"""The ResNet image towers (RN50, RN101) on the GPU: each new kernel and epilogue against float64 of the same bf16 operands, the
whole tower against the float64 restatement of tests/clip_resnet_oracle.py, the handle's bookkeeping and clip.load.

Rounding model. A kernel reads bf16 operands exactly and accumulates in fp32; its bf16 output rounds once (2^-9 relative per
element, at most 2e-3 norm-wise), so kernel bars are 6e-3 norm-wise as in test_lpips_gpu.py; fp32-only paths (the stem's
backward from a bf16 dz) are held to 1e-5.

The whole tower rounds every stored activation (about 60 for RN50, 110 for RN101) and every weight to bf16. Its attention pool
amplifies what reaches it: in float64, one bf16-sized relative perturbation (rms 2^-9 / sqrt 3) of the attention-pool tokens moves
the embeddings by 0.04 % (RN50) and 0.21 % (RN101), and the crop gradient by 0.9 % and 3.1 %, for these synthetic weights (33
blocks leave RN101's tokens larger and its attention sharper). Measured on an H100 (three crops per case):
  - embeddings against float64: RN50 0.46-0.49 % per sample at sides 223, 224, 232 and 254, within the project's bf16 bar of
    2e-2; RN101 1.3-2.5 %, five times RN50's as the sensitivity above predicts, held to 3e-2;
  - crop gradient against a float64 backward through the CUDA forward's own ReLU selects, its attention pool reading the CUDA
    forward's last block output (clip_resnet_oracle: `selects`, `pool_input`). Given the selects the trunk is linear, so what is
    left is the rounding of the stored gradients and weights plus the pool's own bf16 roundings (tokens, q/k/v, attention output:
    about sqrt 3 times the single-rounding figure above, 1.6 % for RN50 and 5.4 % for RN101). Measured 2.1-2.2 % (RN50) and
    6.9-7.7 % (RN101); bars 5e-2 and 1e-1;
  - crop gradient against plain float64: 15-16 % (RN50) and 29-30 % (RN101), the ReLU selects that bf16 activations flip; bars
    2.5e-1 and 4e-1, a bound on the bf16 design as LPIPS' plain bar is.
"""
import os

import pytest
import torch
import torch.nn.functional as F

from aphantasia_b200 import _lib, clip
import clip_resnet_oracle as O

pytestmark = pytest.mark.gpu


def _st():
    return torch.cuda.current_stream().cuda_stream


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16)


def _nchw(x):
    return x.permute(0, 3, 1, 2).double()


@pytest.mark.parametrize('side', [224, 232, 223, 254])
def test_stem_conv_fwd_and_crop_gradient(side):
    torch.manual_seed(side)
    N, h = 2, (side - 1) // 2 + 1
    img = torch.randn(N, 3, side, side, device='cuda')
    w = torch.randn(32, 3, 3, 3, device='cuda') * 0.3
    b = torch.randn(32, device='cuda') * 0.1
    out = torch.full((N, h, h, 64), float('nan'), device='cuda', dtype=torch.bfloat16)
    _lib.check(_lib.lib().aph_rn_stem_test(1, img.data_ptr(), w.data_ptr(), b.data_ptr(), out.data_ptr(), N, side, _st()), 'stem fwd')
    ref = F.relu(F.conv2d(img.double(), w.double(), b.double(), stride=2, padding=1))
    torch.cuda.synchronize()
    assert torch.isfinite(out).all() and (out[..., 32:] == 0).all()
    assert _rel(_nchw(out[..., :32]), ref) < 6e-3
    dz = torch.randn(N, h, h, 64, device='cuda').bfloat16()
    g = torch.full((N, 3, side, side), float('nan'), device='cuda')
    _lib.check(_lib.lib().aph_rn_stem_test(0, dz.data_ptr(), w.data_ptr(), None, g.data_ptr(), N, side, _st()), 'stem bwd')
    gref = torch.nn.grad.conv2d_input((N, 3, side, side), w.double(), _nchw(dz[..., :32]), stride=2, padding=1)
    torch.cuda.synchronize()
    assert torch.isfinite(g).all() and _rel(g, gref) < 1e-5


@pytest.mark.parametrize('h', [116, 112, 63, 29, 14])
def test_average_pool_and_adjoint(h):
    """Forward and adjoint (with and without the ReLU select), odd sides floor. The forward sums the window's four bf16 values
    in fp32 in (0,0) (0,1) (1,0) (1,1) order, scales by 1/4 and rounds once to nearest; the adjoint scales by 1/4 exactly: both
    exact against an fp32 restatement of that order."""
    torch.manual_seed(h)
    N, C = 2, 64
    x = torch.randn(N, C, h, h, device='cuda').bfloat16()
    xh = _nhwc(x)
    out = torch.full((N, h // 2, h // 2, C), float('nan'), device='cuda', dtype=torch.bfloat16)
    _lib.check(_lib.lib().aph_rn_pool_test(1, xh.data_ptr(), None, out.data_ptr(), N, h, h, C, _st()), 'pool fwd')
    e = 2 * (h // 2)
    xf = xh[:, :e, :e].float()
    want = ((((xf[:, 0::2, 0::2] + xf[:, 0::2, 1::2]) + xf[:, 1::2, 0::2]) + xf[:, 1::2, 1::2]) * 0.25).bfloat16()
    torch.cuda.synchronize()
    assert torch.equal(out, want)
    dy = torch.randn(N, C, h // 2, h // 2, device='cuda').bfloat16()
    dyh = _nhwc(dy)
    xr = x.double().requires_grad_(True)
    (want,) = torch.autograd.grad(F.avg_pool2d(xr, 2), xr, dy.double())
    for m in (None, xh):
        dx = torch.full((N, h, h, C), float('nan'), device='cuda', dtype=torch.bfloat16)
        _lib.check(_lib.lib().aph_rn_pool_test(0, dyh.data_ptr(), None if m is None else m.data_ptr(), dx.data_ptr(), N, h, h, C, _st()),
                   'pool bwd')
        ref = want if m is None else torch.where(x.double() > 0, want, torch.zeros_like(want))
        torch.cuda.synchronize()
        assert torch.equal(_nchw(dx), ref)


@pytest.mark.parametrize('M, N, K, variant', [(1000, 64, 256, 0), (1000, 2048, 256, 0), (2176, 2048, 256, 1), (2176, 2048, 2048, 1)],
                         ids=['128x64', '128x128', 'pingpong', '128x256'])
def test_gemm_resnet_epilogues(M, N, K, variant):
    """The four ResNet epilogue kinds on every schedule the tower's 1x1 GEMMs run: 128 x 64 tiles (N = 64), cooperative 128 x 128,
    ping-pong 128 x 128 (many tiles, short K) and cooperative 128 x 256 (many tiles, long K); M is not a multiple of the tile.
    The kernel-variant counter proves the schedule. Bars 6e-3, the selects exact (masked elements are exactly zero)."""
    torch.manual_seed(N + K)
    A = torch.randn(M, K, device='cuda').bfloat16()
    B = (torch.randn(N, K, device='cuda') * K ** -0.5).bfloat16()
    bias = torch.randn(N, device='cuda') * 0.3
    res = torch.randn(M, N, device='cuda').bfloat16()
    mask = torch.randn(M, N, device='cuda').bfloat16()
    acc = A.double() @ B.double().t()
    count = lambda kind: _lib.lib().aph_gemm_variant_launches(variant, kind)
    cases = [(7, bias, None, None, 1, F.relu(acc + bias.double())),
             (8, bias, res, None, 1, F.relu(acc + bias.double() + res.double())),
             (9, None, None, mask, 0, torch.where(mask.double() > 0, acc, torch.zeros_like(acc))),
             (10, None, res, mask, 0, torch.where(mask.double() > 0, acc + res.double(), torch.zeros_like(acc)))]
    ptr = lambda t: None if t is None else t.data_ptr()
    for kind, b, r, m, relu, want in cases:
        before = count(kind)
        out = torch.full((M, N), float('nan'), device='cuda', dtype=torch.bfloat16)
        _lib.check(_lib.lib().aph_gemm_rn_epi_test(A.data_ptr(), B.data_ptr(), M, N, K, ptr(b), ptr(r), ptr(m), relu, out.data_ptr(), _st()),
                   'rn epi')
        torch.cuda.synchronize()
        assert count(kind) == before + 1, (kind, variant)
        assert torch.isfinite(out).all() and _rel(out, want) < 6e-3, kind
        if m is not None:
            assert (out.double()[mask.double() <= 0] == 0).all()


@pytest.mark.parametrize('h', [112, 116, 56, 58, 28, 29, 14, 7])
def test_conv3x3_at_every_map_size(h):
    """The 3x3 convolution at every map size of sides 224 and 232 (112/116 stem, 56/58, 28/29, 14, 7), forward and masked data
    gradient, with the tower's channel counts for that size: bar 6e-3."""
    c = {112: 64, 116: 64, 56: 64, 58: 64, 28: 128, 29: 128, 14: 256, 7: 512}[h]
    torch.manual_seed(h)
    N = 2
    x = torch.relu(torch.randn(N, c, h, h, device='cuda')).bfloat16()
    wt = torch.randn(c, c, 3, 3, device='cuda') * (2.0 / (9 * c)) ** 0.5
    wb = wt.bfloat16().double()
    bias = torch.randn(c, device='cuda') * 0.1
    out = torch.full((N, h, h, c), float('nan'), device='cuda', dtype=torch.bfloat16)
    xh = _nhwc(x)
    _lib.check(_lib.lib().aph_lpips_conv_test(1, xh.data_ptr(), wt.data_ptr(), bias.data_ptr(), None, out.data_ptr(), N, h, h, c, c, _st()),
               'conv fwd')
    torch.cuda.synchronize()
    assert torch.isfinite(out).all() and _rel(_nchw(out), F.relu(F.conv2d(x.double(), wb, bias.double(), padding=1))) < 6e-3
    dy = torch.randn(N, c, h, h, device='cuda').bfloat16()
    dyh = _nhwc(dy)
    dx = torch.full((N, h, h, c), float('nan'), device='cuda', dtype=torch.bfloat16)
    _lib.check(_lib.lib().aph_lpips_conv_test(0, dyh.data_ptr(), wt.data_ptr(), None, xh.data_ptr(), dx.data_ptr(), N, h, h, c, c, _st()),
               'conv bwd')
    want = torch.nn.grad.conv2d_input((N, c, h, h), wb, dy.double(), padding=1)
    want = torch.where(x.double() > 0, want, torch.zeros_like(want))
    torch.cuda.synchronize()
    assert torch.isfinite(dx).all() and _rel(_nchw(dx), want) < 6e-3


def test_tokens_and_adjoint():
    """Token formation (mean of 49 rows in fp32, + positional embedding, one rounding: 6e-3) and its adjoint with the select
    (fp32 sum, one rounding: 6e-3; masked elements exactly zero)."""
    torch.manual_seed(5)
    S, C = 3, 2048
    x = torch.relu(torch.randn(S, 49, C, device='cuda')).bfloat16()
    pos = torch.randn(50, C, device='cuda') * 0.1
    tok = torch.full((S, 50, C), float('nan'), device='cuda', dtype=torch.bfloat16)
    _lib.check(_lib.lib().aph_rn_tokens_test(1, x.data_ptr(), pos.data_ptr(), tok.data_ptr(), S, C, _st()), 'tokens fwd')
    xd = x.double()
    want = torch.cat([xd.mean(1, keepdim=True), xd], 1) + pos.double()
    torch.cuda.synchronize()
    assert torch.isfinite(tok).all() and _rel(tok, want) < 6e-3
    dtok = torch.randn(S, 50, C, device='cuda').bfloat16()
    dz = torch.full((S, 49, C), float('nan'), device='cuda', dtype=torch.bfloat16)
    _lib.check(_lib.lib().aph_rn_tokens_test(0, dtok.data_ptr(), x.data_ptr(), dz.data_ptr(), S, C, _st()), 'tokens bwd')
    d = dtok.double()
    want = torch.where(xd > 0, d[:, 1:] + d[:, :1] / 49, torch.zeros_like(xd))
    torch.cuda.synchronize()
    assert torch.isfinite(dz).all() and _rel(dz, want) < 6e-3 and (dz.double()[xd <= 0] == 0).all()


def _tower(name, seed=0):
    sd = clip.synthetic_resnet_state_dict(seed=seed, **clip._MODELS[name])
    return sd, clip.ModifiedResNet(sd)


def _selects(vis, S):
    """The CUDA forward's ReLU selects (output > 0), NCHW, in the order clip_resnet_oracle.forward applies its ReLUs, and its last
    block's output (NCHW float64)."""
    import ctypes as C
    chans = [32, 32, 64]
    for i, n in enumerate(vis.layers):
        chans += [64 << i, 64 << i, 256 << i] * n
    out = []
    for k, c in enumerate(chans):
        ptr, numel = C.c_void_p(), C.c_int64()
        _lib.check(_lib.lib().aph_rn_saved_test(vis.handle, k, C.byref(ptr), C.byref(numel)), 'aph_rn_saved_test')
        cs = 64 if k < 3 else c                                # the stem's maps carry 64 channels, 32-63 zero
        hw = round((numel.value // (S * cs)) ** 0.5)
        assert S * hw * hw * cs == numel.value
        t = _device_view(ptr.value, numel.value).view(torch.bfloat16).view(S, hw, hw, cs)
        out.append((t[..., :c] > 0).permute(0, 3, 1, 2).contiguous())
    return out, t.permute(0, 3, 1, 2).double()                # and the last block's output


def _device_view(ptr, n):
    """A torch view of n 16-bit elements of device memory at ptr (through the CUDA array interface; no copy)."""
    class _Mem:
        __cuda_array_interface__ = {'shape': (n,), 'typestr': '<i2', 'data': (ptr, False), 'version': 3}
    return torch.as_tensor(_Mem(), device='cuda')


@pytest.mark.parametrize('name, side', [('RN50', 224), ('RN50', 232), ('RN101', 224), ('RN101', 232), ('RN50', 223), ('RN50', 254)])
def test_tower_against_float64(name, side):
    """Embeddings per sample against float64; the crop gradient against a float64 backward through the CUDA forward's own ReLU
    selects, and against plain float64 (bars, their derivation and measured values: module docstring)."""
    torch.manual_seed(side)
    sd, vis = _tower(name)
    S = 3
    x = torch.randn(S, 3, side, side, device='cuda')
    g = torch.randn(S, vis.output_dim, device='cuda')
    xr = x.clone().requires_grad_(True)
    e = vis(xr)
    (gx,) = torch.autograd.grad(e, xr, g)
    e, gx = e.detach(), gx.detach()
    sel, y4 = _selects(vis, S)                                 # the backward leaves the saved forward in place
    osd = {k[len('visual.'):]: v.cuda() for k, v in sd.items() if k.startswith('visual.')}
    er, gr = O.forward_backward(osd, x, g)
    _, gs = O.forward_backward(osd, x, g, selects=sel, pool_input=y4)
    errs = [_rel(e[i], er[i]) for i in range(S)]
    print('%s side %d: embedding errors %s, gradient error %.4f (CUDA selects), %.4f (plain)'
          % (name, side, ['%.4f' % v for v in errs], _rel(gx, gs), _rel(gx, gr)))
    ebar, sbar, gbar = (2e-2, 5e-2, 2.5e-1) if name == 'RN50' else (3e-2, 1e-1, 4e-1)
    assert torch.isfinite(e).all() and max(errs) < ebar
    assert torch.isfinite(gx).all() and _rel(gx, gs) < sbar and _rel(gx, gr) < gbar
    vis.close()


def _rn_bytes(layers, S, O):
    """aph_rn_bytes from the formula of include/aphb200.h."""
    D, h1 = 2048, 127
    h0 = h1 // 2
    w = 4 * (864 + 32 + 2 * 64) + 2 * 2 * 2 * 9 * 64 * 64
    act = S * (3 * h1 * h1 * 64 + h0 * h0 * 64)
    emax = h1 * h1 * 64
    hin, cin = h0, 64
    for i, n in enumerate(layers):
        P = 64 << i
        E = 4 * P
        for j in range(n):
            stride = 2 if (i > 0 and j == 0) else 1
            down = stride > 1 or cin != E
            hout = hin // stride
            w += 2 * 2 * (P * cin + E * P + (E * cin if down else 0)) + 2 * 2 * 9 * P * P + 4 * (2 * P + E + (E if down else 0))
            act += S * (2 * hin * hin * P + hout * hout * E)
            emax = max(emax, hin * hin * max(cin, P), hout * hout * E)
            hin, cin = hout, E
    w += 4 * 50 * D + 2 * 2 * 3 * D * D + 4 * 3 * D + 2 * 2 * O * D + 4 * O
    return w + 2 * (act + 6 * S * emax + 10 * 50 * S * D + S * O) + 4 * S * O


def test_handle_bookkeeping_and_repeatability():
    """aph_rn_bytes follows the header formula and aph_device_bytes returns to its start after close; two backward calls are
    bit-identical; an --enforce-style pair of grad-tracked forwards before one backward gives the gradients of separate calls."""
    torch.cuda.synchronize()
    start = _lib.lib().aph_device_bytes()
    sd, vis = _tower('RN50', seed=2)
    vis._ensure(4)
    assert _lib.lib().aph_rn_bytes(vis.handle) == _rn_bytes((3, 4, 6, 3), 4, 1024)
    torch.manual_seed(0)
    a = torch.randn(4, 3, 232, 232, device='cuda')
    b = torch.randn(4, 3, 232, 232, device='cuda')
    g = torch.randn(4, 1024, device='cuda')
    sep = []
    for x in (a, b):
        xr = x.clone().requires_grad_(True)
        e = vis(xr)
        sep.append(torch.autograd.grad(e, xr, g)[0])
    xr = a.clone().requires_grad_(True)
    e = vis(xr)
    again = torch.autograd.grad(e, xr, g)[0]
    assert torch.equal(again, sep[0])
    xa, xb = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
    ea, eb = vis(xa), vis(xb)                         # the second forward overwrites the first one's activations
    ga, gb = torch.autograd.grad((ea * g).sum() + (eb * g).sum(), (xa, xb))
    assert torch.equal(ga, sep[0]) and torch.equal(gb, sep[1]) and vis.recomputes >= 1
    vis.close()
    del vis
    torch.cuda.synchronize()
    assert _lib.lib().aph_device_bytes() == start


@pytest.mark.parametrize('text', [False, True])
def test_clip_load_resnet_weights(tmp_path, monkeypatch, text):
    """clip.load('RN50') from APH_CLIP_WEIGHTS_RN50: an fp16 state dict holding num_batches_tracked as OpenAI's archives do, with
    and without a text tower of out_dim 1024; the tower computes what the synthetic fp32 weights give to the bf16 bar."""
    sd = clip.synthetic_resnet_state_dict(seed=7, **clip._MODELS['RN50'])
    full = dict(sd)
    if text:
        full.update(clip.synthetic_text_state_dict(layers=2, out_dim=1024, seed=7))
    path = tmp_path / 'RN50.pt'
    torch.save({k: (v.half() if v.is_floating_point() else v) for k, v in full.items()}, str(path))
    monkeypatch.setenv('APH_CLIP_WEIGHTS_RN50', str(path))
    model, _ = clip.load('RN50')
    assert isinstance(model.visual, clip.ModifiedResNet) and model.visual.input_resolution == 224 and model.embed_dim == 1024
    assert (model.transformer is not None) == text
    x = torch.randn(2, 3, 224, 224, device='cuda')
    e = model.encode_image(x)
    half = {k[len('visual.'):]: (v.half().double() if v.is_floating_point() else v).cuda() for k, v in sd.items() if k.startswith('visual.')}
    er = O.forward(half, x.double())
    assert max(_rel(e[i], er[i]) for i in range(2)) < 2e-2
    if text:
        t = model.encode_text(clip.tokenize(['a red square']).cuda())
        assert t.shape == (1, 1024) and torch.isfinite(t).all()
    model.visual.close()
