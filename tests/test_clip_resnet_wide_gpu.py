"""The wide ResNet image towers (RN50x4, RN50x16, RN50x64) on the GPU: the 128 x 64 GEMM tiles for N % 128 == 64, the stem and
token kernels at the new widths and grids, the whole towers against the float64 restatement of tests/clip_resnet_oracle.py, the
handle's bookkeeping, the 640-wide text tower and the sampler at 288, 384 and 448.

Kernel bars follow tests/test_clip_resnet_gpu.py: one bf16 rounding of the output, 6e-3 norm-wise; fp32-only paths 1e-5.

Whole towers. Every stored activation and weight is bf16, and the attention pool amplifies what reaches it, as for RN50 / RN101
(tests/test_clip_resnet_gpu.py derives those bars from the pool's sensitivity). How much it amplifies depends on how large the
pool's tokens are, and with synthetic_resnet_state_dict's default residual-branch scale of 0.25 they keep growing past RN101's
33 blocks: in float64, one bf16-sized relative perturbation (rms 2^-9 / sqrt 3) of the pool's input moves the crop gradient by
1.2 % at RN50x4 (26 blocks) but by 23 % at RN50x16 (40 blocks) and 250 % at RN50x64 (64 blocks), whose softmax is then nearly
one-hot and no comparison can bound its gradient. So these towers' weights scale the branch by 0.25, 0.18 and 0.15 (BRANCH),
which keeps the pool's input at rms 4.2, 4.2 and 5.4 (RN50 2.6, RN101 7.1) and the gradient's sensitivity at 1.2, 1.4 and
1.7 % (RN50 0.8 %, RN101 2.6 %), its mean largest attention weight per head at 0.34, 0.28 and 0.44 (measured on the CPU, one
crop at the model's resolution). Bars, fixed per tower like RN50's: embeddings 2e-2 per sample (the project's bf16 bar);
crop gradient against a float64 backward through the CUDA forward's own ReLU selects and last block output 5e-2 (RN50's);
against plain float64 3e-1, RN50's 2.5e-1 widened for the ReLU selects that bf16 activations flip in 26 to 64 blocks rather
than 16. Measured on an H100 (700 W), two crops per case:
  - RN50x4 at 287, 288, 296, 318: embeddings 0.69-0.88 %, gradient 2.5-3.2 % (plain 19.9-21.1 %);
  - RN50x16 at 384, 392: embeddings 0.61-0.70 %, gradient 2.9 % (plain 20.6-20.8 %);
  - RN50x64 at 448: embeddings 0.99 %, gradient 3.1 % (plain 22.0 %).
"""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from aphantasia_b200 import _lib, clip
import clip_resnet_oracle as O

pytestmark = pytest.mark.gpu


def _st():
    return torch.cuda.current_stream().cuda_stream


def _rel(a, b):
    a = torch.as_tensor(a).double().cpu() if not torch.is_tensor(a) else a.detach().double().cpu()
    b = torch.as_tensor(b).double().cpu() if not torch.is_tensor(b) else b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def _nchw(x):
    return x.permute(0, 3, 1, 2).double()


def _old_variant(M, N, K, sms):
    """The kernel variant launch_gemm picked for (M, N, K) before N % 128 == 64 ran 128 x 64 tiles: 0 small-problem, 1 large."""
    m_tiles = (M + 127) // 128
    if N == 64:
        return 0
    if m_tiles * (N // 128) >= 2 * sms and K <= 1024:
        return 1
    return 1 if N % 256 == 0 and m_tiles * (N // 256) >= sms else 0


def _epilogue_cases(M, N, K, seed):
    torch.manual_seed(seed)
    A = torch.randn(M, K, device='cuda').bfloat16()
    B = (torch.randn(N, K, device='cuda') * K ** -0.5).bfloat16()
    bias = torch.randn(N, device='cuda') * 0.3
    res = torch.randn(M, N, device='cuda').bfloat16()
    mask = torch.randn(M, N, device='cuda').bfloat16()
    acc = A.double() @ B.double().t()
    ptr = lambda t: None if t is None else t.data_ptr()
    L = _lib.lib()

    def rn(b, r, m, relu):
        return lambda out: L.aph_gemm_rn_epi_test(A.data_ptr(), B.data_ptr(), M, N, K, ptr(b), ptr(r), ptr(m), relu, out.data_ptr(), _st())

    def plain(b):
        return lambda out: L.aph_gemm_epi_test(A.data_ptr(), B.data_ptr(), M, N, K, ptr(b), None, None, 0, None, out.data_ptr(), None, 0, 0,
                                               _st())
    zero = torch.zeros_like(acc)
    return [(1, plain(None), acc, None), (2, plain(bias), acc + bias.double(), None),
            (7, rn(bias, None, None, 1), F.relu(acc + bias.double()), None),
            (8, rn(bias, res, None, 1), F.relu(acc + bias.double() + res.double()), None),
            (9, rn(None, None, mask, 0), torch.where(mask.double() > 0, acc, zero), mask),
            (10, rn(None, res, mask, 0), torch.where(mask.double() > 0, acc + res.double(), zero), mask)]


@pytest.mark.parametrize('N', [192, 320, 576])
def test_gemm_narrow_tiles_at_n_mod_128_eq_64(N):
    """The bf16, bias-bf16 and four ResNet epilogues at N % 128 == 64 against float64 (6e-3; selects exact). M is large enough
    that a 128-wide schedule would be the ping-pong one, and not a multiple of the tile: the variant counter proves the 128 x 64
    small-problem tile ran."""
    M, K = 40000 - 37, 256
    L = _lib.lib()
    for kind, launch, want, mask in _epilogue_cases(M, N, K, N):
        before = [L.aph_gemm_variant_launches(v, kind) for v in (0, 1)]
        out = torch.full((M, N), float('nan'), device='cuda', dtype=torch.bfloat16)
        _lib.check(launch(out), 'gemm kind %d' % kind)
        torch.cuda.synchronize()
        assert [L.aph_gemm_variant_launches(v, kind) for v in (0, 1)] == [before[0] + 1, before[1]], kind
        assert torch.isfinite(out).all() and _rel(out, want) < 6e-3, (kind, _rel(out, want))
        if mask is not None:
            assert (out.double()[mask.double() <= 0] == 0).all()


@pytest.mark.parametrize('M, N, K', [(1000, 64, 256), (40000, 64, 256), (1000, 128, 256), (1000, 2048, 256), (40000, 256, 256),
                                     (40000, 256, 2048), (1000, 512, 2048), (2176, 2048, 2048), (20000, 1024, 512)])
def test_gemm_existing_shapes_keep_their_variant(M, N, K):
    """Every (N, K) the towers launched before (N = 64 or a multiple of 128) runs the variant the previous rule chose."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    want_v = _old_variant(M, N, K, sms)
    L = _lib.lib()
    for kind, launch, want, _ in _epilogue_cases(M, N, K, M + N + K)[2:4]:
        before = L.aph_gemm_variant_launches(want_v, kind)
        other = L.aph_gemm_variant_launches(1 - want_v, kind)
        out = torch.empty((M, N), device='cuda', dtype=torch.bfloat16)
        _lib.check(launch(out), 'gemm')
        torch.cuda.synchronize()
        assert L.aph_gemm_variant_launches(want_v, kind) == before + 1 and L.aph_gemm_variant_launches(1 - want_v, kind) == other
        assert _rel(out, want) < 6e-3


@pytest.mark.parametrize('cout, side', [(40, 288), (48, 384), (56, 351), (64, 448), (40, 318)])
def test_stem_conv_at_every_width(cout, side):
    torch.manual_seed(cout + side)
    N, h = 2, (side - 1) // 2 + 1
    img = torch.randn(N, 3, side, side, device='cuda')
    w = torch.randn(cout, 3, 3, 3, device='cuda') * 0.3
    b = torch.randn(cout, device='cuda') * 0.1
    out = torch.full((N, h, h, 64), float('nan'), device='cuda', dtype=torch.bfloat16)
    L = _lib.lib()
    _lib.check(L.aph_rn_stem_test(1, img.data_ptr(), w.data_ptr(), b.data_ptr(), out.data_ptr(), N, side, _st(), cout), 'stem fwd')
    ref = F.relu(F.conv2d(img.double(), w.double(), b.double(), stride=2, padding=1))
    torch.cuda.synchronize()
    assert torch.isfinite(out).all() and (out[..., cout:] == 0).all()
    assert _rel(_nchw(out[..., :cout]), ref) < 6e-3
    dz = torch.randn(N, h, h, 64, device='cuda').bfloat16()
    g = torch.full((N, 3, side, side), float('nan'), device='cuda')
    _lib.check(L.aph_rn_stem_test(0, dz.data_ptr(), w.data_ptr(), None, g.data_ptr(), N, side, _st(), cout), 'stem bwd')
    gref = torch.nn.grad.conv2d_input((N, 3, side, side), w.double(), _nchw(dz[..., :cout]), stride=2, padding=1)
    torch.cuda.synchronize()
    assert torch.isfinite(g).all() and _rel(g, gref) < 1e-5
    assert L.aph_rn_stem_test(1, img.data_ptr(), w.data_ptr(), b.data_ptr(), out.data_ptr(), N, side, _st(), 36) != 0


@pytest.mark.parametrize('grid, C', [(9, 2560), (12, 3072), (14, 4096)])
def test_tokens_at_every_grid(grid, C):
    torch.manual_seed(grid)
    S, P = 2, grid * grid
    x = torch.relu(torch.randn(S, P, C, device='cuda')).bfloat16()
    pos = torch.randn(P + 1, C, device='cuda') * 0.1
    tok = torch.full((S, P + 1, C), float('nan'), device='cuda', dtype=torch.bfloat16)
    L = _lib.lib()
    _lib.check(L.aph_rn_tokens_test(1, x.data_ptr(), pos.data_ptr(), tok.data_ptr(), S, C, _st(), grid), 'tokens fwd')
    xd = x.double()
    want = torch.cat([xd.mean(1, keepdim=True), xd], 1) + pos.double()
    torch.cuda.synchronize()
    assert torch.isfinite(tok).all() and _rel(tok, want) < 6e-3
    dtok = torch.randn(S, P + 1, C, device='cuda').bfloat16()
    dz = torch.full((S, P, C), float('nan'), device='cuda', dtype=torch.bfloat16)
    _lib.check(L.aph_rn_tokens_test(0, dtok.data_ptr(), x.data_ptr(), dz.data_ptr(), S, C, _st(), grid), 'tokens bwd')
    d = dtok.double()
    want = torch.where(xd > 0, d[:, 1:] + d[:, :1] / P, torch.zeros_like(xd))
    torch.cuda.synchronize()
    assert torch.isfinite(dz).all() and _rel(dz, want) < 6e-3 and (dz.double()[xd <= 0] == 0).all()


_SD = {}
# The synthetic weights' residual-branch scale per tower (synthetic_resnet_state_dict's branch_scale; module docstring).
BRANCH = {'RN50x4': 0.25, 'RN50x16': 0.18, 'RN50x64': 0.15}


def _state_dict(name, seed=0):
    if (name, seed) not in _SD:
        _SD.clear()                                  # one model's weights at a time (RN50x64: 420 M parameters)
        _SD[(name, seed)] = clip.synthetic_resnet_state_dict(seed=seed, branch_scale=BRANCH[name], **clip._MODELS[name])
    return _SD[(name, seed)]


def _device_view(ptr, n):
    class _Mem:
        __cuda_array_interface__ = {'shape': (n,), 'typestr': '<i2', 'data': (ptr, False), 'version': 3}
    return torch.as_tensor(_Mem(), device='cuda')


def _selects(vis, S):
    """The CUDA forward's ReLU selects at the real channel counts (NCHW, clip_resnet_oracle's order) and its last block's output."""
    w = vis.width
    real = [w // 2, w // 2, w]
    run = [64, 64, clip.pad64(w)]
    for i, n in enumerate(vis.layers):
        p = w << i
        real += [p, p, 4 * p] * n
        run += [clip.pad64(p), clip.pad64(p), 4 * p] * n
    out = []
    for k, (c, cs) in enumerate(zip(real, run)):
        ptr, numel = C.c_void_p(), C.c_int64()
        _lib.check(_lib.lib().aph_rn_saved_test(vis.handle, k, C.byref(ptr), C.byref(numel)), 'aph_rn_saved_test')
        hw = round((numel.value // (S * cs)) ** 0.5)
        assert S * hw * hw * cs == numel.value, (k, numel.value, cs)
        t = _device_view(ptr.value, numel.value).view(torch.bfloat16).view(S, hw, hw, cs)
        assert (t[..., c:] == 0).all(), k                    # the padded channels stay exactly zero
        out.append((t[..., :c] > 0).permute(0, 3, 1, 2).contiguous())
    return out, t.permute(0, 3, 1, 2).double()


# (embeddings per sample, crop gradient against the CUDA-select float64 backward, crop gradient against plain float64)
BARS = {'RN50x4': (2e-2, 5e-2, 3e-1), 'RN50x16': (2e-2, 5e-2, 3e-1), 'RN50x64': (2e-2, 5e-2, 3e-1)}


@pytest.mark.parametrize('name, side', [('RN50x4', 288), ('RN50x4', 287), ('RN50x4', 296), ('RN50x4', 318), ('RN50x16', 384),
                                        ('RN50x16', 392), ('RN50x64', 448)])
def test_wide_tower_against_float64(name, side):
    """Embeddings per sample and the crop gradient against float64, to the fixed bars of BARS (derivation and measured values:
    module docstring)."""
    torch.manual_seed(side)
    sd = _state_dict(name)
    vis = clip.ModifiedResNet(sd)
    S = 2
    x = torch.randn(S, 3, side, side, device='cuda')
    g = torch.randn(S, vis.output_dim, device='cuda')
    xr = x.clone().requires_grad_(True)
    e = vis(xr)
    (gx,) = torch.autograd.grad(e, xr, g)
    e, gx = e.detach(), gx.detach()
    sel, y4 = _selects(vis, S)
    osd = {k[len('visual.'):]: v.cuda() for k, v in sd.items() if k.startswith('visual.')}
    er, gr = O.forward_backward(osd, x, g)
    _, gs = O.forward_backward(osd, x, g, selects=sel, pool_input=y4)
    del osd
    errs = [_rel(e[i], er[i]) for i in range(S)]
    print('%s side %d: embedding errors %s, gradient error %.4f (CUDA selects), %.4f (plain)'
          % (name, side, ['%.4f' % v for v in errs], _rel(gx, gs), _rel(gx, gr)))
    ebar, sbar, gbar = BARS[name]
    assert torch.isfinite(e).all() and max(errs) < ebar
    assert torch.isfinite(gx).all() and _rel(gx, gs) < sbar and _rel(gx, gr) < gbar
    vis.close()


def _rn_bytes(layers, width, res, S, O):
    """aph_rn_bytes from the formula of include/aphb200.h."""
    pad = clip.pad64
    C1, SC, D, T = width // 2, pad(width), 32 * width, (res // 32) ** 2 + 1
    h1 = (res + 29) // 2 + 1
    h0 = h1 // 2
    w = 4 * (27 * C1 + C1 + 64 + SC) + 2 * 2 * 9 * 64 * (64 + SC)
    act = S * (2 * h1 * h1 * 64 + h1 * h1 * SC + h0 * h0 * SC)
    emax = h1 * h1 * SC
    hin, cin = h0, SC
    for i, n in enumerate(layers):
        P, E = pad(width << i), 4 * (width << i)
        for j in range(n):
            stride = 2 if (i > 0 and j == 0) else 1
            down = stride > 1 or cin != E
            hout = hin // stride
            w += 2 * 2 * (P * cin + E * P + (E * cin if down else 0)) + 2 * 2 * 9 * P * P + 4 * (2 * P + E + (E if down else 0))
            act += S * (2 * hin * hin * P + hout * hout * E)
            emax = max(emax, hin * hin * max(cin, P), hout * hout * E)
            hin, cin = hout, E
    w += 4 * T * D + 2 * 2 * 3 * D * D + 4 * 3 * D + 2 * 2 * O * D + 4 * O
    return w + 2 * (act + 6 * S * emax + 10 * T * S * D + S * O) + 4 * S * O


def test_wide_handle_bookkeeping_and_repeatability():
    """RN50x4: aph_rn_bytes follows the header formula and aph_device_bytes returns to its start after close; one handle serves
    batch sizes up to its max_batch (per-sample embeddings as from a batch of one); two backward calls are bit-identical; an
    --enforce-style pair of grad-tracked forwards before one backward gives the gradients of separate calls."""
    torch.cuda.synchronize()
    start = _lib.lib().aph_device_bytes()
    m = clip._MODELS['RN50x4']
    vis = clip.ModifiedResNet(_state_dict('RN50x4', seed=2))
    vis._ensure(4)
    assert _lib.lib().aph_rn_bytes(vis.handle) == _rn_bytes(m['layers'], 80, 288, 4, 640)
    epoch = vis._handle_epoch
    torch.manual_seed(0)
    a = torch.randn(4, 3, 296, 296, device='cuda')
    b = torch.randn(4, 3, 296, 296, device='cuda')
    g = torch.randn(4, 640, device='cuda')
    with torch.no_grad():
        full = vis(a)
        for n in (1, 3):
            assert _rel(vis(a[:n]), full[:n]) < 5e-3
    assert vis._handle_epoch == epoch
    sep = []
    for x in (a, b):
        xr = x.clone().requires_grad_(True)
        sep.append(torch.autograd.grad(vis(xr), xr, g)[0])
    xr = a.clone().requires_grad_(True)
    again = torch.autograd.grad(vis(xr), xr, g)[0]
    assert torch.equal(again, sep[0])
    xa, xb = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
    ea, eb = vis(xa), vis(xb)
    ga, gb = torch.autograd.grad((ea * g).sum() + (eb * g).sum(), (xa, xb))
    assert torch.equal(ga, sep[0]) and torch.equal(gb, sep[1]) and vis.recomputes >= 1
    with pytest.raises(ValueError, match='287 <= side <= 318'):
        vis(torch.randn(1, 3, 286, 286, device='cuda'))
    vis.close()
    del vis
    torch.cuda.synchronize()
    assert _lib.lib().aph_device_bytes() == start


def test_clip_load_rn50x4_checkpoint(tmp_path, monkeypatch):
    """clip.load('RN50x4') from an fp16 OpenAI-layout checkpoint with RN50x4's 640-wide text tower: the image tower against
    float64 of the same fp16 weights (2e-2, the embedding bar of the module docstring) and the text tower against the restatement (2e-2, as
    test_text_tower_gpu.py)."""
    import text_oracle as TO
    sd = _state_dict('RN50x4', seed=7)
    text = clip.synthetic_text_state_dict(width=640, layers=2, heads=10, out_dim=640, vocab=1000, seed=7)
    path = tmp_path / 'RN50x4.pt'
    torch.save({k: (v.half() if v.is_floating_point() else v) for k, v in {**sd, **text}.items()}, str(path))
    monkeypatch.setenv('APH_CLIP_WEIGHTS_RN50X4', str(path))
    model, _ = clip.load('RN50x4')
    assert model.visual.input_resolution == 288 and model.embed_dim == 640 and model.transformer.width == 640
    x = torch.randn(2, 3, 288, 288, device='cuda')
    e = model.encode_image(x)
    half = {k[len('visual.'):]: (v.half().double() if v.is_floating_point() else v).cuda() for k, v in sd.items() if k.startswith('visual.')}
    er = O.forward(half, x.double())
    assert max(_rel(e[i], er[i]) for i in range(2)) < 2e-2
    ref = TO.build_text({k: v.half().float() for k, v in text.items()})
    toks = torch.randint(1, 999, (3, 77))
    for i, p in enumerate((76, 20, 41)):              # one end-of-text (the largest id) per prompt
        toks[i, p] = 999
    got = model.encode_text(toks.cuda())
    with torch.no_grad():
        want = ref(toks)
    assert got.shape == (3, 640) and _rel(got, want) < 2e-2
    model.visual.close()


# ---------------------------------------------------------------------------------------------------------- the sampler
@pytest.mark.parametrize('size', [288, 384, 448])
@pytest.mark.parametrize('kind', [0, 1, 2, 3, 4])
def test_sampler_at_wide_sizes(size, kind):
    """slice_imgs at the wide towers' crop sides, every transform kind, against the CPU oracle (oracle/restate.py,
    tests/kornia_oracle.py): the canvas gradient to 1e-4 and the values to 1e-5 x size / 224, the existing sampler tests' bars at
    224. The values' bar grows with the side because the fp32 rounding of the warp stages' source coordinates grows with the
    coordinates themselves: transforms_fast measured 1.2e-5 at 384 and 1.6e-5 at 448 on an H100, the other kinds below 1e-5."""
    import kornia_oracle as KO
    from oracle import restate as R
    from aphantasia_b200 import _rng, transforms
    from aphantasia_b200.utils import slice_imgs
    tf = [None, transforms.normalize(), transforms.transforms_fast, transforms.transforms_custom, transforms.transforms_elastic][kind]
    hw, S = (520, 700), 6
    torch.manual_seed(11); np.random.seed(11)
    canvas = torch.rand(1, 3, *hw)
    cc = canvas.cuda().requires_grad_(True)
    torch.manual_seed(5); np.random.seed(5)
    out = slice_imgs([cc], S, size, tf, 'uniform', 0.4)[0]
    assert out.shape == (S, 3, _rng.out_side(size, kind), _rng.out_side(size, kind))
    torch.manual_seed(5); np.random.seed(5)
    tabs, frame = _rng.draw_crop_table_py(S, hw, size, kind, 'uniform', 0.4)
    co = canvas.clone().requires_grad_(True)
    ref = (KO.sample_crops(co, tabs[0], size, kind, frame) if kind >= 3 else R.sample_crops(co, tabs[0], size, kind))
    torch.manual_seed(6)
    cot = torch.randn(ref.shape)
    (out * cot.cuda()).sum().backward()
    (ref * cot).sum().backward()
    assert _rel(out, ref) < 1e-5 * size / 224, _rel(out, ref)
    assert _rel(cc.grad, co.grad) < 1e-4, _rel(cc.grad, co.grad)
