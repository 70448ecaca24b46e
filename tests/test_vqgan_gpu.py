"""The VQGAN decoder on the GPU (csrc/vqgan.cu) against float64: each new kernel on its own, then the whole decoder of both of the
notebook's configs (forward and d loss / d z, tests/vqgan_oracle.py), the handle's re-pack, generation and repeat rules, and the
notebook's Generate-cell step restated with synthetic weights.

Bars. Every kernel test compares with float64 computed from the same bf16 inputs, so its error is the kernel's own: the bf16
rounding of its output (2^-9 relative) plus fp32 accumulation, held to 1e-2 relative (GroupNorm, convolutions, conversions,
conv_out) and 2e-2 for the attention, whose P and dS are stored in bf16 before the second GEMM. The whole decoder keeps its
activations in bf16 through about 30 layers. Measured on an NVIDIA H100 80GB HBM3 (700 W) against the float64 decoder with
synthetic_decoder_state_dict weights: forward 0.85-1.6 % relative (L2), d loss / d z 1.3-2.7 %, over both configs and every latent
here (the 1 x 1 latent is the worst). The bars are 3e-2 for the forward and 5e-2 for d z, about twice the largest measured error.
The notebook step's d loss / d lats, through the ViT-B/32 crop encoder as well, measured 2.0 % and is held to 6e-2.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import vqgan_oracle as VO
from oracle import restate as R

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def L():
    from aphantasia_b200 import _lib
    assert torch.cuda.is_available()
    return _lib


def _rel(a, b):
    a, b = a.detach().cpu().double(), b.detach().cpu().double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _st():
    return torch.cuda.current_stream().cuda_stream


def _bf(t):
    return t.to(torch.bfloat16).cuda().contiguous()


def _nhwc(t):      # [N, C, H, W] -> [N, H, W, C]
    return t.permute(0, 2, 3, 1).contiguous()


def _nchw(t):
    return t.permute(0, 3, 1, 2).contiguous()


# ---- GroupNorm ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('C', [128, 256, 512])
@pytest.mark.parametrize('H,W', [(1, 1), (7, 13), (37, 61)])
@pytest.mark.parametrize('swish', [0, 1])
def test_groupnorm_fwd_bwd_vs_float64(L, C, H, W, swish):
    g = torch.Generator().manual_seed(C + H * W + swish)
    N = 2
    x = _bf(torch.randn(N, H, W, C, generator=g) * 1.5 + 0.7)
    gamma = (1 + 0.3 * torch.randn(C, generator=g)).cuda()
    beta = (0.3 * torch.randn(C, generator=g)).cuda()
    dout = _bf(torch.randn(N, H, W, C, generator=g))
    resid = _bf(torch.randn(N, H, W, C, generator=g))
    out = torch.empty_like(x)
    stats = torch.empty(N, 32, 2, device='cuda')
    L.check(L.lib().aph_vqgan_gn_test(1, x.data_ptr(), None, gamma.data_ptr(), beta.data_ptr(), swish, None, stats.data_ptr(),
                                      out.data_ptr(), N, H * W, C, _st()), 'gn fwd')
    dx = torch.empty_like(x)
    L.check(L.lib().aph_vqgan_gn_test(0, x.data_ptr(), dout.data_ptr(), gamma.data_ptr(), beta.data_ptr(), swish, resid.data_ptr(),
                                      stats.data_ptr(), dx.data_ptr(), N, H * W, C, _st()), 'gn bwd')
    xr = _nchw(x.double().cpu()).requires_grad_(True)
    y = F.group_norm(xr, 32, gamma.double().cpu(), beta.double().cpu(), eps=1e-6)
    y = y * torch.sigmoid(y) if swish else y
    y.backward(_nchw(dout.double().cpu()))
    assert _rel(out, _nhwc(y)) < 1e-2
    xs = _nchw(x.double().cpu()).reshape(N, 32, -1)
    assert _rel(stats[..., 0], xs.mean(-1)) < 1e-5
    if H * W > 1:
        assert _rel(stats[..., 1], 1 / (xs.var(-1, unbiased=False) + 1e-6).sqrt()) < 1e-4
    assert _rel(dx, _nhwc(xr.grad) + resid.double().cpu()) < 1e-2


# ---- convolutions with the two new epilogues -------------------------------------------------------------------------------
@pytest.mark.parametrize('Cin,Cout,H,W', [(256, 512, 7, 13), (128, 128, 23, 41), (512, 256, 9, 17)])
@pytest.mark.parametrize('resid', [False, True])
def test_conv_bias_and_bias_resid_epilogues(L, Cin, Cout, H, W, resid):
    g = torch.Generator().manual_seed(Cin + Cout + H)
    N = 2
    x = _bf(torch.randn(N, H, W, Cin, generator=g))
    w = (torch.randn(Cout, Cin, 3, 3, generator=g) * (9 * Cin) ** -0.5).cuda()
    b = (0.1 * torch.randn(Cout, generator=g)).cuda()
    r = _bf(torch.randn(N, H, W, Cout, generator=g)) if resid else None
    out = torch.empty(N, H, W, Cout, device='cuda', dtype=torch.bfloat16)
    L.check(L.lib().aph_vqgan_conv_test(x.data_ptr(), w.data_ptr(), b.data_ptr(), r.data_ptr() if resid else None, out.data_ptr(),
                                        N, H, W, Cin, Cout, _st()), 'conv')
    ref = F.conv2d(_nchw(x.double().cpu()), w.double().cpu(), b.double().cpu(), padding=1)
    if resid:
        ref = ref + _nchw(r.double().cpu())
    assert _rel(out, _nhwc(ref)) < 1e-2


# ---- upsample and its adjoint --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('H,W,C', [(1, 1, 64), (31, 56, 512), (5, 9, 128)])
def test_upsample_and_adjoint(L, H, W, C):
    g = torch.Generator().manual_seed(H * W)
    x = _bf(torch.randn(2, H, W, C, generator=g))
    up = torch.empty(2, 2 * H, 2 * W, C, device='cuda', dtype=torch.bfloat16)
    L.check(L.lib().aph_vqgan_up_test(1, x.data_ptr(), up.data_ptr(), 2, H, W, C, _st()), 'up')
    assert torch.equal(up, x.repeat_interleave(2, 1).repeat_interleave(2, 2))
    dy = _bf(torch.randn(2, 2 * H, 2 * W, C, generator=g))
    dx = torch.empty_like(x)
    L.check(L.lib().aph_vqgan_up_test(0, dy.data_ptr(), dx.data_ptr(), 2, H, W, C, _st()), 'up adj')
    # the adjoint sums each 2 x 2 window in fp32 in (0,0) (0,1) (1,0) (1,1) order and rounds once to nearest: exact
    d = dy.float()
    ref = (((d[:, 0::2, 0::2] + d[:, 0::2, 1::2]) + d[:, 1::2, 0::2]) + d[:, 1::2, 1::2]).bfloat16()
    assert torch.equal(dx, ref)


# ---- attention ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('T', [1, 50, 200, 1736, 6944])
def test_attention_fwd_bwd_vs_float64(L, T):
    """one head of width 512; q / k scaled so that the logits have a standard deviation of about 2 (neither uniform nor one-hot).
    T = 50, 200 and 1736 are not multiples of 128: the padded keys must be masked."""
    C, N = 512, 2 if T <= 200 else 1
    g = torch.Generator().manual_seed(T)
    qkv = torch.randn(N, T, 3 * C, generator=g)
    qkv[..., :2 * C] *= 1.4
    qkv = _bf(qkv)
    dout = _bf(torch.randn(N, T, C, generator=g))
    out = torch.empty(N, T, C, device='cuda', dtype=torch.bfloat16)
    L.check(L.lib().aph_vqgan_attn_test(1, qkv.data_ptr(), None, out.data_ptr(), N, T, C, _st()), 'attn fwd')
    dqkv = torch.empty(N, T, 3 * C, device='cuda', dtype=torch.bfloat16)
    L.check(L.lib().aph_vqgan_attn_test(0, qkv.data_ptr(), dout.data_ptr(), dqkv.data_ptr(), N, T, C, _st()), 'attn bwd')
    for n in range(N):
        qr = qkv[n].double().requires_grad_(True)
        q, k, v = qr[:, :C].t()[None], qr[:, C:2 * C].t()[None], qr[:, 2 * C:].t()[None]
        o = VO.attention(q, k, v)[0].t()
        o.backward(dout[n].double())
        assert _rel(out[n], o) < 2e-2, n
        assert _rel(dqkv[n], qr.grad) < 2e-2, n


# ---- the ends -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('C,H,W', [(256, 31, 56), (128, 13, 7), (128, 64, 96)])
def test_layout_conversions_and_conv_out(L, C, H, W):
    g = torch.Generator().manual_seed(C + H)
    N = 2
    z = torch.randn(N, C, H, W, generator=g).cuda()
    zb = torch.empty(N, H, W, C, device='cuda', dtype=torch.bfloat16)
    L.check(L.lib().aph_vqgan_ends_test(0, z.data_ptr(), None, None, zb.data_ptr(), N, C, H, W, _st()), 'nchw->nhwc')
    assert torch.equal(zb, _nhwc(z).to(torch.bfloat16))
    back = torch.empty_like(z)
    L.check(L.lib().aph_vqgan_ends_test(1, zb.data_ptr(), None, None, back.data_ptr(), N, C, H, W, _st()), 'nhwc->nchw')
    assert torch.equal(back, _nchw(zb.float()))
    w = (torch.randn(3, C, 3, 3, generator=g) * (9 * C) ** -0.5).cuda()
    b = torch.tensor([0.1, -0.2, 0.3]).cuda()
    out = torch.empty(N, 3, H, W, device='cuda')
    L.check(L.lib().aph_vqgan_ends_test(2, zb.data_ptr(), w.data_ptr(), b.data_ptr(), out.data_ptr(), N, C, H, W, _st()), 'conv_out')
    a = _nchw(zb.double().cpu()).requires_grad_(True)
    ref = F.conv2d(a, w.double().cpu(), b.double().cpu(), padding=1)
    assert _rel(out, ref) < 1e-5
    go = torch.randn(N, 3, H, W, generator=g).cuda()
    da = torch.empty(N, H, W, C, device='cuda', dtype=torch.bfloat16)
    L.check(L.lib().aph_vqgan_ends_test(3, go.data_ptr(), w.data_ptr(), None, da.data_ptr(), N, C, H, W, _st()), 'conv_out bwd')
    ref.backward(go.double().cpu())
    assert _rel(da, _nhwc(a.grad)) < 1e-2


# ---- the whole decoder --------------------------------------------------------------------------------------------------------
FWD_BAR, DZ_BAR = 3e-2, 5e-2


def _decoder(cfg, seed):
    from aphantasia_b200 import vqgan
    dec = vqgan.Decoder(**cfg)
    sd = vqgan.synthetic_decoder_state_dict(seed, **cfg)
    dec.load_state_dict(sd)
    return dec.cuda().eval(), sd


def _vs_oracle(dec, sd, cfg, N, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(N, cfg['z_channels'], h, w, generator=g)
    zc = z.cuda().requires_grad_(True)
    out = dec(zc)
    cot = torch.randn(out.shape, generator=g)
    out.backward(cot.cuda())
    zr = z.double().cuda().requires_grad_(True)          # float64 on the GPU: the notebook-size oracle is ~5 TFLOP
    ref = VO.decode(sd, zr, cfg['ch_mult'], cfg['num_res_blocks'], dec.attn_levels)
    ref.backward(cot.double().cuda())
    e_f, e_g = _rel(out, ref), _rel(zc.grad, zr.grad)
    print('N=%d latent %dx%d: forward %.2e, dz %.2e' % (N, h, w, e_f, e_g))
    assert tuple(out.shape) == tuple(ref.shape)
    return e_f, e_g, zc, out


@pytest.mark.parametrize('cfg_name', ['F16_CONFIG', 'F8_CONFIG'])
@pytest.mark.parametrize('N,h,w', [(1, 3, 5), (2, 5, 3), (1, 1, 1)])
def test_decoder_small_latents_vs_float64(L, cfg_name, N, h, w):
    from aphantasia_b200 import vqgan
    cfg = getattr(vqgan, cfg_name)
    dec, sd = _decoder(cfg, 7)
    e_f, e_g, _, _ = _vs_oracle(dec, sd, cfg, N, h, w, 11 + N * h)
    assert e_f < FWD_BAR and e_g < DZ_BAR


@pytest.mark.parametrize('cfg_name,h,w', [('F16_CONFIG', 31, 56), ('F8_CONFIG', 62, 112)])
def test_decoder_at_the_notebook_size_vs_float64(L, cfg_name, h, w):
    """900 x 500 in the notebook: latent 31 x 56 at f16 (496 x 896 out), 62 x 112 at f8 (496 x 896)"""
    from aphantasia_b200 import vqgan
    cfg = getattr(vqgan, cfg_name)
    dec, sd = _decoder(cfg, 5)
    e_f, e_g, _, out = _vs_oracle(dec, sd, cfg, 1, h, w, 3)
    assert tuple(out.shape) == (1, 3, 496, 896)
    assert e_f < FWD_BAR and e_g < DZ_BAR


def test_repack_nograd_forward_and_repeats(L):
    """a weight change re-packs the handle; a no_grad forward (the notebook's checkout) between a forward and its backward does
    not corrupt that backward; repeated forwards and backwards are bit-identical (GroupNorm sums in a fixed order, no atomics)"""
    from aphantasia_b200 import vqgan
    cfg = vqgan.F8_CONFIG
    dec, sd = _decoder(cfg, 2)
    g = torch.Generator().manual_seed(1)
    z = torch.randn(1, 256, 4, 6, generator=g).cuda()
    cot = torch.randn(1, 3, 32, 48, generator=g).cuda()

    def step(zz):
        zz = zz.clone().requires_grad_(True)
        out = dec(zz)
        out.backward(cot)
        return out.detach(), zz.grad

    o1, g1 = step(z)
    for _ in range(2):                               # eager, capture, replay
        o2, g2 = step(z)
        assert torch.equal(o1, o2) and torch.equal(g1, g2)
    zz = z.clone().requires_grad_(True)
    out = dec(zz)
    with torch.no_grad():
        other = dec(torch.randn(1, 256, 4, 6, generator=g).cuda())
    assert not torch.equal(other, out)
    rec = dec.recomputes
    out.backward(cot)
    assert dec.recomputes == rec + 1 and torch.equal(zz.grad, g1)
    with torch.no_grad():
        dec.conv_out.bias.add_(0.5)                   # in place: the version counter moves
    o3, _ = step(z)
    assert _rel(o3, o1 + 0.5) < 1e-6
    sd2 = dict(sd)
    sd2['conv_out.bias'] = sd['conv_out.bias'] + 0.5
    ref = VO.decode(sd2, z.double(), cfg['ch_mult'], cfg['num_res_blocks'], dec.attn_levels)
    assert _rel(o3, ref) < FWD_BAR
    dec.load_state_dict(sd)                           # copy_ into the parameters: re-packed again
    o4, _ = step(z)
    assert torch.equal(o4, o1)


def test_notebook_generate_step_vs_oracle(L):
    """CLIP_VQGAN.ipynb's train(i) at a small size with synthetic weights: lats -> Decoder (f8) -> (x + 1) / 2 -> slice_imgs
    (transforms_fast) -> ViT-B/32 encode_image -> -cosine(txt, emb); d loss / d lats against the float64 decoder and the fp32 CLIP
    oracle through the same crop table, then a few AdamW (amsgrad) steps to finite, decreasing-on-average losses."""
    from aphantasia_b200 import _rng, transforms, vqgan
    from aphantasia_b200.clip import CLIP, synthetic_visual_state_dict
    from aphantasia_b200.utils import slice_imgs
    cfg = vqgan.F8_CONFIG
    dec, dsd = _decoder(cfg, 9)
    vsd = synthetic_visual_state_dict(patch=32, seed=0)
    model = CLIP('ViT-B/32', vsd, True)
    txt = model.encode_text(torch.zeros(1, 77, dtype=torch.long)).cuda()
    S, h, w = 4, 28, 28
    g = torch.Generator().manual_seed(4)
    lats0 = torch.randn(1, 256, h, w, generator=g) * 0.5
    lats = lats0.cuda().requires_grad_(True)

    def loss_of(lats, seed):
        torch.manual_seed(seed); np.random.seed(seed)
        img = (dec(lats) + 1.) / 2.
        crops = slice_imgs([img], S, 224, transforms.transforms_fast, 'uniform', 0.4)[0]
        emb = model.encode_image(crops)
        return -torch.cosine_similarity(txt, emb, dim=-1).mean()

    loss = loss_of(lats, 1)
    loss.backward()
    torch.manual_seed(1); np.random.seed(1)
    tabs, _ = _rng.draw_crop_table(S, (8 * h, 8 * w), 224, 2, 'uniform', 0.4)
    lr_ = lats0.double().cuda().requires_grad_(True)
    img = (VO.decode(dsd, lr_, cfg['ch_mult'], cfg['num_res_blocks'], dec.attn_levels) + 1.) / 2.
    emb = R.build_visual(vsd)(R.sample_crops(img.float().cpu(), tabs[0], 224, 2))
    o_loss = -torch.cosine_similarity(txt.cpu(), emb, dim=-1).mean()
    o_loss.backward()
    e = _rel(lats.grad, lr_.grad)
    print('notebook step: loss %.6f (oracle %.6f), d loss / d lats %.2e' % (loss.item(), o_loss.item(), e))
    assert abs(loss.item() - o_loss.item()) < 5e-3
    assert e < 6e-2
    opt = torch.optim.AdamW([lats], lr=0.05, weight_decay=0.1, amsgrad=True)
    losses = []
    for i in range(4):
        opt.zero_grad()
        l = loss_of(lats, 10 + i)
        l.backward()
        opt.step()
        losses.append(l.item())
    assert all(np.isfinite(losses)), losses
    model.visual.close()
