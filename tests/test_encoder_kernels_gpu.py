"""The encoder's attention and LayerNorm kernels on their own, against float64 references computed from the same bf16 / fp32
inputs the kernels get (aph_attn_test, aph_ln_fwd_test, aph_ln_bwd_test), and the whole encoder on weights under which those
kernels matter: LayerNorm affines away from the identity, non-zero attention biases, sharper attention.

Attention: every dispatch bucket of the image tower (T <= 32, <= 64: persistent TMA-fed kernels; <= 112, <= 208, <= 256: one CTA
per (sample, head)) and of the text tower's causal forward (T <= 32, <= 64, <= 112), at and across every bucket edge, 1 and 12
heads, in four logit regimes:
  current   logits with std 0.5, what the synthetic encoder weights give (nearly uniform softmax)
  sharp     std 4
  extreme   even query rows see every logit near -200 (no max subtraction: exp underflows, the row sums to 0), odd rows see one
            key at +200 above the rest; a padded key (logit 0) that leaks into the softmax dominates the -200 rows
  dominant  each row has one key 10 above the rest, at key 0, at T - 1 or at the first key of the last 16-key tile
and at item counts around every persistent grid size the T <= 64 kernels choose (k * SMs +- 1).

Rounding budget of the attention kernels. Q K^T and dO V^T are fp32 sums of exact products of bf16 operands, and the softmax
statistics are fp32: their error is ~1e-6 relative. What costs precision is bf16 rounding, which has a relative error of at
most u = 2^-8 per element and about 0.4 u = 1.6e-3 RMS over random significands. The forward rounds twice: the probabilities
P (the A operand of P V) and the output. The backward rounds P (for dV = P^T dO) or dS = P o (dP - delta) / 8 (for dQ = dS K and
dK = dS^T Q), and then its output. Sums over keys of independently rounded terms keep the relative size of the rounding as
long as they do not cancel, so a (sample, head) block of the output or of dV carries about sqrt(2) * 0.4 u = 2.2e-3 norm-wise.
dQ = dS K and dK = dS^T Q do cancel: each row of dS sums to zero, so with few keys (T = 2), sharp rows or a block whose norm
sits in a few elements (one dominant key), the rounding of dS alone reaches 1e-2 of the result (measured on an H100: up to
1.4e-2 at T = 2, sharp logits). The reference for dQ and dK therefore rounds dS / 8 to bf16 where the kernels do, which
leaves the output rounding and the fp32 arithmetic. Bars: 2u = 7.8e-3 per (sample, head) block for every output, and 1e-2
per output row of the forward (a 64-element row norm scatters more than a block norm).

LayerNorm: every width of NCH_DISPATCH (128 ... 1024), rows that are random, that sit on a common offset of 1e3 with std 1, and
that are nearly constant (variance 1e-8, far below eps = 1e-5). fp32 outputs (mean, rstd, dx) within 1e-5 relative; each bf16
output within one bf16 ulp of the rounded float64 value (plus the fp32 arithmetic's few ulps where the value cancels).
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import restate as R  # noqa: E402

U_BF16 = 2.0 ** -8
BLOCK_BAR = 2 * U_BF16
ROW_BAR = 1e-2
SEQ = [1, 2, 17, 31, 32, 33, 50, 63, 64, 65, 77, 111, 112, 113, 196, 197, 208, 209, 255, 256]
CAUSAL_SEQ = [t for t in SEQ if t <= 112]
REGIMES = ['current', 'sharp', 'extreme', 'dominant']


@pytest.fixture(scope='module')
def L():
    from aphantasia_b200 import _lib
    assert torch.cuda.is_available()
    return _lib


def _p(t):
    return None if t is None else t.data_ptr()


# ---------------------------------------------------------------------------------------------------------------- attention
def make_qkv(S, T, heads, regime, seed):
    """bf16 [S*T, 3*64*heads] (q | k | v) on the GPU whose logits q.k/8 follow `regime` (see the module docstring)"""
    g = torch.Generator().manual_seed(seed)
    sig = 2.0 if regime == 'sharp' else 0.5 ** 0.5
    q = torch.randn(S, heads, T, 64, generator=g) * sig
    k = torch.randn(S, heads, T, 64, generator=g) * sig
    v = torch.randn(S, heads, T, 64, generator=g)
    rows = torch.arange(T)
    if regime == 'extreme':
        q[..., :2] = 0.; k[..., :2] = 0.
        k[..., 0] = 4.                                                          # every key
        star = (torch.arange(S * heads) * 7 + 3) % T                           # one key per (sample, head)
        k.view(S * heads, T, 64)[torch.arange(S * heads), star, 1] = 4.
        q[:, :, rows % 2 == 0, 0] = -400.                                      # logits -200 + N(0, 0.5)
        q[:, :, rows % 2 == 1, 1] = 400.                                       # key `star` at +200
    elif regime == 'dominant':
        q[..., 1:4] = 0.; k[..., 1:4] = 0.
        for m, j in enumerate((0, T - 1, 16 * ((T - 1) // 16))):
            k[:, :, j, 1 + m] = 4.
        q[:, :, rows, 1 + rows % 3] = 20.                                      # row i: +10 on key (0, T-1, last tile)[i % 3]
    x = torch.stack((q, k, v)).permute(1, 3, 0, 2, 4).reshape(S * T, 3 * 64 * heads)
    return x.bfloat16().cuda()


def split_heads(m, S, T, heads, parts):
    """token-major [S*T, parts*D] -> float64 [parts, S, heads, T, 64]"""
    return m.double().reshape(S, T, parts, heads, 64).permute(2, 0, 3, 1, 4)


def ref_attention(qkv, dout, S, T, heads, causal=False):
    """float64 forward output and (with dout) dq, dk, dv, each [S, heads, T, 64]; dq and dk from dS / 8 rounded to bf16"""
    q, k, v = split_heads(qkv, S, T, heads, 3)
    s = q @ k.transpose(-1, -2) / 8.
    if causal:
        s = s.masked_fill(torch.ones(T, T, dtype=torch.bool, device=s.device).triu(1), -math.inf)
    p = torch.softmax(s, -1)
    o = p @ v
    if dout is None:
        return o
    do = split_heads(dout, S, T, heads, 1)[0]
    dp = do @ v.transpose(-1, -2)
    ds = (p * (dp - (p * dp).sum(-1, keepdim=True)) / 8.).to(torch.bfloat16).double()     # the kernels' one rounding of dS
    return o, ds @ k, ds.transpose(-1, -2) @ q, p.transpose(-1, -2) @ do


def run_attention(L, fwd, causal, qkv, dout, S, T, heads):
    D = 64 * heads
    out = torch.full((S * T, D if fwd else 3 * D), float('nan'), device='cuda', dtype=torch.bfloat16)
    L.check(L.lib().aph_attn_test(int(fwd), int(causal), qkv.data_ptr(), _p(dout), out.data_ptr(), S, T, D, heads, L.stream_ptr()),
            'aph_attn_test')
    torch.cuda.synchronize()
    return out


def rel_err(got, ref, dims):
    """max over the leading (block or row) index of ||got - ref|| / ||ref|| over the trailing `dims` dimensions"""
    d, r = (got - ref).flatten(-dims).norm(dim=-1), ref.flatten(-dims).norm(dim=-1)
    return float((d / r.clamp_min(1e-300)).max())


def attention_errors(L, S, T, heads, regime, seed, causal=False, backward=True):
    """runs the kernels once; {name: max relative error}; raises if an output element is not finite"""
    qkv = make_qkv(S, T, heads, regime, seed)
    g = torch.Generator().manual_seed(seed + 1)
    dout = None if causal or not backward else (torch.randn(S * T, 64 * heads, generator=g) * 0.5).bfloat16().cuda()
    out = run_attention(L, True, causal, qkv, None, S, T, heads)
    assert bool(torch.isfinite(out).all()), 'forward output has non-finite elements (unwritten or overflowed)'
    refs = ref_attention(qkv, dout, S, T, heads, causal)
    o_ref = refs[0] if dout is not None else refs
    o = split_heads(out, S, T, heads, 1)[0]
    errs = {'out_block': rel_err(o, o_ref, 2), 'out_row': rel_err(o, o_ref, 1)}
    if dout is not None:
        dqkv = run_attention(L, False, False, qkv, dout, S, T, heads)
        assert bool(torch.isfinite(dqkv).all()), 'dqkv has non-finite elements (unwritten or overflowed)'
        got = split_heads(dqkv, S, T, heads, 3)
        for name, gt, rf in zip(('dq', 'dk', 'dv'), got, refs[1:]):
            errs[name + '_block'] = rel_err(gt, rf, 2)
    return errs


def _check(errs, what):
    bad = {k: v for k, v in errs.items() if v > (ROW_BAR if k.endswith('_row') else BLOCK_BAR)}
    assert not bad, (what, bad)


@pytest.mark.parametrize('regime', REGIMES)
@pytest.mark.parametrize('heads', [1, 12])
@pytest.mark.parametrize('T', SEQ)
def test_attention_fwd_bwd_vs_float64(L, T, heads, regime):
    _check(attention_errors(L, 3, T, heads, regime, seed=T * 100 + heads), (T, heads, regime))


@pytest.mark.parametrize('d', [-1, 0, 1])
@pytest.mark.parametrize('k', [0, 1, 2, 3, 4, 6, 8, 12])
@pytest.mark.parametrize('T', [17, 50])
def test_attention_persistent_item_counts(L, T, k, d):
    """S = k * SMs + d items at one head brackets every grid the persistent kernels choose (SMs x 2, 3, 4, 6 CTAs) and twice
    that, so every CTA walks 1, 2 or more items from both halves of its double buffer; k = 0 is the single item S = 1."""
    if k == 0 and d != 1:
        pytest.skip('S = 1 is k = 0, d = 1')
    S = k * torch.cuda.get_device_properties(0).multi_processor_count + d
    _check(attention_errors(L, S, T, 1, 'current', seed=S + T), (T, S))


@pytest.mark.parametrize('S,T', [(190, 50), (47, 197)])
@pytest.mark.parametrize('regime', ['current', 'sharp'])
def test_attention_benchmark_shapes(L, S, T, regime):
    _check(attention_errors(L, S, T, 12, regime, seed=S), (S, T, regime))


@pytest.mark.parametrize('heads', [1, 12])
def test_attention_single_token_is_exact(L, heads):
    """T = 1: softmax of one logit is exactly 1, so out = v, dQ = dK = 0 and dV = dO bit for bit."""
    S, D = 5, 64 * heads
    qkv = make_qkv(S, 1, heads, 'sharp', 11)
    dout = torch.randn(S, D, device='cuda').bfloat16()
    out = run_attention(L, True, False, qkv, None, S, 1, heads)
    dqkv = run_attention(L, False, False, qkv, dout, S, 1, heads)
    assert torch.equal(out, qkv[:, 2 * D:])
    assert bool((dqkv[:, :2 * D] == 0).all()) and torch.equal(dqkv[:, 2 * D:], dout)
    out_c = run_attention(L, True, True, qkv, None, S, 1, heads)
    assert torch.equal(out_c, qkv[:, 2 * D:])


def test_attention_refuses_unsupported_shapes(L):
    """T = 257 (image tower), T = 113 (causal) and a causal backward return an error and launch nothing."""
    lib = L.lib()
    S, heads, D = 2, 2, 128
    qkv = torch.zeros(S * 257, 3 * D, device='cuda', dtype=torch.bfloat16)
    dout = torch.zeros(S * 257, D, device='cuda', dtype=torch.bfloat16)
    out = torch.zeros(S * 257, 3 * D, device='cuda', dtype=torch.bfloat16)
    n0 = lib.aph_launch_count()
    for fwd, causal, T, msg in ((1, 0, 257, '257'), (0, 0, 257, '257'), (1, 1, 113, '113'), (0, 1, 50, 'backward')):
        rc = lib.aph_attn_test(fwd, causal, qkv.data_ptr(), dout.data_ptr(), out.data_ptr(), S, T, D, heads, L.stream_ptr())
        with pytest.raises(RuntimeError, match=msg):
            L.check(rc, 'aph_attn_test')
    torch.cuda.synchronize()
    assert lib.aph_launch_count() == n0
    assert bool((out == 0).all())


@pytest.mark.parametrize('regime', REGIMES)
@pytest.mark.parametrize('heads', [1, 12])
@pytest.mark.parametrize('T', CAUSAL_SEQ)
def test_causal_attention_vs_float64(L, T, heads, regime):
    _check(attention_errors(L, 3, T, heads, regime, seed=T * 10 + heads, causal=True, backward=False), (T, heads, regime))


@pytest.mark.parametrize('T', [17, 33, 50, 64, 77, 112])
def test_causal_rows_ignore_later_tokens(L, T):
    """Replacing q, k and v of every token after i leaves output rows 0 .. i bit for bit unchanged."""
    S, heads = 2, 12
    D = 64 * heads
    base = make_qkv(S, T, heads, 'sharp', T)
    out0 = run_attention(L, True, True, base, None, S, T, heads).reshape(S, T, D)
    for i in sorted({0, 15, 16, T // 2, T - 2}):
        if not 0 <= i < T - 1:
            continue
        mod = base.clone().reshape(S, T, 3 * D)
        mod[:, i + 1:] = (torch.randn(S, T - i - 1, 3 * D, device='cuda') * 3).bfloat16()
        out = run_attention(L, True, True, mod.reshape(S * T, 3 * D), None, S, T, heads).reshape(S, T, D)
        assert torch.equal(out[:, :i + 1], out0[:, :i + 1]), (T, i)
        assert not torch.equal(out[:, i + 1:], out0[:, i + 1:]), (T, i)


# ---------------------------------------------------------------------------------------------------------------- LayerNorm
WIDTHS = [128, 256, 512, 768, 1024]


def ln_rows(n, D, seed):
    """fp32 [3n, D] on the GPU: n random rows, n rows on a common offset of 1e3 (std 1), n nearly constant rows (var 1e-8)"""
    g = torch.Generator().manual_seed(seed)
    rnd = torch.randn(n, D, generator=g) * 2 + torch.randn(n, 1, generator=g)
    off = 1e3 + torch.randn(n, D, generator=g)
    flat = torch.rand(n, 1, generator=g) * 4 - 2 + 1e-4 * torch.randn(n, D, generator=g)
    return torch.cat((rnd, off, flat)).cuda()


def ln_affine(D, seed):
    g = torch.Generator().manual_seed(seed)
    return ((1 + (torch.rand(D, generator=g) * 2 - 1) * 0.5).cuda(), ((torch.rand(D, generator=g) * 2 - 1) * 0.5).cuda())


def ln_stats64(x):
    x = x.double()
    m = x.mean(1)
    return m, 1. / torch.sqrt(((x - m[:, None]) ** 2).mean(1) + 1e-5)


def bf16_ulp(r):
    """one bf16 ulp at |r| (8-bit significand), r float64"""
    a = r.abs().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(a)) - 7)


def assert_bf16_close(got, ref, floor, what):
    """each bf16 element within one bf16 ulp of the float64 value rounded to bf16, plus `floor` (fp32 arithmetic)"""
    rb = ref.to(torch.bfloat16).double()
    err = (got.double() - rb).abs()
    tol = bf16_ulp(rb) + floor
    assert bool((err <= tol).all()), (what, float((err / tol).max()))


@pytest.mark.parametrize('D', WIDTHS)
def test_ln_fwd_vs_float64(L, D):
    x = ln_rows(23, D, D)
    gamma, beta = ln_affine(D, D + 1)
    rows = x.shape[0]
    y = torch.full((rows, D), float('nan'), device='cuda', dtype=torch.bfloat16)
    mean = torch.full((rows,), float('nan'), device='cuda'); rstd = mean.clone()
    L.check(L.lib().aph_ln_fwd_test(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), y.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
                                    rows, D, L.stream_ptr()), 'aph_ln_fwd_test')
    torch.cuda.synchronize()
    m64, r64 = ln_stats64(x)
    assert float(((mean.double() - m64).abs() / (m64.abs() + 1. / r64)).max()) < 1e-5
    assert float(((rstd.double() - r64).abs() / r64).max()) < 1e-5
    # y from the kernel's own (checked) statistics: x - mean of a 1e3-offset row amplifies the fp32 mean's last bit
    xh = (x.double() - mean.double()[:, None]) * rstd.double()[:, None]
    ref = xh * gamma.double() + beta.double()
    assert_bf16_close(y, ref, 2.0 ** -21 * ((xh * gamma.double()).abs() + beta.double().abs()), ('y', D))


def ln_bwd_case(D, S, T, dy_bf16, seed):
    x = ln_rows(S * T // 3 + 1, D, seed)[:S * T].contiguous()
    gamma, _ = ln_affine(D, seed + 1)
    m64, r64 = ln_stats64(x)
    mean, rstd = m64.float(), r64.float()
    dy = torch.randn(S * T, D, device='cuda')
    dy = dy.bfloat16() if dy_bf16 else dy
    # float64 LayerNorm data-gradient from the fp32 statistics the kernel gets
    xh = (x.double() - mean.double()[:, None]) * rstd.double()[:, None]
    dxh = dy.double() * gamma.double()
    s1, s2 = dxh.mean(1, keepdim=True), (dxh * xh).mean(1, keepdim=True)
    ref = rstd.double()[:, None] * (dxh - s1 - xh * s2)
    floor = 2.0 ** -16 * rstd.double()[:, None] * (dxh.abs() + s1.abs() + (xh * s2).abs())
    return x, gamma, mean, rstd, dy, ref, floor


def run_ln_bwd(L, dy, x, mean, rstd, gamma, dx, dx_bf, rows, T, D, mode, accumulate, dcls=None):
    L.check(L.lib().aph_ln_bwd_test(dy.data_ptr(), int(dy.dtype == torch.bfloat16), x.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
                                    gamma.data_ptr(), _p(dx), dx_bf.data_ptr(), rows, T, D, mode, accumulate, _p(dcls), L.stream_ptr()),
            'aph_ln_bwd_test')
    torch.cuda.synchronize()


def assert_rows_close(got, ref, what):
    e = rel_err(got.double(), ref, 1)
    assert e < 1e-5, (what, e)


@pytest.mark.parametrize('accumulate', [0, 1])
@pytest.mark.parametrize('dy_bf16', [0, 1])
@pytest.mark.parametrize('D', WIDTHS)
def test_ln_bwd_mode0_vs_float64(L, D, dy_bf16, accumulate):
    """mode 0: dx (+)= LN'(dy) on every row; accumulate = 0 must not read dx (prefilled with NaN)."""
    S, T = 3, 50
    x, gamma, mean, rstd, dy, ref, floor = ln_bwd_case(D, S, T, dy_bf16, D + 7 * dy_bf16)
    prior = torch.randn(S * T, D, device='cuda') if accumulate else torch.full((S * T, D), float('nan'), device='cuda')
    dx = prior.clone()
    dx_bf = torch.full((S * T, D), float('nan'), device='cuda', dtype=torch.bfloat16)
    run_ln_bwd(L, dy, x, mean, rstd, gamma, dx, dx_bf, S * T, T, D, 0, accumulate)
    if accumulate:
        ref = ref + prior.double()
        floor = floor + 2.0 ** -22 * prior.double().abs()
    assert_rows_close(dx, ref, ('dx', D))
    assert_bf16_close(dx_bf, ref, floor, ('dx_bf16', D))


@pytest.mark.parametrize('dy_bf16', [0, 1])
@pytest.mark.parametrize('D', WIDTHS)
def test_ln_bwd_mode1_adds_dcls_on_class_rows(L, D, dy_bf16):
    """mode 1: dx = LN'(dy) + dcls[s] on rows s*T only; every row is written and dx is not read."""
    S, T = 3, 50
    x, gamma, mean, rstd, dy, ref, floor = ln_bwd_case(D, S, T, dy_bf16, 3 * D + dy_bf16)
    dcls = torch.randn(S, D, device='cuda') * 3
    dx = torch.full((S * T, D), float('nan'), device='cuda')
    dx_bf = torch.full((S * T, D), float('nan'), device='cuda', dtype=torch.bfloat16)
    run_ln_bwd(L, dy, x, mean, rstd, gamma, dx, dx_bf, S * T, T, D, 1, 0, dcls)
    ref = ref.clone()
    ref[::T] += dcls.double()
    floor = floor.clone()
    floor[::T] += 2.0 ** -22 * dcls.double().abs()
    assert_rows_close(dx, ref, ('dx', D))
    assert_bf16_close(dx_bf, ref, floor, ('dx_bf16', D))


@pytest.mark.parametrize('dy_bf16', [0, 1])
@pytest.mark.parametrize('D', WIDTHS)
def test_ln_bwd_mode2_writes_token_rows_only(L, D, dy_bf16):
    """mode 2 (ln_pre): the class rows are skipped and token t of sample s lands on row s*(T-1) + t-1 of dtok; two guard rows
    past the end and every row are checked, so a stray or missing write shows."""
    S, T = 3, 50
    x, gamma, mean, rstd, dy, ref, floor = ln_bwd_case(D, S, T, dy_bf16, 5 * D + dy_bf16)
    sentinel = -12345.
    dtok = torch.full((S * (T - 1) + 2, D), sentinel, device='cuda', dtype=torch.bfloat16)
    run_ln_bwd(L, dy, x, mean, rstd, gamma, None, dtok, S * T, T, D, 2, 0)
    keep = torch.arange(S * T, device='cuda') % T != 0
    assert bool((dtok[-2:] == sentinel).all()), 'a write past the last token row'
    assert_bf16_close(dtok[:-2], ref[keep], floor[keep], ('dtok', D))


# ---------------------------------------------------------------------------------------------------------------- the encoder
QK_SCALE = 2.0       # scales the q and k rows of every in_proj_weight: logit std ~2.5 instead of 0.5 (measured with the oracle)


def perturbed_visual_state_dict(patch, qk_scale=QK_SCALE, seed=0):
    """synthetic_visual_state_dict with every LayerNorm affine at 1 + U(+-0.5) / U(+-0.5) (distinct per layer), the attention
    biases at U(+-0.2) and the q / k projections scaled by qk_scale, so that a dropped affine, a bias or LayerNorm in the wrong
    slot or a softmax that is wrong away from uniform all move the embeddings."""
    sd = R.synthetic_visual_state_dict(patch, seed)
    g = torch.Generator().manual_seed(7919 + patch + seed)
    uni = lambda shape, b: (torch.rand(shape, generator=g) * 2 - 1) * b
    for k in list(sd):
        v = sd[k]
        if k.endswith(('ln_pre.weight', 'ln_post.weight', 'ln_1.weight', 'ln_2.weight')):
            sd[k] = 1 + uni(v.shape, 0.5)
        elif k.endswith(('ln_pre.bias', 'ln_post.bias', 'ln_1.bias', 'ln_2.bias')):
            sd[k] = uni(v.shape, 0.5)
        elif k.endswith(('attn.in_proj_bias', 'attn.out_proj.bias')):
            sd[k] = uni(v.shape, 0.2)
        elif k.endswith('attn.in_proj_weight'):
            w = v.clone()
            w[:2 * w.shape[1]] *= qk_scale
            sd[k] = w
    return sd


def _run(L, vis, x, cot):
    lib = L.lib()
    S = x.shape[0]
    emb = torch.full((S, 512), float('nan'), device='cuda'); gx = torch.full(tuple(x.shape), float('nan'), device='cuda')
    L.check(lib.aph_vit_fwd(vis.handle, x.data_ptr(), S, emb.data_ptr(), 1, L.stream_ptr()), 'vit_fwd')
    L.check(lib.aph_vit_bwd(vis.handle, cot.data_ptr(), S, gx.data_ptr(), L.stream_ptr()), 'vit_bwd')
    torch.cuda.synchronize()
    return emb, gx


def _inputs(S, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(S, 3, 224, 224, generator=g), torch.randn(S, 512, generator=g) * 0.1


def per_sample_err(a, b):
    a, b = a.detach().cpu().double().flatten(1), b.detach().cpu().double().flatten(1)
    return ((a - b).norm(dim=1) / b.norm(dim=1)).max().item(), float((a - b).norm() / b.norm())


@pytest.mark.parametrize('patch,S', [(32, 3), (16, 2)])
def test_encoder_on_perturbed_weights_vs_oracle(L, patch, S):
    """Forward and data-gradient against the fp32 oracle, per sample and globally, eager / capture / replay bit-identical."""
    from aphantasia_b200.clip import VisionTransformer
    sd = perturbed_visual_state_dict(patch)
    vis = VisionTransformer(sd, max_batch=S)
    x, cot = _inputs(S, 300 + S)
    xo = x.clone().requires_grad_(True)
    eo = R.build_visual(sd)(xo)
    (eo * cot).sum().backward()
    xc, cc = x.cuda(), cot.cuda()
    runs = [_run(L, vis, xc, cc) for _ in range(3)]
    for emb, gx in runs:
        errs = per_sample_err(emb, eo) + per_sample_err(gx, xo.grad)
        assert max(errs) < 2e-2, (patch, S, errs)
    for emb, gx in runs[1:]:
        assert torch.equal(emb, runs[0][0]) and torch.equal(gx, runs[0][1]), 'graph capture / replay differ from the eager call'
    vis.close()


@pytest.mark.parametrize('patch,S', [(32, 190), (16, 47)])
def test_encoder_batch_invariance(L, patch, S):
    """Each sample's embedding and image gradient from the batched call equal that image run alone (S = 1): a wrong
    (sample, head) item, row or tile anywhere in the pipeline shows in the one sample it belongs to."""
    from aphantasia_b200.clip import VisionTransformer
    sd = perturbed_visual_state_dict(patch)
    vis = VisionTransformer(sd, max_batch=S)
    x, cot = (t.cuda() for t in _inputs(S, 500 + S))
    emb, gx = _run(L, vis, x, cot)
    worst = [0., 0.]
    for s in range(S):
        e1, g1 = _run(L, vis, x[s:s + 1].contiguous(), cot[s:s + 1].contiguous())
        worst[0] = max(worst[0], per_sample_err(emb[s:s + 1], e1)[0])
        worst[1] = max(worst[1], per_sample_err(gx[s:s + 1], g1)[0])
    assert worst == [0., 0.], (patch, S, worst)
    vis.close()
