"""The image synthesis kernels on their own, against float64 references computed from the same fp32 inputs the kernels get:
spectrum -> RGB (aph_synth_fft_fwd / _bwd, csrc/synth_fft.cu), wavelet pyramid -> RGB (aph_synth_dwt_fwd / _bwd,
csrc/synth_dwt.cu) and the Adam update, plain (aph_adam_step) and fused into the synthesis backward (aph_synth_fft_bwd_adam).

FFT sizes and the kernel forms they run (the rule of aph_fft_plan_create, evaluated on the host):
  column pass  H <= 750                         two-buffer, 8 columns per CTA (750 is the largest)
               756, 1001, 1331 (factor 7/11/13)  two-buffer, 4 columns (the single-buffer kernel has radices <= 5 only)
               768, 1080, 2160                   single-buffer in-register, 8 columns
               2400 / 3000 / 6144                single-buffer, 7 / 5 / 3 columns (tiles that do not divide Wh = 9)
               8640, 9375                        two-buffer, 1 column, 202.5 / 219.7 KB of shared memory
  row pass     W <= 2559: two row pairs per CTA; 3375 (odd), 3840, 9375: one pair per CTA
  radices 11 and 13 in 11x13, 121x169, 143x143, 1287x1430, 1001, 1331x2197, 64x2541.
Refused: a prime factor above 13, 9408 on either axis (its two-buffer pass needs 220.5 KB), H or W = 1.

Rounding budget, with u = 2^-24 (fp32 unit roundoff). Measured values are from an H100 80GB HBM3 at a 400 W power limit.
  FFT   Each Stockham stage rounds every value once or twice in fp32 and multiplies by an fp32 twiddle (relative error
        <= u); radix 11 and 13 butterflies are plain 11- and 13-term sums. A length-N transform has ~log_R N stages, so the
        two axes together carry ~10-20 roundings of relative size u that add up like a random walk: a few 1e-7 norm-wise,
        relative to the whole transform. The inputs scale * (P [+ shift]) are rounded once in fp32, the fp64 statistics add
        nothing measurable, and the tail (x * contrast / sigma, 3x3 mix, sigmoid) a few u per element. Bar: 2e-6 per channel
        for x_raw and the output (measured <= 2.1e-7), 1e-6 for the statistics: sum x against sqrt(N sum x^2), sum x^2
        and sum g_img . x against the sum of their absolute terms (measured <= 1.2e-7).
        The backward runs the same transforms in the other order: dP / scale = dZ is compared per channel and per radial
        frequency band (f < 0.05, 0.05 - 0.25, >= 0.25), each band against its own norm, so that an error confined to the
        high-frequency bins (80% of the bins, 0.4% of the energy under the script's decay of 1.5) is seen. Bar 2e-6
        (measured <= 4.6e-7; 6.7e-7 at 2x2, where the low band is the DC bin alone).
        The cotangent is random plus twice the normalised linear output, so sum g_img . x (stats[2]) carries a term as
        large as the rest of the gradient and a wrong or missing projection shows. Under the script's 1/f^1.5 scale that
        projection cancels most of the cotangent in the few lowest bins, where the image lives, and dP (dominated by those
        bins) would carry the cancellation: the test on the real scale uses a plain random cotangent.
        A spectrum whose image mean is 300 times its std keeps these bars in the forward: the FFT's error is relative to
        ||x||, which the mean dominates, and the fp64 statistics do not lose the variance to cancellation. Its backward
        forms (x - mean) * dot / ((N-1) sigma^2) from the fp32 x_raw, whose error is relative to the mean, not to sigma:
        bar 300 x 2e-6 for dZ and dP (measured <= 7.9e-5 at a mean of 205 std).
  DWT   Each output value is a sum of (L/2)^2 products per band (4 bands) in fp32, each adjoint value a sum of L^2; the J
        levels chain such sums. Bar: 5e-6 for the forward and for each level's gradient, against that level's own norm,
        widened by sqrt(L / 12) for filters longer than coif2's 12 taps (db20: 40 taps, 1600-term adjoint sums). Measured:
        forward <= 1.6e-7, level gradients <= 4.5e-7, Yl <= 1.2e-6 (Yl collects all J adjoint levels).
        The float64 reference is our restatement of pytorch_wavelets' DWTInverse (mode 'symmetric'), not the third-party
        code itself: parity with pytorch_wavelets is unpinned.
  Adam  One step from the kernels' own fp32 state and the same fp32 gradient, against float64 arithmetic with the same fp32
        lr, betas and eps: m within 2u of the magnitudes of its two terms, v within 3u, p within 2u |p| + 10u |update| (the
        step size and 1 / sqrt(1 - b2^t) are fp32-rounded, and sqrt, the product with it, add, divide and multiply round
        once each, v's error enters through the sqrt) plus the error of m carried through the update. Gradients include
        values near eps (1e-9 .. 1e-7) and zeros.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import restate as R  # noqa: E402

U = 2.0 ** -24
FWD_BAR = 2e-6
GRAD_BAR = 2e-6
STATS_BAR = 1e-6
DWT_BAR = 5e-6
BANDS = ((0., 0.05), (0.05, 0.25), (0.25, 1.))


@pytest.fixture(scope='module')
def L():
    from aphantasia_b200 import _lib
    assert torch.cuda.is_available()
    return _lib


def _p(t):
    return None if t is None else t.data_ptr()


def colmat_host(colors=1.8):
    from aphantasia_b200.image import _color_matrix_host
    return _color_matrix_host(colors)


def colmat64(cm):
    """Mn[d][c] as float64 from the fp32 host array the kernels get"""
    return None if cm is None else torch.tensor([float(v) for v in cm], dtype=torch.float64).reshape(3, 3)


def rel(got, ref):
    got, ref = got.detach().cpu().double(), ref.detach().cpu().double()
    return float((got - ref).norm() / ref.norm().clamp_min(1e-300))


def per_channel(got, ref):
    return max(rel(got[c], ref[c]) for c in range(got.shape[0]))


# ---------------------------------------------------------------------------------------------------------------- float64 tail
def tail64(x, contrast, M, sig):
    """to_valid_rgb(x * contrast / std(x)) in float64: (out, img, linear output)"""
    img = x * contrast / x.std()
    o = img if M is None else torch.einsum('dc,chw->dhw', M, img)
    return (torch.sigmoid(o) if sig else o), img, o


def correlated_cot(o, seed, k=2.):
    """fp32 cotangent: N(0, 1) plus k times the normalised linear output, so that sum g_img . x is large"""
    g = torch.Generator().manual_seed(seed)
    o = o.detach()
    return (torch.randn(tuple(o.shape), generator=g, dtype=torch.float64) + k * (o - o.mean()) / o.std()).float()


def ref_backward(x, img, out, cot):
    (out * cot.double()).sum().backward()
    gx = (img.grad * x.detach())
    return float(gx.sum()), float(gx.abs().sum())


# ---------------------------------------------------------------------------------------------------------------- FFT
def fft_plan(L, H, W):
    plan = C.c_void_p()
    L.check(L.lib().aph_fft_plan_create(C.byref(plan), H, W), 'aph_fft_plan_create')
    return plan


def fft_fwd(L, plan, H, W, P, scale, shift, mode, contrast, cm, sig):
    x = torch.full((3, H, W), float('nan'), device='cuda')
    out = torch.full((3, H, W), float('nan'), device='cuda')
    stats = torch.full((4,), float('nan'), device='cuda', dtype=torch.float64)
    L.check(L.lib().aph_synth_fft_fwd(plan, P.data_ptr(), scale.data_ptr(), _p(shift), mode, contrast, cm, sig, x.data_ptr(),
                                      stats.data_ptr(), out.data_ptr(), L.stream_ptr()), 'aph_synth_fft_fwd')
    return x, stats, out


def fft_bwd(L, plan, H, W, cot, out, x, stats, scale, contrast, cm, sig):
    """the saved output is passed for apply_sigmoid = 0 too (image.py does), so the sigmoid switch alone decides"""
    gp = torch.full((3, H, W // 2 + 1, 2), float('nan'), device='cuda')
    L.check(L.lib().aph_synth_fft_bwd(plan, cot.data_ptr(), out.data_ptr(), x.data_ptr(), stats.data_ptr(), scale.data_ptr(), contrast, cm,
                                      sig, gp.data_ptr(), L.stream_ptr()), 'aph_synth_fft_bwd')
    return gp


def fft_inputs(H, W, seed, scale='white', mode=0, dc_ratio=None):
    """fp32 spectrum [3,H,Wh,2], positive scale [H,Wh] (white: U(0.5, 1.5); decay: the script's fft_scale at 1.5), shift"""
    Wh = W // 2 + 1
    g = torch.Generator().manual_seed(seed)
    P = torch.randn(3, H, Wh, 2, generator=g)
    s = (0.5 + torch.rand(H, Wh, generator=g)) if scale == 'white' else R.fft_scale(H, W, 1.5)
    shift = None
    if mode == 1:
        shift = torch.randn(H, Wh, generator=g) * 0.7
    elif mode == 2:
        shift = torch.randn(3, H, Wh, 2, generator=g) * 0.7
    if dc_ratio is not None:         # image mean = dc_ratio * std: the DC bin carries P[c, 0, 0] * scale / sqrt(H W) per pixel
        P[:, 0, 0, 0] = dc_ratio * float(torch.tensor(float(H * W)).sqrt()) / float(s[0, 0])
        P[:, 0, 0, 1] = 0.
    return P.float(), s.float().contiguous(), shift


def ref_fft(P, s, H, W, shift, mode, contrast, M, sig):
    """float64 forward from the fp32 inputs: dict of x, out, img, o and the leaf p"""
    p = P.double().requires_grad_(True)
    s64 = s.double()[..., None]
    z = s64 * p
    if mode == 1:
        z = z + (s64 * shift.double()[..., None])
    elif mode == 2:
        z = z + s64 * shift.double()
    x = torch.fft.irfftn(torch.view_as_complex(z), s=(H, W), norm='ortho')
    out, img, o = tail64(x, contrast, M, sig)
    img.retain_grad()
    return dict(p=p, x=x, out=out, img=img, o=o)


def band_masks(H, W):
    fy = torch.fft.fftfreq(H, dtype=torch.float64).abs()[:, None]
    fx = torch.fft.rfftfreq(W, dtype=torch.float64)[None, :]
    f = torch.sqrt(fx * fx + fy * fy)
    return [(f >= lo) & (f < hi) for lo, hi in BANDS]


def band_errors(dz, dz_ref, H, W):
    """max over channels of ||error|| / ||ref|| in each radial band (empty bands skipped): [3,H,Wh,2] float64"""
    errs = []
    for m in band_masks(H, W):
        if not bool(m.any()):
            errs.append(0.)
            continue
        errs.append(max(rel(dz[c][m], dz_ref[c][m]) for c in range(3)))
    return errs


def fft_case(L, H, W, seed, mode=0, cm=True, sig=1, contrast=1.25, scale='white', dc_ratio=None, plan=None):
    """one forward + backward through the C ABI against float64; returns {name: error}"""
    cmh = colmat_host() if cm else None
    P, s, shift = fft_inputs(H, W, seed, scale, mode, dc_ratio)
    ref = ref_fft(P, s, H, W, shift, mode, contrast, colmat64(cmh), sig)
    cot = correlated_cot(ref['o'], seed + 1)
    dot, dot_abs = ref_backward(ref['x'], ref['img'], ref['out'], cot)
    own = plan is None
    plan = fft_plan(L, H, W) if own else plan
    try:
        Pc, sc, shc, cc = P.cuda(), s.cuda(), None if shift is None else shift.cuda(), cot.cuda()
        x, stats, out = fft_fwd(L, plan, H, W, Pc, sc, shc, mode, contrast, cmh, sig)
        gp = fft_bwd(L, plan, H, W, cc, out, x, stats, sc, contrast, cmh, sig)
        torch.cuda.synchronize()
    finally:
        if own:
            L.lib().aph_fft_plan_destroy(plan)
    return compare_fft(ref, x, stats, out, gp, s, H, W, dot, dot_abs)


def compare_fft(ref, x, stats, out, gp, s, H, W, dot, dot_abs):
    assert bool(torch.isfinite(x).all() and torch.isfinite(out).all() and torch.isfinite(gp).all()), 'non-finite output'
    xr = ref['x'].detach()
    N = xr.numel()
    st = stats.cpu()
    s1, s2 = float(xr.sum()), float((xr * xr).sum())
    errs = {'x_raw': per_channel(x.cpu(), xr), 'out': per_channel(out.cpu(), ref['out'].detach()),
            'sum_x': abs(float(st[0]) - s1) / math.sqrt(N * s2), 'sum_x2': abs(float(st[1]) - s2) / s2,
            'dot': abs(float(st[2]) - dot) / dot_abs}
    mean = s1 / N
    xc, xrc = x.cpu().double() - float(st[0]) / N, xr - mean
    errs['x_centered'] = per_channel(xc, xrc) / (xr.norm() / xrc.norm()).item()          # the FFT error is relative to ||x||
    dz_ref = ref['p'].grad / s.double()[..., None]
    dz = gp.cpu().double() / s.double()[..., None]
    for b, e in zip(('dZ_low', 'dZ_mid', 'dZ_high'), band_errors(dz, dz_ref, H, W)):
        errs[b] = e
    errs['dP'] = per_channel(gp.cpu(), ref['p'].grad)
    return errs


def check(errs, what, bars=None):
    bars = bars or {}
    limit = {'x_raw': FWD_BAR, 'out': FWD_BAR, 'x_centered': FWD_BAR, 'sum_x': STATS_BAR, 'sum_x2': STATS_BAR, 'dot': STATS_BAR}
    print('errors', what, ' '.join('%s=%.2e' % kv for kv in sorted(errs.items())))
    bad = {k: v for k, v in errs.items() if not v <= bars.get(k, limit.get(k, GRAD_BAR))}
    assert not bad, (what, bad)


FFT_SIZES = [
    (11, 13), (121, 169), (143, 143),                        # radices 11 and 13
    (1287, 1430), (64, 2541),                                # odd H, odd W
    (1001, 1001), (1331, 2197),                              # two-buffer columns, C = 4
    (750, 16), (756, 16), (768, 16),                         # around the column-form switch
    (2400, 16), (3000, 16), (6144, 16),                      # single-buffer, tiles that do not divide Wh = 9
    (8640, 16),                                              # two-buffer, C = 1
    (9375, 16), (16, 9375),                                  # the largest accepted length on each axis
    (64, 3375),                                              # odd W, one row pair per CTA
    (2, 2), (2, 3), (3, 2),
    (720, 1280), (1080, 1920), (2160, 3840),                 # the benchmark canvases
]


@pytest.mark.parametrize('H,W', FFT_SIZES, ids=['%dx%d' % hw for hw in FFT_SIZES])
def test_fft_synthesis_vs_float64(L, H, W):
    """White scale (every bin counts), shift mode 2, colour matrix, sigmoid, contrast 1.25."""
    check(fft_case(L, H, W, seed=H * 31 + W, mode=2), (H, W))


MODES = [(mode, cm, sig) for mode in (0, 1, 2) for cm in (True, False) for sig in (1, 0)]


@pytest.mark.parametrize('mode,cm,sig', MODES, ids=['shift%d-%s-%s' % (m, 'colmat' if c else 'nocolmat', 'sigmoid' if s else 'linear')
                                                    for m, c, s in MODES])
@pytest.mark.parametrize('H,W', [(143, 143), (1080, 24), (30, 3375)], ids=['143x143', '1080x24', '30x3375'])
def test_fft_modes_vs_float64(L, H, W, mode, cm, sig):
    """Every shift mode, with and without the colour matrix, with and without the sigmoid, forward and backward."""
    check(fft_case(L, H, W, seed=mode * 7 + cm * 3 + sig + H, mode=mode, cm=cm, sig=sig, contrast=0.8), (H, W, mode, cm, sig))


@pytest.mark.parametrize('H,W', [(96, 160), (1080, 24)])
def test_fft_dc_dominated_spectrum(L, H, W):
    """Image mean 300 x its std: sum x^2 - (sum x)^2 / N cancels by 9e4 in fp64. Small contrast keeps the sigmoid live."""
    ratio = 300.
    errs = fft_case(L, H, W, seed=H + 5, mode=0, contrast=0.004, dc_ratio=ratio)
    check(errs, ('dc', H, W), {k: ratio * GRAD_BAR for k in errs if k.startswith('d') and k != 'dot'})


def test_fft_real_scale_through_fft_image(L):
    """The script's path: fft_image(decay 1.5) + to_valid_rgb(colors 1.8) at 720x1280, image_f() alone (no sigmoid, no colour
    matrix) and to_valid_rgb(decorrelate=False) (colour matrix NULL), each forward and spectrum gradient against float64,
    the gradient per band of dP / scale."""
    from aphantasia_b200.image import fft_image, to_valid_rgb
    H, W = 720, 1280
    torch.manual_seed(17)
    params, image_f, _ = fft_image([1, 3, H, W], 0.01, 1.5, None)
    P = params[0].detach().cpu()[0]
    s = image_f.scale.cpu()
    assert torch.equal(s, R.fft_scale(H, W, 1.5))
    for name, fn, M, sig, contrast in (('rgb', to_valid_rgb(image_f, colors=1.8), colmat64(colmat_host(1.8)), 1, 1.1),
                                       ('image_f', image_f, None, 0, 0.9),
                                       ('no_decorrelate', to_valid_rgb(image_f, decorrelate=False), None, 1, 1.0)):
        ref = ref_fft(P, s, H, W, None, 0, contrast, M, sig)
        cot = correlated_cot(ref['o'], 23, k=0.)
        ref_backward(ref['x'], ref['img'], ref['out'], cot)
        params[0].grad = None
        out = fn(contrast=contrast)
        (out * cot.cuda()).sum().backward()
        errs = {'out': per_channel(out[0].cpu(), ref['out'].detach())}
        dz_ref = ref['p'].grad / s.double()[..., None]
        dz = params[0].grad[0].cpu().double() / s.double()[..., None]
        errs.update(zip(('dZ_low', 'dZ_mid', 'dZ_high'), band_errors(dz, dz_ref, H, W)))
        errs['dP'] = per_channel(params[0].grad[0].cpu(), ref['p'].grad)
        check(errs, name)


def test_fft_two_plans_interleaved(L):
    """Two live plans of different sizes, forward A, forward B, backward A, backward B: each owns its scratch."""
    cases = []
    for H, W, seed in ((143, 143, 1), (1080, 96, 2)):
        cmh = colmat_host()
        P, s, _ = fft_inputs(H, W, seed)
        ref = ref_fft(P, s, H, W, None, 0, 1.1, colmat64(cmh), 1)
        cot = correlated_cot(ref['o'], seed)
        dot, dot_abs = ref_backward(ref['x'], ref['img'], ref['out'], cot)
        cases.append(dict(H=H, W=W, P=P.cuda(), s=s, sc=s.cuda(), cot=cot.cuda(), ref=ref, dot=dot, dot_abs=dot_abs, cmh=cmh,
                          plan=fft_plan(L, H, W)))
    try:
        for c in cases:
            c['fwd'] = fft_fwd(L, c['plan'], c['H'], c['W'], c['P'], c['sc'], None, 0, 1.1, c['cmh'], 1)
        for c in cases:
            x, stats, out = c['fwd']
            c['gp'] = fft_bwd(L, c['plan'], c['H'], c['W'], c['cot'], out, x, stats, c['sc'], 1.1, c['cmh'], 1)
        torch.cuda.synchronize()
    finally:
        for c in cases:
            L.lib().aph_fft_plan_destroy(c['plan'])
    for c in cases:
        x, stats, out = c['fwd']
        check(compare_fft(c['ref'], x, stats, out, c['gp'], c['s'], c['H'], c['W'], c['dot'], c['dot_abs']), ('two plans', c['H'], c['W']))


@pytest.mark.parametrize('H,W,msg', [(17, 16, 'prime factor'), (16, 34, 'prime factor'), (9408, 16, 'shared-memory'),
                                     (16, 9408, 'shared-memory'), (1, 16, 'bad arguments'), (16, 1, 'bad arguments')])
def test_fft_plan_refusals(L, H, W, msg):
    lib = L.lib()
    n0 = lib.aph_launch_count()
    plan = C.c_void_p()
    rc = lib.aph_fft_plan_create(C.byref(plan), H, W)
    with pytest.raises(RuntimeError, match=msg):
        L.check(rc, 'aph_fft_plan_create')
    assert plan.value is None
    assert lib.aph_launch_count() == n0


# ---------------------------------------------------------------------------------------------------------------- Adam
def f32(v):
    return float(np.float32(v))


def adam64(p, g, m, v, lr, b1, b2, eps, step):
    """one float64 Adam step from fp32 state and gradient with the kernels' fp32 b1, b2, eps; returns (p, m, v, bounds)"""
    p, g, m, v = (t.cpu().double() for t in (p, g, m, v))
    lr, b1, b2, eps = f32(lr), f32(b1), f32(b2), f32(eps)
    m_err = 2 * U * ((b1 * m).abs() + ((1 - b1) * g).abs())      # m = b1 m + (1 - b1) g may cancel: bound by its terms
    m1 = b1 * m + (1 - b1) * g
    v1 = b2 * v + (1 - b2) * g * g                                 # positive terms
    step_size = lr / (1 - b1 ** step)
    denom = v1.sqrt() / math.sqrt(1 - b2 ** step) + eps
    upd = step_size * m1 / denom
    p1 = p - upd
    p_err = 2 * U * p1.abs() + 10 * U * upd.abs() + step_size * m_err / denom
    return p1, m1, v1, (p_err, m_err, 3 * U * v1)


def adam_ulp_ratio(got, ref):
    """max |got - ref| / bound over p, m, v (<= 1 passes)"""
    return max(float(((g.cpu().double() - r).abs() / b.clamp_min(1e-45)).max()) for g, r, b in zip(got, ref[:3], ref[3]))


def adam_gradients(n, seed):
    """N(0, 1) gradients with a quarter of the elements near eps (1e-9 .. 1e-7) and some exact zeros"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, generator=g)
    small = torch.rand(n, generator=g) < 0.25
    x[small] = x[small].sign() * 10 ** (-9 + 2 * torch.rand(int(small.sum()), generator=g))
    x[torch.rand(n, generator=g) < 0.02] = 0.
    return x


@pytest.mark.parametrize('betas', [(0.9, 0.999), (0.0, 0.999)])
def test_adam_step_vs_float64(L, betas):
    """20 steps of aph_adam_step, lr changed at step 10; each step against float64 Adam from the kernel's own previous state."""
    n = 3 * 4099
    torch.manual_seed(3)
    p = torch.randn(n, device='cuda'); m = torch.zeros_like(p); v = torch.zeros_like(p)
    worst = 0.
    for step in range(1, 21):
        lr = 0.05 if step <= 10 else 0.013
        g = adam_gradients(n, step).cuda()
        ref = adam64(p, g, m, v, lr, *betas, 1e-8, step)
        L.check(L.lib().aph_adam_step(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), n, lr, betas[0], betas[1], 1e-8, step,
                                      L.stream_ptr()), 'aph_adam_step')
        torch.cuda.synchronize()
        worst = max(worst, adam_ulp_ratio((p, m, v), ref))
    print('errors adam', betas, 'worst / bound = %.2f' % worst)
    assert worst <= 1., (betas, worst)


@pytest.mark.parametrize('H,W', [(96, 160), (1080, 96), (2160, 40)])
def test_fused_adam_matches_plain_backward_and_step(L, H, W):
    """aph_synth_fft_bwd_adam (two-buffer column kernel at 96 rows, single-buffer at 1080 and 2160) against
    aph_synth_fft_bwd + aph_adam_step and against float64 Adam on that dP, 4 steps at betas (0.9, 0.999) with an lr change;
    with grad_params non-NULL the fused call writes exactly the plain backward's dP."""
    b1, b2, eps = 0.9, 0.999, 1e-8
    P, s, _ = fft_inputs(H, W, 41)
    p = (P * 0.01).cuda(); m = torch.zeros_like(p); v = torch.zeros_like(p)
    sc, cmh = s.cuda(), colmat_host()
    plan = fft_plan(L, H, W)
    worst = 0.
    try:
        for step in range(1, 5):
            lr = 0.05 if step <= 2 else 0.02
            x, stats, out = fft_fwd(L, plan, H, W, p, sc, None, 0, 1.0, cmh, 1)
            cot = correlated_cot(out.cpu().double(), step).cuda()
            dP = fft_bwd(L, plan, H, W, cot, out, x, stats, sc, 1.0, cmh, 1)
            torch.cuda.synchronize()
            ref = adam64(p, dP, m, v, lr, b1, b2, eps, step)
            pp, mp, vp = p.clone(), m.clone(), v.clone()
            L.check(L.lib().aph_adam_step(pp.data_ptr(), dP.data_ptr(), mp.data_ptr(), vp.data_ptr(), p.numel(), lr, b1, b2, eps, step,
                                          L.stream_ptr()), 'aph_adam_step')
            gp = torch.full_like(dP, float('nan'))
            pw, mw, vw = p.clone(), m.clone(), v.clone()
            L.check(L.lib().aph_synth_fft_bwd_adam(plan, cot.data_ptr(), out.data_ptr(), x.data_ptr(), stats.data_ptr(), sc.data_ptr(), 1.0, cmh,
                                                   1, gp.data_ptr(), pw.data_ptr(), mw.data_ptr(), vw.data_ptr(), lr, b1, b2, eps, step,
                                                   L.stream_ptr()), 'aph_synth_fft_bwd_adam')
            L.check(L.lib().aph_synth_fft_bwd_adam(plan, cot.data_ptr(), out.data_ptr(), x.data_ptr(), stats.data_ptr(), sc.data_ptr(), 1.0, cmh,
                                                   1, None, p.data_ptr(), m.data_ptr(), v.data_ptr(), lr, b1, b2, eps, step,
                                                   L.stream_ptr()), 'aph_synth_fft_bwd_adam')
            torch.cuda.synchronize()
            assert torch.equal(gp, dP), 'the fused backward wrote a different dP'
            assert torch.equal(pw, p) and torch.equal(mw, m) and torch.equal(vw, v), 'writing dP changed the fused update'
            worst = max(worst, adam_ulp_ratio((pp, mp, vp), ref), adam_ulp_ratio((p, m, v), ref))
    finally:
        L.lib().aph_fft_plan_destroy(plan)
    print('errors fused adam', (H, W), 'worst / bound = %.2f' % worst)
    assert worst <= 1., (H, W, worst)


def test_adam_shim_matches_torch_adam_with_momentum(L):
    """aphantasia_b200.optim.Adam at the script's -o adam betas (0.9, 0.999), fused into the synthesis backward, against
    torch.optim.Adam on the same spectrum: 5 steps with an lr change; parameters and both moments."""
    from aphantasia_b200 import optim
    from aphantasia_b200.image import fft_image, to_valid_rgb
    h, w = 96, 160
    torch.manual_seed(8)
    pa, fa, _ = fft_image([1, 3, h, w], 0.07, 1.5, None)
    pb, fb, _ = fft_image([1, 3, h, w], 0.07, 1.5, pa[0].detach().clone())
    ra, rb = to_valid_rgb(fa, colors=1.8), to_valid_rgb(fb, colors=1.8)
    oa = optim.Adam(pa, 0.05, betas=(0.9, 0.999))
    ob = torch.optim.Adam(pb, 0.05, betas=(0.9, 0.999))
    for i in range(5):
        for grp in list(oa.param_groups) + list(ob.param_groups):
            grp['lr'] = 0.05 if i < 3 else 0.01
        cot = torch.randn(1, 3, h, w, device='cuda')
        oa.zero_grad(); (ra() * cot).sum().backward(); oa.step()
        ob.zero_grad(); (rb() * cot).sum().backward(); ob.step()
    assert oa.fused_steps == 5 and pa[0].grad is None
    sa, sb = oa.state[pa[0]], ob.state[pb[0]]
    # The C ABI takes fp32 betas, and the kernels weight the new gradient by 1 - b computed from the rounded b; torch weights
    # it by fp32(1 - b). At b2 = 0.999 the two differ by 1.3e-5 relative. The bias corrections come from the same rounded
    # betas and cancel that factor in the update, so p is compared directly and the moments after removing the factor.
    w1, w2 = (1 - f32(0.9)) / f32(1 - 0.9), (1 - f32(0.999)) / f32(1 - 0.999)
    errs = (rel(pa[0], pb[0]), rel(sa['exp_avg'], sb['exp_avg'] * w1), rel(sa['exp_avg_sq'], sb['exp_avg_sq'] * w2))
    print('errors adam shim', errs, 'moment weights', w1, w2)
    assert max(errs) < 1e-6, errs


# ---------------------------------------------------------------------------------------------------------------- DWT
WAVES = ['haar', 'db2', 'db3', 'db4', 'db8', 'db20', 'sym2', 'sym3', 'coif1', 'coif2']


def dwt_filters32(wave):
    """the fp32 taps the kernels get, and their float64 values"""
    from aphantasia_b200._wavelets import reconstruction_filters
    lo, hi = reconstruction_filters(wave)
    lo32, hi32 = np.asarray(lo, dtype=np.float32), np.asarray(hi, dtype=np.float32)
    olo, ohi = R.wavelet_filters(wave.replace('sym', 'db'))       # sym2 / sym3 are db2 / db3
    assert np.allclose(lo, olo, rtol=0, atol=1e-12) and np.allclose(hi, ohi, rtol=0, atol=1e-12)
    return lo32, hi32, [float(t) for t in lo32], [float(t) for t in hi32]


def dwt_bar(L_taps):
    return DWT_BAR * math.sqrt(max(1., L_taps / 12.))


def dwt_case(L, H, W, wave, seed, contrast=1.15, cm=True, sig=1):
    lo32, hi32, lo64, hi64 = dwt_filters32(wave)
    nt = len(lo32)
    lib = L.lib()
    plan = C.c_void_p()
    L.check(lib.aph_dwt_plan_create(C.byref(plan), H, W, lo32.ctypes.data_as(C.c_void_p), hi32.ctypes.data_as(C.c_void_p), nt),
            'aph_dwt_plan_create')
    try:
        J = C.c_int(); dims = (C.c_int * 32)(); ohw = (C.c_int * 2)()
        L.check(lib.aph_dwt_plan_levels(plan, C.byref(J), dims, ohw), 'aph_dwt_plan_levels')
        J = J.value
        shapes = [(dims[2 * i], dims[2 * i + 1]) for i in range(J)]
        assert shapes == [tuple(t) for t in R.dwt_level_shapes(H, W, nt)], (wave, H, W)
        scales = [f32(v) for v in R.dwt_scales(shapes, 0.3)]
        g = torch.Generator().manual_seed(seed)
        Ys = [torch.randn(3, *shapes[-1], generator=g)] + [torch.randn(3, 3, *hw, generator=g) for hw in shapes]
        cmh = colmat_host() if cm else None
        # float64 reference
        Yo = [y.double()[None].requires_grad_(True) for y in Ys]
        x = R.dwt_inverse(Yo[0], [Yo[i + 1] * scales[i] for i in range(J)], lo64, hi64)[0]
        assert tuple(x.shape[1:]) == (ohw[0], ohw[1]), (wave, H, W, tuple(x.shape), tuple(ohw))
        out_r, img, o = tail64(x, contrast, colmat64(cmh), sig)
        img.retain_grad()
        cot = correlated_cot(o, seed + 1)
        dot, dot_abs = ref_backward(x, img, out_r, cot)
        # kernels
        oh, ow = ohw[0], ohw[1]
        Yc = [y.cuda() for y in Ys]
        xk = torch.full((3, oh, ow), float('nan'), device='cuda'); outk = torch.full_like(xk, float('nan'))
        stats = torch.full((4,), float('nan'), device='cuda', dtype=torch.float64)
        sc = (C.c_float * J)(*scales)
        ptrs = (C.c_void_p * (J + 1))(*[y.data_ptr() for y in Yc])
        L.check(lib.aph_synth_dwt_fwd(plan, ptrs, sc, contrast, cmh, sig, xk.data_ptr(), stats.data_ptr(), outk.data_ptr(), L.stream_ptr()),
                'aph_synth_dwt_fwd')
        grads = [torch.full_like(y, float('nan')) for y in Yc]
        gptrs = (C.c_void_p * (J + 1))(*[t.data_ptr() for t in grads])
        L.check(lib.aph_synth_dwt_bwd(plan, cot.cuda().data_ptr(), outk.data_ptr(), xk.data_ptr(), stats.data_ptr(), sc, contrast, cmh, sig,
                                      gptrs, L.stream_ptr()), 'aph_synth_dwt_bwd')
        torch.cuda.synchronize()
    finally:
        lib.aph_dwt_plan_destroy(plan)
    xr = x.detach()
    N = xr.numel()
    s1, s2 = float(xr.sum()), float((xr * xr).sum())
    st = stats.cpu()
    errs = {'x_raw': per_channel(xk.cpu(), xr), 'out': per_channel(outk.cpu(), out_r.detach()),
            'sum_x': abs(float(st[0]) - s1) / math.sqrt(N * s2), 'sum_x2': abs(float(st[1]) - s2) / s2,
            'dot': abs(float(st[2]) - dot) / dot_abs, 'grad_Yl': rel(grads[0], Yo[0].grad[0])}
    for i in range(J):
        errs['grad_level%d' % (i + 1)] = rel(grads[i + 1], Yo[i + 1].grad[0])
    return errs, nt


DWT_CASES = [(64, 96, w) for w in WAVES] + [(135, 240, w) for w in ('db3', 'coif2', 'db8')] + [(33, 47, w) for w in WAVES]


@pytest.mark.parametrize('H,W,wave', DWT_CASES, ids=['%dx%d-%s' % c for c in DWT_CASES])
def test_dwt_synthesis_vs_float64(L, H, W, wave):
    """Every built-in wavelet, even (64x96) and odd sizes (135x240, 33x47: ll rows and columns are trimmed; at 33x47 the
    coarse bands of db20 are about as long as the filter). Forward, statistics, and the gradient of Yl and of every level."""
    errs, nt = dwt_case(L, H, W, wave, seed=H * 3 + W + len(wave))
    bar = dwt_bar(nt)
    check(errs, (H, W, wave), {k: bar for k in errs if k in ('x_raw', 'out') or k.startswith('grad')})


@pytest.mark.parametrize('H,W', [(720, 1280), (1080, 1920)])
def test_dwt_coif2_script_sizes_through_dwt_image(L, H, W):
    """dwt_image's default coif2 + to_valid_rgb at the script's default 1280x720 and at 1920x1080 against float64."""
    from aphantasia_b200.image import dwt_image, to_valid_rgb
    torch.manual_seed(H)
    Ys, gen, _ = dwt_image([1, 3, H, W], 'coif2', 0.3, 1.8, None)
    lo32, hi32, lo64, hi64 = dwt_filters32('coif2')
    assert gen.level_hw == [tuple(t) for t in R.dwt_level_shapes(H, W, 12)]
    scales = [f32(v) for v in gen.scales]
    Yo = [y.detach().cpu().double().requires_grad_(True) for y in Ys]
    x = R.dwt_inverse(Yo[0], [Yo[i + 1] * scales[i] for i in range(gen.J)], lo64, hi64)[0]
    out_r, img, o = tail64(x, 1.0, colmat64(colmat_host(1.8)), 1)
    img.retain_grad()
    cot = correlated_cot(o, 5)
    ref_backward(x, img, out_r, cot)
    rgb = to_valid_rgb(gen, colors=1.8)()
    (rgb * cot.cuda()[None]).sum().backward()
    errs = {'out': per_channel(rgb[0].cpu(), out_r.detach()), 'grad_Yl': rel(Ys[0].grad, Yo[0].grad)}
    for i in range(gen.J):
        errs['grad_level%d' % (i + 1)] = rel(Ys[i + 1].grad, Yo[i + 1].grad)
    check(errs, ('coif2', H, W))


@pytest.mark.parametrize('taps,msg', [(5, 'filter length 5'), (42, 'filter length 42'), (0, 'filter length 0')])
def test_dwt_plan_refusals(L, taps, msg):
    lib = L.lib()
    n0 = lib.aph_launch_count()
    f = (C.c_float * 64)(*([0.1] * 64))
    plan = C.c_void_p()
    rc = lib.aph_dwt_plan_create(C.byref(plan), 64, 96, f, f, taps)
    with pytest.raises(RuntimeError, match=msg):
        L.check(rc, 'aph_dwt_plan_create')
    assert plan.value is None
    assert lib.aph_launch_count() == n0
