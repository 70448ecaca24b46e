"""GPU: aphantasia_b200.optim (Adam / AdamW updated inside the generators' synthesis backwards) against the stock torch optimiser.

For each generator at a non-square 360x640 (fft_image, dwt_image with coif2, pixel_image) and each of the scripts' four -opt
choices, 20 steps from one fixed upstream gradient grad_out (loss = <rgb, grad_out>) with a --prog-style lr edit before every
step. Both sides start every step from the same parameters and moments (the fused side's are copied into the stock side after
each comparison), so every step is checked on its own: parameters, exp_avg, exp_avg_sq and max_exp_avg_sq, element by element,
as max |fused - stock| / max |stock| per tensor. The gradients are bit-identical (same kernels).

The library takes the betas as fp32 (the C ABI of aph_adam_step and the fused backwards), so 1 - beta2 is 1 - fp32(0.999) =
9.99987e-4 where torch, from the Python float, uses 1e-3: a relative difference of 1.3e-5 in the new term of exp_avg_sq (and
3.6e-7 in exp_avg's for beta1 = 0.9), and in the bias corrections. The stock optimiser here therefore gets the fp32 values of
the betas, and what remains is fp32 operation order: bar 1e-6 per step (measured on an H100: at most 1.9e-7 over every
generator and -opt choice). test_scripts_double_betas_differ_by_the_fp32_betas_only bounds the difference with the scripts' own
betas (measured: 1.3e-5, the size of the 1 - beta2 difference)."""
import copy

import numpy as np
import pytest
import torch

from test_fused_optim_host import OPT_CHOICES

pytestmark = pytest.mark.gpu
H, W, STEPS = 360, 640, 20
BAR = 1e-6


def _make(kind, seed):
    """(params, rgb closure) of one generator, seeded"""
    from aphantasia_b200 import image
    torch.manual_seed(seed)
    if kind == 'fft':
        params, gen, _ = image.fft_image([1, 3, H, W], 0.01, 1.0)
    elif kind == 'dwt':
        params, gen, _ = image.dwt_image([1, 3, H, W], 'coif2', 0.3, 1.)
    else:
        params, gen, _ = image.pixel_image([1, 3, H, W], sd=1.)
    return params, image.to_valid_rgb(gen, colors=1.5)


def _f32_betas(kw):
    return dict(kw, betas=tuple(float(np.float32(b)) for b in kw.get('betas', (0.9, 0.999))))


def _pair(kind, choice, lr=0.05, f32_betas=True):
    """the same generator twice: (params, rgb, ours) and (params, rgb, stock)"""
    from aphantasia_b200 import optim
    cls, kw = OPT_CHOICES[choice]
    kw = _f32_betas(kw) if f32_betas else kw
    pa, fa = _make(kind, 0)
    pb, fb = _make(kind, 0)
    for a, b in zip(pa, pb):
        assert torch.equal(a, b)
    oa = getattr(optim, cls)(pa, lr, **kw)
    ob = {'Adam': optim._stock_adam, 'AdamW': optim._stock_adamw}[cls](pb, lr, **kw)
    return (pa, fa, oa), (pb, fb, ob)


def _grad_out(seed=7):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return torch.randn(1, 3, H, W, device='cuda', generator=g)


def _step(side, grad_out, lr, n_synth=1):
    params, rgb, opt = side
    for group in opt.param_groups:
        group['lr'] = lr
    opt.zero_grad()
    loss = sum((rgb() * grad_out).sum() for _ in range(n_synth))
    loss.backward()
    opt.step()


def _tensors(side):
    params, _, opt = side
    out = {}
    for i, p in enumerate(params):
        out['p%d' % i] = p.detach()
        for k, v in opt.state[p].items():
            if k != 'step':
                out['%s%d' % (k, i)] = v
    return out


def _compare(a, b):
    ta, tb = _tensors(a), _tensors(b)
    assert sorted(ta) == sorted(tb)
    return max(float((ta[k] - tb[k]).abs().max() / tb[k].abs().max().clamp_min(1e-30)) for k in ta)


def _resync(a, b):
    """copies the fused side's parameters and moments into the stock side"""
    with torch.no_grad():
        ta, tb = _tensors(a), _tensors(b)
        for k in ta:
            tb[k].copy_(ta[k])
    for pa, pb in zip(a[0], b[0]):
        assert float(a[2].state[pa]['step']) == float(b[2].state[pb]['step'])


@pytest.mark.parametrize('kind', ['fft', 'dwt', 'pixel'])
@pytest.mark.parametrize('choice', sorted(OPT_CHOICES))
def test_fused_matches_stock_every_step(kind, choice):
    a, b = _pair(kind, choice)
    go = _grad_out()
    worst, start = 0., [p.detach().clone() for p in a[0]]
    for i in range(STEPS):
        lr = 0.05 + (i / STEPS) * (0.01 - 0.05)                  # clip_fft.py --prog: lr0 -> lr1 over the steps (:288-291)
        _step(a, go, lr)
        _step(b, go, lr)
        err = _compare(a, b)
        assert err < BAR, (i, err)
        worst = max(worst, err)
        _resync(a, b)
    assert a[2].fused_steps == STEPS and all(p.grad is None for p in a[0])
    assert all(not torch.equal(p, q) for p, q in zip(a[0], start))
    print('fused vs stock %s %s: max relative error per step %.2e' % (kind, choice, worst))


@pytest.mark.parametrize('kind', ['fft', 'dwt', 'pixel'])
@pytest.mark.parametrize('choice', ['adam', 'adamw_custom'])
def test_scripts_double_betas_differ_by_the_fp32_betas_only(kind, choice):
    """Against torch with the scripts' own betas (0.9 / 0.999 as Python floats): every tensor within 3e-5 of it per step, the
    fp32 betas' 1.3e-5 in 1 - beta2 and what it does to the bias correction (module docstring)."""
    a, b = _pair(kind, choice, f32_betas=False)
    go = _grad_out()
    worst = 0.
    for i in range(STEPS):
        _step(a, go, 0.05)
        _step(b, go, 0.05)
        worst = max(worst, _compare(a, b))
        _resync(a, b)
    print('fused vs stock with double betas %s %s: max relative error per step %.2e' % (kind, choice, worst))
    assert worst < 3e-5


@pytest.mark.parametrize('kind', ['fft', 'dwt', 'pixel'])
def test_lr_edits_take_effect(kind):
    """The same run with lr edited before one step and without: the update of that step scales with the edit."""
    a, b = _pair(kind, 'adam_custom')
    go = _grad_out()
    _step(a, go, 0.05)
    _step(b, go, 0.05)
    _resync(a, b)
    before = [p.detach().clone() for p in a[0]]
    _step(a, go, 0.01)
    _step(b, go, 0.05)
    da = sum(float((p - q).abs().sum()) for p, q in zip(a[0], before))
    db = sum(float((p - q).abs().sum()) for p, q in zip(b[0], before))
    assert abs(da / db - 0.2) < 1e-3, (da, db)


@pytest.mark.parametrize('kind', ['fft', 'dwt', 'pixel'])
@pytest.mark.parametrize('choice', ['adam_custom', 'adamw_custom'])
def test_two_syntheses_take_the_unfused_path(kind, choice):
    """--enforce synthesises twice per step: neither backward is the whole gradient, so step() updates from .grad."""
    a, b = _pair(kind, choice)
    go = _grad_out()
    for i in range(4):
        _step(a, go, 0.05, n_synth=2)
        _step(b, go, 0.05, n_synth=2)
        assert _compare(a, b) < BAR
        _resync(a, b)
    assert a[2].fused_steps == 0
    _step(a, go, 0.05)                                         # one synthesis again: fused
    assert a[2].fused_steps == 1


@pytest.mark.parametrize('kind', ['fft', 'dwt', 'pixel'])
@pytest.mark.parametrize('choice', ['adam', 'adamw_custom'])
def test_load_state_dict_from_stock_continues_the_trajectory(kind, choice):
    """illustrip.py --smooth / illustra.py: a stock optimiser's state_dict loaded into ours (and ours into a stock one) over
    the same parameters continues with the same steps."""
    from aphantasia_b200 import optim
    cls, kw = OPT_CHOICES[choice]
    kw = _f32_betas(kw)
    a, b = _pair(kind, choice)
    go = _grad_out()
    for i in range(5):
        _step(b, go, 0.05)
    with torch.no_grad():
        for p, q in zip(a[0], b[0]):
            p.copy_(q)
    a = (a[0], a[1], getattr(optim, cls)(a[0], 0.05, **kw))
    a[2].load_state_dict(copy.deepcopy(b[2].state_dict()))      # torch's load shares the saved tensors
    for i in range(5):
        _step(a, go, 0.05)
        _step(b, go, 0.05)
        assert _compare(a, b) < BAR
        _resync(a, b)
    assert a[2].fused_steps == 5 and float(a[2].state[a[0][0]]['step']) == 10.
    stock = {'Adam': optim._stock_adam, 'AdamW': optim._stock_adamw}[cls](b[0], 0.05, **kw)
    stock.load_state_dict(copy.deepcopy(a[2].state_dict()))
    b = (b[0], b[1], stock)
    _step(a, go, 0.05)
    _step(b, go, 0.05)
    assert _compare(a, b) < BAR
