"""Host-side rules of aphantasia_b200.optim (no GPU): which torch.optim.Adam / AdamW constructions resolve to the fused optimiser,
that the C declarations of the library agree with the ctypes table argument by argument, and that the optimiser's state_dict is
torch's, so state moves between it and the stock optimiser in both directions."""
import ctypes as C
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# the four -opt choices of clip_fft.py:108-115 / illustrip.py:411-418 (illustra.py's adamw is adamw_custom), as constructor calls
OPT_CHOICES = {
    'adam': ('Adam', dict()),
    'adam_custom': ('Adam', dict(betas=(.0, .999))),
    'adamw': ('AdamW', dict(weight_decay=0.01)),
    'adamw_custom': ('AdamW', dict(weight_decay=0.01, betas=(.0, .999), amsgrad=True)),
}


class _Gen:
    """stands in for a generator object: the registry only needs something weakly referable"""


def _generator_params(kind):
    """CPU stand-ins for each generator's parameter list, registered as the generators register them: the spectrum of
    fft_image, the J+1 wavelet tensors of dwt_image (one param group), the picture of pixel_image (its own constructor)."""
    from aphantasia_b200 import image, optim
    if kind == 'pixel':
        t = torch.zeros(1, 3, 4, 6, requires_grad=True)
        return [t], image.PixelImage(t)
    gen = _Gen()
    params = [torch.zeros(1, 3, 4, 4, 2, requires_grad=True)] if kind == 'fft' else \
        [torch.zeros(1, 3, 2, 2, requires_grad=True)] + [torch.zeros(1, 3, 3, 4 >> i, 4 >> i, requires_grad=True) for i in range(2)]
    for p in params:
        optim.register_generator(p, gen)
    return params, gen


@pytest.fixture
def routed(monkeypatch):
    """optim.install() with our two classes replaced by recorders (they need CUDA parameters): yields the list of
    (class name, args, kwargs) of the constructions routed to ours; the stock classes run as they are."""
    from aphantasia_b200 import optim
    made = []
    monkeypatch.setattr(optim, 'Adam', lambda plist, *a, **kw: made.append(('Adam', a, kw)) or 'ours')
    monkeypatch.setattr(optim, 'AdamW', lambda plist, *a, **kw: made.append(('AdamW', a, kw)) or 'ours')
    optim.install()
    try:
        yield made
    finally:
        optim.uninstall()


@pytest.mark.parametrize('kind', ['fft', 'dwt', 'pixel'])
@pytest.mark.parametrize('choice', sorted(OPT_CHOICES))
def test_every_opt_choice_over_every_generator_resolves_to_ours(routed, kind, choice):
    params, gen = _generator_params(kind)
    cls, kw = OPT_CHOICES[choice]
    assert getattr(torch.optim, cls)(params, 0.05, **kw) == 'ours'
    assert routed[-1][0] == cls


@pytest.mark.parametrize('cls,kw', [('Adam', dict(maximize=True)), ('Adam', dict(foreach=True)), ('Adam', dict(fused=True)),
                                    ('Adam', dict(capturable=True)), ('Adam', dict(differentiable=True)),
                                    ('Adam', dict(weight_decay=0.01)), ('AdamW', dict(maximize=True)), ('AdamW', dict(foreach=True)),
                                    ('AdamW', dict(fused=True))])
def test_unsupported_options_resolve_to_stock(routed, cls, kw):
    from aphantasia_b200 import optim
    params, gen = _generator_params('fft')
    opt = getattr(torch.optim, cls)(params, 0.05, **kw)
    assert type(opt) is {'Adam': optim._stock_adam, 'AdamW': optim._stock_adamw}[cls] and routed == []


def test_foreign_and_mixed_parameters_resolve_to_stock(routed):
    """CPPN weights and any tensor that no generator owns keep the stock optimiser, alone or mixed with ours."""
    from aphantasia_b200 import optim
    params, gen = _generator_params('pixel')
    foreign = torch.nn.Linear(2, 2)
    for cls in ('Adam', 'AdamW'):
        stock = {'Adam': optim._stock_adam, 'AdamW': optim._stock_adamw}[cls]
        assert type(getattr(torch.optim, cls)(foreign.parameters(), 0.01)) is stock
        assert type(getattr(torch.optim, cls)(params + [foreign.weight], 0.01)) is stock
        assert type(getattr(torch.optim, cls)([{'params': params}], 0.01)) is stock
    assert routed == []


def test_without_install_nothing_is_routed():
    from aphantasia_b200 import optim
    assert torch.optim.Adam is optim._stock_adam and torch.optim.AdamW is optim._stock_adamw


# ---------------------------------------------------------------------------------------------- the C declarations
_CTYPE = {'int': C.c_int, 'float': C.c_float, 'int64_t': C.c_int64, 'uint64_t': C.c_uint64, 'double': C.c_double}


def _declarations():
    hdr = open(os.path.join(ROOT, 'include', 'aphb200.h')).read()
    hdr = re.sub(r'/\*.*?\*/', ' ', hdr, flags=re.S)
    return {m.group(2): (m.group(1), [a.strip() for a in m.group(3).split(',') if a.strip() and a.strip() != 'void'])
            for m in re.finditer(r'\b(int|int64_t|const char\*)\s+(aph_\w+)\s*\(([^)]*)\)\s*;', hdr)}


def test_header_declarations_match_the_ctypes_table():
    """Every declared entry point has as many arguments in _lib._SIGS as in the header, scalars of the same ctypes type and
    pointers as pointers: a widened declaration that the table missed would read garbage for the new arguments."""
    from aphantasia_b200 import _lib
    decls = _declarations()
    assert set(decls) == set(_lib._SIGS)
    for name, (ret, args) in decls.items():
        res, types = _lib._SIGS[name]
        assert len(types) == len(args), (name, args, types)
        for a, t in zip(args, types):
            if '*' in a:
                # a device address may also travel as a 64-bit integer (aph_allreduce_sym's signal pads)
                assert t in (C.c_void_p, C.c_char_p, C.c_uint64) or issubclass(t, C._Pointer), (name, a, t)
            else:
                base = re.sub(r'\s*\w+$', '', a.replace('const ', '')).strip()
                assert t is _CTYPE[base], (name, a, t)
    for name in ('aph_adam_step', 'aph_synth_fft_bwd_adam', 'aph_pixel_bwd', 'aph_synth_dwt_bwd'):
        args = decls[name][1]
        assert any(re.search(r'\bweight_decay$', a) for a in args) and any(re.search(r'\bvmax$', a) for a in args), name


def test_optional_tails_start_after_the_stream():
    """The Adam arguments of the widened entry points follow `void* stream`: a call of the plain form (ending at the stream)
    is completed with 0 / NULL, which is no decay, no AMSGrad and, for the generator backwards, no update."""
    from aphantasia_b200 import _lib
    decls = _declarations()
    for name, tail in _lib.OPTIONAL_TAIL.items():
        args = decls[name][1]
        assert args[len(args) - len(tail) - 1] == 'void* stream', name
        assert all(v in (None, 0) for v in tail), name


# ---------------------------------------------------------------------------------------------- state_dict
def _filled(opt, seed):
    """gives every parameter of `opt` torch's AdamW/AMSGrad state with seeded values, as after some steps"""
    g = torch.Generator().manual_seed(seed)
    for group in opt.param_groups:
        for p in group['params']:
            opt.state[p] = {'step': torch.tensor(7.), 'exp_avg': torch.randn(p.shape, generator=g),
                            'exp_avg_sq': torch.rand(p.shape, generator=g), 'max_exp_avg_sq': 1 + torch.rand(p.shape, generator=g)}


def _same(a, b):
    assert a['param_groups'] == b['param_groups']
    assert sorted(a['state']) == sorted(b['state'])
    for i in a['state']:
        assert sorted(a['state'][i]) == sorted(b['state'][i])
        for k, v in a['state'][i].items():
            assert torch.equal(v, b['state'][i][k]), (i, k)


@pytest.mark.parametrize('choice', sorted(OPT_CHOICES))
def test_state_dict_round_trip_ours_stock_ours(choice):
    from aphantasia_b200 import optim
    cls, kw = OPT_CHOICES[choice]
    params = [torch.zeros(3, 4), torch.zeros(2, 5)]
    ours = getattr(optim, cls)(params, 0.05, **kw)
    stock = {'Adam': optim._stock_adam, 'AdamW': optim._stock_adamw}[cls](params, 0.05, **kw)
    assert ours.state_dict()['param_groups'] == stock.state_dict()['param_groups']      # same keys and values, before any step
    _filled(ours, 1)
    if not kw.get('amsgrad'):
        for st in ours.state.values():
            del st['max_exp_avg_sq']
    ours._updated.add(id(params[0]))
    sd1 = ours.state_dict()
    assert all('fused_done' not in st and len(st) == (4 if kw.get('amsgrad') else 3) for st in sd1['state'].values())
    stock.load_state_dict(sd1)
    sd2 = stock.state_dict()
    _same(sd1, sd2)
    back = getattr(optim, cls)(params, 0.05, **kw)
    back.load_state_dict(sd2)
    _same(sd1, back.state_dict())
    assert back._updated == set()


def test_state_dict_from_a_stock_run_loads_into_ours():
    """illustrip.py --smooth / illustra.py without the switch on the saving side: a stock AdamW's state after real CPU steps."""
    from aphantasia_b200 import optim
    p = torch.randn(4, 3, requires_grad=True)
    stock = optim._stock_adamw([p], 0.05, weight_decay=0.01, betas=(.0, .999), amsgrad=True)
    for i in range(3):
        p.grad = torch.randn(4, 3)
        stock.step()
    stock.param_groups[0]['lr'] = 0.02                       # a --prog edit travels with the groups
    ours = optim.AdamW([p], 0.05, weight_decay=0.01, betas=(.0, .999), amsgrad=True)
    ours.load_state_dict(stock.state_dict())
    _same(stock.state_dict(), ours.state_dict())
    assert ours.param_groups[0]['lr'] == 0.02 and float(ours.state[p]['step']) == 3.
