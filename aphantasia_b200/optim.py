"""Adam and AdamW behind torch.optim's interface, running in libaphb200.so (SURVEY.md 8 row f2).

The scripts build one of four optimisers over the generator's parameters (clip_fft.py:108-115, illustrip.py:411-418,
illustra.py:282-285) and call zero_grad() / loss.backward() / step() per iteration:
    -opt adam          torch.optim.Adam(params, lr)
    -opt adam_custom   torch.optim.Adam(params, lr, betas=(.0, .999))
    -opt adamw         torch.optim.AdamW(params, lr, weight_decay=0.01)
    -opt adamw_custom  torch.optim.AdamW(params, lr, weight_decay=0.01, betas=(.0, .999), amsgrad=True)   (illustra.py's adamw)
`Adam` / `AdamW` here keep that interface (param_groups with a mutable 'lr' -- the --prog schedule writes it,
clip_fft.py:288-291 --, zero_grad, step, and torch's own state_dict / load_state_dict layout, which the video scripts use to carry
the moments from frame to frame and line to line) and run torch's update rule (csrc/adam.cuh). When exactly one grad-tracked
synthesis of the parameters' generator -- fft_image, dwt_image or pixel_image -- ran since the last step(), the update is fused
into that synthesis' backward, where the gradient is formed: the gradient is never written and step() launches nothing. Otherwise
(--enforce synthesises twice per step) step() updates each parameter in one launch (aph_adam_step).

Opt-in for an unmodified script: `APH_FUSED_ADAM=1 python -m aphantasia_b200.run clip_fft.py ...` makes `torch.optim.Adam` and
`torch.optim.AdamW` resolve to these classes when (and only when) every parameter belongs to one of our generators and no
unsupported option (maximize, capturable, differentiable, foreach, fused, or Adam's coupled weight_decay) is set; anything else --
CPPN weights included -- gets the stock optimiser.
"""
import weakref

import torch

from . import _trace
from ._lib import check, lib, stream_ptr

_GENERATORS = weakref.WeakValueDictionary()        # id(param tensor) -> FFTImage / DWTImage / PixelImage
_UNSUPPORTED = ('maximize', 'capturable', 'differentiable', 'foreach', 'fused')


def register_generator(param, gen):
    _GENERATORS[id(param)] = gen


class Adam(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False, *,
                 decoupled_weight_decay=False, **unsupported):
        if any(unsupported.get(k) for k in _UNSUPPORTED) or set(unsupported) - set(_UNSUPPORTED) or \
                (weight_decay != 0 and not decoupled_weight_decay):
            raise NotImplementedError('aphantasia_b200.optim: Adam / AdamW with decoupled weight_decay and amsgrad only '
                                      '(no coupled weight_decay, maximize, capturable, differentiable, foreach, fused)')
        defaults = dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay, amsgrad=bool(amsgrad), maximize=False,
                        foreach=None, capturable=False, differentiable=False, fused=None,
                        decoupled_weight_decay=bool(decoupled_weight_decay))
        super().__init__(params, defaults)
        self.fused_steps = 0
        self._updated = set()          # id(p) of parameters a synthesis backward updated since the last step(); never saved
        gens = {id(g): g for g in (_GENERATORS.get(id(p)) for group in self.param_groups for p in group['params']) if g is not None}
        for gen in gens.values():
            gen.fused_opt = weakref.ref(self)

    def _state(self, p, group):
        """torch's per-parameter state, created on first use as torch does: step (a CPU fp32 tensor), exp_avg, exp_avg_sq and,
        with amsgrad, max_exp_avg_sq."""
        if not (p.is_cuda and p.dtype == torch.float32 and p.is_contiguous()):
            raise RuntimeError('aphantasia_b200.optim: parameters must be contiguous fp32 CUDA tensors')
        st = self.state[p]
        if not st:
            st['step'] = torch.tensor(0.)
            st['exp_avg'] = torch.zeros_like(p, memory_format=torch.contiguous_format)
            st['exp_avg_sq'] = torch.zeros_like(p, memory_format=torch.contiguous_format)
        if group['amsgrad'] and 'max_exp_avg_sq' not in st:
            st['max_exp_avg_sq'] = torch.zeros_like(p, memory_format=torch.contiguous_format)
        for k in ('exp_avg', 'exp_avg_sq', 'max_exp_avg_sq'):
            if k in st and not st[k].is_contiguous():
                st[k] = st[k].contiguous()
        return st

    def _scalars(self, group, step):
        b1, b2 = group['betas']
        return float(group['lr']), float(b1), float(b2), float(group['eps']), float(group['weight_decay']), int(step)

    def _fused_args(self, params):
        """Called from a synthesis backward that holds the whole gradient of `params` (its generator's parameters, one
        grad-tracked synthesis since the last step()): advances their state by one step and returns
        ([(p, exp_avg, exp_avg_sq, max_exp_avg_sq or None)], (lr, b1, b2, eps, weight_decay, step)) for the kernel, or None
        when they cannot take one update together (not all in one group of this optimiser, or at different steps)."""
        group = next((g for g in self.param_groups if any(q is params[0] for q in g['params'])), None)
        if group is None or not all(any(q is p for q in group['params']) for p in params):
            return None
        sts = [self._state(p, group) for p in params]
        if len({float(st['step']) for st in sts}) != 1:
            return None
        for p, st in zip(params, sts):
            st['step'] += 1
            self._updated.add(id(p))
        self.fused_steps += 1
        _trace.optim_step(fused=True)
        return ([(p, st['exp_avg'], st['exp_avg_sq'], st.get('max_exp_avg_sq')) for p, st in zip(params, sts)],
                self._scalars(group, sts[0]['step']))

    @torch.no_grad()
    def step(self, closure=None):
        loss = closure() if closure is not None else None
        for group in self.param_groups:
            for p in group['params']:
                gen = _GENERATORS.get(id(p))
                if gen is not None:
                    gen.pending_fwd = 0
                if id(p) in self._updated:          # the update already happened inside the synthesis backward
                    self._updated.discard(id(p))
                    continue
                if p.grad is None:
                    continue
                st = self._state(p, group)
                st['step'] += 1
                lr, b1, b2, eps, wd, step = self._scalars(group, st['step'])
                g = p.grad.contiguous()
                vmax = st.get('max_exp_avg_sq') if group['amsgrad'] else None
                check(lib().aph_adam_step(p.data_ptr(), g.data_ptr(), st['exp_avg'].data_ptr(), st['exp_avg_sq'].data_ptr(), p.numel(),
                                          lr, b1, b2, eps, step, stream_ptr(), wd, vmax.data_ptr() if vmax is not None else None),
                      'aph_adam_step')
                _trace.optim_step(fused=False)
        return loss


class AdamW(Adam):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, amsgrad=False, **unsupported):
        super().__init__(params, lr, betas, eps, weight_decay, amsgrad, decoupled_weight_decay=True, **unsupported)


_stock_adam, _stock_adamw = torch.optim.Adam, torch.optim.AdamW


def _ours(plist, weight_decay, decoupled, kw):
    supported = not any(kw.get(k) for k in _UNSUPPORTED) and not set(kw) - set(_UNSUPPORTED) and (decoupled or weight_decay == 0)
    return supported and len(plist) > 0 and all(isinstance(p, torch.Tensor) and id(p) in _GENERATORS for p in plist)


def _adam_factory(params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False, **kw):
    plist = list(params)
    if _ours(plist, weight_decay, kw.get('decoupled_weight_decay', False), {k: v for k, v in kw.items() if k != 'decoupled_weight_decay'}):
        return Adam(plist, lr, betas, eps, weight_decay, amsgrad, decoupled_weight_decay=bool(kw.get('decoupled_weight_decay')))
    return _stock_adam(plist, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=amsgrad, **kw)


def _adamw_factory(params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, amsgrad=False, **kw):
    plist = list(params)
    if _ours(plist, weight_decay, True, kw):
        return AdamW(plist, lr, betas, eps, weight_decay, amsgrad)
    return _stock_adamw(plist, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=amsgrad, **kw)


def install():
    """Routes torch.optim.Adam(...) / AdamW(...) over our generators' parameters to the fused implementation (APH_FUSED_ADAM=1)."""
    torch.optim.Adam, torch.optim.AdamW = _adam_factory, _adamw_factory


def uninstall():
    torch.optim.Adam, torch.optim.AdamW = _stock_adam, _stock_adamw
