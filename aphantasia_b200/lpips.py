"""LPIPS (lpips v0.1, net='vgg') on libaphb200.so: the image-composition loss of clip_fft.py --sync (clip_fft.py:220,270).

    sim_loss = lpips.LPIPS(net='vgg', verbose=False).cuda()
    loss += w * sim_loss(F.interpolate(img_out, sim_size, ...), img_in, normalize=True).squeeze()

Supported: net='vgg', lpips=True, spatial=False, in0 and in1 of one shape [N,3,H,W] (H, W >= 16), fp32 or fp64, gradient with
respect to in0. The value and the data gradient run in CUDA (csrc/lpips.cu): VGG16 in bf16 on wgmma, conv1_1 and the head in fp32.

Weights: torchvision's VGG16 state dict from $APH_LPIPS_VGG or torch.hub's checkpoint cache (vgg16-397923af.pth), the lpips
linear layers from $APH_LPIPS_LIN (lpips' weights/v0.1/vgg.pth). Without them, seeded synthetic weights are used, loudly.
"""
import os
from ctypes import c_int64 as C_int64, c_void_p as C_void_p

import torch

from . import _trace
from ._lib import check, lib, require_cuda, stream_ptr

__all__ = ['LPIPS']

VGG_CONVS = (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28)          # torchvision vgg16().features indices of the 13 convolutions
VGG_CH = ((3, 64), (64, 64), (64, 128), (128, 128), (128, 256), (256, 256), (256, 256), (256, 512), (512, 512), (512, 512),
          (512, 512), (512, 512), (512, 512))
TAP_CH = (64, 128, 256, 512, 512)                                     # relu1_2, relu2_2, relu3_3, relu4_3, relu5_3
SHIFT = (-.030, -.088, -.188)
SCALE = (.458, .448, .450)
VGG_CHECKPOINT = 'vgg16-397923af.pth'


def _log(msg):
    print(' [aphantasia_b200] ' + msg)


def vgg_state_dict_path():
    """$APH_LPIPS_VGG, else torchvision's cached checkpoint under torch.hub.get_dir(), else None."""
    p = os.environ.get('APH_LPIPS_VGG')
    if p:
        return p if os.path.isfile(p) else None
    p = os.path.join(torch.hub.get_dir(), 'checkpoints', VGG_CHECKPOINT)
    return p if os.path.isfile(p) else None


def synthetic_vgg_state_dict(seed=0):
    """torchvision's VGG initialisation (kaiming_normal_, fan_out, relu; zero bias) under a private generator: the global RNG,
    which the script's crop draws replay, is untouched."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for i, (ci, co) in zip(VGG_CONVS, VGG_CH):
        sd['features.%d.weight' % i] = torch.randn(co, ci, 3, 3, generator=g) * (2.0 / (co * 9)) ** 0.5
        sd['features.%d.bias' % i] = torch.zeros(co)
    return sd


def synthetic_lin_state_dict(seed=1):
    """Non-negative linear weights (lpips trains its lin layers under a clamp at zero) of mean 1/C per tap."""
    g = torch.Generator().manual_seed(seed)
    return {'lin%d.model.1.weight' % t: (torch.rand(1, c, 1, 1, generator=g) * (2.0 / c)) for t, c in enumerate(TAP_CH)}


def load_vgg_state_dict():
    """(state dict of the 13 convolutions, synthetic?) -- only `features.{i}.weight|bias` of the conv layers are kept."""
    p = vgg_state_dict_path()
    if p is None:
        _log('no VGG16 weights ($APH_LPIPS_VGG or %s in the torch hub cache) available: LPIPS uses seeded synthetic VGG16 weights'
             % VGG_CHECKPOINT)
        return synthetic_vgg_state_dict(), True
    sd = torch.load(p, map_location='cpu')
    keep = {}
    for i, (ci, co) in zip(VGG_CONVS, VGG_CH):
        for kind, shape in (('weight', (co, ci, 3, 3)), ('bias', (co,))):
            k = 'features.%d.%s' % (i, kind)
            if k not in sd or tuple(sd[k].shape) != shape:
                raise ValueError('LPIPS: %s lacks %s of shape %s' % (p, k, shape))
            keep[k] = sd[k].float()
    return keep, False


def load_lin_state_dict():
    """(lin{t}.model.1.weight [1,C,1,1] for t = 0..4, synthetic?) from $APH_LPIPS_LIN."""
    p = os.environ.get('APH_LPIPS_LIN')
    if not p or not os.path.isfile(p):
        _log('no LPIPS linear weights ($APH_LPIPS_LIN, lpips weights/v0.1/vgg.pth) available: LPIPS uses seeded synthetic '
             'non-negative linear weights')
        return synthetic_lin_state_dict(), True
    sd = torch.load(p, map_location='cpu')
    keep = {}
    for t, c in enumerate(TAP_CH):
        k = 'lin%d.model.1.weight' % t
        if k not in sd or tuple(sd[k].shape) != (1, c, 1, 1):
            raise ValueError('LPIPS: %s lacks %s of shape (1, %d, 1, 1)' % (p, k, c))
        keep[k] = sd[k].float()
    return keep, False


def _unsupported(what):
    return NotImplementedError('aphantasia_b200.lpips: %s is not supported; supported is LPIPS(net=\'vgg\', lpips=True, '
                               'spatial=False) on two [N,3,H,W] fp32 / fp64 CUDA tensors of one shape, differentiable in in0' % what)


class _LPIPSFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, in0, in1, model, normalize):
        out = model._forward(in0, in1, normalize, save=in0.requires_grad)
        ctx.model, ctx.generation, ctx.shape, ctx.dtype = model, model._last_generation, tuple(in0.shape), in0.dtype
        return out

    @staticmethod
    def backward(ctx, g):
        m = ctx.model
        g = g.detach().reshape(-1).float().contiguous()
        gi = torch.empty(ctx.shape, device=g.device, dtype=torch.float32)
        check(lib().aph_lpips_bwd(m._handle, g.data_ptr(), ctx.generation, gi.data_ptr(), stream_ptr()), 'aph_lpips_bwd')
        return gi.to(ctx.dtype), None, None, None


class LPIPS:
    """lpips.LPIPS with the upstream signature. Only net='vgg', lpips=True, spatial=False run; everything else raises."""

    def __init__(self, pretrained=True, net='alex', version='0.1', lpips=True, spatial=False, pnet_rand=False, pnet_tune=False,
                 use_dropout=True, model_path=None, eval_mode=True, verbose=True, vgg_state_dict=None, lin_state_dict=None):
        if net != 'vgg':
            raise _unsupported("net='%s'" % net)
        if not lpips:
            raise _unsupported('lpips=False (the baseline without linear layers)')
        if spatial:
            raise _unsupported('spatial=True')
        if version != '0.1':
            raise _unsupported("version='%s'" % version)
        if vgg_state_dict is None:
            vgg_state_dict, self.synthetic_vgg = load_vgg_state_dict()
        else:
            self.synthetic_vgg = False
        if lin_state_dict is None:
            lin_state_dict, self.synthetic_lin = load_lin_state_dict()
        else:
            self.synthetic_lin = False
        self._sd = {k: v.detach().float().contiguous() for k, v in list(vgg_state_dict.items()) + list(lin_state_dict.items())
                    if k.startswith('lin') or any(k == 'features.%d.%s' % (i, t) for i in VGG_CONVS for t in ('weight', 'bias'))}
        self._handle = None
        self._ref = None                      # (key tuple, the tensor itself: keeps its storage from being reused under the key)
        self._last_generation = -1
        if verbose:
            print('Setting up [LPIPS] perceptual loss: trunk [vgg], v[%s], spatial [off]' % version)

    def _ensure(self):
        if self._handle is not None:
            return
        h = C_void_p()
        check(lib().aph_lpips_create(h), 'aph_lpips_create')
        self._handle = h.value
        st = stream_ptr()
        for k, v in self._sd.items():
            d = v.cuda()
            check(lib().aph_lpips_load_tensor(self._handle, k.encode(), d.data_ptr(), d.numel(), st), 'aph_lpips_load_tensor')
            torch.cuda.current_stream().synchronize()           # `d` dies with this iteration
        check(lib().aph_lpips_finalize(self._handle), 'aph_lpips_finalize')

    def __del__(self):
        h = getattr(self, '_handle', None)
        if h is not None and lib is not None:
            try:
                torch.cuda.synchronize()
                lib().aph_lpips_destroy(h)
            except Exception:
                pass
            self._handle = None

    # nn.Module surface used by the scripts
    def cuda(self, *a, **k): return self
    def eval(self): return self
    def to(self, *a, **k): return self
    def train(self, mode=True): return self
    def requires_grad_(self, flag=True): return self
    def parameters(self): return iter(())

    def _forward(self, in0, in1, normalize, save):
        self._ensure()
        N, _, H, W = in0.shape
        key = (in1.data_ptr(), tuple(in1.shape), tuple(in1.stride()), in1._version, in1.dtype, in1.device, bool(normalize))
        if self._ref is not None and self._ref[0] == key:
            ref_ptr, ref_key = 0, self._ref[2]
        else:
            x1 = in1.detach().float().contiguous()
            self._ref = (key, in1, (hash(key) & 0x7FFFFFFFFFFFFFFF) | 1)
            ref_ptr, ref_key = x1.data_ptr(), self._ref[2]
        x0 = in0.detach().float().contiguous()
        out = torch.empty(N, device=in0.device, dtype=torch.float32)
        gen = C_int64()
        check(lib().aph_lpips_fwd(self._handle, x0.data_ptr(), ref_ptr, ref_key, N, H, W, int(bool(normalize)), out.data_ptr(),
                                  int(save), gen, stream_ptr()), 'aph_lpips_fwd')
        if ref_ptr:
            x1.record_stream(torch.cuda.current_stream())
        self._last_generation = gen.value
        _trace.lpips()
        return out.reshape(N, 1, 1, 1).to(in0.dtype)

    def forward(self, in0, in1, retPerLayer=False, normalize=False):
        if retPerLayer:
            raise _unsupported('retPerLayer=True')
        for name, t in (('in0', in0), ('in1', in1)):
            if not isinstance(t, torch.Tensor) or t.dtype not in (torch.float32, torch.float64):
                raise _unsupported('%s of type %s' % (name, getattr(t, 'dtype', type(t).__name__)))
            if t.dim() != 4 or t.shape[1] != 3:
                raise _unsupported('%s of shape %s' % (name, tuple(t.shape)))
        if in0.shape != in1.shape:
            raise _unsupported('inputs of different shapes %s and %s' % (tuple(in0.shape), tuple(in1.shape)))
        if torch.is_grad_enabled() and in1.requires_grad:
            raise _unsupported('a gradient with respect to in1')
        require_cuda(in0, 'LPIPS in0')
        require_cuda(in1, 'LPIPS in1')
        if in0.shape[2] < 16 or in0.shape[3] < 16:
            raise ValueError('LPIPS: images of %dx%d are below VGG16\'s 16x16' % tuple(in0.shape[2:]))
        return _LPIPSFn.apply(in0, in1, self, bool(normalize))

    __call__ = forward

