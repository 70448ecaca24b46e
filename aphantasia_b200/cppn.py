"""The CPPN generator of cppn.py (cppn.py:71-116) on libaphb200.so: a per-pixel MLP from the (x, y) coordinate to RGB.

    snet = CPPN(2, nf, layers, 3, act_fn='unbias').cuda()
    img = snet(mgrid)                       # mgrid [N,2,H,W] -> [N,3,H,W]

`ConvLayer` and `CPPN` keep the original's constructor, state-dict keys (`net.{i}.conv.weight` / `.bias`) and random draws, so a
seeded run starts from the original's weights and the script's own `load_cppn` / `export_data` work unchanged. The parameters
stay ordinary nn.Parameters (the script's torch.optim.Adam updates them); the forward and the weight gradient run in CUDA
(csrc/cppn.cu): for nf <= 64 one launch forward, two backward; wider nets run layer by layer as TF32 GEMMs. Supported: nf_in 2,
nf_out 3, nf a multiple of 8 in [8, 256], 1 to 32 layers.
"""
import ctypes as C
import math

import torch
import torch.nn as nn

from . import _trace
from ._lib import Handle, check, lib, require_cuda, stream_ptr

__all__ = ['ConvLayer', 'CPPN']

ACTS = {'unbias': 0, 'comp': 1, 'relu': 2}


class ConvLayer(nn.Module):
    """A 1x1 convolution and the name of its activation, drawn as the original draws it: nn.Conv2d's default init, then
    normal_(0, sqrt(1 / nf_in)) on the weight and uniform_(-.5, .5) on the bias."""

    def __init__(self, nf_in, nf_out, act_fn='relu'):
        super().__init__()
        self.nf_in = nf_in
        self.conv = nn.Conv2d(nf_in, nf_out, 1, 1)
        self.act_name = act_fn if act_fn in ACTS else 'sigmoid'
        with torch.no_grad():
            self.conv.weight.normal_(0., math.sqrt(1. / self.nf_in))
            self.conv.bias.uniform_(-.5, .5)


def _unsupported(what):
    return NotImplementedError('aphantasia_b200.cppn: %s is not supported; supported is CPPN(nf_in=2, nf_hid, num_layers, nf_out=3) '
                               'with nf_hid a multiple of 8 in [8, 256] and 1 <= num_layers <= 32' % what)


class _CppnFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, net, coords, *params):
        x = coords.detach().float().contiguous()
        N, _, H, W = x.shape
        out = torch.empty(N, 3, H, W, device=x.device, dtype=torch.float32)
        ptrs = (C.c_void_p * len(params))(*[p.data_ptr() for p in params])
        check(lib().aph_cppn_fwd(net._handle, x.data_ptr(), N, H, W, ptrs, out.data_ptr(), stream_ptr()), 'aph_cppn_fwd')
        _trace.cppn()
        ctx.net = net
        ctx.save_for_backward(x, *params)
        return out

    @staticmethod
    def backward(ctx, g):
        x, *params = ctx.saved_tensors
        N, _, H, W = x.shape
        g = g.detach().float().contiguous()
        grads = [torch.empty_like(p) for p in params]
        ptrs = (C.c_void_p * len(params))(*[p.data_ptr() for p in params])
        gptrs = (C.c_void_p * len(grads))(*[t.data_ptr() for t in grads])
        check(lib().aph_cppn_bwd(ctx.net._handle, x.data_ptr(), N, H, W, ptrs, g.data_ptr(), gptrs, stream_ptr()), 'aph_cppn_bwd')
        return (None, None) + tuple(grads)


class CPPN(nn.Module):
    """cppn.py's CPPN: layer 0 (nf_in -> nf_hid), num_layers - 1 hidden layers, an output layer with a sigmoid."""

    def __init__(self, nf_in=2, nf_hid=16, num_layers=9, nf_out=3, act_fn='unbias'):
        super().__init__()
        if nf_in != 2:
            raise _unsupported('nf_in = %s' % nf_in)
        if nf_out != 3:
            raise _unsupported('nf_out = %s' % nf_out)
        if act_fn not in ACTS:
            raise _unsupported("act_fn = '%s'" % act_fn)
        self._handle = Handle('aph_cppn', int(nf_hid), int(num_layers), ACTS[act_fn], error=NotImplementedError)
        self.act_fn = act_fn
        nf_hid_in = nf_hid if act_fn == 'relu' else nf_hid * 2
        net = [ConvLayer(nf_in, nf_hid, act_fn)]
        for _ in range(num_layers - 1):
            net.append(ConvLayer(nf_hid_in, nf_hid, act_fn))
        net.append(ConvLayer(nf_hid_in, nf_out, 'sigmoid'))
        self.net = nn.Sequential(*net)

    def _params(self):
        ps = []
        for layer in self.net:
            for p in (layer.conv.weight, layer.conv.bias):
                if not (p.is_cuda and p.dtype == torch.float32 and p.is_contiguous()):
                    raise RuntimeError('aphantasia_b200.cppn: parameters must be contiguous fp32 CUDA tensors (call .cuda() first); '
                                       'there is no CPU path')
                ps.append(p)
        return ps

    def forward(self, coords):
        if not coords.is_cuda:
            coords = coords.cuda()                  # the original moves the coordinates to the GPU (cppn.py:115)
        require_cuda(coords, 'CPPN coordinates')
        if coords.dim() != 4 or coords.shape[1] != 2:
            raise _unsupported('coordinates of shape %s' % (tuple(coords.shape),))
        out = _CppnFn.apply(self, coords, *self._params())
        if not torch.is_grad_enabled():
            from .utils import PreviewTensor
            out = out.as_subclass(PreviewTensor)    # the per-step preview's .cpu() goes through the pinned ring
        return out
