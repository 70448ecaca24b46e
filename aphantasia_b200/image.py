"""Image parameterisations -- drop-in for /root/reference/aphantasia/image.py (hot-path entry points).

fft_image / to_valid_rgb keep the reference's signatures and return types (image.py:152-177, 14-29); the
arithmetic runs in libaphb200.so (csrc/synth_fft.cu) through torch.autograd.Function wrappers so that
`loss.backward()` deposits `params[0].grad` exactly as the reference's autograd does.
"""
import ctypes as C
import os

import numpy as np
import torch

from . import _dist, _pool
from ._lib import check, lib, require_cuda, stream_ptr


def _color_matrix_host(colors):
    """Mn[d][c] such that out_d = sum_c Mn[d][c] * img_c  (image.py:15-22: einsum('nchw,cd->ndhw', img, M.T))."""
    m = torch.tensor([[0.26, 0.09, 0.02], [0.27, 0.00, -0.05], [0.27, -0.09, 0.03]])
    m = m / torch.tensor([colors, 1., 1.])
    m = m / m.norm(dim=0).max()
    # colcorr_t = m.T ; out[d] = sum_c img[c] * colcorr_t[c, d] = sum_c m[d, c] * img[c]
    return (C.c_float * 9)(*[float(v) for v in m.reshape(-1)])


def rfft2d_freqs(h, w):
    """image.py:122-128."""
    fy = np.fft.fftfreq(h)[:, None]
    w2 = (w + 1) // 2 if w % 2 == 1 else w // 2 + 1
    fx = np.fft.fftfreq(w)[:w2]
    return np.sqrt(fx * fx + fy * fy)


class _SynthFFT(torch.autograd.Function):
    @staticmethod
    def forward(ctx, params, gen, shift, contrast, colmat, sigmoid):
        require_cuda(params, 'spectrum parameters')
        h, w = gen.h, gen.w
        p = params.detach().contiguous().float()
        x_raw = _pool.empty((3, h, w))
        out = _pool.empty((1, 3, h, w))
        stats = _pool.empty((4,), torch.float64)
        mode, sh = 0, None
        if shift is not None:
            sh = shift.detach().to(p.device, torch.float32).contiguous()
            if sh.numel() == h * gen.wh:
                mode = 1
            elif sh.numel() == 3 * h * gen.wh * 2:
                mode = 2
            else:
                raise ValueError('fft_image: unsupported shift shape %s' % (tuple(shift.shape),))
        check(lib().aph_synth_fft_fwd(gen.plan, p.data_ptr(), gen.scale.data_ptr(), sh.data_ptr() if sh is not None else None, mode,
                                      float(contrast), colmat, int(sigmoid), x_raw.data_ptr(), stats.data_ptr(), out.data_ptr(),
                                      stream_ptr()), 'aph_synth_fft_fwd')
        ctx.gen, ctx.contrast, ctx.colmat, ctx.sigmoid = gen, float(contrast), colmat, int(sigmoid)
        ctx.save_for_backward(x_raw, stats, out)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        x_raw, stats, out = ctx.saved_tensors
        gen = ctx.gen
        g = grad_out.contiguous().float()
        fo = gen.fused_opt
        opt = fo[0]() if (fo is not None and gen.pending_fwd == 1) else None
        if opt is not None:
            # row f2: exactly one grad-tracked synthesis since the last optimizer.step() -> this backward IS the whole gradient of
            # the spectrum; Adam runs in the last FFT pass (dP never leaves registers) and step() finds nothing left to do
            m, v, lr, b1, b2, eps, step = opt._fused_args(fo[1], fo[2])
            p = gen.params
            check(lib().aph_synth_fft_bwd_adam(gen.plan, g.data_ptr(), out.data_ptr(), x_raw.data_ptr(), stats.data_ptr(), gen.scale.data_ptr(),
                                               ctx.contrast, ctx.colmat, ctx.sigmoid, None, p.data_ptr(), m.data_ptr(), v.data_ptr(),
                                               lr, b1, b2, eps, step, stream_ptr()), 'aph_synth_fft_bwd_adam')
            return None, None, None, None, None, None
        gp = _pool.empty((1, 3, gen.h, gen.wh, 2))
        check(lib().aph_synth_fft_bwd(gen.plan, g.data_ptr(), out.data_ptr(), x_raw.data_ptr(), stats.data_ptr(), gen.scale.data_ptr(),
                                      ctx.contrast, ctx.colmat, ctx.sigmoid, gp.data_ptr(), stream_ptr()), 'aph_synth_fft_bwd')
        return gp, None, None, None, None, None


class FFTImage:
    """The `image_f` closure of fft_image (image.py:164-175) as a callable object, so to_valid_rgb can fuse into it."""

    def __init__(self, params, h, w, decay_power):
        self.params, self.h, self.w, self.wh = params, h, w, w // 2 + 1
        freqs = rfft2d_freqs(h, w)
        scale = 1. / np.maximum(freqs, 4. / max(h, w)) ** decay_power      # image.py:159-161 (float64 on the host)
        scale *= np.sqrt(h * w)
        self.scale = torch.tensor(scale).float().contiguous().cuda()
        plan = C.c_void_p()
        check(lib().aph_fft_plan_create(C.byref(plan), h, w), 'aph_fft_plan_create')
        self.plan = plan
        self.fused_opt, self.pending_fwd = None, 0          # aphantasia_b200.optim.Adam hooks in here (row f2)
        from .optim import register_generator
        register_generator(params, self)

    def __del__(self):
        try:
            if getattr(self, 'plan', None):
                lib().aph_fft_plan_destroy(self.plan)
        except Exception:
            pass

    def fused(self, shift, contrast, colmat, sigmoid):
        if torch.is_grad_enabled() and self.params.requires_grad:
            self.pending_fwd += 1
        return _SynthFFT.apply(self.params, self, shift, contrast, colmat, sigmoid)

    def __call__(self, shift=None, contrast=1., *noargs, **nokwargs):
        return self.fused(shift, contrast, None, False)


def resume_fft(resume=None, shape=None, decay=None, colors=1.6, sd=0.01):
    """image.py:130-150. Image-file resume (img2fft) is init-time and out of scope; .pt / tensor resume is kept."""
    size = None
    if resume is None:
        params_shape = [*shape[:3], shape[3] // 2 + 1, 2]
        params = 0.01 * torch.randn(*params_shape)
        if _dist.world() > 1:                      # every rank must start from rank 0's draw
            params = params.cuda(); torch.distributed.broadcast(params, 0)
        params = params.cuda()
    elif isinstance(resume, str):
        if os.path.isfile(resume):
            if os.path.splitext(resume)[1].lower()[1:] in ['jpg', 'png', 'tif', 'bmp']:
                raise NotImplementedError('aphantasia_b200: resuming from an image file (img2fft) is not on the CUDA hot path')
            params = torch.load(resume)
            if isinstance(params, list): params = params[0]
            params = params.detach().cuda()
            params *= sd
        else:
            print(' Snapshot not found:', resume); exit()
    else:
        if isinstance(resume, list): resume = resume[0]
        params = resume.cuda()
    return params, size


def fft_image(shape, sd=0.01, decay_power=1.0, resume=None):
    """Drop-in for image.py:152-177: returns ([spectrum_param], image_f, size)."""
    _dist.init()
    params, size = resume_fft(resume, shape, decay_power, sd=sd)
    spectrum_real_imag_t = params.requires_grad_(True)
    if size is not None: shape[2:] = size
    [h, w] = list(shape[2:])
    return [spectrum_real_imag_t], FFTImage(spectrum_real_imag_t, h, w, decay_power), size


class _SynthPixel(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, contrast, fixcontrast, colmat, sigmoid):
        require_cuda(x, 'pixel parameters')
        xi = x.detach().contiguous().float()
        assert xi.shape[0] == 1 and xi.shape[1] == 3, 'pixel_image expects [1,3,H,W]'
        hw = xi.shape[2] * xi.shape[3]
        out = torch.empty_like(xi)
        stats = torch.empty(4, device=xi.device, dtype=torch.float64)
        check(lib().aph_pixel_fwd(xi.data_ptr(), hw, float(contrast), int(bool(fixcontrast)), colmat, int(sigmoid), stats.data_ptr(),
                                  out.data_ptr(), stream_ptr()), 'aph_pixel_fwd')
        ctx.args = (hw, float(contrast), int(bool(fixcontrast)), colmat, int(sigmoid))
        ctx.save_for_backward(xi, stats, out)
        return out

    @staticmethod
    def backward(ctx, g):
        xi, stats, out = ctx.saved_tensors
        hw, contrast, fix, colmat, sig = ctx.args
        g = g.contiguous().float()
        gx = torch.empty_like(xi)
        check(lib().aph_pixel_bwd(g.data_ptr(), out.data_ptr(), xi.data_ptr(), stats.data_ptr(), hw, contrast, fix, colmat, sig, gx.data_ptr(),
                                  stream_ptr()), 'aph_pixel_bwd')
        return gx, None, None, None, None


class PixelImage:
    """The `image_f` closure of pixel_image (image.py:112-118) as a callable object (fusable by to_valid_rgb)."""

    def __init__(self, image_t):
        self.image_t = image_t

    def fused(self, shift, contrast, colmat, sigmoid, fixcontrast=False):
        return _SynthPixel.apply(self.image_t, contrast, fixcontrast, colmat, sigmoid)

    def __call__(self, shift=None, contrast=1., fixcontrast=False):
        return self.fused(shift, contrast, None, False, fixcontrast)


def pixel_image(shape, resume=None, sd=1., *noargs, **nokwargs):
    """Drop-in for image.py:98-119 (illustrip's default generator): returns ([image_t], image_f, size)."""
    _dist.init()
    size = None
    if resume is None:
        image_t = torch.randn(*shape) * sd
    elif isinstance(resume, str):
        raise NotImplementedError('aphantasia_b200: pixel_image resume from an image file (un_rgb) is init-time, out of the hot path')
    else:
        if isinstance(resume, list): resume = resume[0]
        image_t = resume
    image_t = image_t.cuda()
    if resume is None and _dist.world() > 1:
        torch.distributed.broadcast(image_t, 0)
    image_t = image_t.requires_grad_(True)
    return [image_t], PixelImage(image_t), size


class _ValidRGB(torch.autograd.Function):
    @staticmethod
    def forward(ctx, img, colmat):
        require_cuda(img, 'image')
        x = img.detach().contiguous().float()
        assert x.shape[0] == 1 and x.shape[1] == 3, 'to_valid_rgb expects [1,3,H,W]'
        out = torch.empty_like(x)
        check(lib().aph_valid_rgb_fwd(x.data_ptr(), x.shape[2] * x.shape[3], colmat, out.data_ptr(), stream_ptr()), 'aph_valid_rgb_fwd')
        ctx.colmat = colmat
        ctx.save_for_backward(out)
        return out

    @staticmethod
    def backward(ctx, g):
        out, = ctx.saved_tensors
        g = g.contiguous().float()
        gi = torch.empty_like(out)
        check(lib().aph_valid_rgb_bwd(g.data_ptr(), out.data_ptr(), out.shape[2] * out.shape[3], ctx.colmat, gi.data_ptr(), stream_ptr()),
              'aph_valid_rgb_bwd')
        return gi, None


def _maybe_preview(t):
    """Under torch.no_grad() (the script's preview branch, clip_fft.py:298-299) hand back a tensor whose .cpu() uses the pinned
    read-back ring (utils.PreviewTensor, row f1)."""
    if not torch.is_grad_enabled() and t.is_cuda and not t.requires_grad:
        from .utils import PreviewTensor
        return t.as_subclass(PreviewTensor)
    return t


def to_valid_rgb(image_f, colors=1., decorrelate=True):
    """Drop-in for image.py:14-29. Fuses colour decorrelation + sigmoid into the synthesis kernel when
    `image_f` is one of ours; otherwise applies the stand-alone kernel to whatever image_f returns."""
    colmat = _color_matrix_host(colors) if decorrelate else None

    def inner(*args, **kwargs):
        if isinstance(image_f, (FFTImage, DWTImage, PixelImage)):
            shift = args[0] if len(args) > 0 else kwargs.get('shift', None)
            contrast = args[1] if len(args) > 1 else kwargs.get('contrast', 1.)
            if isinstance(image_f, PixelImage):
                return _maybe_preview(image_f.fused(shift, contrast, colmat, True, args[2] if len(args) > 2 else kwargs.get('fixcontrast', False)))
            return _maybe_preview(image_f.fused(shift, contrast, colmat, True))
        return _ValidRGB.apply(image_f(*args, **kwargs), colmat)
    return inner


class _SynthDWT(torch.autograd.Function):
    @staticmethod
    def forward(ctx, gen, contrast, colmat, sigmoid, *Ys):
        for y in Ys:
            require_cuda(y, 'wavelet parameters')
        ys = [y.detach().contiguous().float() for y in Ys]
        ho, wo = gen.out_hw
        dev = ys[0].device
        x_raw = torch.empty(3, ho, wo, device=dev, dtype=torch.float32)
        out = torch.empty(1, 3, ho, wo, device=dev, dtype=torch.float32)
        stats = torch.empty(4, device=dev, dtype=torch.float64)
        ptrs = (C.c_void_p * len(ys))(*[y.data_ptr() for y in ys])
        check(lib().aph_synth_dwt_fwd(gen.plan, ptrs, gen.scales_c, float(contrast), colmat, int(sigmoid), x_raw.data_ptr(), stats.data_ptr(),
                                      out.data_ptr(), stream_ptr()), 'aph_synth_dwt_fwd')
        ctx.gen, ctx.contrast, ctx.colmat, ctx.sigmoid, ctx.shapes = gen, float(contrast), colmat, int(sigmoid), [tuple(y.shape) for y in Ys]
        ctx.save_for_backward(x_raw, stats, out)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        x_raw, stats, out = ctx.saved_tensors
        gen = ctx.gen
        g = grad_out.contiguous().float()
        grads = [torch.empty(sh, device=g.device, dtype=torch.float32) for sh in ctx.shapes]
        ptrs = (C.c_void_p * len(grads))(*[t.data_ptr() for t in grads])
        check(lib().aph_synth_dwt_bwd(gen.plan, g.data_ptr(), out.data_ptr(), x_raw.data_ptr(), stats.data_ptr(), gen.scales_c, ctx.contrast,
                                      ctx.colmat, ctx.sigmoid, ptrs, stream_ptr()), 'aph_synth_dwt_bwd')
        return (None, None, None, None) + tuple(grads)


class DWTImage:
    """The `image_f` closure of dwt_image (image.py:66-69) as a callable object (fusable by to_valid_rgb)."""

    def __init__(self, shape, wave, sharp):
        from ._wavelets import reconstruction_filters
        h, w = int(shape[2]), int(shape[3])
        rec_lo, rec_hi = reconstruction_filters(wave)
        L = len(rec_lo)
        plan = C.c_void_p()
        check(lib().aph_dwt_plan_create(C.byref(plan), h, w, (C.c_float * L)(*rec_lo), (C.c_float * L)(*rec_hi), L), 'aph_dwt_plan_create')
        self.plan = plan
        J = C.c_int()
        dims = (C.c_int * 32)(); ohw = (C.c_int * 2)()
        check(lib().aph_dwt_plan_levels(plan, C.byref(J), dims, ohw), 'aph_dwt_plan_levels')
        self.J = J.value
        self.level_hw = [(dims[2 * i], dims[2 * i + 1]) for i in range(self.J)]
        self.out_hw = (ohw[0], ohw[1])
        h0, w0 = self.level_hw[0]
        self.scales = [((h0 * w0) / (hh * ww)) ** (1. - sharp) for (hh, ww) in self.level_hw]      # image.py:73-80
        self.scales_c = (C.c_float * self.J)(*[float(v) for v in self.scales])
        self.Ys = None

    def param_shapes(self):
        hJ, wJ = self.level_hw[-1]
        return [(1, 3, hJ, wJ)] + [(1, 3, 3, hh, ww) for (hh, ww) in self.level_hw]

    def __del__(self):
        try:
            if getattr(self, 'plan', None):
                lib().aph_dwt_plan_destroy(self.plan)
        except Exception:
            pass

    def fused(self, shift, contrast, colmat, sigmoid):
        return _SynthDWT.apply(self, contrast, colmat, sigmoid, *self.Ys)

    def __call__(self, shift=None, contrast=1.):
        return self.fused(shift, contrast, None, False)


def dwt_image(shape, wave='coif2', sharp=0.3, colors=1., resume=None):
    """Drop-in for image.py:61-71 / init_dwt :33-59: returns (Ys, image_f, size) with Ys = [Yl, Yh_1 (finest) .. Yh_J]
    ~ N(0,1) leaves. Resume from a .pt list / tensors is kept; image-file resume (img2dwt) is init-time, out of scope."""
    _dist.init()
    gen = DWTImage(shape, wave, sharp)
    if resume is None:
        Ys = [torch.randn(*sh) for sh in gen.param_shapes()]          # same draw order as init_dwt (image.py:42)
        if _dist.world() > 1:
            Ys = [y.cuda() for y in Ys]
            for y in Ys: torch.distributed.broadcast(y, 0)
        Ys = [y.cuda() for y in Ys]
    elif isinstance(resume, str):
        if not os.path.isfile(resume):
            print(' Snapshot not found:', resume); exit()
        if os.path.splitext(resume)[1].lower()[1:] in ['jpg', 'png', 'tif', 'bmp']:
            raise NotImplementedError('aphantasia_b200: resuming from an image file (img2dwt) is not on the CUDA hot path')
        Ys = [y.detach().cuda() for y in torch.load(resume)]
    else:
        Ys = [y.cuda() for y in resume]
    assert [tuple(y.shape) for y in Ys] == gen.param_shapes(), 'dwt_image: parameter shapes do not match this size / wavelet'
    Ys = [y.requires_grad_(True) for y in Ys]
    gen.Ys = Ys
    return Ys, gen, None
