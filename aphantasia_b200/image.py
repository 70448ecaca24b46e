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
from ._lib import Handle, check, lib, require_cuda, stream_ptr


def _color_correlation(colors):
    """The normalised colour matrix m (fp32) of to_valid_rgb / un_rgb; colcorr_t = m.T  (image.py:15-19, 186-190)."""
    m = torch.tensor([[0.26, 0.09, 0.02], [0.27, 0.00, -0.05], [0.27, -0.09, 0.03]])
    m = m / torch.tensor([colors, 1., 1.])
    return m / m.norm(dim=0).max()


def _color_matrix_host(colors):
    """Mn[d][c] such that out_d = sum_c Mn[d][c] * img_c  (image.py:15-22: einsum('nchw,cd->ndhw', img, M.T))."""
    m = _color_correlation(colors)
    # colcorr_t = m.T ; out[d] = sum_c img[c] * colcorr_t[c, d] = sum_c m[d, c] * img[c]
    return (C.c_float * 9)(*[float(v) for v in m.reshape(-1)])


# ---- starting from an image file (image.py:82-107, 130-150, 185-220) ---------------------------------------------------------
def _is_image_file(path):
    """resume_fft's / init_dwt's test (image.py:45, 138): .jpeg and .tiff are not in the list and go to torch.load."""
    return os.path.splitext(path)[1].lower()[1:] in ['jpg', 'png', 'tif', 'bmp']


def _rgb_u8(img):
    """A decoded picture as contiguous uint8 [H,W,3] under utils.img_read's channel rules (grey -> 3 channels, RGBA -> RGB)."""
    img = np.asarray(img)
    if img.dtype != np.uint8:
        raise ValueError('aphantasia_b200: starting from an image needs 8-bit colour (a uint8 array); this one is %s' % img.dtype)
    if img.ndim == 2 or (img.ndim == 3 and img.shape[2] == 1):
        img = np.dstack((img, img, img))
    if img.ndim == 3 and img.shape[2] == 4:
        img = img[:, :, :3]
    if img.ndim != 3 or img.shape[2] != 3:
        raise ValueError('aphantasia_b200: expected a grey, RGB or RGBA picture, got an array of shape %s' % (img.shape,))
    return np.require(img, requirements=['C', 'W'])          # a decoder's read-only buffer is copied: torch shares writable memory only


def _un_rgb(img, colors, gain):
    """gain * un_rgb(img, colors) as a CUDA tensor [1,3,H,W] (aph_un_rgb: one upload of 3 bytes per pixel)."""
    img = _rgb_u8(img)
    h, w = img.shape[:2]
    inv = torch.linalg.inv(_color_correlation(colors).T)           # inv(colcorr_t) in fp32, as image.py:191
    # einsum('nchw,cd->ndhw', x, inv): out_d = sum_c inv[c, d] x_c, so Minv[d][c] = inv[c][d]
    minv = (C.c_float * 9)(*[float(v) for v in inv.T.reshape(-1)])
    src = torch.from_numpy(img).cuda()
    out = torch.empty(1, 3, h, w, device=src.device)
    check(lib().aph_un_rgb(src.data_ptr(), h, w, minv, float(gain), out.data_ptr(), stream_ptr()), 'aph_un_rgb')
    return out


def un_rgb(image, colors=1.):
    """Drop-in for image.py:185-197 on a uint8 HWC picture: CUDA tensor [1,3,H,W]."""
    return _un_rgb(image, colors, 1.)


def _prime_factors(n):
    out, p = [], 2
    while p * p <= n:
        while n % p == 0:
            out.append(p); n //= p
        p += 1
    return out + ([n] if n > 1 else [])


def _check_fft_size(h, w):
    """The FFT generator's lengths are products of primes <= 13: refuse any other picture size before any GPU work."""
    for n in (w, h):
        f = _prime_factors(n)
        if f and f[-1] > 13:
            raise ValueError('%d×%d: %d = %s; the FFT generator needs prime factors ≤ 13; crop or resize the image, or use --dwt'
                             % (w, h, n, '·'.join(str(v) for v in f)))


def _analysis_scale(h, wh, decay, sd):
    """sd * 500000 / un_spectrum's scale, float64 on the host, cast once (image.py:199-206, 218-219, 147). un_spectrum
    recovers w from the half-spectrum width, (wh - 1) * 2: for an odd image width that is W - 1, and so are its frequencies."""
    w = (wh - 1) * 2
    scale = 1. / np.maximum(rfft2d_freqs(h, w), 1. / max(w, h)) ** decay
    scale *= np.sqrt(w * h)
    return torch.tensor(sd * 500000. / scale).float()


def _img2fft(img, decay, colors, sd):
    """sd * img2fft(img, decay, colors): [1,3,H,W//2+1,2] on the GPU (aph_un_rgb, then aph_fft_analyze)."""
    img = _rgb_u8(img)
    h, w = img.shape[:2]
    _check_fft_size(h, w)
    plan = Handle('aph_fft_plan', h, w)
    x = _un_rgb(img, colors, 1.)
    ascale = _analysis_scale(h, w // 2 + 1, decay, sd).cuda()
    spectrum = torch.empty(1, 3, h, w // 2 + 1, 2, device=x.device)
    check(lib().aph_fft_analyze(plan, x.data_ptr(), ascale.data_ptr(), spectrum.data_ptr(), stream_ptr()), 'aph_fft_analyze')
    return spectrum


def img2fft(img_in, decay=1., colors=1.):
    """Drop-in for image.py:208-220: the spectrum parameters [1,3,H,W//2+1,2] (CUDA) of the picture img_in."""
    return _img2fft(img_in, decay, colors, 1.)


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


# ---- one FFT plan per (H, W) and one radial scale per (H, W, decay) for the life of the process. illustrip.py builds a new
# fft_image every frame (illustrip.py:409); a plan of its own would cost four cudaMalloc on creation and four device-synchronising
# cudaFree when the previous frame's generator is dropped, plus an upload of the scale.
# Sharing a plan is safe because no plan buffer carries data from one API call to the next (csrc/synth_fft.cu): the twiddles are
# written once at creation and only read; T and gimg are scratch that every call (aph_synth_fft_fwd / _bwd / _bwd_adam,
# aph_fft_analyze) writes before it reads them within that same call. Calls issued on one stream therefore never see each other's
# scratch, whichever generator issues them; generators sharing a plan must not run their calls concurrently on different streams.
_fft_plans = {}
_fft_scales = {}
fft_plans_created = 0          # plans this process has created for fft_image generators


def _shared_fft_plan(h, w):
    global fft_plans_created
    plan = _fft_plans.get((h, w))
    if plan is None:
        plan = C.c_void_p()
        check(lib().aph_fft_plan_create(C.byref(plan), h, w), 'aph_fft_plan_create')
        _fft_plans[(h, w)] = plan
        fft_plans_created += 1
    return plan


def _shared_fft_scale(h, w, decay_power):
    key = (h, w, float(decay_power))
    scale = _fft_scales.get(key)
    if scale is None:
        freqs = rfft2d_freqs(h, w)
        s = 1. / np.maximum(freqs, 4. / max(h, w)) ** decay_power      # image.py:159-161 (float64 on the host)
        s *= np.sqrt(h * w)
        scale = _fft_scales[key] = torch.tensor(s).float().contiguous().cuda()
    return scale


class _Generator:
    """An `image_f` closure as a callable object. Its fused(colmat, sigmoid, *args, **kwargs) parses the closure's arguments
    and runs the synthesis with to_valid_rgb's colour matrix and sigmoid fused into its last kernel; a plain call has neither."""

    def __call__(self, *args, **kwargs):
        return self.fused(None, False, *args, **kwargs)


class FFTImage(_Generator):
    """The `image_f` closure of fft_image (image.py:164-175) as a callable object, so to_valid_rgb can fuse into it."""

    def __init__(self, params, h, w, decay_power):
        self.params, self.h, self.w, self.wh = params, h, w, w // 2 + 1
        self.scale = _shared_fft_scale(h, w, decay_power)
        self.plan = _shared_fft_plan(h, w)
        self.fused_opt, self.pending_fwd = None, 0          # aphantasia_b200.optim.Adam hooks in here (row f2)
        from .optim import register_generator
        register_generator(params, self)

    def fused(self, colmat, sigmoid, /, shift=None, contrast=1., *noargs, **nokwargs):
        if torch.is_grad_enabled() and self.params.requires_grad:
            self.pending_fwd += 1
        return _SynthFFT.apply(self.params, self, shift, contrast, colmat, sigmoid)


def resume_fft(resume=None, shape=None, decay=None, colors=1.6, sd=0.01):
    """image.py:130-150. An image file is analysed on the GPU with resume_fft's own colors (fft_image passes none) and returns
    its (H, W); every rank computes the same bits from the same file."""
    size = None
    if resume is None:
        params_shape = [*shape[:3], shape[3] // 2 + 1, 2]
        params = 0.01 * torch.randn(*params_shape)
        if _dist.world() > 1:                      # every rank must start from rank 0's draw
            params = params.cuda(); torch.distributed.broadcast(params, 0)
        params = params.cuda()
    elif isinstance(resume, str):
        if os.path.isfile(resume):
            if _is_image_file(resume):
                from .utils import img_read
                img_in = img_read(resume)
                params = _img2fft(img_in, decay, colors, sd)          # `params *= sd` is folded into the analysis scale
                size = img_in.shape[:2]
            else:
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


class PixelImage(_Generator):
    """The `image_f` closure of pixel_image (image.py:112-118) as a callable object (fusable by to_valid_rgb)."""

    def __init__(self, image_t):
        self.image_t = image_t

    def fused(self, colmat, sigmoid, /, shift=None, contrast=1., fixcontrast=False, *noargs, **nokwargs):
        return _SynthPixel.apply(self.image_t, contrast, fixcontrast, colmat, sigmoid)


def pixel_image(shape, resume=None, sd=1., *noargs, **nokwargs):
    """Drop-in for image.py:98-119 (illustrip's default generator): returns ([image_t], image_f, size)."""
    _dist.init()
    size = None
    if resume is None:
        image_t = torch.randn(*shape) * sd
    elif isinstance(resume, str):
        if not os.path.isfile(resume):
            print(' Image not found:', resume); exit()
        from .utils import img_read
        img_in = img_read(resume)
        image_t = _un_rgb(img_in, 2., 3.3)
        size = img_in.shape[:2]
        print(resume, size)
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
        if isinstance(image_f, _Generator):
            return _maybe_preview(image_f.fused(colmat, True, *args, **kwargs))
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


class DWTImage(_Generator):
    """The `image_f` closure of dwt_image (image.py:66-69) as a callable object (fusable by to_valid_rgb)."""

    def __init__(self, shape, wave, sharp):
        from ._wavelets import reconstruction_filters
        h, w = int(shape[2]), int(shape[3])
        rec_lo, rec_hi = reconstruction_filters(wave)
        L = len(rec_lo)
        self.plan = Handle('aph_dwt_plan', h, w, (C.c_float * L)(*rec_lo), (C.c_float * L)(*rec_hi), L)
        J = C.c_int()
        dims = (C.c_int * 32)(); ohw = (C.c_int * 2)()
        check(lib().aph_dwt_plan_levels(self.plan, C.byref(J), dims, ohw), 'aph_dwt_plan_levels')
        self.J = J.value
        self.level_hw = [(dims[2 * i], dims[2 * i + 1]) for i in range(self.J)]
        self.out_hw = (ohw[0], ohw[1])
        self.scales = _dwt_scales(self.level_hw, sharp)
        self.scales_c = (C.c_float * self.J)(*[float(v) for v in self.scales])
        self.Ys = None

    def param_shapes(self):
        hJ, wJ = self.level_hw[-1]
        return [(1, 3, hJ, wJ)] + [(1, 3, 3, hh, ww) for (hh, ww) in self.level_hw]

    def fused(self, colmat, sigmoid, /, shift=None, contrast=1., *noargs, **nokwargs):
        return _SynthDWT.apply(self, contrast, colmat, sigmoid, *self.Ys)


def _dwt_scales(level_hw, sharp):
    """image.py:73-80 from the band sizes, finest first."""
    h0, w0 = level_hw[0]
    return [((h0 * w0) / (hh * ww)) ** (1. - sharp) for (hh, ww) in level_hw]


def dwt_scale(Ys, sharp):
    """Drop-in for image.py:73-80."""
    return _dwt_scales([tuple(y.shape[3:5]) for y in Ys[1:]], sharp)


def _img2dwt(img, gen, colors, sharp=0.3):
    """img2dwt (image.py:82-94) on the plan of `gen`, which has the picture's size: [Yl, Yh_1 .. Yh_J] CUDA tensors, each
    Yh_i divided by its scale at `sharp`."""
    x = _un_rgb(img, colors, 1.)
    Ys = [torch.empty(sh, device=x.device) for sh in gen.param_shapes()]
    inv = (C.c_float * gen.J)(*[1. / s for s in _dwt_scales(gen.level_hw, sharp)])
    ptrs = (C.c_void_p * len(Ys))(*[y.data_ptr() for y in Ys])
    check(lib().aph_dwt_analyze(gen.plan, x.data_ptr(), inv, ptrs, stream_ptr()), 'aph_dwt_analyze')
    return Ys


def img2dwt(img_in, wave='coif2', sharp=0.3, colors=1.):
    """Drop-in for image.py:82-94: the wavelet parameters [Yl, Yh_1 (finest) .. Yh_J] (CUDA) of the picture img_in."""
    img = _rgb_u8(img_in)
    gen = DWTImage([1, 3, *img.shape[:2]], wave, sharp)
    return _img2dwt(img, gen, colors, sharp)


def _init_dwt(resume, shape, wave, sharp, colors):
    """init_dwt (image.py:33-59) with the generator built for the size it settles on, the picture's for an image file:
    (gen, Ys, size). The picture's bands are divided by the scales at init_dwt's sharp = 0.3 whatever `sharp` is."""
    size, img_in = None, None
    if isinstance(resume, str):
        if not os.path.isfile(resume):
            print(' Snapshot not found:', resume); exit()
        if _is_image_file(resume):
            from .utils import img_read
            img_in = _rgb_u8(img_read(resume))
            size = img_in.shape[:2]
            shape = [1, 3, *size]
    gen = DWTImage(shape, wave, sharp)
    if resume is None:
        Ys = [torch.randn(*sh) for sh in gen.param_shapes()]          # same draw order as init_dwt (image.py:42)
        if _dist.world() > 1:
            Ys = [y.cuda() for y in Ys]
            for y in Ys: torch.distributed.broadcast(y, 0)
        Ys = [y.cuda() for y in Ys]
    elif img_in is not None:
        Ys = _img2dwt(img_in, gen, colors)
        print(' loaded image', resume, img_in.shape, 'level', len(Ys) - 1)
    elif isinstance(resume, str):
        Ys = [y.detach().cuda() for y in torch.load(resume)]
    else:
        Ys = [y.cuda() for y in resume]
    return gen, Ys, size


def init_dwt(resume=None, shape=None, wave=None, colors=None):
    """Drop-in for image.py:33-59: (Ys, None, None, size); the pytorch_wavelets transforms it also returns do not exist here."""
    _, Ys, size = _init_dwt(resume, shape, wave, 0.3, colors)
    return Ys, None, None, size


def dwt_image(shape, wave='coif2', sharp=0.3, colors=1., resume=None):
    """Drop-in for image.py:61-71 / init_dwt :33-59: returns (Ys, image_f, size) with Ys = [Yl, Yh_1 (finest) .. Yh_J]
    ~ N(0,1) leaves, or the analysis of an image file at that file's size (returned as `size`), or a .pt list / tensors."""
    _dist.init()
    gen, Ys, size = _init_dwt(resume, shape, wave, sharp, colors)
    assert [tuple(y.shape) for y in Ys] == gen.param_shapes(), 'dwt_image: parameter shapes do not match this size / wavelet'
    Ys = [y.requires_grad_(True) for y in Ys]
    gen.Ys = Ys
    return Ys, gen, size
