"""The per-frame camera motion of illustrip.py on the GPU: torchvision's tensor `affine` as one kernel (csrc/motion.cu).

illustrip.py moves the canvas every frame with frame_transform (illustrip.py:130-138):

    T.functional.affine(img, angle, tuple(shift), scale, shear, fill=0, interpolation=T.InterpolationMode.BILINEAR)

On a CUDA tensor torchvision builds the matrix on the host, uploads it with a blocking pageable copy, materialises a grid,
appends a ones-plane (a copy of the canvas), runs grid_sample and blends with the sampled mask: about ten launches. The
launcher (run.py) installs `affine` below in place of `torchvision.transforms.functional.affine`. It sends a call to
aph_affine_fwd only when the kernel computes exactly that call: a float32 CUDA 4-D contiguous tensor that requires no
gradient, BILINEAR, fill 0 (a number or a list of zeros) and the default centre. Every other call goes to the stock function
unchanged. The inverse matrix comes from torchvision's own _get_inverse_affine_matrix, so it is torchvision's by construction.
"""
import ctypes as C
import numbers

import numpy as np
import torch
import torchvision.transforms.functional as TF
from torchvision.transforms.functional import InterpolationMode

from . import _trace
from ._lib import check, lib, stream_ptr

stock_affine = TF.affine


def _number(x):
    """A Python float from what the script passes: a number, a NumPy scalar or a one-element array (illustrip's scale)."""
    return float(np.asarray(x, dtype=np.float64).reshape(-1)[0]) if isinstance(x, np.ndarray) else float(x)


def _zero_fill(fill):
    if isinstance(fill, numbers.Number):
        return fill == 0
    if isinstance(fill, (list, tuple)):
        return len(fill) > 0 and all(isinstance(v, numbers.Number) and v == 0 for v in fill)
    return False


def _routable(img, interpolation, fill, center):
    return (isinstance(img, torch.Tensor) and img.is_cuda and img.dtype == torch.float32 and img.dim() == 4
            and img.is_contiguous() and not img.requires_grad and interpolation == InterpolationMode.BILINEAR
            and center is None and fill is not None and _zero_fill(fill) and img.numel() > 0)


def inverse_matrix(angle, translate, scale, shear):
    """torchvision's inverse matrix for centre (0, 0), from the argument types the script passes (affine's own
    normalisation of `shear`: a number means [shear, 0], one element means [s, s])."""
    if isinstance(shear, (numbers.Number, np.ndarray)) and np.ndim(shear) == 0:
        shear = [_number(shear), 0.0]
    else:
        shear = [_number(s) for s in shear]
        if len(shear) == 1:
            shear = [shear[0], shear[0]]
    m = TF._get_inverse_affine_matrix([0.0, 0.0], _number(angle), [_number(t) for t in translate], _number(scale), shear)
    return [_number(v) for v in m]


def affine_gpu(img, matrix):
    """out [N,C,H,W] = the kernel's affine warp of img (float32 CUDA, contiguous) by the 6-element inverse matrix."""
    n, c, h, w = img.shape
    out = torch.empty_like(img)
    check(lib().aph_affine_fwd(img.data_ptr(), n * c, h, w, (C.c_double * 6)(*matrix), out.data_ptr(), stream_ptr()),
          'aph_affine_fwd')
    return out


def affine(img, angle, translate, scale, shear, interpolation=InterpolationMode.NEAREST, fill=None, center=None, **kwargs):
    """torchvision.transforms.functional.affine with the kernel under it for the calls it computes exactly."""
    if kwargs or isinstance(interpolation, int) or not _routable(img, interpolation, fill, center):
        return stock_affine(img, angle, translate, scale, shear, interpolation=interpolation, fill=fill, center=center, **kwargs)
    # the stock function's argument checks, so a bad call fails here as it does there
    if not isinstance(angle, (int, float)):
        raise TypeError('Argument angle should be int or float')
    if not isinstance(translate, (list, tuple)) or len(translate) != 2:
        raise TypeError('Argument translate should be a sequence of length 2')
    if scale <= 0.0:
        raise ValueError('Argument scale should be positive')
    _trace.affine()
    return affine_gpu(img, inverse_matrix(angle, translate, scale, shear))


def install():
    """Routes torchvision.transforms.functional.affine (what `T.functional.affine` resolves to at call time) through
    `affine`. Idempotent."""
    if TF.affine is not affine:
        TF.affine = affine
