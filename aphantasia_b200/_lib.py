"""ctypes binding of libaphb200.so (the C ABI declared in include/aphb200.h).

The product path has NO fallback: if the CUDA library is missing or a call fails, this raises.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libaphb200.so')

_lib = None

c_f32p = C.c_void_p   # device pointers are passed as integers (tensor.data_ptr())
_SIGS = {
    'aph_version': (C.c_int, []),
    'aph_last_error': (C.c_char_p, []),
    'aph_launch_count': (C.c_int64, []),
    'aph_device_bytes': (C.c_int64, []),
    'aph_fft_plan_create': (C.c_int, [C.POINTER(C.c_void_p), C.c_int, C.c_int]),
    'aph_fft_plan_destroy': (C.c_int, [C.c_void_p]),
    'aph_synth_fft_fwd': (C.c_int, [C.c_void_p, c_f32p, c_f32p, c_f32p, C.c_int, C.c_float, C.c_void_p, C.c_int,
                                    c_f32p, C.c_void_p, c_f32p, C.c_void_p]),
    'aph_synth_fft_bwd': (C.c_int, [C.c_void_p, c_f32p, c_f32p, c_f32p, C.c_void_p, c_f32p, C.c_float, C.c_void_p, C.c_int,
                                    c_f32p, C.c_void_p]),
    'aph_un_rgb': (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_float, c_f32p, C.c_void_p]),
    'aph_fft_analyze': (C.c_int, [C.c_void_p, c_f32p, c_f32p, c_f32p, C.c_void_p]),
    'aph_dwt_analyze': (C.c_int, [C.c_void_p, c_f32p, C.c_void_p, C.c_void_p, C.c_void_p]),
    'aph_dwt_plan_create': (C.c_int, [C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int]),
    'aph_dwt_plan_destroy': (C.c_int, [C.c_void_p]),
    'aph_dwt_plan_levels': (C.c_int, [C.c_void_p, C.POINTER(C.c_int), C.c_void_p, C.c_void_p]),
    'aph_synth_dwt_fwd': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_int, c_f32p, C.c_void_p, c_f32p, C.c_void_p]),
    'aph_synth_dwt_bwd': (C.c_int, [C.c_void_p, c_f32p, c_f32p, c_f32p, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int]),
    'aph_pixel_fwd': (C.c_int, [c_f32p, C.c_int64, C.c_float, C.c_int, C.c_void_p, C.c_int, C.c_void_p, c_f32p, C.c_void_p]),
    'aph_pixel_bwd': (C.c_int, [c_f32p, c_f32p, c_f32p, C.c_void_p, C.c_int64, C.c_float, C.c_int, C.c_void_p, C.c_int, c_f32p, C.c_void_p,
                                c_f32p, c_f32p, c_f32p, c_f32p, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int]),
    'aph_valid_rgb_fwd': (C.c_int, [c_f32p, C.c_int64, C.c_void_p, c_f32p, C.c_void_p]),
    'aph_valid_rgb_bwd': (C.c_int, [c_f32p, c_f32p, C.c_int64, C.c_void_p, c_f32p, C.c_void_p]),
    'aph_affine_fwd': (C.c_int, [c_f32p, C.c_int, C.c_int, C.c_int, C.c_void_p, c_f32p, C.c_void_p]),
    'aph_sample_fwd': (C.c_int, [c_f32p, C.c_int, C.c_int, C.c_int, C.c_int, c_f32p, C.c_int, C.c_int, C.c_int, c_f32p, C.c_void_p]),
    'aph_sample_fwd_patches': (C.c_int, [c_f32p, C.c_int, C.c_int, C.c_int, C.c_int, c_f32p, C.c_int, C.c_int, C.c_int, c_f32p, C.c_void_p, C.c_int,
                                         C.POINTER(C.c_int), C.c_void_p]),
    'aph_sample_bwd_scaled': (C.c_int, [c_f32p, C.c_int, C.c_int, C.c_int, C.c_int, c_f32p, C.c_int, C.c_int, C.c_int, C.c_float, c_f32p, C.c_void_p]),
    'aph_rng_crop_tables': (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.POINTER(C.c_int32), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                      C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, C.c_void_p]),
    'aph_vit_create': (C.c_int, [C.POINTER(C.c_void_p), C.c_void_p]),
    'aph_vit_destroy': (C.c_int, [C.c_void_p]),
    'aph_vit_load_tensor': (C.c_int, [C.c_void_p, C.c_char_p, c_f32p, C.c_int64, C.c_void_p]),
    'aph_vit_finalize': (C.c_int, [C.c_void_p]),
    'aph_vit_fwd': (C.c_int, [C.c_void_p, c_f32p, C.c_int, c_f32p, C.c_int, C.c_void_p]),
    'aph_vit_patch_operand': (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    'aph_vit_fwd_prepatched': (C.c_int, [C.c_void_p, C.c_int, c_f32p, C.c_int, C.c_void_p]),
    'aph_vit_bwd': (C.c_int, [C.c_void_p, c_f32p, C.c_int, c_f32p, C.c_void_p]),
    'aph_vit_fwd_sized': (C.c_int, [C.c_void_p, c_f32p, C.c_int, C.c_int, c_f32p, C.c_int, C.c_void_p]),
    'aph_vit_bwd_sized': (C.c_int, [C.c_void_p, c_f32p, C.c_int, C.c_int, c_f32p, C.c_void_p]),
    'aph_vit_bytes': (C.c_int64, [C.c_void_p]),
    'aph_rn_create': (C.c_int, [C.POINTER(C.c_void_p), C.c_void_p]),
    'aph_rn_destroy': (C.c_int, [C.c_void_p]),
    'aph_rn_load_tensor': (C.c_int, [C.c_void_p, C.c_char_p, c_f32p, C.c_int64, C.c_void_p]),
    'aph_rn_finalize': (C.c_int, [C.c_void_p]),
    'aph_rn_fwd': (C.c_int, [C.c_void_p, c_f32p, C.c_int, C.c_int, c_f32p, C.c_int, C.c_void_p]),
    'aph_rn_bwd': (C.c_int, [C.c_void_p, c_f32p, C.c_int, C.c_int, c_f32p, C.c_void_p]),
    'aph_rn_bytes': (C.c_int64, [C.c_void_p]),
    'aph_rn_saved_test': (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_int64)]),
    'aph_rn_stem_test': (C.c_int, [C.c_int, C.c_void_p, c_f32p, c_f32p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    'aph_rn_pool_test': (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    'aph_rn_tokens_test': (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    'aph_gemm_rn_epi_test': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, c_f32p, C.c_void_p, C.c_void_p, C.c_int,
                                       C.c_void_p, C.c_void_p]),
    'aph_text_create': (C.c_int, [C.POINTER(C.c_void_p), C.c_void_p]),
    'aph_text_destroy': (C.c_int, [C.c_void_p]),
    'aph_text_load_tensor': (C.c_int, [C.c_void_p, C.c_char_p, c_f32p, C.c_int64, C.c_void_p]),
    'aph_text_finalize': (C.c_int, [C.c_void_p]),
    'aph_text_fwd': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, c_f32p, C.c_void_p]),
    'aph_text_bytes': (C.c_int64, [C.c_void_p]),
    'aph_gemm_bf16_tn': (C.c_int, [C.c_void_p, C.c_void_p, c_f32p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    'aph_gemm_epi_test': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, c_f32p, c_f32p, C.c_void_p, C.c_int, c_f32p, C.c_void_p, C.c_void_p,
                                    C.c_int, C.c_int, C.c_void_p]),
    'aph_gemm_epi_strided_test': (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, c_f32p, c_f32p, C.c_int, C.c_void_p,
                                            C.c_int, c_f32p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    'aph_gemm_variant_launches': (C.c_int64, [C.c_int, C.c_int]),
    'aph_attn_test': (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    'aph_attn_long_test': (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    'aph_ln_fwd_test': (C.c_int, [c_f32p, c_f32p, c_f32p, C.c_void_p, c_f32p, c_f32p, C.c_int, C.c_int, C.c_void_p]),
    'aph_ln_bwd_test': (C.c_int, [C.c_void_p, C.c_int, c_f32p, c_f32p, c_f32p, c_f32p, c_f32p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                  C.c_int, c_f32p, C.c_void_p]),
    'aph_prof_gemm': (C.c_int, [C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_int)]),
    'aph_sim_fwd': (C.c_int, [c_f32p, C.c_int, c_f32p, C.c_int, C.c_int, C.c_int, c_f32p, c_f32p, c_f32p, C.c_void_p]),
    'aph_derivat_fwd': (C.c_int, [c_f32p, C.c_int, C.c_int, C.c_int, C.c_void_p, c_f32p, C.c_void_p]),
    'aph_derivat_bwd': (C.c_int, [c_f32p, C.c_int, C.c_int, C.c_int, c_f32p, c_f32p, C.c_void_p]),
    'aph_derivat_sobel_fwd': (C.c_int, [c_f32p, C.c_int, C.c_int, C.c_int, C.c_void_p, c_f32p, C.c_void_p]),
    'aph_derivat_sobel_bwd': (C.c_int, [c_f32p, C.c_int, C.c_int, C.c_int, c_f32p, c_f32p, C.c_void_p]),
    'aph_cppn_create': (C.c_int, [C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_int]),
    'aph_cppn_destroy': (C.c_int, [C.c_void_p]),
    'aph_cppn_bytes': (C.c_int64, [C.c_void_p]),
    'aph_cppn_fwd': (C.c_int, [C.c_void_p, c_f32p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p), c_f32p, C.c_void_p]),
    'aph_cppn_bwd': (C.c_int, [C.c_void_p, c_f32p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p), c_f32p, C.POINTER(C.c_void_p),
                               C.c_void_p]),
    'aph_head_fwd':(C.c_int, [c_f32p, C.c_int, C.c_int, c_f32p, c_f32p, c_f32p, C.c_void_p]),
    'aph_head_bwd': (C.c_int, [c_f32p, c_f32p, C.c_int, C.c_int, c_f32p, C.c_void_p]),
    'aph_synth_fft_bwd_adam': (C.c_int, [C.c_void_p, c_f32p, c_f32p, c_f32p, C.c_void_p, c_f32p, C.c_float, C.c_void_p, C.c_int,
                                         c_f32p, c_f32p, c_f32p, c_f32p, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int, C.c_void_p,
                                         C.c_float, c_f32p]),
    'aph_lpips_create': (C.c_int, [C.POINTER(C.c_void_p)]),
    'aph_lpips_destroy': (C.c_int, [C.c_void_p]),
    'aph_lpips_load_tensor': (C.c_int, [C.c_void_p, C.c_char_p, c_f32p, C.c_int64, C.c_void_p]),
    'aph_lpips_finalize': (C.c_int, [C.c_void_p]),
    'aph_lpips_fwd': (C.c_int, [C.c_void_p, c_f32p, c_f32p, C.c_uint64, C.c_int, C.c_int, C.c_int, C.c_int, c_f32p, C.c_int,
                                C.POINTER(C.c_int64), C.c_void_p]),
    'aph_lpips_bwd': (C.c_int, [C.c_void_p, c_f32p, C.c_int64, c_f32p, C.c_void_p]),
    'aph_lpips_conv_test': (C.c_int, [C.c_int, C.c_void_p, c_f32p, c_f32p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                      C.c_int, C.c_void_p]),
    'aph_lpips_conv0_test': (C.c_int, [C.c_int, C.c_void_p, c_f32p, c_f32p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    'aph_lpips_pool_test': (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    'aph_allreduce_sym': (C.c_int, [C.c_uint64, C.c_void_p, C.c_uint64, C.c_int, C.c_int, C.c_int64, C.c_void_p, C.c_void_p]),
    'aph_adam_step': (C.c_int, [c_f32p, c_f32p, c_f32p, c_f32p, C.c_int64, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int, C.c_void_p,
                                C.c_float, c_f32p]),
}
# Entry points whose last arguments are optional (the fused / extended Adam update): a call that stops after `stream` gets
# these values for them, so a call written for the plain form binds unchanged.
_ADAM_OFF = (None, None, None, None, 0., 0., 0., 0., 0., 0)
OPTIONAL_TAIL = {'aph_adam_step': (0., None), 'aph_synth_fft_bwd_adam': (0., None), 'aph_pixel_bwd': _ADAM_OFF,
                 'aph_synth_dwt_bwd': _ADAM_OFF}
EXPORTS = tuple(_SIGS)


class VitConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ('patch', 'width', 'layers', 'heads', 'out_dim', 'res', 'max_batch', 'reserved')]


class RnConfig(C.Structure):
    _fields_ = [('layers', C.c_int32 * 4)] + [(n, C.c_int32) for n in ('width', 'heads', 'out_dim', 'res', 'max_batch', 'reserved')]


class TextConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ('width', 'layers', 'heads', 'out_dim', 'context', 'vocab', 'max_batch', 'reserved')]


def lib():
    """Loads libaphb200.so once. Raises (never falls back) if it is missing."""
    global _lib
    if _lib is None:
        if not os.path.isfile(LIB_PATH):
            raise RuntimeError('aphantasia_b200: %s not built. Run `python -c "import __graft_entry__ as g; g.build()"` '
                               '(or `make -C aphantasia_b200/csrc`). There is no CPU fallback.' % LIB_PATH)
        l = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGS.items():
            f = getattr(l, name)
            f.restype, f.argtypes = res, args
        for name, tail in OPTIONAL_TAIL.items():
            setattr(l, name, _with_optional_tail(getattr(l, name), tail))
        _lib = l
    return _lib


def _with_optional_tail(f, tail):
    full = len(f.argtypes)

    def call(*args):
        if len(args) == full - len(tail):
            args += tail
        return f(*args)
    call.__name__, call.argtypes, call.restype = f.__name__, f.argtypes, f.restype
    return call


def check(rc, what, error=RuntimeError):
    if rc != 0:
        raise error('%s failed (rc=%d): %s' % (what, rc, lib().aph_last_error().decode('utf-8', 'replace')))


class Handle:
    """One library object `<api>`, made by `<api>_create(&handle, *args)` and owned from then on: close() (or garbage
    collection) destroys it once, after the device's pending work, which may still use it, has finished. ctypes takes it
    wherever the ABI takes the handle. A create that fails raises `error`."""

    def __init__(self, api, *args, error=RuntimeError):
        self.api, self.loaded = api, False
        h = C.c_void_p()
        check(getattr(lib(), api + '_create')(C.byref(h), *args), api + '_create', error)
        self._as_parameter_ = h

    def load(self, state_dict, prefix=''):
        """`<api>_load_tensor` for every fp32 tensor of `state_dict` (key = prefix + its key), then `<api>_finalize`: `loaded`
        once that succeeds. A failed load raises RuntimeError and leaves the handle owned and not loaded."""
        import torch
        load, st = getattr(lib(), self.api + '_load_tensor'), stream_ptr()
        for k, v in state_dict.items():
            d = v.cuda()
            check(load(self, (prefix + k).encode(), d.data_ptr(), d.numel(), st), '%s_load_tensor(%s)' % (self.api, k))
        torch.cuda.current_stream().synchronize()      # the staging copies `d` die with this scope
        check(getattr(lib(), self.api + '_finalize')(self), self.api + '_finalize')
        self.loaded = True

    def close(self):
        h = self.__dict__.pop('_as_parameter_', None)
        self.loaded = False
        if h is not None:
            import torch
            if torch.cuda.is_initialized():
                torch.cuda.synchronize()
            getattr(lib(), self.api + '_destroy')(h)

    def __del__(self):
        try:
            self.close()
        except Exception:          # interpreter shutdown: the modules this needs may be gone
            pass


def stream_ptr():
    import torch
    return torch.cuda.current_stream().cuda_stream


def require_cuda(t, name):
    import torch
    if not (isinstance(t, torch.Tensor) and t.is_cuda):
        raise RuntimeError('aphantasia_b200: %s must be a CUDA tensor; this implementation has no CPU path' % name)
