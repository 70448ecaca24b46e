"""The image generators' colour tail and the fp64 block sums, read from the sources: one forward tail kernel and its two adjoints
live in synth_common.cuh, every fp64 block sum that ends in an atomic goes through block_atomic_add_d, and to_valid_rgb hands its
arguments to the generator's own parse."""
import os
import re

from test_device_memory_host import ROOT, _sources
from test_launch_plumbing_host import _function, _outside

KERNEL = re.compile(r'__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s+)?(\w+)\s*\(')


def test_fp64_block_sums_go_through_one_helper():
    srcs = _sources()
    helper = _function(srcs['aph_common.cuh'], 'block_atomic_add_d')
    assert '__shared__ double' in helper and 'warp_sum_d(' in helper and 'atomicAdd(' in helper
    assert 'blockDim.x >> 5' in helper
    rest = _outside(srcs, 'aph_common.cuh', helper)
    # the LPIPS head writes fixed-order per-block partials without atomics: a different determinism contract
    assert [name for name, text in rest.items() if '__shared__ double' in text] == ['lpips.cu']
    calls = {name: len(re.findall(r'\bwarp_sum_d\s*\(', text)) for name, text in rest.items()}
    calls['aph_common.cuh'] -= 1                                          # its definition
    assert {name: n for name, n in calls.items() if n} == {}
    users = {name: text.count('block_atomic_add_d(') for name, text in rest.items() if name != 'aph_common.cuh'}
    assert {name: n for name, n in users.items() if n} == {'synth_common.cuh': 1, 'synth_fft.cu': 1, 'synth_dwt.cu': 2, 'loss.cu': 2}


def test_the_tail_kernels_are_defined_once_in_synth_common():
    defs = {}
    for name, text in _sources().items():
        for m in KERNEL.finditer(text):
            defs.setdefault(m.group(1), []).append(name)
    assert 'k_rgb_fwd' not in defs
    for kernel in ('k_finish', 'k_finish_bwd', 'k_norm_bwd'):
        assert defs.get(kernel) == ['synth_common.cuh'], (kernel, defs.get(kernel))
    assert re.search(r'template <bool NORM>\s*static __global__ void __launch_bounds__\(256\) k_finish\(',
                     _sources()['synth_common.cuh'])


def test_to_valid_rgb_leaves_argument_parsing_to_the_generators():
    text = open(os.path.join(ROOT, 'aphantasia_b200', 'image.py')).read()
    body = re.search(r'\ndef to_valid_rgb\(.*?(?=\n\S)', text, re.S).group(0)
    assert 'PixelImage' not in body and 'fixcontrast' not in body
    assert body.count('isinstance(') == 1 and body.count('.fused(') == 1


def test_generators_parse_the_closures_arguments_and_ignore_extra_ones(monkeypatch):
    """What each generator's synthesis receives from a plain call and through to_valid_rgb, with the autograd Functions
    replaced by recorders (no GPU): shift / contrast (/ fixcontrast) by position or keyword, anything else ignored."""
    import torch
    from aphantasia_b200 import image
    seen = []
    for fn in ('_SynthFFT', '_SynthDWT', '_SynthPixel'):
        monkeypatch.setattr(getattr(image, fn), 'apply', lambda *a: seen.append(a) or torch.zeros(1))
    fft, dwt, pix = (object.__new__(cls) for cls in (image.FFTImage, image.DWTImage, image.PixelImage))
    fft.params, fft.pending_fwd = torch.zeros(1), 0
    dwt.Ys = [torch.zeros(1)]
    pix.image_t = torch.zeros(1)
    cm = list(image._color_matrix_host(1.5))

    def synth(gen, *args, rgb=False, **kwargs):
        """(shift, contrast, fixcontrast, colmat as a list or None, sigmoid) that the call passed to the synthesis"""
        (image.to_valid_rgb(gen, colors=1.5) if rgb else gen)(*args, **kwargs)
        a = seen[-1]
        if gen is fft:
            shift, contrast, fix, colmat, sig = a[2], a[3], None, a[4], a[5]
        elif gen is dwt:
            shift, contrast, fix, colmat, sig = None, a[1], None, a[2], a[3]
        else:
            shift, contrast, fix, colmat, sig = None, a[1], a[2], a[3], a[4]
        return shift, contrast, fix, None if colmat is None else list(colmat), sig

    assert synth(fft) == (None, 1., None, None, False)
    assert synth(fft, 'S', 2., 'extra', nokey=1) == ('S', 2., None, None, False)
    assert synth(fft, contrast=3., rgb=True, fixcontrast=True) == (None, 3., None, cm, True)
    assert synth(fft, 'S', 2., 'extra', rgb=True, colmat=None, sigmoid=False) == ('S', 2., None, cm, True)
    assert synth(dwt, 'S', 2.) == (None, 2., None, None, False)
    assert synth(dwt, 'S', 2., True, rgb=True, sigmoid=0, colmat=None) == (None, 2., None, cm, True)
    assert synth(pix) == (None, 1., False, None, False)
    assert synth(pix, None, 2., True) == (None, 2., True, None, False)
    assert synth(pix, contrast=1., fixcontrast=True, rgb=True) == (None, 1., True, cm, True)
    assert synth(pix, 'S', 2., True, 'extra', rgb=True, other=0) == (None, 2., True, cm, True)
