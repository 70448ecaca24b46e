"""Sampler -> encoder hand-over of the patch-embedding operand (SURVEY.md 2.4 k10-k12).

The reference hands `slice_imgs`' fp32 batch to `model.encode_image` (/root/reference/clip_fft.py:250-254); the first thing the
encoder does with it is the im2col of conv1. When exactly one image encoder is alive, it is a ViT and its input resolution is the crop size,
the sampler's last stage writes that bf16 patch-major operand straight into the encoder handle's buffer (aph_sample_fwd_patches)
and stamps the fp32 batch it returns; `encode_image` on that very tensor (same object, not modified in place, no other forward of
the model in between) then skips k_patchify (aph_vit_fwd_prepatched). Anything else -- two encoders (--dualmod), a derived tensor,
APH_PATCH_FUSE=0 -- takes the plain route, with identical results (the operand is the same bf16 rounding of the same fp32 values).
"""
import os
import weakref

import torch

_consumers = weakref.WeakSet()


def register(vis):
    _consumers.add(vis)


def target(size, windowed=False):
    """The one live encoder that will consume [*,3,size,size] batches, or None. windowed: the batch may be larger than the
    encoder's input resolution r by less than one patch (r <= size < r + patch, the size + 8 batches of transforms_custom /
    transforms_elastic): conv1 reads its top-left r x r window, and that window is the operand."""
    if os.environ.get('APH_PATCH_FUSE', '1') == '0':
        return None
    live = list(_consumers)
    if len(live) != 1 or getattr(live[0], 'patch_size', 0) is None:      # a ResNet tower takes no patch operand
        return None
    r = live[0].input_resolution
    if not (r == size or (windowed and r <= size < r + live[0].patch_size)):
        return None
    return live[0]


def stamp(out, vis, S):
    out._aph_patch = (weakref.ref(vis), vis._patch_gen, vis._handle_epoch, out._version, S)


def matches(x, vis):
    st = getattr(x, '_aph_patch', None)
    if st is None:
        return False
    ref, gen, epoch, ver, S = st
    return ref() is vis and gen == vis._patch_gen and epoch == vis._handle_epoch and x._version == ver and x.shape[0] == S \
        and x.dtype == torch.float32 and x.is_contiguous()
