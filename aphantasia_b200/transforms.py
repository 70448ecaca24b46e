"""Augmentation pipelines -- drop-in for /root/reference/aphantasia/transforms.py (names clip_fft.py reads).

In the reference these are Python closures applied per crop. Here `transforms_fast` and `normalize()` are
*spec-carrying* callables: slice_imgs recognises them and runs the whole pipeline inside the fused CUDA
sampler (csrc/sample.cu). The kornia-based pipelines (custom / elastic / lucent / openai) are outside the
CUDA hot path (SURVEY.md section 2.1) and raise when selected.
"""
import torch

from . import _rng

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)


class SamplerTransform:
    """A transform the fused sampler implements natively. `kind` is one of _rng.TF_*."""

    def __init__(self, kind, name):
        self.kind, self.name = kind, name

    def __call__(self, x):
        # stand-alone use (reference: transform(cut) on a [N,3,s,s] tensor): identity crop through the same kernel
        from .utils import apply_transform_standalone
        return apply_transform_standalone(x, self)

    def __repr__(self):
        return 'SamplerTransform(%s)' % self.name


def normalize():
    """transforms.py:102-109 (CLIP mean/std)."""
    return SamplerTransform(_rng.TF_NORMALIZE, 'normalize')


# transforms.py:165-170: RandomPerspective(0.33, .2) -> RandomErasing(.2) -> random_rotate_fast -> normalize
transforms_fast = SamplerTransform(_rng.TF_FAST, 'fast')


class _Unsupported:
    def __init__(self, name):
        self.name = name

    def __call__(self, x):
        raise NotImplementedError('aphantasia_b200: transform "%s" needs kornia and is outside the CUDA hot path; '
                                  'use --transform fast (default) or none' % self.name)


transforms_custom = _Unsupported('custom')
transforms_elastic = _Unsupported('elastic')
transforms_lucent = _Unsupported('lucent')
transforms_openai = _Unsupported('openai')
device = torch.device('cuda:0' if torch.cuda.is_available() else 'cpu')
