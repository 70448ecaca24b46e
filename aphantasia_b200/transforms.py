"""Augmentation pipelines -- drop-in for /root/reference/aphantasia/transforms.py (names clip_fft.py reads).

In the reference these are Python closures applied per crop. Here `transforms_fast`, `transforms_custom`,
`transforms_elastic` and `normalize()` are *spec-carrying* callables: slice_imgs recognises them and runs the whole
pipeline inside the fused CUDA sampler (csrc/sample.cu). `transforms_custom` and `transforms_elastic` pad each crop
by 4 pixels, so slice_imgs returns [count, 3, size + 8, size + 8] with them, as the reference does; the reference
builds their rotation, elastic and jitter stages on kornia, which the sampler restates (DESIGN.md section 1).
`transforms_lucent` / `transforms_openai` are selected by no script and raise.
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
# transforms.py:156-163: pad(4, constant 0.5) -> random_rotate -> jitter(8) -> normalize
transforms_custom = SamplerTransform(_rng.TF_CUSTOM, 'custom')
# transforms.py:147-154: pad(4, constant 0.5) -> RandomErasing(.2) -> random_rotate -> random_elastic -> jitter(8) -> normalize
transforms_elastic = SamplerTransform(_rng.TF_ELASTIC, 'elastic')


class _Unsupported:
    def __init__(self, name):
        self.name = name

    def __call__(self, x):
        raise NotImplementedError('aphantasia_b200: transform "%s" is not implemented in the fused sampler; '
                                  'use --transform fast (default), custom, elastic or none' % self.name)


transforms_lucent = _Unsupported('lucent')
transforms_openai = _Unsupported('openai')
device = torch.device('cuda:0' if torch.cuda.is_available() else 'cpu')
