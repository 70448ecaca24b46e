"""Drop-in for taming.modules.vqvae.quantize. CLIP_VQGAN.ipynb constructs a quantizer in its VQModel but never calls it: the
optimised latent goes straight to the decoder. These stand-ins take the constructor's arguments and hold no parameters, so a
checkpoint's `quantize.*` keys are left over by `load_state_dict(strict=False)`. Calling one raises."""
import torch.nn as nn


class _Unsupported(nn.Module):
    def __init__(self, *args, **kwargs):
        super().__init__()
        self.args, self.kwargs = args, kwargs

    def forward(self, *args, **kwargs):
        raise NotImplementedError('%s: the quantizer is a parameter-free stand-in here; only the VQGAN decoder runs on the GPU '
                                  '(the notebook optimises the latent directly and never quantizes it)' % type(self).__name__)


class VectorQuantizer2(_Unsupported):
    """taming's VectorQuantizer2(n_e, e_dim, beta, remap=None, unknown_index='random', sane_index_shape=False, legacy=True)"""


class GumbelQuantize(_Unsupported):
    """taming's GumbelQuantize(num_hiddens, embedding_dim, n_embed, straight_through=True, kl_weight=5e-4, temp_init=1.0,
    use_vqinterface=True, remap=None, unknown_index='random')"""


VectorQuantizer = VectorQuantizer2
