"""Drop-in for taming.modules.diffusionmodules.model: the Decoder -> aphantasia_b200.vqgan.Decoder (forward and d loss / d z on
the GPU; the weights are constants, see that module)."""
from aphantasia_b200.vqgan import AttnBlock, Decoder, ResnetBlock, Upsample  # noqa: F401
