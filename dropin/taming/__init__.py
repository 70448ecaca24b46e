"""Drop-in `taming` package (CLIP_VQGAN.ipynb: `from taming.modules.diffusionmodules.model import Decoder` and the two quantizers
its VQModel constructs). Only the decoder runs, on aphantasia_b200.vqgan; the encoder and the quantizers' arithmetic are not here."""
