"""aphantasia_b200 -- H100-native (sm_90a) hot path of eps696/aphantasia behind the reference's own
Python entry points (fft_image, dwt_image, to_valid_rgb, slice_imgs, sim_func, clip model.encode_image).

The package is host glue only: torch owns device memory / streams / autograd plumbing, all arithmetic of
the path runs in hand-written CUDA kernels of libaphb200.so (include/aphb200.h). There is no CPU path.
Put `dropin/` on PYTHONPATH to expose the reference's module names (`aphantasia`, `clip`).
"""
__version__ = '0.1.0'
