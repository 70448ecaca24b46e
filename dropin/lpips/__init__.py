"""Drop-in for the lpips package -> aphantasia_b200.lpips (clip_fft.py --sync: lpips.LPIPS(net='vgg'))."""
from aphantasia_b200.lpips import *  # noqa: F401,F403
import aphantasia_b200.lpips as _m
globals().update({k: v for k, v in vars(_m).items() if not k.startswith("__")})
