"""eps.progress_bar -> aphantasia_b200.progress_bar. Its last upd() waits for the asynchronous JPEG writes, before cppn.py reads the
frame directory (cppn.py:314)."""
from aphantasia_b200.progress_bar import *  # noqa: F401,F403
import aphantasia_b200.progress_bar as _m
globals().update({k: v for k, v in vars(_m).items() if not k.startswith("__")})
