"""Env-gated run trace (the reference never prints its loss, SURVEY.md section 5): APH_TRACE=<file.json> makes sim_func
record every similarity value (one D2H read per call -- only when tracing) and, at interpreter exit, writes
{sims, encode_image_calls, launches, wall_s, encode_text_calls, text_tower}. Used by the script-level tests and the logs under profiles/."""
import atexit
import json
import os
import time

PATH = os.environ.get('APH_TRACE')
_state = {'sims': [], 'encodes': 0, 'text_encodes': 0, 'text_tower': 'stand-in', 't0': time.time()}


def enabled():
    return PATH is not None


def sim(value):
    if PATH is not None:
        _state['sims'].append(float(value))


def encode():
    _state['encodes'] += 1


def encode_text():
    _state['text_encodes'] += 1


def text_tower(kind):
    """'cuda' (the text encoder runs in libaphb200.so) or 'stand-in' (seeded embeddings): the last CLIP model built."""
    _state['text_tower'] = kind


def _dump():
    from . import _lib
    out = {'sims': _state['sims'], 'encode_image_calls': _state['encodes'], 'wall_s': time.time() - _state['t0'],
           'launches': int(_lib.lib().aph_launch_count()) if _lib._lib is not None else 0,
           'encode_text_calls': _state['text_encodes'], 'text_tower': _state['text_tower']}
    with open(PATH, 'w') as f:
        json.dump(out, f)


if PATH is not None:
    atexit.register(_dump)
