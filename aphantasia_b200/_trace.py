"""Env-gated run trace (the reference never prints its loss, SURVEY.md section 5): APH_TRACE=<file.json> makes sim_func
record every similarity value (one D2H read per call -- only when tracing) and, at interpreter exit, writes
{sims, encode_image_calls, launches, wall_s, encode_text_calls, text_tower, lpips_calls, affine_calls,
cppn_calls, optim_steps_fused, optim_steps_unfused}. Used by the script-level tests and the logs under profiles/."""
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


def lpips():
    _state['lpips'] = _state.get('lpips', 0) + 1


def affine():
    _state['affine'] = _state.get('affine', 0) + 1


def cppn():
    _state['cppn'] = _state.get('cppn', 0) + 1


def optim_step(fused):
    """One update by aphantasia_b200.optim: of a generator's parameters inside its synthesis backward (fused), or of one
    parameter in step() (unfused)."""
    k = 'optim_fused' if fused else 'optim_unfused'
    _state[k] = _state.get(k, 0) + 1


def text_tower(kind):
    """'cuda' (the text encoder runs in libaphb200.so) or 'stand-in' (seeded embeddings): the last CLIP model built."""
    _state['text_tower'] = kind


def _dump():
    from . import _lib
    out = {'sims': _state['sims'], 'encode_image_calls': _state['encodes'], 'wall_s': time.time() - _state['t0'],
           'launches': int(_lib.lib().aph_launch_count()) if _lib._lib is not None else 0,
           'encode_text_calls': _state['text_encodes'], 'text_tower': _state['text_tower'], 'lpips_calls': _state.get('lpips', 0),
           'affine_calls': _state.get('affine', 0), 'cppn_calls': _state.get('cppn', 0),
           'optim_steps_fused': _state.get('optim_fused', 0), 'optim_steps_unfused': _state.get('optim_unfused', 0)}
    with open(PATH, 'w') as f:
        json.dump(out, f)


if PATH is not None:
    atexit.register(_dump)
