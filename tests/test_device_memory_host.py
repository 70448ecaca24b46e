"""Device-memory ownership, read from the sources: only the owner types of csrc/aph_common.cuh (DeviceAllocs, Scratch,
StreamTemp) allocate or free device memory, so every handle, plan and temporary gives back what it took on every path, and
aph_device_bytes() can count all of it."""
import os
import re

from aphantasia_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'aphantasia_b200', 'csrc')
ALLOC = re.compile(r'\bcuda(Malloc|Free)(Async)?\b')


def _sources():
    """{file name: its text without comments} for every CUDA source of the library"""
    out = {}
    for name in sorted(os.listdir(CSRC)):
        if name.endswith(('.cu', '.cuh')):
            text = open(os.path.join(CSRC, name)).read()
            out[name] = re.sub(r'//[^\n]*|/\*.*?\*/', '', text, flags=re.S)
    return out


def _body(text, start):
    """the brace-balanced body of the function whose signature begins at `start`"""
    i = text.index('{', start)
    depth = 0
    for j in range(i, len(text)):
        depth += {'{': 1, '}': -1}.get(text[j], 0)
        if depth == 0:
            return text[i:j + 1]
    raise AssertionError('unbalanced braces after offset %d' % start)


def test_device_memory_is_allocated_and_freed_only_by_the_owner_types():
    srcs = _sources()
    assert 'aph_common.cuh' in srcs and len(srcs) > 10
    assert ALLOC.search(srcs['aph_common.cuh'])
    users = {name: sorted({m.group(0) for m in ALLOC.finditer(text)}) for name, text in srcs.items() if name != 'aph_common.cuh'}
    assert {name: calls for name, calls in users.items() if calls} == {}


def test_no_destroy_frees_by_hand():
    destroys = {}
    for name, text in _sources().items():
        for m in re.finditer(r'extern "C" int (aph_\w+_destroy)\s*\(', text):
            destroys[m.group(1)] = _body(text, m.end())
    assert set(destroys) >= {'aph_vit_destroy', 'aph_text_destroy', 'aph_lpips_destroy', 'aph_cppn_destroy', 'aph_fft_plan_destroy',
                             'aph_dwt_plan_destroy'}
    assert [fn for fn, body in destroys.items() if 'cudaFree' in body] == []


def test_device_bytes_is_declared_and_bound():
    hdr = open(os.path.join(ROOT, 'include', 'aphb200.h')).read()
    assert re.search(r'\bint64_t aph_device_bytes\(void\);', hdr)
    assert 'aph_device_bytes' in _lib.EXPORTS
