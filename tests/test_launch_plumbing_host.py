"""Launch configuration, read from the sources: one helper raises a kernel's shared-memory limit (smem_at_least), one function
encodes tensor maps, one helper sizes the grid-stride launches (stride_blocks), and the encoder's graph cache is keyed on what
it replays, so that each of these decisions is made in one place."""
import re

from test_device_memory_host import _body, _sources


def _function(text, name):
    """the body of the function `name` defined in `text`"""
    m = re.search(r'\b%s\s*\([^;{]*\)\s*\{' % name, text)
    assert m, name
    return _body(text, m.start())


def _outside(srcs, file, body):
    """every source with `body` cut out of `file`"""
    assert body in srcs[file]
    return {name: text.replace(body, '') if name == file else text for name, text in srcs.items()}


def test_shared_memory_limits_are_raised_only_by_the_helper():
    srcs = _sources()
    helper = _function(srcs['aph_common.cuh'], 'smem_at_least')
    assert 'cudaFuncAttributeMaxDynamicSharedMemorySize' in helper and 'cudaFuncAttributePreferredSharedMemoryCarveout' in helper
    rest = _outside(srcs, 'aph_common.cuh', helper)
    assert [name for name, text in rest.items() if 'cudaFuncSetAttribute' in text] == []
    callers = {name for name, text in rest.items() if 'smem_at_least(' in text}
    assert callers >= {'vit_gemm.cu', 'conv_tc.cu', 'cppn.cu', 'vit_attn_tc.cuh', 'text.cu', 'sample.cu', 'synth_fft.cu'}


def test_no_function_local_launch_flag_remains():
    flags = {name: re.findall(r'\n[ \t]+static\s+(?:bool|size_t)\s+\w+\s*[=;]', text) for name, text in _sources().items()}
    assert {name: found for name, found in flags.items() if found} == {}


def test_tensor_maps_are_encoded_by_one_function():
    srcs = _sources()
    encoder = _function(srcs['vit_gemm.cu'], 'encode_tmap')
    assert 'cudaGetDriverEntryPoint' in encoder and 'CU_TENSOR_MAP_SWIZZLE_128B' in encoder
    rest = _outside(srcs, 'vit_gemm.cu', encoder)
    for token in ('cudaGetDriverEntryPoint', 'cuTensorMapEncodeTiled', 'CU_TENSOR_MAP_SWIZZLE_128B', 'CU_TENSOR_MAP_DATA_TYPE'):
        assert [name for name, text in rest.items() if token in text] == [], token


def test_grid_stride_block_counts_come_from_the_helper():
    srcs = _sources()
    helper = _function(srcs['aph_common.cuh'], 'stride_blocks')
    assert '+ 255) / 256' in helper and 'num_sms()' in helper
    rest = _outside(srcs, 'aph_common.cuh', helper)
    # a statement that divides by the block size and caps by the SM count is a grid-stride block count written out again
    inline = {name: [s.strip() for s in text.split(';') if '+ 255) / 256' in s and 'num_sms()' in s] for name, text in rest.items()}
    assert {name: found for name, found in inline.items() if found} == {}
    assert [name for name, text in rest.items() if re.search(r'\b(grid_for|pack_grid)\b', text)] == []


def test_the_graph_cache_is_keyed_on_batch_size_and_flag_and_owns_its_graphs():
    vit = _sources()['vit.cu']
    assert 'run_cached' not in vit and '~VitImpl' not in vit
    cache = _body(vit, vit.index('struct GraphCache'))
    entry = re.search(r'struct Entry\s*\{([^}]*)\}', cache).group(1)
    assert '*' not in entry and 'void' not in entry, entry
    params = re.search(r'\bint run\(([^)]*)\)', cache).group(1)
    assert [p.strip() for p in params.split(',')] == ['int S', 'int flag', 'cudaStream_t& st', 'Body body']
    assert vit.count('cudaGraphExecDestroy') == cache.count('cudaGraphExecDestroy') == 2     # the destructor and the LRU eviction
    assert re.search(r'GraphCache fwd_graphs, bwd_graphs;', vit)
