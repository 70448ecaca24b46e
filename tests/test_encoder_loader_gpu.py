"""The weight-loading contract of the image and text encoder handles (aph_vit_* / aph_text_*), at small geometries: a tensor
with the wrong element count, an unknown key and a bad layer index are refused with a message that names them, finalize
names a tensor that was never loaded, and the Python wrappers keep (and close() frees) a handle whose load failed."""
import contextlib
import ctypes as C

import pytest
import torch

from aphantasia_b200 import _lib, clip

pytestmark = pytest.mark.gpu
LAYERS, WIDTH = 2, 128
FIELDS = ('ln_1.weight', 'ln_1.bias', 'ln_2.weight', 'ln_2.bias', 'attn.in_proj_weight', 'attn.in_proj_bias',
          'attn.out_proj.weight', 'attn.out_proj.bias', 'mlp.c_fc.weight', 'mlp.c_fc.bias', 'mlp.c_proj.weight', 'mlp.c_proj.bias')


def _image_sd():
    return clip.synthetic_visual_state_dict(patch=32, width=WIDTH, layers=LAYERS, heads=2, out_dim=128, res=64, seed=0)


def _text_sd():
    return clip.synthetic_text_state_dict(width=WIDTH, layers=LAYERS, heads=2, out_dim=128, context=16, vocab=500, seed=0)


class Tower:
    """One tower through the raw C ABI: its entry points, config, key prefix and a state dict on the GPU."""

    def __init__(self, name):
        if name == 'image':
            self.api, self.prefix, sd = 'aph_vit', 'visual.', _image_sd()
            self.cfg = _lib.VitConfig(32, WIDTH, LAYERS, 2, 128, 64, 2, 0)
        else:
            self.api, self.prefix, sd = 'aph_text', '', _text_sd()
            self.cfg = _lib.TextConfig(WIDTH, LAYERS, 2, 128, 16, 500, 2, 0)
        self.sd = {k: v.contiguous().cuda() for k, v in sd.items()}

    def fn(self, what):
        return getattr(_lib.lib(), '%s_%s' % (self.api, what))

    def block_key(self, layer, field):
        return '%stransformer.resblocks.%s.%s' % (self.prefix, layer, field)

    @contextlib.contextmanager
    def handle(self):
        h = C.c_void_p()
        assert self.fn('create')(C.byref(h), C.byref(self.cfg)) == 0, _error()
        try:
            yield h
        finally:
            torch.cuda.synchronize()         # the loads are asynchronous: they finish before the handle and `sd` go
            self.fn('destroy')(h)

    def load(self, h, key, t, numel=None):
        return self.fn('load_tensor')(h, key.encode(), t.data_ptr(), t.numel() if numel is None else numel, _lib.stream_ptr())


def _error():
    return _lib.lib().aph_last_error().decode()


@pytest.fixture(params=['image', 'text'])
def tower(request):
    return Tower(request.param)


@pytest.mark.parametrize('field', FIELDS)
def test_block_tensor_with_wrong_size_is_refused(tower, field):
    key = tower.block_key(1, field)
    n = tower.sd[key].numel()
    buf = torch.zeros(n + WIDTH, device='cuda')
    with tower.handle() as h:
        for bad in (n - 1, n + WIDTH):
            assert tower.load(h, key, buf, bad) == 2
            msg = _error()
            assert key in msg and 'expected %d elements, got %d' % (n, bad) in msg, msg
        assert tower.load(h, key, buf, n) == 0, _error()


def test_unknown_keys_and_bad_layer_indices_are_refused(tower):
    buf = torch.zeros(4 * WIDTH, device='cuda')
    with tower.handle() as h:
        for key in (tower.prefix + 'ln_mid.weight', tower.block_key(0, 'attn.qkv_weight'), tower.block_key(0, 'ln_1')):
            assert tower.load(h, key, buf, WIDTH) == 2
            assert 'unknown tensor %s' % key in _error()
        for layer in (LAYERS, -1, 'x'):
            key = tower.block_key(layer, 'ln_1.weight')
            assert tower.load(h, key, buf, WIDTH) == 2
            assert 'bad layer index in %s' % key in _error()


def test_finalize_names_the_missing_tensor(tower):
    assert len(tower.sd) == (8 if tower.api == 'aph_vit' else 5) + LAYERS * len(FIELDS)
    for missing in tower.sd:
        with tower.handle() as h:
            for k, v in tower.sd.items():
                if k != missing:
                    assert tower.load(h, k, v) == 0, _error()
            assert tower.fn('finalize')(h) == 2
            # the image tower's message names the key with its 'visual.' prefix, like the state dict
            assert 'tensor %s was never loaded' % missing in _error(), (missing, _error())
    with tower.handle() as h:
        for k, v in tower.sd.items():
            assert tower.load(h, k, v) == 0, _error()
        assert tower.fn('finalize')(h) == 0, _error()


@pytest.mark.parametrize('name', ['image', 'text'])
def test_wrapper_owns_the_handle_of_a_failed_load(name):
    """A state dict with one tensor of the wrong size: _ensure raises, and the wrapper still holds the handle it created, so
    close() frees it instead of leaking it."""
    if name == 'image':
        sd = _image_sd()
        key = 'visual.transformer.resblocks.1.mlp.c_fc.bias'
        sd[key] = torch.zeros(4 * WIDTH - 1)
        model, nbytes = clip.VisionTransformer(sd), _lib.lib().aph_vit_bytes
    else:
        sd = _text_sd()
        key = 'transformer.resblocks.1.mlp.c_fc.bias'
        sd[key] = torch.zeros(4 * WIDTH - 1)
        model, nbytes = clip.TextTransformer(sd), _lib.lib().aph_text_bytes
    with pytest.raises(RuntimeError, match='expected %d elements, got %d' % (4 * WIDTH, 4 * WIDTH - 1)):
        model._ensure(2)
    assert model.handle is not None and nbytes(model.handle) > 0
    model.close()
    assert model.handle is None
