"""The weight-loading contract of the handles that take a state dict: the image and text encoders (aph_vit_* / aph_text_*, at
small geometries) and LPIPS (aph_lpips_*). A tensor with the wrong element count, an unknown key and a bad layer index are
refused with a message that names them, finalize names a tensor that was never loaded, and the Python wrappers keep (and
close() frees) a handle whose load failed."""
import contextlib
import ctypes as C

import pytest
import torch

from aphantasia_b200 import _lib, clip, lpips

pytestmark = pytest.mark.gpu
LAYERS, WIDTH = 2, 128
FIELDS = ('ln_1.weight', 'ln_1.bias', 'ln_2.weight', 'ln_2.bias', 'attn.in_proj_weight', 'attn.in_proj_bias',
          'attn.out_proj.weight', 'attn.out_proj.bias', 'mlp.c_fc.weight', 'mlp.c_fc.bias', 'mlp.c_proj.weight', 'mlp.c_proj.bias')


def _image_sd():
    return clip.synthetic_visual_state_dict(patch=32, width=WIDTH, layers=LAYERS, heads=2, out_dim=128, res=64, seed=0)


def _text_sd():
    return clip.synthetic_text_state_dict(width=WIDTH, layers=LAYERS, heads=2, out_dim=128, context=16, vocab=500, seed=0)


def _lpips_sd():
    return {**lpips.synthetic_vgg_state_dict(), **lpips.synthetic_lin_state_dict()}


class Tower:
    """One handle kind through the raw C ABI: its entry points, create arguments, key prefix and a state dict on the GPU."""

    def __init__(self, name):
        if name == 'image':
            self.api, self.prefix, sd = 'aph_vit', 'visual.', _image_sd()
            self.cfg = [C.byref(_lib.VitConfig(32, WIDTH, LAYERS, 2, 128, 64, 2, 0))]
        elif name == 'text':
            self.api, self.prefix, sd = 'aph_text', '', _text_sd()
            self.cfg = [C.byref(_lib.TextConfig(WIDTH, LAYERS, 2, 128, 16, 500, 2, 0))]
        else:
            self.api, self.prefix, sd, self.cfg = 'aph_lpips', '', _lpips_sd(), []
        self.sd = {k: v.contiguous().cuda() for k, v in sd.items()}

    def fn(self, what):
        return getattr(_lib.lib(), '%s_%s' % (self.api, what))

    def block_key(self, layer, field):
        return '%stransformer.resblocks.%s.%s' % (self.prefix, layer, field)

    @contextlib.contextmanager
    def handle(self):
        h = C.c_void_p()
        assert self.fn('create')(C.byref(h), *self.cfg) == 0, _error()
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


@pytest.fixture(params=['image', 'text', 'lpips'])
def any_handle(request):
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


@pytest.mark.parametrize('key', ['features.0.weight', 'features.0.bias', 'features.2.weight', 'features.28.weight',
                                 'features.28.bias', 'lin0.model.1.weight', 'lin4.model.1.weight'])
def test_lpips_tensor_with_wrong_size_is_refused(key):
    """conv1_1's fp32 copy, a packed 3x3 convolution, a bias and a linear layer each check their element count."""
    tower = Tower('lpips')
    n = tower.sd[key].numel()
    buf = torch.zeros(n + 64, device='cuda')
    with tower.handle() as h:
        for bad in (n - 1, n + 64):
            assert tower.load(h, key, buf, bad) == 2
            msg = _error()
            assert key in msg and 'expected %d elements, got %d' % (n, bad) in msg, msg
        assert tower.load(h, key, buf, n) == 0, _error()


def test_lpips_unknown_keys_are_refused():
    """A ReLU or max-pool index of VGG16's features, a sixth linear layer and anything else: no such tensor."""
    tower = Tower('lpips')
    buf = torch.zeros(64 * 27, device='cuda')
    with tower.handle() as h:
        for key in ('features.3.weight', 'features.1.bias', 'features.30.weight', 'lin5.model.1.weight', 'lin0.model.0.weight',
                    'classifier.0.weight', 'features.0'):
            assert tower.load(h, key, buf, 64) == 2
            assert 'unknown tensor %s' % key in _error(), _error()


def test_finalize_names_the_missing_tensor(any_handle):
    tower = any_handle
    assert len(tower.sd) == {'aph_vit': 8 + LAYERS * len(FIELDS), 'aph_text': 5 + LAYERS * len(FIELDS), 'aph_lpips': 2 * 13 + 5}[tower.api]
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


@pytest.mark.parametrize('name', ['image', 'text', 'lpips'])
def test_wrapper_owns_the_handle_of_a_failed_load(name):
    """A state dict with one tensor of the wrong size: building the handle raises, the wrapper still holds the handle it created
    (not loaded), a second attempt raises the load's error again, and close() frees the handle instead of leaking it."""
    if name == 'image':
        sd = _image_sd()
        sd['visual.transformer.resblocks.1.mlp.c_fc.bias'] = torch.zeros(4 * WIDTH - 1)
        model, n = clip.VisionTransformer(sd), 4 * WIDTH
        build, held = (lambda: model._ensure(2)), (lambda: model.handle)
    elif name == 'text':
        sd = _text_sd()
        sd['transformer.resblocks.1.mlp.c_fc.bias'] = torch.zeros(4 * WIDTH - 1)
        model, n = clip.TextTransformer(sd), 4 * WIDTH
        build, held = (lambda: model._ensure(2)), (lambda: model.handle)
    else:
        lin = lpips.synthetic_lin_state_dict()
        lin['lin4.model.1.weight'] = torch.zeros(511)
        model, n = lpips.LPIPS(net='vgg', verbose=False, vgg_state_dict=lpips.synthetic_vgg_state_dict(), lin_state_dict=lin), 512
        build, held = model._ensure, (lambda: model._handle)
    for _ in range(2):
        with pytest.raises(RuntimeError, match='expected %d elements, got %d' % (n, n - 1)):
            build()
        h = held()
        assert h is not None and not h.loaded
    if name != 'lpips':
        assert ({'image': _lib.lib().aph_vit_bytes, 'text': _lib.lib().aph_text_bytes}[name])(h) > 0
    model.close()
    assert held() is None and not hasattr(h, '_as_parameter_')
