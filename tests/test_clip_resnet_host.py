"""The ResNet image towers' host side (no GPU): the model table and its refusals, the synthetic state dict against the
ModifiedResNet architecture, the BatchNorm fold, the q/k/v stacking order and the crop-side rule."""
import pytest
import torch
import torch.nn.functional as F

from aphantasia_b200 import clip

ARCH = {'RN50': ((3, 4, 6, 3), 1024), 'RN101': ((3, 4, 23, 3), 512)}


def _visual(sd):
    return {k[len('visual.'):]: v for k, v in sd.items() if k.startswith('visual.')}


def test_model_table_and_refusals():
    for name, (layers, out_dim) in ARCH.items():
        assert name in clip.available_models()
        assert clip._MODELS[name] == dict(layers=layers, width=64, heads=32, out_dim=out_dim, res=224)
    for name in ('RN50x4', 'RN50x16', 'RN50x64', 'ViT-L/14@336px'):
        with pytest.raises(RuntimeError, match='not available'):
            clip.load(name)


@pytest.mark.parametrize('name', sorted(ARCH))
def test_synthetic_state_dict_matches_the_architecture(name):
    layers, out_dim = ARCH[name]
    sd = _visual(clip.synthetic_resnet_state_dict(seed=1, **clip._MODELS[name]))
    assert clip.is_resnet({'visual.' + k: v for k, v in sd.items()})
    want = {'conv1.weight': (32, 3, 3, 3), 'conv2.weight': (32, 32, 3, 3), 'conv3.weight': (64, 32, 3, 3),
            'attnpool.positional_embedding': (50, 2048), 'attnpool.c_proj.weight': (out_dim, 2048), 'attnpool.c_proj.bias': (out_dim,)}
    for n in 'qkv':
        want['attnpool.%s_proj.weight' % n], want['attnpool.%s_proj.bias' % n] = (2048, 2048), (2048,)

    def bn(p, c):
        for k in ('weight', 'bias', 'running_mean', 'running_var'):
            want['%s.%s' % (p, k)] = (c,)
        want[p + '.num_batches_tracked'] = ()
    for i, c in enumerate((32, 32, 64)):
        bn('bn%d' % (i + 1), c)
    cin = 64
    for i, n in enumerate(layers):
        P = 64 << i
        for j in range(n):
            p = 'layer%d.%d.' % (i + 1, j)
            want[p + 'conv1.weight'], want[p + 'conv2.weight'], want[p + 'conv3.weight'] = (P, cin, 1, 1), (P, P, 3, 3), (4 * P, P, 1, 1)
            bn(p + 'bn1', P); bn(p + 'bn2', P); bn(p + 'bn3', 4 * P)
            if j == 0:                      # every stage's first block changes the stride or the width
                want[p + 'downsample.0.weight'] = (4 * P, cin, 1, 1)
                bn(p + 'downsample.1', 4 * P)
            cin = 4 * P
    assert {k: tuple(v.shape) for k, v in sd.items()} == want
    # non-trivial running statistics, so that a missing fold shows
    assert (sd['layer2.0.bn1.running_mean'].abs() > 0).all() and (sd['layer2.0.bn1.running_var'] != 1).all()


def test_fold_matches_conv_then_batch_norm():
    """conv -> BN (eval, float64) equals the folded conv with its new bias to 1e-12, for a 3x3, a 1x1 and the stem's padding."""
    sd = _visual(clip.synthetic_resnet_state_dict(layers=(1, 1, 1, 1), seed=3))
    f = clip.fold_resnet_state_dict(sd)
    g = torch.Generator().manual_seed(0)

    def ref(x, conv, bn, pad):
        y = F.conv2d(x, sd[conv].double(), padding=pad)
        return F.batch_norm(y, sd[bn + '.running_mean'].double(), sd[bn + '.running_var'].double(), sd[bn + '.weight'].double(),
                            sd[bn + '.bias'].double(), training=False, eps=1e-5)
    x = torch.randn(2, 64, 9, 9, generator=g, dtype=torch.float64)
    got = F.conv2d(x, f['layer1.0.conv2.weight'], f['layer1.0.conv2.bias'], padding=1)
    assert (got - ref(x, 'layer1.0.conv2.weight', 'layer1.0.bn2', 1)).abs().max() < 1e-12
    got = F.conv2d(x, f['layer1.0.conv1.weight'][:, :, None, None], f['layer1.0.conv1.bias'])
    assert (got - ref(x, 'layer1.0.conv1.weight', 'layer1.0.bn1', 0)).abs().max() < 1e-12
    got = F.conv2d(x, f['layer1.0.downsample.weight'][:, :, None, None], f['layer1.0.downsample.bias'])
    assert (got - ref(x, 'layer1.0.downsample.0.weight', 'layer1.0.downsample.1', 0)).abs().max() < 1e-12
    # stem: 32 channels zero-padded to 64 on both sides of conv2, on the input side of conv3
    x32 = torch.randn(2, 32, 9, 9, generator=g, dtype=torch.float64)
    x64 = torch.cat([x32, torch.zeros_like(x32)], 1)
    got = F.conv2d(x64, f['conv2.weight'], f['conv2.bias'], padding=1)
    assert (got[:, :32] - ref(x32, 'conv2.weight', 'bn2', 1)).abs().max() < 1e-12 and (got[:, 32:] == 0).all()
    got = F.conv2d(x64, f['conv3.weight'], f['conv3.bias'], padding=1)
    assert (got - ref(x32, 'conv3.weight', 'bn3', 1)).abs().max() < 1e-12
    assert f['conv1.weight'].shape == (32, 3, 3, 3)


def test_qkv_stacking_order():
    sd = _visual(clip.synthetic_resnet_state_dict(layers=(1, 1, 1, 1), seed=4))
    f = clip.fold_resnet_state_dict(sd)
    w, b = f['attnpool.qkv.weight'], f['attnpool.qkv.bias']
    assert w.shape == (6144, 2048) and b.shape == (6144,)
    for i, n in enumerate('qkv'):
        assert torch.equal(w[2048 * i:2048 * (i + 1)], sd['attnpool.%s_proj.weight' % n].double())
        assert torch.equal(b[2048 * i:2048 * (i + 1)], sd['attnpool.%s_proj.bias' % n].double())


def _final_map(side):
    h = (side - 1) // 2 + 1
    for _ in range(4):
        h //= 2
    return h


def test_side_rule():
    """The tower accepts exactly the sides whose final map is 7 x 7, and names that range when it refuses one."""
    lo, hi = clip.RN_SIDES
    assert [s for s in range(160, 320) if _final_map(s) == 7] == list(range(lo, hi + 1))
    assert (lo, hi) == (223, 254)
    vis = clip.ModifiedResNet.__new__(clip.ModifiedResNet)
    for side in (lo, 224, 232, hi):
        vis.check_input(torch.empty(2, 3, side, side))
    for shape in ((2, 3, 222, 222), (2, 3, 255, 255), (2, 3, 224, 232), (2, 1, 224, 224)):
        with pytest.raises(ValueError, match='223 <= side <= 254'):
            vis.check_input(torch.empty(shape))


def test_patch_operand_is_never_written_for_a_resnet():
    """A live ResNet tower counts as an image encoder for the sampler's patch hand-over but is never its target: alone it takes
    no patch operand, and with a ViT alive as well (clip_fft.py --dualmod) the sampler takes the plain route."""
    from aphantasia_b200 import _patchlink

    class Vit:                       # the attributes _patchlink reads from clip.VisionTransformer
        input_resolution, patch_size, _patch_gen, _handle_epoch = 224, 16, 0, 1

    rn = clip.ModifiedResNet.__new__(clip.ModifiedResNet)
    rn.input_resolution = 224
    saved = list(_patchlink._consumers)
    _patchlink._consumers.clear()
    try:
        _patchlink.register(rn)
        assert _patchlink.target(224) is None and _patchlink.target(232, windowed=True) is None
        v = Vit()
        _patchlink.register(v)
        assert _patchlink.target(224) is None and _patchlink.target(232, windowed=True) is None
        _patchlink._consumers.discard(rn)
        assert _patchlink.target(224) is v            # the ViT alone takes the fused route again
    finally:
        _patchlink._consumers.clear()
        for c in saved:
            _patchlink.register(c)
