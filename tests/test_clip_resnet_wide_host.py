"""The wide ResNet image towers' host side (no GPU): the model table, the channel-padding fold at every padded width, the per-model
crop sides, the checkpoint rules of clip.load and the optional trailing arguments of the tower's test entries."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from aphantasia_b200 import _lib, clip

WIDE = {'RN50x4': ((4, 6, 10, 6), 80, 40, 640, 288), 'RN50x16': ((6, 8, 18, 8), 96, 48, 768, 384),
        'RN50x64': ((3, 15, 36, 10), 128, 64, 1024, 448)}


def _visual(sd):
    return {k[len('visual.'):]: v for k, v in sd.items() if k.startswith('visual.')}


def _small(width, seed):
    """A one-block-per-stage ModifiedResNet of the given width: every padded shape of the full tower at that width."""
    return _visual(clip.synthetic_resnet_state_dict(layers=(1, 1, 1, 1), width=width, heads=width // 2, out_dim=128, res=224, seed=seed))


def test_model_table():
    for name, (layers, width, heads, out_dim, res) in WIDE.items():
        assert name in clip.available_models() and name in clip.CHECKPOINT_ONLY
        assert clip._MODELS[name] == dict(layers=layers, width=width, heads=heads, out_dim=out_dim, res=res)
        assert heads * 64 == 32 * width and out_dim % 128 == 0 and res % 32 == 0
    assert 'ViT-L/14@336px' not in clip.available_models()


@pytest.mark.parametrize('width', [80, 96, 112, 128])
def test_fold_pads_with_exact_zeros_and_folds_to_1e_12(width):
    """Every convolution but the stem's first comes out at pad64 channels on both sides, the padding exactly 0 in weights and
    biases; the real part of each BN-folded convolution equals conv -> BN (eval, float64) to 1e-12, and a zero-padded input gives
    exactly zero padded outputs."""
    sd = _small(width, seed=width)
    f = clip.fold_resnet_state_dict(sd)
    pad = clip.pad64
    assert f['conv1.weight'].shape == (width // 2, 3, 3, 3) and f['conv1.bias'].shape == (width // 2,)
    g = torch.Generator().manual_seed(0)

    def ref(x, conv, bn, p):
        y = F.conv2d(x, sd[conv].double(), padding=p)
        return F.batch_norm(y, sd[bn + '.running_mean'].double(), sd[bn + '.running_var'].double(), sd[bn + '.weight'].double(),
                            sd[bn + '.bias'].double(), training=False, eps=1e-5)
    convs = [('conv2', 'bn2', 1), ('conv3', 'bn3', 1)]
    for i in range(1, 5):
        b = 'layer%d.0.' % i
        convs += [(b + 'conv1', b + 'bn1', 0), (b + 'conv2', b + 'bn2', 1), (b + 'conv3', b + 'bn3', 0),
                  (b + 'downsample', b + 'downsample.1', 0)]
    for key, bn, p in convs:
        src = key + ('.0.weight' if key.endswith('downsample') else '.weight')
        co, ci = sd[src].shape[:2]
        w, bias = f[key + '.weight'], f[key + '.bias']
        assert w.shape[:2] == (pad64 := pad(co), pad(ci)) and bias.shape == (pad64,), key
        w4 = w if w.dim() == 4 else w[:, :, None, None]
        assert (w4[co:] == 0).all() and (w4[:, ci:] == 0).all() and (bias[co:] == 0).all(), key
        x = torch.randn(1, ci, 6, 6, generator=g, dtype=torch.float64)
        xp = torch.cat([x, torch.zeros(1, pad(ci) - ci, 6, 6, dtype=torch.float64)], 1)
        got = F.conv2d(xp, w4, bias, padding=p)
        assert (got[:, :co] - ref(x, src, bn, p)).abs().max() < 1e-12, key
        assert (got[:, co:] == 0).all(), key


def test_fold_padded_widths_of_the_models():
    """RN50x4: stem 40 -> 64 and 80 -> 128, planes 80 -> 128 and 160 -> 192; RN50x16: 48 -> 64, 96 -> 128, planes 96 -> 128;
    RN50x64 unpadded. fp32 output (the handle's) equals the float64 fold rounded."""
    for width, stem3, planes in ((80, 128, (128, 192, 320, 640)), (96, 128, (128, 192, 384, 768)), (128, 128, (128, 256, 512, 1024))):
        sd = _small(width, seed=1)
        f = clip.fold_resnet_state_dict(sd)
        assert f['conv2.weight'].shape == (64, 64, 3, 3) and f['conv3.weight'].shape == (stem3, 64, 3, 3)
        assert tuple(f['layer%d.0.conv2.weight' % (i + 1)].shape[0] for i in range(4)) == planes
        assert f['layer1.0.conv1.weight'].shape == (planes[0], stem3)
        assert tuple(f['layer%d.0.conv3.weight' % (i + 1)].shape for i in range(4)) == tuple((4 * (width << i), planes[i]) for i in range(4))
        f32 = clip.fold_resnet_state_dict(sd, dtype=torch.float32)
        assert list(f32) == list(f) and all(f32[k].dtype == torch.float32 and torch.equal(f32[k], f[k].float()) for k in f)


@pytest.mark.parametrize('name', ['RN50', 'RN101'])
def test_fold_of_rn50_and_rn101_is_unchanged(name):
    """The stem keeps its 32 -> 64 padding and nothing else changes: the padding rule reproduces the RN50-only fold exactly."""
    sd = _visual(clip.synthetic_resnet_state_dict(seed=5, **clip._MODELS[name]))
    f = clip.fold_resnet_state_dict(sd)
    eps = 1e-5

    def fold(conv, bn):
        s = sd[bn + '.weight'].double() / torch.sqrt(sd[bn + '.running_var'].double() + eps)
        return sd[conv].double() * s.view(-1, 1, 1, 1), sd[bn + '.bias'].double() - sd[bn + '.running_mean'].double() * s
    w2, b2 = fold('conv2.weight', 'bn2')
    w3, b3 = fold('conv3.weight', 'bn3')
    want2 = torch.zeros(64, 64, 3, 3, dtype=torch.float64); want2[:32, :32] = w2
    want3 = torch.zeros(64, 64, 3, 3, dtype=torch.float64); want3[:, :32] = w3
    assert torch.equal(f['conv2.weight'], want2) and torch.equal(f['conv2.bias'][:32], b2) and (f['conv2.bias'][32:] == 0).all()
    assert torch.equal(f['conv3.weight'], want3) and torch.equal(f['conv3.bias'], b3)
    w, b = fold('layer3.1.conv2.weight', 'layer3.1.bn2')
    assert torch.equal(f['layer3.1.conv2.weight'], w) and torch.equal(f['layer3.1.conv2.bias'], b)
    w, b = fold('layer4.0.downsample.0.weight', 'layer4.0.downsample.1')
    assert torch.equal(f['layer4.0.downsample.weight'], w.flatten(1)) and torch.equal(f['layer4.0.downsample.bias'], b)
    assert all(v.dtype == torch.float64 for v in f.values())


def _final_map(side):
    h = (side - 1) // 2 + 1
    for _ in range(4):
        h //= 2
    return h


@pytest.mark.parametrize('name', ['RN50', 'RN50x4', 'RN50x16', 'RN50x64'])
def test_side_ranges(name):
    """Each tower takes exactly the sides whose final map is res/32 x res/32, its size + 8 crops included."""
    res = clip._MODELS[name]['res']
    lo, hi = clip.rn_sides(res)
    assert [s for s in range(res - 64, res + 64) if _final_map(s) == res // 32] == list(range(lo, hi + 1))
    assert lo <= res + 8 <= hi
    vis = clip.ModifiedResNet.__new__(clip.ModifiedResNet)
    vis.input_resolution = res
    for side in (lo, res, res + 8, hi):
        vis.check_input(torch.empty(1, 3, side, side))
    g = res // 32
    for side in (lo - 1, hi + 1):
        with pytest.raises(ValueError, match='%d <= side <= %d \\(a %d x %d final map\\)' % (lo, hi, g, g)):
            vis.check_input(torch.empty(1, 3, side, side))
    assert clip.RN_SIDES == (223, 254) and clip.ModifiedResNet.input_resolution == 224


@pytest.mark.parametrize('name', sorted(WIDE))
def test_refused_without_a_checkpoint(name, monkeypatch):
    monkeypatch.delenv('APH_CLIP_WEIGHTS', raising=False)
    monkeypatch.delenv(clip.weights_variable(name), raising=False)
    with pytest.raises(RuntimeError, match='not available.*%s' % clip.weights_variable(name)):
        clip.load(name)
    assert clip.weights_variable(name) == 'APH_CLIP_WEIGHTS_' + name.upper()


def test_architecture_check_against_the_name(tmp_path, monkeypatch):
    """A checkpoint whose layers, width or resolution differ from the name's is refused, naming both; a matching one builds the
    tower (the handle itself is made on the first call)."""
    sd = clip.synthetic_resnet_state_dict(layers=(1, 1, 1, 1), width=80, heads=40, out_dim=640, res=288, seed=2)
    path = tmp_path / 'wrong.pt'
    torch.save({k: (v.half() if v.is_floating_point() else v) for k, v in sd.items()}, str(path))
    monkeypatch.setenv('APH_CLIP_WEIGHTS_RN50X4', str(path))
    with pytest.raises(RuntimeError, match=r'layers \(1, 1, 1, 1\), width 80, resolution 288, not RN50x4 \(layers \(4, 6, 10, 6\)'):
        clip.load('RN50x4')
    vit = tmp_path / 'vit.pt'
    torch.save(clip.synthetic_visual_state_dict(layers=1, seed=0), str(vit))
    monkeypatch.setenv('APH_CLIP_WEIGHTS_RN50X16', str(vit))
    with pytest.raises(RuntimeError, match='no ResNet image tower, not RN50x16'):
        clip.load('RN50x16')
    assert clip.resnet_architecture(sd) == ((1, 1, 1, 1), 80, 288)
    full = clip.synthetic_resnet_state_dict(seed=0, **clip._MODELS['RN50x4'])
    assert clip.resnet_architecture(full) == ((4, 6, 10, 6), 80, 288)
    good = tmp_path / 'RN50x4.pt'
    torch.save(full, str(good))
    monkeypatch.setenv('APH_CLIP_WEIGHTS_RN50X4', str(good))
    model, _ = clip.load('RN50x4')
    assert not model.synthetic and model.visual.input_resolution == 288 and model.visual.layers == (4, 6, 10, 6)
    assert model.visual.width == 80 and model.visual.heads == 40 and model.embed_dim == 640 and model.visual.handle is None


def test_optional_tails():
    """The stem and token test entries take the stem width and the map grid as a trailing argument that defaults to 0 (RN50's
    32 and 7), so calls written for the plain form bind unchanged."""
    for name in ('aph_rn_stem_test', 'aph_rn_tokens_test'):
        assert _lib.OPTIONAL_TAIL[name] == (0,)
        res, args = _lib._SIGS[name]
        assert args[-2] is ctypes.c_void_p and args[-1] is ctypes.c_int


def test_branch_scale_changes_only_the_last_batch_norm_of_each_branch():
    """synthetic_resnet_state_dict's branch_scale defaults to 0.25 (the weights RN50 / RN101 and the scripts get) and scales the
    affine of each residual branch's last BatchNorm and nothing else."""
    kw = dict(layers=(1, 2, 1, 1), width=80, heads=40, out_dim=128, res=224, seed=4)
    base = clip.synthetic_resnet_state_dict(**kw)
    assert all(torch.equal(v, base[k]) for k, v in clip.synthetic_resnet_state_dict(branch_scale=0.25, **kw).items())
    low = clip.synthetic_resnet_state_dict(branch_scale=0.15, **kw)
    for k, v in base.items():
        if k.endswith('.bn3.weight') and '.layer' in k:
            assert torch.allclose(low[k], v * 0.6, rtol=1e-6), k
        else:
            assert torch.equal(low[k], v), k
