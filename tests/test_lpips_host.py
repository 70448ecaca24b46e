"""CPU checks of the LPIPS layer: the float64 restatement (tests/lpips_oracle.py) against an independent torch composition,
the weight loaders, and every refusal of aphantasia_b200.lpips.LPIPS."""
import os

import pytest
import torch
import torch.nn.functional as F

from aphantasia_b200 import lpips as L
import lpips_oracle as O


def _composition(in0, in1, vgg_sd, lin_sd):
    """LPIPS spelled out with F.conv2d / F.max_pool2d on the state dict, F.normalize and an einsum for the lin layers."""
    convs = [i for i in L.VGG_CONVS]
    pools_after = {3, 8, 15, 22}
    tap_after = {3, 8, 15, 22, 29}

    def feats(x):
        x = (2 * x.double() - 1 - torch.tensor(O.SHIFT, dtype=torch.float64).view(1, 3, 1, 1)) / torch.tensor(O.SCALE, dtype=torch.float64).view(1, 3, 1, 1)
        out = []
        for i in convs:
            x = F.relu(F.conv2d(x, vgg_sd['features.%d.weight' % i].double(), vgg_sd['features.%d.bias' % i].double(), padding=1))
            if i + 1 in tap_after:
                out.append(x)
            if i + 1 in pools_after:
                x = F.max_pool2d(x, 2, 2)
        return out

    val = 0
    for t, (a, b) in enumerate(zip(feats(in0), feats(in1))):
        d = (F.normalize(a, dim=1, eps=1e-30) - F.normalize(b, dim=1, eps=1e-30)) ** 2
        w = lin_sd['lin%d.model.1.weight' % t].double().reshape(-1)
        val = val + torch.einsum('nchw,c->nhw', d, w).mean(dim=(1, 2)).view(-1, 1, 1, 1)
    return val


def _perturbed_vgg(seed):
    sd = L.synthetic_vgg_state_dict()
    g = torch.Generator().manual_seed(seed)
    for k in sd:
        if k.endswith('.bias'):
            sd[k] = 0.05 * torch.randn(sd[k].shape, generator=g)
        else:
            sd[k] = sd[k] * (1 + 0.3 * torch.randn(sd[k].shape, generator=g))
    return sd


def test_oracle_matches_torch_composition():
    """Value and in0-gradient of the restatement equal an independently written composition (float64: 1e-9 relative)."""
    vgg, lin = _perturbed_vgg(3), L.synthetic_lin_state_dict()
    g = torch.Generator().manual_seed(0)
    in0 = torch.rand(2, 3, 37, 45, generator=g, dtype=torch.float64).requires_grad_(True)
    in1 = torch.rand(2, 3, 37, 45, generator=g, dtype=torch.float64)
    a = O.lpips(in0, in1, vgg, lin)
    ga, = torch.autograd.grad(a.sum(), in0)
    b = _composition(in0, in1, vgg, lin)
    gb, = torch.autograd.grad(b.sum(), in0)
    assert a.shape == (2, 1, 1, 1)
    assert torch.allclose(a, b, rtol=1e-9, atol=0)
    assert float((ga - gb).norm() / gb.norm()) < 1e-9


def test_oracle_zero_norm_pixels_give_finite_gradient():
    """A flat region and a negative bias leave whole tap pixels at zero: the gradient is finite (the ReLU select removes the
    NaN of the norm's derivative)."""
    vgg, lin = L.synthetic_vgg_state_dict(), L.synthetic_lin_state_dict()
    vgg['features.2.bias'] = torch.full((64,), -0.4)
    in0 = torch.full((1, 3, 32, 32), 0.5, dtype=torch.float64)
    in0[..., 8:24, 8:24] = torch.rand(3, 16, 16, dtype=torch.float64, generator=torch.Generator().manual_seed(1))
    in0.requires_grad_(True)
    in1 = torch.rand(1, 3, 32, 32, dtype=torch.float64, generator=torch.Generator().manual_seed(2))
    feats = O.vgg_features(vgg)
    f = O.taps(feats, (2 * in0.detach() - 1 - torch.tensor(O.SHIFT, dtype=torch.float64).view(1, 3, 1, 1))
               / torch.tensor(O.SCALE, dtype=torch.float64).view(1, 3, 1, 1))[0]
    assert (f.abs().sum(dim=1) == 0).any(), 'the case has no all-zero relu1_2 pixel'
    v = O.lpips(in0, in1, vgg, lin, feats=feats)
    g, = torch.autograd.grad(v.sum(), in0)
    assert torch.isfinite(g).all() and g.abs().sum() > 0


def test_synthetic_weights_keys_shapes_and_rng():
    """The synthetic state dicts have exactly the keys and shapes the real ones have; the lin weights are non-negative; building
    them leaves the global RNG alone (the script's crop draws replay it)."""
    before = torch.get_rng_state().clone()
    vgg, lin = L.synthetic_vgg_state_dict(), L.synthetic_lin_state_dict()
    assert torch.equal(before, torch.get_rng_state())
    assert sorted(vgg) == sorted('features.%d.%s' % (i, k) for i in L.VGG_CONVS for k in ('weight', 'bias'))
    for i, (ci, co) in zip(L.VGG_CONVS, L.VGG_CH):
        assert vgg['features.%d.weight' % i].shape == (co, ci, 3, 3) and vgg['features.%d.bias' % i].shape == (co,)
        std = float(vgg['features.%d.weight' % i].std())
        assert abs(std / (2.0 / (9 * co)) ** 0.5 - 1) < 0.2          # kaiming_normal_, fan_out, relu
    assert sorted(lin) == ['lin%d.model.1.weight' % t for t in range(5)]
    for t, c in enumerate(L.TAP_CH):
        assert lin['lin%d.model.1.weight' % t].shape == (1, c, 1, 1) and (lin['lin%d.model.1.weight' % t] >= 0).all()
    assert torch.equal(vgg['features.0.weight'], L.synthetic_vgg_state_dict()['features.0.weight'])


def test_loaders_read_files_and_fall_back_loudly(tmp_path, monkeypatch, capsys):
    """$APH_LPIPS_VGG / $APH_LPIPS_LIN are read (classifier keys dropped, wrong shapes refused); without them the synthetic
    weights come with a log line."""
    monkeypatch.setenv('APH_LPIPS_VGG', str(tmp_path / 'missing.pth'))
    monkeypatch.delenv('APH_LPIPS_LIN', raising=False)
    sd, synth = L.load_vgg_state_dict()
    assert synth and 'synthetic VGG16 weights' in capsys.readouterr().out
    sd, synth = L.load_lin_state_dict()
    assert synth and 'synthetic non-negative linear weights' in capsys.readouterr().out

    full = dict(_perturbed_vgg(5))
    full['classifier.0.weight'] = torch.zeros(4, 4)
    p = tmp_path / 'vgg16.pth'
    torch.save(full, str(p))
    monkeypatch.setenv('APH_LPIPS_VGG', str(p))
    sd, synth = L.load_vgg_state_dict()
    assert not synth and 'classifier.0.weight' not in sd and torch.equal(sd['features.28.bias'], full['features.28.bias'])
    lin = L.synthetic_lin_state_dict(seed=7)
    q = tmp_path / 'vgg.pth'
    torch.save(lin, str(q))
    monkeypatch.setenv('APH_LPIPS_LIN', str(q))
    sd2, synth = L.load_lin_state_dict()
    assert not synth and torch.equal(sd2['lin4.model.1.weight'], lin['lin4.model.1.weight'])

    full['features.5.weight'] = torch.zeros(128, 64, 1, 1)
    torch.save(full, str(p))
    with pytest.raises(ValueError, match='features.5.weight'):
        L.load_vgg_state_dict()


def test_hub_cache_location(tmp_path, monkeypatch):
    """Without $APH_LPIPS_VGG the weights come from torchvision's checkpoint cache under torch.hub.get_dir()."""
    monkeypatch.delenv('APH_LPIPS_VGG', raising=False)
    monkeypatch.setattr(torch.hub, 'get_dir', lambda: str(tmp_path))
    assert L.vgg_state_dict_path() is None
    os.makedirs(tmp_path / 'checkpoints')
    torch.save({}, str(tmp_path / 'checkpoints' / L.VGG_CHECKPOINT))
    assert L.vgg_state_dict_path() == str(tmp_path / 'checkpoints' / L.VGG_CHECKPOINT)


@pytest.mark.parametrize('kw, what', [({'net': 'alex'}, "net='alex'"), ({'net': 'squeeze'}, "net='squeeze'"),
                                      ({'net': 'vgg', 'spatial': True}, 'spatial=True'),
                                      ({'net': 'vgg', 'lpips': False}, 'lpips=False')])
def test_unsupported_constructions_raise(kw, what):
    with pytest.raises(NotImplementedError, match="net='vgg'") as e:
        L.LPIPS(verbose=False, **kw)
    assert what in str(e.value)


def _model():
    return L.LPIPS(net='vgg', verbose=False, vgg_state_dict=L.synthetic_vgg_state_dict(), lin_state_dict=L.synthetic_lin_state_dict())


def test_unsupported_calls_raise():
    """retPerLayer, a gradient with respect to in1, other dtypes and mismatched shapes are refused before any GPU work."""
    m = _model()
    assert m.cuda() is m and m.eval() is m and m.to('cuda') is m
    a, b = torch.rand(1, 3, 32, 32), torch.rand(1, 3, 32, 32)
    with pytest.raises(NotImplementedError, match='retPerLayer'):
        m(a, b, retPerLayer=True)
    with pytest.raises(NotImplementedError, match='in1'):
        m(a, b.requires_grad_(True))
    with pytest.raises(NotImplementedError, match='float16'):
        m(a.half(), b.detach().half())
    with pytest.raises(NotImplementedError, match='different shapes'):
        m(a, torch.rand(1, 3, 32, 40))


def test_dropin_reexports():
    import importlib
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, os.path.join(root, 'dropin'))
    try:
        sys.modules.pop('lpips', None)
        mod = importlib.import_module('lpips')
        assert mod.LPIPS is L.LPIPS
    finally:
        sys.path.remove(os.path.join(root, 'dropin'))
        sys.modules.pop('lpips', None)
