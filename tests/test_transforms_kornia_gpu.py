"""GPU tests of transforms_custom / transforms_elastic in the fused sampler (kinds 3 and 4) and of the encoder's windowed input.

The sampler is held to the existing sampler bars against the CPU restatement (tests/kornia_oracle.py): 1e-5 on the values and
1e-4 on the canvas gradient, norm-wise. The encoder must read the top-left input_resolution window of a size + 8 batch exactly
as it reads a copy of that window, and its image gradient must have an exactly zero margin.
"""
import ctypes as C
import gc
import glob
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import kornia_oracle as KO
from oracle import restate as R

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rel(a, b):
    a = torch.as_tensor(np.asarray(a.detach().cpu() if torch.is_tensor(a) else a)).double()
    b = torch.as_tensor(np.asarray(b.detach().cpu() if torch.is_tensor(b) else b)).double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _seed(s):
    torch.manual_seed(int(s)); np.random.seed(int(s))


def _tf(kind):
    from aphantasia_b200 import transforms
    return {3: transforms.transforms_custom, 4: transforms.transforms_elastic}[kind]


# ---------------------------------------------------------------------------------------------- slice_imgs against the oracle
@pytest.mark.parametrize('kind', [3, 4])
@pytest.mark.parametrize('hw,S,size,align,macro', [((360, 640), 24, 224, 'uniform', 0.4), ((720, 1280), 190, 224, 'uniform', 0.4),
                                                   ((240, 320), 12, 224, 'overscan', 0.4), ((64, 96), 16, 32, 'uniform', 0.5),
                                                   ((360, 640), 12, 224, 'uniform', 0.)],
                         ids=['360p', 'c2', 'overscan', 'size32', 'macro0'])
def test_slice_imgs_vs_oracle(kind, hw, S, size, align, macro):
    from aphantasia_b200 import _rng
    from aphantasia_b200.utils import slice_imgs
    _seed(11)
    canvas = torch.rand(1, 3, *hw)
    cc = canvas.cuda().requires_grad_(True)
    _seed(5)
    out = slice_imgs([cc], S, size, _tf(kind), align, macro)[0]
    assert out.shape == (S, 3, size + 8, size + 8)
    _seed(5)
    tabs, frame = _rng.draw_crop_table_py(S, hw, size, kind, align, macro)
    co = canvas.clone().requires_grad_(True)
    ref = KO.sample_crops(co, tabs[0], size, kind, frame)
    _seed(6)
    cot = torch.randn(ref.shape)
    (out * cot.cuda()).sum().backward()
    (ref * cot).sum().backward()
    e_out, e_grad = _rel(out, ref), _rel(cc.grad, co.grad)
    print('kind %d %s S=%d: rel out %.2e grad %.2e' % (kind, hw, S, e_out, e_grad))
    assert e_out < 1e-5 and e_grad < 1e-4


def _abi(kind, S=24, size=224, H=300, W=420, seed=3):
    """Canvas, device table and the sampler's forward / backward through the C ABI."""
    from aphantasia_b200 import _rng
    from aphantasia_b200._lib import check, lib, stream_ptr
    _seed(seed)
    tabs, _ = _rng.draw_crop_table_py(S, (H, W), size, kind, 'uniform', 0.4)
    t = torch.from_numpy(tabs[0]).cuda()
    side = size + 8

    def fwd(x):
        out = torch.empty(S, 3, side, side, device='cuda')
        check(lib().aph_sample_fwd(x.data_ptr(), H, W, 0, 0, t.data_ptr(), S, size, kind, out.data_ptr(), stream_ptr()), 'fwd')
        return out

    def bwd(g, gscale=1., k=kind):
        gc_ = torch.full((1, 3, H, W), float('nan'), device='cuda')
        check(lib().aph_sample_bwd_scaled(g.data_ptr(), H, W, 0, 0, t.data_ptr(), S, size, k, gscale, gc_.data_ptr(), stream_ptr()), 'bwd')
        return gc_
    return fwd, bwd, (S, side, H, W)


@pytest.mark.parametrize('kind', [3, 4])
def test_sampler_backward_is_the_adjoint_of_the_forward(kind):
    """<S(x) - S(0), y> = <x, S^T y>: the backward is the exact adjoint of the forward's linear part."""
    fwd, bwd, (S, side, H, W) = _abi(kind)
    x = torch.rand(1, 3, H, W, device='cuda')
    y = torch.randn(S, 3, side, side, device='cuda')
    lhs = ((fwd(x) - fwd(torch.zeros_like(x))).double() * y.double()).sum().item()
    rhs = (x.double() * bwd(y).double()).sum().item()
    print('kind %d: <Sx - S0, y> = %.9g, <x, S^T y> = %.9g' % (kind, lhs, rhs))
    assert abs(lhs - rhs) <= 1e-5 * abs(rhs)


@pytest.mark.parametrize('kind', [3, 4])
def test_gscale_scales_the_gradient_only_and_the_scratches_stay_clean(kind):
    fwd, bwd, (S, side, H, W) = _abi(kind)
    x = torch.rand(1, 3, H, W, device='cuda')
    y = torch.randn(S, 3, side, side, device='cuda')
    out0 = fwd(x)
    g1 = bwd(y)
    g2 = bwd(y, 0.375)
    assert torch.equal(fwd(x), out0)
    assert _rel(g2, 0.375 * g1) < 1e-6 and torch.isfinite(g1).all()
    # the transforms_fast scratch (kept all-zero between calls) and this kind's scratch do not leak into each other
    fast_fwd, fast_bwd, (_, fside, _, _) = _abi(2)
    yf = torch.randn(S, 3, fside, fside, device='cuda')
    f0 = fast_bwd(yf)
    bwd(y)
    assert _rel(fast_bwd(yf), f0) < 1e-6
    assert _rel(bwd(y), g1) < 1e-6


# ---------------------------------------------------------------------------------------------- encoder on the size + 8 batch
def _model(name):
    from aphantasia_b200.clip import CLIP, synthetic_visual_state_dict
    gc.collect()
    return CLIP(name, synthetic_visual_state_dict(patch=32 if name == 'ViT-B/32' else 16, seed=0), True)


@pytest.mark.parametrize('name,S', [('ViT-B/32', 6), ('ViT-B/16', 5)])
def test_encode_image_reads_the_top_left_window(name, S):
    from aphantasia_b200 import _lib
    model = _model(name)
    g = torch.Generator('cuda').manual_seed(7)
    for it in range(3):                                  # eager, graph capture, graph replay
        x232 = torch.randn(S, 3, 232, 232, device='cuda', generator=g).requires_grad_(True)
        x224 = x232.detach()[:, :, :224, :224].clone().requires_grad_(True)
        cot = torch.randn(S, 512, device='cuda', generator=g)
        e232 = model.encode_image(x232)
        (e232 * cot).sum().backward()
        e224 = model.encode_image(x224)
        (e224 * cot).sum().backward()
        assert torch.equal(e232, e224), it
        assert torch.equal(x232.grad[:, :, :224, :224], x224.grad), it
        assert not x232.grad[:, :, 224:, :].any() and not x232.grad[:, :, :, 224:].any(), it
        assert x224.grad.abs().sum() > 0
    before = _lib.lib().aph_launch_count()
    for bad in ((S, 3, 223, 223), (S, 3, 256 if name == 'ViT-B/32' else 240, 256 if name == 'ViT-B/32' else 240), (S, 3, 232, 224),
                (S, 1, 224, 224), (3, 224, 224)):
        with pytest.raises(ValueError, match='encode_image'):
            model.encode_image(torch.zeros(bad, device='cuda'))
    assert _lib.lib().aph_launch_count() == before


@pytest.mark.parametrize('kind', [3, 4])
def test_fused_patch_operand_of_the_window(kind):
    from aphantasia_b200 import _patchlink
    from aphantasia_b200.utils import slice_imgs
    model = _model('ViT-B/32')
    assert _patchlink.target(232, windowed=True) is model.visual
    canvas = torch.rand(1, 3, 360, 640, device='cuda', generator=torch.Generator('cuda').manual_seed(3))
    _seed(4)
    crops = slice_imgs([canvas], 24, 224, _tf(kind), 'uniform', 0.4)[0]
    n0 = model.visual.prepatched_forwards
    emb = model.encode_image(crops)
    assert model.visual.prepatched_forwards == n0 + 1
    plain = model.encode_image(crops.clone())
    assert model.visual.prepatched_forwards == n0 + 1
    assert torch.equal(emb, plain)


@pytest.mark.parametrize('kind', [3, 4])
def test_full_step_config2_vs_oracle(kind):
    """1280x720 FFT, S=190, ViT-B/32, mix loss with transforms_custom / _elastic, under the existing full-step bars."""
    from aphantasia_b200 import _rng
    from aphantasia_b200.image import fft_image, to_valid_rgb
    from aphantasia_b200.utils import sim_func, slice_imgs
    from aphantasia_b200.clip import synthetic_visual_state_dict
    h, w, S = 720, 1280, 190
    model = _model('ViT-B/32')
    sd = synthetic_visual_state_dict(patch=32, seed=0)
    _seed(0)
    params, image_f, _ = fft_image([1, 3, h, w], 0.07, 1.5, None)
    rgb_f = to_valid_rgb(image_f, colors=1.8)
    g = torch.Generator().manual_seed(1234)
    txt = torch.randn(1, 512, generator=g); txt = (10. * txt / txt.norm()).cuda()
    _seed(1)
    crops = slice_imgs([rgb_f()], S, 224, _tf(kind), 'uniform', 0.4)[0]
    emb = model.encode_image(crops)
    loss = -1. * sim_func(txt, emb, 'mix')
    loss.backward()
    _seed(1)
    tabs, _ = _rng.draw_crop_table(S, (h, w), 224, kind, 'uniform', 0.4)
    o_loss, o_grad, o_emb = KO.reference_step(params[0].detach().cpu(), R.fft_scale(h, w, 1.5), (h, w), R.color_matrix(1.8), tabs[0],
                                              R.build_visual(sd), txt.cpu(), kind, 'mix')
    e_emb, e_grad = _rel(emb, o_emb), _rel(params[0].grad, o_grad)
    print('kind %d: loss ours %.6f oracle %.6f; rel emb %.3e grad %.3e' % (kind, loss.item(), o_loss.item(), e_emb, e_grad))
    assert e_emb < 2e-2 and e_grad < 2e-2
    assert abs(loss.item() - o_loss.item()) < 2e-3


def test_standalone_transform_draws_once_per_call():
    from aphantasia_b200 import _rng, transforms
    x = torch.rand(3, 3, 224, 224, device='cuda')
    for kind, tf in ((3, transforms.transforms_custom), (4, transforms.transforms_elastic)):
        _seed(9)
        out = tf(x)
        assert out.shape == (3, 3, 232, 232)
        _seed(9)
        row = np.zeros((1, _rng.CROP_PARAM_FLOATS), np.float32)
        row[0, _rng.F_CSIZE] = 224
        row[0, _rng.F_FLAGS] = _rng.draw_kornia(row[0], 224, kind == 4)
        for i in range(3):
            assert _rel(out[i:i + 1], KO.sample_crops(x[i:i + 1].cpu(), row, 224, kind)) < 1e-5


# ---------------------------------------------------------------------------------------------- the unmodified script
SCRIPT = os.environ.get('APH_REF_SCRIPT') or os.path.join(ROOT, 'oracle', '_ref', 'clip_fft.py')


@pytest.mark.skipif(not os.path.isfile(SCRIPT), reason='no copy of the original clip_fft.py: build() stages one into oracle/_ref/')
@pytest.mark.parametrize('tf', ['custom', 'elastic'])
def test_unmodified_clip_fft_with_transform(tmp_path, tf):
    out_dir = str(tmp_path / 'out')
    trace = str(tmp_path / 'trace.json')
    env = dict(os.environ, PYTHONPATH=ROOT, APH_TRACE=trace)
    cmd = [sys.executable, '-m', 'aphantasia_b200.run', SCRIPT, '-t', 'red square', '--size', '224-224', '--samples', '4', '--steps', '10',
           '-tf', tf, '--out_dir', out_dir, '-nv']
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=str(tmp_path), env=env)
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-3000:])
    tr = json.load(open(trace))
    assert tr['encode_image_calls'] == 10 and len(tr['sims']) == 10
    assert tr['sims'][-1] > tr['sims'][0], tr['sims']
    assert len(glob.glob(os.path.join(out_dir, '*', '*.jpg'))) == 10
