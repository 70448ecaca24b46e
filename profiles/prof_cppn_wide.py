"""Times the wide CPPN nets of cppn.py --nf (csrc/cppn.cu, 72 <= nf <= 256: layer by layer, the hidden layers as TF32 wgmma GEMMs)
and the script's training step at --nf 256.

    python profiles/prof_cppn_wide.py > cppn_wide_times.json

Reports, with the card's name, power limit and maximum SM clock:
  generator : CUDA-event times of the forward and of forward + backward (autograd, as the script calls it) at 512x512, 10 layers,
              nf 128 and 256, each activation; the same module as eager torch ops (1x1 nn.Conv2d per layer with TF32 allowed, as
              prof_cppn.py does for the narrow nets) in the same call, alternated round by round; achieved TFLOP/s from the FLOPs
              counted from shapes (forward + backward = 4x the forward's FLOPs, the backward recomputing the forward);
  step      : cppn.py's training step at 512x512, nf 256, 10 layers, ViT-B/32, 50 crops, normalize, overscan, macro 0.4,
              Adam 0.003: steps/s over a synchronised window.
"""
import json
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'profiles'))

from aphantasia_b200.cppn import CPPN  # noqa: E402
from prof_cppn import card, events_ms, flops_fwd, mgrid  # noqa: E402


def eager_forward(net, coords):
    """The original module's arithmetic as torch ops on the same parameters (cppn.py:88-116)."""
    x = coords
    for i, layer in enumerate(net.net):
        z = F.conv2d(x, layer.conv.weight, layer.conv.bias)
        if i == len(net.net) - 1:
            return torch.sigmoid(z)
        if net.act_fn == 'relu':
            x = (F.relu(z) - 0.40) / 0.58
            continue
        t = torch.atan(z)
        x = torch.cat([t / 0.67, (t * t - 0.45) / 0.396], 1) if net.act_fn == 'unbias' else torch.cat([t / 0.67, t * t / 0.6], 1)


def time_generator(rounds=5, reps=10, H=512, W=512, layers=10):
    torch.backends.cudnn.allow_tf32 = True
    out = []
    for nf in (128, 256):
        for act in ('unbias', 'comp', 'relu'):
            torch.manual_seed(0)
            net = CPPN(2, nf, layers, 3, act_fn=act).cuda()
            coords = mgrid(H, W)
            gout = torch.randn(1, 3, H, W, device='cuda')

            def ours_fwd():
                with torch.no_grad():
                    net(coords)

            def ours_fb():
                net(coords).backward(gout)

            def eager_fwd():
                with torch.no_grad():
                    eager_forward(net, coords)

            def eager_fb():
                eager_forward(net, coords).backward(gout)
            fns = {'cuda_fwd': ours_fwd, 'cuda_fwd_bwd': ours_fb, 'eager_fwd': eager_fwd, 'eager_fwd_bwd': eager_fb}
            for fn in fns.values():
                for _ in range(3):
                    fn()
            times = {k: [] for k in fns}
            for _ in range(rounds):
                for k, fn in fns.items():
                    times[k].append(events_ms(fn, reps))
            f = flops_fwd(nf, layers, H, W, act)
            med = {k: float(np.median(v)) for k, v in times.items()}
            with torch.no_grad():
                diff = float((net(coords).as_subclass(torch.Tensor) - eager_forward(net, coords)).abs().max())
            out.append({'nf': nf, 'layers': layers, 'act': act, 'frame': '%dx%d' % (W, H), 'gflop_fwd': round(f / 1e9, 2),
                        'median_ms': {k: round(v, 3) for k, v in med.items()},
                        'spread_ms': {k: [round(min(v), 3), round(max(v), 3)] for k, v in times.items()},
                        'tflops': {'cuda_fwd': round(f / med['cuda_fwd'] / 1e9, 1), 'cuda_fwd_bwd': round(4 * f / med['cuda_fwd_bwd'] / 1e9, 1)},
                        'speedup_vs_eager': {'fwd': round(med['eager_fwd'] / med['cuda_fwd'], 2),
                                             'fwd_bwd': round(med['eager_fwd_bwd'] / med['cuda_fwd_bwd'], 2)},
                        'max_abs_diff_vs_eager': diff})
            del net
            torch.cuda.empty_cache()
    return out


def time_step(nf=256, steps=20):
    """cppn.py's training step at --nf 256 (its other defaults), device-resident, one synchronise per window"""
    import time
    from aphantasia_b200 import transforms
    from aphantasia_b200.clip import load
    from aphantasia_b200.utils import slice_imgs
    model, _ = load('ViT-B/32')
    txt = model.encode_text(torch.zeros(1, 77, dtype=torch.long).cuda()).detach()
    torch.manual_seed(0); np.random.seed(0)
    net = CPPN(2, nf, 10, 3, act_fn='unbias').cuda()
    coords = mgrid(512, 512)
    opt = torch.optim.Adam(net.parameters(), 0.003)
    norm = transforms.normalize()

    def step():
        img = net(coords)
        sliced = slice_imgs([img], 50, 224, norm, 'overscan', 0.4)
        enc = model.encode_image(sliced[-1])
        loss = -torch.cosine_similarity(txt, enc, dim=-1).mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
    for _ in range(3):
        step()
    walls = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            step()
        torch.cuda.synchronize()
        walls.append((time.perf_counter() - t0) * 1e3 / steps)
    return {'frame': '512x512', 'nf': nf, 'layers': 10, 'model': 'ViT-B/32', 'samples': 50, 'step_ms': [round(w, 3) for w in walls],
            'steps_per_s_median': round(1e3 / float(np.median(walls)), 2)}


if __name__ == '__main__':
    assert torch.cuda.is_available(), 'prof_cppn_wide.py measures on the GPU'
    print(json.dumps({'card': card(), 'generator': time_generator(), 'step': time_step()}, indent=1))
