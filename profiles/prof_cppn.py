"""Times the CPPN generator of cppn.py (csrc/cppn.cu) and the script's training step.

    python profiles/prof_cppn.py > cppn_times.json

Reports, with the card's name and power limit:
  generator : CUDA-event times of the forward and of forward + backward (autograd, as the script calls it) at 512x512 and
              1280x720, nf 24 / 64, 10 layers, `unbias`; the same module as eager torch ops (F.conv2d per layer, atan, cat, sigmoid;
              cuDNN with torch's default allow_tf32) in the same call, alternated round by round; achieved TFLOP/s from the FLOPs
              counted below (the backward recomputes the forward: forward + backward = 4x the forward's FLOPs);
  step      : cppn.py's training step at its defaults (512x512, nf 24, 10 layers, ViT-B/32, 50 crops, normalize, overscan,
              macro 0.4, Adam 0.003): generator, sampler, encoder, cosine loss, backward, Adam; wall time per step with one
              synchronise per step window.
"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from aphantasia_b200 import transforms  # noqa: E402
from aphantasia_b200.clip import load  # noqa: E402
from aphantasia_b200.cppn import CPPN  # noqa: E402
from aphantasia_b200.utils import slice_imgs  # noqa: E402


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as ex:
        return 'unknown (%r)' % (ex,)


def mgrid(H, W):
    xs, ys = np.linspace(-1, 1, num=W), np.linspace(-1, 1, num=H)
    return torch.from_numpy(np.stack(np.meshgrid(xs, ys), axis=0)[None].astype(np.float32)).cuda()


def flops_fwd(nf, layers, H, W, act='unbias'):
    """Multiply-adds x 2 of the forward per frame: 2 -> nf, (layers - 1) x kh -> nf, kh -> 3."""
    kh = nf if act == 'relu' else 2 * nf
    return 2. * H * W * (2 * nf + (layers - 1) * kh * nf + kh * 3)


def eager_forward(net, coords):
    """The original module's arithmetic as torch ops on the same parameters (cppn.py:88-116)."""
    x = coords
    for i, layer in enumerate(net.net):
        z = F.conv2d(x, layer.conv.weight, layer.conv.bias)
        if i == len(net.net) - 1:
            return torch.sigmoid(z)
        t = torch.atan(z)
        x = torch.cat([t / 0.67, (t * t - 0.45) / 0.396], 1)


def events_ms(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def time_generator(rounds=5, reps=20):
    out = []
    for nf in (24, 64):
        for H, W in ((512, 512), (720, 1280)):
            torch.manual_seed(0)
            net = CPPN(2, nf, 10, 3, act_fn='unbias').cuda()
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
            f = flops_fwd(nf, 10, H, W)
            med = {k: float(np.median(v)) for k, v in times.items()}
            with torch.no_grad():
                diff = float((net(coords).as_subclass(torch.Tensor) - eager_forward(net, coords)).abs().max())
            out.append({'nf': nf, 'layers': 10, 'act': 'unbias', 'frame': '%dx%d' % (W, H), 'gflop_fwd': round(f / 1e9, 3),
                        'gflop_fwd_bwd': round(4 * f / 1e9, 3), 'median_ms': {k: round(v, 4) for k, v in med.items()},
                        'spread_ms': {k: [round(min(v), 4), round(max(v), 4)] for k, v in times.items()},
                        'tflops': {'cuda_fwd': round(f / med['cuda_fwd'] / 1e9, 2), 'cuda_fwd_bwd': round(4 * f / med['cuda_fwd_bwd'] / 1e9, 2)},
                        'speedup_vs_eager': {'fwd': round(med['eager_fwd'] / med['cuda_fwd'], 2),
                                             'fwd_bwd': round(med['eager_fwd_bwd'] / med['cuda_fwd_bwd'], 2)},
                        'max_abs_diff_vs_eager': diff})
    return out


def time_step(steps=30):
    model, _ = load('ViT-B/32')
    txt = model.encode_text(torch.zeros(1, 77, dtype=torch.long).cuda()).detach()
    torch.manual_seed(0); np.random.seed(0)
    net = CPPN(2, 24, 10, 3, act_fn='unbias').cuda()
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
    for _ in range(5):
        step()
    walls = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            step()
        torch.cuda.synchronize()
        walls.append((time.perf_counter() - t0) * 1e3 / steps)
    return {'frame': '512x512', 'nf': 24, 'layers': 10, 'model': 'ViT-B/32', 'samples': 50, 'step_ms': [round(w, 3) for w in walls],
            'steps_per_s_median': round(1e3 / float(np.median(walls)), 2)}


def main():
    assert torch.cuda.is_available(), 'prof_cppn.py measures on the GPU'
    res = {'card': card(), 'cudnn_allow_tf32': torch.backends.cudnn.allow_tf32, 'generator': time_generator(), 'step': time_step()}
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
