"""Times the optimiser step stock (torch.optim.Adam / AdamW, foreach) against fused (aphantasia_b200.optim: the update runs
inside the synthesis backward), alternated in one process.

    python profiles/prof_fused_optim.py > fused_optim_times.json

Reports, with the card's name, power limit and maximum SM clock:
  steps  : for each generator at 1280x720 (fft_image, dwt_image coif2, pixel_image) and each -opt choice of the scripts, one
           generator step (synthesis forward, backward from a fixed upstream gradient, optimiser step) with the stock optimiser,
           with the fused one, and without any optimiser (backward only); optimiser work = step - backward only. Wall time per
           step over a window that ends in a device synchronise, and device time between CUDA events; medians of alternated
           rounds;
  frames : illustrip.py's frame (profiles/prof_illustrip.py's loop body, default flags, -opt adam_custom) for --gen RGB and
           --gen FFT, stock against fused, alternated frame blocks, wall time per frame with one synchronise per block."""
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import prof_illustrip as PI  # noqa: E402

from aphantasia_b200 import image, optim  # noqa: E402
from aphantasia_b200.clip import load  # noqa: E402

H, W = PI.H, PI.W
CHOICES = {'adam': ('Adam', {}), 'adam_custom': ('Adam', dict(betas=(.0, .999))), 'adamw': ('AdamW', dict(weight_decay=0.01)),
           'adamw_custom': ('AdamW', dict(weight_decay=0.01, betas=(.0, .999), amsgrad=True))}


def generator(kind):
    torch.manual_seed(0)
    if kind == 'fft':
        params, gen, _ = image.fft_image([1, 3, H, W], 0.01, 1.0)
    elif kind == 'dwt':
        params, gen, _ = image.dwt_image([1, 3, H, W], 'coif2', 0.3, 1.)
    else:
        params, gen, _ = image.pixel_image([1, 3, H, W], sd=1.)
    return params, image.to_valid_rgb(gen, colors=1.5)


def time_steps(rounds=9, reps=100):
    grad_out = torch.randn(1, 3, H, W, device='cuda')
    out = {}
    for kind in ('fft', 'dwt', 'pixel'):
        out[kind] = {}
        for choice, (cls, kw) in CHOICES.items():
            variants = {}
            for name in ('stock', 'fused', 'backward_only'):
                params, rgb = generator(kind)
                opt = None
                if name == 'stock':
                    opt = {'Adam': optim._stock_adam, 'AdamW': optim._stock_adamw}[cls](params, 0.05, **kw)
                elif name == 'fused':
                    opt = getattr(optim, cls)(params, 0.05, **kw)

                def step(params=params, rgb=rgb, opt=opt):
                    if opt is not None:
                        opt.zero_grad()
                    else:
                        for p in params:
                            p.grad = None
                    (rgb() * grad_out).sum().backward()
                    if opt is not None:
                        opt.step()
                variants[name] = step
            for fn in variants.values():
                for _ in range(5):
                    fn()
            wall = {n: [] for n in variants}
            dev = {n: [] for n in variants}
            for _ in range(rounds):
                for n, fn in variants.items():
                    wall[n].append(PI.wall_ms(fn, reps))
                    dev[n].append(PI.events_ms(fn, reps))
            med = lambda xs: float(np.median(xs))
            r = {n: {'wall_ms': round(med(wall[n]), 4), 'device_ms': round(med(dev[n]), 4)} for n in variants}
            for n in ('stock', 'fused'):
                r[n]['optimiser_wall_ms'] = round(med(wall[n]) - med(wall['backward_only']), 4)
                r[n]['optimiser_device_ms'] = round(med(dev[n]) - med(dev['backward_only']), 4)
            r['spread_wall_ms'] = {n: round(max(wall[n]) - min(wall[n]), 4) for n in variants}
            out[kind][choice] = r
    return out


def time_frames(model, txt, rounds=7, frames=10):
    out = {}
    for gen in ('RGB', 'FFT'):
        with tempfile.TemporaryDirectory() as tmp:
            torch.manual_seed(0); np.random.seed(0)
            sides = {'stock': PI.make_frame(gen, model, txt, tmp), 'fused': PI.make_frame(gen, model, txt, tmp)}

            def frame(name):
                (optim.install if name == 'fused' else optim.uninstall)()      # the frame builds its optimiser in its motion phase
                try:
                    for _, fn in sides[name]:
                        fn()
                finally:
                    optim.uninstall()
            for name in sides:
                for _ in range(3):
                    frame(name)
            ms = {n: [] for n in sides}
            for _ in range(rounds):
                for name in sides:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for _ in range(frames):
                        frame(name)
                    torch.cuda.synchronize()
                    ms[name].append((time.perf_counter() - t0) * 1e3 / frames)
            out[gen] = {n: {'frame_ms_median': round(float(np.median(v)), 3), 'frame_ms_min': round(min(v), 3),
                            'frame_ms_max': round(max(v), 3)} for n, v in ms.items()}
    return out


def main():
    assert torch.cuda.is_available(), 'prof_fused_optim.py measures on the GPU'
    res = {'card (name, power limit, max SM clock)': PI.card(), 'canvas': '%dx%d' % (W, H), 'steps': time_steps()}
    model, _ = load('ViT-B/32')
    txt = model.encode_text(torch.zeros(1, 77, dtype=torch.long).cuda()).detach()
    PI.motion.install()
    res['illustrip_frames'] = time_frames(model, txt)
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
