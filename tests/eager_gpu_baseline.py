"""Not a pytest module: times the oracle restatement of the reference step as plain PyTorch-eager CUDA ops on the GPU box.

BASELINE.md section 3, item 5 ("second baseline"): the reference has no GPU kernels of its own; on a GPU it runs
as a few hundred ATen launches per crop plus cuBLAS/cuDNN inside CLIP. the original project is not part of this repository, so
the op sequence executed here is oracle/restate.py (same per-crop interpolate / grid_sample / normalise loop, same CLIP
module layout), placed on the device with torch.set_default_device('cuda') -- the device-context mode costs about a
microsecond per op, small against the ~10 us of an eager launch. CLIP runs in fp16 as clip.load() does on a GPU.

    python tests/eager_gpu_baseline.py [steps] > eager_gpu_baseline.json
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

H, W, S = 720, 1280, 190


VARIANTS = (('fp16_clip_with_weight_grads', torch.float16, True), ('fp16_clip_frozen', torch.float16, False),
            ('fp32_clip_frozen', torch.float32, False))


def measure(steps=8, names=None):
    from aphantasia_b200 import _rng
    from aphantasia_b200.clip import synthetic_visual_state_dict
    from oracle import restate as R
    torch.manual_seed(0); np.random.seed(0)
    tabs, _ = _rng.draw_crop_table(S, (H, W), 224, _rng.TF_FAST, 'uniform', 0.4)
    params0 = 0.01 * torch.randn(1, 3, H, W // 2 + 1, 2)
    scale, cm = R.fft_scale(H, W, 1.5).cuda(), R.color_matrix(1.8).cuda()
    g = torch.Generator().manual_seed(1234)
    txt = torch.randn(1, 512, generator=g); txt = (10. * txt / txt.norm()).cuda()
    sd = synthetic_visual_state_dict(patch=32, seed=0)
    prev_dev = torch.get_default_device()
    torch.set_default_device('cuda')
    results = {}
    for name, dtype, wgrad in VARIANTS:
        if names is not None and name not in names:
            continue
        vis = R.build_visual(sd).cuda()
        if dtype == torch.float16:                   # clip.model.convert_weights: everything but the LayerNorms goes to fp16
            vis.half()
            for m in vis.modules():
                if isinstance(m, torch.nn.LayerNorm):
                    m.float()
        vis.requires_grad_(wgrad)
        p = params0.cuda().requires_grad_(True)
        opt = torch.optim.Adam([p], 0.05, betas=(.0, .999))

        def step():
            rgb = R.valid_rgb(R.synth_fft(p, scale, H, W, None, 1.), cm)
            crops = R.sample_crops(rgb, tabs[0], 224, 2)
            emb = vis(crops.to(dtype)).float()
            loss = -1. * R.sim_func(txt, emb, 'mix')
            opt.zero_grad()
            loss.backward()
            opt.step()
            return loss.item()

        for _ in range(2):
            step()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            last = step()
        e1.record(); torch.cuda.synchronize()
        t = e0.elapsed_time(e1) / 1e3 / steps
        results[name] = {'steps_per_s': 1.0 / t, 'ms_per_step': 1e3 * t, 'loss': last}
        del vis, p, opt
        torch.cuda.empty_cache()
    torch.set_default_device(prev_dev)
    return results


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 8
    results = measure(steps)
    print(json.dumps({'workload': 'C2: 1280x720 FFT, S=190, ViT-B/32, transforms_fast, mix loss, Adam; PyTorch-eager CUDA ops (oracle restatement)',
                      'steps': steps, 'device': torch.cuda.get_device_name(0), 'results': results}))


if __name__ == '__main__':
    main()
