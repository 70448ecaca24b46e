"""Times LPIPS (net='vgg') forward + canvas gradient at 360 x 640 (clip_fft.py --sync's sim size for the 1280 x 720 canvas) and at
1080 x 1920 (a 3840 x 2160 canvas), with the achieved rate from the FLOP count of the 13 convolutions (forward, and the same again
for the data gradient), and the whole --sync step at 1280 x 720 against the plain step: fft_image -> slice_imgs (fast transforms)
-> ViT-B/32 -> mix similarity (+ LPIPS of the bicubic-resized canvas against a fixed picture) -> backward -> Adam. The plain step
has S = 190 crops (--samples 200 x 0.95), the --sync step S = 95 (halved first). CUDA events, median of 10 after 3 warm-ups.
Synthetic weights (the timing does not depend on their values). Reads the card's name and power limit in the same run.

    python profiles/prof_lpips.py > lpips_times.json
"""
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from aphantasia_b200 import lpips as L, transforms  # noqa: E402
from aphantasia_b200.clip import CLIP, synthetic_visual_state_dict  # noqa: E402
from aphantasia_b200.image import fft_image, to_valid_rgb  # noqa: E402
from aphantasia_b200.utils import sim_func, slice_imgs  # noqa: E402


def conv_flops(h, w):
    """2 * pixels * C_out * 9 * C_in summed over the 13 convolutions of VGG16 features[0:30] (floor-mode pools)."""
    total, lvl = 0, 0
    for i, (ci, co) in zip(L.VGG_CONVS, L.VGG_CH):
        hh, ww = h, w
        for _ in range(lvl):
            hh, ww = hh // 2, ww // 2
        total += 2 * hh * ww * co * 9 * ci
        if i + 1 in (3, 8, 15, 22):           # features[i + 1] is the tap's ReLU; a max-pool follows
            lvl += 1
    return total


def timed(fn, reps=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def main():
    torch.backends.cudnn.benchmark = False
    rows = {}
    m = L.LPIPS(net='vgg', verbose=False, vgg_state_dict=L.synthetic_vgg_state_dict(), lin_state_dict=L.synthetic_lin_state_dict())
    for h, w in ((360, 640), (1080, 1920)):
        torch.manual_seed(0)
        ref = torch.rand(1, 3, h, w, device='cuda')
        x = torch.rand(1, 3, h, w, device='cuda', requires_grad=True)

        def fwd_bwd():
            v = m(x, ref, normalize=True)
            torch.autograd.grad(v.sum(), x)

        def fwd():
            with torch.no_grad():
                m(x, ref, normalize=True)

        t_fb, t_f = timed(fwd_bwd), timed(fwd)
        fl = conv_flops(h, w)
        rows['%dx%d' % (h, w)] = {'fwd_ms': t_f, 'fwd_bwd_ms': t_fb, 'conv_gflop_fwd': fl / 1e9,
                                  'tflops_fwd': fl / t_f / 1e9, 'tflops_fwd_bwd': 2 * fl / t_fb / 1e9}

    # the whole step at 1280 x 720 (clip_fft.py:239-295 with --sync, reference features cached after the first call)
    H, W = 720, 1280
    model = CLIP('ViT-B/32', synthetic_visual_state_dict(patch=32, seed=0), True)
    txt = model.encode_text(torch.zeros(1, 77, dtype=torch.long)).cuda()
    img_in = F.interpolate(torch.rand(1, 3, H, W, device='cuda', dtype=torch.float64), (H // 2, W // 2), mode='bicubic',
                           align_corners=True).float()
    for name, S, sync in (('step_plain_S190', 190, False), ('step_sync_S95', 95, True)):
        torch.manual_seed(0); np.random.seed(0)
        params, image_f, _ = fft_image([1, 3, H, W], 0.07, 1.5, None)
        rgb_f = to_valid_rgb(image_f, colors=1.8)
        opt = torch.optim.Adam(params, 0.05)

        def step():
            img_out = rgb_f()
            crops = slice_imgs([img_out], S, 224, transforms.transforms_fast, 'overscan', 0.4)[0]
            loss = -sim_func(txt, model.encode_image(crops), 'mix')
            if sync:
                loss = loss + 0.5 * m(F.interpolate(img_out, (H // 2, W // 2), mode='bicubic', align_corners=True).float(), img_in,
                                      normalize=True).squeeze()
            opt.zero_grad()
            loss.backward()
            opt.step()

        rows[name + '_ms'] = timed(step)
    rows['sync_over_plain'] = rows['step_sync_S95_ms'] / rows['step_plain_S190_ms']
    rows['gpu'] = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                                 capture_output=True, text=True).stdout.strip()
    print(json.dumps(rows))


if __name__ == '__main__':
    main()
