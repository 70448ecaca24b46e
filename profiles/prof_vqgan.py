"""The VQGAN decoder of CLIP_VQGAN.ipynb on one GPU, at the notebook's default 900 x 500 (latent 31 x 56 at f16, 62 x 112 at f8,
496 x 896 out). For both decoders it reports:
  - the CUDA decoder's forward and forward + d loss / d z, with achieved TFLOP/s from the count below;
  - the same decoder as eager fp32 torch (tests/vqgan_oracle.py in fp32, weights requiring grad: what the notebook runs, weight
    gradients included) and under bf16 autocast;
  - FLOPs from shapes: 2 x the multiply-accumulates of every convolution, 1x1 convolution and attention GEMM of the forward; the
    data gradient costs the same again, so forward + d z counts twice the forward.
Then the notebook's Generate-cell step at samples = 60 (lats -> decoder -> (x + 1) / 2 -> slice_imgs(transforms_fast) -> ViT-B/32
-> cosine loss -> backward -> AdamW amsgrad) with synthetic weights, steps/s. Every timing runs 3 warm-up calls first (the first
call runs eagerly, the second captures the CUDA graph, later ones replay it). The card name and its power limit are printed with
the numbers.
Usage: python profiles/prof_vqgan.py [--steps 10]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from aphantasia_b200 import transforms, vqgan  # noqa: E402
from aphantasia_b200.clip import CLIP, synthetic_visual_state_dict  # noqa: E402
from aphantasia_b200.utils import slice_imgs  # noqa: E402
import vqgan_oracle as VO  # noqa: E402

LATENTS = {'F16_CONFIG': (31, 56), 'F8_CONFIG': (62, 112)}


def flops(cfg, h, w):
    """2 x the forward's multiply-accumulates"""
    ch, mult, nrb, zc = cfg['ch'], cfg['ch_mult'], cfg['num_res_blocks'], cfg['z_channels']
    attn = vqgan._attn_levels(mult, cfg['resolution'], cfg['attn_resolutions'])
    L = len(mult)
    px = h * w
    bi = ch * mult[-1]
    m = px * 9 * zc * bi

    def res(px, ci, co):
        return px * 9 * (ci * co + co * co) + (px * ci * co if ci != co else 0)

    def att(px, c):
        return px * 4 * c * c + 2 * px * px * c

    m += 2 * res(px, bi, bi) + att(px, bi)
    for i in reversed(range(L)):
        bo = ch * mult[i]
        for _ in range(nrb + 1):
            m += res(px, bi, bo)
            bi = bo
            if i in attn:
                m += att(px, bi)
        if i:
            px *= 4
            m += px * 9 * bi * bi
    m += px * 9 * bi * 3
    return 2 * m


def _time(fn, steps, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    a = ap.parse_args()
    try:
        power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'], capture_output=True,
                               text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = 'unknown'
    res = {'gpu': torch.cuda.get_device_name(0), 'power_limit': power}
    for name, (h, w) in LATENTS.items():
        cfg = getattr(vqgan, name)
        sd = vqgan.synthetic_decoder_state_dict(0, **cfg)
        dec = vqgan.Decoder(**cfg)
        dec.load_state_dict(sd)
        dec = dec.cuda().eval()
        z = torch.randn(1, 256, h, w, device='cuda')
        zr = z.clone().requires_grad_(True)
        g = torch.randn(1, 3, 8 * h if name == 'F8_CONFIG' else 16 * h, 8 * w if name == 'F8_CONFIG' else 16 * w, device='cuda')
        with torch.no_grad():
            fwd = _time(lambda: dec(z), a.steps)
        both = _time(lambda: torch.autograd.grad(dec(zr), zr, g), a.steps)
        wsd = {k: v.cuda().requires_grad_(True) for k, v in sd.items()}
        lev = dec.attn_levels

        def eager(zz):
            return VO.decode(wsd, zz, cfg['ch_mult'], cfg['num_res_blocks'], lev)

        def eager_both():
            out = eager(zr)
            torch.autograd.backward(out, g)            # the notebook's parameters require grad: weight gradients too

        with torch.no_grad():
            e_fwd = _time(lambda: eager(z), a.steps)
        e_both = _time(eager_both, a.steps)
        with torch.autocast('cuda', dtype=torch.bfloat16):
            with torch.no_grad():
                b_fwd = _time(lambda: eager(z), a.steps)
            b_both = _time(eager_both, a.steps)
        del wsd
        f = flops(cfg, h, w)
        res[name] = {'latent': [h, w], 'gflop_fwd': f / 1e9, 'fwd_ms': fwd, 'fwd_plus_dz_ms': both,
                     'fwd_tflops': f / fwd / 1e9, 'fwd_plus_dz_tflops': 2 * f / both / 1e9,
                     'eager_fp32_fwd_ms': e_fwd, 'eager_fp32_fwd_plus_bwd_ms': e_both,
                     'eager_bf16_autocast_fwd_ms': b_fwd, 'eager_bf16_autocast_fwd_plus_bwd_ms': b_both}
        if name == 'F8_CONFIG':
            model = CLIP('ViT-B/32', synthetic_visual_state_dict(patch=32, seed=0), True)
            txt = model.encode_text(torch.zeros(1, 77, dtype=torch.long)).cuda()
            lats = (torch.randn(1, 256, h, w, device='cuda') * 0.5).requires_grad_(True)
            opt = torch.optim.AdamW([lats], lr=0.1, weight_decay=0.1, amsgrad=True)
            torch.manual_seed(0); np.random.seed(0)

            def step():
                opt.zero_grad()
                img = (dec(lats) + 1.) / 2.
                crops = slice_imgs([img], 60, 224, transforms.transforms_fast, 'uniform', 0.4)[0]
                loss = -torch.cosine_similarity(txt, model.encode_image(crops), dim=-1).mean()
                loss.backward()
                opt.step()

            ms = _time(step, a.steps)
            res['notebook_step_f8_samples60'] = {'ms': ms, 'steps_per_s': 1e3 / ms}
            model.visual.close()
        dec._handle.close()
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
