"""The wide ResNet image towers on one GPU, at the crop counts clip_fft.py's defaults give them (samples 200 x the script's
per-model memory scale x 0.95 for the default transforms: RN50x4 30 crops of 288, RN50x16 11 of 384; RN50x64, which clip_fft.py
does not list, at 11 crops of 448, since cppn.py's defaults give it a single crop: 50 x 0.04 x 0.95). For each it reports:
  - the tower's forward and forward + data gradient, with TFLOP/s from the useful MAC count (real channel counts; the README's
    counting, 6.01 GMAC for RN50) and, separately, the extra MACs of the zero channel padding to multiples of 64;
  - the same tower as eager fp16 torch ops (tests/clip_resnet_oracle.py in fp16: cuDNN convolutions) on the same GPU;
  - device-resident steps/s of the 1280x720 FFT step (profiles/prof_clip_resnet.py's step at the tower's crop side).
Every timing runs 3 warm-up calls first. The card name, its power limit and its maximum SM clock are printed with the numbers.
Usage: python profiles/prof_clip_resnet_wide.py [--steps 10] [--models RN50x4,RN50x16,RN50x64]"""
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
sys.path.insert(0, os.path.join(ROOT, 'profiles'))
from aphantasia_b200 import _lib, _rng, clip  # noqa: E402
import clip_resnet_oracle as O  # noqa: E402
import prof_clip_resnet as P  # noqa: E402

BATCH = {'RN50x4': 30, 'RN50x16': 11, 'RN50x64': 11}


def macs(layers, width, res, out_dim, padded=False):
    """Forward multiply-accumulates per crop of side res; padded: at the channel counts the tower runs (pad64)."""
    R = clip.pad64 if padded else (lambda c: c)
    c1, h1 = width // 2, (res - 1) // 2 + 1
    m = h1 * h1 * c1 * 27 + h1 * h1 * 9 * (R(c1) * R(c1) + R(c1) * R(width))
    h, cin = h1 // 2, width
    for i, n in enumerate(layers):
        p = width << i
        for j in range(n):
            stride = 2 if (i > 0 and j == 0) else 1
            ho = h // stride
            m += h * h * R(cin) * R(p) + h * h * R(p) * R(p) * 9 + ho * ho * R(p) * 4 * p
            if stride > 1 or cin != 4 * p:
                m += ho * ho * R(cin) * 4 * p
            h, cin = ho, 4 * p
    D, T = 32 * width, (res // 32) ** 2 + 1
    return m + T * D * 3 * D + (width // 2) * T * T * 64 * 2 + D * out_dim


class WideStep(P.ResNetStep):
    """prof_clip_resnet.ResNetStep (synthesis, sampler, tower forward, mix loss, tower data gradient, sampler backward, synthesis
    backward, Adam) with crops of the tower's side."""

    def __init__(self, vis, S, size):
        super().__init__(vis, S)
        self.size = size
        tabs = [torch.from_numpy(np.ascontiguousarray(_rng.draw_crop_table(S, (P.H, P.W), size, _rng.TF_FAST, 'uniform', 0.4)[0][0]))
                for _ in range(4)]
        self.tables = torch.stack(tabs).cuda()
        self.crops = torch.empty(S, 3, size, size, device='cuda'); self.g_crops = torch.empty_like(self.crops)

    def step(self):
        lib, ck, st, S, z = self.lib, _lib.check, _lib.stream_ptr(), self.S, self.size
        tab = self.tables[self.i % self.tables.shape[0]]
        self.i += 1
        ck(lib.aph_synth_fft_fwd(self.gen.plan, self.params.data_ptr(), self.gen.scale.data_ptr(), None, 0, 1.0, self.colmat, 1,
                                 self.x_raw.data_ptr(), self.stats.data_ptr(), self.rgb.data_ptr(), st), 'synth_fwd')
        ck(lib.aph_sample_fwd(self.rgb.data_ptr(), P.H, P.W, 0, 0, tab.data_ptr(), S, z, 2, self.crops.data_ptr(), st), 'sample_fwd')
        ck(lib.aph_rn_fwd(self.vis.handle, self.crops.data_ptr(), S, z, self.emb.data_ptr(), 1, st), 'rn_fwd')
        ck(lib.aph_sim_fwd(self.txt.data_ptr(), 1, self.emb.data_ptr(), S, self.O, 1, self.loss.data_ptr(), None, self.g_emb.data_ptr(), st), 'sim')
        self.g_emb.mul_(-1.0)
        ck(lib.aph_rn_bwd(self.vis.handle, self.g_emb.data_ptr(), S, z, self.g_crops.data_ptr(), st), 'rn_bwd')
        ck(lib.aph_sample_bwd_scaled(self.g_crops.data_ptr(), P.H, P.W, 0, 0, tab.data_ptr(), S, z, 2, 1.0, self.g_rgb.data_ptr(), st), 'sample_bwd')
        ck(lib.aph_synth_fft_bwd(self.gen.plan, self.g_rgb.data_ptr(), self.rgb.data_ptr(), self.x_raw.data_ptr(), self.stats.data_ptr(),
                                 self.gen.scale.data_ptr(), 1.0, self.colmat, 1, self.g_params.data_ptr(), st), 'synth_bwd')
        self.t += 1
        ck(lib.aph_adam_step(self.params.data_ptr(), self.g_params.data_ptr(), self.m.data_ptr(), self.v.data_ptr(), self.params.numel(),
                             0.05, 0.0, 0.999, 1e-8, self.t, st), 'adam')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--models', default='RN50x4,RN50x16,RN50x64')
    a = ap.parse_args()
    try:
        card = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        card = 'unknown'
    res = {'gpu': torch.cuda.get_device_name(0), 'power_limit, max_sm_clock': card}
    for name in a.models.split(','):
        cfg = clip._MODELS[name]
        S, z = BATCH[name], cfg['res']
        sd = clip.synthetic_resnet_state_dict(**cfg)
        vis = clip.ModifiedResNet(sd, max_batch=S)
        x = torch.randn(S, 3, z, z, device='cuda')
        g = torch.randn(S, cfg['out_dim'], device='cuda')
        xr = x.clone().requires_grad_(True)
        with torch.no_grad():
            fwd_ms = P._time(lambda: vis(x), a.steps)
        both_ms = P._time(lambda: torch.autograd.grad(vis(xr), xr, g), a.steps)
        step = WideStep(vis, S, z)
        step_ms = P._time(step.step, a.steps)
        del step
        mac = macs(cfg['layers'], cfg['width'], z, cfg['out_dim'])
        pad = macs(cfg['layers'], cfg['width'], z, cfg['out_dim'], padded=True) - mac
        hsd = {k[len('visual.'):]: v.cuda() for k, v in sd.items() if k.startswith('visual.')}
        del sd
        xh = x.half().requires_grad_(True)
        with torch.no_grad():
            eager_fwd = P._time(lambda: O.forward(hsd, x, dtype=torch.float16), a.steps)
        eager_both = P._time(lambda: torch.autograd.grad(O.forward(hsd, xh, dtype=torch.float16), xh, g.half()), a.steps)
        res[name] = {'S': S, 'side': z, 'gmac_per_crop': mac / 1e9, 'padding_gmac_per_crop': pad / 1e9,
                     'fwd_ms': fwd_ms, 'fwd_plus_bwd_ms': both_ms,
                     'fwd_tflops': 2 * mac * S / fwd_ms / 1e9, 'fwd_plus_bwd_tflops': 4 * mac * S / both_ms / 1e9,
                     'eager_fp16_fwd_ms': eager_fwd, 'eager_fp16_fwd_plus_bwd_ms': eager_both,
                     'fft_step_ms': step_ms, 'fft_step_steps_per_s': 1e3 / step_ms}
        print(json.dumps({name: res[name]}), flush=True)
        vis.close()
        del hsd, vis
        torch.cuda.empty_cache()
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
