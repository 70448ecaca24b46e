"""The ResNet image towers on one GPU. For RN50 at S = 100 crops and RN101 at S = 66 (the crop counts clip_fft.py --samples 200
gives them) it reports:
  - device-resident steps/s of the 1280x720 FFT step (bench.py's DeviceStep with the ViT replaced by the ResNet: synthesis,
    sampler, tower forward, mix loss, tower data gradient, sampler backward, synthesis backward, Adam; C-ABI calls only);
  - the tower's forward and forward + data gradient, with achieved TFLOP/s from the MAC count below;
  - the same tower as eager fp16 torch ops (tests/clip_resnet_oracle.py in fp16: cuDNN convolutions) on the same GPU.
Every timing runs 3 warm-up calls first: the first call of a batch size runs eagerly, the second captures the CUDA graph, later
ones replay it. The card name and its power limit are printed with the numbers.
Usage: python profiles/prof_clip_resnet.py [--steps 20]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from aphantasia_b200 import _lib, _rng, clip  # noqa: E402
from aphantasia_b200.image import FFTImage, _color_matrix_host  # noqa: E402
import clip_resnet_oracle as O  # noqa: E402

H, W = 720, 1280


def macs(layers, side=224, out_dim=1024):
    """(useful forward multiply-accumulates per crop, the extra ones of the stem's zero padding to 64 channels)."""
    h1 = (side - 1) // 2 + 1
    m = h1 * h1 * 32 * 27 + h1 * h1 * 9 * (32 * 32 + 32 * 64)
    padding = h1 * h1 * 9 * (64 * 64 - 32 * 32) + h1 * h1 * 9 * (64 * 64 - 32 * 64)
    h, cin = h1 // 2, 64
    for i, n in enumerate(layers):
        P = 64 << i
        for j in range(n):
            stride = 2 if (i > 0 and j == 0) else 1
            ho = h // stride
            m += h * h * cin * P + h * h * P * P * 9 + ho * ho * P * 4 * P
            if stride > 1 or cin != 4 * P:
                m += ho * ho * cin * 4 * P
            h, cin = ho, 4 * P
    D = 2048
    m += 50 * D * 3 * D + 32 * 50 * 50 * 64 * 2 + D * out_dim
    return m, padding


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


class ResNetStep:
    """bench.py's device-resident FFT step with the ResNet tower as the encoder (crops of 224, transforms_fast, mix loss)."""

    def __init__(self, vis, S):
        self.lib, self.vis, self.S, self.O = _lib.lib(), vis, S, vis.output_dim
        dev = torch.device('cuda')
        torch.manual_seed(0); np.random.seed(0)
        self.params = (0.01 * torch.randn(1, 3, H, W // 2 + 1, 2)).to(dev)
        self.gen = FFTImage(self.params, H, W, 1.5)
        self.colmat = _color_matrix_host(1.8)
        g = torch.Generator().manual_seed(1234)
        txt = torch.randn(1, self.O, generator=g); self.txt = (10. * txt / txt.norm()).to(dev)
        tabs = [torch.from_numpy(np.ascontiguousarray(_rng.draw_crop_table(S, (H, W), 224, _rng.TF_FAST, 'uniform', 0.4)[0][0]))
                for _ in range(4)]
        self.tables = torch.stack(tabs).to(dev)
        f32 = dict(device=dev, dtype=torch.float32)
        self.x_raw, self.rgb = torch.empty(3, H, W, **f32), torch.empty(3, H, W, **f32)
        self.stats = torch.zeros(4, device=dev, dtype=torch.float64)
        self.crops = torch.empty(S, 3, 224, 224, **f32); self.g_crops = torch.empty_like(self.crops)
        self.emb = torch.empty(S, self.O, **f32); self.g_emb = torch.empty_like(self.emb)
        self.loss = torch.zeros((), **f32)
        self.g_rgb = torch.empty(3, H, W, **f32); self.g_params = torch.empty_like(self.params)
        self.m, self.v = torch.zeros_like(self.params), torch.zeros_like(self.params)
        self.t, self.i = 0, 0

    def step(self):
        lib, ck, st, S = self.lib, _lib.check, _lib.stream_ptr(), self.S
        tab = self.tables[self.i % self.tables.shape[0]]
        self.i += 1
        ck(lib.aph_synth_fft_fwd(self.gen.plan, self.params.data_ptr(), self.gen.scale.data_ptr(), None, 0, 1.0, self.colmat, 1,
                                 self.x_raw.data_ptr(), self.stats.data_ptr(), self.rgb.data_ptr(), st), 'synth_fwd')
        ck(lib.aph_sample_fwd(self.rgb.data_ptr(), H, W, 0, 0, tab.data_ptr(), S, 224, 2, self.crops.data_ptr(), st), 'sample_fwd')
        ck(lib.aph_rn_fwd(self.vis.handle, self.crops.data_ptr(), S, 224, self.emb.data_ptr(), 1, st), 'rn_fwd')
        ck(lib.aph_sim_fwd(self.txt.data_ptr(), 1, self.emb.data_ptr(), S, self.O, 1, self.loss.data_ptr(), None, self.g_emb.data_ptr(), st), 'sim')
        self.g_emb.mul_(-1.0)
        ck(lib.aph_rn_bwd(self.vis.handle, self.g_emb.data_ptr(), S, 224, self.g_crops.data_ptr(), st), 'rn_bwd')
        ck(lib.aph_sample_bwd_scaled(self.g_crops.data_ptr(), H, W, 0, 0, tab.data_ptr(), S, 224, 2, 1.0, self.g_rgb.data_ptr(), st), 'sample_bwd')
        ck(lib.aph_synth_fft_bwd(self.gen.plan, self.g_rgb.data_ptr(), self.rgb.data_ptr(), self.x_raw.data_ptr(), self.stats.data_ptr(),
                                 self.gen.scale.data_ptr(), 1.0, self.colmat, 1, self.g_params.data_ptr(), st), 'synth_bwd')
        self.t += 1
        ck(lib.aph_adam_step(self.params.data_ptr(), self.g_params.data_ptr(), self.m.data_ptr(), self.v.data_ptr(), self.params.numel(),
                             0.05, 0.0, 0.999, 1e-8, self.t, st), 'adam')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    a = ap.parse_args()
    try:
        power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'], capture_output=True,
                               text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = 'unknown'
    res = {'gpu': torch.cuda.get_device_name(0), 'power_limit': power}
    for name, S in (('RN50', 100), ('RN101', 66)):
        cfg = clip._MODELS[name]
        sd = clip.synthetic_resnet_state_dict(**cfg)
        vis = clip.ModifiedResNet(sd, max_batch=S)
        step = ResNetStep(vis, S)
        step_ms = _time(step.step, a.steps)
        x = torch.randn(S, 3, 224, 224, device='cuda')
        g = torch.randn(S, cfg['out_dim'], device='cuda')
        xr = x.clone().requires_grad_(True)
        with torch.no_grad():
            fwd_ms = _time(lambda: vis(x), a.steps)
        both_ms = _time(lambda: torch.autograd.grad(vis(xr), xr, g), a.steps)
        mac, pad = macs(cfg['layers'], 224, cfg['out_dim'])
        hsd = {k[len('visual.'):]: v.cuda() for k, v in sd.items() if k.startswith('visual.')}
        xh = x.half().requires_grad_(True)
        with torch.no_grad():
            eager_fwd = _time(lambda: O.forward(hsd, x, dtype=torch.float16), a.steps)
        eager_both = _time(lambda: torch.autograd.grad(O.forward(hsd, xh, dtype=torch.float16), xh, g.half()), a.steps)
        res[name] = {'S': S, 'fft_step_steps_per_s': 1e3 / step_ms, 'fft_step_ms': step_ms,
                     'gmac_per_crop': mac / 1e9, 'stem_padding_gmac_per_crop': pad / 1e9,
                     'fwd_ms': fwd_ms, 'fwd_plus_bwd_ms': both_ms,
                     'fwd_tflops': 2 * mac * S / fwd_ms / 1e9, 'fwd_plus_bwd_tflops': 4 * mac * S / both_ms / 1e9,
                     'eager_fp16_fwd_ms': eager_fwd, 'eager_fp16_fwd_plus_bwd_ms': eager_both}
        vis.close()
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
