"""Times BASELINE config 3's device-resident step (clip_fft.py --dwt, 1920x1080, ViT-B/16, --samples 200 -> 47 crops) with the
wavelets db3 (6 taps), coif4 (24), coif6 (36) and sym20 (40): the DWT synthesis forward and its adjoint cost grows with L^2.

The step is bench.py's DeviceStep with the wavelet generator in place of the spectrum: direct C-ABI calls on resident buffers,
aph_synth_dwt_fwd -> aph_sample_fwd -> aph_vit_fwd -> aph_sim_fwd -> aph_vit_bwd -> aph_sample_bwd_scaled -> aph_synth_dwt_bwd
with the Adam update fused in (what APH_FUSED_ADAM=1 runs). Synthetic ViT-B/16 weights, seeded. Every wavelet is built and warmed
up first; then ROUNDS rounds time STEPS steps of each wavelet in turn (CUDA events around the whole window), and one more
step per wavelet is split by events into synthesis forward, synthesis backward + Adam, and the rest. Medians are printed as
one JSON line with the card's name, power limit and SM clocks.

    python profiles/prof_dwt_waves.py > dwt_waves.json
"""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from aphantasia_b200 import _lib, _rng  # noqa: E402
from aphantasia_b200._wavelets import reconstruction_filters  # noqa: E402
from aphantasia_b200.clip import VisionTransformer, synthetic_visual_state_dict  # noqa: E402
from aphantasia_b200.image import DWTImage, _color_matrix_host  # noqa: E402

H, W, S, PATCH = 1080, 1920, 47, 16
WAVES = ('db3', 'coif4', 'coif6', 'sym20')
STEPS, WARMUP, ROUNDS, TABLES = 20, 5, 5, 8


def _ptrs(ts):
    return (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


class DWTStep:
    def __init__(self, wave, vis, txt, tables):
        self.lib, self.ck = _lib.lib(), _lib.check
        self.vis, self.txt, self.tables = vis, txt, tables
        self.gen = DWTImage([1, 3, H, W], wave, 0.3)
        self.taps = len(reconstruction_filters(wave)[0])
        g = torch.Generator().manual_seed(0)
        self.Ys = [(0.1 * torch.randn(sh, generator=g)).cuda() for sh in self.gen.param_shapes()]
        self.m = [torch.zeros_like(y) for y in self.Ys]
        self.v = [torch.zeros_like(y) for y in self.Ys]
        self.colmat = _color_matrix_host(1.8)
        oh, ow = self.gen.out_hw
        self.hw = (oh, ow)
        f32 = dict(device='cuda', dtype=torch.float32)
        self.x_raw = torch.empty(3, oh, ow, **f32); self.rgb = torch.empty(3, oh, ow, **f32); self.g_rgb = torch.empty_like(self.rgb)
        self.stats = torch.zeros(4, device='cuda', dtype=torch.float64)
        self.crops = torch.empty(S, 3, 224, 224, **f32); self.g_crops = torch.empty_like(self.crops)
        self.emb = torch.empty(S, 512, **f32); self.g_emb = torch.empty_like(self.emb)
        self.loss = torch.zeros((), **f32)
        self.t = 0
        self.ev = None

    def _mark(self, name):
        if self.ev is not None:
            e = torch.cuda.Event(enable_timing=True); e.record(); self.ev.append((name, e))

    def step(self, i):
        lib, ck, st = self.lib, self.ck, _lib.stream_ptr()
        oh, ow = self.hw
        tab = self.tables[i % self.tables.shape[0]]
        self._mark('start')
        ck(lib.aph_synth_dwt_fwd(self.gen.plan, _ptrs(self.Ys), self.gen.scales_c, 1.0, self.colmat, 1, self.x_raw.data_ptr(),
                                 self.stats.data_ptr(), self.rgb.data_ptr(), st), 'synth_dwt_fwd')
        self._mark('synth_fwd')
        ck(lib.aph_sample_fwd(self.rgb.data_ptr(), oh, ow, 0, 0, tab.data_ptr(), S, 224, 2, self.crops.data_ptr(), st), 'sample_fwd')
        ck(lib.aph_vit_fwd(self.vis.handle, self.crops.data_ptr(), S, self.emb.data_ptr(), 1, st), 'vit_fwd')
        ck(lib.aph_sim_fwd(self.txt.data_ptr(), 1, self.emb.data_ptr(), S, 512, 1, self.loss.data_ptr(), None, self.g_emb.data_ptr(), st), 'sim')
        self.g_emb.mul_(-1.0)
        ck(lib.aph_vit_bwd(self.vis.handle, self.g_emb.data_ptr(), S, self.g_crops.data_ptr(), st), 'vit_bwd')
        ck(lib.aph_sample_bwd_scaled(self.g_crops.data_ptr(), oh, ow, 0, 0, tab.data_ptr(), S, 224, 2, 1.0, self.g_rgb.data_ptr(), st),
           'sample_bwd')
        self._mark('encoder')
        self.t += 1
        ck(lib.aph_synth_dwt_bwd(self.gen.plan, self.g_rgb.data_ptr(), self.rgb.data_ptr(), self.x_raw.data_ptr(), self.stats.data_ptr(),
                                 self.gen.scales_c, 1.0, self.colmat, 1, None, st, _ptrs(self.Ys), _ptrs(self.m), _ptrs(self.v), None,
                                 0.05, 0.0, 0.999, 1e-8, 0.0, self.t), 'synth_dwt_bwd')
        self._mark('synth_bwd_adam')


def window_ms(step, n, first):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for i in range(n):
        step.step(first + i)
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def main():
    torch.manual_seed(0); np.random.seed(0)
    vis = VisionTransformer(synthetic_visual_state_dict(patch=PATCH, seed=0), max_batch=S)
    txt = torch.randn(1, 512, generator=torch.Generator().manual_seed(1234))
    txt = (10. * txt / txt.norm()).cuda()
    tabs = [torch.from_numpy(np.ascontiguousarray(_rng.draw_crop_table(S, (H, W), 224, _rng.TF_FAST, 'uniform', 0.4)[0][0]))
            for _ in range(TABLES)]
    tables = torch.stack(tabs).cuda()
    steps = {w: DWTStep(w, vis, txt, tables) for w in WAVES}
    for st in steps.values():
        window_ms(st, WARMUP, 0)
        assert torch.isfinite(st.loss).item() and all(bool(torch.isfinite(y).all()) for y in st.Ys)
    times = {w: [] for w in WAVES}
    for r in range(ROUNDS):
        for w in (WAVES if r % 2 == 0 else WAVES[::-1]):
            times[w].append(window_ms(steps[w], STEPS, WARMUP + r * STEPS))
    rows = {}
    for w, st in steps.items():
        st.ev = []
        st.step(0); torch.cuda.synchronize()
        split = {n1: e0.elapsed_time(e1) for (_, e0), (n1, e1) in zip(st.ev[:-1], st.ev[1:])}
        rows[w] = {'taps': st.taps,
                   'step_ms_median': float(np.median(times[w])), 'step_ms_runs': [round(t, 3) for t in times[w]],
                   'split_ms': {k: round(v, 3) for k, v in split.items()}}
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm,clocks.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({'workload': 'config 3 device-resident step, %dx%d, S=%d, ViT-B/%d, fused Adam' % (W, H, S, PATCH),
                      'steps_per_run': STEPS, 'runs': ROUNDS, 'gpu': gpu, 'waves': rows}))


if __name__ == '__main__':
    main()
