"""Times the spectrum -> RGB synthesis (forward and backward, C ABI calls on resident buffers) at the BASELINE canvas sizes.

    python profiles/prof_synth.py > synth_times.json
Algorithmic HBM bytes (DESIGN.md 4): forward = params + scale read, x_raw + out written (+ the complex intermediate T written and
read once, L2-resident at 720p); backward = grad_out + out + x_raw read, grad_params written (+ g_img and T round trips)."""
import ctypes as C
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from aphantasia_b200 import _lib  # noqa: E402
from aphantasia_b200.image import FFTImage, _color_matrix_host  # noqa: E402


def main():
    lib, ck = _lib.lib(), _lib.check
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, 'MEASURED_PEAKS.json')))
    except Exception:
        pass
    hbm = peaks.get('hbm_gbs', 6650.0)
    out = {'hbm_gbs_peak': hbm, 'rows': []}
    flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')
    for (h, w) in ((720, 1280), (1080, 1920), (2160, 3840)):
        wh = w // 2 + 1
        p = (0.01 * torch.randn(1, 3, h, wh, 2)).cuda()
        gen = FFTImage(p, h, w, 1.5)
        cm = _color_matrix_host(1.8)
        f32 = dict(device='cuda', dtype=torch.float32)
        x_raw = torch.empty(3, h, w, **f32); rgb = torch.empty(3, h, w, **f32); stats = torch.zeros(4, device='cuda', dtype=torch.float64)
        g = torch.randn(3, h, w, **f32); gp = torch.empty_like(p)
        st = _lib.stream_ptr()

        def fwd():
            ck(lib.aph_synth_fft_fwd(gen.plan, p.data_ptr(), gen.scale.data_ptr(), None, 0, 1.0, cm, 1, x_raw.data_ptr(), stats.data_ptr(), rgb.data_ptr(), st), 'fwd')

        def bwd():
            ck(lib.aph_synth_fft_bwd(gen.plan, g.data_ptr(), rgb.data_ptr(), x_raw.data_ptr(), stats.data_ptr(), gen.scale.data_ptr(), 1.0, cm, 1, gp.data_ptr(), st), 'bwd')
        res = {}
        for name, fn in (('fwd', fwd), ('bwd', bwd)):
            for _ in range(3):
                fn()
            tot = 0.
            for _ in range(10):
                flush.fill_(1)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(); fn(); e1.record(); torch.cuda.synchronize()
                tot += e0.elapsed_time(e1)
            res[name] = tot / 10
        n_spec, n_img = 3 * h * wh * 8, 3 * h * w * 4
        alg_f = n_spec + h * wh * 4 + 2 * n_img            # params + scale -> x_raw + out
        alg_b = 3 * n_img + n_spec + h * wh * 4            # grad_out + out + x_raw (+ scale) -> grad_params
        out['rows'].append({'canvas': '%dx%d' % (w, h), 'fwd_ms': round(res['fwd'], 4), 'bwd_ms': round(res['bwd'], 4),
                            'fwd_alg_MB': round(alg_f / 1e6, 1), 'bwd_alg_MB': round(alg_b / 1e6, 1),
                            'fwd_frac_of_hbm': round(alg_f / (res['fwd'] * 1e-3) / 1e9 / hbm, 3), 'bwd_frac_of_hbm': round(alg_b / (res['bwd'] * 1e-3) / 1e9 / hbm, 3)})
    print(json.dumps(out, indent=1))


if __name__ == '__main__':
    main()
