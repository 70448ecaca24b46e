"""Times starting from a picture file: fft_image(..., path) and coif2 dwt_image(..., path) on a 3840 x 2160 PNG, end to end
and split into decode (PIL, host clock), upload (3 bytes per pixel, CUDA events) and kernels (aph_un_rgb + aph_fft_analyze or
aph_dwt_analyze, CUDA events), median of 5 after one warm-up. Init-time work: run once per run of the script.

    python profiles/prof_resume.py > resume_times.json
"""
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from aphantasia_b200 import _lib, image  # noqa: E402
from aphantasia_b200.utils import img_read  # noqa: E402


def events_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); r = fn(); b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b), r


def wall_ms(fn):
    torch.cuda.synchronize(); t = time.perf_counter(); r = fn(); torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3, r


def main():
    lib, ck, st = _lib.lib(), _lib.check, _lib.stream_ptr
    h, w = 2160, 3840
    rng = np.random.RandomState(0)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    img = np.stack([128 + 90 * np.sin(2 * np.pi * (xx / w * (k + 1) + yy / h * (2 - k))) for k in range(3)], -1)
    img = np.clip(img + rng.normal(0, 20, (h, w, 3)), 0, 255).astype(np.uint8)
    rows = {}
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, 'pic.png')
        Image.fromarray(img).save(path)
        rows['png_bytes'] = os.path.getsize(path)
        minv = (C.c_float * 9)(*[float(v) for v in torch.linalg.inv(image._color_correlation(1.6).T).T.reshape(-1)])
        fplan = C.c_void_p()
        ck(lib.aph_fft_plan_create(C.byref(fplan), h, w), 'plan')
        dgen = image.DWTImage([1, 3, h, w], 'coif2', 0.3)
        ascale = image._analysis_scale(h, w // 2 + 1, 1.5, 0.07).cuda()
        spec = torch.empty(1, 3, h, w // 2 + 1, 2, device='cuda')
        Ys = [torch.empty(sh, device='cuda') for sh in dgen.param_shapes()]
        ptrs = (C.c_void_p * len(Ys))(*[y.data_ptr() for y in Ys])
        inv = (C.c_float * dgen.J)(*[1. / s for s in dgen.scales])
        x = torch.empty(1, 3, h, w, device='cuda')
        host_src = torch.from_numpy(img)
        parts = {k: [] for k in ('decode', 'upload', 'un_rgb', 'fft_analyze', 'dwt_analyze', 'fft_image_total', 'dwt_image_total')}
        for it in range(6):
            t = time.perf_counter(); dec = img_read(path); td = (time.perf_counter() - t) * 1e3
            tu, src = events_ms(lambda: host_src.cuda())
            tr, _ = events_ms(lambda: ck(lib.aph_un_rgb(src.data_ptr(), h, w, minv, 1.0, x.data_ptr(), st()), 'un_rgb'))
            tf, _ = events_ms(lambda: ck(lib.aph_fft_analyze(fplan, x.data_ptr(), ascale.data_ptr(), spec.data_ptr(), st()), 'fft'))
            tw, _ = events_ms(lambda: ck(lib.aph_dwt_analyze(dgen.plan, x.data_ptr(), inv, ptrs, st()), 'dwt'))
            tfi, _ = wall_ms(lambda: image.fft_image([1, 3, 64, 64], 0.07, 1.5, path))
            tdi, _ = wall_ms(lambda: image.dwt_image([1, 3, 64, 64], 'coif2', 0.3, 1.8, path))
            assert dec.shape == img.shape
            if it:
                for k, v in zip(parts, (td, tu, tr, tf, tw, tfi, tdi)):
                    parts[k].append(v)
        lib.aph_fft_plan_destroy(fplan)
    rows.update({k + '_ms': float(np.median(v)) for k, v in parts.items()})
    rows['gpu'] = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                                 capture_output=True, text=True).stdout.strip()
    rows['size'] = [h, w]
    print(json.dumps(rows))


if __name__ == '__main__':
    main()
