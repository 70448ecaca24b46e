"""Sampler cost per transform kind: aph_sample_fwd + aph_sample_bwd_scaled for transforms_fast (2), transforms_custom (3) and
transforms_elastic (4) at C2's geometry (1280x720 canvas, S = 190) and C3's (1920x1080, S = 47), by CUDA events over many calls
after a warm-up; the forward of every kind (0-4) on a frame too large for k_resize's per-warp crop rows; then one step per kind
through the drop-in entry points (FFT synthesis -> slice_imgs -> encode_image -> mix loss -> backward, ViT-B/32 at C2), timed the
same way. Prints one JSON line with the card's name, power limit and SM clock, read in
the same run. Usage: python profiles/prof_sampler_kinds.py [--reps 200] [--steps 30]"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _time(fn, reps):
    import torch
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def sampler(kind, H, W, S, reps):
    import numpy as np
    import torch
    from aphantasia_b200 import _rng
    from aphantasia_b200._lib import check, lib, stream_ptr
    torch.manual_seed(0); np.random.seed(0)
    tabs, _ = _rng.draw_crop_table(S, (H, W), 224, kind, 'uniform', 0.4)
    t = torch.from_numpy(tabs[0]).cuda()
    side = _rng.out_side(224, kind)
    canvas = torch.rand(1, 3, H, W, device='cuda')
    out = torch.empty(S, 3, side, side, device='cuda')
    g = torch.randn(S, 3, side, side, device='cuda')
    gc = torch.empty(1, 3, H, W, device='cuda')
    fwd = lambda: check(lib().aph_sample_fwd(canvas.data_ptr(), H, W, 0, 0, t.data_ptr(), S, 224, kind, out.data_ptr(), stream_ptr()), 'fwd')
    bwd = lambda: check(lib().aph_sample_bwd_scaled(g.data_ptr(), H, W, 0, 0, t.data_ptr(), S, 224, kind, 1., gc.data_ptr(), stream_ptr()), 'bwd')
    return _time(fwd, reps), _time(bwd, reps)


def sampler_large_frame(kind, reps, S=190):
    """Forward only, on the frame of tests/test_gpu_parity.py::test_sampler_large_frame_every_kind_vs_oracle: a 300x420 canvas wrap-padded by
    3000 / 2950 pixels (6300 x 6320), whose short side is too long for k_resize's per-warp crop rows; S crops of random side."""
    import numpy as np
    import torch
    from aphantasia_b200 import _rng
    from aphantasia_b200._lib import check, lib, stream_ptr
    H, W, pad_top, pad_left = 300, 420, 3000, 2950
    fh, fw = H + 2 * pad_top, W + 2 * pad_left
    torch.manual_seed(0); np.random.seed(0)
    tab = np.zeros((S, _rng.CROP_PARAM_FLOATS), np.float32)
    for row in tab:
        cs = np.random.randint(224, min(fh, fw) + 1)
        row[_rng.F_OFFY], row[_rng.F_OFFX], row[_rng.F_CSIZE] = np.random.randint(fh - cs + 1), np.random.randint(fw - cs + 1), cs
        row[_rng.F_ROT:_rng.F_ROT + 4] = (1., 0., 0., 1.)
        if kind == _rng.TF_FAST:
            row[_rng.F_FLAGS] = _rng.draw_fast(row, 224)
        elif kind >= _rng.TF_CUSTOM:
            row[_rng.F_FLAGS] = _rng.draw_kornia(row, 224, kind == _rng.TF_ELASTIC)
    t = torch.from_numpy(tab).cuda()
    side = _rng.out_side(224, kind)
    canvas = torch.rand(1, 3, H, W, device='cuda')
    out = torch.empty(S, 3, side, side, device='cuda')
    return _time(lambda: check(lib().aph_sample_fwd(canvas.data_ptr(), H, W, pad_top, pad_left, t.data_ptr(), S, 224, kind, out.data_ptr(),
                                                    stream_ptr()), 'fwd'), reps)


def step(kind, steps):
    import numpy as np
    import torch
    from aphantasia_b200 import transforms
    from aphantasia_b200.clip import CLIP, synthetic_visual_state_dict
    from aphantasia_b200.image import fft_image, to_valid_rgb
    from aphantasia_b200.utils import sim_func, slice_imgs
    tf = {2: transforms.transforms_fast, 3: transforms.transforms_custom, 4: transforms.transforms_elastic}[kind]
    model = CLIP('ViT-B/32', synthetic_visual_state_dict(patch=32, seed=0), True)
    torch.manual_seed(0); np.random.seed(0)
    params, image_f, _ = fft_image([1, 3, 720, 1280], 0.07, 1.5, None)
    rgb_f = to_valid_rgb(image_f, colors=1.8)
    txt = torch.randn(1, 512, device='cuda')

    def one():
        loss = -1. * sim_func(txt, model.encode_image(slice_imgs([rgb_f()], 190, 224, tf, 'uniform', 0.4)[0]), 'mix')
        loss.backward()
    ms = _time(one, steps)
    model.visual.close()
    return ms


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=200)
    ap.add_argument('--steps', type=int, default=30)
    a = ap.parse_args()
    out = {}
    for geo, (H, W, S) in (('c2', (720, 1280, 190)), ('c3', (1080, 1920, 47))):
        for kind in (2, 3, 4):
            f, b = sampler(kind, H, W, S, a.reps)
            out['%s_kind%d_fwd_ms' % (geo, kind)] = round(f, 4)
            out['%s_kind%d_bwd_ms' % (geo, kind)] = round(b, 4)
    for kind in (0, 1, 2, 3, 4):
        out['large_frame_kind%d_fwd_ms' % kind] = round(sampler_large_frame(kind, a.reps), 4)
    for kind in (2, 3, 4):
        out['c2_step_kind%d_ms' % kind] = round(step(kind, a.steps), 3)
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    out['gpu'] = q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
