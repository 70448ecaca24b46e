"""Generates reference_golden_transforms.npz from the REAL reference (/root/reference), build container only.

    python tests/golden/make_golden_transforms.py

Runs the reference's own slice_imgs with its transforms_custom / transforms_elastic (oracle/ref_import.py loads the modules in
place; nothing is copied). kornia is absent, so its four functions the pipelines call are stubs that record what they receive
(angle and centre, the image warp_affine gets, k / sigma / alpha / noise of elastic_transform2d, the translation) and then apply
tests/kornia_oracle.py's restatement. Everything else -- the crop, the resize, pad, RandomErasing, normalise and every random
draw -- is the reference's. Pinned here:
  * trf_<case>_*: the per-crop parameters in the sampler's table layout and both generator states after the call;
  * val_<case>_*: on a small frame, the input of every warp_affine call (pad + erase values) and slice_imgs' output.
"""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F
import torchvision.transforms.functional as TF

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from oracle import ref_import  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
ref = ref_import.load()
import kornia_oracle as KO  # noqa: E402

FLAG_ERASE, FLAG_ROT, FLAG_JITTER, FLAG_ELASTIC = 2, 4, 8, 16


def seed(s):
    torch.manual_seed(s); np.random.seed(s)


def install_stubs(rec):
    K = sys.modules['kornia.geometry.transform']
    sys.modules['kornia'].geometry = sys.modules['kornia.geometry']
    sys.modules['kornia.geometry'].transform = K

    def get_rotation_matrix2d(center, angle, scale):
        rec[-1].update(angle=float(angle[0]), center=center[0].tolist(), scale=scale[0].tolist())
        return torch.tensor(KO.kornia_rotation_matrix(float(angle[0]), float(center[0, 0])), dtype=torch.float32)[None]

    def warp_affine(src, M, dsize, **k):
        rec[-1]['warp_in'] = src.detach().clone()
        rec[-1]['dsize'] = tuple(dsize)
        # restated from the recorded angle and centre in float64 (the float32 M differs from it by rounding only)
        return KO.warp_affine(src, KO.kornia_rotation_matrix(rec[-1]['angle'], rec[-1]['center'][0]))

    def elastic_transform2d(image, noise, kernel_size, sigma, alpha, **k):
        rec[-1].update(elastic=(kernel_size[0], kernel_size[1], sigma[0], sigma[1], alpha[0], alpha[1]), noise_max=float(noise.abs().max()))
        return KO.elastic_zero_noise(image)

    def translate(image, translation, **k):
        rec[-1]['shift'] = translation[0].tolist()
        return KO.translate(image, int(translation[0, 0]), int(translation[0, 1]))

    K.get_rotation_matrix2d, K.warp_affine, K.elastic_transform2d, K.translate = get_rotation_matrix2d, warp_affine, elastic_transform2d, translate


def run_slice(canvas, count, size, kind, align, macro, s):
    """The reference slice_imgs with transforms_custom (3) / transforms_elastic (4); returns its output and the records."""
    rec = []
    o_interp, o_erase = F.interpolate, TF.erase

    def interp(x, *a, **k):
        rec.append(dict(cut=x.detach().clone(), erase=None, elastic=None))
        return o_interp(x, *a, **k)

    def erase(img, i, j, h, w, v, *a, **k):
        rec[-1]['erase'] = (i, j, h, w)
        return o_erase(img, i, j, h, w, v, *a, **k)

    install_stubs(rec)
    import torchvision.transforms.transforms as TT
    F.interpolate, TF.erase, TT.F.erase = interp, erase, erase
    try:
        seed(s)
        tf = ref.transforms.transforms_elastic if kind == 4 else ref.transforms.transforms_custom
        out = ref.utils.slice_imgs([canvas], count, size, tf, align, macro)[0]
        tstate = torch.get_rng_state().numpy().copy()
        _, key, pos = np.random.get_state()[:3]
    finally:
        F.interpolate, TF.erase, TT.F.erase = o_interp, o_erase, o_erase
    return out, rec, tstate, np.append(np.asarray(key, np.int64), pos)


def table_of(rec, index_canvas):
    """Records -> rows of the sampler's table layout (include/aphb200.h). Crop offsets come from the index canvas (channel 0 = y,
    channel 1 = x) the crop was cut from; F_ROT is left to the test (the restated inverse of the recorded angle)."""
    arr = np.zeros((len(rec), 24), np.float32)
    extra = np.zeros((len(rec), 10), np.float64)        # centre x, y, k_x, k_y, sigma_x, sigma_y, alpha_x, alpha_y, |noise|max, dsize
    for c, r in enumerate(rec):
        flags = FLAG_ROT | FLAG_JITTER
        if index_canvas:
            arr[c, 0:3] = (float(r['cut'][0, 0, 0, 0]), float(r['cut'][0, 1, 0, 0]), r['cut'].shape[-1])
        if r['erase'] is not None and tuple(r['erase'][2:]) != tuple(r['warp_in'].shape[-2:]):
            flags |= FLAG_ERASE
            arr[c, 12:16] = r['erase']
        if r['elastic'] is not None:
            flags |= FLAG_ELASTIC
            extra[c, 2:8] = r['elastic']
            extra[c, 8] = r['noise_max']
        arr[c, 3] = flags
        arr[c, 20] = r['angle']
        arr[c, 21:23] = r['shift']
        extra[c, 0:2] = r['center']
        extra[c, 9] = r['dsize'][0]
    return arr, extra


def main():
    g = {}
    # ---- 1. parameters and generator states after the call ---------------------------------------------------------------
    cases = [('c2c', (720, 1280), 190, 224, 3, 'uniform', 0.4, 123),
             ('c2e', (720, 1280), 190, 224, 4, 'uniform', 0.4, 321),
             ('central_e', (300, 420), 16, 224, 4, 'central', 0.4, 7),
             ('over_c', (240, 320), 12, 224, 3, 'overscan', 0.4, 11),
             ('over_e', (240, 320), 12, 224, 4, 'overscan', 0., 12),
             ('small_c', (64, 96), 8, 32, 3, 'uniform', 0.5, 5),
             ('small_e', (64, 96), 24, 32, 4, 'uniform', 0.5, 6),
             ('macro0_e', (256, 256), 9, 224, 4, 'uniform', 0., 3)]
    for name, (H, W), cnt, size, kind, align, macro, s in cases:
        yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing='ij')
        canvas = torch.stack([yy, xx, torch.zeros_like(yy)])[None]
        if 'over' in align:           # the index canvas must survive the wrap padding: record offsets in the padded frame
            fh, fw = (int(1.5 * H), int(1.5 * W))
            yy, xx = torch.meshgrid(torch.arange(fh, dtype=torch.float32), torch.arange(fw, dtype=torch.float32), indexing='ij')
            pad_frame = torch.stack([yy, xx, torch.zeros_like(yy)])[None]
            o_pad = ref.utils.pad_up_to
            ref.utils.pad_up_to = lambda *a, **k: pad_frame
            try:
                _, rec, ts, ns = run_slice(canvas, cnt, size, kind, align, macro, s)
            finally:
                ref.utils.pad_up_to = o_pad
        else:
            _, rec, ts, ns = run_slice(canvas, cnt, size, kind, align, macro, s)
        arr, extra = table_of(rec, True)
        g['trf_%s_table' % name] = arr
        g['trf_%s_extra' % name] = extra
        g['trf_%s_torch_after' % name] = ts
        g['trf_%s_np_after' % name] = ns
        g['trf_%s_cfg' % name] = np.array([H, W, cnt, size, kind, macro, s], np.float64)
        g['trf_%s_align' % name] = np.array(align)
        print(name, 'erase hits', int(((arr[:, 3].astype(int) & FLAG_ERASE) > 0).sum()), 'of', len(arr))

    # ---- 2. values on a small frame: the warp_affine inputs (pad + erase) and the output (normalise) ----------------------
    for name, hw, cnt, size, kind, align, macro, s in [('small_c', (64, 96), 6, 32, 3, 'uniform', 0.5, 5),
                                                         ('small_e', (64, 96), 24, 32, 4, 'uniform', 0.5, 6),
                                                         ('over_e', (80, 120), 6, 32, 4, 'overscan', 0.4, 13)]:
        seed(100 + s)
        canvas = torch.rand(1, 3, *hw).half().float()            # fp16-exact values: stored compactly
        out, rec, _, _ = run_slice(canvas, cnt, size, kind, align, macro, s)
        arr, _ = table_of(rec, False)
        g['val_%s_canvas' % name] = canvas.numpy().astype(np.float16)
        g['val_%s_cfg' % name] = np.array([hw[0], hw[1], cnt, size, kind, macro, s], np.float64)
        g['val_%s_align' % name] = np.array(align)
        g['val_%s_params' % name] = arr                            # erase / angle / shift / flags (offsets: from the replay)
        g['val_%s_warp_in' % name] = torch.cat([r['warp_in'] for r in rec]).numpy()
        g['val_%s_out' % name] = out.detach().numpy()

    path = os.path.join(OUT, 'reference_golden_transforms.npz')
    np.savez_compressed(path, **g)
    print('wrote', path, os.path.getsize(path) // 1024, 'KiB,', len(g), 'arrays')


if __name__ == '__main__':
    main()
