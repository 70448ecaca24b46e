"""Times illustrip.py's frame at 1280x720 with its default flags (ViT-B/32, 95 crops after the script's 0.95 factor, overscan,
transforms_fast, macro 0.3, adam_custom, opt_step 1), for the RGB generator (default) and --gen FFT.

    python profiles/prof_illustrip.py > illustrip_times.json

Reports, with the card's name and power limit:
  motion   : frame_transform (affine + center_crop) with the script's argument types, stock torchvision against the routed kernel;
  fft_init : fft_image construction per frame with the shared plan, and with a plan created per generator and the previous
             frame's plan destroyed (what each frame cost before plans were shared);
  split    : one frame, phase by phase with a device synchronise after each phase (motion, synth, sampler, encoder, loss,
             backward, Adam, preview), and the same frame without intermediate synchronises;
  launches : per frame, kernels of libaphb200.so (aph_launch_count) and all CUDA kernels (torch.profiler)."""
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'dropin'))
import torchvision.transforms.functional as TF  # noqa: E402
from torchvision.transforms import InterpolationMode as IM  # noqa: E402

from aphantasia_b200 import _lib, image, motion, transforms  # noqa: E402
from aphantasia_b200.clip import load  # noqa: E402
from aphantasia_b200.image import fft_image, pixel_image, to_valid_rgb  # noqa: E402
from aphantasia_b200.utils import latent_anima, sim_func, slice_imgs  # noqa: E402

H, W = 720, 1280


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as ex:
        return 'unknown (%r)' % (ex,)


def events_ms(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def wall_ms(fn, reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / reps


def motion_args(n):
    """The script's per-frame arguments (illustrip.py:301-314, 381-384) for RGB defaults, in its types."""
    np.random.seed(0)
    sc = latent_anima([1], n, 100, uniform=True, cubic=True, start_lat=[-0.3], seed=1)
    sc = 1 + (sc + 0.3) * 0.012
    sh = (0.5 - latent_anima([2], n, 100, uniform=True, cubic=True, start_lat=[.5, .5], seed=2)) * 10. * abs(sc - 1) / 0.012
    an = (0.5 - latent_anima([1], n, 100, uniform=True, cubic=True, start_lat=[.5], seed=3)) * 0.8 * abs(sc - 1) / 0.012
    se = (0.5 - latent_anima([1], n, 100, uniform=True, cubic=True, start_lat=[.5], seed=4)) * 0.4 * abs(sc - 1) / 0.012
    return [(an[k][0], tuple(sh[k]), sc[k], se[k][0]) for k in range(n)]


def frame_transform(img, args):
    angle, shift, scale, shear = args
    img = TF.affine(img, angle, shift, scale, shear, fill=0, interpolation=IM.BILINEAR)
    return TF.center_crop(img, [H, W])


def time_motion():
    args = motion_args(200)
    out = {}
    img = torch.randn(1, 3, H, W, device='cuda')
    for name, fn in (('stock_torchvision', motion.stock_affine), ('routed_kernel', motion.affine)):
        TF.affine = fn
        k = [0]

        def step():
            frame_transform(img, args[k[0] % len(args)]); k[0] += 1
        for _ in range(10):
            step()
        out[name + '_ms'] = round(wall_ms(step, 200), 4)            # includes the host work and the stock path's blocking copy
        out[name + '_device_ms'] = round(events_ms(step, 200), 4)
    TF.affine = motion.stock_affine
    return out


def time_fft_init(frames=50):
    p = 0.01 * torch.randn(1, 3, H, W // 2 + 1, 2, device='cuda')

    def shared():
        params, image_f, _ = fft_image([1, 3, H, W], sd=1, resume=p.clone())
        return image_f

    prev = {'plan': None}

    def per_generator():
        # the former behaviour: a plan per generator, the previous frame's plan freed when its generator is dropped
        image._fft_plans.pop((H, W), None)
        image._fft_scales.clear()
        gen = shared()
        if prev['plan'] is not None:
            _lib.lib().aph_fft_plan_destroy(prev['plan'])
        prev['plan'] = gen.plan
        return gen
    res = {}
    for name, fn in (('per_generator_plan', per_generator), ('shared_plan', shared)):
        for _ in range(3):
            fn()
        res[name + '_ms'] = round(wall_ms(fn, frames), 4)
    image._fft_plans[(H, W)] = prev['plan']          # the last plan stays in use as the shared one
    return res


def make_frame(gen, model, txt, tmpdir):
    """One frame of illustrip.py's loop body (illustrip.py:379-484) for --gen RGB / FFT with default flags, as phases."""
    samples, colors, contrast, lr = int(100 * 0.95), 2.3, 1.2, 0.1
    st = {'params_tmp': None, 'k': 0}
    if gen == 'RGB':
        p, _, _ = pixel_image([1, 3, H, W], None)
        st['params_tmp'] = p[0].detach()
    else:
        st['params_tmp'], _ = image.resume_fft(None, [1, 3, H, W], decay=1.5, sd=1)
    margs = motion_args(400)
    txt_enc = [[txt, 0.7], [txt, 0.3]]

    def motion_phase():
        a = margs[st['k'] % len(margs)]; st['k'] += 1
        if gen == 'RGB':
            st['params_tmp'] = frame_transform(st['params_tmp'], a)
            st['params'], f, _ = pixel_image([1, 3, H, W], resume=st['params_tmp'])
        else:
            c = torch.view_as_complex(st['params_tmp'])
            img = frame_transform(torch.fft.irfftn(c, s=[H, W], norm='ortho'), a)
            st['params_tmp'] = torch.view_as_real(torch.fft.rfftn(img, s=[H, W], dim=[2, 3], norm='ortho'))
            st['params'], f, _ = fft_image([1, 3, H, W], sd=1, resume=st['params_tmp'])
        st['opt'] = torch.optim.Adam(st['params'], lr, betas=(.0, .999))
        st['image_f'] = to_valid_rgb(f, colors=colors)

    def synth_phase():
        noise = 2. * (torch.rand(1, 1, H, W // 2 + 1, 1) - 0.5).cuda()
        st['img_out'] = st['image_f'](noise, fixcontrast=False)

    def sampler_phase():
        st['sliced'] = slice_imgs([st['img_out']], samples, 224, transforms.transforms_fast, 'overscan', 0.3)[0]

    def encoder_phase():
        st['enc'] = model.encode_image(st['sliced'])

    def loss_phase():
        loss = 0
        if gen == 'RGB':
            loss += abs(st['img_out'].mean((2, 3)) - 0.45).mean()
            loss += abs(st['img_out'].std((2, 3)) - 0.17).mean()
        for enc, wt in txt_enc:
            loss -= wt * sim_func(enc, st['enc'], 'mix')
        st['loss'] = loss
        del st['img_out'], st['sliced'], st['enc']
        torch.cuda.empty_cache()

    def backward_phase():
        st['opt'].zero_grad()
        st['loss'].backward()

    def adam_phase():
        st['opt'].step()
        st['params_tmp'] = st['params'][0].detach().clone()

    def preview_phase():
        with torch.no_grad():
            img_t = st['image_f'](contrast=contrast, fixcontrast=False)[0].permute(1, 2, 0)
            img_np = torch.clip(img_t * 255, 0, 255).cpu().numpy().astype(np.uint8)
        from imageio import imsave
        imsave(os.path.join(tmpdir, '%06d.jpg' % st['k']), img_np, quality=95)

    return [('motion', motion_phase), ('synth', synth_phase), ('sampler', sampler_phase), ('encoder', encoder_phase),
            ('loss', loss_phase), ('backward', backward_phase), ('adam', adam_phase), ('preview', preview_phase)]


def time_frames(model, txt, frames=30):
    out = {}
    lib = _lib.lib()
    for gen in ('RGB', 'FFT'):
        with tempfile.TemporaryDirectory() as tmp:
            torch.manual_seed(0); np.random.seed(0)
            phases = make_frame(gen, model, txt, tmp)

            def frame():
                for _, fn in phases:
                    fn()
            for _ in range(5):
                frame()
            split = {name: 0. for name, _ in phases}
            for _ in range(frames):
                for name, fn in phases:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    fn()
                    torch.cuda.synchronize()
                    split[name] += (time.perf_counter() - t0) * 1e3
            free_ms = wall_ms(frame, frames)
            torch.cuda.synchronize()
            n0 = lib.aph_launch_count()
            frame()
            torch.cuda.synchronize()
            aph_launches = lib.aph_launch_count() - n0
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                frame()
                torch.cuda.synchronize()
            kernels = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and 'memcpy' not in e.name.lower()
                          and 'memset' not in e.name.lower())
            out[gen] = {'split_ms_synchronised': {k: round(v / frames, 3) for k, v in split.items()},
                        'sum_of_split_ms': round(sum(split.values()) / frames, 3), 'frame_ms_unsynchronised': round(free_ms, 3),
                        'frames_per_s_unsynchronised': round(1e3 / free_ms, 2), 'launches_libaphb200': int(aph_launches),
                        'cuda_kernels_all': int(kernels)}
    return out


def main():
    assert torch.cuda.is_available(), 'prof_illustrip.py measures on the GPU'
    model, _ = load('ViT-B/32')
    txt = model.encode_text(torch.zeros(1, 77, dtype=torch.long).cuda()).detach()
    res = {'card': card(), 'canvas': '%dx%d' % (W, H), 'motion': time_motion(), 'fft_init': time_fft_init()}
    motion.install()                      # as the launcher does: the frames below run the routed affine
    res['frames'] = time_frames(model, txt)
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
