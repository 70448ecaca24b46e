"""ViT-L/14 on the GPU, synthetic weights, CUDA events after warm-up. Prints one JSON line with the card's name and power limit:
  - the encoder's forward and data-gradient (aph_vit_fwd / aph_vit_bwd, graph-cached as in the optimisation loop) at S = 8
    (the notebook's sample budget for ViT-L/14) and S = 200;
  - attention kernel times at S = 200, 16 heads: T = 197 and 256 with both the resident kernels (aph_attn_test) and the
    streaming kernels (aph_attn_long_test), and T = 257 (streaming, what ViT-L/14 runs);
  - the encoder's GEMM work (sum of 2 M N K over its GEMM shapes, the patch GEMMs at their padded K / N of 640) over the
    encoder's event time: a lower bound on the GEMMs' own rate, since that time includes attention and LayerNorm;
  - a whole optimisation step at 1280x720, --samples 200 (S = 190 crops, as bench.py counts them), transforms_fast, mix loss,
    Adam, ViT-L/14, timed over K steps with no host read inside the window.
Usage: python profiles/prof_vit_l14.py [--reps 20] [--steps 20]"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

VITL14 = dict(patch=14, width=1024, layers=24, heads=16, out_dim=768, res=224)


def gemm_flops(S, patch=14, D=1024, layers=24, out=768, res=224):
    """(forward, backward) sum of 2 M N K over the encoder's GEMMs (csrc/vit.cu); the last block runs its MLP and out_proj on
    the S class rows only"""
    g = res // patch
    T, Mp, Kp = g * g + 1, S * g * g, (3 * patch * patch + 127) // 128 * 128
    M = S * T
    f = 2 * Mp * D * Kp + 2 * S * out * D
    b = 2 * S * D * out + 2 * Mp * Kp * D
    for l in range(layers):
        Mr = S if l == layers - 1 else M
        f += 2 * M * 3 * D * D + 2 * Mr * D * D + 2 * Mr * 4 * D * D + 2 * Mr * D * 4 * D
        b += 2 * Mr * 4 * D * D + 2 * Mr * D * 4 * D + 2 * Mr * D * D + 2 * M * D * 3 * D
    return f, b


def events_ms(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    import numpy as np
    import torch
    from aphantasia_b200 import _lib, transforms
    from aphantasia_b200.clip import CLIP, VisionTransformer, synthetic_visual_state_dict
    from aphantasia_b200.image import fft_image, to_valid_rgb
    from aphantasia_b200.utils import sim_func, slice_imgs
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--steps', type=int, default=20)
    a = ap.parse_args()
    lib, st = _lib.lib(), _lib.stream_ptr
    out = {}
    sd = synthetic_visual_state_dict(seed=0, **VITL14)

    # ---- encoder forward / backward
    vis = VisionTransformer(sd, max_batch=200)
    for S in (8, 200):
        x = torch.rand(S, 3, 224, 224, device='cuda')
        emb = torch.empty(S, 768, device='cuda'); gx = torch.empty_like(x)
        cot = torch.randn(S, 768, device='cuda') * 0.1
        fwd = lambda: _lib.check(lib.aph_vit_fwd(vis.handle, x.data_ptr(), S, emb.data_ptr(), 1, st()), 'fwd')
        bwd = lambda: _lib.check(lib.aph_vit_bwd(vis.handle, cot.data_ptr(), S, gx.data_ptr(), st()), 'bwd')
        for _ in range(3):                       # eager, capture, replay
            fwd(); bwd()
        tf = events_ms(fwd, a.reps)
        fwd()
        tb = events_ms(bwd, a.reps)
        ff, fb = gemm_flops(S)
        out['enc_S%d_fwd_ms' % S], out['enc_S%d_bwd_ms' % S] = round(tf, 3), round(tb, 3)
        out['enc_S%d_gemm_tflops_fwd' % S] = round(ff / tf / 1e9, 1)
        out['enc_S%d_gemm_tflops_bwd' % S] = round(fb / tb / 1e9, 1)
        del x, emb, gx, cot
    vis.close()
    del vis
    torch.cuda.empty_cache()

    # ---- attention kernels
    S, H = 200, 16
    D = 64 * H
    for T in (197, 256, 257):
        qkv = (torch.randn(S * T, 3 * D, device='cuda') * 0.7).bfloat16()
        dout = (torch.randn(S * T, D, device='cuda') * 0.5).bfloat16()
        o = torch.empty(S * T, D, device='cuda', dtype=torch.bfloat16)
        dq = torch.empty(S * T, 3 * D, device='cuda', dtype=torch.bfloat16)
        fams = [('stream', lambda f, d, y: lib.aph_attn_long_test(f, qkv.data_ptr(), d, y, S, T, D, H, st()))]
        if T <= 256:
            fams.append(('resident', lambda f, d, y: lib.aph_attn_test(f, 0, qkv.data_ptr(), d, y, S, T, D, H, st())))
        for name, call in fams:
            tf = events_ms(lambda: _lib.check(call(1, None, o.data_ptr()), name), a.reps)
            tb = events_ms(lambda: _lib.check(call(0, dout.data_ptr(), dq.data_ptr()), name), a.reps)
            out['attn_T%d_%s_fwd_ms' % (T, name)], out['attn_T%d_%s_bwd_ms' % (T, name)] = round(tf, 3), round(tb, 3)
        del qkv, dout, o, dq
    torch.cuda.empty_cache()

    # ---- a whole step at 1280x720, S = 190
    torch.manual_seed(0); np.random.seed(0)
    params, image_f, _ = fft_image([1, 3, 720, 1280], 0.07, 1.5, None)
    rgb_f = to_valid_rgb(image_f, colors=1.8)
    model = CLIP('ViT-L/14', sd, True)
    g = torch.Generator().manual_seed(1234)
    txt = torch.randn(1, 768, generator=g); txt = (10. * txt / txt.norm()).cuda()
    opt = torch.optim.Adam(params, 0.05, betas=(.0, .999))
    losses = []

    def step():
        crops = slice_imgs([rgb_f(None)], 190, 224, transforms.transforms_fast, 'uniform', 0.4)[0]
        loss = -1. * sim_func(txt, model.encode_image(crops), 'mix')
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.detach())
    for _ in range(5):
        step()
    t = events_ms(step, a.steps)
    out['step_1280x720_S190_ms'] = round(t, 2)
    out['step_1280x720_S190_steps_per_s'] = round(1e3 / t, 3)
    out['step_loss_finite'] = bool(torch.isfinite(torch.stack(losses)).all())
    fs, bs = gemm_flops(190)
    out['step_encoder_gemm_tflop'] = round((fs + bs) / 1e12, 2)
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    out['gpu'] = q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
