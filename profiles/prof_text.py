"""Latency of one CLIP text encode (aph_text_fwd, ViT-B text geometry: width 512, 12 layers, context 77, vocab 49408) with
synthetic weights, by CUDA events over repeated calls after a warm-up. Prints one JSON line with the card's name and power
limit. Usage: python profiles/prof_text.py [--reps 50]"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    import torch
    from aphantasia_b200 import _lib, clip
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=50)
    a = ap.parse_args()
    tower = clip.TextTransformer(clip.synthetic_text_state_dict(seed=0))
    out = {}
    for n in (1, 4):
        toks = torch.zeros(n, 77, dtype=torch.long)
        toks[:, 0], toks[:, 1:6], toks[:, 6] = 49406, 320, 49407
        toks = toks.cuda()
        for _ in range(5):
            tower(toks)
        torch.cuda.synchronize()
        l0 = _lib.lib().aph_launch_count()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.reps):
            tower(toks)
        e1.record()
        torch.cuda.synchronize()
        out['n%d_ms' % n] = e0.elapsed_time(e1) / a.reps
        out['n%d_launches' % n] = (_lib.lib().aph_launch_count() - l0) // a.reps
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    out['gpu'] = q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
