"""Generates reference_golden_cppn.npz from the REAL cppn.py of the original project (/root/reference), build container only.

    python tests/golden/make_golden_cppn.py

The script's own ConvLayer / CPPN run on the CPU in fp32 (tests/cppn_oracle.load_original_script stubs `clip`, `eps` and
`googletrans`; `.cuda()` is the identity while this runs). Nothing of the original is copied, only these values, per case
`c<i>` (activation, nf, layers, H, W):
  * meta: [act index (0 unbias, 1 comp, 2 relu), nf, layers, H, W, seed];
  * p<k>: the state dict after torch.manual_seed(seed) and CPPN(2, nf, layers, 3, act_fn), in state-dict order;
  * coords: the script's get_mgrid(H, W) as fp32, out: CPPN.forward(coords);
  * gout: a fixed random cotangent, g<k>: the weight gradients of sum(out * gout).
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from oracle import ref_import  # noqa: E402
import cppn_oracle  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
ACTS = ('unbias', 'comp', 'relu')
CASES = [(act, nf, layers, H, W) for act in ACTS for (nf, layers, H, W) in ((8, 1, 1, 1), (8, 2, 5, 7), (24, 3, 9, 13), (16, 10, 6, 4))]


def main():
    cuda_t, cuda_m = torch.Tensor.cuda, torch.nn.Module.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    torch.nn.Module.cuda = lambda self, *a, **k: self
    try:
        mod = cppn_oracle.load_original_script(os.path.join(ref_import.REF_ROOT, 'cppn.py'))
        data = {}
        for i, (act, nf, layers, H, W) in enumerate(CASES):
            seed = 100 + i
            torch.manual_seed(seed)
            net = mod.CPPN(2, nf, layers, 3, act_fn=act)
            sd = net.state_dict()
            coords = torch.from_numpy(mod.get_mgrid(H, W).astype(np.float32))
            out = net(coords)
            g = torch.Generator().manual_seed(1000 + i)
            gout = torch.randn(out.shape, generator=g)
            (out * gout).sum().backward()
            data['c%d_meta' % i] = np.array([ACTS.index(act), nf, layers, H, W, seed], dtype=np.int64)
            for k, (name, v) in enumerate(sd.items()):
                data['c%d_p%d' % (i, k)] = v.numpy().copy()
            for k, p in enumerate(net.parameters()):
                data['c%d_g%d' % (i, k)] = p.grad.numpy().copy()
            data['c%d_coords' % i] = coords.numpy()
            data['c%d_out' % i] = out.detach().numpy()
            data['c%d_gout' % i] = gout.numpy()
        np.savez_compressed(os.path.join(OUT, 'reference_golden_cppn.npz'), **data)
        print('wrote %d cases' % len(CASES))
    finally:
        torch.Tensor.cuda, torch.nn.Module.cuda = cuda_t, cuda_m


if __name__ == '__main__':
    main()
