"""Test infrastructure: float64 restatement of cppn.py's CPPN (cppn.py:71-116), its backward, and kornia's Sobel
`spatial_gradient` as `derivat(img, mode='sobel')` uses it (aphantasia/utils.py:262-264).

`tf32=True` rounds the operands of the hidden layers' three products (forward z = x W^T, data gradient dx = dz W, weight gradient
dW = dz^T x) as the kernel does: each operand is first an fp32 value (the kernel holds it in fp32), then rounded by
cvt.rna.tf32.f32 (nearest, ties away from zero, 10 mantissa bits). Everything else is float64. Layer 0 and the output layer are
not rounded: the kernel runs them in fp32 (csrc/cppn.cu).

The network is pinned by tests/golden/reference_golden_cppn.npz (the original classes, fp32 on the CPU). kornia is absent here,
so the Sobel part restates its documented semantics and is parity-unpinned: the Sobel kernel [[-1,0,1],[-2,0,2],[-1,0,1]] (and
its transpose) normalised by the sum of its absolute values (8), replicate padding, cross-correlation, output [N,C,2,H,W].
"""
import os
import sys
import types

import numpy as np

OFF_DIV = {'unbias': (0.45, 0.396), 'comp': (0.0, 0.6)}


def tf32(a):
    """fp32 value of `a`, rounded to TF32 as cvt.rna.tf32.f32 does, returned as float64."""
    u = np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)
    u = (u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)
    return u.view(np.float32).astype(np.float64)


def _act(z, act):
    if act == 'relu':
        return (np.maximum(z, 0.) - 0.4) / 0.58, None
    off, div = OFF_DIV[act]
    t = np.arctan(z)
    return np.concatenate([t / 0.67, (t * t - off) / div], axis=1), t


def _act_grad(dx, z, t, act):
    if act == 'relu':
        return dx / 0.58 * (z > 0)
    nf = z.shape[1]
    return (dx[:, :nf] / 0.67 + dx[:, nf:] * 2. * t / OFF_DIV[act][1]) / (1. + z * z)


def _pixels(coords):
    c = np.asarray(coords, dtype=np.float64)
    N, _, H, W = c.shape
    return c.transpose(0, 2, 3, 1).reshape(-1, 2), (N, H, W)


def forward(coords, params, act, tf32_ops=True):
    """coords [N,2,H,W], params [W0, b0, ..., W_L, b_L] (W as [out,in] or [out,in,1,1]) -> (out [N,3,H,W], cache)."""
    R = tf32 if tf32_ops else (lambda a: np.asarray(a, dtype=np.float64))
    X, (N, H, W) = _pixels(coords)
    Ws = [np.asarray(params[2 * i], dtype=np.float64).reshape(np.shape(params[2 * i])[0], -1) for i in range(len(params) // 2)]
    bs = [np.asarray(params[2 * i + 1], dtype=np.float64) for i in range(len(params) // 2)]
    L = len(Ws) - 1
    z = X @ Ws[0].T + bs[0]
    zs, xs, ts = [z], [X], []
    for l in range(1, L):
        x, t = _act(z, act)
        ts.append(t); xs.append(x)
        z = R(x) @ R(Ws[l]).T + bs[l]
        zs.append(z)
    x, t = _act(z, act)
    ts.append(t); xs.append(x)
    y = 1. / (1. + np.exp(-(x @ Ws[L].T + bs[L])))
    out = y.reshape(N, H, W, 3).transpose(0, 3, 1, 2)
    return out, dict(Ws=Ws, zs=zs, xs=xs, ts=ts, y=y, act=act, R=R, shape=(N, H, W))


def backward(cache, grad_out):
    """d sum(out * grad_out) / d params, in the order of params."""
    Ws, zs, xs, ts, y, act, R = (cache[k] for k in ('Ws', 'zs', 'xs', 'ts', 'y', 'act', 'R'))
    L = len(Ws) - 1
    g = np.asarray(grad_out, dtype=np.float64).transpose(0, 2, 3, 1).reshape(-1, 3)
    dzo = g * y * (1. - y)
    grads = [None] * (2 * (L + 1))
    grads[2 * L], grads[2 * L + 1] = dzo.T @ xs[L], dzo.sum(0)
    dx = dzo @ Ws[L]
    for l in range(L - 1, -1, -1):
        dz = _act_grad(dx, zs[l], ts[l], act)
        if l > 0:
            grads[2 * l], grads[2 * l + 1] = R(dz).T @ R(xs[l]), dz.sum(0)
            dx = R(dz) @ R(Ws[l])
        else:
            grads[0], grads[1] = dz.T @ xs[0], dz.sum(0)
    return grads


SOBEL_X = np.array([[-1., 0., 1.], [-2., 0., 2.], [-1., 0., 1.]]) / 8.


def sobel_gradient(img):
    """unpinned: kornia.filters.spatial_gradient(img, 'sobel', order=1, normalized=True): [N,C,H,W] -> [N,C,2,H,W] (x, y)."""
    x = np.asarray(img, dtype=np.float64)
    H, W = x.shape[2:]
    p = np.pad(x, ((0, 0), (0, 0), (1, 1), (1, 1)), mode='edge')
    out = np.zeros(x.shape[:2] + (2, H, W))
    for d, k in enumerate((SOBEL_X, SOBEL_X.T)):
        for i in range(3):
            for j in range(3):
                out[:, :, d] += k[i, j] * p[:, :, i:i + H, j:j + W]
    return out


def sobel_derivat(img, upstream=1.):
    """(mean |spatial_gradient(img)|, its gradient with respect to img times upstream; sign(0) = 0)."""
    x = np.asarray(img, dtype=np.float64)
    H, W = x.shape[2:]
    g = sobel_gradient(x)
    s = np.sign(g) * upstream / g.size
    gp = np.zeros(x.shape[:2] + (H + 2, W + 2))
    for d, k in enumerate((SOBEL_X, SOBEL_X.T)):
        for i in range(3):
            for j in range(3):
                gp[:, :, i:i + H, j:j + W] += k[i, j] * s[:, :, d]
    gp[:, :, 1] += gp[:, :, 0]; gp[:, :, -2] += gp[:, :, -1]          # replicate padding's adjoint: fold the pads back
    gp[:, :, :, 1] += gp[:, :, :, 0]; gp[:, :, :, -2] += gp[:, :, :, -1]
    return float(np.abs(g).mean()), gp[:, :, 1:-1, 1:-1]


def load_original_script(path):
    """Executes the original cppn.py (module body only: __name__ is not '__main__') with `clip`, `eps` and `googletrans`
    stubbed, the original `aphantasia` package (oracle/ref_import) importable and shader_expo.py from the script's directory.
    Returns the module. The loader's stand-ins for packages absent here (imageio, kornia, ...) and its `.cuda()` shim are taken
    back afterwards, so that they do not leak into the tests that run after the caller."""
    import torch
    from oracle import ref_import
    before = set(sys.modules)
    cuda_t, cuda_m = torch.Tensor.cuda, torch.nn.Module.cuda
    try:
        ns = ref_import.load()
    finally:
        for k in [k for k in sys.modules if k not in before and getattr(sys.modules[k], '__aph_stub__', False)]:
            del sys.modules[k]
        torch.Tensor.cuda, torch.nn.Module.cuda = cuda_t, cuda_m
    saved = {k: sys.modules.get(k) for k in ('aphantasia', 'aphantasia.utils', 'aphantasia.transforms', 'clip', 'eps',
                                             'eps.progress_bar', 'eps.data_load', 'googletrans', 'shader_expo')}
    pkg = types.ModuleType('aphantasia')
    pkg.utils, pkg.transforms = ns.utils, ns.transforms
    stubs = {'aphantasia': pkg, 'aphantasia.utils': ns.utils, 'aphantasia.transforms': ns.transforms,
             'clip': types.ModuleType('clip'), 'eps': types.ModuleType('eps'), 'googletrans': types.ModuleType('googletrans')}
    pb, dl = types.ModuleType('eps.progress_bar'), types.ModuleType('eps.data_load')
    pb.ProgressBar = None
    for n in ('basename', 'img_list', 'img_read', 'file_list', 'save_cfg'):
        setattr(dl, n, None)
    stubs['eps.progress_bar'], stubs['eps.data_load'] = pb, dl
    stubs['googletrans'].Translator = None
    sys.modules.update(stubs)
    sys.path.insert(0, os.path.dirname(os.path.abspath(path)))
    try:
        mod = types.ModuleType('ref_cppn_script')
        mod.__file__ = path
        with open(path, 'rb') as f:
            exec(compile(f.read(), path, 'exec'), mod.__dict__)
        return mod
    finally:
        sys.path.pop(0)
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
