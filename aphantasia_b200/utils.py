"""Sampler, loss and helper names -- drop-in for /root/reference/aphantasia/utils.py.

slice_imgs (utils.py:218-254) and sim_func (utils.py:276-295) are the hot-path entry points: the host
replays the reference's RNG order into a parameter table (_rng.py) and two fused CUDA launches each way do the rest
(csrc/sample.cu; csrc/loss.cu for the loss). The remaining names are the thin IO helpers clip_fft.py imports.
"""
import collections.abc
import math
import os

import numpy as np
import torch
import torch.nn.functional as F

import ctypes as C

from . import _dist, _patchlink, _rng, _trace
from . import _pool as _tpool
from ._lib import check, lib, require_cuda, stream_ptr


# ---------------------------------------------------------------------------------------------- sampler
class _SliceImgs(torch.autograd.Function):
    @staticmethod
    def forward(ctx, canvas, table_dev, meta, vis=None):
        H, W, pad_top, pad_left, S, size, kind, scale = meta
        x = canvas.detach().contiguous().float()
        side = _rng.out_side(size, kind)
        out = _tpool.empty((S, 3, side, side))
        if vis is not None and S > 0:
            # the encoder that will consume this batch takes its patch operand straight from the sampler's last stage (_patchlink)
            vis._ensure(S)
            ptr, patch, grid = C.c_void_p(), C.c_int(), C.c_int()
            check(lib().aph_vit_patch_operand(vis.handle, S, C.byref(ptr), C.byref(patch), C.byref(grid)), 'aph_vit_patch_operand')
            check(lib().aph_sample_fwd_patches(x.data_ptr(), H, W, pad_top, pad_left, table_dev.data_ptr(), S, size, kind, out.data_ptr(),
                                               ptr, patch.value, C.byref(C.c_int()), stream_ptr()), 'aph_sample_fwd_patches')
            vis._patch_gen += 1                     # whatever the buffer held before is gone
        else:
            check(lib().aph_sample_fwd(x.data_ptr(), H, W, pad_top, pad_left, table_dev.data_ptr(), S, size, kind, out.data_ptr(),
                                       stream_ptr()), 'aph_sample_fwd')
        ctx.meta = meta
        ctx.save_for_backward(table_dev)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        table_dev, = ctx.saved_tensors
        H, W, pad_top, pad_left, S, size, kind, scale = ctx.meta
        g = grad_out.contiguous().float()
        gc = _dist.symm_empty((1, 3, H, W)) if (_dist.world() > 1 and (3 * H * W) % 4 == 0) else None      # symmetric memory: own all-reduce kernel
        if gc is None:
            gc = _tpool.empty((1, 3, H, W))
        # each rank's loss is a mean over its own shard: its canvas gradient enters the sum over ranks with weight S_local / S_total
        # (`scale`, folded into the scatter kernel)
        check(lib().aph_sample_bwd_scaled(g.data_ptr(), H, W, pad_top, pad_left, table_dev.data_ptr(), S, size, kind, float(scale), gc.data_ptr(),
                                          stream_ptr()), 'aph_sample_bwd_scaled')
        if _dist.world() > 1:
            _dist.all_reduce_sum_(gc)
        return gc, None, None, None


def _transform_kind(transform):
    if transform is None:
        return _rng.TF_NONE
    kind = getattr(transform, 'kind', None)
    if kind is None:
        raise NotImplementedError('aphantasia_b200.slice_imgs: only transform=None, transforms.normalize(), transforms_fast, '
                                  'transforms_custom and transforms_elastic run in the fused sampler (got %r)' % (transform,))
    return kind


_pinned = {}          # table shape -> ring of pinned staging buffers with the event of the copy that last read each
_PIN_RING = 4


def _table_to_device(tab, device):
    """H2D of the per-step crop table through reused pinned staging buffers (async on the current stream). A ring, because the
    host may run a step ahead of the GPU (the script does not synchronise every step): a single buffer could be overwritten
    with step k+1's table before the copy of step k has executed. A slot is reused only after its copy event has completed."""
    key = tuple(tab.shape)
    ring = _pinned.get(key)
    if ring is None:
        ring = _pinned[key] = {'bufs': [torch.empty(tab.shape, dtype=torch.float32).pin_memory() for _ in range(_PIN_RING)],
                               'evs': [None] * _PIN_RING, 'next': 0}
    i = ring['next']
    ring['next'] = (i + 1) % _PIN_RING
    if ring['evs'][i] is not None:
        ring['evs'][i].synchronize()          # normally completed long ago
    else:
        ring['evs'][i] = torch.cuda.Event()
    buf = ring['bufs'][i]
    buf.numpy()[...] = tab
    out = buf.to(device, non_blocking=True)
    ring['evs'][i].record()
    return out


def slice_imgs(imgs, count, size=224, transform=None, align='uniform', macro=0.):
    """Drop-in for utils.py:218-254. Returns a list with one [count_local,3,side,side] tensor per input image
    (count_local == count on one GPU; the contiguous shard of this rank under torchrun). side = size, or size + 8 for
    transforms_custom / transforms_elastic, whose pad(4) the reference applies after the resize."""
    _dist.init()
    kind = _transform_kind(transform)
    for img in imgs:
        require_cuda(img, 'slice_imgs input')
    hw = tuple(imgs[0].shape[2:])
    assert all(tuple(i.shape[2:]) == hw for i in imgs), 'slice_imgs: all images must share one size'
    tables, (pad_top, pad_left, fh, fw) = _rng.draw_crop_table(count, hw, size, kind, align, macro, n_imgs=len(imgs))
    lo, hi = _rng.shard_range(count, _dist.rank(), _dist.world())
    sliced = []
    for img, tab in zip(imgs, tables):
        assert img.shape[0] == 1 and img.shape[1] == 3, 'slice_imgs expects [1,3,H,W] images'
        local = np.ascontiguousarray(tab[lo:hi])
        tdev = _table_to_device(local, img.device)
        meta = (hw[0], hw[1], pad_top, pad_left, hi - lo, size, kind, float(hi - lo) / float(count))
        side = _rng.out_side(size, kind)
        vis = _patchlink.target(side, windowed=side != size) if len(imgs) == 1 else None
        gen0 = vis._patch_gen if vis is not None else 0
        out = _SliceImgs.apply(img, tdev, meta, vis)
        if vis is not None and vis._patch_gen != gen0:
            _patchlink.stamp(out, vis, hi - lo)
        sliced.append(out)
    return sliced


def apply_transform_standalone(x, transform):
    """transform(x) outside slice_imgs: every image of the batch is an identity crop (csize == size). As in the reference
    (torchvision draws get_params ONCE per call, transforms.py:165-170), one parameter row is drawn per call and applied to
    every image of the batch. transforms_custom / transforms_elastic return [N,3,s+8,s+8]."""
    require_cuda(x, 'transform input')
    n, c, h, w = x.shape
    assert c == 3 and h == w, 'fused transforms expect [N,3,s,s]'
    tab = np.zeros((1, _rng.CROP_PARAM_FLOATS), np.float32)
    tab[0, _rng.F_CSIZE] = h
    tab[0, _rng.F_ROT:_rng.F_ROT + 4] = (1., 0., 0., 1.)
    if transform.kind == _rng.TF_FAST:
        tab[0, _rng.F_FLAGS] = _rng.draw_fast(tab[0], h)
    elif transform.kind in (_rng.TF_CUSTOM, _rng.TF_ELASTIC):
        tab[0, _rng.F_FLAGS] = _rng.draw_kornia(tab[0], h, transform.kind == _rng.TF_ELASTIC)
    tdev = torch.from_numpy(tab).to(x.device)
    meta = (h, w, 0, 0, 1, h, transform.kind, 1.)
    return torch.cat([_SliceImgs.apply(x[i:i + 1], tdev, meta, None) for i in range(n)], 0)


# ---------------------------------------------------------------------------------------------- loss
class _SimFused(torch.autograd.Function):
    @staticmethod
    def forward(ctx, v1, v2, kind):
        a = v1.detach().contiguous().float().reshape(-1, v1.shape[-1])
        b = v2.detach().contiguous().float().reshape(-1, v2.shape[-1])
        S, D = b.shape
        val = torch.empty((), device=b.device, dtype=torch.float32)
        g1 = torch.empty_like(a) if ctx.needs_input_grad[0] else None
        g2 = torch.empty_like(b) if ctx.needs_input_grad[1] else None
        check(lib().aph_sim_fwd(a.data_ptr(), a.shape[0], b.data_ptr(), S, D, kind, val.data_ptr(),
                                g1.data_ptr() if g1 is not None else None, g2.data_ptr() if g2 is not None else None, stream_ptr()),
              'aph_sim_fwd')
        ctx.shapes = (v1.shape, v2.shape)
        ctx.save_for_backward(*[t for t in (g1, g2) if t is not None])
        ctx.has = (g1 is not None, g2 is not None)
        return val

    @staticmethod
    def backward(ctx, g):
        saved = list(ctx.saved_tensors)
        g1 = saved.pop(0) if ctx.has[0] else None
        g2 = saved.pop(0) if ctx.has[1] else None
        return (g * g1).reshape(ctx.shapes[0]) if g1 is not None else None, (g * g2).reshape(ctx.shapes[1]) if g2 is not None else None, None


def dot_compare(v1, v2, cossim_pow=0):
    dot = (v1 * v2).sum()
    mag = torch.sqrt(torch.sum(v2 ** 2))
    cossim = dot / (1e-6 + mag)
    return dot * cossim ** cossim_pow


def sim_func(v1, v2, type=None):
    """Drop-in for utils.py:276-295. The script's defaults ('mix'; plain cosine with --dualmod) run in one fused
    kernel; the rarely used 'spher' / 'ang' / 'dot' variants are composed from torch ops on the [S,512] embeddings."""
    fused_kind = None
    if type is not None and 'mix' in type:
        fused_kind = 1
    elif type is None or not any(k in type for k in ('spher', 'ang', 'dot')):
        fused_kind = 0
    if fused_kind is not None and v1.is_cuda and v2.is_cuda and v1.dim() == 2 and v2.dim() == 2 and v1.shape[-1] == v2.shape[-1]:
        out = None
        if v1.shape[0] in (1, v2.shape[0]):
            out = _SimFused.apply(v1, v2, fused_kind)
        elif v2.shape[0] == 1:                               # both similarities are symmetric in their arguments
            out = _SimFused.apply(v2, v1, fused_kind)
        if out is not None:
            if _trace.enabled():
                _trace.sim(out.item())
            return out
    if type is not None and 'mix' in type:
        coss = torch.cosine_similarity(v1, v2, dim=-1).mean()
        a = F.normalize(v1, dim=-1); b = F.normalize(v2, dim=-1)
        spher = torch.abs((a - b).norm(dim=-1).div(2).arcsin().pow(2).mul(2)).mean()
        return coss - 0.25 * spher
    elif type is not None and 'spher' in type:
        a = F.normalize(v1, dim=-1); b = F.normalize(v2, dim=-1)
        return (a - b).norm(dim=-1).div(2).arcsin().pow(2).mul(2)
    elif type is not None and 'ang' in type:
        return 1 - torch.acos(torch.cosine_similarity(v1, v2, dim=-1)).mean() / np.pi
    elif type is not None and 'dot' in type:
        return dot_compare(v1, v2, cossim_pow=1)
    return torch.cosine_similarity(v1, v2, dim=-1).mean()


# ---------------------------------------------------------------------------------------------- helpers clip_fft.py imports
def old_torch():
    ver = [int(i) for i in torch.__version__.split('.')[:2]]
    return True if (ver[0] < 2 and ver[1] < 8) else False


def txt_clean(txt):
    return txt.translate(str.maketrans(dict.fromkeys(list("\n',.вЂ”|!?/:;\\"), ""))).replace(' ', '_').replace('"', '')


def basename(file):
    return os.path.splitext(os.path.basename(file))[0]


# ---- preview read-back and write-out (SURVEY.md 8 row f1). clip_fft.py:297-306 runs, every `opt_step` (default: EVERY step),
#   img = image_f(contrast=a.contrast).cpu().numpy()[0];  checkout(img, '%04d.jpg')
# i.e. a forward-only synthesis, an 11 MB device->host read-back and a JPEG encode (~25 ms on the host -- several GPU steps).
# Here (i) image_f under no_grad returns a tensor whose .cpu() lands in a ring of PINNED host buffers (one async copy + one event
# wait instead of a pageable staging copy), (ii) checkout() recognises a view of such a buffer and hands it to the encoder pool
# WITHOUT copying it, (iii) clip / convert / JPEG-encode run on the pool. A ring slot is reused only when nothing references it
# any more (the encoder's reference and the script's `img` both gone), so holding on to a frame stays safe.
_pending = []
_pool = None


class _PinnedFrame(torch.Tensor):
    """CPU tensor living in a pinned ring slot; .numpy() returns the slot's ONE ndarray object, so that views of it
    (`.numpy()[0]`) keep that object referenced and the ring can tell when a slot is free again."""
    _aph_arr = None

    def numpy(self, *args, **kwargs):
        return self._aph_arr


class _PreviewRing:
    MAX_SLOTS = 24

    def __init__(self):
        self.slots = {}                      # shape -> [(pinned CPU tensor, its ndarray), ...]

    def owner_of(self, arr):
        """True if `arr` (an ndarray) is a view of a ring slot."""
        b = arr
        while isinstance(b, np.ndarray) and b.base is not None and isinstance(b.base, np.ndarray):
            b = b.base
        return any(b is a for ring in self.slots.values() for (_t, a) in ring)

    def fetch(self, dev_tensor):
        import sys
        shape = tuple(dev_tensor.shape)
        ring = self.slots.setdefault(shape, [])
        slot = None
        for entry in ring:
            if sys.getrefcount(entry[1]) <= 2:     # the ring's tuple + getrefcount's argument: no view of the slot is alive
                slot = entry
                break
        plain = dev_tensor.as_subclass(torch.Tensor)
        if slot is None:
            if len(ring) >= self.MAX_SLOTS:        # every slot is still referenced (encoder backlog): ordinary pageable copy
                return plain.cpu()
            t = torch.empty(shape, dtype=dev_tensor.dtype).pin_memory()
            slot = (t, t.numpy())
            ring.append(slot)
        slot[0].copy_(plain, non_blocking=True)
        ev = torch.cuda.Event(); ev.record(); ev.synchronize()
        out = slot[0].as_subclass(_PinnedFrame)
        out._aph_arr = slot[1]
        return out


_ring = _PreviewRing()


class PreviewTensor(torch.Tensor):
    """What image_f returns under torch.no_grad(): an ordinary CUDA tensor whose .cpu() uses the pinned ring."""

    def cpu(self, *args, **kwargs):
        if args or kwargs or not self.is_cuda:
            return self.as_subclass(torch.Tensor).cpu(*args, **kwargs)
        return _ring.fetch(self)


def _drain_saves():
    while _pending:
        _pending.pop(0).result()


def _imsave(path, img):
    try:
        from imageio import imsave
    except ImportError:                 # imageio absent and dropin/ not on the path: same PIL encoder dropin/imageio wraps
        from PIL import Image
        Image.fromarray(img).save(path, **({'quality': 95} if path.lower().endswith(('.jpg', '.jpeg')) else {}))
        return
    imsave(path, img)


def _encode_save(fname, chw):
    # utils.py:98-100: transpose to HWC, clip(img*255, 0, 255) -> uint8. Done channel-major on contiguous memory, then ONE
    # transposing uint8 copy: the encoder gets a C-contiguous HWC buffer (a strided view costs PIL an extra 10 ms tobytes()).
    x = np.multiply(chw, np.float32(255.))
    np.clip(x, 0, 255, out=x)
    img = np.ascontiguousarray(np.transpose(x.astype(np.uint8), (1, 2, 0)))
    # encode under a temporary name in the same directory, then rename: a reader of the directory (ffmpeg, img_list) never
    # sees a half-written frame. The temporary keeps the extension so the encoder still picks the format from it.
    base, ext = os.path.splitext(fname)
    tmp = '%s.tmp%d%s' % (base, os.getpid(), ext)
    _imsave(tmp, img)
    os.replace(tmp, fname)


def _submit_save(fname, chw):
    global _pool
    if os.environ.get('APH_SYNC_SAVE', '0') == '1':
        _encode_save(fname, chw)
        return
    if _pool is None:
        import atexit
        from concurrent.futures import ThreadPoolExecutor
        ncpu = len(os.sched_getaffinity(0)) if hasattr(os, 'sched_getaffinity') else (os.cpu_count() or 4)
        _pool = ThreadPoolExecutor(max_workers=int(os.environ.get('APH_SAVE_THREADS', str(max(2, min(8, ncpu // 2))))))
        atexit.register(_drain_saves)
    while _pending and _pending[0].done():
        _pending.pop(0).result()
    while len(_pending) > 64:          # bound the queue (and host memory) if the encoder cannot keep up
        _pending.pop(0).result()
    _pending.append(_pool.submit(_encode_save, fname, chw))


def img_list(path, subdir=None):
    _drain_saves()
    if subdir is True:
        files = [os.path.join(dp, f) for dp, dn, fn in os.walk(path) for f in fn]
    else:
        files = [os.path.join(path, f) for f in os.listdir(path)]
    files = [f for f in files if os.path.splitext(f.lower())[1][1:] in ['jpg', 'jpeg', 'png', 'ppm', 'tif']]
    return sorted([f for f in files if os.path.isfile(f)])


def _pil_imread(path):
    """imageio.imread's decoding through PIL (what dropin/imageio uses): palette images come back as RGB(A) colours."""
    from PIL import Image
    with Image.open(path) as im:
        if im.mode == 'P':
            im = im.convert('RGBA' if 'transparency' in im.info else 'RGB')
        return np.asarray(im)


def img_read(path):
    try:
        from imageio import imread
    except ImportError:
        imread = _pil_imread
    img = imread(path)
    if (img.ndim == 2) or (img.shape[2] == 1):
        img = np.dstack((img, img, img))
    if img.shape[2] == 4:
        img = img[:, :, :3]
    return img


def checkout(img, fname=None, verbose=False):
    """utils.py:94-100: CHW float -> HWC uint8 -> file (rank 0 only under torchrun). The cv2 preview is dropped."""
    if fname is not None and _dist.rank() == 0:
        if isinstance(img, np.ndarray) and img.dtype == np.float32 and _ring.owner_of(img):
            _submit_save(fname, img)                                   # a view of a pinned ring slot: no copy, the slot stays referenced
        else:
            _submit_save(fname, np.array(img, dtype=np.float32))       # private copy; conversion + encode happen off-thread


class _Derivat(torch.autograd.Function):
    @staticmethod
    def forward(ctx, img):
        x = img.detach().contiguous().float()
        C, H, W = x.shape[0] * x.shape[1], x.shape[2], x.shape[3]
        sums = torch.empty(2, device=x.device, dtype=torch.float64)
        val = torch.empty((), device=x.device, dtype=torch.float32)
        check(lib().aph_derivat_fwd(x.data_ptr(), C, H, W, sums.data_ptr(), val.data_ptr(), stream_ptr()), 'aph_derivat_fwd')
        ctx.save_for_backward(x)
        return val

    @staticmethod
    def backward(ctx, g):
        x, = ctx.saved_tensors
        up = g.detach().float().reshape(1).contiguous()
        grad = torch.empty_like(x)
        check(lib().aph_derivat_bwd(x.data_ptr(), x.shape[0] * x.shape[1], x.shape[2], x.shape[3], up.data_ptr(), grad.data_ptr(), stream_ptr()),
              'aph_derivat_bwd')
        return grad


class _DerivatSobel(torch.autograd.Function):
    @staticmethod
    def forward(ctx, img):
        x = img.detach().contiguous().float()
        C, H, W = x.shape[0] * x.shape[1], x.shape[2], x.shape[3]
        sums = torch.empty(1, device=x.device, dtype=torch.float64)
        val = torch.empty((), device=x.device, dtype=torch.float32)
        check(lib().aph_derivat_sobel_fwd(x.data_ptr(), C, H, W, sums.data_ptr(), val.data_ptr(), stream_ptr()), 'aph_derivat_sobel_fwd')
        ctx.save_for_backward(x)
        return val

    @staticmethod
    def backward(ctx, g):
        x, = ctx.saved_tensors
        up = g.detach().float().reshape(1).contiguous()
        grad = torch.empty_like(x)
        check(lib().aph_derivat_sobel_bwd(x.data_ptr(), x.shape[0] * x.shape[1], x.shape[2], x.shape[3], up.data_ptr(), grad.data_ptr(),
                                          stream_ptr()), 'aph_derivat_sobel_bwd')
        return grad


def derivat(img, mode='sobel'):
    """utils.py:256-268. clip_fft.py:272 passes mode='naiv' (the finite-difference branch), cppn.py:292 mode='sobel'
    (mean |kornia spatial_gradient|): each is one fused reduction kernel + its adjoint (csrc/loss.cu). 'scharr' is not provided."""
    if mode == 'scharr':
        raise NotImplementedError("aphantasia_b200.derivat: mode='scharr' is not provided; 'sobel' and the finite-difference mode are")
    require_cuda(img, 'derivat input')
    if mode == 'sobel':
        assert img.dim() == 4, 'derivat expects [N,C,H,W]'
        return _DerivatSobel.apply(img)
    assert img.dim() == 4 and img.shape[2] > 1 and img.shape[3] > 1, 'derivat expects [N,C,H,W]'
    return _Derivat.apply(img)


class _Head(torch.autograd.Function):
    @staticmethod
    def forward(ctx, emb, w, b):
        e = emb.detach().contiguous().float()
        S, D = e.shape
        out = torch.empty(S, 1, device=e.device, dtype=torch.float32)
        check(lib().aph_head_fwd(e.data_ptr(), S, D, w.data_ptr(), b.data_ptr(), out.data_ptr(), stream_ptr()), 'aph_head_fwd')
        ctx.save_for_backward(w)
        ctx.shape = (S, D)
        return out

    @staticmethod
    def backward(ctx, g):
        w, = ctx.saved_tensors
        S, D = ctx.shape
        g = g.contiguous().float()
        ge = torch.empty(S, D, device=g.device, dtype=torch.float32)
        check(lib().aph_head_bwd(g.data_ptr(), w.data_ptr(), S, D, ge.data_ptr(), stream_ptr()), 'aph_head_bwd')
        return ge, None, None


class AestheticHead:
    """What clip_fft.py needs from the nn.Linear(512, 1) the reference returns (utils.py:410-413): .cuda(), __call__([S,512]) -> [S,1]."""

    def __init__(self, weight, bias, synthetic):
        self.weight, self.bias, self.synthetic = weight.reshape(-1).float().contiguous(), bias.reshape(-1).float().contiguous(), synthetic

    def cuda(self):
        self.weight, self.bias = self.weight.cuda(), self.bias.cuda()
        return self

    def eval(self): return self
    def half(self): return self
    def float(self): return self

    def __call__(self, emb):
        require_cuda(emb, 'aesthetic head input')
        if not self.weight.is_cuda:
            self.cuda()
        return _Head.apply(emb, self.weight, self.bias)


def aesthetic_model(clip_model='ViT-B/32'):
    """utils.py:402-413: the LAION linear aesthetic predictor on CLIP embeddings. The reference downloads
    sa_0_4_<model>_linear.pth; here it is read from the working directory (the reference's own cache location) or
    $APH_AEST_WEIGHTS if present, otherwise -- no network in this environment -- a seeded synthetic head is used, loudly."""
    nf = 768 if clip_model == 'ViT-L/14' else 512 if clip_model in ['ViT-B/16', 'ViT-B/32'] else None
    if nf is None:
        return None
    name = clip_model.replace('/', '_').replace('-', '_').lower()
    for path in (os.environ.get('APH_AEST_WEIGHTS'), 'sa_0_4_%s_linear.pth' % name):
        if path and os.path.isfile(path):
            sd = torch.load(path, map_location='cpu')
            return AestheticHead(sd['weight'], sd['bias'], False)
    print(' [aphantasia_b200] no aesthetic-predictor weights (sa_0_4_%s_linear.pth) available: using a seeded synthetic linear head' % name)
    g = torch.Generator().manual_seed(4321)
    return AestheticHead((torch.rand(nf, generator=g) * 2 - 1) * nf ** -0.5, torch.zeros(1), True)


def plot_text(txt, size=224):
    raise NotImplementedError('aphantasia_b200: plot_text needs matplotlib; never called by clip_fft.py')


# ---------------------------------------------------------------------------------------------- helpers illustrip.py / illustra.py import
# (illustrip.py:28, illustra.py:19). Host-side list, path and timeline helpers; the values they return are the original's
# (utils.py:32-38, 47-59, 102-126, 149-216, 299-396), bit for bit where NumPy / SciPy compute them.
def intrl(a, b, step=2):
    """Replaces every `step`-th entry of list `a` (from index `step` on) by the entry of `b` at that index, in place."""
    assert len(a) == len(b), ' diff lengths: %d %d' % (len(a), len(b))
    assert step > 1
    for k in range(step, len(a), step):
        a[k] = b[k]
    return a


def file_list(path, ext=None, subdir=None):
    """Sorted paths of the files in `path` (recursively with subdir=True); ext: a suffix string, or a list of extensions."""
    if subdir is True:
        found = [os.path.join(d, f) for d, _, names in os.walk(path) for f in names]
    else:
        found = [os.path.join(path, f) for f in os.listdir(path)]
    if isinstance(ext, list):
        found = [f for f in found if os.path.splitext(f.lower())[1][1:] in ext]
    elif isinstance(ext, str):
        found = [f for f in found if f.endswith(ext)]
    elif ext is not None:
        print(' Unknown extension/type for file list!')
    return sorted(f for f in found if os.path.isfile(f))


def cvshow(img):
    """The original opens an OpenCV preview window; there is no display to show it on, so this does nothing."""


def _write_dict(d, out, indent=''):
    for k in sorted(d.keys()):
        v = d[k]
        if isinstance(v, collections.abc.Mapping):
            out(indent + str(k), ' \n')
            _write_dict(v, out, indent + '   ')
        else:
            out('%s%s: %s' % (indent, str(k), str(v)), ' \n')


def save_cfg(args, dir='./', file='config.txt'):
    """Writes the arguments (a Namespace or a dict), sorted by name, one `name: value ` line each, to dir/file; prints
    them when file is None."""
    if dir != '':
        os.makedirs(dir, exist_ok=True)
    try:
        args = vars(args)
    except TypeError:
        pass
    if file is None:
        _write_dict(args, lambda line, end: print(line))
    else:
        with open(os.path.join(dir, file), 'w') as f:
            _write_dict(args, lambda line, end: f.write(line + end))


def tile_pad(xt, padding, symm=False):
    """Pads the last two axes by (left, right, top, bottom) by repeating the image (symm=True: mirroring it), for any pad
    length: every padded index maps back into the image through a periodic index map."""
    h, w = xt.shape[-2:]
    left, right, top, bottom = padding

    def wrap(idx, lo, hi):
        period = hi - lo
        if symm is True:
            m = np.fmod(idx - lo, 2 * period)
            m = np.where(m < 0, m + 2 * period, m)
            m = np.where(m >= period, 2 * period - m, m) + lo
        else:
            m = np.remainder(idx - lo, period) + lo
        return np.array(m, dtype=idx.dtype)

    cols = wrap(np.arange(-left, w + right), -0.5, w - 0.5)
    rows = wrap(np.arange(-top, h + bottom), -0.5, h - 0.5)
    xx, yy = np.meshgrid(cols, rows)
    return xt[..., yy, xx]


def pad_up_to(x, size, type='centr'):
    """Pads [..., H, W] up to size = (H', W') with tile_pad: centred by default, at the far side with 'side' in type,
    mirrored with 'symm' in type."""
    if list(x.shape[2:]) == list(size):
        return x
    padding = []
    for have, want in zip(list(x.shape[2:])[::-1], list(size)[::-1]):     # width first, then height
        extra = want - have
        first = 0 if 'side' in type.lower() else extra // 2
        padding += [first, extra - first]
    return tile_pad(x, padding, symm=('symm' in type.lower()))


def smoothstep(x, NN=1., xmin=0., xmax=1.):
    """The order-N smoothstep polynomial of x clipped to [xmin, xmax], N = ceil(NN); a fractional NN averages it with x."""
    import scipy.special
    N = math.ceil(NN)
    x = np.clip((x - xmin) / (xmax - xmin), 0, 1)
    poly = 0
    for n in range(N + 1):
        poly += scipy.special.comb(N + n, n) * scipy.special.comb(2 * N + 1, N - n) * (-x) ** n
    poly *= x ** (N + 1)
    return (x + poly) / 2 if NN != N else poly


def _steps01(num_steps, smooth):
    xs = [k / (num_steps - 1) for k in range(num_steps)]
    return [smoothstep(x, smooth) for x in xs] if smooth > 0 else xs


def slerp(z1, z2, num_steps=None, x=None, smooth=0.5):
    """Torch tensors z1 -> z2: the straight line between them, rescaled at each point to |z1| over the norm of the line
    from z1 to z2 rescaled to |z1|. num_steps points from 0 to 1, or the single point x; concatenated along axis 0."""
    n1 = z1.norm()
    z2_on_sphere = z2 * (n1 / z2.norm())
    xs = _steps01(num_steps, 0) if num_steps is not None else [x]
    if smooth > 0:
        xs = [smoothstep(t, smooth) for t in xs]
    out = []
    for t in xs:
        plain = z1 + (z2 - z1) * t
        norm = (z1 + (z2_on_sphere - z1) * t).norm()
        if norm != 0:
            point = plain * (n1 / norm)
        out.append(point)          # a zero norm repeats the previous point, as the original does
    return torch.cat(out)


def get_z(shape, rnd, uniform=False):
    return rnd.uniform(0., 1., shape) if uniform else rnd.randn(*shape)


def lerp(z1, z2, num_steps, smooth=0.):
    return np.array([z1 + (z2 - z1) * t for t in _steps01(num_steps, smooth)])


def slerp_np(z1, z2, num_steps, smooth=0.):
    """NumPy slerp (see slerp) with num_steps points from z1 to z2."""
    n1 = np.linalg.norm(z1)
    z2_on_sphere = z2 * (n1 / np.linalg.norm(z2))
    out = []
    for t in _steps01(num_steps, smooth):
        plain = z1 + (z2 - z1) * t
        out.append(plain * (n1 / np.linalg.norm(z1 + (z2_on_sphere - z1) * t)))
    return np.array(out)


def cublerp(points, steps, fstep, looped=True):
    """Cubic spline through `steps` key points placed fstep frames apart, closed by the first point (looped) or the last:
    steps * fstep + 1 frames."""
    from scipy.interpolate import CubicSpline
    keys = np.array([k * fstep for k in range(steps + 1)])
    closing = points[0] if looped is True else points[-1]
    spline = CubicSpline(keys, np.concatenate((points, np.expand_dims(closing, 0))))
    return spline(np.arange(steps * fstep + 1))


def _clock_seed():
    """What the original's latent_anima does without a seed: reseed NumPy's global stream from the clock
    (np.random.seed(int((time.time() % 1) * 9999)), whose None return becomes the seed) and draw the key latents from a
    RandomState seeded by the OS. Returns that RandomState's seed, drawn here so it can be shared: under torchrun rank 0's
    clock value and seed are broadcast, so that every rank moves its replicated canvas the same way and continues the same
    NumPy stream (the crop replay reads it)."""
    import time
    vals = np.array([int((time.time() % 1) * 9999)] + list(np.frombuffer(os.urandom(16), np.uint32)), np.int64)
    if _dist.world() > 1:
        t = torch.from_numpy(vals).to('cuda' if _dist.backend_is_nccl() else 'cpu')
        torch.distributed.broadcast(t, 0)
        vals = t.cpu().numpy()
    np.random.seed(int(vals[0]))
    return vals[1:].astype(np.uint32)


def latent_anima(shape, frames, transit, key_latents=None, smooth=0.5, uniform=False, cubic=False, gauss=False, start_lat=None,
                 seed=None, looped=True, verbose=False):
    """A timeline of `frames` latents of `shape`: key latents drawn (or given) every `transit` frames, joined by a cubic
    spline (cubic=True) or by lerp (uniform=True) / slerp segments, optionally smoothed by a wrapped Gaussian."""
    if key_latents is None:
        transit = int(max(1, min(frames // 2, transit)))
    steps = max(1, math.ceil(frames / transit))
    log = ' timeline: %d steps by %d' % (steps, transit)
    rnd = np.random.RandomState(_clock_seed() if seed is None else seed)
    if key_latents is None:
        key_latents = np.array([get_z(shape, rnd, uniform) for _ in range(steps)])
    if start_lat is not None:
        key_latents[0] = start_lat

    if transit == 1:
        latents = key_latents
    elif cubic:
        latents = cublerp(key_latents, steps, transit, looped)
        log += ', cubic'
    else:
        parts = [np.expand_dims(key_latents[0], 0)]
        for k in range(steps):
            nxt = (k + 1) % steps if looped is True else min(k + 1, steps - 1)
            join = lerp if uniform is True else slerp_np
            parts.append(join(key_latents[k], key_latents[nxt], transit, smooth=smooth))
        latents = np.concatenate(parts)
    latents = np.array(latents)

    if gauss:
        from scipy.ndimage import gaussian_filter
        blurred = gaussian_filter(latents, [transit, 0, 0], mode='wrap')
        latents = blurred / np.linalg.norm(blurred, axis=-1, keepdims=True) * math.sqrt(np.prod(shape))
        log += ', gauss'
    if verbose:
        print(log)
    return latents[1:] if latents.shape[0] > frames else latents
