"""Test infrastructure: CPU restatement of transforms_custom / transforms_elastic (reference aphantasia/transforms.py:147-163) on
top of oracle.restate's crop + bicubic resize, for the fused sampler's kinds 3 and 4.

The reference builds the rotation, elastic and jitter stages on kornia, which is absent here. The functions marked "unpinned"
restate kornia's documented semantics, with sampling positions in float64 (the exact map; kornia itself works in float32);
the rotation convention is cross-checked against OpenCV's warpAffine
(test_transforms_kornia_host.py). The reference's own pad, erase and normalise values, the per-crop parameters and the input of
every kornia call are pinned by tests/golden/reference_golden_transforms.npz (tests/golden/make_golden_transforms.py).
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import restate as R

KORNIA_PAD = 4
F_ANGLE, F_JIT_DX, F_JIT_DY = 20, 21, 22
FLAG_ELASTIC = 16


def kornia_rotation_matrix(angle, c):
    """unpinned: kornia get_rotation_matrix2d (OpenCV getRotationMatrix2D convention), scale 1, centre (c, c) -> [2, 3] float64."""
    a, b = math.cos(math.radians(angle)), math.sin(math.radians(angle))
    return np.array([[a, b, (1 - a) * c - b * c], [-b, a, b * c + (1 - a) * c]])


def warp_affine(img, M):
    """unpinned: kornia warp_affine(img, M, dsize=(s, s)) with align_corners=True, bilinear, zeros: out(p) = img(M^-1 p) in pixel
    coordinates; taps outside the image weigh 0 (no renormalisation)."""
    return warp_inverse(img, np.linalg.inv(np.vstack([np.asarray(M, dtype=np.float64).reshape(2, 3), [0, 0, 1]]))[:2])


def warp_inverse(img, Mi):
    """warp_affine given the inverse map Mi [2, 3] (destination pixel -> source pixel)."""
    s = img.shape[-1]
    yy, xx = np.meshgrid(np.arange(s, dtype=np.float64), np.arange(s, dtype=np.float64), indexing='ij')
    sx = Mi[0, 0] * xx + Mi[0, 1] * yy + Mi[0, 2]
    sy = Mi[1, 0] * xx + Mi[1, 1] * yy + Mi[1, 2]
    grid = torch.tensor(np.stack([2 * sx / (s - 1) - 1, 2 * sy / (s - 1) - 1], -1), dtype=torch.float64)[None]
    out = F.grid_sample(img.double(), grid.expand(img.shape[0], s, s, 2), mode='bilinear', padding_mode='zeros', align_corners=True)
    return out.to(img.dtype)


def elastic_zero_noise(img):
    """unpinned: kornia elastic_transform2d with noise = 0: grid_sample(align_corners=False) of the identity mesh built with the
    align_corners=True convention (linspace(-1, 1, s)), i.e. source index j s / (s - 1) - 1/2 per axis."""
    s = img.shape[-1]
    lin = torch.linspace(-1, 1, s, dtype=torch.float64)
    gy, gx = torch.meshgrid(lin, lin, indexing='ij')
    grid = torch.stack([gx, gy], -1)[None].expand(img.shape[0], s, s, 2)
    return F.grid_sample(img.double(), grid, mode='bilinear', padding_mode='zeros', align_corners=False).to(img.dtype)


def translate(img, dx, dy):
    """unpinned: kornia translate by an integer (dx, dy): out(x, y) = img(x - dx, y - dy), zeros outside."""
    out = torch.zeros_like(img)
    s = img.shape[-1]
    out[..., dy:, dx:] = img[..., :s - dy, :s - dx]
    return out


def pad_erase(cut, row, elastic):
    """transforms.py:38-43 pad(4, constant 0.5), then for elastic the RandomErasing rectangle (TV:_functional_tensor.py:931-938)."""
    cut = F.pad(cut, [KORNIA_PAD] * 4, mode='constant', value=0.5)
    if elastic and int(row[R.F_FLAGS]) & R.FLAG_ERASE:
        i, j, h, w = (int(row[k]) for k in (R.F_ER_I, R.F_ER_J, R.F_ER_H, R.F_ER_W))
        cut = cut.clone()
        cut[..., i:i + h, j:j + w] = 0
    return cut


def kornia_stages(cut, row, elastic):
    """After the resize: pad -> [erase] -> random_rotate -> [random_elastic] -> jitter(8); normalise is the caller's."""
    cut = pad_erase(cut, row, elastic)
    # the table's float32 inverse rotation about c = (s - 1) / 2 (the sampler's operand), applied in float64
    c = (cut.shape[-1] - 1) / 2
    r = np.asarray(row[R.F_ROT:R.F_ROT + 4], np.float64)
    cut = warp_inverse(cut, np.array([[r[0], r[1], c - r[0] * c - r[1] * c], [r[2], r[3], c - r[2] * c - r[3] * c]]))
    if elastic:
        cut = elastic_zero_noise(cut)
    return translate(cut, int(row[F_JIT_DX]), int(row[F_JIT_DY]))


def sample_crops(canvas, table, size=224, kind=3, frame=None):
    """slice_imgs with transforms_custom (kind 3) or transforms_elastic (kind 4): canvas [1,3,H,W] -> [S,3,size+8,size+8]."""
    assert kind in (3, 4)
    if frame is not None:
        canvas = R.wrap_pad(canvas, frame)
    mean = torch.tensor(R.CLIP_MEAN).view(1, 3, 1, 1)
    std = torch.tensor(R.CLIP_STD).view(1, 3, 1, 1)
    cuts = []
    for row in np.asarray(table):
        oy, ox, cs = int(row[R.F_OFFY]), int(row[R.F_OFFX]), int(row[R.F_CSIZE])
        cut = F.interpolate(canvas[:, :, oy:oy + cs, ox:ox + cs], (size, size), mode='bicubic', align_corners=True)
        cuts.append((kornia_stages(cut, row, kind == 4) - mean) / std)
    return torch.cat(cuts, 0)


def reference_step(params, scale, hw, colcorr_t, table, visual, txt_emb, kind, sim='mix', size=224, contrast=1.):
    """oracle.restate.reference_step with transforms_custom / _elastic: the encoder (conv1, kernel = stride = patch) reads the
    top-left input_resolution window of the size + 8 crops."""
    h, w = hw
    p = params.detach().clone().requires_grad_(True)
    rgb = R.valid_rgb(R.synth_fft(p, scale, h, w, None, contrast), colcorr_t)
    crops = sample_crops(rgb, table, size, kind)
    r = visual.input_resolution
    emb = visual(crops[:, :, :r, :r].contiguous())
    loss = -1. * R.sim_func(txt_emb, emb, sim)
    loss.backward()
    return loss.detach(), p.grad, emb.detach()
