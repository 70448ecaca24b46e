"""Host-side replay of the reference's per-crop random draws -> crop parameter table.

The reference draws its sampling / augmentation randomness on the host, per crop, from two generators
(torch's default CPU generator and NumPy's global legacy RandomState), in a data-dependent order:

  /root/reference/aphantasia/utils.py:222-228   rnd_size, rnd_offx, rnd_offy  (torch.rand / randn, [count])
  /root/reference/aphantasia/utils.py:244       torch.rand(1) < macro         (per crop, always drawn)
  /root/reference/aphantasia/utils.py:245-247   csize / offsetx / offsety     (fp32 tensor lerp, .int() trunc)
  torchvision transforms.py:811,829-846         RandomPerspective: rand(1) < p, then 8x randint on hit
  torchvision transforms.py:1727,1697-1714      RandomErasing: rand(1) < p, then <=10x (uniform_, uniform_), randint x2
  /root/reference/aphantasia/transforms.py:75   np.random.choice(angles)      (NumPy global RNG)

This module performs the *same calls in the same order* (so identical seeds give identical crops) and
packs the result into a float32 table [count, CROP_PARAM_FLOATS] that one CUDA launch consumes
(include/aphb200.h: aph_sample_fwd). No image data is touched here.
"""
import math

import numpy as np
import torch

CROP_PARAM_FLOATS = 24
# field offsets inside one table row (all stored as float32; integer fields are exact: |v| < 2^24)
F_OFFY, F_OFFX, F_CSIZE, F_FLAGS = 0, 1, 2, 3
F_PERSP = 4          # 8 floats a..h  (output -> input mapping, torchvision convention)
F_ER_I, F_ER_J, F_ER_H, F_ER_W = 12, 13, 14, 15
F_ROT = 16           # theta00, theta01, theta10, theta11 (inverse affine matrix, float32)
F_ANGLE = 20         # degrees (informational)
F_JIT_DX, F_JIT_DY = 21, 22    # custom / elastic: integer jitter shift
FLAG_PERSP, FLAG_ERASE, FLAG_ROT, FLAG_JITTER, FLAG_ELASTIC = 1, 2, 4, 8, 16

# transform kinds understood by the fused sampler
TF_NONE, TF_NORMALIZE, TF_FAST, TF_CUSTOM, TF_ELASTIC = 0, 1, 2, 3, 4
KORNIA_PAD = 4       # pad(4) of transforms_custom / transforms_elastic: their output side is size + 8


def out_side(size, kind):
    """Side of the crops slice_imgs returns for transform `kind`."""
    return size + 2 * KORNIA_PAD if kind in (TF_CUSTOM, TF_ELASTIC) else size

FAST_ANGLES = list(range(-30, 30)) + 20 * [0]   # reference transforms.py:168
PERSP_DISTORTION, PERSP_P = 0.33, 0.2           # reference transforms.py:166
ERASE_P, ERASE_SCALE, ERASE_RATIO = 0.2, (0.02, 0.33), (0.3, 3.3)  # transforms.py:167 + torchvision defaults


def perspective_coeffs(startpoints, endpoints):
    """8 perspective coefficients, float64 least squares then cast to float32.
    Same construction as torchvision functional.py:674-704 (what RandomPerspective executes)."""
    a = torch.zeros(8, 8, dtype=torch.float64)
    for i, (p1, p2) in enumerate(zip(endpoints, startpoints)):
        a[2 * i, :] = torch.tensor([p1[0], p1[1], 1, 0, 0, 0, -p2[0] * p1[0], -p2[0] * p1[1]])
        a[2 * i + 1, :] = torch.tensor([0, 0, 0, p1[0], p1[1], 1, -p2[1] * p1[0], -p2[1] * p1[1]])
    b = torch.tensor(startpoints, dtype=torch.float64).view(8)
    return torch.linalg.lstsq(a, b, driver='gels').solution.to(torch.float32).tolist()


def inverse_rotation_matrix(angle):
    """theta = [cos, sin, -sin, cos] of the inverse affine matrix for a pure rotation about (0,0)
    (torchvision functional.py:1029-1052 with center=translate=shear=0, scale=1)."""
    rot = math.radians(angle)
    a = math.cos(rot); b = -math.sin(rot); c = math.sin(rot); d = math.cos(rot)
    return [d, -b, -c, a]


def kornia_inverse_rotation(angle):
    """Pixel-space inverse of kornia's get_rotation_matrix2d (OpenCV convention: positive = counter-clockwise on screen):
    source = c + [[cos, -sin], [sin, cos]] (dest - c), as [r00, r01, r10, r11]."""
    rot = math.radians(angle)
    return [math.cos(rot), -math.sin(rot), math.sin(rot), math.cos(rot)]


def draw_erase(row, side):
    """RandomErasing(p=0.2), value=0 (torchvision transforms.py:1697-1727) on an image of side `side`: FLAG_ERASE or 0."""
    if not torch.rand(1) < ERASE_P:
        return 0
    area = side * side
    log_ratio = torch.log(torch.tensor(ERASE_RATIO))
    for _ in range(10):
        erase_area = area * torch.empty(1).uniform_(ERASE_SCALE[0], ERASE_SCALE[1]).item()
        aspect = torch.exp(torch.empty(1).uniform_(log_ratio[0], log_ratio[1])).item()
        h = int(round(math.sqrt(erase_area * aspect)))
        w = int(round(math.sqrt(erase_area / aspect)))
        if not (h < side and w < side):
            continue
        i = torch.randint(0, side - h + 1, size=(1,)).item()
        j = torch.randint(0, side - w + 1, size=(1,)).item()
        row[F_ER_I], row[F_ER_J], row[F_ER_H], row[F_ER_W] = i, j, h, w
        return FLAG_ERASE
    return 0


def draw_kornia(row, size, elastic):
    """Draws one crop's transforms_custom / transforms_elastic parameters into `row` (reference transforms.py:147-163, in order):
    elastic only: RandomErasing on the padded (size + 8) image (torch); random_rotate: np.random.choice(angles); elastic only:
    random_elastic's rand(2), randint(8, 64), rand() (zero noise: drawn, without effect on the output); jitter(8): dx, dy."""
    flags = FLAG_ROT | FLAG_JITTER
    if elastic:
        flags |= draw_erase(row, size + 2 * KORNIA_PAD)
    angle = float(np.random.choice(FAST_ANGLES))
    row[F_ROT:F_ROT + 4] = kornia_inverse_rotation(angle)
    row[F_ANGLE] = angle
    if elastic:
        np.random.rand(2)
        np.random.randint(8, 64)
        np.random.rand()
        flags |= FLAG_ELASTIC
    row[F_JIT_DX] = np.random.choice(8)
    row[F_JIT_DY] = np.random.choice(8)
    return flags


def draw_fast(row, size):
    """Draws one crop's transforms_fast parameters into `row` (numpy float32 view), reference order."""
    flags = 0
    # RandomPerspective(0.33, p=0.2)
    if torch.rand(1) < PERSP_P:
        half = size // 2
        d = int(PERSP_DISTORTION * half)
        ri = lambda lo, hi: int(torch.randint(lo, hi, size=(1,)).item())
        tl = [ri(0, d + 1), ri(0, d + 1)]
        tr = [ri(size - d - 1, size), ri(0, d + 1)]
        br = [ri(size - d - 1, size), ri(size - d - 1, size)]
        bl = [ri(0, d + 1), ri(size - d - 1, size)]
        start = [[0, 0], [size - 1, 0], [size - 1, size - 1], [0, size - 1]]
        row[F_PERSP:F_PERSP + 8] = perspective_coeffs(start, [tl, tr, br, bl])
        flags |= FLAG_PERSP
    flags |= draw_erase(row, size)
    # random_rotate_fast: always executed, even for angle 0
    angle = float(np.random.choice(FAST_ANGLES))
    row[F_ROT:F_ROT + 4] = inverse_rotation_matrix(angle)
    row[F_ANGLE] = angle
    flags |= FLAG_ROT
    return flags


def draw_crop_table(count, canvas_hw, size=224, kind=TF_FAST, align='uniform', macro=0., n_imgs=1):
    """Crop tables for one slice_imgs call, from the native replay (libaphb200.so: aph_rng_crop_tables);
    draw_crop_table_py below is the executable specification it is tested against."""
    return draw_crop_table_native(count, canvas_hw, size, kind, align, macro, n_imgs)


def _frame(H, W, align):
    if 'over' in align:
        fh, fw = (2 * H, 2 * W) if align == 'overmax' else (int(1.5 * H), int(1.5 * W))
    else:
        fh, fw = H, W
    return (fh - H) // 2, (fw - W) // 2, fh, fw


_NP_INPLACE = None     # (bit_generator, address of its mt19937_state) once verified; False if the layout check failed


def _numpy_state_address():
    """Address of the global legacy RandomState's `mt19937_state { uint32_t key[624]; int pos; }` (numpy/random/src/mt19937/
    mt19937.h), so the native replay can continue NumPy's stream in place: np.random.get_state() + set_state() cost 88 us per
    slice_imgs call, more than the replay itself. The layout is verified once against the public state; None -> copy path."""
    global _NP_INPLACE
    import ctypes as C
    rs = np.random.mtrand._rand
    if _NP_INPLACE is None:
        try:
            bg = rs._bit_generator
            addr = int(bg.ctypes.state_address)
            name, key, pos = np.random.get_state()[:3]
            raw = np.frombuffer((C.c_uint32 * 625).from_address(addr), dtype=np.uint32)
            ok = name == 'MT19937' and np.array_equal(raw[:624], np.asarray(key, dtype=np.uint32)) and int(raw[624]) == int(pos)
            _NP_INPLACE = (bg, addr) if ok else False
        except Exception:
            _NP_INPLACE = False
    if _NP_INPLACE and rs._bit_generator is _NP_INPLACE[0]:
        return _NP_INPLACE[1]
    return None


def draw_crop_table_native(count, canvas_hw, size=224, kind=TF_FAST, align='uniform', macro=0., n_imgs=1):
    """Same draws as draw_crop_table_py, but the per-crop loop continues both Mersenne-Twister streams in C."""
    import ctypes as C
    from ._lib import check, lib
    H, W = int(canvas_hw[0]), int(canvas_hw[1])
    rnd_size = torch.rand(count)
    if align == 'central':
        rnd_offx = torch.clip(torch.randn(count) * 0.2 + 0.5, 0., 1.)
        rnd_offy = torch.clip(torch.randn(count) * 0.2 + 0.5, 0., 1.)
    else:
        rnd_offx = torch.rand(count)
        rnd_offy = torch.rand(count)
    pad_top, pad_left, fh, fw = _frame(H, W, align)
    tstate = torch.get_rng_state()
    tabs = np.empty((n_imgs, count, CROP_PARAM_FLOATS), dtype=np.float32)
    addr = _numpy_state_address()
    if addr is not None:                     # NumPy's key[] / pos are advanced where they live
        key_ptr, pos_ptr, np_state = addr, C.cast(addr + 624 * 4, C.POINTER(C.c_int32)), None
    else:
        name, key, pos, has_gauss, cached = np.random.get_state()
        key = np.ascontiguousarray(key, dtype=np.uint32)
        cpos = C.c_int32(int(pos))
        key_ptr, pos_ptr, np_state = key.ctypes.data, C.byref(cpos), (name, key, has_gauss, cached)
    check(lib().aph_rng_crop_tables(tstate.data_ptr(), tstate.numel(), key_ptr, pos_ptr, rnd_size.data_ptr(), rnd_offx.data_ptr(),
                                    rnd_offy.data_ptr(), count, H, W, fh, fw, size, kind, float(macro), n_imgs, tabs.ctypes.data),
          'aph_rng_crop_tables')
    torch.set_rng_state(tstate)
    if np_state is not None:
        np.random.set_state((np_state[0], np_state[1], int(cpos.value), np_state[2], np_state[3]))
    return [tabs[i] for i in range(n_imgs)], (pad_top, pad_left, fh, fw)


def draw_crop_table_py(count, canvas_hw, size=224, kind=TF_FAST, align='uniform', macro=0., n_imgs=1):
    """Replays slice_imgs' draws (reference utils.py:218-254) for `n_imgs` canvases of equal size.

    Returns a list (one per input image) of float32 numpy tables [count, CROP_PARAM_FLOATS] and the
    (pad_top, pad_left, padded_h, padded_w) of the wrap-padded sampling frame ('over*' aligns).
    """
    H, W = int(canvas_hw[0]), int(canvas_hw[1])
    rnd_size = torch.rand(count)
    if align == 'central':
        rnd_offx = torch.clip(torch.randn(count) * 0.2 + 0.5, 0., 1.)
        rnd_offy = torch.clip(torch.randn(count) * 0.2 + 0.5, 0., 1.)
    else:
        rnd_offx = torch.rand(count)
        rnd_offy = torch.rand(count)
    sz_max = torch.min(torch.tensor([H, W]))
    if 'over' in align:
        fh, fw = (2 * H, 2 * W) if align == 'overmax' else (int(1.5 * H), int(1.5 * W))
    else:
        fh, fw = H, W
    pad_top, pad_left = (fh - H) // 2, (fw - W) // 2      # pad_up_to 'centr' (utils.py:183-184)

    lerp = lambda x, a, b: x * (b - a) + a                # utils.py:219-220 (`map`)
    tables = []
    for _ in range(n_imgs):
        tab = np.zeros((count, CROP_PARAM_FLOATS), dtype=np.float32)
        for c in range(count):
            sz_min = 0.9 * sz_max if torch.rand(1) < macro else size
            csize = lerp(rnd_size[c], sz_min, sz_max).int()
            offx = lerp(rnd_offx[c], 0, fw - csize).int()
            offy = lerp(rnd_offy[c], 0, fh - csize).int()
            row = tab[c]
            row[F_OFFY], row[F_OFFX], row[F_CSIZE] = int(offy), int(offx), int(csize)
            row[F_ROT:F_ROT + 4] = (1., 0., 0., 1.)
            flags = 0
            if kind == TF_FAST:
                flags = draw_fast(row, size)
            elif kind in (TF_CUSTOM, TF_ELASTIC):
                flags = draw_kornia(row, size, kind == TF_ELASTIC)
            row[F_FLAGS] = flags
        tables.append(tab)
    return tables, (pad_top, pad_left, fh, fw)


def shard_range(count, rank, world):
    """Contiguous, balanced shard [lo, hi) of the crop index for `rank` of `world`
    (190 over 8 -> 24x6 + 23x2; 87 over 4 -> 22,22,22,21)."""
    base, rem = divmod(count, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)
