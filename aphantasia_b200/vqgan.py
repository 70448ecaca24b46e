"""The VQGAN decoder of CLIP_VQGAN.ipynb (taming.modules.diffusionmodules.model.Decoder) on the GPU, forward and d loss / d z.

`Decoder(**ddconfig)` is an nn.Module with taming's parameter names and shapes, so a parent's `load_state_dict(sd, strict=False)`,
`.cuda()` and `.eval()` work as in the notebook. Its forward runs the `aph_vqgan` handle (csrc/vqgan.cu): bf16 NHWC activations,
3x3 convolutions on tensor cores, GroupNorm statistics in fp32 partials summed in fp64. The weights are constants of the handle,
as the CLIP encoders' are: the backward returns d loss / d z only, and no parameter receives a gradient. The handle is packed from
the parameters on first use and re-packed when one of them changed (its storage or its version counter).
"""
import ctypes as C
from collections import OrderedDict

import torch
import torch.nn as nn

from ._lib import Handle, VqganConfig, check, lib, require_cuda, stream_ptr

MAX_TOKENS = 16384          # T of the attention's T x T scores per image (include/aphb200.h APH_VQGAN_MAX_TOKENS)

# the two decoders of the notebook's models (configs/*.yaml of taming's checkpoints)
F16_CONFIG = dict(double_z=False, z_channels=256, resolution=256, in_channels=3, out_ch=3, ch=128, ch_mult=(1, 1, 2, 2, 4),
                  num_res_blocks=2, attn_resolutions=[16], dropout=0.0)      # vqgan_imagenet_f16_1024 / _16384
F8_CONFIG = dict(double_z=False, z_channels=256, resolution=256, in_channels=3, out_ch=3, ch=128, ch_mult=(1, 1, 2, 4),
                 num_res_blocks=2, attn_resolutions=[32], dropout=0.0)       # gumbel_f8_8192


def _norm(c):
    return nn.GroupNorm(num_groups=32, num_channels=c, eps=1e-6, affine=True)


class ResnetBlock(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.in_channels, self.out_channels = cin, cout
        self.norm1, self.conv1 = _norm(cin), nn.Conv2d(cin, cout, 3, 1, 1)
        self.norm2, self.conv2 = _norm(cout), nn.Conv2d(cout, cout, 3, 1, 1)
        if cin != cout:
            self.nin_shortcut = nn.Conv2d(cin, cout, 1, 1, 0)


class AttnBlock(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.in_channels = c
        self.norm = _norm(c)
        self.q, self.k, self.v, self.proj_out = (nn.Conv2d(c, c, 1, 1, 0) for _ in range(4))


class Upsample(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, 1, 1)


def _attn_levels(ch_mult, resolution, attn_resolutions):
    """taming's rule: level i (0 the finest) has attention when its curr_res, resolution // 2**i, is in attn_resolutions"""
    return [i for i in range(len(ch_mult)) if resolution // 2 ** i in attn_resolutions]


def check_config(ch, out_ch, ch_mult=(1, 2, 4, 8), num_res_blocks=2, attn_resolutions=(), dropout=0.0, resamp_with_conv=True,
                 resolution=256, z_channels=256, give_pre_end=False, **_ignored):
    """Raises NotImplementedError naming the limit for a config the CUDA decoder does not run."""
    if give_pre_end:
        raise NotImplementedError('VQGAN Decoder: give_pre_end=True is not supported (the CUDA decoder ends in conv_out)')
    if not resamp_with_conv:
        raise NotImplementedError('VQGAN Decoder: resamp_with_conv=False is not supported (Upsample runs its 3x3 convolution)')
    if dropout != 0:
        raise NotImplementedError('VQGAN Decoder: dropout=%r is not supported (eval mode only: dropout must be 0)' % (dropout,))
    if out_ch != 3:
        raise NotImplementedError('VQGAN Decoder: out_ch=%d is not supported (3 only)' % out_ch)
    if not 1 <= len(ch_mult) <= 8:
        raise NotImplementedError('VQGAN Decoder: %d levels are not supported (1 to 8)' % len(ch_mult))
    widths = [ch * m for m in ch_mult]
    for c in widths + [z_channels]:
        if c <= 0 or c % 64 or c > 2048:
            raise NotImplementedError('VQGAN Decoder: channel count %d is not supported (multiples of 64 up to 2048)' % c)
    attn = set(_attn_levels(ch_mult, resolution, attn_resolutions))
    gemm = {widths[-1]} | {widths[i] for i in attn}
    gemm |= {c for i in range(len(widths) - 1) if widths[i] != widths[i + 1] for c in (widths[i], widths[i + 1])}
    for c in sorted(gemm):
        if c % 128:
            raise NotImplementedError('VQGAN Decoder: width %d runs a nin_shortcut or attention, which need a multiple of 128' % c)


class Decoder(nn.Module):
    """taming's Decoder (temb_ch = 0), eval mode. forward(z [N, z_channels, h, w]) -> [N, 3, h 2^(L-1), w 2^(L-1)] fp32 on the
    GPU; its backward gives d loss / d z only (the weights are constants). h w is at most MAX_TOKENS (the attention's ceiling)."""

    def __init__(self, *, ch, out_ch, ch_mult=(1, 2, 4, 8), num_res_blocks, attn_resolutions, dropout=0.0, resamp_with_conv=True,
                 in_channels=3, resolution, z_channels, give_pre_end=False, **ignorekwargs):
        super().__init__()
        check_config(ch, out_ch, ch_mult, num_res_blocks, attn_resolutions, dropout, resamp_with_conv, resolution, z_channels, give_pre_end)
        self.ch, self.temb_ch, self.num_resolutions, self.num_res_blocks = ch, 0, len(ch_mult), num_res_blocks
        self.resolution, self.in_channels, self.give_pre_end, self.z_channels = resolution, in_channels, give_pre_end, z_channels
        self.ch_mult = tuple(ch_mult)
        self.attn_levels = _attn_levels(ch_mult, resolution, attn_resolutions)
        block_in = ch * ch_mult[-1]
        curr_res = resolution // 2 ** (self.num_resolutions - 1)
        self.z_shape = (1, z_channels, curr_res, curr_res)
        self.conv_in = nn.Conv2d(z_channels, block_in, 3, 1, 1)
        self.mid = nn.Module()
        self.mid.block_1, self.mid.attn_1, self.mid.block_2 = ResnetBlock(block_in, block_in), AttnBlock(block_in), ResnetBlock(block_in, block_in)
        self.up = nn.ModuleList()
        for i_level in reversed(range(self.num_resolutions)):
            block, attn = nn.ModuleList(), nn.ModuleList()
            block_out = ch * ch_mult[i_level]
            for _ in range(num_res_blocks + 1):
                block.append(ResnetBlock(block_in, block_out))
                block_in = block_out
                if curr_res in attn_resolutions:
                    attn.append(AttnBlock(block_in))
            up = nn.Module()
            up.block, up.attn = block, attn
            if i_level != 0:
                up.upsample = Upsample(block_in)
                curr_res *= 2
            self.up.insert(0, up)
        self.norm_out = _norm(block_in)
        self.conv_out = nn.Conv2d(block_in, out_ch, 3, 1, 1)
        self._handle, self._max = None, (0, 0)
        self._packed = None
        self._generation, self._handle_epoch, self.recomputes = 0, 0, 0      # see _Decode

    def __getstate__(self):
        state = self.__dict__.copy()
        state['_handle'], state['_max'], state['_packed'] = None, (0, 0), None
        return state

    def _signature(self):
        return tuple((p.data_ptr(), p._version) for p in self.parameters())

    def _ensure(self, n, tokens):
        """(Re)creates the handle when the call needs a larger arena, and (re)packs the weights when a parameter changed."""
        if self._handle is None or n > self._max[0] or tokens > self._max[1]:
            if self._handle is not None:
                self._handle.close()
            self._handle, self._packed = None, None
            n, tokens = max(n, self._max[0]), max(tokens, self._max[1])
            mult = (C.c_int32 * 8)(*self.ch_mult)
            mask = sum(1 << i for i in self.attn_levels)
            cfg = VqganConfig(self.z_channels, self.ch, mult, self.num_resolutions, self.num_res_blocks, mask, 3, int(n), int(tokens))
            self._handle = Handle('aph_vqgan', C.byref(cfg))
            self._max = (int(n), int(tokens))
            self._handle_epoch += 1
        sig = self._signature()
        if sig != self._packed:
            with torch.no_grad():
                self._handle.load(pack_state_dict(self.state_dict()))
            self._packed = sig
            self._handle_epoch += 1

    def _fwd(self, zi, out, save):
        n, _, h, w = zi.shape
        check(lib().aph_vqgan_fwd(self._handle, zi.data_ptr(), n, h, w, out.data_ptr(), int(save), stream_ptr()), 'aph_vqgan_fwd')

    def forward(self, z):
        if not isinstance(z, torch.Tensor) or z.dim() != 4 or z.shape[1] != self.z_channels:
            raise ValueError('VQGAN Decoder: expected z [N, %d, h, w], got %s' % (self.z_channels, tuple(z.shape)))
        for i in self.attn_levels + [self.num_resolutions - 1]:
            t = z.shape[2] * z.shape[3] * 4 ** (self.num_resolutions - 1 - i)
            if t > MAX_TOKENS:
                raise ValueError('VQGAN Decoder: the attention at %d x %d would run over %d tokens, above the limit of %d '
                                 '(its T x T scores are materialised)' % (z.shape[2] << (self.num_resolutions - 1 - i),
                                                                          z.shape[3] << (self.num_resolutions - 1 - i), t, MAX_TOKENS))
        require_cuda(z, 'VQGAN Decoder input')
        return _Decode.apply(z, self)


class _Decode(torch.autograd.Function):
    @staticmethod
    def forward(ctx, z, dec):
        zi = z.detach().contiguous().float()
        n, _, h, w = zi.shape
        dec._ensure(n, h * w)
        f = 2 ** (dec.num_resolutions - 1)
        out = torch.empty(n, 3, h * f, w * f, device=zi.device, dtype=torch.float32)
        need_bwd = z.requires_grad
        dec._fwd(zi, out, need_bwd)
        # The handle owns ONE activation arena, and every forward overwrites it (a no_grad forward too: the notebook's checkout).
        # Each forward gets a generation stamp; a backward whose stamp is stale re-runs its forward from the saved input first
        # (deterministic kernels: identical activations), as _EncodeImage does.
        dec._generation += 1
        ctx.dec, ctx.shape = dec, tuple(zi.shape)
        if need_bwd:
            ctx.generation, ctx.handle_epoch = dec._generation, dec._handle_epoch
            ctx.save_for_backward(zi)
        return out

    @staticmethod
    def backward(ctx, g):
        dec = ctx.dec
        zi, = ctx.saved_tensors
        g = g.contiguous().float()
        n, _, h, w = ctx.shape
        if ctx.generation != dec._generation or ctx.handle_epoch != dec._handle_epoch:
            dec._ensure(n, h * w)
            dec._fwd(zi, torch.empty_like(g), True)
            dec._generation += 1
            dec.recomputes += 1
        dz = torch.empty(ctx.shape, device=g.device, dtype=torch.float32)
        check(lib().aph_vqgan_bwd(dec._handle, g.data_ptr(), n, h, w, dz.data_ptr(), stream_ptr()), 'aph_vqgan_bwd')
        return dz, None


def pack_state_dict(sd):
    """taming's decoder keys (without "decoder.") -> the handle's: each AttnBlock's q, k, v stacked into "<p>.qkv.weight" [3C, C]
    and "<p>.qkv.bias", the 1x1 kernels (nin_shortcut, proj_out) flattened to [C_out, C_in]; fp32, contiguous."""
    out = OrderedDict()
    for k, v in sd.items():
        v = v.detach().float()
        p, _, leaf = k.rpartition('.')
        mod = p.rpartition('.')[2]
        if mod in ('q', 'k', 'v'):
            if mod == 'q':
                base = p[:-2]
                parts = [sd['%s.%s.%s' % (base, m, leaf)].detach().float() for m in ('q', 'k', 'v')]
                t = torch.cat(parts, 0)
                out['%s.qkv.%s' % (base, leaf)] = (t.reshape(t.shape[0], -1) if leaf == 'weight' else t).contiguous()
            continue
        if mod in ('nin_shortcut', 'proj_out') and leaf == 'weight':
            v = v.reshape(v.shape[0], -1)
        out[k] = v.contiguous()
    return out


def synthetic_decoder_state_dict(seed=0, **ddconfig):
    """A decoder state dict in taming's key layout whose weights exercise the kernels: GroupNorm affines away from (1, 0),
    residual branches scaled so that the stream stays of order one, and q / k scaled so that the softmax is neither uniform
    nor one-hot (logits of standard deviation about 2 on normalised input)."""
    g = torch.Generator().manual_seed(seed)
    skel = Decoder(**ddconfig)
    sd = OrderedDict()
    for k, v in skel.state_dict().items():
        uni = lambda a: (torch.rand(v.shape, generator=g, dtype=torch.float64) * 2 - 1) * a
        gauss = lambda s: torch.randn(v.shape, generator=g, dtype=torch.float64) * s
        name = k.rsplit('.', 2)
        leaf, mod = name[-1], name[-2]
        if mod.startswith('norm'):
            t = 1 + uni(0.3) if leaf == 'weight' else uni(0.3)
        elif leaf == 'bias':
            t = uni(0.05)
        else:
            fan_in = v[0].numel()
            s = fan_in ** -0.5
            if mod in ('q', 'k'):
                s *= 1.4
            elif mod in ('conv2', 'proj_out'):
                s *= 0.3                  # the residual branches
            t = gauss(s)
        sd[k] = t.float()
    return sd
