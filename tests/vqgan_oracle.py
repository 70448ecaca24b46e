"""Float64 restatement of taming's Decoder (taming.modules.diffusionmodules.model, temb_ch = 0, eval mode) in torch.nn.functional,
from a state dict in taming's key layout. taming itself is not installed here, so parity with taming is unpinned: this follows
its forward as written (ResnetBlock, AttnBlock, nearest x2 + conv Upsample, GroupNorm(32, eps 1e-6), swish = x sigmoid(x))."""
import torch
import torch.nn.functional as F


def _gn(sd, p, x):
    return F.group_norm(x, 32, sd[p + '.weight'], sd[p + '.bias'], eps=1e-6)


def _conv(sd, p, x):
    w = sd[p + '.weight']
    return F.conv2d(x, w, sd[p + '.bias'], padding=w.shape[-1] // 2)


def _swish(x):
    return x * torch.sigmoid(x)


def resnet_block(sd, p, x):
    h = _conv(sd, p + '.conv1', _swish(_gn(sd, p + '.norm1', x)))
    h = _conv(sd, p + '.conv2', _swish(_gn(sd, p + '.norm2', h)))
    if p + '.nin_shortcut.weight' in sd:
        x = _conv(sd, p + '.nin_shortcut', x)
    return x + h


def attention(q, k, v):
    """q, k, v [b, c, t] -> [b, c, t]: softmax(q^T k c^-1/2) over the keys, applied to v"""
    c = q.shape[1]
    w = torch.softmax(torch.bmm(q.permute(0, 2, 1), k) * c ** -0.5, dim=2)
    return torch.bmm(v, w.permute(0, 2, 1))


def attn_block(sd, p, x):
    h = _gn(sd, p + '.norm', x)
    b, c, hh, ww = h.shape
    q, k, v = (_conv(sd, '%s.%s' % (p, m), h).reshape(b, c, hh * ww) for m in ('q', 'k', 'v'))
    return x + _conv(sd, p + '.proj_out', attention(q, k, v).reshape(b, c, hh, ww))


def decode(sd, z, ch_mult, num_res_blocks, attn_levels):
    """z [N, z_channels, h, w] -> [N, 3, h 2^(L-1), w 2^(L-1)], in the dtype and on the device of z (float64 for the oracle)"""
    sd = {k: v.to(z) for k, v in sd.items()}
    h = _conv(sd, 'conv_in', z)
    h = resnet_block(sd, 'mid.block_1', h)
    h = attn_block(sd, 'mid.attn_1', h)
    h = resnet_block(sd, 'mid.block_2', h)
    for i in reversed(range(len(ch_mult))):
        for j in range(num_res_blocks + 1):
            h = resnet_block(sd, 'up.%d.block.%d' % (i, j), h)
            if i in attn_levels:
                h = attn_block(sd, 'up.%d.attn.%d' % (i, j), h)
        if i != 0:
            h = _conv(sd, 'up.%d.upsample.conv' % i, F.interpolate(h, scale_factor=2.0, mode='nearest'))
    return _conv(sd, 'conv_out', _swish(_gn(sd, 'norm_out', h)))
