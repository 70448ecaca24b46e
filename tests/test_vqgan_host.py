"""The VQGAN decoder's host side (no GPU): taming's parameter names and shapes for the notebook's two decoders, loading a
taming-layout checkpoint through a stand-in for the notebook's VQModel, the handle's key packing, every refusal and the
attention's token ceiling, and the `taming` drop-in."""
import os
import sys

import pytest
import torch
import torch.nn as nn

from aphantasia_b200 import vqgan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _expected_shapes(cfg):
    """taming's Decoder parameters, written out from its constructor"""
    ch, mult, nrb, zc = cfg['ch'], cfg['ch_mult'], cfg['num_res_blocks'], cfg['z_channels']
    L = len(mult)
    out = {}

    def conv(p, co, ci, k):
        out[p + '.weight'], out[p + '.bias'] = (co, ci, k, k), (co,)

    def norm(p, c):
        out[p + '.weight'], out[p + '.bias'] = (c,), (c,)

    def res(p, ci, co):
        norm(p + '.norm1', ci); conv(p + '.conv1', co, ci, 3); norm(p + '.norm2', co); conv(p + '.conv2', co, co, 3)
        if ci != co:
            conv(p + '.nin_shortcut', co, ci, 1)

    def attn(p, c):
        norm(p + '.norm', c)
        for m in ('q', 'k', 'v', 'proj_out'):
            conv('%s.%s' % (p, m), c, c, 1)

    bi = ch * mult[-1]
    res_ = cfg['resolution'] // 2 ** (L - 1)
    conv('conv_in', bi, zc, 3)
    res('mid.block_1', bi, bi); attn('mid.attn_1', bi); res('mid.block_2', bi, bi)
    for i in reversed(range(L)):
        bo = ch * mult[i]
        for j in range(nrb + 1):
            res('up.%d.block.%d' % (i, j), bi, bo)
            bi = bo
            if res_ in cfg['attn_resolutions']:
                attn('up.%d.attn.%d' % (i, j), bi)
        if i:
            conv('up.%d.upsample.conv' % i, bi, bi, 3)
            res_ *= 2
    norm('norm_out', bi); conv('conv_out', 3, bi, 3)
    return out


@pytest.mark.parametrize('name', ['F16_CONFIG', 'F8_CONFIG'])
def test_parameter_names_and_shapes_are_tamings(name):
    cfg = getattr(vqgan, name)
    dec = vqgan.Decoder(**cfg)
    got = {k: tuple(v.shape) for k, v in dec.state_dict().items()}
    assert got == _expected_shapes(cfg)
    assert 'up.%d.block.0.nin_shortcut.weight' % (len(cfg['ch_mult']) - 2) in got
    attn_level = len(cfg['ch_mult']) - 1
    assert dec.attn_levels == [attn_level]
    assert got['up.%d.attn.2.q.weight' % attn_level] == (512, 512, 1, 1)
    assert got['conv_out.weight'] == (3, 128, 3, 3) and got['conv_in.weight'] == (512, 256, 3, 3)


class _VQModel(nn.Module):
    """the notebook's VQModel as far as the decoder's step goes: decoder, quantize, quant_conv, post_quant_conv (the encoder's
    checkpoint keys are left over, as are the quantizer's)"""
    def __init__(self, ddconfig, n_embed, embed_dim, gumbel):
        super().__init__()
        from taming.modules.diffusionmodules.model import Decoder
        from taming.modules.vqvae.quantize import GumbelQuantize, VectorQuantizer2
        self.decoder = Decoder(**ddconfig)
        self.quantize = (GumbelQuantize(ddconfig['z_channels'], embed_dim, n_embed=n_embed) if gumbel
                         else VectorQuantizer2(n_embed, embed_dim, beta=0.25))
        self.quant_conv = nn.Conv2d(ddconfig['z_channels'], embed_dim, 1)
        self.post_quant_conv = nn.Conv2d(embed_dim, ddconfig['z_channels'], 1)


@pytest.fixture
def taming():
    sys.path.insert(0, os.path.join(ROOT, 'dropin'))
    try:
        yield
    finally:
        sys.path.remove(os.path.join(ROOT, 'dropin'))
        for k in [k for k in sys.modules if k == 'taming' or k.startswith('taming.')]:
            del sys.modules[k]


@pytest.mark.parametrize('name,gumbel', [('F16_CONFIG', False), ('F8_CONFIG', True)])
def test_a_taming_checkpoint_loads_with_strict_false(taming, name, gumbel):
    cfg = getattr(vqgan, name)
    dec_sd = vqgan.synthetic_decoder_state_dict(3, **cfg)
    ckpt = {'decoder.' + k: v for k, v in dec_sd.items()}
    ckpt.update({'encoder.conv_in.weight': torch.zeros(128, 3, 3, 3), 'quantize.embedding.weight': torch.zeros(1024, 256),
                 'quantize.proj.weight': torch.zeros(8192, 256, 1, 1), 'post_quant_conv.weight': torch.ones(256, 256, 1, 1),
                 'post_quant_conv.bias': torch.zeros(256)})
    model = _VQModel(cfg, 1024, 256, gumbel).eval()
    missing, unexpected = model.load_state_dict(ckpt, strict=False)
    assert not [k for k in missing if k.startswith('decoder.')]
    assert set(unexpected) >= {'quantize.embedding.weight', 'quantize.proj.weight', 'encoder.conv_in.weight'}
    for k, v in dec_sd.items():
        assert torch.equal(model.decoder.state_dict()[k], v), k
    assert list(model.quantize.parameters()) == []
    with pytest.raises(NotImplementedError, match='stand-in'):
        model.quantize(torch.zeros(1, 256, 2, 2))


def test_pack_stacks_qkv_and_flattens_the_1x1_kernels():
    sd = vqgan.synthetic_decoder_state_dict(1, **vqgan.F8_CONFIG)
    packed = vqgan.pack_state_dict(sd)
    p = 'mid.attn_1'
    assert torch.equal(packed[p + '.qkv.weight'], torch.cat([sd[p + '.q.weight'], sd[p + '.k.weight'], sd[p + '.v.weight']]).reshape(1536, 512))
    assert torch.equal(packed[p + '.qkv.bias'], torch.cat([sd[p + '.q.bias'], sd[p + '.k.bias'], sd[p + '.v.bias']]))
    assert packed[p + '.proj_out.weight'].shape == (512, 512)
    assert packed['up.2.block.0.nin_shortcut.weight'].shape == (256, 512)
    assert not [k for k in packed if k.endswith(('.q.weight', '.k.bias', '.v.weight'))]
    assert sum(v.numel() for v in packed.values()) == sum(v.numel() for v in sd.values())


def test_synthetic_weights_exercise_the_kernels():
    sd = vqgan.synthetic_decoder_state_dict(0, **vqgan.F16_CONFIG)
    g = sd['mid.block_1.norm1.weight']
    assert 0.05 < float((g - 1).abs().mean()) and 0.05 < float(sd['mid.block_1.norm1.bias'].abs().mean())
    assert sd['mid.block_1.conv2.weight'].std() < 0.5 * sd['mid.block_1.conv1.weight'].std()
    assert sd['mid.attn_1.q.weight'].std() > sd['mid.attn_1.v.weight'].std()
    assert all(torch.equal(a, b) for a, b in zip(sd.values(), vqgan.synthetic_decoder_state_dict(0, **vqgan.F16_CONFIG).values()))


@pytest.mark.parametrize('change,match', [
    (dict(give_pre_end=True), 'give_pre_end'),
    (dict(resamp_with_conv=False), 'resamp_with_conv'),
    (dict(dropout=0.1), 'dropout'),
    (dict(out_ch=4), 'out_ch'),
    (dict(ch=96), 'multiples of 64'),
    (dict(z_channels=200), 'multiples of 64'),
    (dict(ch=64, ch_mult=(1, 3)), 'multiple of 128'),
    (dict(ch=64, ch_mult=(1, 1)), 'multiple of 128'),
    (dict(ch_mult=(1,) * 9), 'levels'),
])
def test_unsupported_configs_are_refused(change, match):
    cfg = dict(vqgan.F8_CONFIG, **change)
    with pytest.raises(NotImplementedError, match=match):
        vqgan.Decoder(**cfg)


def test_the_attention_token_ceiling():
    dec = vqgan.Decoder(**vqgan.F8_CONFIG)
    assert vqgan.MAX_TOKENS == 16384
    hdr = open(os.path.join(ROOT, 'include', 'aphb200.h')).read()
    assert '#define APH_VQGAN_MAX_TOKENS 16384' in hdr
    with pytest.raises(ValueError, match='16384'):
        dec(torch.zeros(1, 256, 128, 129))
    with pytest.raises(ValueError, match='z \\[N, 256, h, w\\]'):
        dec(torch.zeros(1, 3, 8, 8))
    if not torch.cuda.is_available():          # at the ceiling the shape passes, and the CPU tensor is refused next
        with pytest.raises(RuntimeError, match='no CPU path'):
            dec(torch.zeros(1, 256, 128, 128))
