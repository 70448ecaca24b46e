"""Drop-in for the OpenAI `clip` package as used by /root/reference/clip_fft.py (:19,119,121,133,150,216,254):
`clip.load(name, jit=False) -> (model, preprocess)`, `clip.tokenize`, `model.encode_image`, `model.encode_text`,
`model.visual.input_resolution`.

The image encoder (ViT-B/32, ViT-B/16, ViT-L/14) runs forward and data-gradient in libaphb200.so (csrc/vit.cu: wgmma
GEMMs + fused kernels); the ResNet encoders RN50, RN101, RN50x4, RN50x16 and RN50x64 in csrc/rn.cu (the same GEMM and 3x3
convolution, BatchNorm folded on the host). Weights: an OpenAI state dict if `APH_CLIP_WEIGHTS_<NAME>=<file.pt>` or
`APH_CLIP_WEIGHTS=<file.pt>` is set (a TorchScript archive as OpenAI ships them, or a plain state dict), else seeded synthetic
weights of the same architecture. RN50x4, RN50x16 and RN50x64 have no synthetic fallback: they need a checkpoint.
The text encoder (csrc/text.cu, forward only) runs once per prompt before the optimisation loop when the weights hold
the text tower; `tokenize` uses CLIP's BPE vocabulary from `APH_CLIP_BPE=<bpe_simple_vocab_16e6.txt.gz>` or from that
file next to the weights. Without text weights `encode_text` returns a deterministic seeded embedding per prompt, and
without a vocabulary `tokenize` encodes the prompt's UTF-8 bytes (both loudly).
"""
import ctypes as C
import hashlib
import os
import zipfile
from collections import OrderedDict

import torch

from .. import _patchlink, _pool, _trace
from .._lib import Handle, RnConfig, TextConfig, VitConfig, check, lib, require_cuda, stream_ptr
from ._bpe import SimpleTokenizer

_MODELS = {'ViT-B/32': dict(patch=32, width=768, layers=12, heads=12, out_dim=512, res=224),
           'ViT-B/16': dict(patch=16, width=768, layers=12, heads=12, out_dim=512, res=224),
           'ViT-L/14': dict(patch=14, width=1024, layers=24, heads=16, out_dim=768, res=224),
           'RN50': dict(layers=(3, 4, 6, 3), width=64, heads=32, out_dim=1024, res=224),
           'RN101': dict(layers=(3, 4, 23, 3), width=64, heads=32, out_dim=512, res=224),
           'RN50x4': dict(layers=(4, 6, 10, 6), width=80, heads=40, out_dim=640, res=288),
           'RN50x16': dict(layers=(6, 8, 18, 8), width=96, heads=48, out_dim=768, res=384),
           'RN50x64': dict(layers=(3, 15, 36, 10), width=128, heads=64, out_dim=1024, res=448)}
# The wide ResNets load from an OpenAI checkpoint only: no benchmark or script default needs them without one, and a synthetic
# RN50x64 alone is 420 M parameters to draw.
CHECKPOINT_ONLY = ('RN50x4', 'RN50x16', 'RN50x64')
RN_SIDES = (223, 254)      # the crop sides whose ResNet map is 7 x 7 at the attention pool (RN50, RN101: resolution 224)


def rn_sides(res):
    """The crop sides a ResNet of input resolution `res` takes: those whose final map is res/32 x res/32."""
    return res - 1, res + 30


def weights_variable(name):
    """The environment variable that names `name`'s checkpoint (APH_CLIP_WEIGHTS serves every model)."""
    return 'APH_CLIP_WEIGHTS_' + name.replace('/', '').replace('-', '').upper()


def available_models():
    return list(_MODELS)


def synthetic_visual_state_dict(patch=32, width=768, layers=12, heads=12, out_dim=512, res=224, seed=0):
    """Seeded synthetic weights in the OpenAI key layout, PyTorch-default-style init (private generator:
    the global RNG stream the sampler replays is left untouched)."""
    g = torch.Generator().manual_seed(seed)
    T = (res // patch) ** 2 + 1

    def uni(shape, bound):
        return (torch.rand(shape, generator=g) * 2 - 1) * bound

    def nrm(shape, std):
        return torch.randn(shape, generator=g) * std
    sd = OrderedDict()
    sd['visual.class_embedding'] = nrm((width,), width ** -0.5)
    sd['visual.positional_embedding'] = nrm((T, width), width ** -0.5)
    sd['visual.proj'] = nrm((width, out_dim), width ** -0.5)
    sd['visual.conv1.weight'] = uni((width, 3, patch, patch), (3 * patch * patch) ** -0.5)
    for n in ('ln_pre', 'ln_post'):
        sd['visual.%s.weight' % n] = torch.ones(width); sd['visual.%s.bias' % n] = torch.zeros(width)
    for i in range(layers):
        p = 'visual.transformer.resblocks.%d.' % i
        sd[p + 'attn.in_proj_weight'] = uni((3 * width, width), (6. / (4 * width)) ** 0.5)
        sd[p + 'attn.in_proj_bias'] = torch.zeros(3 * width)
        sd[p + 'attn.out_proj.weight'] = uni((width, width), width ** -0.5)
        sd[p + 'attn.out_proj.bias'] = torch.zeros(width)
        sd[p + 'ln_1.weight'] = torch.ones(width); sd[p + 'ln_1.bias'] = torch.zeros(width)
        sd[p + 'mlp.c_fc.weight'] = uni((4 * width, width), width ** -0.5)
        sd[p + 'mlp.c_fc.bias'] = uni((4 * width,), width ** -0.5)
        sd[p + 'mlp.c_proj.weight'] = uni((width, 4 * width), (4 * width) ** -0.5)
        sd[p + 'mlp.c_proj.bias'] = uni((width,), (4 * width) ** -0.5)
        sd[p + 'ln_2.weight'] = torch.ones(width); sd[p + 'ln_2.bias'] = torch.zeros(width)
    return sd


def synthetic_resnet_state_dict(layers=(3, 4, 6, 3), width=64, heads=32, out_dim=1024, res=224, seed=0, branch_scale=0.25):
    """Seeded synthetic ModifiedResNet weights in the OpenAI key layout ("visual." prefix). Convolutions have He-normal weights
    and every BatchNorm non-trivial running statistics and affine (so that a missing or wrong fold shows); the last BatchNorm of
    each residual branch is scaled by `branch_scale`: 0.25 keeps the residual stream of order one through 33 blocks, deeper
    towers need less."""
    g = torch.Generator().manual_seed(seed)
    embed = width * 32

    def uni(shape, bound):
        return (torch.rand(shape, generator=g) * 2 - 1) * bound

    def conv(co, ci, k):
        return torch.randn((co, ci, k, k), generator=g) * (2. / (ci * k * k)) ** 0.5

    sd = OrderedDict()

    def bn(p, c, scale=1.):
        sd[p + '.weight'] = scale * (1 + uni((c,), 0.2))
        sd[p + '.bias'] = uni((c,), 0.1)
        sd[p + '.running_mean'] = uni((c,), 0.2)
        sd[p + '.running_var'] = 1 + uni((c,), 0.5)
        sd[p + '.num_batches_tracked'] = torch.tensor(0)
    v = 'visual.'
    for i, (ci, co) in enumerate(((3, width // 2), (width // 2, width // 2), (width // 2, width))):
        sd[v + 'conv%d.weight' % (i + 1)] = conv(co, ci, 3)
        bn(v + 'bn%d' % (i + 1), co)
    cin = width
    for i, n in enumerate(layers):
        planes = width << i
        for j in range(n):
            p = v + 'layer%d.%d.' % (i + 1, j)
            sd[p + 'conv1.weight'] = conv(planes, cin, 1); bn(p + 'bn1', planes)
            sd[p + 'conv2.weight'] = conv(planes, planes, 3); bn(p + 'bn2', planes)
            sd[p + 'conv3.weight'] = conv(4 * planes, planes, 1); bn(p + 'bn3', 4 * planes, branch_scale)
            if j == 0 and (i > 0 or cin != 4 * planes):
                sd[p + 'downsample.0.weight'] = conv(4 * planes, cin, 1); bn(p + 'downsample.1', 4 * planes)
            cin = 4 * planes
    a = v + 'attnpool.'
    sd[a + 'positional_embedding'] = torch.randn(((res // 32) ** 2 + 1, embed), generator=g) / embed ** 0.5
    for n in ('q_proj', 'k_proj', 'v_proj'):
        sd[a + n + '.weight'] = torch.randn((embed, embed), generator=g) * embed ** -0.5
        sd[a + n + '.bias'] = uni((embed,), 0.02)
    sd[a + 'c_proj.weight'] = torch.randn((out_dim, embed), generator=g) * embed ** -0.5
    sd[a + 'c_proj.bias'] = uni((out_dim,), 0.02)
    return sd


def pad64(c):
    """The channel count the ResNet tower runs a layer of c channels at: c rounded up to a multiple of 64."""
    return (c + 63) // 64 * 64


def fold_resnet_state_dict(sd, eps=1e-5, dtype=torch.float64):
    """The ResNet tower's device tensors from a ModifiedResNet state dict without the "visual." prefix: every BatchNorm (running
    statistics, eps) folded into the convolution before it, w' = w g / sqrt(var + eps), b' = b - mean g / sqrt(var + eps), in
    float64; every convolution but the stem's first zero-padded to pad64 output and input channels, with zero biases in the
    padding (RN50's stem 32 -> 64; RN50x4's 40 -> 64, 80 -> 128 and planes 80 -> 128, 160 -> 192; RN50x16's 48 -> 64,
    96 -> 128 and planes 96 -> 128), so that the padded channels stay exactly 0 through bias, ReLU, residual and pools; 1x1
    weights as [C_out, C_in]; the attention pool's q, k and v projections stacked into one [3 D, D] operand in that order. Each
    tensor is converted to `dtype` before the next one is folded, so the float64 working set is one tensor (RN50x64 holds 420 M
    visual parameters). Keys: see aph_rn_load_tensor."""
    out = OrderedDict()

    def fold(conv, bn):
        s = sd[bn + '.weight'].double() / torch.sqrt(sd[bn + '.running_var'].double() + eps)
        w = sd[conv].double() * s.view(-1, 1, 1, 1)
        return w, sd[bn + '.bias'].double() - sd[bn + '.running_mean'].double() * s

    def put(key, w, bias):
        co, ci = w.shape[:2]
        if (pad64(co), pad64(ci)) != (co, ci):
            wp = torch.zeros((pad64(co), pad64(ci)) + tuple(w.shape[2:]), dtype=torch.float64)
            wp[:co, :ci] = w
            bp = torch.zeros(pad64(co), dtype=torch.float64)
            bp[:co] = bias
            w, bias = wp, bp
        out[key + '.weight'] = (w if w.shape[-1] == 3 else w.flatten(1)).to(dtype)
        out[key + '.bias'] = bias.to(dtype)
    w1, b1 = fold('conv1.weight', 'bn1')
    out['conv1.weight'], out['conv1.bias'] = w1.to(dtype), b1.to(dtype)
    put('conv2', *fold('conv2.weight', 'bn2'))
    put('conv3', *fold('conv3.weight', 'bn3'))
    blocks = sorted({k.rsplit('.', 2)[0] for k in sd if k.startswith('layer') and k.endswith('.conv1.weight')},
                    key=lambda b: tuple(int(t) for t in b[len('layer'):].split('.')))
    for b in blocks:
        for n in ('conv1', 'conv2', 'conv3'):
            put('%s.%s' % (b, n), *fold('%s.%s.weight' % (b, n), '%s.bn%s' % (b, n[-1])))
        if b + '.downsample.0.weight' in sd:
            put(b + '.downsample', *fold(b + '.downsample.0.weight', b + '.downsample.1'))
    a = 'attnpool.'
    out[a + 'positional_embedding'] = sd[a + 'positional_embedding'].double().to(dtype)
    out[a + 'qkv.weight'] = torch.cat([sd[a + n + '_proj.weight'].double() for n in 'qkv']).to(dtype)
    out[a + 'qkv.bias'] = torch.cat([sd[a + n + '_proj.bias'].double() for n in 'qkv']).to(dtype)
    out[a + 'c_proj.weight'] = sd[a + 'c_proj.weight'].double().to(dtype)
    out[a + 'c_proj.bias'] = sd[a + 'c_proj.bias'].double().to(dtype)
    return out


def resnet_architecture(state_dict):
    """(layers, width, input resolution) of a ModifiedResNet state dict with the "visual." prefix, read as OpenAI's build_model
    reads them."""
    sd = state_dict
    layers = tuple(len({k.split('.')[2] for k in sd if k.startswith('visual.layer%d.' % i)}) for i in range(1, 5))
    width = sd['visual.layer1.0.conv1.weight'].shape[0]
    res = 32 * round((sd['visual.attnpool.positional_embedding'].shape[0] - 1) ** 0.5)
    return layers, width, res


def is_resnet(state_dict):
    """OpenAI's loader test for a ModifiedResNet image tower."""
    return 'visual.layer1.0.conv1.weight' in state_dict


_TEXT_KEYS = ('token_embedding.weight', 'positional_embedding', 'ln_final.weight', 'ln_final.bias', 'text_projection')


def synthetic_text_state_dict(width=512, layers=12, heads=8, out_dim=512, context=77, vocab=49408, seed=0):
    """Seeded synthetic text-tower weights in the OpenAI key layout (OpenAI's init scales; LayerNorm affines perturbed so that
    a swapped or dropped LayerNorm shows in a comparison)."""
    assert heads * 64 == width, 'the text tower has head dim 64'
    g = torch.Generator().manual_seed(seed)

    def uni(shape, bound):
        return (torch.rand(shape, generator=g) * 2 - 1) * bound

    def nrm(shape, std):
        return torch.randn(shape, generator=g) * std
    sd = OrderedDict()
    sd['token_embedding.weight'] = nrm((vocab, width), 0.02)
    sd['positional_embedding'] = nrm((context, width), 0.01)
    sd['text_projection'] = nrm((width, out_dim), width ** -0.5)
    sd['ln_final.weight'] = 1 + uni((width,), 0.1); sd['ln_final.bias'] = uni((width,), 0.1)
    for i in range(layers):
        p = 'transformer.resblocks.%d.' % i
        sd[p + 'attn.in_proj_weight'] = uni((3 * width, width), (6. / (4 * width)) ** 0.5)
        sd[p + 'attn.in_proj_bias'] = uni((3 * width,), 0.02)
        sd[p + 'attn.out_proj.weight'] = uni((width, width), width ** -0.5)
        sd[p + 'attn.out_proj.bias'] = uni((width,), 0.02)
        sd[p + 'ln_1.weight'] = 1 + uni((width,), 0.1); sd[p + 'ln_1.bias'] = uni((width,), 0.1)
        sd[p + 'mlp.c_fc.weight'] = uni((4 * width, width), width ** -0.5)
        sd[p + 'mlp.c_fc.bias'] = uni((4 * width,), width ** -0.5)
        sd[p + 'mlp.c_proj.weight'] = uni((width, 4 * width), (4 * width) ** -0.5)
        sd[p + 'mlp.c_proj.bias'] = uni((width,), (4 * width) ** -0.5)
        sd[p + 'ln_2.weight'] = 1 + uni((width,), 0.1); sd[p + 'ln_2.bias'] = uni((width,), 0.1)
    return sd


def has_text_tower(state_dict):
    return all(k in state_dict for k in _TEXT_KEYS) and 'transformer.resblocks.0.attn.in_proj_weight' in state_dict


class _Tower:
    """A tower's device handle (a `Handle` of `_api`), loaded from `self._sd` for batches of up to max_batch samples. It is
    owned from its creation on: when a load or the finalize fails, close() still frees it."""
    _api, _prefix = None, ''
    handle, max_batch = None, 0

    def _build(self, cfg, max_batch):
        self.close()
        self.handle = Handle(self._api, C.byref(cfg))
        self.handle.load(self._sd, self._prefix)
        self.max_batch = int(max_batch)

    def close(self):
        if self.handle is not None:
            self.handle.close()
        self.handle, self.max_batch = None, 0


class TextTransformer(_Tower):
    """Handle-owning forward of clip.model.CLIP's text tower (token embedding -> causal transformer -> ln_final at the
    end-of-text position -> text_projection) through the C ABI. The handle is created on the first call (constructing a
    CLIP needs no GPU) and re-created when a call brings more prompts than it was sized for."""
    _api = 'aph_text'

    def __init__(self, state_dict):
        sd = {k: v for k, v in state_dict.items() if k in _TEXT_KEYS or k.startswith('transformer.resblocks.')}
        self.vocab, self.width = sd['token_embedding.weight'].shape
        self.context = sd['positional_embedding'].shape[0]
        self.layers = len([k for k in sd if k.endswith('.attn.in_proj_weight')])
        self.heads = self.width // 64
        self.output_dim = sd['text_projection'].shape[1]
        self._sd = {k: v.detach().float().contiguous() for k, v in sd.items()}

    def _ensure(self, n):
        if self.handle is not None and n <= self.max_batch:
            return
        self._build(TextConfig(self.width, self.layers, self.heads, self.output_dim, self.context, self.vocab, int(n), 0), n)

    @torch.no_grad()
    def __call__(self, tokens):
        require_cuda(tokens, 'encode_text tokens')
        if tokens.dim() != 2 or tokens.shape[1] != self.context:
            raise ValueError('encode_text: tokens must be [n, %d], got %s' % (self.context, tuple(tokens.shape)))
        t = tokens.detach().to(torch.int64).contiguous()
        lo, hi = (int(v) for v in torch.stack((t.min(), t.max())).cpu())     # one host read per prompt batch, before the loop
        if lo < 0 or hi >= self.vocab:
            raise ValueError('encode_text: token ids must lie in [0, %d), got [%d, %d]' % (self.vocab, lo, hi))
        n = t.shape[0]
        self._ensure(n)
        emb = torch.empty(n, self.output_dim, device=t.device, dtype=torch.float32)
        check(lib().aph_text_fwd(self.handle, t.data_ptr(), n, emb.data_ptr(), stream_ptr()), 'aph_text_fwd')
        return emb


class _EncodeImage(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, vis, prepatched=False):
        require_cuda(x, 'encode_image input')
        xi = x.detach().contiguous().float()
        S = xi.shape[0]
        vis._ensure(S)
        emb = _pool.empty((S, vis.output_dim))
        need_bwd = x.requires_grad
        if prepatched:       # the sampler already wrote this batch as the conv1 operand (_patchlink): no k_patchify
            check(lib().aph_vit_fwd_prepatched(vis.handle, S, emb.data_ptr(), int(need_bwd), stream_ptr()), 'aph_vit_fwd_prepatched')
            vis.prepatched_forwards += 1
        else:
            vis._patch_gen += 1                 # k_patchify overwrites the operand buffer: outstanding stamps are void
            vis._fwd(xi, S, emb, int(need_bwd))
        _trace.encode()
        ctx.vis, ctx.S, ctx.shape = vis, S, tuple(xi.shape)
        if need_bwd:
            # The handle owns ONE activation arena: a later grad-tracked forward of the same model overwrites what this call
            # saved (clip_fft.py --enforce runs encode_image twice before loss.backward(), :254 and :276). Each saving forward
            # gets a generation stamp; a backward whose stamp is stale re-runs its forward from the saved input first
            # (deterministic kernels: identical activations), instead of silently using the other call's activations.
            vis._generation += 1
            ctx.generation = vis._generation
            ctx.handle_epoch = vis._handle_epoch
            ctx.save_for_backward(xi)
        return emb

    @staticmethod
    def backward(ctx, g):
        vis = ctx.vis
        xi, = ctx.saved_tensors
        g = g.contiguous().float()
        if ctx.generation != vis._generation or ctx.handle_epoch != vis._handle_epoch:
            vis._ensure(ctx.S)
            scratch = torch.empty(ctx.S, vis.output_dim, device=g.device, dtype=torch.float32)
            vis._patch_gen += 1
            vis._fwd(xi, ctx.S, scratch, 1)
            vis._generation += 1            # the arena now belongs to this call; any other pending backward must recompute too
            vis.recomputes += 1
        gi = _pool.empty(ctx.shape)
        vis._bwd(g, ctx.S, ctx.shape[-1], gi)
        return gi, None, None


class VisionTransformer(_Tower):
    """Handle-owning mirror of clip.model.VisionTransformer (forward only through the C ABI)."""
    _api, _prefix = 'aph_vit', 'visual.'

    def __init__(self, state_dict, max_batch=None):
        sd = {k[len('visual.'):]: v for k, v in state_dict.items() if k.startswith('visual.')}
        self.width = sd['conv1.weight'].shape[0]
        self.patch_size = sd['conv1.weight'].shape[-1]
        grid = round((sd['positional_embedding'].shape[0] - 1) ** 0.5)
        self.input_resolution = self.patch_size * grid
        self.layers = len([k for k in sd if k.endswith('.attn.in_proj_weight')])
        self.heads = self.width // 64
        self.output_dim = sd['proj'].shape[1]
        self._sd = {k: v.detach().float().contiguous() for k, v in sd.items()}
        self._generation, self.recomputes, self._handle_epoch = 0, 0, 0        # see _EncodeImage
        self._patch_gen, self.prepatched_forwards = 0, 0      # see _patchlink
        _patchlink.register(self)
        if max_batch:
            self._ensure(max_batch)

    def _ensure(self, S):
        """(Re)creates the device handle so that its activation arena holds S samples."""
        if self.handle is not None and S <= self.max_batch:
            return
        self._build(VitConfig(self.patch_size, self.width, self.layers, self.heads, self.output_dim, self.input_resolution, int(S), 0), S)
        self._handle_epoch += 1

    def _fwd(self, xi, S, emb, save_for_bwd):
        side = xi.shape[-1]
        if side == self.input_resolution:
            check(lib().aph_vit_fwd(self.handle, xi.data_ptr(), S, emb.data_ptr(), save_for_bwd, stream_ptr()), 'aph_vit_fwd')
        else:
            check(lib().aph_vit_fwd_sized(self.handle, xi.data_ptr(), S, side, emb.data_ptr(), save_for_bwd, stream_ptr()),
                  'aph_vit_fwd_sized')

    def _bwd(self, g, S, side, gi):
        if side == self.input_resolution:
            check(lib().aph_vit_bwd(self.handle, g.data_ptr(), S, gi.data_ptr(), stream_ptr()), 'aph_vit_bwd')
        else:
            check(lib().aph_vit_bwd_sized(self.handle, g.data_ptr(), S, side, gi.data_ptr(), stream_ptr()), 'aph_vit_bwd_sized')

    def check_input(self, x):
        """conv1 (kernel = stride = patch, no padding) takes [S,3,side,side] with r <= side < r + patch (r = input_resolution) and
        reads its top-left r x r window: the size + 8 batches of transforms_custom / transforms_elastic. Anything else is refused."""
        r, p = self.input_resolution, self.patch_size
        if x.dim() != 4 or x.shape[1] != 3 or x.shape[2] != x.shape[3] or not r <= x.shape[2] < r + p:
            raise ValueError('encode_image: expected images [S, 3, side, side] with %d <= side < %d, got %s' % (r, r + p, tuple(x.shape)))

    def __call__(self, x):
        require_cuda(x, 'encode_image input')
        self.check_input(x)
        return _EncodeImage.apply(x, self, _patchlink.matches(x, self))


class ModifiedResNet(_Tower):
    """Handle-owning mirror of clip.model.ModifiedResNet (eval mode) through the C ABI, forward and data gradient. It reads the
    whole crop: any side in rn_sides(input_resolution) (RN_SIDES at 224), size + 8 under transforms_custom / _elastic included.
    It has no patch operand, so the sampler never writes one for it (_patchlink)."""
    _api = 'aph_rn'
    patch_size = None
    input_resolution = 224         # set per instance from the weights

    def __init__(self, state_dict, max_batch=None):
        sd = {k[len('visual.'):]: v for k, v in state_dict.items() if k.startswith('visual.')}
        self.layers = tuple(len({k.split('.')[1] for k in sd if k.startswith('layer%d.' % i)}) for i in range(1, 5))
        self.width = sd['conv3.weight'].shape[0]
        self.heads = self.width * 32 // 64
        self.output_dim = sd['attnpool.c_proj.weight'].shape[0]
        self.input_resolution = 32 * round((sd['attnpool.positional_embedding'].shape[0] - 1) ** 0.5)
        self._sd = OrderedDict((k, v.contiguous()) for k, v in fold_resnet_state_dict(sd, dtype=torch.float32).items())
        self._generation, self.recomputes, self._handle_epoch = 0, 0, 0        # see _EncodeImage
        self._patch_gen = 0
        _patchlink.register(self)
        if max_batch:
            self._ensure(max_batch)

    def _ensure(self, S):
        if self.handle is not None and S <= self.max_batch:
            return
        self._build(RnConfig((C.c_int32 * 4)(*self.layers), self.width, self.heads, self.output_dim, self.input_resolution, int(S), 0), S)
        self._handle_epoch += 1

    def _fwd(self, xi, S, emb, save_for_bwd):
        check(lib().aph_rn_fwd(self.handle, xi.data_ptr(), S, xi.shape[-1], emb.data_ptr(), save_for_bwd, stream_ptr()), 'aph_rn_fwd')

    def _bwd(self, g, S, side, gi):
        check(lib().aph_rn_bwd(self.handle, g.data_ptr(), S, side, gi.data_ptr(), stream_ptr()), 'aph_rn_bwd')

    def check_input(self, x):
        lo, hi = rn_sides(self.input_resolution)
        g = self.input_resolution // 32
        if x.dim() != 4 or x.shape[1] != 3 or x.shape[2] != x.shape[3] or not lo <= x.shape[2] <= hi:
            raise ValueError('encode_image: the ResNet takes images [S, 3, side, side] with %d <= side <= %d (a %d x %d final map), '
                             'got %s' % (lo, hi, g, g, tuple(x.shape)))

    def __call__(self, x):
        require_cuda(x, 'encode_image input')
        self.check_input(x)
        return _EncodeImage.apply(x, self, False)


class CLIP:
    """What clip_fft.py needs from clip.model.CLIP."""

    def __init__(self, name, state_dict, synthetic):
        self.name, self.synthetic = name, synthetic
        self.visual = ModifiedResNet(state_dict) if is_resnet(state_dict) else VisionTransformer(state_dict)
        self.embed_dim = self.visual.output_dim
        self.transformer = TextTransformer(state_dict) if has_text_tower(state_dict) else None
        _trace.text_tower('cuda' if self.transformer is not None else 'stand-in')

    def encode_image(self, image):
        return self.visual(image)

    def encode_text(self, tokens):
        """With text-tower weights: the CLIP text encoder on the GPU (tokens: CUDA [n, context]) -> [n, embed_dim] fp32, no
        grad. Without them: a deterministic seeded stand-in per token row set, unit norm x 10."""
        _trace.encode_text()
        if self.transformer is not None:
            return self.transformer(tokens)
        dev = tokens.device
        digest = hashlib.sha256(tokens.detach().cpu().numpy().tobytes() + self.name.encode()).digest()
        g = torch.Generator().manual_seed(int.from_bytes(digest[:7], 'little'))
        emb = torch.randn(tokens.shape[0], self.embed_dim, generator=g)
        emb = 10. * emb / emb.norm(dim=-1, keepdim=True)
        return emb.to(dev)

    def eval(self):
        return self

    def cuda(self):
        return self

    def float(self):
        return self


VOCAB_FILE = 'bpe_simple_vocab_16e6.txt.gz'
_weights_dir = None          # directory of the weights file load() used last: its VOCAB_FILE is the default vocabulary
_tokenizers = {}


def vocab_path():
    """The BPE vocabulary in use: APH_CLIP_BPE, else VOCAB_FILE next to the loaded weights, else None (byte-level stand-in)."""
    p = os.environ.get('APH_CLIP_BPE')
    if p:
        if not os.path.isfile(p):
            raise RuntimeError('aphantasia_b200.clip: APH_CLIP_BPE=%s is not a file' % p)
        return p
    if _weights_dir is not None and os.path.isfile(os.path.join(_weights_dir, VOCAB_FILE)):
        return os.path.join(_weights_dir, VOCAB_FILE)
    return None


def _tokenizer():
    p = vocab_path()
    if p is None:
        return None
    if p not in _tokenizers:
        _tokenizers[p] = SimpleTokenizer(p)
    return _tokenizers[p]


def tokenize(texts, context_length=77, truncate=False):
    """clip.tokenize: LongTensor [n, context_length] = [sot] + BPE ids + [eot], zero padded. RuntimeError when a prompt does
    not fit and truncate is False; truncate=True cuts it and ends it with eot.
    Without a vocabulary (see vocab_path): the byte-level stand-in (start 49406, UTF-8 bytes, end 49407, cut to fit)."""
    if isinstance(texts, str):
        texts = [texts]
    tok = _tokenizer()
    out = torch.zeros(len(texts), context_length, dtype=torch.long)
    if tok is None:
        for i, t in enumerate(texts):
            b = list(t.encode('utf-8'))[:context_length - 2]
            toks = [49406] + b + [49407]
            out[i, :len(toks)] = torch.tensor(toks)
        return out
    for i, t in enumerate(texts):
        toks = [tok.sot] + tok.encode(t) + [tok.eot]
        if len(toks) > context_length:
            if not truncate:
                raise RuntimeError('Input %s is too long for context length %d' % (t, context_length))
            toks = toks[:context_length]
            toks[-1] = tok.eot
        out[i, :len(toks)] = torch.tensor(toks)
    return out


def _read_weights(path):
    """OpenAI's TorchScript archive (torch.load refuses those under weights_only) or a plain state dict -> fp32 state dict
    without the JIT model's non-tensor attributes."""
    if _is_torchscript(path):
        sd = torch.jit.load(path, map_location='cpu').state_dict()
    else:
        sd = torch.load(path, map_location='cpu')
        if hasattr(sd, 'state_dict'):
            sd = sd.state_dict()
    return OrderedDict((k, v.float() if v.is_floating_point() else v) for k, v in sd.items()
                       if k not in ('input_resolution', 'context_length', 'vocab_size'))


def _is_torchscript(path):
    """torch.jit.save archives carry compiled code and a constants table; torch.save archives do not."""
    if not zipfile.is_zipfile(path):
        return False
    with zipfile.ZipFile(path) as z:
        return any(n.endswith('/constants.pkl') for n in z.namelist())


def load(name, device=None, jit=False, download_root=None):
    """clip.load: returns (model, preprocess). `preprocess` is unused by the scripts (None)."""
    global _weights_dir
    if name not in _MODELS:
        raise RuntimeError('aphantasia_b200.clip: model %s not available (the CUDA hot path covers %s)' % (name, available_models()))
    var = weights_variable(name)
    path = os.environ.get(var, os.environ.get('APH_CLIP_WEIGHTS'))
    if path and os.path.isfile(path):
        sd = _read_weights(path)
        synthetic = False
        if name in CHECKPOINT_ONLY:
            m = _MODELS[name]
            want = (m['layers'], m['width'], m['res'])
            got = resnet_architecture(sd) if is_resnet(sd) else None
            if got != want:
                held = 'a ResNet of layers %s, width %d, resolution %d' % got if got else 'no ResNet image tower'
                raise RuntimeError('aphantasia_b200.clip: %s holds %s, not %s (layers %s, width %d, resolution %d)'
                                   % ((path, held, name) + want))
        _weights_dir = os.path.dirname(os.path.abspath(path))
        if has_text_tower(sd) and vocab_path() is None:
            print(' [aphantasia_b200.clip] WARNING: no BPE vocabulary (set APH_CLIP_BPE=<%s> or put it next to %s): prompts will be '
                  'byte-tokenized and the text encoder will not see CLIP tokens' % (VOCAB_FILE, path))
    elif name in CHECKPOINT_ONLY:
        raise RuntimeError('aphantasia_b200.clip: model %s not available without its OpenAI checkpoint: set %s=<%s.pt> (or '
                           'APH_CLIP_WEIGHTS)' % (name, var, name))
    else:
        synth = synthetic_resnet_state_dict if name.startswith('RN') else synthetic_visual_state_dict
        sd = synth(seed=int(os.environ.get('APH_CLIP_SEED', '0')), **_MODELS[name])
        synthetic = True
        print(' [aphantasia_b200.clip] no CLIP weights available: using seeded synthetic %s weights and seeded text embeddings' % name)
    return CLIP(name, sd, synthetic), None
