"""Drop-in for the OpenAI `clip` package as used by /root/reference/clip_fft.py (:19,119,121,133,150,216,254):
`clip.load(name, jit=False) -> (model, preprocess)`, `clip.tokenize`, `model.encode_image`, `model.encode_text`,
`model.visual.input_resolution`.

The image encoder (ViT-B/32, ViT-B/16) runs forward and data-gradient in libaphb200.so (csrc/vit.cu: wgmma
GEMMs + fused kernels). Weights: an OpenAI state dict if `APH_CLIP_WEIGHTS=<file.pt>` is set, else seeded
synthetic weights of the same architecture (there are no CLIP weights or network in this environment).
The text encoder runs once before the optimisation loop and is not part of the hot path: without real weights
`encode_text` returns a deterministic seeded embedding per prompt (loudly).
"""
import ctypes as C
import hashlib
import os
from collections import OrderedDict

import torch

from .. import _patchlink, _pool, _trace
from .._lib import VitConfig, check, lib, require_cuda, stream_ptr

_MODELS = {'ViT-B/32': dict(patch=32, width=768, layers=12, heads=12, out_dim=512, res=224),
           'ViT-B/16': dict(patch=16, width=768, layers=12, heads=12, out_dim=512, res=224)}


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
            check(lib().aph_vit_fwd(vis.handle, xi.data_ptr(), S, emb.data_ptr(), int(need_bwd), stream_ptr()), 'aph_vit_fwd')
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
            check(lib().aph_vit_fwd(vis.handle, xi.data_ptr(), ctx.S, scratch.data_ptr(), 1, stream_ptr()), 'aph_vit_fwd (recompute)')
            vis._generation += 1            # the arena now belongs to this call; any other pending backward must recompute too
            vis.recomputes += 1
        gi = _pool.empty(ctx.shape)
        check(lib().aph_vit_bwd(vis.handle, g.data_ptr(), ctx.S, gi.data_ptr(), stream_ptr()), 'aph_vit_bwd')
        return gi, None, None


class VisionTransformer:
    """Handle-owning mirror of clip.model.VisionTransformer (forward only through the C ABI)."""

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
        self.handle, self.max_batch = None, 0
        self._generation, self.recomputes, self._handle_epoch = 0, 0, 0        # see _EncodeImage
        self._patch_gen, self._patch_written, self.prepatched_forwards = 0, False, 0      # see _patchlink
        _patchlink.register(self)
        if max_batch:
            self._ensure(max_batch)

    def _ensure(self, S):
        """(Re)creates the device handle so that its activation arena holds S samples."""
        if self.handle is not None and S <= self.max_batch:
            return
        self.close()
        cfg = VitConfig(self.patch_size, self.width, self.layers, self.heads, self.output_dim, self.input_resolution, int(S), 0)
        h = C.c_void_p()
        check(lib().aph_vit_create(C.byref(h), C.byref(cfg)), 'aph_vit_create')
        st = stream_ptr()
        for k, v in self._sd.items():
            d = v.cuda()
            check(lib().aph_vit_load_tensor(h, ('visual.' + k).encode(), d.data_ptr(), d.numel(), st), 'aph_vit_load_tensor(%s)' % k)
        torch.cuda.current_stream().synchronize()      # staging copies `d` die with this scope
        check(lib().aph_vit_finalize(h), 'aph_vit_finalize')
        self.handle, self.max_batch = h, int(S)
        self._handle_epoch += 1

    def close(self):
        if self.handle is not None:
            lib().aph_vit_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __call__(self, x):
        return _EncodeImage.apply(x, self, _patchlink.matches(x, self))


class CLIP:
    """What clip_fft.py needs from clip.model.CLIP."""

    def __init__(self, name, state_dict, synthetic):
        self.name, self.synthetic = name, synthetic
        self.visual = VisionTransformer(state_dict)
        self.embed_dim = self.visual.output_dim

    def encode_image(self, image):
        return self.visual(image)

    def encode_text(self, tokens):
        """Deterministic seeded stand-in (no text-tower weights / BPE vocab in this environment), unit norm x 10."""
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


def tokenize(texts, context_length=77, truncate=False):
    """Byte-level stand-in for clip.tokenize: LongTensor [n, 77] (start 49406, bytes, end 49407, zero padded)."""
    if isinstance(texts, str):
        texts = [texts]
    out = torch.zeros(len(texts), context_length, dtype=torch.long)
    for i, t in enumerate(texts):
        b = list(t.encode('utf-8'))[:context_length - 2]
        toks = [49406] + b + [49407]
        out[i, :len(toks)] = torch.tensor(toks)
    return out


def load(name, device=None, jit=False, download_root=None):
    """clip.load: returns (model, preprocess). `preprocess` is unused by the scripts (None)."""
    if name not in _MODELS:
        raise RuntimeError('aphantasia_b200.clip: model %s not available (the CUDA hot path covers %s)' % (name, available_models()))
    path = os.environ.get('APH_CLIP_WEIGHTS_' + name.replace('/', '').replace('-', '').upper(), os.environ.get('APH_CLIP_WEIGHTS'))
    if path and os.path.isfile(path):
        sd = torch.load(path, map_location='cpu')
        if hasattr(sd, 'state_dict'):
            sd = sd.state_dict()
        synthetic = False
    else:
        sd = synthetic_visual_state_dict(seed=int(os.environ.get('APH_CLIP_SEED', '0')), **_MODELS[name])
        synthetic = True
        print(' [aphantasia_b200.clip] no CLIP weights available: using seeded synthetic %s weights and seeded text embeddings' % name)
    return CLIP(name, sd, synthetic), None
