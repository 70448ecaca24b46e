"""CLIP text encoder, host side: the BPE tokenizer against HuggingFace's CLIPTokenizer, the tokenize() contract, the text-tower
restatement against HuggingFace's CLIPTextModelWithProjection, and loading OpenAI's TorchScript checkpoints."""
import os
from collections import OrderedDict

import pytest
import torch
import torch.nn as nn

import text_oracle as TO
from aphantasia_b200 import clip

PROMPTS = ['red square', 'A Red  Square,  on   blue!', "don't stop", "it's 3:1 | 42 cats", 'with-hyphens and_underscores', 'blue circle']


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


@pytest.fixture
def vocab(tmp_path, monkeypatch):
    gz, vj, mt, n = TO.write_vocab(str(tmp_path / 'vocab'))
    monkeypatch.setenv('APH_CLIP_BPE', gz)
    return gz, vj, mt, n


def test_bpe_matches_hf_tokenizer(vocab):
    transformers = pytest.importorskip('transformers')
    gz, vj, mt, n = vocab
    hf = transformers.CLIPTokenizer(vj, mt)
    ours = clip._bpe.SimpleTokenizer(gz)
    assert (ours.sot, ours.eot, ours.vocab_size) == (n - 2, n - 1, n)
    assert len(ours.bpe_ranks) == 40
    for p in PROMPTS:
        want = hf(p)['input_ids']
        assert [ours.sot] + ours.encode(p) + [ours.eot] == want, p
    # the merges are used: a merged word is fewer ids than its bytes
    assert len(ours.encode('red square')) < len('redsquare')


def test_tokenize_contract_with_vocabulary(vocab):
    gz, _, _, n = vocab
    tok = clip.tokenize(PROMPTS)
    assert tok.dtype == torch.long and tok.shape == (len(PROMPTS), 77)
    ref = clip._bpe.SimpleTokenizer(gz)
    for i, p in enumerate(PROMPTS):
        ids = [n - 2] + ref.encode(p) + [n - 1]
        assert tok[i, :len(ids)].tolist() == ids and not tok[i, len(ids):].any()
    assert clip.tokenize('red square', context_length=16).shape == (1, 16)
    long_prompt = ' '.join(['cats stop'] * 40)
    with pytest.raises(RuntimeError, match='too long'):
        clip.tokenize(long_prompt)
    t = clip.tokenize(long_prompt, truncate=True)
    assert t.shape == (1, 77) and t[0, 0] == n - 2 and t[0, -1] == n - 1 and (t[0] == n - 1).sum() == 1
    assert t[0, 1:76].tolist() == ref.encode(long_prompt)[:75]


def test_tokenize_without_vocabulary_is_the_byte_stand_in(monkeypatch):
    monkeypatch.delenv('APH_CLIP_BPE', raising=False)
    monkeypatch.setattr(clip, '_weights_dir', None)
    for p in PROMPTS + ['x' * 200]:
        b = list(p.encode('utf-8'))[:75]
        want = torch.zeros(1, 77, dtype=torch.long)
        want[0, :len(b) + 2] = torch.tensor([49406] + b + [49407])
        assert torch.equal(clip.tokenize(p), want)


def test_vocabulary_next_to_the_weights_is_found(tmp_path, monkeypatch):
    monkeypatch.delenv('APH_CLIP_BPE', raising=False)
    gz, _, _, n = TO.write_vocab(str(tmp_path))
    monkeypatch.setattr(clip, '_weights_dir', str(tmp_path))
    assert clip.vocab_path() == gz and clip.tokenize('red')[0, 0] == n - 2


def test_text_restatement_matches_hf():
    """OpenAI-layout text-tower restatement vs the independent HuggingFace CLIP text model (small geometry, varied EOT
    positions including the last one)."""
    transformers = pytest.importorskip('transformers')
    from transformers import CLIPTextConfig, CLIPTextModelWithProjection
    width, layers, heads, out, ctx, vocab = 128, 2, 2, 64, 16, 300
    sd = clip.synthetic_text_state_dict(width, layers, heads, out, ctx, vocab, seed=3)
    ours = TO.build_text(sd)
    cfg = CLIPTextConfig(vocab_size=vocab, hidden_size=width, intermediate_size=4 * width, num_hidden_layers=layers, num_attention_heads=heads,
                         max_position_embeddings=ctx, projection_dim=out, hidden_act='quick_gelu', layer_norm_eps=1e-5,
                         eos_token_id=vocab - 1, bos_token_id=vocab - 2, pad_token_id=0, attn_implementation='eager')
    hf = CLIPTextModelWithProjection(cfg).eval()
    t = hf.text_model
    with torch.no_grad():
        t.embeddings.token_embedding.weight.copy_(sd['token_embedding.weight'])
        t.embeddings.position_embedding.weight.copy_(sd['positional_embedding'])
        t.final_layer_norm.weight.copy_(sd['ln_final.weight']); t.final_layer_norm.bias.copy_(sd['ln_final.bias'])
        hf.text_projection.weight.copy_(sd['text_projection'].T)
        for i, l in enumerate(t.encoder.layers):
            g = lambda k: sd['transformer.resblocks.%d.%s' % (i, k)]
            wq, wk, wv = g('attn.in_proj_weight').chunk(3); bq, bk, bv = g('attn.in_proj_bias').chunk(3)
            l.self_attn.q_proj.weight.copy_(wq); l.self_attn.q_proj.bias.copy_(bq)
            l.self_attn.k_proj.weight.copy_(wk); l.self_attn.k_proj.bias.copy_(bk)
            l.self_attn.v_proj.weight.copy_(wv); l.self_attn.v_proj.bias.copy_(bv)
            l.self_attn.out_proj.weight.copy_(g('attn.out_proj.weight')); l.self_attn.out_proj.bias.copy_(g('attn.out_proj.bias'))
            l.layer_norm1.weight.copy_(g('ln_1.weight')); l.layer_norm1.bias.copy_(g('ln_1.bias'))
            l.layer_norm2.weight.copy_(g('ln_2.weight')); l.layer_norm2.bias.copy_(g('ln_2.bias'))
            l.mlp.fc1.weight.copy_(g('mlp.c_fc.weight')); l.mlp.fc1.bias.copy_(g('mlp.c_fc.bias'))
            l.mlp.fc2.weight.copy_(g('mlp.c_proj.weight')); l.mlp.fc2.bias.copy_(g('mlp.c_proj.bias'))
    g = torch.Generator().manual_seed(0)
    toks = torch.zeros(4, ctx, dtype=torch.long)
    for r, e in enumerate([1, 5, 9, ctx - 1]):                  # EOT at position e, random ids before it, zero padding after
        toks[r, 0] = vocab - 2
        toks[r, 1:e] = torch.randint(1, vocab - 2, (e - 1,), generator=g)
        toks[r, e] = vocab - 1
    with torch.no_grad():
        a = ours(toks)
        b = hf(input_ids=toks).text_embeds
    assert a.shape == (4, out) and _rel(a, b) < 1e-5


def _scripted_checkpoint(sd):
    """A TorchScript archive holding `sd` under its keys, as OpenAI's released checkpoints are."""
    class Ckpt(nn.Module):
        def forward(self, x):
            return x * 2
    root = Ckpt()
    for k, v in sd.items():
        *path, leaf = k.split('.')
        m = root
        for p in path:
            if not hasattr(m, p):
                m.add_module(p, nn.Module())
            m = getattr(m, p)
        if v.is_floating_point():
            m.register_parameter(leaf, nn.Parameter(v, requires_grad=False))
        else:
            m.register_buffer(leaf, v)
    return torch.jit.trace(root, torch.zeros(1))


def test_load_accepts_torchscript_checkpoints(tmp_path, monkeypatch):
    """fp16 OpenAI-layout TorchScript archive via APH_CLIP_WEIGHTS -> a non-synthetic CLIP whose text and visual tensors are
    the saved ones in fp32 (torch.load refuses such archives under torch >= 2.6)."""
    sd = OrderedDict()
    sd.update((k, v.half()) for k, v in clip.synthetic_visual_state_dict(patch=32, width=128, layers=1, heads=2, out_dim=128, seed=1).items())
    sd.update((k, v.half()) for k, v in clip.synthetic_text_state_dict(128, 1, 2, 128, 77, 600, seed=2).items())
    for k, v in (('input_resolution', 224), ('context_length', 77), ('vocab_size', 600)):
        sd[k] = torch.tensor(v)
    path = str(tmp_path / 'ViT-B-32.pt')
    torch.jit.save(_scripted_checkpoint(sd), path)
    monkeypatch.setenv('APH_CLIP_WEIGHTS', path)
    monkeypatch.delenv('APH_CLIP_BPE', raising=False)
    model, _ = clip.load('ViT-B/32', jit=False)
    assert not model.synthetic and model.transformer is not None
    for k, v in sd.items():
        if k.startswith('visual.'):
            got = model.visual._sd[k[len('visual.'):]]
        elif v.is_floating_point():
            got = model.transformer._sd[k]
        else:
            continue
        assert got.dtype == torch.float32 and torch.equal(got, v.float()), k
    assert (model.transformer.width, model.transformer.layers, model.transformer.vocab, model.transformer.context) == (128, 1, 600, 77)


def test_clip_without_text_weights_keeps_the_stand_in():
    sd = clip.synthetic_visual_state_dict(patch=32, width=128, layers=1, heads=2, out_dim=128, seed=0)
    model = clip.CLIP('ViT-B/32', sd, True)
    assert model.transformer is None
    e = model.encode_text(torch.zeros(1, 77, dtype=torch.long))
    assert e.shape == (1, 128) and abs(float(e.norm()) - 10.) < 1e-4
