"""Test infrastructure for the CLIP text encoder: a CPU restatement of the published text tower (OpenAI clip/model.py
CLIP.encode_text; pinned to HuggingFace's CLIPTextModelWithProjection by test_text_tower_host.py) and a synthetic BPE
vocabulary written in OpenAI's format and in HuggingFace's (vocab.json + merges.txt)."""
import gzip
import json
import os
from collections import Counter, OrderedDict

import torch
import torch.nn as nn

from aphantasia_b200.clip._bpe import EOT, SOT, bytes_to_unicode
from oracle import restate as R


class CausalResidualAttentionBlock(R.ResidualAttentionBlock):
    """oracle.restate's block with an attention mask: -inf strictly above the diagonal (query i sees keys 0..i)."""

    def forward(self, x):
        T = x.shape[0]
        mask = torch.full((T, T), float('-inf')).triu_(1)
        y = self.ln_1(x)
        x = x + self.attn(y, y, y, need_weights=False, attn_mask=mask)[0]
        return x + self.mlp(self.ln_2(x))


class TextTransformer(nn.Module):
    def __init__(self, width=512, layers=12, heads=8, out_dim=512, context=77, vocab=49408):
        super().__init__()
        self.token_embedding = nn.Embedding(vocab, width)
        self.positional_embedding = nn.Parameter(torch.empty(context, width))
        self.transformer = nn.Module()
        self.transformer.resblocks = nn.Sequential(*[CausalResidualAttentionBlock(width, heads) for _ in range(layers)])
        self.ln_final = R.LayerNorm(width)
        self.text_projection = nn.Parameter(torch.empty(width, out_dim))

    def forward(self, tokens):
        x = self.token_embedding(tokens) + self.positional_embedding
        x = self.transformer.resblocks(x.permute(1, 0, 2)).permute(1, 0, 2)
        x = self.ln_final(x)
        return x[torch.arange(x.shape[0]), tokens.argmax(dim=-1)] @ self.text_projection


def build_text(state_dict):
    sd = {k: v for k, v in state_dict.items() if not k.startswith('visual.')}
    vocab, width = sd['token_embedding.weight'].shape
    layers = len([k for k in sd if k.startswith('transformer.resblocks.') and k.endswith('.attn.in_proj_weight')])
    m = TextTransformer(width, layers, width // 64, sd['text_projection'].shape[1], sd['positional_embedding'].shape[0], vocab)
    m.load_state_dict(OrderedDict((k, v.float()) for k, v in sd.items()))
    return m.float().eval()


CORPUS = ('red square red square a red square on blue blue circle circle don\'t stop it\'s cats cats with hyphens and '
          'underscores squares stop stopping reds')


def _learn_merges(words, n):
    """Plain BPE training (most frequent adjacent pair, ties by order) over byte symbols: n merges that are all valid."""
    be = bytes_to_unicode()
    corpus = Counter()
    for w in words:
        s = tuple(be[b] for b in w.encode('utf-8'))
        corpus[s[:-1] + (s[-1] + '</w>',)] += 1
    merges = []
    for _ in range(n):
        counts = Counter()
        for s, c in corpus.items():
            for p in zip(s[:-1], s[1:]):
                counts[p] += c
        if not counts:
            break
        best = max(sorted(counts), key=lambda p: counts[p])
        merges.append(best)
        nxt = Counter()
        for s, c in corpus.items():
            out, i = [], 0
            while i < len(s):
                if i < len(s) - 1 and (s[i], s[i + 1]) == best:
                    out.append(s[i] + s[i + 1]); i += 2
                else:
                    out.append(s[i]); i += 1
            nxt[tuple(out)] += c
        corpus = nxt
    return merges


def write_vocab(directory, n_merges=40):
    """Writes bpe_simple_vocab_16e6.txt.gz (OpenAI format) plus vocab.json / merges.txt (HuggingFace format) with the same
    merges; returns (gz path, vocab.json path, merges.txt path, vocabulary size)."""
    import regex
    from aphantasia_b200.clip._bpe import _PAT
    words = regex.findall(_PAT, CORPUS, regex.IGNORECASE)
    merges = _learn_merges(words, n_merges)
    os.makedirs(directory, exist_ok=True)
    gz = os.path.join(directory, 'bpe_simple_vocab_16e6.txt.gz')
    with gzip.open(gz, 'wt', encoding='utf-8') as f:
        f.write('"bpe_simple_vocab_16e6.txt#version: 0.2\n' + ''.join('%s %s\n' % m for m in merges))
    vocab = list(bytes_to_unicode().values())
    vocab += [v + '</w>' for v in vocab]
    vocab += [a + b for a, b in merges] + [SOT, EOT]
    vj, mt = os.path.join(directory, 'vocab.json'), os.path.join(directory, 'merges.txt')
    with open(vj, 'w', encoding='utf-8') as f:
        json.dump({v: i for i, v in enumerate(vocab)}, f)
    with open(mt, 'w', encoding='utf-8') as f:
        f.write('#version: 0.2\n' + ''.join('%s %s\n' % m for m in merges))
    return gz, vj, mt, len(vocab)
