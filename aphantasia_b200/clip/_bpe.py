"""CLIP's byte-level BPE tokenizer, written from the published algorithm (Radford et al. 2021, after GPT-2's byte-level BPE;
Sennrich et al. 2016 for BPE itself).

Vocabulary file: OpenAI's `bpe_simple_vocab_16e6.txt.gz` format -- gzip text, one header line, then one merge pair per line
("a b"). At most 48 894 merges are used (49 408 ids in all for the real file). Ids are assigned in this order: the 256
byte symbols, the same with the end-of-word marker `</w>`, one per merge (the merged string), then `<|startoftext|>` and
`<|endoftext|>`: so those two are the last ids (49406 / 49407 for the real file).
"""
import functools
import gzip
import html
import re

try:
    import regex
except ImportError:          # only needed once a vocabulary is in use; the byte-level stand-in works without it
    regex = None

MAX_MERGES = 49152 - 256 - 2
SOT, EOT = '<|startoftext|>', '<|endoftext|>'
# contractions, runs of letters, single digits, runs of other non-space characters
_PAT = r"""<\|startoftext\|>|<\|endoftext\|>|'s|'t|'re|'ve|'m|'ll|'d|[\p{L}]+|[\p{N}]|[^\s\p{L}\p{N}]+"""


@functools.lru_cache()
def bytes_to_unicode():
    """Reversible byte -> printable unicode character table: printable Latin-1 bytes map to themselves, the other 68 bytes to
    code points 256.. in byte order (so no byte symbol is whitespace or a control character)."""
    bs = list(range(ord('!'), ord('~') + 1)) + list(range(ord('\xa1'), ord('\xac') + 1)) + list(range(ord('\xae'), ord('\xff') + 1))
    cs = list(bs)
    n = 0
    for b in range(256):
        if b not in bs:
            bs.append(b)
            cs.append(256 + n)
            n += 1
    return dict(zip(bs, (chr(c) for c in cs)))


def _pairs(word):
    return set(zip(word[:-1], word[1:]))


def clean(text):
    try:
        import ftfy
        text = ftfy.fix_text(text)
    except ImportError:
        pass
    text = html.unescape(html.unescape(text)).strip()
    return re.sub(r'\s+', ' ', text).strip().lower()


class SimpleTokenizer:
    def __init__(self, path):
        if regex is None:
            raise RuntimeError('aphantasia_b200.clip: the BPE tokenizer needs the `regex` module (\\p{L} / \\p{N} classes)')
        with gzip.open(path, 'rt', encoding='utf-8') as f:
            lines = f.read().split('\n')[1:]
        merges = [tuple(l.split()) for l in lines if l.strip()][:MAX_MERGES]
        self.byte_encoder = bytes_to_unicode()
        vocab = list(self.byte_encoder.values())
        vocab += [v + '</w>' for v in vocab]
        vocab += [''.join(m) for m in merges]
        vocab += [SOT, EOT]
        self.encoder = {v: i for i, v in enumerate(vocab)}
        self.bpe_ranks = {m: i for i, m in enumerate(merges)}
        self.cache = {SOT: SOT, EOT: EOT}
        self.pat = regex.compile(_PAT, regex.IGNORECASE)
        self.sot, self.eot, self.vocab_size = self.encoder[SOT], self.encoder[EOT], len(vocab)

    def bpe(self, token):
        """Space-separated BPE symbols of one pre-token: merge the lowest-ranked adjacent pair until none is in the table."""
        if token in self.cache:
            return self.cache[token]
        word = tuple(token[:-1]) + (token[-1] + '</w>',)
        pairs = _pairs(word)
        while pairs:
            first, second = min(pairs, key=lambda p: self.bpe_ranks.get(p, float('inf')))
            if (first, second) not in self.bpe_ranks:
                break
            merged, i = [], 0
            while i < len(word):
                if i < len(word) - 1 and word[i] == first and word[i + 1] == second:
                    merged.append(first + second)
                    i += 2
                else:
                    merged.append(word[i])
                    i += 1
            word = tuple(merged)
            if len(word) == 1:
                break
            pairs = _pairs(word)
        out = ' '.join(word)
        self.cache[token] = out
        return out

    def encode(self, text):
        ids = []
        for tok in self.pat.findall(clean(text)):
            tok = ''.join(self.byte_encoder[b] for b in tok.encode('utf-8'))
            ids.extend(self.encoder[s] for s in self.bpe(tok).split(' '))
        return ids
