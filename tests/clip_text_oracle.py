"""fp32 oracle of the CLIP text tower (test infrastructure; ``clip.model.CLIP.encode_text`` on the upstream key layout), a synthetic
BPE vocabulary in CLIP's file format, the same tower re-keyed for ``transformers.CLIPTextModelWithProjection``, and the plan
interpreter extended with the text tower's ops (TOKEN_EMBED, ROW_GATHER, causal ATTN_FWD)."""
from __future__ import annotations

import collections
import gzip
import json
import math

import torch as th
import torch.nn.functional as F

from clip_guided_diffusion_b200.tokenizer import clean
from tests.plan_interp import Interp


# ---------------------------------------------------------------- fp32 oracle
def encode_text(sd: dict, ids: th.Tensor) -> th.Tensor:
    """ids int [n, T] -> fp32 [n, D]: token + positional embedding, causal pre-LN residual blocks (QuickGELU MLP), ln_final,
    the row of the largest id (EOT) of each sequence, text_projection"""
    f = {k: v.detach().double() for k, v in sd.items() if not k.startswith("visual.")}
    ids = ids.long()
    n, T = ids.shape
    w = f["ln_final.weight"].shape[0]
    heads, d = w // 64, 64
    x = f["token_embedding.weight"][ids] + f["positional_embedding"][:T]
    mask = th.full((T, T), float("-inf"), dtype=th.float64).triu(1)
    layers = len({k.split(".")[2] for k in f if k.startswith("transformer.resblocks.")})
    for i in range(layers):
        p = f"transformer.resblocks.{i}."
        y = F.layer_norm(x, (w,), f[p + "ln_1.weight"], f[p + "ln_1.bias"], 1e-5)
        q, k, v = (y @ f[p + "attn.in_proj_weight"].t() + f[p + "attn.in_proj_bias"]).split(w, dim=-1)
        q, k, v = (t.view(n, T, heads, d).transpose(1, 2) for t in (q, k, v))
        a = th.softmax(q @ k.transpose(-1, -2) / math.sqrt(d) + mask, dim=-1) @ v
        x = x + a.transpose(1, 2).reshape(n, T, w) @ f[p + "attn.out_proj.weight"].t() + f[p + "attn.out_proj.bias"]
        y = F.layer_norm(x, (w,), f[p + "ln_2.weight"], f[p + "ln_2.bias"], 1e-5)
        u = y @ f[p + "mlp.c_fc.weight"].t() + f[p + "mlp.c_fc.bias"]
        x = x + (u * th.sigmoid(1.702 * u)) @ f[p + "mlp.c_proj.weight"].t() + f[p + "mlp.c_proj.bias"]
    x = F.layer_norm(x, (w,), f["ln_final.weight"], f["ln_final.bias"], 1e-5)
    return (x[th.arange(n), ids.argmax(dim=-1)] @ f["text_projection"]).float()


# ---------------------------------------------------------------- transformers' layout
def hf_text_model(sd: dict, context_length: int, vocab_size: int):
    """``CLIPTextModelWithProjection`` holding the same weights; eos_token_id = 2 makes it pool at the argmax id like CLIP"""
    from transformers import CLIPTextConfig, CLIPTextModelWithProjection
    w = sd["ln_final.weight"].shape[0]
    layers = len({k.split(".")[2] for k in sd if k.startswith("transformer.resblocks.")})
    cfg = CLIPTextConfig(vocab_size=vocab_size, hidden_size=w, intermediate_size=4 * w, num_hidden_layers=layers, num_attention_heads=w // 64,
                         max_position_embeddings=context_length, hidden_act="quick_gelu", projection_dim=sd["text_projection"].shape[1],
                         layer_norm_eps=1e-5, eos_token_id=2, attn_implementation="eager")
    m = CLIPTextModelWithProjection(cfg).eval()
    hk = {"text_model.embeddings.token_embedding.weight": sd["token_embedding.weight"],
          "text_model.embeddings.position_embedding.weight": sd["positional_embedding"],
          "text_model.final_layer_norm.weight": sd["ln_final.weight"], "text_model.final_layer_norm.bias": sd["ln_final.bias"],
          "text_projection.weight": sd["text_projection"].t()}
    for i in range(layers):
        p, q = f"transformer.resblocks.{i}.", f"text_model.encoder.layers.{i}."
        for name, t in zip("qkv", sd[p + "attn.in_proj_weight"].split(w)):
            hk[q + f"self_attn.{name}_proj.weight"] = t
        for name, t in zip("qkv", sd[p + "attn.in_proj_bias"].split(w)):
            hk[q + f"self_attn.{name}_proj.bias"] = t
        for src, dst in (("attn.out_proj", "self_attn.out_proj"), ("ln_1", "layer_norm1"), ("ln_2", "layer_norm2"), ("mlp.c_fc", "mlp.fc1"),
                         ("mlp.c_proj", "mlp.fc2")):
            hk[q + dst + ".weight"] = sd[p + src + ".weight"]
            hk[q + dst + ".bias"] = sd[p + src + ".bias"]
    missing, unexpected = m.load_state_dict({k: v.float() for k, v in hk.items()}, strict=False)
    assert not unexpected and all("position_ids" in k for k in missing), (missing, unexpected)
    return m


# ---------------------------------------------------------------- synthetic vocabulary
# GPT-2's published byte alphabet (Radford et al. 2019, encoder.py), written out here rather than taken from the package: ids 0..187
# are the printable bytes ! .. ~, ¡ .. ¬, ® .. ÿ as themselves, ids 188..255 the other 68 bytes in byte order as chr(256), chr(257), ...
# CLIP's vocabulary starts with these 256 symbols, then the same 256 with </w>.
PRINTABLE_BYTES = [*range(0x21, 0x7F), *range(0xA1, 0xAD), *range(0xAE, 0x100)]
OTHER_BYTES = [b for b in range(256) if b not in PRINTABLE_BYTES]
BYTE_SYMBOL = {**{b: chr(b) for b in PRINTABLE_BYTES}, **{b: chr(256 + k) for k, b in enumerate(OTHER_BYTES)}}
SYMBOLS = [chr(b) for b in PRINTABLE_BYTES] + [chr(256 + k) for k in range(len(OTHER_BYTES))]
# ids of the published CLIP vocabulary (bpe_simple_vocab_16e6.txt.gz) that depend on this order alone
PUBLISHED_IDS = {"!": 0, '"': 1, "a": 64, "ÿ": 187, chr(256): 188, "\u0120": 220, chr(323): 255, "!</w>": 256, "a</w>": 320,
                 ".</w>": 269, ",</w>": 267, "1</w>": 272}

CORPUS = ("a lighthouse on a rocky coast at sunset, oil painting by an old master.  it's the painter's 2nd work; they're sure we've "
          "seen 3 boats & 12 birds!! i'm told you'll find the red fox, she'd said.  a photograph of a cat sitting in a window, "
          "trending on artstation, 4k, highly detailed, cinematic lighting, matte painting of mountains and rivers in the morning. ")


def synthetic_merges(n_merges: int = 400, corpus: str = CORPUS) -> "list[tuple[str, str]]":
    """byte-level BPE merges learned from `corpus` (most frequent adjacent pair first, ties by the pair): a well-formed merges list"""
    import regex
    pat = regex.compile(r"""'s|'t|'re|'ve|'m|'ll|'d|[\p{L}]+|[\p{N}]|[^\s\p{L}\p{N}]+""", regex.IGNORECASE)
    words = collections.Counter()
    for t in pat.findall(clean(corpus)):
        s = "".join(BYTE_SYMBOL[b] for b in t.encode("utf-8"))
        words[tuple(s[:-1]) + (s[-1] + "</w>",)] += 1
    merges = []
    while len(merges) < n_merges:
        pairs = collections.Counter()
        for wd, c in words.items():
            for a, b in zip(wd, wd[1:]):
                pairs[(a, b)] += c
        if not pairs:
            break
        best = max(pairs, key=lambda p: (pairs[p], p))
        merges.append(best)
        merged = collections.Counter()
        for wd, c in words.items():
            out, i = [], 0
            while i < len(wd):
                if i + 1 < len(wd) and (wd[i], wd[i + 1]) == best:
                    out.append(wd[i] + wd[i + 1])
                    i += 2
                else:
                    out.append(wd[i])
                    i += 1
            merged[tuple(out)] += c
        words = merged
    return merges


def write_vocab(path, merges) -> int:
    """CLIP's format: gzip text, a version line, one merge per line.  Returns the vocabulary size (512 + merges + 2)."""
    with gzip.open(path, "wt", encoding="utf-8") as f:
        f.write("#version: 0.2\n" + "\n".join(" ".join(m) for m in merges) + "\n")
    return 512 + len(merges) + 2


def write_hf_vocab(dirpath, merges):
    """the CLIP vocabulary of these merges as transformers' vocab.json / merges.txt, laid out from the published byte order above"""
    vocab = SYMBOLS + [s + "</w>" for s in SYMBOLS] + ["".join(m) for m in merges] + ["<|startoftext|>", "<|endoftext|>"]
    with open(f"{dirpath}/vocab.json", "w", encoding="utf-8") as f:
        json.dump({t: i for i, t in enumerate(vocab)}, f)
    with open(f"{dirpath}/merges.txt", "w", encoding="utf-8") as f:
        f.write("#version: 0.2\n" + "\n".join(" ".join(m) for m in merges) + "\n")
    return f"{dirpath}/vocab.json", f"{dirpath}/merges.txt"


# ---------------------------------------------------------------- plan interpreter with the text tower's ops
class TextInterp(Interp):
    def op_ATTN_FWD(self, op):
        if not op.flags & 1:
            return super().op_ATTN_FWD(op)
        B, heads, T, d = op.i[:4]
        obs, ors, ohs = op.i[7:10]
        q, k, v = (t.float() for t in self._attn_views(op, op.p[:3]))
        s = ((q @ k.transpose(-1, -2)) * op.f[0]).masked_fill(th.ones(T, T, dtype=th.bool).triu(1), float("-inf"))
        self.V(op.p[4], (B, heads, T), (heads * T, T, 1)).copy_(th.logsumexp(s, dim=-1))
        self.V(op.p[3], (B, heads, T, d), (obs, ohs, ors, 1)).copy_(th.softmax(s, dim=-1) @ v)

    def op_TOKEN_EMBED(self, op):
        n, T, w, V = op.i[:4]
        ids = self.V(op.p[0], (n, T), (T, 1)).long()
        table = self.V(op.p[1], (V, w), (w, 1)).float()
        pos = self.V(op.p[2], (T, w), (w, 1))
        self.V(op.p[3], (n, T, w), (T * w, w, 1)).copy_(table[ids] + pos)

    def op_ROW_GATHER(self, op):
        rows, w, ldx, ldy, n_src = op.i[:5]
        x = self.V(op.p[0], (n_src, w), (ldx, 1))
        idx = self.V(op.p[1], (rows,), (1,)).long()
        self.V(op.p[2], (rows, w), (ldy, 1)).copy_(x[idx])
