"""CLIP text tower (``clip.model.CLIP.encode_text``) as a forward-only H100 op plan.

Replaces the eager ``clip_model.encode_text(clip.tokenize(txt))`` of the reference's ``encode_text_prompt`` (cgd/clip_util.py:104-108),
run once per text prompt set and run, outside the sampling loop.  The weights are the text half of the same CLIP state_dict the
visual tower loads (upstream key layout: ``token_embedding``, ``positional_embedding``, ``transformer.resblocks.N``, ``ln_final``,
``text_projection``).  The ops, in order:

    TOKEN_EMBED -> layers x (ln_1, qkv, causal ATTN_FWD, out_proj + residual, ln_2, c_fc, QuickGELU (GELU: OpenCLIP), c_proj + residual)
    -> ROW_GATHER of each sequence's end-of-text row -> ln_final -> fp32 text_projection (LINEAR_SMALL)

Linear layers run on the wgmma GEMM kernel with fp16 operands and fp32 accumulation, like the ViT (the reference's CUDA path loads
CLIP in fp16, cgd/clip_util.py:64-65); LayerNorm statistics, softmax and the projection are fp32.  ln_final runs on the gathered rows
only: LayerNorm is per row, so gathering first gives the same embeddings as the reference's ln_final over every token.
"""
from __future__ import annotations

from dataclasses import dataclass

import torch as th

from .plan import Act, Plan, pack_conv


@dataclass
class TextConfig:
    width: int = 512
    layers: int = 12
    context_length: int = 77
    vocab_size: int = 49408
    output_dim: int = 512
    act: str = "quick_gelu"  # the MLP's activation: "quick_gelu" (OpenAI CLIP) or "gelu" (exact erf GELU, OpenCLIP)

    @property
    def heads(self):
        return self.width // 64


def text_config_from_state_dict(sd: dict, act: str = "quick_gelu") -> TextConfig:
    """clip.model.build_model's reading of the text half: width = ln_final size, heads = width / 64, layers = the non-visual
    transformer.resblocks.N, context = positional_embedding rows, vocab = token_embedding rows, D = text_projection columns.  The MLP
    activation is not in the keys: `act` ("gelu" for the OpenCLIP towers)"""
    need = ("token_embedding.weight", "positional_embedding", "ln_final.weight", "text_projection")
    missing = [k for k in need if k not in sd]
    if missing:
        raise ValueError(f"the CLIP state_dict has no text tower (missing {', '.join(missing)}): text prompts need a full CLIP "
                         "checkpoint, or pass target_embeds= / weights=")
    layers = len({k.split(".")[2] for k in sd if k.startswith("transformer.resblocks.")})
    return TextConfig(width=sd["ln_final.weight"].shape[0], layers=layers, context_length=sd["positional_embedding"].shape[0],
                      vocab_size=sd["token_embedding.weight"].shape[0], output_dim=sd["text_projection"].shape[1], act=act)


class TextB200:
    """encode_text for ``n_prompts`` token sequences of ``cfg.context_length``.  ``encode(ids)`` takes the int32 token ids
    (``tokenize``'s output) and returns the fp32 [n_prompts, D] embeddings.  Build it once per run, then drop it."""

    def __init__(self, cfg: TextConfig, state_dict: dict, n_prompts: int, device="cuda"):
        self.cfg, self.n = cfg, int(n_prompts)
        self.sd = state_dict
        self.plan = Plan()
        self._build()
        self.plan.finalize(device)
        del self.sd

    def _w(self, key):
        return self.sd[key].detach().float().cpu()

    def _const(self, key):
        return self.plan.const(self._w(key), "f", key)

    def _pack(self, pre, wkey, bkey):
        return pack_conv(self.plan, self._w(pre + wkey), self._w(pre + bkey), need_bwd=False, name=pre + wkey)

    def _build(self):
        p, cfg, n = self.plan, self.cfg, self.n
        w, T, D = cfg.width, cfg.context_length, cfg.output_dim
        rows = n * T
        self.ids = p.new(rows, "i32", "ids")
        self.eot_rows = p.new(n, "i32", "eot_rows")
        self.embeds = p.new(n * D, "f", "embeds")
        p.mark("text_fwd")
        table = p.const(self._w("token_embedding.weight"), "h", "token_embedding")
        x = Act(p.new(rows * w, "h", "tok"), 0, 1, 1, rows, w, w)
        p.emit("TOKEN_EMBED", i=[n, T, w, cfg.vocab_size], p=[(self.ids, 0), (table, 0), (self._const("positional_embedding"), 0), (x.buf, 0)],
               tag="token_embed")
        for li in range(cfg.layers):
            pre = f"transformer.resblocks.{li}"
            y = p.layer_norm(x, self._const(pre + ".ln_1.weight"), self._const(pre + ".ln_1.bias"), name=pre + ".ln_1")
            qkv = p.conv(y, self._pack(pre, ".attn.in_proj_weight", ".attn.in_proj_bias"), name=pre + ".qkv")
            a = p.attention(qkv, cfg.heads, T, n, legacy_order=False, causal=True, name=pre + ".attn")
            x = p.conv(a, self._pack(pre, ".attn.out_proj.weight", ".attn.out_proj.bias"), res=x, name=pre + ".out_proj")
            y = p.layer_norm(x, self._const(pre + ".ln_2.weight"), self._const(pre + ".ln_2.bias"), name=pre + ".ln_2")
            u = p.conv(y, self._pack(pre, ".mlp.c_fc.weight", ".mlp.c_fc.bias"), name=pre + ".c_fc")
            g = p.quick_gelu(u, name=pre + ".gelu", exact=cfg.act == "gelu")
            x = p.conv(g, self._pack(pre, ".mlp.c_proj.weight", ".mlp.c_proj.bias"), res=x, name=pre + ".c_proj")
        eot = Act(p.new(n * w, "h", "eot"), 0, 1, 1, n, w, w)
        p.emit("ROW_GATHER", i=[n, w, x.ld, eot.ld, rows], p=[(x.buf, x.eoff), (self.eot_rows, 0), (eot.buf, 0)], tag="eot_rows")
        c = p.layer_norm(eot, self._const("ln_final.weight"), self._const("ln_final.bias"), name="ln_final")
        proj_t = p.const(self._w("text_projection").t().contiguous(), "f", "text_projection^T")  # [D, w]
        p.emit("LINEAR_SMALL", flags=4, i=[n, w, D, w, D], p=[(c.buf, 0), (proj_t, 0), None, (self.embeds, 0)], tag="text_projection")
        p.mark("text_end")

    def encode(self, ids: th.Tensor) -> th.Tensor:
        """ids: integer [n_prompts, context_length] (SOT .. EOT, zero padded) -> fp32 [n_prompts, D] on the plan's device.  Each
        sequence is pooled at its largest id, the end-of-text token (clip.model.CLIP.encode_text: text.argmax(dim=-1))."""
        cfg = self.cfg
        ids = th.as_tensor(ids).cpu()
        if tuple(ids.shape) != (self.n, cfg.context_length):
            raise ValueError(f"token ids of shape {tuple(ids.shape)}: this tower encodes [{self.n}, {cfg.context_length}]")
        if int(ids.min()) < 0 or int(ids.max()) >= cfg.vocab_size:
            raise ValueError(f"token ids must lie in [0, {cfg.vocab_size}) (the checkpoint's vocabulary): got [{int(ids.min())}, {int(ids.max())}]")
        rows = th.arange(self.n) * cfg.context_length + ids.long().argmax(dim=-1)
        self.plan.view(self.ids).copy_(ids.reshape(-1).to(th.int32))
        self.plan.view(self.eot_rows).copy_(rows.to(th.int32))
        self.plan.run()
        return self.plan.view(self.embeds, (self.n, cfg.output_dim)).float().clone()


__all__ = ["TextB200", "TextConfig", "text_config_from_state_dict"]
