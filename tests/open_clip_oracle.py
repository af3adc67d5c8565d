"""Test infrastructure for the OpenCLIP towers (vit.OPEN_CLIP_CONFIGS): fp32 oracles with a head width and an MLP activation, the same
weights re-keyed for the independent ``transformers`` CLIP towers, and the plan interpreter extended with QGELU_FWD flags 1 (exact GELU)
and CONV flags 8 (acc * GELU'(u)).

The vision oracle is oracle/clip_vit.py's ``CLIPVisualOnly`` built from a config whose head count is width / head_width, with its MLP
activations swapped for ``nn.GELU()`` when the tower's act is "gelu"; the OpenAI defaults build the unchanged oracle."""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch as th
import torch.nn as nn
import torch.nn.functional as F

from oracle.clip_vit import CLIPVisualOnly, ViTConfig as OViTConfig
from tests.clip_text_oracle import TextInterp


# ---------------------------------------------------------------- oracles
@dataclass
class OViTHeadsConfig(OViTConfig):
    head_width: int = 64

    @property
    def heads(self):
        return self.width // self.head_width


def vision_oracle(cfg, sd: dict) -> CLIPVisualOnly:
    """oracle of the product ViTConfig `cfg` (width, layers, head_width, act) holding the `visual.*` weights of `sd`"""
    ocfg = OViTHeadsConfig(cfg.input_resolution, cfg.patch_size, cfg.width, cfg.layers, cfg.output_dim, cfg.head_width)
    m = CLIPVisualOnly(ocfg)
    if cfg.act == "gelu":
        for blk in m.visual.transformer.resblocks:
            blk.mlp.gelu = nn.GELU()
    m.load_state_dict({k: v for k, v in sd.items() if k.startswith("visual.")})
    return m.eval()


def encode_text(sd: dict, ids: th.Tensor, act: str = "quick_gelu") -> th.Tensor:
    """float64 encode_text (tests/clip_text_oracle.py's, with the MLP activation `act`): ids int [n, T] -> fp32 [n, D]"""
    f = {k: v.detach().double() for k, v in sd.items() if not k.startswith("visual.")}
    ids = ids.long()
    n, T = ids.shape
    w = f["ln_final.weight"].shape[0]
    heads, d = w // 64, 64
    x = f["token_embedding.weight"][ids] + f["positional_embedding"][:T]
    mask = th.full((T, T), float("-inf"), dtype=th.float64).triu(1)
    gelu = F.gelu if act == "gelu" else (lambda u: u * th.sigmoid(1.702 * u))
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
        x = x + gelu(u) @ f[p + "mlp.c_proj.weight"].t() + f[p + "mlp.c_proj.bias"]
    x = F.layer_norm(x, (w,), f["ln_final.weight"], f["ln_final.bias"], 1e-5)
    return (x[th.arange(n), ids.argmax(dim=-1)] @ f["text_projection"]).float()


# ---------------------------------------------------------------- transformers' layout
def hf_vision_model(cfg, sd: dict):
    """``CLIPVisionModelWithProjection`` with cfg's heads (num_attention_heads = width / head_width) and activation, holding `sd`"""
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection
    w = cfg.width
    hf_cfg = CLIPVisionConfig(hidden_size=w, intermediate_size=4 * w, projection_dim=cfg.output_dim, num_hidden_layers=cfg.layers,
                              num_attention_heads=cfg.heads, image_size=cfg.input_resolution, patch_size=cfg.patch_size,
                              hidden_act=cfg.act, layer_norm_eps=1e-5, attention_dropout=0.0)
    hf_cfg._attn_implementation = "eager"
    m = CLIPVisionModelWithProjection(hf_cfg).eval()
    new = {"vision_model.embeddings.class_embedding": sd["visual.class_embedding"],
           "vision_model.embeddings.patch_embedding.weight": sd["visual.conv1.weight"],
           "vision_model.embeddings.position_embedding.weight": sd["visual.positional_embedding"],
           "vision_model.pre_layrnorm.weight": sd["visual.ln_pre.weight"], "vision_model.pre_layrnorm.bias": sd["visual.ln_pre.bias"],
           "vision_model.post_layernorm.weight": sd["visual.ln_post.weight"], "vision_model.post_layernorm.bias": sd["visual.ln_post.bias"],
           "visual_projection.weight": sd["visual.proj"].t().contiguous()}
    for i in range(cfg.layers):
        s, d = f"visual.transformer.resblocks.{i}.", f"vision_model.encoder.layers.{i}."
        for n, ww, bb in zip(("q_proj", "k_proj", "v_proj"), sd[s + "attn.in_proj_weight"].chunk(3, 0), sd[s + "attn.in_proj_bias"].chunk(3, 0)):
            new[d + f"self_attn.{n}.weight"], new[d + f"self_attn.{n}.bias"] = ww, bb
        for a, b in (("attn.out_proj", "self_attn.out_proj"), ("ln_1", "layer_norm1"), ("ln_2", "layer_norm2"), ("mlp.c_fc", "mlp.fc1"),
                     ("mlp.c_proj", "mlp.fc2")):
            new[d + b + ".weight"], new[d + b + ".bias"] = sd[s + a + ".weight"], sd[s + a + ".bias"]
    missing, unexpected = m.load_state_dict({k: v.float() for k, v in new.items()}, strict=False)
    missing = [k for k in missing if "position_ids" not in k]
    assert not missing and not unexpected, (missing, unexpected)
    return m


def hf_text_model(sd: dict, cfg):
    """``CLIPTextModelWithProjection`` of the TextConfig `cfg` (its act) holding `sd`; eos_token_id = 2 pools at the argmax id like CLIP"""
    from transformers import CLIPTextConfig, CLIPTextModelWithProjection
    w = cfg.width
    hcfg = CLIPTextConfig(vocab_size=cfg.vocab_size, hidden_size=w, intermediate_size=4 * w, num_hidden_layers=cfg.layers,
                          num_attention_heads=cfg.heads, max_position_embeddings=cfg.context_length, hidden_act=cfg.act,
                          projection_dim=cfg.output_dim, layer_norm_eps=1e-5, eos_token_id=2, attn_implementation="eager")
    m = CLIPTextModelWithProjection(hcfg).eval()
    hk = {"text_model.embeddings.token_embedding.weight": sd["token_embedding.weight"],
          "text_model.embeddings.position_embedding.weight": sd["positional_embedding"],
          "text_model.final_layer_norm.weight": sd["ln_final.weight"], "text_model.final_layer_norm.bias": sd["ln_final.bias"],
          "text_projection.weight": sd["text_projection"].t()}
    for i in range(cfg.layers):
        p, q = f"transformer.resblocks.{i}.", f"text_model.encoder.layers.{i}."
        for name, t, b in zip("qkv", sd[p + "attn.in_proj_weight"].split(w), sd[p + "attn.in_proj_bias"].split(w)):
            hk[q + f"self_attn.{name}_proj.weight"], hk[q + f"self_attn.{name}_proj.bias"] = t, b
        for src, dst in (("attn.out_proj", "self_attn.out_proj"), ("ln_1", "layer_norm1"), ("ln_2", "layer_norm2"), ("mlp.c_fc", "mlp.fc1"),
                         ("mlp.c_proj", "mlp.fc2")):
            hk[q + dst + ".weight"], hk[q + dst + ".bias"] = sd[p + src + ".weight"], sd[p + src + ".bias"]
    missing, unexpected = m.load_state_dict({k: v.float() for k, v in hk.items()}, strict=False)
    assert not unexpected and all("position_ids" in k for k in missing), (missing, unexpected)
    return m


# ---------------------------------------------------------------- float64 references of the new kernel bits
def gelu_f64(u):
    u = u.double()
    return 0.5 * u * (1 + th.erf(u / math.sqrt(2)))


def gelu_grad_f64(u):
    u = u.double()
    return 0.5 * (1 + th.erf(u / math.sqrt(2))) + u * th.exp(-0.5 * u * u) / math.sqrt(2 * math.pi)


# ---------------------------------------------------------------- plan interpreter
class OpenClipInterp(TextInterp):
    """TextInterp plus QGELU_FWD flags 1 and CONV flags 8 (fp32 math, fp16 where the kernels store fp16)"""

    def op_QGELU_FWD(self, op):
        if not op.flags & 1:
            return super().op_QGELU_FWD(op)
        u = self.flat(op.p[0], op.i[0]).float()
        self.flat(op.p[1], op.i[0]).copy_(F.gelu(u))

    def op_CONV(self, op):
        if not op.flags & 8:
            return super().op_CONV(op)
        assert not op.flags & 4 and op.p[2] is None and op.p[3] is not None and op.i[6] == 1, "CONV flags 8: a 1x1 dgrad with a res operand"
        NB, H, W, Cin, Cout, Npad = op.i[:6]
        A = self.V(op.p[0], (NB, H, W, Cin), (*op.i[7:10], 1)).float()
        Wp = self.V(op.p[1], (Npad, Cin), (Cin, 1)).float()[:Cout]
        u = self.V(op.p[3], (NB, H, W, Cout), (*op.i[13:16], 1)).float()
        self.V(op.p[4], (NB, H, W, Cout), (*op.i[10:13], 1)).copy_((A @ Wp.t()) * gelu_grad_f64(u).float())
