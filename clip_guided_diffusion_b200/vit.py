"""CLIP visual tower (``clip.model.VisionTransformer``) as an H100 op plan: encode_image forward and input gradient.

Replaces [3P] ``clip_model.encode_image`` (called at cgd/cgd.py:194) and its autograd backward (cgd/cgd.py:228).
Weights come from a state_dict in upstream key layout (``visual.*``, SURVEY.md Appendix A.3, A.5).  The input is
not an image tensor but the patch matrix that the cutout kernel writes directly in patch order, so the patch
"convolution" is a plain GEMM.  Linear layers run on the wgmma GEMM kernel with fp16 operands / fp32
accumulation (the reference's CUDA path loads CLIP in fp16, cgd/clip_util.py:64-65); LayerNorm statistics,
softmax and the final projection are fp32.
"""
from __future__ import annotations

from dataclasses import dataclass

import torch as th

from .plan import Act, Plan, pack_conv, _round_up


@dataclass
class ViTConfig:
    input_resolution: int = 224
    patch_size: int = 32
    width: int = 768
    layers: int = 12
    output_dim: int = 512

    @property
    def heads(self):
        return self.width // 64

    @property
    def grid(self):
        return self.input_resolution // self.patch_size

    @property
    def tokens(self):
        return self.grid ** 2 + 1

    @property
    def kpad(self):
        """patch vector length 3*P*P zero-padded to a multiple of 64 (TMA K slices)"""
        return _round_up(3 * self.patch_size ** 2, 64)


VIT_CONFIGS = {
    "ViT-B/32": ViTConfig(224, 32, 768, 12, 512),
    "ViT-B/16": ViTConfig(224, 16, 768, 12, 512),
    "ViT-L/14": ViTConfig(224, 14, 1024, 24, 768),
    "ViT-L/14@336px": ViTConfig(336, 14, 1024, 24, 768),  # in CLIP_MODEL_URLS (cgd/clip_util.py:28): 24 x 24 patches + class token = 577 tokens
}


def vit_config_from_state_dict(sd: dict) -> ViTConfig:
    w = sd["visual.conv1.weight"]
    width, _, ps, _ = w.shape
    tokens = sd["visual.positional_embedding"].shape[0]
    grid = int(round((tokens - 1) ** 0.5))
    layers = len({k.split(".")[3] for k in sd if k.startswith("visual.transformer.resblocks.")})
    return ViTConfig(grid * ps, ps, width, layers, sd["visual.proj"].shape[1])


class ViTB200:
    """encode_image for n = cutn*B cutouts.  ``patches`` (fp16 [n, grid^2, kpad]) is the plan's input buffer;
    ``embeds`` (fp32 [n, D]) its output; ``d_embeds`` -> ``d_patches`` the backward."""

    def __init__(self, cfg: ViTConfig, state_dict: dict, n_images: int, device="cuda", conv_impl: int = 0, build_backward=True,
                 plan: Plan = None, parts: int = 1, suffix: str = "", share: "ViTB200" = None):
        """parts > 1 builds `parts` independent op lists over equal slices of the image batch (shared packed weights, shared
        patches / embeds buffers) so that the engine can run them on parallel streams: at 16 cutouts every ViT GEMM occupies a
        fraction of the SMs for a latency-bound ~8 us, two half-batches side by side hide each other's latency."""
        self.cfg, self.n = cfg, n_images
        self.parts = parts if (parts > 1 and n_images % parts == 0) else 1
        self.sd = state_dict
        self.own_plan = plan is None
        self.plan = plan or Plan(conv_impl=conv_impl)
        # `share`: another tower on the same plan whose packed weights are reused (engines with several cutout counts:
        # progressive_cutout, cgd/cgd.py:167-175); `suffix` keeps the range marks of the towers apart
        self.suffix = suffix
        self._wcache, self._ccache = (share._wcache, share._ccache) if share is not None else ({}, {})
        self._build(build_backward)
        if self.own_plan:
            self.plan.finalize(device)
        del self.sd

    def _w(self, key):
        return self.sd["visual." + key].detach().float().cpu()

    def _const(self, key):
        if key not in self._ccache:
            self._ccache[key] = self.plan.const(self._w(key), "f", key)
        return self._ccache[key]

    def _pack(self, wkey, bkey, name, **kw):
        if name not in self._wcache:
            w = self._w(wkey)
            if kw.pop("flatten", False):
                w = w.reshape(w.shape[0], -1)
            self._wcache[name] = pack_conv(self.plan, w, self._w(bkey) if bkey else None, name=name, **kw)
        return self._wcache[name]

    def part_ranges(self, which: str):
        """[(mark_a, mark_b)] of the forward ("fwd") or backward ("bwd") op range of every part"""
        sfx = self.suffix
        names = [f"vit_{which}{sfx}"] + [f"vit_{which}_p{k}{sfx}" for k in range(1, self.parts)]
        ends = names[1:] + [("vit_bwd" if which == "fwd" else "vit_end") + sfx]
        return list(zip(names, ends))

    def _build(self, build_backward):
        p, cfg, n = self.plan, self.cfg, self.n
        D, kp, G2 = cfg.output_dim, cfg.kpad, cfg.grid ** 2
        self.patches = p.new(n * G2 * kp, "h", "patches")
        self.embeds = p.new(n * D, "f", "embeds")
        self.d_embeds = p.new(n * D, "f", "d_embeds")
        self.d_patches = p.new(n * G2 * kp, "h", "d_patches")
        nk = n // self.parts
        saved_tape, p._tape = p._tape, []
        tapes, heads = [], []
        for k in range(self.parts):
            p.mark(("vit_fwd" if k == 0 else f"vit_fwd_p{k}") + self.suffix)
            heads.append(self._build_forward(k, nk, build_backward))
            tapes.append(p._tape)
            p._tape = []
        p.mark("vit_bwd" + self.suffix)
        if build_backward:
            for k in range(self.parts):
                if k:
                    p.mark(f"vit_bwd_p{k}" + self.suffix)
                p._tape = tapes[k]
                self._build_backward(k, nk, *heads[k])
        p._tape = saved_tape
        p.mark("vit_end" + self.suffix)

    def _build_forward(self, k, n, build_backward):
        p, cfg = self.plan, self.cfg
        w, T, G2, D, kp = cfg.width, cfg.tokens, cfg.grid ** 2, cfg.output_dim, cfg.kpad
        rows = n * T
        # patch embedding: tok[n, 1+g, :] = patches[n, g, :] @ conv1^T   (no bias)
        wpatch = self._pack("conv1.weight", None, "conv1", need_bwd=build_backward, cin_pad=kp, flatten=True)
        tok = Act(p.new(rows * w, "h", "tok"), 0, 1, 1, rows, w, w)
        p._emit_conv((self.patches, k * n * G2 * kp), (G2 * kp, G2 * kp, kp), n, 1, G2, kp, wpatch.fwd, wpatch.fwd_npad, w, 1, None, None, None,
                     (tok.buf, w), (T * w, T * w, w), tag="patch_embed")
        p.emit("VIT_EMBED", i=[n, T, w], p=[(tok.buf, 0), (self._const("class_embedding"), 0), (self._const("positional_embedding"), 0)],
               tag="cls+pos")
        x = p.layer_norm(tok, self._const("ln_pre.weight"), self._const("ln_pre.bias"), name="ln_pre")
        for li in range(cfg.layers):
            pre = f"transformer.resblocks.{li}"
            y = p.layer_norm(x, self._const(pre + ".ln_1.weight"), self._const(pre + ".ln_1.bias"), name=pre + ".ln_1")
            qkv = p.conv(y, self._pack(pre + ".attn.in_proj_weight", pre + ".attn.in_proj_bias", pre + ".in_proj"), name=pre + ".qkv")
            a = p.attention(qkv, cfg.heads, T, n, legacy_order=False, name=pre + ".attn")
            x = p.conv(a, self._pack(pre + ".attn.out_proj.weight", pre + ".attn.out_proj.bias", pre + ".out_proj"), res=x, name=pre + ".out_proj")
            y = p.layer_norm(x, self._const(pre + ".ln_2.weight"), self._const(pre + ".ln_2.bias"), name=pre + ".ln_2")
            u = p.conv(y, self._pack(pre + ".mlp.c_fc.weight", pre + ".mlp.c_fc.bias", pre + ".c_fc"), name=pre + ".c_fc")
            g = p.quick_gelu(u, name=pre + ".gelu")
            x = p.conv(g, self._pack(pre + ".mlp.c_proj.weight", pre + ".mlp.c_proj.bias", pre + ".c_proj"), res=x, name=pre + ".c_proj")
        # ln_post on the class token of every image, then the fp32 projection
        c = p.layer_norm(x, self._const("ln_post.weight"), self._const("ln_post.bias"), rows=n, ldx=T * w, name="ln_post")
        if "proj^T" not in self._ccache:
            proj = self._w("proj")  # [w, D]
            self._ccache["proj^T"] = p.const(proj.t().contiguous(), "f", "proj^T")
            self._ccache["proj"] = p.const(proj.contiguous(), "f", "proj")
        p.emit("LINEAR_SMALL", flags=4, i=[n, w, D, w, D], p=[(c.buf, 0), (self._ccache["proj^T"], 0), None, (self.embeds, k * n * D)], tag="proj")
        return tok, c, wpatch

    def _build_backward(self, k, n, tok, c, wpatch):
        p, cfg = self.plan, self.cfg
        w, T, G2, D, kp = cfg.width, cfg.tokens, cfg.grid ** 2, cfg.output_dim, cfg.kpad
        dc = Act(p.new(n * w, "h", "d_cls"), 0, 1, 1, n, w, w)
        p.emit("LINEAR_SMALL", flags=8, i=[n, D, w, D, w], p=[(self.d_embeds, k * n * D), (self._ccache["proj"], 0), None, (dc.buf, 0)], tag="d_proj")
        p._grads[c.key()] = dc
        p.backward()
        d_tok = p.grad_of(tok)
        assert d_tok is not None and d_tok.ld == w
        # d_patches[n, g, :] = d_tok[n, 1+g, :] @ conv1
        p._emit_conv((d_tok.buf, d_tok.eoff + w), (T * w, T * w, w), n, 1, G2, w, wpatch.bwd, wpatch.bwd_npad, kp, 1, None, None, None,
                     (self.d_patches, k * n * G2 * kp), (G2 * kp, G2 * kp, kp), tag="d_patch_embed")

    # ---- run-time API (stand-alone use; the fused step drives the shared plan directly)
    def encode_patches(self, patches: th.Tensor = None) -> th.Tensor:
        if patches is not None:
            self.plan.view(self.patches, patches.shape).copy_(patches)
        self.plan.run_range("vit_fwd" + self.suffix, "vit_bwd" + self.suffix)
        return self.plan.view(self.embeds, (self.n, self.cfg.output_dim))

    def backward_patches(self, d_embeds: th.Tensor = None) -> th.Tensor:
        if d_embeds is not None:
            self.plan.view(self.d_embeds, d_embeds.shape).copy_(d_embeds)
        self.plan.run_range("vit_bwd" + self.suffix, "vit_end" + self.suffix)
        return self.plan.view(self.d_patches, (self.n, self.cfg.grid ** 2, self.cfg.kpad))
