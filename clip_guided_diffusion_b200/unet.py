"""ADM UNet (guided-diffusion ``UNetModel``) as an H100 op plan: forward and input-gradient backward.

Replaces [3P] ``guided_diffusion.unet.UNetModel.forward`` and the autograd walk of it that the reference triggers
with ``th.autograd.grad(loss, x)`` (cgd/cgd.py:228); constructed from the same flags the reference merges at
cgd/script_util.py:305-316 and from a state_dict in upstream key layout (SURVEY.md Appendix A.1, A.5), so real
checkpoints load unchanged.  All convolutions (3x3, 1x1, qkv / proj) run on the wgmma implicit-GEMM kernel;
activations are pixel-major fp16 like the reference's ``convert_to_fp16`` trunk (cgd/script_util.py:322-323);
GroupNorm statistics, the timestep-embedding MLP and all accumulation are fp32.
"""
from __future__ import annotations

from dataclasses import dataclass

import torch as th

from .plan import Act, ConvW, Plan, pack_conv


@dataclass
class UNetConfig:
    """Shape-defining flags (data/diffusion_model_flags.py merged over guided-diffusion defaults)."""
    image_size: int = 256
    model_channels: int = 256
    num_res_blocks: int = 2
    channel_mult: tuple = (1, 1, 2, 2, 4, 4)
    attention_resolutions: tuple = (32, 16, 8)
    num_heads: int = 4
    num_head_channels: int = 64
    class_cond: bool = True
    num_classes: int = 1000
    use_new_attention_order: bool = False
    in_channels: int = 3
    out_channels: int = 6
    rescale_timesteps: bool = False
    noise_schedule: str = "linear"

    @property
    def attention_ds(self):
        return tuple(self.image_size // int(r) for r in self.attention_resolutions)


def config_for(image_size: int, class_cond: bool = True) -> UNetConfig:
    """The four published checkpoints (data/diffusion_model_flags.py:1-120)."""
    mult = {512: (0.5, 1, 1, 2, 2, 4, 4), 256: (1, 1, 2, 2, 4, 4), 128: (1, 1, 2, 3, 4), 64: (1, 2, 3, 4)}[image_size]
    base = dict(image_size=image_size, class_cond=class_cond, channel_mult=mult)
    if image_size == 64:
        return UNetConfig(model_channels=192, num_res_blocks=3, use_new_attention_order=True, noise_schedule="cosine", **base)
    if image_size == 128:
        return UNetConfig(model_channels=256, num_heads=4, num_head_channels=-1, **base)
    if image_size == 512:
        return UNetConfig(model_channels=256, rescale_timesteps=True, **base)
    return UNetConfig(model_channels=256, **base)


def topology(cfg: UNetConfig):
    """Block list of the network (same walk as guided_diffusion.unet.UNetModel.__init__): input blocks after the stem,
    the middle width, output blocks (with the width of the skip each one concatenates)."""
    mc = cfg.model_channels
    blocks_in, blocks_out = [], []
    ch = int(cfg.channel_mult[0] * mc)
    skip_chs = [ch]
    ds = 1
    idx = 1
    for level, mult in enumerate(cfg.channel_mult):
        for _ in range(cfg.num_res_blocks):
            cout = int(mult * mc)
            blocks_in.append(dict(prefix=f"input_blocks.{idx}", cin=ch, cout=cout, attn=ds in cfg.attention_ds, down=False))
            ch = cout
            skip_chs.append(ch)
            idx += 1
        if level != len(cfg.channel_mult) - 1:
            blocks_in.append(dict(prefix=f"input_blocks.{idx}", cin=ch, cout=ch, attn=False, down=True))
            skip_chs.append(ch)
            ds *= 2
            idx += 1
    mid_ch = ch
    idx = 0
    for level, mult in list(enumerate(cfg.channel_mult))[::-1]:
        for i in range(cfg.num_res_blocks + 1):
            ich = skip_chs.pop()
            cout = int(mc * mult)
            up = bool(level and i == cfg.num_res_blocks)
            blocks_out.append(dict(prefix=f"output_blocks.{idx}", cin=ch + ich, cout=cout, attn=ds in cfg.attention_ds, up=up, ich=ich))
            ch = cout
            if up:
                ds //= 2
            idx += 1
    return blocks_in, mid_ch, blocks_out


IN_PAD = 64  # image channels are zero-padded to one 64-channel K slice for the stem conv / head dgrad


class UNetB200:
    """Drop-in for the reference's ``gd_model``: ``model(x, timesteps, y) -> [B, 6, H, W]`` plus
    ``backward_input()`` (what autograd does for the reference).  One instance is bound to one (batch, H, W)."""

    def __init__(self, cfg: UNetConfig, state_dict: dict, batch: int, height: int = None, width: int = None, device="cuda",
                 conv_impl: int = 0, seed_scale: float = 1.0, build_backward: bool = True, plan: Plan = None):
        self.cfg = cfg
        self.B = batch
        self.H = height or cfg.image_size
        self.W = width or cfg.image_size
        # every level but the last halves the image and the output path doubles it back onto the skip connection: sizes that are not a
        # multiple of 2^(levels - 1) (image_size + height_offset / width_offset, cgd/cgd.py:244) make the reference fail in th.cat of
        # the first mismatching skip; said here, before anything is packed
        step = 2 ** (len(cfg.channel_mult) - 1)
        if self.H % step or self.W % step or self.H <= 0 or self.W <= 0:
            raise ValueError(f"image {self.H}x{self.W}: height and width must be positive multiples of {step} for this {len(cfg.channel_mult)}-level UNet "
                             "(image_size + height_offset / width_offset)")
        self.num_classes = cfg.num_classes if cfg.class_cond else None
        self.dtype = th.float16
        self.seed_scale = float(seed_scale)
        self.sd = {k: v for k, v in state_dict.items()}
        self.own_plan = plan is None
        self.plan = plan or Plan(conv_impl=conv_impl)
        self._build(build_backward)
        if self.own_plan:
            self.plan.finalize(device)
        self.device = th.device(device)
        del self.sd

    # ------------------------------------------------------------------ helpers
    def _w(self, key):
        return self.sd[key].detach().float().cpu()

    def _const(self, key):
        return self.plan.const(self._w(key), "f", key)

    def _conv_w(self, prefix, need_bwd=True, cin_pad=None) -> ConvW:
        return pack_conv(self.plan, self._w(prefix + ".weight"), self._w(prefix + ".bias"), need_bwd=need_bwd, cin_pad=cin_pad, name=prefix)

    def _resblock_prepare(self, prefix, cout):
        """Register one ResBlock's emb_layers Linear (e = Linear(SiLU(emb)) -> [B, 2*Cout] fp32, x-independent: no backward).
        All of them are evaluated by ONE weight-streaming launch in the prelude (`_emit_emb_layers`): ~30 launches of 8 MB fp32
        each (0.43 ms per step) become one pass over the concatenated fp16 weights (the reference's emb_layers are fp16 too:
        convert_to_fp16 covers the ResBlocks, cgd/script_util.py:322-323)."""
        cout2 = 2 * cout
        e = self.plan.new(self.B * cout2, "f", prefix + ".emb_layers.1_e")
        self._emb_jobs.append((prefix + ".emb_layers.1", cout2, e))
        return e

    def _emit_emb_layers(self):
        p = self.plan
        ted = 4 * self.cfg.model_channels
        W = th.cat([self._w(k + ".weight") for k, _, _ in self._emb_jobs], dim=0)
        b = th.cat([self._w(k + ".bias") for k, _, _ in self._emb_jobs], dim=0)
        base = self._emb_jobs[0][2].off
        tab = []
        for _, cout2, e in self._emb_jobs:
            assert (e.off - base) % 4 == 0
            off = (e.off - base) // 4
            tab += [[off + c, cout2] for c in range(cout2)]
        n_total = W.shape[0]
        p.emit("LINEAR_SMALL", flags=1 | 16, i=[self.B, ted, n_total, ted, n_total],
               p=[(self.emb, 0), (p.const(W, "h", "emb_layers.W"), 0), (p.const(b, "f", "emb_layers.b"), 0), (self._emb_jobs[0][2], 0),
                  (p.const(th.tensor(tab, dtype=th.int32), "i32", "emb_layers.scatter"), 0)], tag="emb_layers (all ResBlocks)")

    def _resblock(self, x: Act, prefix: str, cout: int, e_buf, up=False, down=False, out: Act = None) -> Act:
        p = self.plan
        h = p.group_norm(x, self._const(prefix + ".in_layers.0.weight"), self._const(prefix + ".in_layers.0.bias"), silu=True,
                         name=prefix + ".in_gn")
        xs = x
        if up:
            h, xs = p.up2(h, prefix + ".h_up"), p.up2(x, prefix + ".x_up")
        elif down:
            h, xs = p.pool2(h, prefix + ".h_down"), p.pool2(x, prefix + ".x_down")
        h = p.conv(h, self._conv_w(prefix + ".in_layers.2"), name=prefix + ".conv1")
        h = p.group_norm(h, self._const(prefix + ".out_layers.0.weight"), self._const(prefix + ".out_layers.0.bias"), emb=(e_buf, 0),
                         silu=True, name=prefix + ".out_gn")
        if x.C != cout:
            xs = p.conv(xs, self._conv_w(prefix + ".skip_connection"), name=prefix + ".skip")
        return p.conv(h, self._conv_w(prefix + ".out_layers.3"), res=xs, out=out, name=prefix + ".conv2")

    def _attnblock(self, x: Act, prefix: str, out: Act = None) -> Act:
        p, cfg = self.plan, self.cfg
        C = x.C
        heads = cfg.num_heads if cfg.num_head_channels == -1 else C // cfg.num_head_channels
        xn = p.group_norm(x, self._const(prefix + ".norm.weight"), self._const(prefix + ".norm.bias"), silu=False, name=prefix + ".norm")
        qkv = p.conv(xn, self._conv_w(prefix + ".qkv"), name=prefix + ".qkv")
        a = p.attention(qkv, heads, x.HW, x.N, legacy_order=not cfg.use_new_attention_order, name=prefix + ".attn")
        return p.conv(a, self._conv_w(prefix + ".proj_out"), res=x, out=out, name=prefix + ".proj")

    # ------------------------------------------------------------------ whole network
    def _build(self, build_backward: bool):
        p, cfg, B, H, W = self.plan, self.cfg, self.B, self.H, self.W
        mc = cfg.model_channels
        ted = 4 * mc
        # ---- I/O buffers (fp32 NCHW at the boundary, like the reference's tensors)
        self.x_in = p.new(B * 3 * H * W, "f", "x")
        self.t_in = p.new(B, "f", "t")
        self.y_in = p.new(B, "i64", "y")
        self.out = p.new(B * cfg.out_channels * H * W, "f", "model_out")
        self.seed = p.new(B * H * W * IN_PAD, "h", "d_out_seed")  # channels 0..5 written by the guidance kernel, rest stay 0
        self.dx = p.new(B * 3 * H * W, "f", "dx")

        # ---- prelude: timestep / class embedding and every ResBlock's scale-shift vector (x-independent)
        p.mark("unet_emb")
        te = p.new(B * mc, "f", "t_sin")
        p.emit("TIMESTEP_EMB", i=[B, mc], f=[1.0], p=[(self.t_in, 0), (te, 0)], tag="timestep_embedding")
        h1 = p.new(B * ted, "f", "te_h1")
        self.emb = p.new(B * ted, "f", "emb")
        p.emit("LINEAR_SMALL", i=[B, mc, ted, mc, ted], p=[(te, 0), (self._const("time_embed.0.weight"), 0), (self._const("time_embed.0.bias"), 0), (h1, 0)],
               tag="time_embed.0")
        p.emit("LINEAR_SMALL", flags=1, i=[B, ted, ted, ted, ted],
               p=[(h1, 0), (self._const("time_embed.2.weight"), 0), (self._const("time_embed.2.bias"), 0), (self.emb, 0)], tag="time_embed.2")
        if cfg.class_cond:
            p.emit("LABEL_ADD", i=[B, ted], p=[(self.emb, 0), (self._const("label_emb.weight"), 0), (self.y_in, 0)], tag="label_emb")

        blocks_in, mid_ch, blocks_out = topology(cfg)
        # scale-shift vectors (prelude ops must precede the trunk)
        self._emb_jobs = []
        for b in blocks_in:
            b["e"] = self._resblock_prepare(b["prefix"] + ".0", b["cout"])
        mid_e = [self._resblock_prepare("middle_block.0", mid_ch), self._resblock_prepare("middle_block.2", mid_ch)]
        for b in blocks_out:
            b["e"] = self._resblock_prepare(b["prefix"] + ".0", b["cout"])
            if b["up"]:
                b["e_up"] = self._resblock_prepare(b["prefix"] + (".2" if b["attn"] else ".1"), b["cout"])

        self._emit_emb_layers()

        # ---- forward trunk
        p.mark("unet_fwd")
        x0 = Act(p.new(B * H * W * IN_PAD, "h", "x_pm"), 0, B, H, W, IN_PAD, IN_PAD)
        p.emit("NCHW_TO_PM", i=[B, 3, H * W, IN_PAD], f=[1.0], p=[(self.x_in, 0), (x0.buf, 0)], tag="x->pixel-major")
        stem_w = self._conv_w("input_blocks.0.0", need_bwd=build_backward, cin_pad=IN_PAD)
        # torch.cat([h, hs.pop()], dim=1) of every output block without a copy: the concatenated tensor of output block k is
        # allocated when its skip half is produced on the way down; the stem / input-block convs write the skip half and the
        # preceding block writes the h half straight into it (TMA stores with the wide row stride), consumers read the halves as
        # strided views.  46 copy launches and 2 x 0.25 GB of traffic per step at 256x256 disappear.
        n_skips = len(blocks_in) + 1
        cats = [None] * len(blocks_out)

        def skip_slot(j, Hc, Wc):
            """storage of hs[j]: the skip half of the output block that will pop it"""
            k = n_skips - 1 - j
            bo = blocks_out[k]
            cats[k] = p.act(B, Hc, Wc, bo["cin"], bo["prefix"] + ".cat")
            return cats[k].cslice(bo["cin"] - bo["ich"], bo["cin"])

        def h_slot(k):
            """storage of the h half of output block k (None past the last block)"""
            if k >= len(blocks_out):
                return None
            bo = blocks_out[k]
            return cats[k].cslice(0, bo["cin"] - bo["ich"])

        h = p.conv(x0, ConvW(stem_w.fwd, stem_w.fwd_npad, None, 0, stem_w.bias, IN_PAD, stem_w.cout, 9), out=skip_slot(0, H, W), name="stem")
        stem_out = h
        hs = [h]
        for j, b in enumerate(blocks_in, start=1):
            Ho, Wo = (h.H // 2, h.W // 2) if b["down"] else (h.H, h.W)
            slot = skip_slot(j, Ho, Wo)
            h = self._resblock(h, b["prefix"] + ".0", b["cout"], b["e"], down=b["down"], out=None if b["attn"] else slot)
            if b["attn"]:
                h = self._attnblock(h, b["prefix"] + ".1", out=slot)
            hs.append(h)
        h = self._resblock(h, "middle_block.0", mid_ch, mid_e[0])
        h = self._attnblock(h, "middle_block.1")
        h = self._resblock(h, "middle_block.2", mid_ch, mid_e[1], out=h_slot(0))
        for k, b in enumerate(blocks_out):
            skip = hs.pop()
            assert h.buf is cats[k].buf and skip.buf is cats[k].buf and h.C + skip.C == cats[k].C
            p.concat_view(cats[k], h, skip)
            h = cats[k]
            nxt = h_slot(k + 1)
            last = "up" if b["up"] else ("attn" if b["attn"] else "res")
            h = self._resblock(h, b["prefix"] + ".0", b["cout"], b["e"], out=nxt if last == "res" else None)
            if b["attn"]:
                h = self._attnblock(h, b["prefix"] + ".1", out=nxt if last == "attn" else None)
            if b["up"]:
                h = self._resblock(h, b["prefix"] + (".2" if b["attn"] else ".1"), b["cout"], b["e_up"], up=True, out=nxt)
        hn = p.group_norm(h, self._const("out.0.weight"), self._const("out.0.bias"), silu=True, name="out.gn")
        head_w = self._conv_w("out.2", need_bwd=build_backward)
        HW = H * W
        oc = cfg.out_channels
        p._emit_conv(p._ap(hn), p._strides(hn), B, H, W, hn.C, head_w.fwd, head_w.fwd_npad, oc, 9, head_w.bias, None, None,
                     (self.out, 0), (oc * HW, W, 1), out_f32=True, out_sc=HW, tag="head")
        p.mark("unet_bwd")
        if not build_backward:
            p.mark("unet_end")
            return

        # ---- backward: head dgrad from the seed, reverse tape, stem dgrad to fp32 NCHW
        seed_act = Act(self.seed, 0, B, H, W, IN_PAD, IN_PAD)
        d_hn = p.act(B, H, W, hn.C, "d_head")
        p._emit_conv(p._ap(seed_act), p._strides(seed_act), B, H, W, IN_PAD, head_w.bwd, head_w.bwd_npad, hn.C, 9, None, None, None,
                     p._ap(d_hn), p._strides(d_hn), tag="d_head")
        p._grads[hn.key()] = d_hn
        p.backward()
        d_stem = p.grad_of(stem_out)
        assert d_stem is not None
        p._emit_conv(p._ap(d_stem), p._strides(d_stem), B, H, W, d_stem.C, stem_w.bwd, stem_w.bwd_npad, 3, 9, None, None, None,
                     (self.dx, 0), (3 * HW, W, 1), out_f32=True, out_sc=HW, tag="d_stem")
        p.mark("unet_end")

    # ------------------------------------------------------------------ run-time API
    def _v(self, buf, shape):
        return self.plan.view(buf, shape)

    def set_inputs(self, x: th.Tensor, timesteps: th.Tensor, y: th.Tensor = None):
        self._v(self.x_in, (self.B, 3, self.H, self.W)).copy_(x)
        self._v(self.t_in, (self.B,)).copy_(timesteps)
        if self.cfg.class_cond:
            assert y is not None, "class-conditional UNet needs y"
            self._v(self.y_in, (self.B,)).copy_(y)

    def run_forward(self):
        self.plan.run_range("unet_emb", "unet_bwd")

    def run_backward(self):
        self.plan.run_range("unet_bwd", "unet_end")

    @property
    def out_view(self):
        return self._v(self.out, (self.B, self.cfg.out_channels, self.H, self.W))

    @property
    def dx_view(self):
        return self._v(self.dx, (self.B, 3, self.H, self.W))

    @property
    def seed_view(self):
        return self._v(self.seed, (self.B, self.H * self.W, IN_PAD))

    def __call__(self, x, timesteps, y=None):
        """model(x, timesteps, y) -> [B, 6, H, W] fp32 (a view of the plan's output buffer, valid until the next call)."""
        self.set_inputs(x, timesteps, y)
        self.run_forward()
        return self.out_view

    forward = __call__

    def backward_input(self, d_out: th.Tensor = None) -> th.Tensor:
        """dL/dx for dL/d(model_out) = d_out [B, 6, H, W] (or the seed already written by the guidance kernel)."""
        if d_out is not None:
            sv = self.seed_view
            sv[:, :, :self.cfg.out_channels].copy_((d_out * self.seed_scale).reshape(self.B, self.cfg.out_channels, -1).permute(0, 2, 1))
        self.run_backward()
        return self.dx_view

    def parameters(self):  # guided-diffusion loops ask next(model.parameters()).device
        yield self.plan.arena

    def convert_to_fp16(self):  # cgd/script_util.py:322-323 -- the trunk is fp16 by construction
        return self

    def eval(self):
        return self

    def requires_grad_(self, flag=False):
        return self
