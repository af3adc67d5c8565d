"""CLIP ``ModifiedResNet`` towers (RN50, RN101, RN50x4, RN50x16: the other `clip_model_name`s of cgd/clip_util.py:17) as an op list on the same kernels
as the ViT tower: every layer is the wgmma conv (BatchNorm folded into weights and bias at build time -- the reference runs the
tower in eval mode, cgd/clip_util.py:64), ReLU, 2x2 average pooling, the small-T attention kernel for AttentionPool2d.

Two layout tricks keep it on the existing kernels:
* the stem's 3x3 **stride-2** conv runs as a stride-1 3x3 conv over the space-to-depth image: the cutout kernel already writes
  cutouts in "patch order" ``[n, g*g, (c, ky, kx)]`` (that is how the ViT's patch conv became a GEMM); with patch size 2 that IS the
  2x2 space-to-depth tensor ``[n, 112, 112, 12 -> 64]``, and the stride-2 taps (a - 1 in {-1, 0, +1} of pixel row 2i) land on block
  offsets {-1, 0} with in-block rows {1, 0, 1} -- a 3x3 kernel over blocks whose +1 taps are zero (`stem_s2d_weight`).
* widths that are not multiples of 64 (the stem's 32 channels; the 40 / 80 / 160-wide layers of RN50x4, the 48 / 96-wide layers of
  RN50x16) are zero-padded to the next multiple on the host (`_conv_bn`: weight rows / columns and the folded bias), so activations stay
  multiples of the 64-channel TMA K-slice; the padded outputs are relu(0 * x + 0) = 0 and their gradients meet zero weight columns.

[3P] clip/model.py (clip-anytorch 2.6.0) is not in /root/reference: restated from the published architecture (oracle/clip_rn.py,
parity unpinned, RN50 = 38,316,896 visual parameters).
"""
from __future__ import annotations

from dataclasses import dataclass

import torch as th

from .plan import Act, Plan, pack_conv


@dataclass
class RNConfig:
    layers: tuple = (3, 4, 6, 3)
    output_dim: int = 1024
    input_resolution: int = 224
    width: int = 64
    patch_size: int = 2  # space-to-depth factor of the stride-2 stem conv (what the engine asks the cutout kernel for)
    kpad: int = 64       # 3 * 2 * 2 = 12 values per block, padded to one 64-channel K-slice

    @property
    def heads(self):
        return self.width * 32 // 64

    @property
    def embed_dim(self):
        return self.width * 32

    @property
    def grid(self):
        return self.input_resolution // self.patch_size

    @property
    def tokens(self):
        return (self.input_resolution // 32) ** 2 + 1


RN_CONFIGS = {"RN50": RNConfig((3, 4, 6, 3), 1024, 224, 64), "RN101": RNConfig((3, 4, 23, 3), 512, 224, 64),
              "RN50x4": RNConfig((4, 6, 10, 6), 640, 288, 80), "RN50x16": RNConfig((6, 8, 18, 8), 768, 384, 96)}


def ceil64(c: int) -> int:
    return -(-c // 64) * 64


def rn_config_from_state_dict(sd: dict) -> RNConfig:
    width = sd["visual.layer1.0.conv1.weight"].shape[0]
    layers = tuple(len({k.split(".")[2] for k in sd if k.startswith(f"visual.layer{i}.")}) for i in (1, 2, 3, 4))
    spacial = int(round((sd["visual.attnpool.positional_embedding"].shape[0] - 1) ** 0.5))
    return RNConfig(layers, sd["visual.attnpool.c_proj.weight"].shape[0], spacial * 32, width)


def fold_bn(w: th.Tensor, bn: dict, eps: float = 1e-5):
    """eval-mode BatchNorm2d after a bias-free conv: (w * s, beta - mean * s), s = gamma / sqrt(var + eps)"""
    s = bn["weight"].float() / th.sqrt(bn["running_var"].float() + eps)
    return w.float() * s.view(-1, 1, 1, 1), bn["bias"].float() - bn["running_mean"].float() * s


def stem_s2d_weight(w: th.Tensor) -> th.Tensor:
    """[Co, 3, 3, 3] stride-2 pad-1 kernel -> [Co, 12, 3, 3] stride-1 pad-1 kernel over the 2x2 space-to-depth image whose channels are
    ordered (c, ky, kx).  Output pixel i reads input rows 2i + a - 1: a = 0 -> block i-1, in-block row 1; a = 1 -> block i, row 0;
    a = 2 -> block i, row 1.  Block offset -1 / 0 is tap 0 / 1 of the new kernel; tap 2 (offset +1) stays zero."""
    co = w.shape[0]
    out = th.zeros(co, 12, 3, 3)
    place = {0: (0, 1), 1: (1, 0), 2: (1, 1)}  # a -> (tap index, in-block position)
    for a, (ta, ky) in place.items():
        for b, (tb, kx) in place.items():
            for c in range(3):
                out[:, c * 4 + ky * 2 + kx, ta, tb] = w[:, c, a, b]
    return out


def _pad_channels(w: th.Tensor, b: th.Tensor, cout: int, cin: int):
    wp = th.zeros(cout, cin, *w.shape[2:])
    wp[:w.shape[0], :w.shape[1]] = w
    bp = th.zeros(cout)
    bp[:b.shape[0]] = b
    return wp, bp


class RNB200:
    """encode_image for n = cutn*B cutouts with a ModifiedResNet tower; same surface as ``vit.ViTB200``: ``patches`` (fp16
    [n, grid^2, kpad], the space-to-depth cutouts) in, ``embeds`` (fp32 [n, D]) out, ``d_embeds`` -> ``d_patches`` backward."""

    def __init__(self, cfg: RNConfig, state_dict: dict, n_images: int, device="cuda", conv_impl: int = 0, build_backward=True,
                 plan: Plan = None, parts: int = 1, suffix: str = "", share: "RNB200" = None):
        self.cfg, self.n, self.parts = cfg, n_images, 1
        self.sd = state_dict
        self.own_plan = plan is None
        self.plan = plan or Plan(conv_impl=conv_impl)
        self.suffix = suffix
        self._wcache, self._ccache = (share._wcache, share._ccache) if share is not None else ({}, {})
        self._build(build_backward)
        if self.own_plan:
            self.plan.finalize(device)
        del self.sd

    # ---- weights
    def _w(self, key):
        return self.sd["visual." + key].detach().float().cpu()

    def _bn(self, prefix):
        return {k: self._w(f"{prefix}.{k}") for k in ("weight", "bias", "running_mean", "running_var")}

    def _conv_bn(self, conv, bn, name, s2d=False):
        """packed (conv + folded BatchNorm), both channel counts zero-padded to multiples of 64; cached per tower family"""
        if name not in self._wcache:
            w, b = fold_bn(self._w(conv + ".weight"), self._bn(bn))
            if s2d:
                w = stem_s2d_weight(w)
            if w.shape[0] % 64 or w.shape[1] % 64:
                w, b = _pad_channels(w, b, ceil64(w.shape[0]), ceil64(w.shape[1]))
            self._wcache[name] = pack_conv(self.plan, w, b, need_bwd=True, name=name)
        return self._wcache[name]

    def _const(self, key, t=None):
        if key not in self._ccache:
            self._ccache[key] = self.plan.const(self._w(key) if t is None else t, "f", key)
        return self._ccache[key]

    def part_ranges(self, which: str):
        sfx = self.suffix
        return [(f"vit_{which}{sfx}", ("vit_bwd" if which == "fwd" else "vit_end") + sfx)]

    # ---- graph
    def _bottleneck(self, x: Act, prefix: str, stride: int, has_down: bool) -> Act:
        p = self.plan
        out = p.relu(p.conv(x, self._conv_bn(prefix + ".conv1", prefix + ".bn1", prefix + ".conv1"), name=prefix + ".conv1"), name=prefix + ".relu1")
        out = p.relu(p.conv(out, self._conv_bn(prefix + ".conv2", prefix + ".bn2", prefix + ".conv2"), name=prefix + ".conv2"), name=prefix + ".relu2")
        if stride > 1:
            out = p.pool2(out, name=prefix + ".avgpool")
        identity = x
        if has_down:
            if stride > 1:
                identity = p.pool2(x, name=prefix + ".downsample.-1")
            identity = p.conv(identity, self._conv_bn(prefix + ".downsample.0", prefix + ".downsample.1", prefix + ".downsample"),
                              name=prefix + ".downsample")
        out = p.conv(out, self._conv_bn(prefix + ".conv3", prefix + ".bn3", prefix + ".conv3"), res=identity, name=prefix + ".conv3")
        return p.relu(out, name=prefix + ".relu3")

    def _build(self, build_backward):
        p, cfg, n = self.plan, self.cfg, self.n
        g, kp, D, C = cfg.grid, cfg.kpad, cfg.output_dim, cfg.embed_dim
        assert cfg.width % 16 == 0 and cfg.input_resolution % 32 == 0 and kp == 64
        self.patches = p.new(n * g * g * kp, "h", "patches")
        self.embeds = p.new(n * D, "f", "embeds")
        self.d_embeds = p.new(n * D, "f", "d_embeds")
        saved_tape, p._tape = p._tape, []
        p.mark("vit_fwd" + self.suffix)
        x0 = Act(self.patches, 0, n, g, g, kp, kp)
        w = cfg.width
        h = p.relu(p.conv(x0, self._conv_bn("conv1", "bn1", "stem.conv1", s2d=True), name="stem.conv1"), name="stem.relu1")
        h = p.relu(p.conv(h, self._conv_bn("conv2", "bn2", "stem.conv2"), name="stem.conv2"), name="stem.relu2")
        h = p.relu(p.conv(h, self._conv_bn("conv3", "bn3", "stem.conv3"), name="stem.conv3"), name="stem.relu3")
        h = p.pool2(h, name="stem.avgpool")
        inplanes = w
        for li, (blocks, planes, stride) in enumerate(zip(cfg.layers, (w, 2 * w, 4 * w, 8 * w), (1, 2, 2, 2)), start=1):
            for bi in range(blocks):
                st = stride if bi == 0 else 1
                h = self._bottleneck(h, f"layer{li}.{bi}", st, st > 1 or inplanes != planes * 4)
                inplanes = planes * 4
        # AttentionPool2d: tokens, fused q/k/v projection, attention over all tokens (only the mean token's row is used), c_proj
        T = cfg.tokens
        tok = p.attnpool_embed(h, self._const("attnpool.positional_embedding"))
        if "attnpool.qkv" not in self._wcache:
            wq = th.cat([self._w(f"attnpool.{k}_proj.weight") for k in "qkv"])
            bq = th.cat([self._w(f"attnpool.{k}_proj.bias") for k in "qkv"])
            self._wcache["attnpool.qkv"] = pack_conv(p, wq, bq, need_bwd=True, name="attnpool.qkv")
        qkv = p.conv(tok, self._wcache["attnpool.qkv"], name="attnpool.qkv")
        a = p.attention(qkv, cfg.heads, T, n, legacy_order=False, name="attnpool.attn")
        c = p.gather_rows(a, n, T * a.ld, name="attnpool.query_row")
        wc = self._w("attnpool.c_proj.weight")  # [D, C]
        p.emit("LINEAR_SMALL", flags=4, i=[n, C, D, C, D],
               p=[(c.buf, 0), (self._const("attnpool.c_proj.weight"), 0), (self._const("attnpool.c_proj.bias"), 0), (self.embeds, 0)], tag="attnpool.c_proj")
        p.mark("vit_bwd" + self.suffix)
        if build_backward:
            dc = Act(p.new(n * C, "h", "d_query_row"), 0, 1, 1, n, C, C)
            p.emit("LINEAR_SMALL", flags=8, i=[n, D, C, D, C],
                   p=[(self.d_embeds, 0), (self._const("attnpool.c_proj.weight^T", wc.t().contiguous()), 0), None, (dc.buf, 0)], tag="d_attnpool.c_proj")
            p._grads[c.key()] = dc
            p.backward()
            d0 = p.grad_of(x0)
            assert d0 is not None and d0.eoff == 0 and d0.ld == kp
            self.d_patches = d0.buf
        else:
            self.d_patches = p.new(n * g * g * kp, "h", "d_patches")
        p._tape = saved_tape
        p.mark("vit_end" + self.suffix)

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
