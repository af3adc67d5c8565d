"""Parameter inventories (upstream state_dict key -> shape) and seeded synthetic weights.

Real checkpoints (``256x256_diffusion.pt``, CLIP ``ViT-B-32.pt``) load through ``torch.load`` exactly as in the reference
(cgd/script_util.py:316-317, cgd/clip_util.py:47-69) and are handed to ``UNetB200`` / ``ViTB200`` as plain state_dicts.
There is no network here, so benchmarks and tests use seeded random weights in the same key layout (timing is
value-independent).  Upstream zero-initialises every ResBlock ``out_layers.3``, attention ``proj_out`` and ``out.2``;
those are initialised non-zero here or the network would be trivially zero (SURVEY.md 8c).
"""
from __future__ import annotations

import math

import torch as th

from .unet import UNetConfig, topology
from .vit import ViTConfig


def unet_param_shapes(cfg: UNetConfig) -> dict:
    mc = cfg.model_channels
    ted = 4 * mc
    sh = {"time_embed.0.weight": (ted, mc), "time_embed.0.bias": (ted,), "time_embed.2.weight": (ted, ted), "time_embed.2.bias": (ted,)}
    if cfg.class_cond:
        sh["label_emb.weight"] = (cfg.num_classes, ted)
    ch0 = int(cfg.channel_mult[0] * mc)
    sh["input_blocks.0.0.weight"] = (ch0, cfg.in_channels, 3, 3)
    sh["input_blocks.0.0.bias"] = (ch0,)

    def res(prefix, cin, cout):
        sh[prefix + ".in_layers.0.weight"] = (cin,)
        sh[prefix + ".in_layers.0.bias"] = (cin,)
        sh[prefix + ".in_layers.2.weight"] = (cout, cin, 3, 3)
        sh[prefix + ".in_layers.2.bias"] = (cout,)
        sh[prefix + ".emb_layers.1.weight"] = (2 * cout, ted)
        sh[prefix + ".emb_layers.1.bias"] = (2 * cout,)
        sh[prefix + ".out_layers.0.weight"] = (cout,)
        sh[prefix + ".out_layers.0.bias"] = (cout,)
        sh[prefix + ".out_layers.3.weight"] = (cout, cout, 3, 3)
        sh[prefix + ".out_layers.3.bias"] = (cout,)
        if cin != cout:
            sh[prefix + ".skip_connection.weight"] = (cout, cin, 1, 1)
            sh[prefix + ".skip_connection.bias"] = (cout,)

    def attn(prefix, c):
        sh[prefix + ".norm.weight"] = (c,)
        sh[prefix + ".norm.bias"] = (c,)
        sh[prefix + ".qkv.weight"] = (3 * c, c, 1)
        sh[prefix + ".qkv.bias"] = (3 * c,)
        sh[prefix + ".proj_out.weight"] = (c, c, 1)
        sh[prefix + ".proj_out.bias"] = (c,)

    blocks_in, mid_ch, blocks_out = topology(cfg)
    for b in blocks_in:
        res(b["prefix"] + ".0", b["cin"], b["cout"])
        if b["attn"]:
            attn(b["prefix"] + ".1", b["cout"])
    res("middle_block.0", mid_ch, mid_ch)
    attn("middle_block.1", mid_ch)
    res("middle_block.2", mid_ch, mid_ch)
    for b in blocks_out:
        res(b["prefix"] + ".0", b["cin"], b["cout"])
        if b["attn"]:
            attn(b["prefix"] + ".1", b["cout"])
        if b["up"]:
            res(b["prefix"] + (".2" if b["attn"] else ".1"), b["cout"], b["cout"])
    sh["out.0.weight"] = (ch0,)
    sh["out.0.bias"] = (ch0,)
    sh["out.2.weight"] = (cfg.out_channels, ch0, 3, 3)
    sh["out.2.bias"] = (cfg.out_channels,)
    return sh


def vit_param_shapes(cfg: ViTConfig) -> dict:
    w, D = cfg.width, cfg.output_dim
    sh = {"visual.conv1.weight": (w, 3, cfg.patch_size, cfg.patch_size), "visual.class_embedding": (w,),
          "visual.positional_embedding": (cfg.tokens, w), "visual.ln_pre.weight": (w,), "visual.ln_pre.bias": (w,)}
    for i in range(cfg.layers):
        p = f"visual.transformer.resblocks.{i}"
        sh.update({p + ".attn.in_proj_weight": (3 * w, w), p + ".attn.in_proj_bias": (3 * w,), p + ".attn.out_proj.weight": (w, w),
                   p + ".attn.out_proj.bias": (w,), p + ".ln_1.weight": (w,), p + ".ln_1.bias": (w,), p + ".mlp.c_fc.weight": (4 * w, w),
                   p + ".mlp.c_fc.bias": (4 * w,), p + ".mlp.c_proj.weight": (w, 4 * w), p + ".mlp.c_proj.bias": (w,),
                   p + ".ln_2.weight": (w,), p + ".ln_2.bias": (w,)})
    sh.update({"visual.ln_post.weight": (w,), "visual.ln_post.bias": (w,), "visual.proj": (w, D)})
    return sh


def text_param_shapes(cfg) -> dict:
    """CLIP text tower (``text.TextConfig``) in upstream key layout: the keys of a full CLIP state_dict outside ``visual.*``"""
    w = cfg.width
    sh = {"token_embedding.weight": (cfg.vocab_size, w), "positional_embedding": (cfg.context_length, w)}
    for i in range(cfg.layers):
        p = f"transformer.resblocks.{i}"
        sh.update({p + ".attn.in_proj_weight": (3 * w, w), p + ".attn.in_proj_bias": (3 * w,), p + ".attn.out_proj.weight": (w, w),
                   p + ".attn.out_proj.bias": (w,), p + ".ln_1.weight": (w,), p + ".ln_1.bias": (w,), p + ".mlp.c_fc.weight": (4 * w, w),
                   p + ".mlp.c_fc.bias": (4 * w,), p + ".mlp.c_proj.weight": (w, 4 * w), p + ".mlp.c_proj.bias": (w,),
                   p + ".ln_2.weight": (w,), p + ".ln_2.bias": (w,)})
    sh.update({"ln_final.weight": (w,), "ln_final.bias": (w,), "text_projection": (w, cfg.output_dim)})
    return sh


def rn_param_shapes(cfg) -> dict:
    """CLIP ModifiedResNet visual tower ([3P] clip/model.py) in upstream key layout, BatchNorm buffers included"""
    w = cfg.width
    sh = {}

    def conv_bn(conv, bn, cout, cin, k):
        sh[conv + ".weight"] = (cout, cin, k, k)
        for suffix in ("weight", "bias", "running_mean", "running_var"):
            sh[f"{bn}.{suffix}"] = (cout,)

    conv_bn("visual.conv1", "visual.bn1", w // 2, 3, 3)
    conv_bn("visual.conv2", "visual.bn2", w // 2, w // 2, 3)
    conv_bn("visual.conv3", "visual.bn3", w, w // 2, 3)
    inplanes = w
    for li, (blocks, planes, stride) in enumerate(zip(cfg.layers, (w, 2 * w, 4 * w, 8 * w), (1, 2, 2, 2)), start=1):
        for bi in range(blocks):
            pre = f"visual.layer{li}.{bi}"
            st = stride if bi == 0 else 1
            conv_bn(pre + ".conv1", pre + ".bn1", planes, inplanes, 1)
            conv_bn(pre + ".conv2", pre + ".bn2", planes, planes, 3)
            conv_bn(pre + ".conv3", pre + ".bn3", planes * 4, planes, 1)
            if st > 1 or inplanes != planes * 4:
                conv_bn(pre + ".downsample.0", pre + ".downsample.1", planes * 4, inplanes, 1)
            inplanes = planes * 4
    C = cfg.embed_dim
    sh["visual.attnpool.positional_embedding"] = (cfg.tokens, C)
    for k in "kqv":
        sh[f"visual.attnpool.{k}_proj.weight"] = (C, C)
        sh[f"visual.attnpool.{k}_proj.bias"] = (C,)
    sh["visual.attnpool.c_proj.weight"] = (cfg.output_dim, C)
    sh["visual.attnpool.c_proj.bias"] = (cfg.output_dim,)
    return sh


def seeded_rn_state_dict(cfg, seed: int = 77) -> dict:
    """He-initialised convs (the last conv of every block damped so that 16 residual additions keep O(1) activations), BatchNorm with
    non-trivial running statistics"""
    g = th.Generator().manual_seed(seed)
    sd = {}
    for name, shape in rn_param_shapes(cfg).items():
        if name.endswith("running_mean"):
            t = th.randn(shape, generator=g) * 0.1
        elif name.endswith("running_var"):
            t = 1.0 + 0.2 * th.rand(shape, generator=g)
        elif name.endswith("positional_embedding"):
            t = th.randn(shape, generator=g) * shape[1] ** -0.5
        elif len(shape) >= 2:
            gain = 0.25 if name.endswith("conv3.weight") else 1.0
            t = th.randn(shape, generator=g) * gain * (2.0 / math.prod(shape[1:])) ** 0.5
        elif name.endswith("bias"):
            t = th.randn(shape, generator=g) * 0.05
        else:
            t = 1.0 + 0.1 * th.randn(shape, generator=g)
        sd[name] = t
    return sd


def lpips_param_shapes() -> dict:
    """lpips.LPIPS(net='vgg') v0.1: ``net.sliceK.<vgg16.features index>.{weight,bias}`` + ``linK.model.1.weight`` (SURVEY.md A.4)"""
    from .lpips import CHANNELS, SLICES
    sh, cin = {}, 3
    for k, idxs in enumerate(SLICES):
        for i in idxs:
            sh[f"net.slice{k + 1}.{i}.weight"] = (CHANNELS[k], cin, 3, 3)
            sh[f"net.slice{k + 1}.{i}.bias"] = (CHANNELS[k],)
            cin = CHANNELS[k]
        sh[f"lin{k}.model.1.weight"] = (1, CHANNELS[k], 1, 1)
    return sh


def seeded_lpips_state_dict(seed: int = 77) -> dict:
    """synthetic LPIPS weights: He-initialised convs (activations stay O(1) through 13 ReLU layers), non-negative lin weights"""
    g = th.Generator().manual_seed(seed)
    sd = {}
    for name, shape in lpips_param_shapes().items():
        if name.startswith("lin"):
            sd[name] = th.rand(shape, generator=g) * 0.2
        elif name.endswith("weight"):
            sd[name] = th.randn(shape, generator=g) * (2.0 / (shape[1] * 9)) ** 0.5
        else:
            sd[name] = th.randn(shape, generator=g) * 0.05
    return sd


def seeded_state_dict(shapes: dict, seed: int = 1234) -> dict:
    """fp16-range-safe synthetic weights: conv/linear N(0, 1/fan_in), biases N(0, 0.02), norm gains 1 + N(0, 0.1),
    embeddings N(0, 0.5) (SURVEY.md 8d)."""
    g = th.Generator().manual_seed(seed)
    sd = {}
    for name, shape in shapes.items():
        if name.endswith("label_emb.weight"):
            t = th.randn(shape, generator=g) * 0.5
        elif name.endswith("positional_embedding") or name.endswith("visual.proj"):
            t = th.randn(shape, generator=g) * shape[0] ** -0.5
        elif len(shape) >= 2:
            t = th.randn(shape, generator=g) * math.sqrt(1.0 / math.prod(shape[1:]))
        elif name.endswith("bias"):
            t = th.randn(shape, generator=g) * 0.02
        elif name.endswith("weight"):
            t = 1.0 + 0.1 * th.randn(shape, generator=g)
        else:
            t = th.randn(shape, generator=g) * 0.1
        sd[name] = t
    return sd
