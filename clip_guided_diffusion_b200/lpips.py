"""LPIPS-VGG16 perceptual loss against an init image, as an H100 op plan: value and gradient with respect to x_in.

Replaces [3P] ``lpips.LPIPS(net='vgg')`` as the reference uses it (cgd/cgd.py:147-148 lazy construction, 220-224
``lpips_vgg(x_in, init_tensor).sum() * init_scale`` inside the differentiated loss; SURVEY.md A.4, K21, section 8f row 3).  The
13 conv3x3 layers run on the wgmma implicit-GEMM kernel (forward and dgrad), ReLU / 2x2 max-pool / the per-tap normalise-diff-
lin-mean with its analytic gradient are the kernels of csrc/lpips.cu.  The init image's features are constant: they are
computed once by the same forward ops and stored channel-normalised.  State dict keys follow the upstream layout
(``net.sliceK.<vgg16.features index>.{weight,bias}``, ``linK.model.1.weight``).
"""
from __future__ import annotations

import torch as th

from .plan import Buf, Plan, pack_conv

SHIFT = (-0.030, -0.088, -0.188)
SCALE = (0.458, 0.448, 0.450)
SLICES = ((0, 2), (5, 7), (10, 12, 14), (17, 19, 21), (24, 26, 28))  # torchvision vgg16.features conv indices per LPIPS slice
CHANNELS = (64, 128, 256, 512, 512)
IN_PAD = 64


class LpipsB200:
    """loss[b] = LPIPS(x_in[b], init) ; g_dst += init_scale * d loss / d x_in.  ``x_src`` / ``g_dst`` are fp32 NCHW [B,3,H,W]
    buffers of the plan (the engine's blended x_in and its x_in-gradient accumulator)."""

    def __init__(self, state_dict: dict, batch: int, height: int, width: int, plan: Plan, x_src: Buf, g_dst: Buf, init_scale: float,
                 grad_scale: float = 1024.0):
        assert height % 16 == 0 and width % 16 == 0, "four 2x2 max-pools"
        self.plan, self.B, self.H, self.W = plan, batch, height, width
        self.init_scale, self.grad_scale = float(init_scale), float(grad_scale)
        self.x_src = x_src
        p, B, H, W = plan, batch, height, width
        sd = {k: v.detach().float().cpu() for k, v in state_dict.items()}
        self.loss = p.new(B, "f", "lpips_loss")
        p.mark("lpips")
        p.emit("FILL", i=[B], f=[0.0], p=[(self.loss, 0)], tag="lpips loss = 0")
        x0 = p.act(B, H, W, IN_PAD, "lpips_x")
        p.emit("NCHW_TO_PM", flags=4, i=[B, 3, H * W, IN_PAD], f=[1.0, *SHIFT, *(1.0 / s for s in SCALE)], p=[(x_src, 0), (x0.buf, 0)],
               tag="ScalingLayer -> pixel-major")
        saved_tape, p._tape = p._tape, []
        h, cin = x0, 3
        self.taps = []
        for k, idxs in enumerate(SLICES):
            if k:
                h = p.maxpool2(h, name=f"lpips.pool{k}")
            for i in idxs:
                w = sd[f"net.slice{k + 1}.{i}.weight"]
                if cin == 3:  # zero-pad the image channels to one 64-wide K slice in both orientations
                    w = th.cat([w, th.zeros(w.shape[0], IN_PAD - 3, 3, 3)], dim=1)
                cw = pack_conv(p, w, sd[f"net.slice{k + 1}.{i}.bias"], need_bwd=True, name=f"lpips.conv{i}")
                h = p.relu(p.conv(h, cw, name=f"lpips.conv{i}"), name=f"lpips.relu{i}")
                cin = CHANNELS[k]
            self.taps.append(h)
        p.mark("lpips_tap")
        self.targets, dfs = [], []
        for k, h in enumerate(self.taps):
            tn = p.new(h.H * h.W * h.C, "h", f"lpips.target{k}")  # normalised init-image features, broadcast over the batch
            wl = p.const(sd[f"lin{k}.model.1.weight"].reshape(-1), "f", f"lpips.lin{k}")
            df = p.act(h.N, h.H, h.W, h.C, f"lpips.d_tap{k}")
            p.emit("LPIPS_TAP", i=[B, h.H * h.W, h.C, 1], f=[self.init_scale * self.grad_scale],
                   p=[p._ap(h), (tn, 0), (wl, 0), p._ap(df), (self.loss, 0)], tag=f"lpips tap {k}")
            self.targets.append(tn)
            dfs.append(df)
        p.mark("lpips_bwd")
        for h, df in zip(self.taps, dfs):
            p._grads[h.key()] = df
        p.backward()
        p._tape = saved_tape
        dx0 = p.grad_of(x0)
        assert dx0 is not None and dx0.C == IN_PAD
        p.emit("PM_TO_NCHW", flags=2 | 4, i=[B, 3, H * W, dx0.ld], f=[1.0 / self.grad_scale, *(1.0 / s for s in SCALE)],
               p=[p._ap(dx0), (g_dst, 0)], tag="d ScalingLayer, += x_in gradient")
        p.mark("lpips_end")

    def set_init_image(self, init: th.Tensor, runner=None):
        """init: [1 or B, 3, H, W] in [-1, 1] (cgd/cgd.py:116-120).  Runs the VGG forward ops on it and stores the channel-
        normalised tap features (set-up time, not on the per-step path)."""
        p = self.plan
        img = init.detach().float()
        if img.shape[0] != 1:
            img = img[:1]
        xs = p.view(self.x_src, (self.B, 3, self.H, self.W))
        keep = xs.clone()
        xs.copy_(img.to(xs.device).expand(self.B, -1, -1, -1))
        (runner or p.run_range)("lpips", "lpips_tap")
        for h, tn in zip(self.taps, self.targets):
            f = p.view(h.buf, (h.N, h.H * h.W, h.C))[0].float()
            p.view(tn, (h.H * h.W, h.C)).copy_((f / (f.pow(2).sum(-1, keepdim=True).sqrt() + 1e-10)).half())
        xs.copy_(keep)

    def loss_value(self) -> th.Tensor:
        """per-image ``lpips_vgg(x_in, init)`` of the last step (logging, cgd/cgd.py:223)"""
        return self.plan.view(self.loss, (self.B,))
