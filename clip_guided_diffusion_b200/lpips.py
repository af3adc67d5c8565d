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


def vgg_trunk(p: Plan, sd: dict, n: int, height: int, width: int, src: Buf, prefix: str = "lpips", convs: list = None):
    """ScalingLayer + VGG16 up to relu5_3 on ``n`` fp32 NCHW images at ``src``, forward ops emitted into ``p`` with their backward on
    ``p._tape``.  ``sd``: fp32 upstream-layout weights; ``convs``: the 13 packed layers of an earlier trunk of the same plan to share
    (None packs them here).  Returns (pixel-major input, the five tap activations, the packed layers)."""
    x0 = p.act(n, height, width, IN_PAD, f"{prefix}_x")
    p.emit("NCHW_TO_PM", flags=4, i=[n, 3, height * width, IN_PAD], f=[1.0, *SHIFT, *(1.0 / s for s in SCALE)], p=[(src, 0), (x0.buf, 0)],
           tag="ScalingLayer -> pixel-major")
    h, cin, taps, packed = x0, 3, [], []
    for k, idxs in enumerate(SLICES):
        if k:
            h = p.maxpool2(h, name=f"{prefix}.pool{k}")
        for i in idxs:
            if convs is None:
                w = sd[f"net.slice{k + 1}.{i}.weight"]
                if cin == 3:  # zero-pad the image channels to one 64-wide K slice in both orientations
                    w = th.cat([w, th.zeros(w.shape[0], IN_PAD - 3, 3, 3)], dim=1)
                cw = pack_conv(p, w, sd[f"net.slice{k + 1}.{i}.bias"], need_bwd=True, name=f"lpips.conv{i}")
            else:
                cw = convs[len(packed)]
            packed.append(cw)
            h = p.relu(p.conv(h, cw, name=f"{prefix}.conv{i}"), name=f"{prefix}.relu{i}")
            cin = CHANNELS[k]
        taps.append(h)
    return x0, taps, packed


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
        saved_tape, p._tape = p._tape, []
        x0, self.taps, _ = vgg_trunk(p, sd, B, H, W, x_src)
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


# ---------------------------------------------------------------------------------------------------------------------------------
# LPIPS(net='vgg') under torch.autograd
#
# ``LPIPS()(in0, in1)`` is the ``lpips`` package's call with both inputs differentiable.  One plan per (H, W, N0, N1), built on the first
# call with that shape: trunk 0 on in0's rows and trunk 1 on in1's rows over one set of packed weights, each with its own backward tape,
# and the ops of csrc/lpips.cu (include/cgd_b200.h CGD_OP_LPIPS_*), in these ranges:
#
#     lp_fwd0 / lp_fwd1      in0 / in1 staging -> ScalingLayer (NCHW_TO_PM flags 4) -> VGG16 to relu5_3
#     lp_tap                 LPIPS_PAIR_FWD per tap -> LPIPS_LOSS: loss [B]
#     lp_seed                LPIPS_SEED: one power of two per trunk row from d_loss alone
#     lp_seed01 / 0 / 1      LPIPS_PAIR_BWD per tap, seeds of both sides / in0's / in1's
#     lp_bwd0 / lp_bwd1      VGG16 backward of that trunk -> PM_TO_NCHW flags 4 | 8 (inverse ScalingLayer, unscale): d in0 / d in1
#
# The host runs only the seed and backward ranges of the inputs that need a gradient.  Decisions:
# 1. No padding: every shape gets its own plan (the arena is sized for it; DESIGN.md section 2).
# 2. Inputs may be fp32, fp16 or bf16 (copied exactly into fp32 staging); the loss is fp32 [B, 1, 1, 1], gradients come back in each
#    input's dtype.
# 3. Every forward bumps its plan's generation counter; a backward whose forward is no longer the plan's latest raises (its
#    activations are overwritten), so does create_graph=True.  retain_graph=True may run a backward twice, with the same bits.
# 4. No weight gradients: the weights are constants of the plans.

# LPIPS_SEED's target for |d_loss| * scale: measured with scripts/lpips_seed_band.py (DESIGN.md section 2)
LPIPS_SEED_BAND = 2.0 ** 23

_INPUT_DTYPES = (th.float32, th.float16, th.bfloat16)


def _fwd_blocks(hw: int) -> int:
    """LPIPS_PAIR_FWD CTAs per image: about 64 pixels (8 per warp) each"""
    return max(1, min(4096, -(-hw // 64)))


class LpipsPairPlan:
    """the plan of one (H, W, N0, N1): see the ranges above"""

    def __init__(self, convs_sd: dict, height: int, width: int, n0: int, n1: int, device=None):
        self.H, self.W, self.N = height, width, (n0, n1)
        B = self.B = max(n0, n1)
        p = self.plan = Plan()
        hw = height * width
        self.x = [p.new(n * 3 * hw, "f", f"lpips_in{s}") for s, n in enumerate(self.N)]
        self.dx = [p.new(n * 3 * hw, "f", f"lpips_d_in{s}") for s, n in enumerate(self.N)]
        self.d_loss = p.new(B, "f", "lpips_d_loss")
        self.dyn = p.new(n0 + n1, "f", "lpips_seed_scale")
        self.loss = p.new(B, "f", "lpips_loss")
        x0, taps, tapes, convs = [], [], [], None
        for s, n in enumerate(self.N):
            p.mark(f"lp_fwd{s}")
            p._tape = []
            xs, ts, convs = vgg_trunk(p, convs_sd, n, height, width, self.x[s], prefix=f"lpips{s}", convs=convs)
            x0.append(xs)
            taps.append(ts)
            tapes.append(p._tape)
        p._tape = []
        p.mark("lp_tap")
        wl = [p.const(convs_sd[f"lin{k}.model.1.weight"].reshape(-1), "f", f"lpips.lin{k}") for k in range(5)]
        parts, nblk = [], []
        for k, (f0, f1) in enumerate(zip(taps[0], taps[1])):
            thw = f0.H * f0.W
            nblk.append(_fwd_blocks(thw))
            parts.append(p.new(B * nblk[-1], "f", f"lpips.partial{k}"))
            p.emit("LPIPS_PAIR_FWD", i=[B, thw, f0.C, n0, n1, nblk[-1]], p=[p._ap(f0), p._ap(f1), (wl[k], 0), (parts[-1], 0)], tag=f"lpips pair tap {k}")
        p.emit("LPIPS_LOSS", i=[B, *nblk], f=[1.0 / (t.H * t.W) for t in taps[0]], p=[*((b, 0) for b in parts), (self.loss, 0)], tag="lpips loss")
        p.mark("lp_seed")
        p.emit("LPIPS_SEED", i=[B, n0, n1], f=[LPIPS_SEED_BAND], p=[(self.d_loss, 0), (self.dyn, 0)], tag="seed of the lpips backward")
        dfs = [[p.act(t.N, t.H, t.W, t.C, f"lpips{s}.d_tap{k}") for k, t in enumerate(taps[s])] for s in range(2)]
        for name, flags in (("lp_seed01", 3), ("lp_seed0", 1), ("lp_seed1", 2)):
            p.mark(name)
            for k, (f0, f1) in enumerate(zip(taps[0], taps[1])):
                p.emit("LPIPS_PAIR_BWD", flags=flags, i=[B, f0.H * f0.W, f0.C, n0, n1],
                       p=[p._ap(f0), p._ap(f1), (wl[k], 0), (self.d_loss, 0), (self.dyn, 0), p._ap(dfs[0][k]) if flags & 1 else None,
                          p._ap(dfs[1][k]) if flags & 2 else None], tag=f"lpips pair tap {k} seeds ({name})")
        for s, n in enumerate(self.N):
            p.mark(f"lp_bwd{s}")
            for t, df in zip(taps[s], dfs[s]):
                p._grads[t.key()] = df
            p._tape = tapes[s]
            p.backward()
            dx0 = p.grad_of(x0[s])
            assert dx0 is not None and dx0.C == IN_PAD
            p.emit("PM_TO_NCHW", flags=4 | 8, i=[n, 3, hw, dx0.ld], f=[1.0, *(1.0 / sc for sc in SCALE)], p=[p._ap(dx0), (self.dx[s], 0), (self.dyn, s * n0)],
                   tag=f"d ScalingLayer, unscale: d in{s}")
        p.mark("lp_end")
        if device is not None:
            p.finalize(device)
        self.generation = 0

    def forward(self, in0: th.Tensor, in1: th.Tensor) -> int:
        """stage both inputs, run both trunks and the loss; returns the forward's generation"""
        for s, x in enumerate((in0, in1)):
            self.plan.view(self.x[s], tuple(x.shape)).copy_(x.detach())
        self.generation += 1
        self.plan.run_range("lp_fwd0", "lp_seed")
        return self.generation

    def value(self) -> th.Tensor:
        return self.plan.view(self.loss, (self.B, 1, 1, 1)).clone()

    def backward(self, generation: int, d_loss: th.Tensor, need: tuple) -> list:
        """[d in0 | None, d in1 | None] (fp32) from d loss [B, 1, 1, 1] of the forward ``generation``"""
        if th.is_grad_enabled():
            raise RuntimeError("double backward (create_graph=True) through LPIPS is not supported")
        if generation != self.generation:
            raise RuntimeError("backward through LPIPS after a later LPIPS call with the same shapes: its activations are overwritten.  "
                               "Take the gradient of each call before the next one of the same shapes")
        p = self.plan
        p.view(self.d_loss, (self.B,)).copy_(d_loss.reshape(self.B))
        p.run_range("lp_seed", "lp_seed01")
        seeds = ("lp_seed01", "lp_seed0") if all(need) else ("lp_seed0", "lp_seed1") if need[0] else ("lp_seed1", "lp_bwd0")
        p.run_range(*seeds)
        out = []
        for s, ends in enumerate((("lp_bwd0", "lp_bwd1"), ("lp_bwd1", "lp_end"))):
            if need[s]:
                p.run_range(*ends)
                out.append(p.view(self.dx[s], (self.N[s], 3, self.H, self.W)).clone())
            else:
                out.append(None)
        return out


class _LpipsFunction(th.autograd.Function):
    """LPIPS under autograd: forward = both trunks + loss; backward = the seeds and trunk backwards of the inputs that need a gradient.
    The backward re-enters the plan's activations, so it must follow that plan's latest forward."""

    @staticmethod
    def forward(ctx, in0, in1, plan):
        ctx.plan, ctx.gen, ctx.dtypes = plan, plan.forward(in0, in1), (in0.dtype, in1.dtype)
        return plan.value()

    @staticmethod
    def backward(ctx, d_loss):
        need = tuple(ctx.needs_input_grad[:2])
        g = ctx.plan.backward(ctx.gen, d_loss, need)
        return (g[0].to(ctx.dtypes[0]) if need[0] else None), (g[1].to(ctx.dtypes[1]) if need[1] else None), None


class LPIPS:
    """``lpips.LPIPS(net='vgg')`` (v0.1, eval mode) on this package's kernels: ``LPIPS()(in0, in1)`` -> fp32 [N, 1, 1, 1], differentiable
    in both inputs.  Weights from ``lpips_state_dict=`` (upstream keys ``net.sliceK.<idx>.{weight,bias}``, ``linK.model.1.weight``) or
    from the installed ``lpips`` package."""

    def __init__(self, net: str = "vgg", *, lpips_state_dict: dict = None, device="cuda"):
        if net != "vgg":
            raise ValueError(f"LPIPS(net={net!r}): only net='vgg' is implemented")
        from .cgd import _lpips_sd
        self.sd = {k: v.detach().float().cpu() for k, v in _lpips_sd(lpips_state_dict).items()}
        device = th.device(device)
        if device.type == "cuda" and device.index is None:
            device = th.device("cuda", th.cuda.current_device())
        self.device = device
        self.plans: dict = {}

    # the no-op chain of the reference's construction: lpips.LPIPS(net='vgg').to(device) (and .eval() / .requires_grad_(False))
    def eval(self):
        return self

    def requires_grad_(self, flag=False):
        return self

    def to(self, device=None, *a, **k):
        if device is not None and not isinstance(device, th.dtype) and th.device(device).type != self.device.type:
            raise RuntimeError(f"the LPIPS model lives on {self.device}; construct one per device")
        return self

    def plan_for(self, height: int, width: int, n0: int, n1: int) -> LpipsPairPlan:
        key = (height, width, n0, n1)
        if key not in self.plans:
            self.plans[key] = LpipsPairPlan(self.sd, height, width, n0, n1, self.device)
        return self.plans[key]

    def _check(self, in0, in1):
        for name, x in (("in0", in0), ("in1", in1)):
            if not isinstance(x, th.Tensor) or x.dim() != 4 or x.shape[1] != 3:
                raise ValueError(f"LPIPS takes [N, 3, H, W] images, got {name} "
                                 f"{tuple(x.shape) if isinstance(x, th.Tensor) else type(x).__name__}")
            if x.dtype not in _INPUT_DTYPES:
                raise ValueError(f"LPIPS takes fp32, fp16 or bf16 images, got {name} in {x.dtype}")
            if x.device != self.device:
                raise ValueError(f"LPIPS: {name} is on {x.device}, the model on {self.device}")
        if in0.shape[2:] != in1.shape[2:]:
            raise ValueError(f"LPIPS: in0 is {tuple(in0.shape[2:])} and in1 {tuple(in1.shape[2:])} pixels: the sizes must agree")
        H, W = in0.shape[2:]
        if H % 16 or W % 16 or H == 0 or W == 0:
            raise ValueError(f"LPIPS: {H}x{W} images: height and width must be positive multiples of 16 (four 2x2 max-pools)")
        n0, n1 = in0.shape[0], in1.shape[0]
        if n0 < 1 or n1 < 1 or not (n0 == n1 or n0 == 1 or n1 == 1):
            raise ValueError(f"LPIPS: batches of {n0} and {n1} images: they must be equal, or one of them 1 (broadcast)")

    def forward(self, in0: th.Tensor, in1: th.Tensor, retPerLayer: bool = False, normalize: bool = False) -> th.Tensor:  # noqa: N803
        """the lpips package's ``forward``: [N0, 3, H, W] and [N1, 3, H, W] in [-1, 1] ([0, 1] with ``normalize=True``), N0 == N1 or either
        1 -> fp32 [max(N0, N1), 1, 1, 1].  With grad mode on and an input that requires grad, the result has a ``grad_fn``."""
        if retPerLayer:
            raise ValueError("LPIPS(retPerLayer=True) is not supported: the per-layer values are reduced on the device")
        self._check(in0, in1)
        if normalize:
            in0, in1 = 2 * in0 - 1, 2 * in1 - 1
        plan = self.plan_for(in0.shape[2], in0.shape[3], in0.shape[0], in1.shape[0])
        if th.is_grad_enabled() and (in0.requires_grad or in1.requires_grad):
            return _LpipsFunction.apply(in0, in1, plan)
        plan.forward(in0, in1)
        return plan.value()

    __call__ = forward
