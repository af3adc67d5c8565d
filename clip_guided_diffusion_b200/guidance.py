"""The guided sampling step engine: UNet fwd -> cond_fn (cutouts, CLIP fwd/bwd, losses) -> UNet dgrad -> update.

Replaces the L1 <-> L3 <-> L2 ping-pong the reference executes once per timestep (SURVEY.md 3.2 / 3.3):
``p_mean_variance`` + ``cond_fn`` (cgd/cgd.py:151-239) + ``-autograd.grad`` (cgd/cgd.py:228) + the ancestral / DDIM
update.  One op plan holds both networks and every guidance kernel in a single arena; a whole step (918 kernel launches for
bench.py's cfg2: 256², ViT-B/32, 16 cutouts) is replayed from one CUDA graph, fed per step by one small pinned H2D copy (scalars,
cutout windows, t, y).

Surfaces kept (SURVEY.md 8b): ``cond_fn(x, t, out, y=None)``, ``MakeCutouts``, ``model(x, timesteps, y)``.
"""
from __future__ import annotations

import itertools

import numpy as np
import torch as th

from . import _lib
from ._lib import SC
from .plan import Plan
from .unet import IN_PAD, UNetB200, UNetConfig
from .rn import RNB200, RNConfig
from .vit import ViTB200, ViTConfig

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)  # cgd/clip_util.py:45
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)


class MakeCutouts(th.nn.Module):
    """cgd/modules.py:5-66 surface: same constructor, ``cached_coords``, ``cache_coordinates`` and the same CPU-generator
    draw order (3 draws per cutout: size, offsetx, offsety).  ``forward`` runs the batched CUDA cutout kernel and
    returns ``[cutn*B, 3, cut_size, cut_size]`` fp32 (un-normalised pooled cutouts, like the reference)."""

    def __init__(self, cut_size: int, num_cutouts: int, cutout_size_power: float = 1.0, use_augs: bool = False):
        super().__init__()
        self.cut_size, self.cutn, self.cut_pow = cut_size, num_cutouts, cutout_size_power
        self.cached_coords = None
        # use_augs (cgd/modules.py:12-24): flip / affine / perspective / grayscale / noise run inside the cutout kernels
        # (csrc/augs.cu) from parameters drawn in torchvision's order (augs.py); `augs` stays an attribute like the reference's
        self.use_augs = bool(use_augs)
        self.augs = th.nn.Identity()

    def _generate_coords(self, side_x: int, side_y: int, cutn: int):
        max_size = min(side_y, side_x)
        min_size = min(side_y, side_x, self.cut_size)
        coords = []
        for _ in range(cutn):
            size = int(th.rand([]) ** self.cut_pow * (max_size - min_size) + min_size)
            offsetx = th.randint(0, side_x - size + 1, ()).item()
            offsety = th.randint(0, side_y - size + 1, ()).item()
            coords.append((offsetx, offsety, size))
        return coords

    def cache_coordinates(self, side_x: int, side_y: int):
        self.cached_coords = self._generate_coords(side_x, side_y, self.cutn)

    def coords_for(self, side_x, side_y, use_cache=False, num_cutouts_override=None):
        cutn = num_cutouts_override if num_cutouts_override is not None else self.cutn
        if use_cache and self.cached_coords is not None:
            if len(self.cached_coords) < cutn:  # the reference fails one line later, at .view([current_cutn, n, -1]) (cgd/cgd.py:194-195)
                raise RuntimeError(f"{cutn} cutouts requested but only {len(self.cached_coords)} cached: cached_cutouts with "
                                   "progressive_cutout needs num_cutouts >= 16 (the schedule's middle count is max(8, n // 2))")
            return self.cached_coords[:cutn]
        return self._generate_coords(side_x, side_y, cutn)

    def forward(self, input: th.Tensor, use_cache: bool = False, num_cutouts_override: int = None):
        """with grad mode on and ``input.requires_grad`` the result has a ``grad_fn`` whose backward is the gather transpose of the same
        windows (CUTOUTS_BWD / CUTOUTS_AUG_BWD flags 4) and returns d / d input in input's dtype; otherwise a plain tensor"""
        B, C, H, W = input.shape
        assert C == 3
        if not input.is_floating_point():
            raise ValueError(f"MakeCutouts takes a floating-point image batch, got {input.dtype}")
        coords = self.coords_for(H, W, use_cache, num_cutouts_override)  # sic: (H, W) passed as (side_x, side_y), modules.py:52
        cdev = th.tensor(coords, dtype=th.int32, device=input.device)
        prm = noise = None
        if self.use_augs:  # parameters and noise are drawn here, in the reference's order, whether or not a gradient follows
            from . import augs
            Smax = min(H, W)
            noise = th.zeros(len(coords), 4, B, 3, Smax, Smax, device=input.device)
            prm = augs.draw_aug_params(coords, B, H, W, noise_device=input.device, noise_out=noise).to(input.device)
        if th.is_grad_enabled() and input.requires_grad:
            return _CutoutsFunction.apply(input, cdev, self.cut_size, prm, noise)
        return _cutouts_fwd(input.detach().float().contiguous(), cdev, self.cut_size, prm, noise)


def _cutouts_fwd(x: th.Tensor, cdev: th.Tensor, cs: int, prm=None, noise=None) -> th.Tensor:
    """pooled cutouts [cutn*B, 3, cs, cs] fp32 of x [B, 3, H, W] (fp32, contiguous) at the windows cdev (int32 [cutn, 3]); with ``prm``
    (and ``noise``) the use_augs pipeline"""
    B, _, H, W = x.shape
    n = cdev.shape[0]
    if prm is not None:  # the reference applies its augmentations to the raw cutout values: feed 2x - 1, mean 0 / std 1
        out = th.empty(n * B, 1, 3 * cs * cs, dtype=th.float16, device=x.device)
        _lib.run_op("CUTOUTS_AUG_FWD", i=[B, H, W, n, cs, cs, 3 * cs * cs, noise.shape[-1]], f=[0.0, 0.0, 0.0, 1.0, 1.0, 1.0],
                    p=[x * 2 - 1, cdev, out, prm, noise])
        return out.view(n * B, 3, cs, cs).float()
    # mean 0.5 / std 0.5 with the kernel's (x + 1) / 2 yield the raw pooled value; flags 1 = fp32 output like the reference's
    # adaptive_avg_pool2d (the fused step writes fp16 straight into the CLIP tower's patch buffer instead)
    out32 = th.empty(n * B, 3, cs, cs, dtype=th.float32, device=x.device)
    _lib.run_op("CUTOUTS_FWD", flags=1, i=[B, H, W, n, cs, cs, 3 * cs * cs], f=[0.5] * 6, p=[x, cdev, out32], what="cgd_cutouts_fwd")
    return out32


class _CutoutsFunction(th.autograd.Function):
    """``MakeCutouts.forward`` under autograd.  Stateless: the windows (and the use_augs parameters) travel in the graph, so several calls
    can share one backward.  The backward reads fp32 d cutouts, which is the patch layout with P = cs (flags 4): the pool gather
    (deterministic) with std 0.5 undoing the forward's mean 0.5 / std 0.5 fold, or the use_augs scatter with scale 2 undoing its x * 2 - 1."""

    @staticmethod
    def forward(ctx, input, cdev, cs, prm, noise):
        ctx.save_for_backward(cdev, prm)
        ctx.geo = (tuple(input.shape), input.dtype, cs)
        return _cutouts_fwd(input.detach().float().contiguous(), cdev, cs, prm, noise)

    @staticmethod
    @th.autograd.function.once_differentiable
    def backward(ctx, d):
        cdev, prm = ctx.saved_tensors
        (B, _, H, W), dtype, cs = ctx.geo
        dims = [B, H, W, cdev.shape[0], cs, cs, 3 * cs * cs]
        d = d.float().contiguous()
        if prm is None:
            dx = th.empty(B, 3, H, W, device=d.device)
            _lib.run_op("CUTOUTS_BWD", flags=4, i=dims, f=[0.0, 0.0, 0.0, 0.5, 0.5, 0.5, 1.0], p=[d, cdev, dx])
        else:
            dx = th.zeros(B, 3, H, W, device=d.device)  # the use_augs backward scatters into dx
            _lib.run_op("CUTOUTS_AUG_BWD", flags=4, i=dims, f=[0.0, 0.0, 0.0, 1.0, 1.0, 1.0, 2.0], p=[d, cdev, dx, prm])
        return dx.to(dtype), None, None, None, None


class EngineModel:
    """What the loops and ``p_sample`` receive as ``model``: ``model(x, timesteps, y) -> [B, 6, H, W]``."""

    def __init__(self, engine):
        self.engine = engine
        self.num_classes = engine.unet.num_classes
        self.dtype = th.float16

    def __call__(self, x, timesteps, y=None):
        """with grad mode on and ``x.requires_grad`` (an input gradient is wanted: a PyTorch cond_fn's ``th.autograd.grad(loss, x)``)
        the result is a fresh tensor with a ``grad_fn`` whose backward runs the UNet input-gradient plan; otherwise a view of the
        engine's output buffer, valid until the next UNet forward"""
        eng = self.engine
        if th.is_grad_enabled() and isinstance(x, th.Tensor) and x.requires_grad:
            return _UNetFunction.apply(x, eng, timesteps, y)
        eng.forward_generation += 1
        return eng.unet(x, timesteps, y)

    def parameters(self):
        yield self.engine.plan.arena

    def eval(self):
        return self

    def requires_grad_(self, flag=False):
        return self

    def convert_to_fp16(self):
        return self

    def to(self, device=None, *a, **k):  # cgd/script_util.py:318 chains .requires_grad_(False).eval().to(device)
        if device is not None and th.device(device).type != self.engine.device.type:
            raise RuntimeError(f"the engine lives on {self.engine.device}; build a GuidedStepB200 per device")
        return self

    def load_state_dict(self, state_dict, strict=True):
        """cgd/script_util.py:317 ``model.load_state_dict(th.load(checkpoint_path))``: re-pack a checkpoint in upstream key layout
        into the kernel layouts (K-major fp16 tiles, tap-flipped dgrad copies, the fused emb_layers matrix) IN PLACE -- the engine's
        op lists, TMA descriptors and captured CUDA graphs hold addresses and stay valid.  The packing code runs once more on the
        host against a shadow plan (seconds, like construction); shapes must match the architecture the engine was built for."""
        from . import weights as W
        from .plan import Plan
        eng = self.engine
        want = W.unet_param_shapes(eng.unet.cfg)
        missing = [k for k in want if k not in state_dict]
        unexpected = [k for k in state_dict if k not in want]
        bad = [k for k in want if k in state_dict and tuple(state_dict[k].shape) not in (tuple(want[k]), tuple(want[k]) + (1,))]
        if bad:
            raise RuntimeError("size mismatch for " + ", ".join(f"{k}: {tuple(state_dict[k].shape)} vs {tuple(want[k])}" for k in bad[:4]))
        if missing or (strict and unexpected):
            raise RuntimeError(f"Error(s) in loading state_dict: missing {missing[:4]}{'...' if len(missing) > 4 else ''}, "
                               f"unexpected {unexpected[:4]}{'...' if len(unexpected) > 4 else ''}")
        shadow = Plan(conv_impl=eng.plan.conv_impl)
        for flag in ("grid_gn", "fused_gn", "cluster_splitk"):
            setattr(shadow, flag, getattr(eng.plan, flag))
        UNetB200(eng.unet.cfg, state_dict, batch=eng.B, height=eng.H, width=eng.W, device="cpu", seed_scale=eng.unet.seed_scale, plan=shadow,
                 build_backward=bool(eng.towers) or eng.input_grad)
        eng.plan.reload_consts(shadow, first=0)  # the UNet is the first network of the engine's plan
        if eng.device.type == "cuda":
            th.cuda.synchronize(eng.device)
        import collections
        return collections.namedtuple("IncompatibleKeys", "missing_keys unexpected_keys")(missing, unexpected)


class _UNetFunction(th.autograd.Function):
    """``model(x, t, y)`` under autograd: forward = the UNet forward range; backward = GRAD_SEED -> UNet input-gradient plan ->
    GRAD_UNSCALE.  The backward re-enters the activations of the engine's arena, so it must follow the latest UNet forward."""

    @staticmethod
    def forward(ctx, x, eng, timesteps, y):
        ctx.eng, ctx.gen = eng, eng.autograd_forward(x, timesteps, y)
        return eng.unet.out_view.clone()

    @staticmethod
    def backward(ctx, d_out):
        return ctx.eng.autograd_backward(ctx.gen, d_out=d_out), None, None, None


class _PMVFunction(th.autograd.Function):
    """the package's ``p_mean_variance`` under autograd: forward = UNet forward + PMV_BLEND; backward = PMV_BWD -> GRAD_SEED -> UNet
    input-gradient plan -> GRAD_UNSCALE (+ the direct x terms of pred_xstart and mean)"""

    @staticmethod
    def forward(ctx, x, eng, diffusion, t_index, y):
        out = eng.unet_forward(diffusion, x.detach(), t_index, y)
        ctx.eng, ctx.gen = eng, eng.forward_generation
        return tuple(out[k].clone() for k in PMV_KEYS)

    @staticmethod
    def backward(ctx, *grads):
        return ctx.eng.autograd_backward(ctx.gen, pmv_grads=grads), None, None, None, None


PMV_KEYS = ("pred_xstart", "mean", "variance", "log_variance")


def _as_list(v):
    """a list or tuple (one item per CLIP tower) -> list(v); anything else is one item -> [v]"""
    return list(v) if isinstance(v, (list, tuple)) else [v]


def check_tower_options(n_towers: int, use_augs: bool, cutout_resize: str):
    """several CLIP towers run with the reference's adaptive_avg_pool2d cutouts and no augmentations"""
    if n_towers > 1 and use_augs:
        raise NotImplementedError("use_augs with several CLIP towers (the augmentation parameters are drawn for one tower's cutouts)")
    if n_towers > 1 and cutout_resize == "lanczos3":
        raise NotImplementedError("cutout_resize='lanczos3' with several CLIP towers (the resampling tables are built for one tower)")


def clip_tower(cfg, state_dict, **kw):
    """the CLIP visual tower of `cfg`: a ViT (vit.py) or a ModifiedResNet (rn.py); both expose patches / embeds / d_embeds / d_patches"""
    return (RNB200 if isinstance(cfg, RNConfig) else ViTB200)(cfg, state_dict, **kw)


class _Tower:
    """one CLIP tower of the engine: its config, the buffers of its cutout windows (``coords``) and targets, the slot of its CLIP loss, one tower instance
    per cutout count, and the ResizeRight tables of its windows (``rr``: the y axis's, which serve the x axis too on a square image;
    ``rr_x``: the x axis's own on a non-square image, else None)"""

    def __init__(self, cfg, tag, cutn, coords, targets, loss):
        self.cfg, self.tag, self.cutn, self.coords, self.targets, self.loss = cfg, tag, cutn, coords, targets, loss
        self.by_count = {}
        self.rr = self.rr_x = None  # ResizeRight, per axis: (left [cutn, cs], weights [cutn, cs, T_MAX], taps [cutn], inverse [cutn, min(H, W), 2])

    def sfx(self, c):
        """range-mark suffix: the cutout count's ("@c", "" for the default count), then the tower's ("", "#1", "#2", ...)"""
        return ("" if c == self.cutn else f"@{c}") + self.tag


class _Fork(tuple):
    """schedule entry: the op ranges of one CLIP forward or backward, one per batch slice (vit_streams); run on parallel streams"""


ALL_REDUCE = "all_reduce"  # schedule entry: the host all-reduces the partial sums of the sharded RMS clamp (fg_ws) over the ranks


class GuidedStepB200:
    """Engine for one (local batch, H, W, cutn, CLIP towers) configuration on one GPU.

    ``vit_cfg`` / ``vit_sd``: one CLIP visual tower, or equal-length sequences of them (an ensemble).  Every tower cuts its own windows at
    its own resolution and gets its own targets; their CLIP losses are summed (the reference's CLIP block once per tower) and share the
    prompt weights.  The towers run one after another inside the step; the first stores its cutout gradient, the others add theirs
    (CUTOUTS_BWD flags 2), in tower order."""

    def __init__(self, unet_cfg: UNetConfig, unet_sd: dict, vit_cfg: ViTConfig = None, vit_sd: dict = None, *, batch: int,
                 height: int = None, width: int = None, num_cutouts: int = 16, max_prompts: int = 1, clip_guidance_scale=1000.0,
                 tv_scale=150.0, range_scale=50.0, sat_scale=0.0, use_magnitude=False, device="cuda", seed_scale=0.0,
                 vit_grad_scale=1.0, conv_impl=0, rank: int = 0, world_size: int = 1, use_graph: bool = True, vit_streams: int = 1,
                 cutn_variants: tuple = (), lpips_sd: dict = None, init_scale: float = 0.0, cutout_resize: str = "pool",
                 use_augs: bool = False, input_grad: bool = False):
        """``input_grad``: also build the input-gradient path of ``model()`` and of ``p_mean_variance`` under torch.autograd (the UNet
        backward even without a CLIP tower, and the GRAD_SEED / GRAD_UNSCALE / PMV_BWD ranges after the step's), so any PyTorch cond_fn
        can guide a run"""
        self.device = th.device(device)
        self.input_grad = bool(input_grad)
        self.B = batch
        self.rank, self.world = rank, world_size
        self.global_batch = batch * world_size
        self.H = height or unet_cfg.image_size
        self.W = width or unet_cfg.image_size
        self.cutn = num_cutouts if vit_cfg is not None else 0
        cfgs = _as_list(vit_cfg) if vit_cfg is not None else []
        sds = _as_list(vit_sd) if vit_cfg is not None else []
        if vit_cfg is not None and (not cfgs or len(sds) != len(cfgs)):
            raise ValueError(f"vit_cfg / vit_sd: one CLIP tower or equal-length non-empty sequences (got {len(cfgs)} configs, {len(sds)} state_dicts)")
        check_tower_options(len(cfgs), use_augs, cutout_resize)
        self.T = len(cfgs)
        self.P = max_prompts
        self.scales = dict(cgs=float(clip_guidance_scale), tv=float(tv_scale), rng=float(range_scale), sat=float(sat_scale))
        self.use_magnitude = bool(use_magnitude)
        self.mag_sync = False
        self.seed_scale, self.vit_grad_scale = float(seed_scale), float(vit_grad_scale)
        self.use_graph = use_graph and self.device.type == "cuda"
        self.plan = p = Plan(conv_impl=conv_impl)
        B, H, W, HW = self.B, self.H, self.W, self.H * self.W
        self.unet = UNetB200(unet_cfg, unet_sd, batch=B, height=H, width=W, device=device, seed_scale=seed_scale or 1.0, plan=p,
                             build_backward=bool(cfgs) or self.input_grad)
        n3 = B * 3 * HW
        self.sc = p.new(SC["COUNT"], "f", "scalars")
        self.noise = p.new(n3, "f", "noise")
        self.x0 = p.new(n3, "f", "pred_xstart")
        self.mean = p.new(n3, "f", "mean")
        self.var = p.new(n3, "f", "variance")
        self.logvar = p.new(n3, "f", "log_variance")
        self.x_inb = p.new(n3, "f", "x_in")
        self.g = p.new(n3, "f", "g")
        self.sample = p.new(n3, "f", "sample")
        self.loss = p.new(4 * B, "f", "losses")  # [clip | tv | range | sat] per image
        p.mark("pmv")
        p.emit("PMV_BLEND", i=[B, HW, 3 * B], p=[(self.unet.x_in, 0), (self.unet.out, 0), (self.sc, 0), (self.x0, 0), (self.mean, 0),
                                                 (self.var, 0), (self.logvar, 0), (self.x_inb, 0), (self.loss, B)], tag="p_mean_variance+blend")
        p.mark("cond")
        self.lpips = None
        self.towers = []
        self.loss_towers = None
        self.use_augs = bool(use_augs and cfgs)
        # {cutout count: the towers' instances for that count, in tower order}; its keys are the counts the engine runs: num_cutouts and
        # the further counts of progressive_cutout (cgd/cgd.py:167-175), each with its own activations and op ranges ("...@c" marks),
        # sharing the packed weights of the default count
        self.vits = {}
        if cfgs:
            cutn = self.cutn
            # cutout resampling: "pool" = adaptive_avg_pool2d like the reference's MakeCutouts (cgd/modules.py:63); "lanczos3" =
            # the vendored ResizeRight resampler north_star names (cgd/ResizeRight/resize_right.py, host tables in resize_right.py)
            if cutout_resize not in ("pool", "lanczos3"):
                raise ValueError("cutout_resize must be 'pool' or 'lanczos3'")
            for c in cutn_variants:
                if not 0 < int(c) <= cutn:
                    raise ValueError(f"cutn_variants must lie in (0, {cutn}), got {c}")
            counts = sorted({cutn, *(int(c) for c in cutn_variants)})
            self.weights = p.new(self.P, "f", "prompt_weights")
            self.g_clip = p.new(n3, "f", "g_clip")
            self.dx_direct = p.new(n3, "f", "dx_direct")
            self.fg_ws = p.new(128, "f", "final_grad_ws")
            # clip terms of towers 1..: [T - 1, B] (tower 0's stays in `loss`); SPHERICAL stores them, nothing needs zeroing
            self.loss_towers = p.new((self.T - 1) * B, "f", "losses_towers") if self.T > 1 else None
            if use_augs:  # the augmentation parameters of every window and the four noise fields per cutout
                from .augs import AUG_NP
                self.aug_smax = min(H, W)
                self.aug_prm = p.new(cutn * AUG_NP, "f", "aug_params")
                self.aug_noise = p.new(cutn * 4 * B * 3 * self.aug_smax * self.aug_smax, "f", "aug_noise")
                if cutout_resize == "lanczos3":  # the augmented crops ResizeRight resamples, then their gradient (one buffer, used in turn)
                    self.aug_crop = p.new(cutn * B * 3 * self.aug_smax * self.aug_smax, "f", "aug_crop")
            for m, (cfg, sd) in enumerate(zip(cfgs, sds)):  # range marks of towers 1.. suffixed "#m", tower 0 keeps the plain ones
                tag = f"#{m}" if m else ""
                tw = _Tower(cfg, tag, cutn, p.new(cutn * 3, "i32", "cutout_coords" + tag), p.new(self.P * cfg.output_dim, "f", "target_embeds" + tag),
                            (self.loss, 0) if m == 0 else (self.loss_towers, (m - 1) * B))
                cs = cfg.input_resolution
                if cutout_resize == "lanczos3":
                    from .resize_right import T_MAX
                    # the device tables hold T_MAX = 16 taps per output: lanczos3 with antialiasing needs ceil(6 * S / cs) of them, and
                    # the largest window the reference draws is min(H, W) (cgd/modules.py:40) -- checked here, once, not in the middle of a run
                    if -(-6 * min(H, W) // cs) > T_MAX:
                        raise ValueError(f"cutout_resize='lanczos3': windows up to {min(H, W)} px down to {cs} px need {-(-6 * min(H, W) // cs)} "
                                         f"taps, the device tables hold {T_MAX} (images up to {T_MAX * cs // 6} px)")
                    # a crop is S x S inside a square image; on a non-square one the reference's slicing clips it to Sy x Sx (quirk B3), so
                    # the x axis gets its own tables
                    axis = lambda a: (p.new(cutn * cs, "i32", "rr_left" + a), p.new(cutn * cs * T_MAX, "f", "rr_weights" + a),  # noqa: E731
                                      p.new(cutn, "i32", "rr_taps" + a), p.new(cutn * min(H, W) * 2, "i32", "rr_inverse" + a))
                    tw.rr = axis("")
                    tw.rr_x = axis("_x") if H != W else None
                for c in sorted(counts, key=lambda v: v != cutn):  # the default count first: the others share its weights
                    tw.by_count[c] = clip_tower(cfg, sd, n_images=c * B, device=device, plan=p, parts=vit_streams, suffix=tw.sfx(c),
                                                share=tw.by_count.get(cutn))
                self.towers.append(tw)
            self.vits = {c: tuple(tw.by_count[c] for tw in self.towers) for c in counts}
            # per cutout count (the default count last: its ranges end at "guide"), then per tower in tower order
            for c, (m, tw) in itertools.product(sorted(counts, key=lambda v: v == cutn), enumerate(self.towers)):
                self._emit_cutouts(tw, c, accumulate=m > 0)
            if lpips_sd is not None and init_scale != 0:
                from .lpips import LpipsB200
                # d (init_scale * lpips_vgg(x_in, init).sum()) / d x_in is added to the x_in gradient the cutout backward left in g_clip
                self.lpips = LpipsB200(lpips_sd, B, H, W, p, self.x_inb, self.g_clip, init_scale)
            p.mark("guide")
            # seed_scale > 0: static loss scale; seed_scale = 0 (default): per-image power-of-two scale chosen on the device every step
            dyn = self.seed_scale == 0.0
            if dyn:
                self.seed_f32 = p.new(n3, "f", "seed_f32")
                self.seed_dyn = p.new(2 * B, "f", "seed_dyn")
            p.emit("GUIDE_GRAD", flags=1 if dyn else 0, i=[B, H, W, IN_PAD, self.global_batch],
                   f=[self.scales["tv"], self.scales["rng"], self.scales["sat"], self.seed_scale],
                   p=[(self.x_inb, 0), (self.x0, 0), (self.g_clip, 0), (self.sc, 0), (self.unet.seed, 0), (self.dx_direct, 0), (self.loss, B)]
                   + ([(self.seed_f32, 0), (self.seed_dyn, 0)] if dyn else []), tag="tv+range+sat")
            if dyn:
                p.emit("SEED_QUANT", i=[B, HW, IN_PAD], p=[(self.seed_f32, 0), (self.seed_dyn, 0), (self.unet.seed, 0)], tag="seed scale")
            p.mark("final")
            # use_magnitude clamps by the RMS of the WHOLE batch (cgd/cgd.py:229-232).  With the batch sharded over ranks FINAL_GRAD
            # only writes its partial sums, the host all-reduces the 128 floats (the step's one data-path collective, 512 bytes)
            # and MAG_CLAMP applies the clamp; a single rank keeps the two-launch FINAL_GRAD.
            self.mag_sync = self.use_magnitude and self.world > 1
            p.emit("FINAL_GRAD", flags=(1 if self.use_magnitude else 0) | (2 if dyn else 0) | (4 if self.mag_sync else 0), i=[B, HW],
                   f=[1.0 / self.seed_scale if not dyn else 0.0, 0.05],
                   p=[(self.dx_direct, 0), (self.unet.dx, 0), (self.g, 0), (self.fg_ws, 0)] + ([(self.seed_dyn, 0)] if dyn else []), tag="-grad")
            if self.mag_sync:
                p.mark("mag")
                p.emit("MAG_CLAMP", i=[n3, self.global_batch * 3 * HW], f=[0.05], p=[(self.g, 0), (self.fg_ws, 0)], tag="rms clamp")
        n = n3
        p.mark("upd_anc_g")
        p.emit("SAMPLE_ANCESTRAL", i=[n], p=[(self.mean, 0), (self.var, 0), (self.logvar, 0), (self.g, 0), (self.noise, 0), (self.sc, 0), (self.sample, 0)])
        p.mark("upd_anc")
        p.emit("SAMPLE_ANCESTRAL", i=[n], p=[(self.mean, 0), (self.var, 0), (self.logvar, 0), None, (self.noise, 0), (self.sc, 0), (self.sample, 0)])
        p.mark("upd_ddim_g")
        p.emit("SAMPLE_DDIM", i=[n], p=[(self.unet.x_in, 0), (self.x0, 0), (self.g, 0), (self.noise, 0), (self.sc, 0), (self.sample, 0)])
        p.mark("upd_ddim")
        p.emit("SAMPLE_DDIM", i=[n], p=[(self.unet.x_in, 0), (self.x0, 0), None, (self.noise, 0), (self.sc, 0), (self.sample, 0)])
        p.mark("engine_end")
        if self.input_grad:  # after engine_end and after every other buffer: the step's ops and offsets stay what they are without it
            self._emit_input_grad()
        p.finalize(device)
        self.model = EngineModel(self)
        self.shape = (B, 3, H, W)
        # The pinned staging slot of a step: one region per device buffer the host uploads, in this order (int64 classes first, for
        # alignment).  The host runs ahead of the GPU (a step is ~1 ms of host work and ~10 ms of device work, and nothing
        # synchronises between saved frames), so the async copies of step k may still be queued when the host stages step k+1: the
        # slots are a ring of STAGE_SLOTS, each guarded by the event recorded after its copies were enqueued.
        staged = [self.unet.y_in, self.sc, self.unet.t_in] + ([self.aug_prm] if self.use_augs else [])
        for tw in self.towers:
            staged += [tw.coords] + list(tw.rr or ()) + list(tw.rr_x or ())
        self._slot, size = {}, 0
        for b in staged:  # arena offset of the device buffer -> offset of its region in the slot
            self._slot[b.off], size = size, size + b.nbytes
        pin = self.device.type == "cuda"
        self._stage_ring = [th.zeros(size, dtype=th.uint8, pin_memory=pin) for _ in range(self.STAGE_SLOTS)]
        self._stage_events = [None] * self.STAGE_SLOTS
        self._stage_i = 0
        self._graphs = {}
        self._side_streams = [th.cuda.Stream(device=self.device) for _ in range(max((vt.parts for vt in self.vits.get(self.cutn, ())),
                                                                                    default=1) - 1)] if self.device.type == "cuda" else []
        self._last_out = None
        self._fwd_valid = False
        # bumped by every UNet forward (fused step, unet_forward, model()): an autograd backward or an update whose forward is no longer
        # the latest would differentiate or read someone else's activations
        self.forward_generation = 0
        self._pmv_generation = None
        self.h2d_bytes = 0
        self.d2h_bytes = 0

    def _emit_input_grad(self):
        """the ops of the autograd bridge, each in its own range: PMV_BWD (ag_pmv_bwd), GRAD_SEED (ag_seed), GRAD_UNSCALE without
        (ag_unscale) and with the direct x term (ag_unscale_d)"""
        p, B, HW = self.plan, self.B, self.H * self.W
        n3 = B * 3 * HW
        self.ag_d_out = p.new(B * 6 * HW, "f", "ag_d_model_out")
        self.ag_dyn = p.new(2 * B, "f", "ag_seed_dyn")
        self.ag_dx = p.new(n3, "f", "ag_dx")
        self.ag_dx_direct = p.new(n3, "f", "ag_dx_direct")
        self.ag_pmv_grads = p.new(4 * n3, "f", "ag_pmv_grads")  # upstream grads of pred_xstart | mean | variance | log_variance
        p.mark("ag_pmv_bwd")
        p.emit("PMV_BWD", i=[B, HW], p=[(self.sc, 0), (self.var, 0)] + [(self.ag_pmv_grads, k * n3) for k in range(4)]
               + [(self.ag_d_out, 0), (self.ag_dx_direct, 0)], tag="d p_mean_variance")
        p.mark("ag_seed")
        p.emit("GRAD_SEED", i=[B, HW, IN_PAD], p=[(self.ag_d_out, 0), (self.ag_dyn, 0), (self.unet.seed, 0)], tag="seed of model() backward")
        p.mark("ag_unscale")
        p.emit("GRAD_UNSCALE", i=[B, HW, IN_PAD], p=[(self.unet.dx, 0), None, (self.ag_dyn, 0), (self.unet.seed, 0), (self.ag_dx, 0)],
               tag="dx of model()")
        p.mark("ag_unscale_d")
        p.emit("GRAD_UNSCALE", i=[B, HW, IN_PAD], p=[(self.unet.dx, 0), (self.ag_dx_direct, 0), (self.ag_dyn, 0), (self.unet.seed, 0), (self.ag_dx, 0)],
               tag="dx of p_mean_variance")
        p.mark("ag_end")

    def _emit_cutouts(self, tw, c, accumulate):
        """cutouts -> CLIP (the tower's own op ranges) -> spherical loss -> cutout gradient into g_clip, for `c` windows of tower `tw`;
        `accumulate`: add to g_clip (towers 1..) instead of storing (tower 0), a deterministic sum in tower order"""
        p, B, H, W = self.plan, self.B, self.H, self.W
        sfx, vt = tw.sfx(c), tw.by_count[c]
        cs, ps, kp, D = tw.cfg.input_resolution, tw.cfg.patch_size, tw.cfg.kpad, tw.cfg.output_dim
        dims, win = [B, H, W, c, cs, ps, kp], (tw.coords, 0)
        fwd_f, bwd_f = [*CLIP_MEAN, *CLIP_STD], [0, 0, 0, *CLIP_STD, 1.0 / self.vit_grad_scale]
        p.mark("cut_fwd" + sfx)
        # ResizeRight: flags 1 = the x axis's own tables (non-square images), 2 = resample the augmented crops of aug_crop (use_augs)
        rr_flags = (1 if tw.rr_x else 0) | (2 if self.use_augs else 0)
        smax = min(H, W)
        if tw.rr:
            if self.use_augs:  # crop -> the torchvision pipeline at crop resolution -> ResizeRight, in the reference's order
                p.emit("CUTOUTS_AUG_FWD", flags=1, i=dims + [smax], p=[(self.x_inb, 0), win, (self.aug_crop, 0), (self.aug_prm, 0), (self.aug_noise, 0)],
                       tag="make_cutouts(use_augs crops)")
            p.emit("CUTOUTS_RR_FWD", flags=rr_flags, i=dims + ([smax] if self.use_augs else []), f=fwd_f,
                   p=[(self.aug_crop if self.use_augs else self.x_inb, 0), win, (vt.patches, 0), *((b, 0) for b in tw.rr[:3]),
                      *((b, 0) for b in (tw.rr_x or ())[:3])], tag="make_cutouts(resize_right lanczos3)+normalize")
        elif self.use_augs:
            p.emit("CUTOUTS_AUG_FWD", i=dims + [self.aug_smax], f=fwd_f, p=[(self.x_inb, 0), win, (vt.patches, 0), (self.aug_prm, 0), (self.aug_noise, 0)],
                   tag="make_cutouts(use_augs)+normalize")
        else:
            p.emit("CUTOUTS_FWD", i=dims, f=fwd_f, p=[(self.x_inb, 0), win, (vt.patches, 0)], tag="make_cutouts+normalize")
        p.mark("sph" + sfx)
        p.emit("SPHERICAL", i=[c, B, self.P, D], f=[self.scales["cgs"], self.vit_grad_scale],
               p=[(vt.embeds, 0), (tw.targets, 0), (self.weights, 0), (vt.d_embeds, 0), tw.loss], tag="spherical_dist_loss")
        p.mark("cut_bwd" + sfx)
        if tw.rr:
            p.emit("CUTOUTS_RR_BWD", flags=rr_flags, i=dims + [smax], f=bwd_f,
                   p=[(vt.d_patches, 0), win, (self.aug_crop if self.use_augs else self.g_clip, 0)]
                   + [(b, 0) for t in (tw.rr, tw.rr_x) if t for b in (t[0], t[1], t[3])], tag="d_make_cutouts(resize_right)")
            if self.use_augs:  # d crop -> through the augmentations, scattered into g_clip
                p.emit("FILL", i=[B * 3 * H * W], f=[0.0], p=[(self.g_clip, 0)], tag="zero g_clip")
                p.emit("CUTOUTS_AUG_BWD", flags=1, i=dims + [smax], f=[0, 0, 0, 1, 1, 1, 1.0], p=[(self.aug_crop, 0), win, (self.g_clip, 0), (self.aug_prm, 0)],
                       tag="d_make_cutouts(use_augs crops)")
        elif self.use_augs:
            p.emit("FILL", i=[B * 3 * H * W], f=[0.0], p=[(self.g_clip, 0)], tag="zero g_clip")
            p.emit("CUTOUTS_AUG_BWD", i=dims, f=bwd_f, p=[(vt.d_patches, 0), win, (self.g_clip, 0), (self.aug_prm, 0)], tag="d_make_cutouts(use_augs)")
        else:
            p.emit("CUTOUTS_BWD", flags=2 if accumulate else 0, i=dims, f=bwd_f, p=[(vt.d_patches, 0), win, (self.g_clip, 0)], tag="d_make_cutouts")
        p.mark("cut_end" + sfx)

    # ------------------------------------------------------------------ views
    def v(self, buf, shape=None):
        return self.plan.view(buf, shape)

    def img(self, buf):
        return self.plan.view(buf, self.shape)

    def set_init_image(self, init: th.Tensor, runner=None):
        """init image in [-1, 1] for the LPIPS init loss (cgd/cgd.py:116-120, 220-224); engines built with lpips_sd only"""
        if self.lpips is None:
            raise RuntimeError("engine built without the LPIPS loss (pass lpips_sd= and init_scale != 0)")
        self.lpips.set_init_image(init, runner)

    def set_targets(self, target_embeds, weights: th.Tensor):
        """target_embeds [P, D] (un-normalised is fine: the loss normalises, cgd/losses.py:12-13), or one [P, D_m] per tower of an
        ensemble; weights [P] (shared by the towers) already divided by their |sum| like cgd/cgd.py:102-105."""
        per = _as_list(target_embeds)
        if self.T > 1 and isinstance(target_embeds, th.Tensor):
            raise ValueError(f"engine built with {self.T} CLIP towers: target_embeds must be a sequence of {self.T} [P, D_m] tensors")
        if len(per) != self.T:
            raise ValueError(f"engine built with {self.T} CLIP tower(s), got {len(per)} target tensors")
        for tw, te in zip(self.towers, per):
            if tuple(te.shape) != (self.P, tw.cfg.output_dim):
                raise ValueError(f"engine was built for {self.P} prompt(s) of width {tw.cfg.output_dim}, got {tuple(te.shape)}")
        if self.B > 1 and self.P > 1:
            raise RuntimeError("the reference's spherical-loss broadcast is only defined for batch 1 or a single prompt (quirk B1)")
        for tw, te in zip(self.towers, per):
            self.v(tw.targets, (self.P, tw.cfg.output_dim)).copy_(te.detach().float())
        self.v(self.weights, (self.P,)).copy_(weights.detach().float())

    # ------------------------------------------------------------------ RNG (torch generators: seed parity, SURVEY 8e)
    def local_rows(self, t: th.Tensor) -> th.Tensor:
        return t[self.rank * self.B:(self.rank + 1) * self.B]

    def draw_initial_noise(self, shape=None) -> th.Tensor:
        full = th.randn(self.global_batch, 3, self.H, self.W, device=self.device)
        return self.local_rows(full).contiguous()

    def draw_noise(self) -> th.Tensor:
        """th.randn_like(x) of the reference; with several ranks every rank draws the full batch and keeps its rows."""
        if self.world == 1:
            return self.img(self.noise).normal_()
        full = th.randn(self.global_batch, 3, self.H, self.W, device=self.device)
        self.img(self.noise).copy_(self.local_rows(full))
        return self.img(self.noise)

    def gather_final(self, t: th.Tensor) -> th.Tensor:
        """The run's single collective (SURVEY 8e): every rank's rows of ``t`` ([B_local, ...], e.g. the final sample or
        pred_xstart) -> [B_global, ...] in rank order on every rank.  One ``all_gather_into_tensor`` (NCCL over NVLink; gloo in the
        CPU tests) into a buffer allocated once per shape -- no list of outputs, no copies, no per-call channel set-up after the
        first.  A single rank returns its tensor unchanged."""
        if self.world == 1:
            return t
        import torch.distributed as dist
        t = t.contiguous()
        key = (tuple(t.shape), t.dtype)
        bufs = self.__dict__.setdefault("_gather_bufs", {})
        out = bufs.get(key)
        if out is None:
            out = bufs[key] = th.empty((self.world * t.shape[0],) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
        dist.all_gather_into_tensor(out, t)
        return out

    def draw_classes(self) -> th.Tensor:
        full = th.randint(0, self.unet.num_classes, (self.global_batch,), device=self.device)
        return self.local_rows(full)

    # ------------------------------------------------------------------ the step's op ranges
    def schedule(self, mode, cutn=None, guided=True) -> list:
        """The op ranges of one step in launch order: (mark_a, mark_b) pairs, a ``_Fork`` for the CLIP forward and the CLIP backward of
        each tower, and ``ALL_REDUCE`` where the sharded RMS clamp all-reduces its partial sums.  A guided step runs UNet forward ->
        p_mean_variance -> per tower (cutouts, CLIP fwd, loss, CLIP bwd, cutout gradient) -> LPIPS -> tv / range / sat -> UNet dgrad ->
        -grad (+ clamp) -> update; an unguided one (reduce_clip's skipped steps) UNet forward -> p_mean_variance -> update."""
        steps = [("unet_emb", "unet_bwd"), ("pmv", "cond")]
        if guided and self.towers:
            c = self.cutn if cutn is None else cutn
            if c not in self.vits:
                raise ValueError(f"engine built for cutout counts {sorted(self.vits)}, got {cutn}")
            for tw in self.towers:
                sfx, vt = tw.sfx(c), tw.by_count[c]
                steps += [("cut_fwd" + sfx, "sph" + sfx), _Fork(vt.part_ranges("fwd")), ("sph" + sfx, "cut_bwd" + sfx),
                          _Fork(vt.part_ranges("bwd")), ("cut_bwd" + sfx, "cut_end" + sfx)]
            steps += [("lpips", "lpips_end")] if self.lpips is not None else []
            steps += [("guide", "final"), ("unet_bwd", "unet_end")]
            steps += [("final", "mag"), ALL_REDUCE, ("mag", "upd_anc_g")] if self.mag_sync else [("final", "upd_anc_g")]
        if mode == "ancestral":
            return steps + [("upd_anc_g", "upd_anc") if guided else ("upd_anc", "upd_ddim_g")]
        return steps + [("upd_ddim_g", "upd_ddim") if guided else ("upd_ddim", "engine_end")]

    def _run_all(self, mode, runner=None, cutn=None):
        """one guided step launched range by range, without a CUDA graph; ``runner(mark_a, mark_b)`` stands in for
        ``plan.run_range`` (the tests interpret op lists with it)"""
        self.forward_generation += 1
        self._launch(self.schedule(mode, cutn), runner)

    def _launch(self, steps, runner=None):
        run = runner or self.plan.run_range
        for e in steps:
            if e == ALL_REDUCE:
                import torch.distributed as dist
                dist.all_reduce(self.v(self.fg_ws))
            elif isinstance(e, _Fork) and len(e) > 1 and runner is None and self._side_streams:
                # one CLIP pass per batch slice on parallel streams (fork / join around the current stream; inside CUDA-graph capture
                # this becomes parallel branches of the graph)
                main = th.cuda.current_stream()
                for s, (a, b) in zip(self._side_streams, e[1:]):
                    s.wait_stream(main)
                    self.plan.run_range(a, b, stream=s.cuda_stream)
                self.plan.run_range(*e[0])
                for s in self._side_streams:
                    main.wait_stream(s)
            else:
                for a, b in (e if isinstance(e, _Fork) else [e]):
                    run(a, b)

    def launches_per_step(self, mode="ddim") -> int:
        m = self.plan.marks
        ranges = [r for e in self.schedule(mode) if e != ALL_REDUCE for r in (e if isinstance(e, _Fork) else [e])]
        return sum(self.plan.num_launches(m[a], m[b] - m[a]) for a, b in ranges)

    # ------------------------------------------------------------------ torch.autograd bridge (input_grad=True)
    def _check_autograd_input(self, x):
        if not self.input_grad:
            raise RuntimeError("input gradients through the engine's UNet need an engine built with GuidedStepB200(..., input_grad=True)")
        if tuple(x.shape) != self.shape:
            raise ValueError(f"engine built for inputs of shape {self.shape}, got {tuple(x.shape)}")

    def autograd_forward(self, x, timesteps, y=None) -> int:
        """the UNet forward of ``model()`` under autograd; returns its forward generation"""
        self._check_autograd_input(x)
        self.unet.set_inputs(x.detach(), timesteps, y)
        self.forward_generation += 1
        self.plan.run_range("unet_emb", "unet_bwd")
        return self.forward_generation

    def p_mean_variance_autograd(self, diffusion, x, t_index, y=None) -> dict:
        """p_mean_variance whose outputs carry a ``grad_fn`` back to ``x`` (through the UNet and the p_mean_variance algebra)"""
        self._check_autograd_input(x)
        out = dict(zip(PMV_KEYS, _PMVFunction.apply(x, self, diffusion, t_index, y)))
        out["engine"] = self
        return out

    def autograd_backward(self, generation, d_out=None, pmv_grads=None) -> th.Tensor:
        """d loss / d x from d loss / d model_out (``d_out``) or from the upstream grads of p_mean_variance's four outputs"""
        if th.is_grad_enabled():
            raise RuntimeError("double backward (create_graph=True) through the engine's UNet is not supported")
        if generation != self.forward_generation:
            raise RuntimeError("backward through the engine's UNet after another UNet forward ran on this engine: its activations are "
                               "overwritten (run the backward of each forward before the next forward)")
        run = self.plan.run_range
        if pmv_grads is not None:
            g = self.v(self.ag_pmv_grads, (4,) + self.shape)
            for k, gk in enumerate(pmv_grads):
                g[k].copy_(gk) if gk is not None else g[k].zero_()
            run("ag_pmv_bwd", "ag_seed")
        else:
            self.v(self.ag_d_out, (self.B, 6, self.H, self.W)).copy_(d_out)
        run("ag_seed", "ag_unscale")
        run("unet_bwd", "unet_end")
        run(*(("ag_unscale_d", "ag_end") if pmv_grads is not None else ("ag_unscale", "ag_unscale_d")))
        return self.img(self.ag_dx).clone()

    def drives(self, cond_fn) -> bool:
        """True for this engine's own CondFnB200: the loops then take the fused / segment guidance kernels instead of autograd"""
        return isinstance(cond_fn, CondFnB200) and cond_fn.engine is self

    # ------------------------------------------------------------------ segment-wise execution (API-parity path)
    def _push_scalars(self, sc: np.ndarray):
        self.v(self.sc).copy_(th.from_numpy(sc), non_blocking=True)

    def unet_forward(self, diffusion, x, t_index: int, y=None, fac_index=None) -> dict:
        if fac_index is None:
            fac_index = t_index
        self._cur_t = t_index
        self._push_scalars(diffusion.scalar_table(t_index, fac_index))
        ts = th.full((self.B,), diffusion.model_timestep(t_index), dtype=th.float32)
        self.unet.set_inputs(x, ts.to(self.device, non_blocking=True), y)
        self.forward_generation += 1
        self._pmv_generation = self.forward_generation
        self._launch(self.schedule("ddim", guided=False)[:2])  # UNet forward, p_mean_variance
        self._fwd_valid = True
        out = {"mean": self.img(self.mean), "variance": self.img(self.var), "log_variance": self.img(self.logvar),
               "pred_xstart": self.img(self.x0), "engine": self}
        self._last_out = out
        return out

    def cond_grad(self, diffusion, coords, fac_index: int) -> th.Tensor:
        """-d(loss)/dx for the last unet_forward (what cond_fn returns)."""
        if not self._fwd_valid:
            raise RuntimeError("cond_fn called without a preceding p_mean_variance on this engine")
        if not self.towers:
            raise RuntimeError("engine built without a CLIP tower")
        if fac_index != self._cur_t:  # quirk B2: fac follows the closure's current_timestep, not t
            sc = diffusion.scalar_table(self._cur_t, fac_index)
            self._push_scalars(sc)
            self.plan.run_range("pmv", "cond")
        steps = self.schedule("ddim", len(self._per_tower(coords)[0]))[2:-1]  # the guidance between p_mean_variance and the update
        k = self._stage_acquire()
        self._stage_windows(self._stage_ring[k], coords)
        self._stage_release(k)
        self._launch(steps)
        return self.img(self.g)

    def update(self, diffusion, mode, t_index, g, noise, eta=0.0) -> th.Tensor:
        if self._pmv_generation is not None and self._pmv_generation != self.forward_generation:
            raise RuntimeError("update after another UNet forward ran on this engine: the step's p_mean_variance buffers and x are "
                               "overwritten (a cond_fn must not call the engine's model itself)")
        if mode == "ddim" and eta != 0.0:
            self.v(self.sc)[SC["ETA"]] = float(eta)
        if noise.data_ptr() != self.v(self.noise).data_ptr():
            self.img(self.noise).copy_(noise)
        if g is not None and g.data_ptr() != self.v(self.g).data_ptr():
            self.img(self.g).copy_(g)
        self._launch(self.schedule(mode, guided=g is not None)[-1:])
        self._fwd_valid = False
        return self.img(self.sample).clone()

    # ------------------------------------------------------------------ fused step (CUDA graphs)
    def can_fuse(self, cond_fn, clip_denoised, denoised_fn) -> bool:
        return (isinstance(cond_fn, CondFnB200) and cond_fn.engine is self and not clip_denoised and denoised_fn is None
                and cond_fn.fusable())

    def _per_tower(self, coords):
        """a step's cutout windows -> one window list per tower: one tower takes a flat window list, an ensemble a sequence of
        them (the same count each); no windows at all (an unguided step) -> empty lists"""
        if self.T <= 1 or not len(coords):
            return [list(coords)] * max(self.T, 1)
        per = [list(c) for c in coords]
        if len(per) != self.T or len({len(c) for c in per}) != 1:
            raise ValueError(f"engine built with {self.T} CLIP towers: expected {self.T} window lists of one length, got "
                             f"{[len(c) for c in per]}")
        return per

    STAGE_SLOTS = 4

    def _stage_acquire(self):
        """next slot of the pinned ring; blocks (host only) until the copies last issued from it have executed"""
        k = self._stage_i % self.STAGE_SLOTS
        self._stage_i += 1
        ev = self._stage_events[k]
        if ev is not None:
            ev.synchronize()
        return k

    def _stage_release(self, k):
        if self.device.type == "cuda":
            ev = self._stage_events[k] or th.cuda.Event()
            ev.record(th.cuda.current_stream(self.device))
            self._stage_events[k] = ev

    def _region(self, st, buf, dtype):
        """the region of device buffer `buf` in the pinned slot `st`, as `dtype`"""
        o = self._slot[buf.off]
        return st[o:o + buf.nbytes].view(dtype)

    def _upload(self, st, buf, nbytes=None):
        """async copy of the first `nbytes` (all) of buf's region of the slot `st` into the device buffer"""
        o, n = self._slot[buf.off], buf.nbytes if nbytes is None else nbytes
        self.plan.arena[buf.off:buf.off + n].copy_(st[o:o + n], non_blocking=True)
        self.h2d_bytes += n

    def stage_step(self, sc: np.ndarray, coords, t_model: float, y=None):
        """One pinned staging slot -> small async H2D copies (classes, scalars, timestep, cutout windows)."""
        k = self._stage_acquire()
        st = self._stage_ring[k]
        self.h2d_bytes = 0
        if y is not None and self.unet.cfg.class_cond:
            if y.device.type == "cpu":
                self._region(st, self.unet.y_in, th.int64).copy_(y)
                self._upload(st, self.unet.y_in)
            else:
                self.v(self.unet.y_in).copy_(y)
        self._region(st, self.sc, th.float32).copy_(th.from_numpy(sc))
        self._upload(st, self.sc)
        self._region(st, self.unet.t_in, th.float32).fill_(t_model)
        self._upload(st, self.unet.t_in)
        self._stage_windows(st, coords)
        self._stage_release(k)

    def _stage_windows(self, st, coords):
        """every tower's cutout windows of this step (and the use_augs parameters / ResizeRight tables drawn or built from them) ->
        the pinned slot `st` -> the device; an unguided step has none"""
        if not self.towers:
            return
        per = self._per_tower(coords)
        for ox, oy, size in itertools.chain(*per):  # windows may be clipped at the border (quirk B3) but not empty
            if not (0 <= ox < self.W and 0 <= oy < self.H and size > 0):
                raise RuntimeError(f"cutout window (x={ox}, y={oy}, size={size}) lies outside the {self.H}x{self.W} image: the reference's "
                                   "adaptive_avg_pool2d raises on the empty crop (non-square images, cgd/modules.py:52,61)")
        for tw, windows in zip(self.towers, per):
            if not windows:
                continue
            w = th.tensor(windows, dtype=th.int32).view(-1)
            self._region(st, tw.coords, th.int32)[:w.numel()].copy_(w)
            self._upload(st, tw.coords, w.numel() * 4)
            if self.use_augs:
                self._stage_augs(st, windows)
            if tw.rr:
                self._stage_resize_tables(st, tw, windows)

    def _stage_augs(self, st, windows):
        """use_augs: this step's flip / affine / perspective / grayscale parameters (CPU generator, torchvision's order) and the four
        noise fields per cutout (device generator, the reference's shapes; full batch drawn, own rows kept when sharded)"""
        from . import augs
        S = self.aug_smax
        noise = self.v(self.aug_noise, (self.cutn, 4, self.B, 3, S, S))
        rows = None if self.world == 1 else (self.rank * self.B, (self.rank + 1) * self.B)
        prm = augs.draw_aug_params(windows, self.global_batch, self.H, self.W, noise_device=self.device, noise_out=noise, rows=rows).view(-1)
        self._region(st, self.aug_prm, th.float32)[:prm.numel()].copy_(prm)
        self._upload(st, self.aug_prm, prm.numel() * 4)

    def _stage_resize_tables(self, st, tw, windows):
        """ResizeRight mode: per-cutout resampling tables of this step's crop extents (cached per extent on the host) -> device; the
        first len(windows) rows, so every cutout count reads its own windows' tables"""
        from . import resize_right as rr
        cs, n, smax = tw.cfg.input_resolution, self.cutn, min(self.H, self.W)
        sets = [tw.rr] + ([tw.rr_x] if tw.rr_x else [])
        views = [(self._region(st, l, th.int32).view(n, cs), self._region(st, w, th.float32).view(n, cs, rr.T_MAX), self._region(st, t, th.int32),
                  self._region(st, i, th.int32).view(n, smax, 2)) for l, w, t, i in sets]
        for k, (ox, oy, S) in enumerate(windows):
            # the crop the reference's slicing leaves, Sy x Sx (clipped at the border, quirk B3); y tables first, then x
            for (pl, pw, pt, pi_), ext in zip(views, (min(S, self.H - oy), min(S, self.W - ox))):
                l, w, T = rr.tables(int(ext), cs)
                pl[k].copy_(l)
                pw[k].copy_(w)
                pt[k] = T
                pi_[k, :ext].copy_(rr.inverse_ranges(l, T, int(ext)))
        for b in itertools.chain(*sets):
            self._upload(st, b)

    def fused_step(self, diffusion, mode, t_index, img, y, cond_fn, eta=0.0) -> dict:
        # RNG order of the reference: the ancestral sampler draws its noise BEFORE cond_fn (whose MakeCutouts draws the windows
        # from the CPU generator), DDIM AFTER it.  On a GPU the two come from different generators and the order is immaterial;
        # it is kept anyway so a CPU run (tests/test_loops_cpu.py) consumes the default generator exactly like the reference.
        fac_index = cond_fn.current_timestep
        # reduce_clip (cgd/cgd.py:157-164): on the steps its rule skips, cond_fn returns zeros -- no cutout windows are drawn, CLIP
        # and both backward passes have nothing to do, the sampler takes its unguided update.  Those steps replay a second, short
        # graph (UNet forward -> p_mean_variance -> update), which is where the option's speed-up comes from.
        guided = not cond_fn.skips_guidance()
        if mode == "ancestral":
            self.draw_noise()
        coords = cond_fn.next_coords(self.H, self.W) if guided else []
        if mode != "ancestral":
            self.draw_noise()
        sc = diffusion.scalar_table(t_index, fac_index, eta)
        self.stage_step(sc, coords, diffusion.model_timestep(t_index), y)
        xin = self.img(self.unet.x_in)
        if img.data_ptr() != xin.data_ptr():
            xin.copy_(img, non_blocking=True)
        self.replay(mode, len(self._per_tower(coords)[0]) if (self.cutn and guided) else None, guided=guided)
        return {"sample": self.img(self.sample).clone(), "pred_xstart": self.img(self.x0).clone()}

    def replay(self, mode, cutn=None, guided=True):
        """one step from CUDA graphs: the schedule cut at its host all-reduce into segments, one graph per segment, captured on first
        use after one eager run (which sets kernel attributes and touches every buffer), then replayed with the all-reduce between"""
        steps = self.schedule(mode, cutn, guided)
        self.forward_generation += 1
        if not self.use_graph:
            self._launch(steps)
            return
        key = (mode, (None if cutn == self.cutn else cutn) if guided else "unguided")
        graphs = self._graphs.get(key)
        if graphs is None:
            self._launch(steps)
            th.cuda.synchronize()
            graphs = self._graphs[key] = []
            cuts = [-1] + [k for k, e in enumerate(steps) if e == ALL_REDUCE] + [len(steps)]
            for a, b in zip(cuts, cuts[1:]):
                graphs.append(th.cuda.CUDAGraph())
                with th.cuda.graph(graphs[-1]):
                    self._launch(steps[a + 1:b])
        for k, g in enumerate(graphs):
            if k:
                self._launch([ALL_REDUCE])
            g.replay()

    def losses(self) -> dict:
        """per-image loss terms of the last step (device->host sync; logging only, like tqdm.write at cgd/cgd.py:234-236)"""
        l = self.v(self.loss, (4, self.B)).cpu()
        per = l[0:1] if self.loss_towers is None else th.cat([l[0:1], self.v(self.loss_towers, (self.T - 1, self.B)).cpu()])
        # "clip": the sum over the towers, in tower order; "clip_per_tower": [T, B]
        d = {"clip": per.sum(0), "clip_per_tower": per, "tv": l[1], "range": l[2], "sat": l[3]}
        if self.lpips is not None:
            d["init"] = self.lpips.loss_value().cpu() * self.lpips.init_scale
        return d


class CondFnB200:
    """The reference's ``cond_fn(x, t, out, y=None)`` closure (cgd/cgd.py:151-239) bound to an engine, including its
    ``current_timestep`` bookkeeping (quirk B2) and the reduce_clip / progressive_cutout / cached_cutouts switches."""

    with_grad = True

    def __init__(self, engine: GuidedStepB200, diffusion, make_cutouts, *, cached_cutouts=False, reduce_clip=False,
                 progressive_cutout=False):
        """``make_cutouts``: one ``MakeCutouts``, or one per CLIP tower of an ensemble engine (in tower order, the same count each)"""
        self.cutouts = _as_list(make_cutouts)
        if not self.cutouts or len({mk.cutn for mk in self.cutouts}) != 1:
            raise ValueError("make_cutouts: one MakeCutouts or a non-empty sequence of them with the same num_cutouts")
        if engine.cutn and len(self.cutouts) != getattr(engine, "T", 1):  # (duck-typed engines without towers count as one)
            raise ValueError(f"engine built with {engine.T} CLIP tower(s), got {len(self.cutouts)} MakeCutouts")
        make_cutouts = self.cutouts[0]
        self.engine, self.diffusion, self.make_cutouts = engine, diffusion, make_cutouts
        self.cached_cutouts, self.reduce_clip, self.progressive_cutout = cached_cutouts, reduce_clip, progressive_cutout
        self.current_timestep = diffusion.num_timesteps - 1  # cgd/cgd.py:265
        # the schedule follows the user's num_cutouts (make_cutouts.cutn); for num_cutouts < 16 its middle count max(8, n // 2)
        # EXCEEDS num_cutouts, so the engine is built for the largest count of the schedule (cgd.py does that)
        counts = self.progressive_counts(make_cutouts.cutn) if progressive_cutout else (make_cutouts.cutn,)
        missing = set(counts) - set(engine.vits)
        if missing and engine.cutn:
            raise ValueError(f"engine built for cutout counts {sorted(engine.vits)}; this cond_fn needs {sorted(set(counts))} "
                             "(GuidedStepB200(num_cutouts=max, cutn_variants=the others))")

    @staticmethod
    def progressive_counts(num_cutouts: int) -> tuple:
        """the three cutout counts of the reference's schedule (cgd/cgd.py:167-175)"""
        return (max(4, num_cutouts // 4), max(8, num_cutouts // 2), num_cutouts)

    def current_cutn(self) -> int:
        n = self.make_cutouts.cutn
        if not self.progressive_cutout:
            return n
        total = self.diffusion.num_timesteps
        pct = (total - self.current_timestep) / total
        lo, mid, hi = self.progressive_counts(n)
        return lo if pct < 0.3 else (mid if pct < 0.7 else hi)

    def fusable(self):
        return True

    def skips_guidance(self) -> bool:
        """reduce_clip's rule (cgd/cgd.py:157-164): below 70 % progress CLIP guidance runs on every 4th step only (the first 20 % are
        skipped altogether through skip_timesteps, cgd/cgd.py:141-144); on the other steps cond_fn returns zeros"""
        if not self.reduce_clip:
            return False
        total = self.diffusion.num_timesteps
        pct = (total - self.current_timestep) / total
        return pct < 0.7 and int((pct - 0.2) * total) % 4 != 0

    def step_done(self):  # cgd/cgd.py:267
        self.current_timestep -= 1

    def next_coords(self, H, W):
        """this step's windows: a flat list for one tower; with several, one list per tower, drawn in tower order (each tower
        with its own min_size = min(H, W, cut_size))"""
        n = self.current_cutn()
        per = [mk.coords_for(H, W, use_cache=self.cached_cutouts, num_cutouts_override=n) for mk in self.cutouts]
        return per[0] if len(per) == 1 else per

    def __call__(self, x, t, out, y=None):
        eng = self.engine
        if out.get("engine") is not eng:
            raise RuntimeError("cond_fn: `out` must come from this engine's p_mean_variance (the UNet backward re-enters its saved "
                               "activations)")
        if self.skips_guidance():  # cgd/cgd.py:157-164
            return th.zeros_like(x)
        coords = self.next_coords(x.shape[2], x.shape[3])
        return eng.cond_grad(self.diffusion, coords, self.current_timestep)
