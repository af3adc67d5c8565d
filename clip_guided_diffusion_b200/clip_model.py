"""``load_clip()``: a CLIP model whose ``encode_image`` runs this package's visual towers (vit.py, rn.py) under torch.autograd.

The reference's entry point is ``cgd/clip_util.py: load_clip(model_name, device) -> (clip_model, clip_size)``; user code calls
``clip_model.encode_image(clip_in)`` and reads ``clip_model.visual.input_resolution``.  Here ``encode_image`` is differentiable: a
PyTorch cond_fn's ``th.autograd.grad(loss, x)`` flows through it into ``clip_in`` and on through the user's cutouts and, with an
``input_grad`` engine's ``engine.model``, through the UNet, so both networks of a guided step run on the device kernels.

One plan holds the tower (built for ``max_images`` images, forward and input gradient) and three ops of csrc/clip_autograd.cu, each in
its own range after the tower's ``vit_end``::

    clip_in -> CLIP_PATCHIFY -> tower forward ("vit_fwd".."vit_bwd") -> embeds
    d_embeds -> CLIP_SEED -> tower backward ("vit_bwd".."vit_end") -> CLIP_UNPATCHIFY -> d clip_in

The host copies the caller's tensor into fixed fp32 staging buffers of the arena and clones the results out, as the UNet bridge
(guidance.py, ``_UNetFunction``) does.  Decisions:

1. One size, padded: a call with N <= ``max_images`` images runs the whole tower; rows N.. are zero in the forward, their embeddings
   are dropped and their gradients are zero.  Images are independent in every op of both towers, so padding cannot change a real row
   beyond the order of a split-K sum.  N > ``max_images`` raises.
2. ``clip_in`` may be fp32, fp16 or bf16 (copied exactly into fp32); the patches are rounded to fp16 once, which is what the
   reference's ``image.type(self.dtype)`` does on its fp16 CUDA model.  Embeddings come back fp32 (the projection is fp32 here), the
   input gradient in ``clip_in``'s dtype.
3. Without grad mode or without ``clip_in.requires_grad``, ``encode_image`` returns a fresh fp32 tensor and records nothing.
4. Every forward bumps a generation counter; a backward whose forward is no longer the latest raises (its activations are
   overwritten), so is ``create_graph=True``.  ``retain_graph=True`` may run a backward twice, with the same bits.
5. No weight gradients: the weights are constants of the plan.
"""
from __future__ import annotations

import torch as th

from .cgd import CACHE_PATH, _clip_tower, _require_cuda
from .guidance import clip_tower
from .plan import Plan
from .text import TextB200, text_config_from_state_dict

# CLIP_SEED's target for the largest |d embeds| of an image: measured with scripts/clip_seed_band.py (DESIGN.md section 2)
CLIP_SEED_BAND = 512.0

_INPUT_DTYPES = (th.float32, th.float16, th.bfloat16)


class ClipVisual:
    """``clip_model.visual``: what callers read of the tower (``input_resolution``, ``output_dim``)"""

    def __init__(self, cfg):
        self.cfg = cfg
        self.input_resolution = cfg.input_resolution
        self.output_dim = cfg.output_dim


class ClipModelB200:
    """A CLIP model for guidance: ``encode_image`` (differentiable, up to ``max_images`` images per call) and ``encode_text``
    (forward only, token ids).  Built by ``load_clip``."""

    def __init__(self, cfg, state_dict: dict, max_images: int = 16, device="cuda"):
        if int(max_images) < 1:
            raise ValueError(f"max_images={max_images}: at least one image per call")
        self.cfg, self.max_images = cfg, int(max_images)
        self.visual = ClipVisual(cfg)
        self.dtype = th.float16  # the precision of the tower's activations, like the reference's fp16 CUDA model
        self._text_sd = {k: v for k, v in state_dict.items() if not k.startswith("visual.")}  # references, for encode_text
        p = self.plan = Plan()
        n, R, D = self.max_images, cfg.input_resolution, cfg.output_dim
        self.tower = clip_tower(cfg, state_dict, n_images=n, device=device, plan=p, build_backward=True)
        self.x_in = p.new(n * 3 * R * R, "f", "clip_in")
        self.d_in = p.new(n * D, "f", "d_embeds_in")
        self.dyn = p.new(n, "f", "clip_seed_scale")
        self.dx = p.new(n * 3 * R * R, "f", "d_clip_in")
        dims = [n, n, R, cfg.patch_size, cfg.kpad]
        p.mark("clip_patchify")
        p.emit("CLIP_PATCHIFY", i=dims, p=[(self.x_in, 0), (self.tower.patches, 0)], tag="clip_in -> patches")
        p.mark("clip_seed")
        p.emit("CLIP_SEED", i=[n, n, D], f=[CLIP_SEED_BAND], p=[(self.d_in, 0), (self.tower.d_embeds, 0), (self.dyn, 0)], tag="seed of encode_image backward")
        p.mark("clip_unpatchify")
        p.emit("CLIP_UNPATCHIFY", i=dims, p=[(self.tower.d_patches, 0), (self.dyn, 0), (self.dx, 0)], tag="d_patches -> d clip_in")
        p.mark("clip_end")
        p.finalize(device)
        self.device = p.arena.device
        self.forward_generation = 0

    # ------------------------------------------------------------------ the reference's clip_model surface
    def encode_image(self, image: th.Tensor) -> th.Tensor:
        """image: [N, 3, R, R] CLIP-normalised, N <= max_images, fp32 / fp16 / bf16 on the model's device -> fp32 [N, D].  With grad
        mode on and ``image.requires_grad`` the result has a ``grad_fn`` whose backward runs the tower's input gradient."""
        self._check_image(image)
        if th.is_grad_enabled() and image.requires_grad:
            return _ClipFunction.apply(image, self)
        self.forward(image)
        return self.embeds(image.shape[0])

    def encode_text(self, text) -> th.Tensor:
        """token ids [P, context] (``clip.tokenize``'s or ``tokenizer.tokenize``'s output) -> fp32 [P, D], forward only, on a one-shot text
        tower released before returning"""
        ids = th.as_tensor(text)
        if ids.dim() == 1:
            ids = ids[None]
        cfg = text_config_from_state_dict(self._text_sd, act=getattr(self.cfg, "act", "quick_gelu"))  # the visual tower's MLP activation
        tower = TextB200(cfg, self._text_sd, ids.shape[0], self.device)
        emb = tower.encode(ids)
        del tower
        return emb

    # the no-op chain of EngineModel: the reference's load_clip calls .eval().requires_grad_(False).to(device)
    def parameters(self):
        yield self.plan.arena

    def eval(self):
        return self

    def requires_grad_(self, flag=False):
        return self

    def to(self, device=None, *a, **k):
        if device is not None and not isinstance(device, th.dtype) and th.device(device).type != self.device.type:
            raise RuntimeError(f"the CLIP model lives on {self.device}; call load_clip once per device")
        return self

    # ------------------------------------------------------------------ the plan's ranges
    def _check_image(self, image):
        R = self.cfg.input_resolution
        if not isinstance(image, th.Tensor) or image.dim() != 4 or image.shape[1] != 3 or tuple(image.shape[2:]) != (R, R):
            raise ValueError(f"encode_image takes [N, 3, {R}, {R}] images (this tower's input resolution), got "
                             f"{tuple(image.shape) if isinstance(image, th.Tensor) else type(image).__name__}")
        if not 1 <= image.shape[0] <= self.max_images:
            raise ValueError(f"encode_image got {image.shape[0]} images: this model was built for 1..{self.max_images} per call "
                             "(load_clip(..., max_images=N))")
        if image.dtype not in _INPUT_DTYPES:
            raise ValueError(f"encode_image takes fp32, fp16 or bf16 images, got {image.dtype}")
        if image.device != self.device:
            raise ValueError(f"encode_image: the images are on {image.device}, the model on {self.device}")

    def forward(self, image: th.Tensor) -> int:
        """stage ``image`` (rows N.. zero), run CLIP_PATCHIFY and the tower forward; returns the forward's generation"""
        n = image.shape[0]
        x = self.plan.view(self.x_in, (self.max_images,) + tuple(image.shape[1:]))
        x[:n].copy_(image.detach())
        x[n:].zero_()
        self.forward_generation += 1
        self.plan.run_range("clip_patchify", "clip_seed")
        self.plan.run_range("vit_fwd", "vit_bwd")
        return self.forward_generation

    def embeds(self, n: int) -> th.Tensor:
        return self.plan.view(self.tower.embeds, (self.max_images, self.cfg.output_dim))[:n].clone()

    def backward(self, generation: int, d_embeds: th.Tensor) -> th.Tensor:
        """d loss / d clip_in (fp32 [N, 3, R, R]) from d loss / d embeds of the forward ``generation``"""
        if th.is_grad_enabled():
            raise RuntimeError("double backward (create_graph=True) through encode_image is not supported")
        if generation != self.forward_generation:
            raise RuntimeError("backward through encode_image after a later encode_image call on this model: its activations are "
                               "overwritten.  Two encode_image calls under one backward are not supported: pass all images to one call "
                               "(up to max_images), or take the gradient of each call before the next")
        n = d_embeds.shape[0]
        d = self.plan.view(self.d_in, (self.max_images, self.cfg.output_dim))
        d[:n].copy_(d_embeds)
        d[n:].zero_()
        self.plan.run_range("clip_seed", "clip_unpatchify")
        self.plan.run_range("vit_bwd", "vit_end")
        self.plan.run_range("clip_unpatchify", "clip_end")
        R = self.cfg.input_resolution
        return self.plan.view(self.dx, (self.max_images, 3, R, R))[:n].clone()


class _ClipFunction(th.autograd.Function):
    """``encode_image`` under autograd: forward = CLIP_PATCHIFY + tower forward; backward = CLIP_SEED -> tower backward ->
    CLIP_UNPATCHIFY.  The backward re-enters the tower's activations, so it must follow the latest forward."""

    @staticmethod
    def forward(ctx, image, model):
        ctx.model, ctx.gen, ctx.dtype = model, model.forward(image), image.dtype
        return model.embeds(image.shape[0])

    @staticmethod
    def backward(ctx, d_embeds):
        return ctx.model.backward(ctx.gen, d_embeds).to(ctx.dtype), None


def load_clip(model_name: str = "ViT-B/32", device: str = "cuda", *, max_images: int = 16, clip_state_dict: dict = None,
              checkpoints_dir: str = CACHE_PATH):
    """cgd/clip_util.py's ``load_clip(model_name, device) -> (clip_model, clip_size)`` on this package's towers.  ``model_name`` is a
    tower name (ViT-B/32, ViT-B/16, ViT-L/14, ViT-L/14@336px, RN50, RN101, RN50x4, RN50x16) whose checkpoint lies under
    ``checkpoints_dir/clip/``, an OpenCLIP tower ``"open_clip:<arch>"`` (vit.OPEN_CLIP_CONFIGS; weights under ``checkpoints_dir/open_clip/``),
    or a path to a CLIP checkpoint file; ``clip_state_dict=`` gives the weights directly (the architecture is read from its keys, except
    for an ``open_clip:`` name, whose architecture the weights are checked against).  ``max_images``: the most images one ``encode_image`` call takes (the reference's ``num_cutouts`` x batch)."""
    _require_cuda(device)
    sd, cfg = _clip_tower(model_name, clip_state_dict, checkpoints_dir)
    model = ClipModelB200(cfg, sd, max_images, device)
    return model, cfg.input_resolution


__all__ = ["CLIP_SEED_BAND", "ClipModelB200", "load_clip"]
