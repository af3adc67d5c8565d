"""Sampler host logic: schedules, respacing and the guided-diffusion step/loop signatures.

Mirrors [3P] ``guided_diffusion.gaussian_diffusion.GaussianDiffusion`` / ``respace.SpacedDiffusion`` as reached
from the reference at cgd/cgd.py:242-262 (loops, kwargs) and cgd/cgd.py:142,154,177,265 (``num_timesteps``,
``sqrt_one_minus_alphas_cumprod``): epsilon prediction, LEARNED_RANGE variance, the fork's ``*_with_grad`` steps
with ``skip_timesteps`` / ``init_image`` / ``randomize_class`` / ``cond_fn_with_grad``.  The float64 numpy tables are
kept (they are part of the surface); all per-pixel algebra runs in the CUDA kernels of the engine
(``guidance.GuidedStepB200``): this file only selects per-timestep scalars and sequences launches.
"""
from __future__ import annotations

import math

import numpy as np
import torch as th

from ._lib import SC


def get_named_beta_schedule(name: str, T: int) -> np.ndarray:
    if name == "linear":
        scale = 1000.0 / T
        return np.linspace(scale * 0.0001, scale * 0.02, T, dtype=np.float64)
    if name == "cosine":
        def abar(s):
            return math.cos((s + 0.008) / 1.008 * math.pi / 2) ** 2
        return np.array([min(1 - abar((i + 1) / T) / abar(i / T), 0.999) for i in range(T)], dtype=np.float64)
    raise NotImplementedError(f"unknown beta schedule: {name}")


def space_timesteps(num_timesteps: int, section_counts) -> set:
    if isinstance(section_counts, str):
        if section_counts.startswith("ddim"):
            desired = int(section_counts[len("ddim"):])
            for stride in range(1, num_timesteps):
                if len(range(0, num_timesteps, stride)) == desired:
                    return set(range(0, num_timesteps, stride))
            raise ValueError(f"cannot create exactly {desired} steps with an integer stride")
        section_counts = [int(x) for x in section_counts.split(",")]
    size_per, extra = divmod(num_timesteps, len(section_counts))
    start, steps = 0, []
    for i, count in enumerate(section_counts):
        size = size_per + (1 if i < extra else 0)
        if size < count:
            raise ValueError(f"cannot divide section of {size} steps into {count}")
        stride = 1 if count <= 1 else (size - 1) / (count - 1)
        cur = 0.0
        for _ in range(count):
            steps.append(start + round(cur))
            cur += stride
        start += size
    return set(steps)


class GaussianDiffusion:
    def __init__(self, betas, rescale_timesteps: bool = False):
        betas = np.array(betas, dtype=np.float64)
        assert betas.ndim == 1 and (betas > 0).all() and (betas <= 1).all()
        self.betas = betas
        self.rescale_timesteps = rescale_timesteps
        self.num_timesteps = int(betas.shape[0])
        alphas = 1.0 - betas
        self.alphas_cumprod = np.cumprod(alphas, axis=0)
        self.alphas_cumprod_prev = np.append(1.0, self.alphas_cumprod[:-1])
        self.alphas_cumprod_next = np.append(self.alphas_cumprod[1:], 0.0)
        self.sqrt_alphas_cumprod = np.sqrt(self.alphas_cumprod)
        self.sqrt_one_minus_alphas_cumprod = np.sqrt(1.0 - self.alphas_cumprod)
        self.log_one_minus_alphas_cumprod = np.log(1.0 - self.alphas_cumprod)
        self.sqrt_recip_alphas_cumprod = np.sqrt(1.0 / self.alphas_cumprod)
        self.sqrt_recipm1_alphas_cumprod = np.sqrt(1.0 / self.alphas_cumprod - 1)
        self.posterior_variance = betas * (1.0 - self.alphas_cumprod_prev) / (1.0 - self.alphas_cumprod)
        self.posterior_log_variance_clipped = np.log(np.append(self.posterior_variance[1], self.posterior_variance[1:]))
        self.posterior_mean_coef1 = betas * np.sqrt(self.alphas_cumprod_prev) / (1.0 - self.alphas_cumprod)
        self.posterior_mean_coef2 = (1.0 - self.alphas_cumprod_prev) * np.sqrt(alphas) / (1.0 - self.alphas_cumprod)
        self.timestep_map = list(range(self.num_timesteps))
        self.original_num_steps = self.num_timesteps

    # ---- per-timestep scalar table consumed by the kernels (include/cgd_b200.h CGD_SC_*)
    def scalar_table(self, t: int, fac_index: int = None, eta: float = 0.0) -> np.ndarray:
        sc = np.zeros(SC["COUNT"], dtype=np.float32)
        sc[SC["SQRT_RECIP_AC"]] = self.sqrt_recip_alphas_cumprod[t]
        sc[SC["SQRT_RECIPM1_AC"]] = self.sqrt_recipm1_alphas_cumprod[t]
        sc[SC["POST_COEF1"]] = self.posterior_mean_coef1[t]
        sc[SC["POST_COEF2"]] = self.posterior_mean_coef2[t]
        sc[SC["MIN_LOG"]] = self.posterior_log_variance_clipped[t]
        sc[SC["MAX_LOG"]] = np.log(self.betas[t])
        sc[SC["NONZERO"]] = 0.0 if t == 0 else 1.0
        sc[SC["SQRT_1M_AC"]] = np.float32(np.sqrt(np.float32(1.0) - np.float32(self.alphas_cumprod[t])))  # (1 - abar).sqrt() in fp32
        sc[SC["AC_PREV"]] = self.alphas_cumprod_prev[t]
        sc[SC["AC"]] = self.alphas_cumprod[t]
        sc[SC["ETA"]] = eta
        if fac_index is not None:  # cgd/cgd.py:177-178: fac indexed by the closure's current_timestep, (1 - fac) in fp64
            fac = self.sqrt_one_minus_alphas_cumprod[fac_index]
            sc[SC["FAC"]] = fac
            sc[SC["ONE_MINUS_FAC"]] = 1.0 - fac
        return sc

    def model_timestep(self, t: int) -> float:
        """what the UNet receives for step index t (SpacedDiffusion's _WrappedModel + rescale_timesteps)"""
        ts = float(self.timestep_map[t])
        if self.rescale_timesteps:
            ts = ts * (1000.0 / self.original_num_steps)
        return ts

    # ---- closed forms on tensors (q_sample is the only one the loops need on the host side)
    def q_sample(self, x_start, t, noise=None):
        if noise is None:
            noise = th.randn_like(x_start)
        ti = _uniform_t(t)
        return float(self.sqrt_alphas_cumprod[ti]) * x_start + float(self.sqrt_one_minus_alphas_cumprod[ti]) * noise

    # ---- one step.  `model` is the engine's UNet handle (guidance.EngineModel)
    def p_mean_variance(self, model, x, t, clip_denoised=True, denoised_fn=None, model_kwargs=None):
        _require(not clip_denoised and denoised_fn is None,
                 "the H100 step implements the reference's configuration (clip_denoised=False, no denoised_fn; cgd/cgd.py:253)")
        engine = _engine_of(model)
        return engine.unet_forward(self, x, _uniform_t(t), (model_kwargs or {}).get("y"))

    def _step(self, mode, model, x, t, clip_denoised, denoised_fn, cond_fn, model_kwargs, eta=0.0, noise=None):
        engine = _engine_of(model)
        ti = _uniform_t(t)
        out = self.p_mean_variance(model, x, t, clip_denoised, denoised_fn, model_kwargs)
        if mode == "ancestral" and noise is None:
            noise = engine.draw_noise()  # drawn BEFORE cond_fn (SURVEY 3.2)
        g = cond_fn(x, t, out, **(model_kwargs or {})) if cond_fn is not None else None
        if mode == "ddim" and noise is None:
            noise = engine.draw_noise()  # drawn AFTER cond_fn, consumed even when eta == 0 (SURVEY 3.3)
        sample = engine.update(self, mode, ti, g, noise, eta)
        return {"sample": sample, "pred_xstart": out["pred_xstart"]}

    def p_sample(self, model, x, t, clip_denoised=True, denoised_fn=None, cond_fn=None, model_kwargs=None):
        _require(cond_fn is None or getattr(cond_fn, "with_grad", False),
                 "cond_fn must be a CondFnB200 (the reference always samples with cond_fn_with_grad=True)")
        return self._step("ancestral", model, x, t, clip_denoised, denoised_fn, cond_fn, model_kwargs)

    def p_sample_with_grad(self, model, x, t, clip_denoised=True, denoised_fn=None, cond_fn=None, model_kwargs=None):
        return self._step("ancestral", model, x, t, clip_denoised, denoised_fn, cond_fn, model_kwargs)

    def ddim_sample(self, model, x, t, clip_denoised=True, denoised_fn=None, cond_fn=None, model_kwargs=None, eta=0.0):
        return self._step("ddim", model, x, t, clip_denoised, denoised_fn, cond_fn, model_kwargs, eta=eta)

    def ddim_sample_with_grad(self, model, x, t, clip_denoised=True, denoised_fn=None, cond_fn=None, model_kwargs=None, eta=0.0):
        return self._step("ddim", model, x, t, clip_denoised, denoised_fn, cond_fn, model_kwargs, eta=eta)

    # ---- loops (same kwargs as the fork's; call site cgd/cgd.py:250-262)
    def _loop(self, mode, model, shape, noise, clip_denoised, denoised_fn, cond_fn, model_kwargs, device, progress,
              skip_timesteps, init_image, randomize_class, eta=0.0):
        engine = _engine_of(model)
        device = device or engine.device
        img = noise if noise is not None else engine.draw_initial_noise(shape)
        if skip_timesteps and init_image is None:
            init_image = th.zeros_like(img)
        indices = list(range(self.num_timesteps - skip_timesteps))[::-1]
        if init_image is not None:
            img = self.q_sample(engine.local_rows(init_image.expand(engine.global_batch, *init_image.shape[1:])
                                                  if init_image.shape[0] == 1 else init_image), indices[0], img)
        model_kwargs = dict(model_kwargs or {})
        if progress:
            from tqdm.auto import tqdm
            indices = tqdm(indices)
        fused = engine.can_fuse(cond_fn, clip_denoised, denoised_fn)
        for i in indices:
            if randomize_class and "y" in model_kwargs:
                model_kwargs["y"] = engine.draw_classes()
            if fused:
                out = engine.fused_step(self, mode, i, img, model_kwargs.get("y"), cond_fn, eta)
            else:
                t = th.full((shape[0],), i, device=device, dtype=th.long)
                out = self._step(mode, model, img, t, clip_denoised, denoised_fn, cond_fn, model_kwargs, eta=eta)
            yield out
            img = out["sample"]

    def p_sample_loop_progressive(self, model, shape, noise=None, clip_denoised=True, denoised_fn=None, cond_fn=None,
                                  model_kwargs=None, device=None, progress=False, skip_timesteps=0, init_image=None,
                                  randomize_class=False, cond_fn_with_grad=False):
        yield from self._loop("ancestral", model, shape, noise, clip_denoised, denoised_fn, cond_fn, model_kwargs, device, progress,
                              skip_timesteps, init_image, randomize_class)

    def ddim_sample_loop_progressive(self, model, shape, noise=None, clip_denoised=True, denoised_fn=None, cond_fn=None,
                                     model_kwargs=None, device=None, progress=False, eta=0.0, skip_timesteps=0, init_image=None,
                                     randomize_class=False, cond_fn_with_grad=False):
        yield from self._loop("ddim", model, shape, noise, clip_denoised, denoised_fn, cond_fn, model_kwargs, device, progress,
                              skip_timesteps, init_image, randomize_class, eta=eta)

    def p_sample_loop(self, model, shape, **kw):
        final = None
        for final in self.p_sample_loop_progressive(model, shape, **kw):
            pass
        return final["sample"]

    def ddim_sample_loop(self, model, shape, **kw):
        final = None
        for final in self.ddim_sample_loop_progressive(model, shape, **kw):
            pass
        return final["sample"]


class SpacedDiffusion(GaussianDiffusion):
    """Sub-sequence of a base process; betas recomputed so the kept alpha-bars are reproduced (respace.py)."""

    def __init__(self, use_timesteps, betas, rescale_timesteps: bool = False):
        self.use_timesteps = set(use_timesteps)
        base = GaussianDiffusion(betas)
        last, new_betas, tmap = 1.0, [], []
        for i, ac in enumerate(base.alphas_cumprod):
            if i in self.use_timesteps:
                new_betas.append(1 - ac / last)
                last = ac
                tmap.append(i)
        super().__init__(new_betas, rescale_timesteps=rescale_timesteps)
        self.timestep_map = tmap
        self.original_num_steps = len(betas)


def create_gaussian_diffusion(steps=1000, noise_schedule="linear", timestep_respacing="", rescale_timesteps=False) -> SpacedDiffusion:
    """[3P] script_util.create_gaussian_diffusion with learn_sigma=True (every published checkpoint)."""
    betas = get_named_beta_schedule(noise_schedule, steps)
    if not timestep_respacing:
        timestep_respacing = [steps]
    return SpacedDiffusion(space_timesteps(steps, timestep_respacing), betas, rescale_timesteps=rescale_timesteps)


# ---------------------------------------------------------------------- helpers
def _require(cond, msg):
    if not cond:
        raise NotImplementedError(msg)


def _engine_of(model):
    eng = getattr(model, "engine", None)
    if eng is None:
        raise TypeError("model must be the UNet handle of a GuidedStepB200 engine (engine.model); the sampling step has no "
                        "PyTorch / CPU fallback")
    return eng


def _uniform_t(t) -> int:
    if isinstance(t, (int, np.integer)):
        return int(t)
    vals = t.tolist() if hasattr(t, "tolist") else list(t)
    if isinstance(vals, (int, float)):
        return int(vals)
    if any(v != vals[0] for v in vals):
        raise NotImplementedError("per-sample timesteps are not supported: the sampling loops use one timestep per batch")
    return int(vals[0])
