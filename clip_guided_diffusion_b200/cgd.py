"""``clip_guided_diffusion(...)`` -- the reference's orchestrator surface (cgd/cgd.py:19-283) over the H100 engine.

Same keyword arguments and the same generator contract (yields ``(batch_idx, png_path)``); set-up stays Python and
runs once (seed, prompt encoding, weight loading, cutout cache), the per-timestep work is the engine's fused step.
Out of scope here, exactly as SURVEY.md section 2 marks them: checkpoint download, W&B, GIF/MP4,
image prompts (the reference's ``encode_image_prompt`` crashes, quirk B5).  The LPIPS init loss (``init_image`` + ``init_scale``)
runs on the engine when the VGG weights are given (``lpips_state_dict=``) or the ``lpips`` package is installed.

Weights: pass ``unet_state_dict`` / ``clip_state_dict`` (upstream key layout), or have the reference's checkpoints on
disk under ``checkpoints_dir`` (``256x256_diffusion.pt`` ..., ``clip/ViT-B-32.pt``).  Text prompts need a text tower:
either pass ``target_embeds`` / ``weights`` directly or have the ``clip`` package importable (used once, outside the hot
path, like cgd/clip_util.py:104-108).
"""
from __future__ import annotations

import os
from pathlib import Path

import torch as th

from . import gaussian_diffusion as gd
from .guidance import CondFnB200, GuidedStepB200, MakeCutouts
from .unet import config_for
from .rn import RN_CONFIGS, rn_config_from_state_dict
from .vit import VIT_CONFIGS, vit_config_from_state_dict

CACHE_PATH = os.path.expanduser("~/.cache/clip-guided-diffusion")  # cgd/script_util.py:18


def parse_prompt(prompt: str):
    """"<text or url>:<weight>" -> (text, weight), weight 1 when absent; a URL keeps its scheme colon (cgd/script_util.py:60-67)"""
    is_url = prompt.startswith(("http://", "https://"))
    vals = prompt.rsplit(":", 2 if is_url else 1)
    if is_url:
        vals = [vals[0] + ":" + vals[1], *vals[2:]]
    vals = vals + ["", "1"][len(vals):]
    return vals[0], float(vals[1])


def alphanumeric_filter(s: str) -> str:  # cgd/script_util.py:81-84: drop everything but word characters and blanks, blanks -> "_"
    import re
    return re.sub(r"[^\w\s]", "", s).replace(" ", "_")


def clean_and_combine_prompts(base_path, txts, batch_idx, max_length=255) -> str:  # cgd/script_util.py:87-90
    return os.path.join(base_path, "_".join(alphanumeric_filter(t) for t in txts)[:max_length], f"{batch_idx:02}")


# checkpoint file names of data/diffusion_model_flags.py (DIFFUSION_LOOKUP[cond|uncond][image_size]["filename"])
DIFFUSION_FILENAMES = {
    (True, 64): "64x64_diffusion.pt", (True, 128): "128x128_diffusion.pt", (True, 256): "256x256_diffusion.pt",
    (True, 512): "512x512_diffusion.pt", (False, 256): "256x256_diffusion_uncond.pt",
    (False, 512): "512x512_diffusion_uncond_finetune_008100.pt",
}


def log_image(image: th.Tensor, prefix_path, prompts, step: int, batch_idx: int) -> str:  # cgd/script_util.py:93-101
    from PIL import Image
    dirname = Path(clean_and_combine_prompts(str(prefix_path), prompts, batch_idx))
    dirname.mkdir(parents=True, exist_ok=True)
    # tvf.to_pil_image(image.add(1).div(2).clamp(0, 1)) of the reference: torchvision converts a float tensor with `mul(255).byte()` --
    # truncation, not rounding (pinned pixel for pixel on tests/golden/script_util_golden.json)
    arr = image.detach().float().add(1).div(2).clamp(0, 1).mul(255).byte().permute(1, 2, 0).cpu().numpy()
    path = str(dirname / f"{step:04d}.png")
    pil = Image.fromarray(arr)
    pil.save(path)
    pil.save("current.png")
    return path


def _load_unet_sd(image_size, class_cond, checkpoints_dir):
    if (class_cond, image_size) not in DIFFUSION_FILENAMES:
        raise ValueError(f"no published {'class-conditional' if class_cond else 'unconditional'} checkpoint at {image_size}x{image_size} "
                         "(data/diffusion_model_flags.py)")
    path = os.path.join(checkpoints_dir, DIFFUSION_FILENAMES[(class_cond, image_size)])
    if not os.path.exists(path):
        raise FileNotFoundError(f"{path} not found: pass unet_state_dict=... or place the guided-diffusion checkpoint there "
                                "(downloads are outside this framework's scope)")
    return th.load(path, map_location="cpu")


def clip_checkpoint_filename(clip_model_name: str) -> str:
    """file names of CLIP_MODEL_URLS (cgd/clip_util.py:20-29): ViT-B-32.pt, RN50x4.pt, ViT-L-14-336px.pt"""
    return clip_model_name.replace("/", "-").replace("@", "-") + ".pt"


def _load_clip_sd(clip_model_name, checkpoints_dir):
    # the reference keeps CLIP archives under CACHE_PATH/clip whatever checkpoints_dir is (cgd/clip_util.py:32-37); look there too
    fname = clip_checkpoint_filename(clip_model_name)
    path = os.path.join(checkpoints_dir, "clip", fname)
    if not os.path.exists(path) and os.path.exists(os.path.join(CACHE_PATH, "clip", fname)):
        path = os.path.join(CACHE_PATH, "clip", fname)
    if not os.path.exists(path):
        raise FileNotFoundError(f"{path} not found: pass clip_state_dict=...")
    try:
        return th.jit.load(path, map_location="cpu").state_dict()
    except RuntimeError:
        return th.load(path, map_location="cpu")


def _encode_text(prompts, clip_model_name, device):
    try:
        import clip  # clip-anytorch, only for the one-shot text tower
    except ImportError as e:
        raise RuntimeError("text prompts need the `clip` package for the (one-shot) text tower, or pass target_embeds=/weights=") from e
    model = clip.load(clip_model_name, jit=False, device=device)[0].eval()
    embeds, weights = [], []
    for p in prompts:
        txt, w = parse_prompt(p)
        embeds.append(model.encode_text(clip.tokenize(txt).to(device)).float())
        weights.append(w)
    return th.cat(embeds), th.tensor(weights)


def _lpips_sd(given):
    """LPIPS(net='vgg') weights in upstream key layout: passed in, or taken from the ``lpips`` package when it is installed"""
    if given is not None:
        return given
    try:
        import lpips  # noqa: WPS433 (optional dependency, like the reference's lazy construction at cgd/cgd.py:147-148)
    except ImportError as e:
        raise RuntimeError("init_scale != 0 needs the LPIPS-VGG weights: pass lpips_state_dict= (keys net.sliceK.N.*, linK.model.1.weight) "
                           "or install the `lpips` package") from e
    return lpips.LPIPS(net="vgg").state_dict()


def _tower_config(clip_sd: dict):
    """ViT-B/32, ViT-B/16, ViT-L/14 (vit.py) or a ModifiedResNet tower -- RN50, RN101, RN50x4, RN50x16 (rn.py; any width that is a
    multiple of 16) -- recognised from the state_dict keys"""
    if "visual.layer1.0.conv1.weight" in clip_sd:
        cfg = rn_config_from_state_dict(clip_sd)
        if cfg.width % 16:
            raise NotImplementedError(f"ModifiedResNet width {cfg.width}: the attention pool needs 64-wide heads (width a multiple of 16)")
        return cfg
    return vit_config_from_state_dict(clip_sd)


def _require_cuda(device):
    if not str(device).startswith("cuda") or not th.cuda.is_available():
        raise RuntimeError("clip_guided_diffusion_b200 runs the sampling step on a CUDA (sm_90a, H100) device only; there is no CPU path")


def clip_guided_diffusion(
    image_size: int = 128, num_cutouts: int = 16, prompts: "list[str]" = [], image_prompts: "list[str]" = [],
    clip_guidance_scale: int = 1000, tv_scale: float = 150, range_scale: float = 50, sat_scale: float = 0, init_scale: float = 0,
    batch_size: int = 1, init_image=None, class_cond: bool = True, cutout_power: float = 1.0, timestep_respacing: str = "1000",
    seed: int = 0, diffusion_steps: int = 1000, skip_timesteps: int = 0, checkpoints_dir: str = CACHE_PATH,
    clip_model_name: str = "ViT-B/32", randomize_class: bool = True, prefix_path=Path("./outputs"), save_frequency: int = 25,
    noise_schedule: str = "linear", dropout: float = 0.0, device: str = "", wandb_project: str = None, wandb_entity: str = None,
    use_augs: bool = False, use_magnitude: bool = False, height_offset: int = 0, width_offset: int = 0, progress: bool = True,
    reduce_clip: bool = False, progressive_cutout: bool = False, cached_cutouts: bool = False,
    # --- additions of this framework (all optional)
    unet_state_dict: dict = None, clip_state_dict: dict = None, target_embeds: th.Tensor = None, weights: th.Tensor = None,
    lpips_state_dict: dict = None, cutout_resize: str = "pool",
    rank: int = 0, world_size: int = 1,
):
    if len(device) == 0:
        device = "cuda"
    _require_cuda(device)
    if image_prompts:
        raise NotImplementedError("image prompts are unsupported (the reference's encode_image_prompt crashes, SURVEY quirk B5)")
    if wandb_project is not None:
        raise NotImplementedError("W&B logging is outside the hot path (SURVEY section 2)")
    th.manual_seed(seed)
    if not use_magnitude and image_size == 64:  # cgd/cgd.py:72-74
        use_magnitude = True
    Path(prefix_path).mkdir(parents=True, exist_ok=True)

    clip_sd = clip_state_dict if clip_state_dict is not None else _load_clip_sd(clip_model_name, checkpoints_dir)
    towers = {**VIT_CONFIGS, **RN_CONFIGS}
    if clip_state_dict is None and clip_model_name not in towers:
        raise NotImplementedError(f"CLIP tower {clip_model_name!r} is not supported (supported: {sorted(towers)})")
    vit_cfg = _tower_config(clip_sd) if clip_state_dict is not None else towers[clip_model_name]
    if target_embeds is None:
        target_embeds, weights = _encode_text(prompts, clip_model_name, device)
    if weights is None:  # target_embeds= given without weights=: every prompt weighs 1 (parse_prompt's default)
        weights = th.ones(target_embeds.shape[0])
    weights = th.as_tensor(weights, dtype=th.float32)
    if weights.sum().abs() < 1e-3:
        raise RuntimeError("The weights must not sum to 0.")
    weights = weights / weights.sum().abs()  # cgd/cgd.py:102-105

    if noise_schedule not in ("linear", "cosine"):  # cgd/script_util.py:302-303
        raise ValueError("linear_or_cosine must be set")
    unet_cfg = config_for(image_size, class_cond)
    # CLI semantics (cgd/script_util.py:307-315): user noise_schedule overrides the checkpoint flag; rescale_timesteps from the flags
    unet_sd = unet_state_dict if unet_state_dict is not None else _load_unet_sd(image_size, class_cond, checkpoints_dir)
    diffusion = gd.create_gaussian_diffusion(diffusion_steps, noise_schedule, timestep_respacing, rescale_timesteps=unet_cfg.rescale_timesteps)
    if reduce_clip and skip_timesteps == 0:  # cgd/cgd.py:141-144
        skip_timesteps = int(diffusion.num_timesteps * 0.2)

    H, W = image_size + height_offset, image_size + width_offset
    local_b = batch_size // world_size
    assert local_b * world_size == batch_size, "batch_size must divide evenly over the ranks"
    # progressive_cutout runs max(4, n // 4), max(8, n // 2), n cutouts (cgd/cgd.py:167-175): the middle count exceeds n when n < 16
    counts = CondFnB200.progressive_counts(num_cutouts) if progressive_cutout else (num_cutouts,)
    engine = GuidedStepB200(unet_cfg, unet_sd, vit_cfg, clip_sd, batch=local_b, height=H, width=W, num_cutouts=max(counts),
                            max_prompts=target_embeds.shape[0], clip_guidance_scale=clip_guidance_scale, tv_scale=tv_scale,
                            range_scale=range_scale, sat_scale=sat_scale, use_magnitude=use_magnitude, device=device, rank=rank,
                            world_size=world_size,
                            cutn_variants=tuple(c for c in counts if c != max(counts)),
                            lpips_sd=_lpips_sd(lpips_state_dict) if (init_image is not None and init_scale != 0) else None,
                            init_scale=init_scale, cutout_resize=cutout_resize, use_augs=use_augs)
    engine.set_targets(target_embeds, weights)
    make_cutouts = MakeCutouts(cut_size=vit_cfg.input_resolution, num_cutouts=num_cutouts, cutout_size_power=cutout_power, use_augs=use_augs)
    if cached_cutouts:
        make_cutouts.cache_coordinates(W, H)  # cgd/cgd.py:113
    cond_fn = CondFnB200(engine, diffusion, make_cutouts, cached_cutouts=cached_cutouts, reduce_clip=reduce_clip,
                         progressive_cutout=progressive_cutout)

    init_tensor = None
    if init_image is not None:
        from PIL import Image
        import numpy as np
        pil = Image.open(init_image).convert("RGB").resize((image_size, image_size))
        init_tensor = th.from_numpy(np.array(pil)).float().div(255).permute(2, 0, 1).unsqueeze(0).mul(2).sub(1).to(device)
        if engine.lpips is not None:  # cgd/cgd.py:147-148, 220-224
            engine.set_init_image(init_tensor)

    model_kwargs = {}
    if class_cond:
        model_kwargs["y"] = th.zeros([local_b], device=device, dtype=th.long)
    loop = diffusion.ddim_sample_loop_progressive if timestep_respacing.startswith("ddim") else diffusion.p_sample_loop_progressive
    samples = loop(engine.model, (local_b, 3, H, W), clip_denoised=False, model_kwargs=model_kwargs, cond_fn=cond_fn, progress=progress,
                   skip_timesteps=skip_timesteps, init_image=init_tensor, randomize_class=randomize_class, cond_fn_with_grad=True)
    cond_fn.current_timestep = diffusion.num_timesteps - 1  # cgd/cgd.py:265
    last_step = diffusion.num_timesteps - skip_timesteps - 1
    for step, sample in enumerate(samples):
        cond_fn.step_done()
        save = step % save_frequency == 0 or cond_fn.current_timestep == -1
        if world_size > 1 and step == last_step:
            # the run's one collective (SURVEY 8e): all ranks' final images -> rank 0, which saves and yields the whole batch;
            # earlier frames stay with the rank that owns the image (no traffic)
            final = engine.gather_final(sample["pred_xstart"])
            if save and rank == 0:
                for batch_idx, image_tensor in enumerate(final):
                    yield batch_idx, log_image(image_tensor, prefix_path, prompts, step, batch_idx)
            continue
        if save:
            for batch_idx, image_tensor in enumerate(sample["pred_xstart"]):
                yield batch_idx + rank * local_b, log_image(image_tensor, prefix_path, prompts, step, batch_idx + rank * local_b)
