"""``clip_guided_diffusion(...)`` -- the reference's orchestrator surface (cgd/cgd.py:19-283) over the H100 engine.

Same keyword arguments and the same generator contract (yields ``(batch_idx, png_path)``); set-up stays Python and
runs once (seed, prompt encoding, weight loading, cutout cache), the per-timestep work is the engine's fused step.
Out of scope here, exactly as SURVEY.md section 2 marks them: checkpoint download, W&B, GIF/MP4.  The LPIPS init loss
(``init_image`` + ``init_scale``) runs on the engine when the VGG weights are given (``lpips_state_dict=``) or the ``lpips`` package
is installed.

Image prompts (``image_prompts=["path:weight", ...]``, local files) are encoded once, before the loop, by ``encode_image_prompt``:
the intent of the reference's function of that name, which itself crashes (quirk B5; image_prompt.py).  Each one adds
``num_cutouts`` target embeddings of weight ``weight / num_cutouts`` after the text prompts' embeddings; the weights of the whole set
are then normalised together (cgd/cgd.py:86-105).

Weights: pass ``unet_state_dict`` / ``clip_state_dict`` (upstream key layout), or have the reference's checkpoints on
disk under ``checkpoints_dir`` (``256x256_diffusion.pt`` ..., ``clip/ViT-B-32.pt``).  Text prompts are encoded once, outside the hot
path (cgd/clip_util.py:104-108), by one of two text towers (``text_encoder=``):
- ``"device"``: this package's own tokenizer and causal text tower (tokenizer.py, text.py), from the same CLIP state_dict as the
  visual tower; needs CLIP's BPE vocabulary file (``bpe_path=``, or ``bpe_simple_vocab_16e6.txt.gz`` under ``checkpoints_dir/clip/``
  or ``CACHE_PATH/clip/``);
- ``"clip"``: the ``clip`` package's eager model (``clip.load(clip_model_name)``, its own checkpoint);
- ``"auto"`` (default): the ``clip`` package if it imports, else the device tower if the vocabulary file is found, else the ``clip``
  path, which raises without the package.
Or pass ``target_embeds`` / ``weights`` directly.  Image prompts use this package's own CLIP visual tower and never import ``clip``.

Several CLIP towers (``clip_model_name=["ViT-B/32", "ViT-B/16", "RN50"]``) guide one run together: each tower cuts its own
``num_cutouts`` windows at its own resolution, gets its own text and image targets, and the CLIP losses are summed (the reference's CLIP
block once per tower; tv / range / sat / LPIPS once).  A name is a tower name or a path to a CLIP checkpoint file (``.pt``: a TorchScript
archive or a plain state_dict, the architecture read from its keys).  ``"open_clip:<arch>"`` names LAION's OpenCLIP ViT towers (ViT-B-32,
ViT-B-32-quickgelu, ViT-B-16, ViT-L-14, ViT-H-14; vit.OPEN_CLIP_CONFIGS): exact-GELU MLPs, ViT-H's 80-wide heads; weights from
``clip_state_dict=`` or ``checkpoints_dir/open_clip/<arch>.{safetensors,bin,pt}`` (then ``CACHE_PATH/open_clip/``), checked against the
architecture.  Their text prompts are always encoded on the device text tower (``text_encoder="clip"`` is refused for them).  With several towers, ``target_embeds=`` is one ``[P, D_m]`` tensor
per tower and ``clip_state_dict=`` one state_dict (or None) per tower; ``use_augs`` and ``cutout_resize="lanczos3"`` take one tower.  ``cutout_resize="lanczos3"``
(ResizeRight instead of adaptive_avg_pool2d) combines with ``height_offset`` / ``width_offset``, ``progressive_cutout`` and ``use_augs``.
"""
from __future__ import annotations

import os
from pathlib import Path

import torch as th

from . import gaussian_diffusion as gd
from .guidance import CondFnB200, GuidedStepB200, MakeCutouts, check_tower_options
from .image_prompt import ImagePromptEncoder, check_local
from .text import TextB200, text_config_from_state_dict
from .tokenizer import find_vocab, load_tokenizer, tokenize  # noqa: F401 (tokenize: public, like clip.tokenize)
from .unet import config_for
from .rn import RN_CONFIGS, rn_config_from_state_dict
from .vit import OPEN_CLIP_CONFIGS, VIT_CONFIGS, check_open_clip_state_dict, vit_config_from_state_dict

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


def _clip_importable() -> bool:
    """does `import clip` succeed?  (a package that is installed but fails to import counts as absent)"""
    try:
        import clip  # noqa: F401
    except Exception:  # noqa: BLE001 -- any import failure means the clip path cannot run
        return False
    return True


def _text_encoder_choice(text_encoder, bpe_path, checkpoints_dir):
    """-> the vocabulary file when the device tower encodes the text prompts, None when `_encode_text` (the `clip` package) does"""
    if text_encoder == "clip" or (text_encoder == "auto" and _clip_importable()):
        return None
    try:
        return find_vocab(bpe_path, checkpoints_dir)
    except FileNotFoundError:
        if text_encoder == "device":
            raise
        return None


def _encode_text_device(prompts, clip_sd, vocab, device, act="quick_gelu"):
    """all text prompts in one pass of a forward-only text tower, in prompt order -> (fp32 [P, D], weights [P]); `act`: the MLP
    activation of the tower (the visual config's, "gelu" for the OpenCLIP towers)"""
    parsed = [parse_prompt(p) for p in prompts]
    cfg = text_config_from_state_dict(clip_sd, act=act)
    ids = load_tokenizer(vocab).tokenize([t for t, _ in parsed], context_length=cfg.context_length)
    tower = TextB200(cfg, clip_sd, len(parsed), device)
    embeds = tower.encode(ids)
    del tower
    return embeds, th.tensor([w for _, w in parsed])


def encode_text_prompt(txt: str, weight: float, clip_model_name: str = "ViT-B/32", device: str = "cuda", *, clip_state_dict: dict = None,
                       checkpoints_dir: str = CACHE_PATH, bpe_path: str = None):
    """cgd/clip_util.py:104-108 (the reference's signature plus the weight and vocabulary sources) -> (fp32 [1, D] on ``device``,
    ``weight``), on this package's text tower: the text half of ``clip_state_dict`` or of the named checkpoint, and the BPE vocabulary
    of ``find_vocab(bpe_path, checkpoints_dir)``.  A text longer than the context raises RuntimeError like ``clip.tokenize``."""
    _require_cuda(device)
    act = "quick_gelu"
    if open_clip_arch(clip_model_name) is not None:
        clip_sd, cfg = _clip_tower(clip_model_name, clip_state_dict, checkpoints_dir)
        act = cfg.act
    else:
        clip_sd = clip_state_dict if clip_state_dict is not None else _load_clip_sd(clip_model_name, checkpoints_dir)
    embeds, _ = _encode_text_device([txt], clip_sd, find_vocab(bpe_path, checkpoints_dir), device, act=act)
    return embeds, weight


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


def _is_checkpoint_path(clip_model_name) -> bool:
    """a CLIP checkpoint file rather than a tower name (the reference's `clip.load(path)` fallback, cgd/clip_util.py:52-56)"""
    return str(clip_model_name).endswith(".pt") or os.path.isfile(str(clip_model_name))


def _load_clip_file(path):
    """a CLIP checkpoint file -> state_dict: a TorchScript archive first, then a plain state_dict (as `_load_clip_sd`)"""
    if not os.path.isfile(path):
        raise FileNotFoundError(f"CLIP checkpoint {path} not found")
    try:
        return th.jit.load(path, map_location="cpu").state_dict()
    except RuntimeError:
        return th.load(path, map_location="cpu")


OPEN_CLIP_PREFIX = "open_clip:"
OPEN_CLIP_SUFFIXES = (".safetensors", ".bin", ".pt")


def open_clip_arch(clip_model_name):
    """"open_clip:<arch>" -> arch (ValueError for an arch not in OPEN_CLIP_CONFIGS); None for any other name"""
    name = str(clip_model_name)
    if not name.startswith(OPEN_CLIP_PREFIX):
        return None
    arch = name[len(OPEN_CLIP_PREFIX):]
    if arch not in OPEN_CLIP_CONFIGS:
        raise ValueError(f"OpenCLIP tower {arch!r} is not supported (supported: {', '.join(OPEN_CLIP_PREFIX + a for a in OPEN_CLIP_CONFIGS)})")
    return arch


def open_clip_checkpoint_paths(arch, checkpoints_dir):
    """where the weights of open_clip:<arch> are looked for, in order: checkpoints_dir/open_clip/<arch>.{safetensors,bin,pt}, then the
    same under CACHE_PATH (the LAION hub repos' open_clip_model.safetensors / open_clip_pytorch_model.bin, renamed)"""
    dirs = [d for d in (checkpoints_dir, CACHE_PATH) if d is not None]
    return [os.path.join(d, "open_clip", arch + s) for d in dict.fromkeys(dirs) for s in OPEN_CLIP_SUFFIXES]


def _load_open_clip_sd(arch, checkpoints_dir):
    places = open_clip_checkpoint_paths(arch, checkpoints_dir)
    path = next((p for p in places if os.path.isfile(p)), None)
    if path is None:
        raise FileNotFoundError(f"no weights for open_clip:{arch} in {', '.join(places)}: place the checkpoint there or pass "
                                "clip_state_dict= (nothing is downloaded)")
    if path.endswith(".safetensors"):
        from safetensors.torch import load_file
        return load_file(path, device="cpu")
    if path.endswith(".bin"):
        return th.load(path, map_location="cpu")
    return _load_clip_file(path)


def _clip_tower(clip_model_name, clip_state_dict, checkpoints_dir):
    """-> (CLIP state_dict, visual tower config): the given state_dict's own architecture, a checkpoint file's (a path) or the named
    tower's checkpoint.  An "open_clip:<arch>" name takes its config from OPEN_CLIP_CONFIGS, never from the keys, and the weights (given
    or found under checkpoints_dir/open_clip/) are checked against it."""
    arch = open_clip_arch(clip_model_name)
    if arch is not None:
        clip_sd = clip_state_dict if clip_state_dict is not None else _load_open_clip_sd(arch, checkpoints_dir)
        check_open_clip_state_dict(arch, clip_sd, text="token_embedding.weight" in clip_sd)
        return clip_sd, OPEN_CLIP_CONFIGS[arch].vision
    if clip_state_dict is None and _is_checkpoint_path(clip_model_name):
        clip_sd = _load_clip_file(str(clip_model_name))
        return clip_sd, _tower_config(clip_sd)
    clip_sd = clip_state_dict if clip_state_dict is not None else _load_clip_sd(clip_model_name, checkpoints_dir)
    towers = {**VIT_CONFIGS, **RN_CONFIGS}
    if clip_state_dict is None and clip_model_name not in towers:
        raise NotImplementedError(f"CLIP tower {clip_model_name!r} is not supported (supported: {sorted(towers)})")
    return clip_sd, (_tower_config(clip_sd) if clip_state_dict is not None else towers[clip_model_name])


def encode_image_prompt(image: str, weight: float, diffusion_size: int, num_cutouts: int, clip_model_name: str = "ViT-B/32",
                        device: str = "cuda", *, clip_state_dict: dict = None, checkpoints_dir: str = CACHE_PATH):
    """cgd/clip_util.py:90-101 (the reference's signature plus the weight source) -> (embeds fp32 [num_cutouts, D] on ``device``,
    ``[weight / num_cutouts] * num_cutouts``).  ``image`` is a local file; the cutout windows are drawn from the CPU default
    generator.  For callers that assemble ``target_embeds=`` / ``weights=`` themselves: append the result after the text prompts'
    embeddings, as ``clip_guided_diffusion(image_prompts=...)`` does."""
    _require_cuda(device)
    clip_sd, cfg = _clip_tower(clip_model_name, clip_state_dict, checkpoints_dir)
    return ImagePromptEncoder(cfg, clip_sd, num_cutouts, device).encode(image, weight, diffusion_size)


def _tower_list(clip_model_name, clip_state_dict):
    """-> (names, state_dicts): `clip_model_name` is one name or a non-empty sequence of them; `clip_state_dict` None, one
    state_dict (one tower) or a sequence of the names' length"""
    names = [clip_model_name] if isinstance(clip_model_name, (str, os.PathLike)) else list(clip_model_name)
    if not names:
        raise ValueError("clip_model_name: a tower name, a checkpoint path or a non-empty sequence of them")
    if clip_state_dict is None:
        sds = [None] * len(names)
    elif isinstance(clip_state_dict, dict):
        if len(names) != 1:
            raise ValueError(f"{len(names)} CLIP towers: clip_state_dict must be a sequence of {len(names)} state_dicts (or None)")
        sds = [clip_state_dict]
    else:
        sds = list(clip_state_dict)
        if len(sds) != len(names):
            raise ValueError(f"{len(names)} CLIP towers but {len(sds)} clip_state_dict entries")
    return names, sds


def _require_cuda(device):
    if not str(device).startswith("cuda") or not th.cuda.is_available():
        raise RuntimeError("clip_guided_diffusion_b200 runs the sampling step on a CUDA (sm_90a, H100) device only; there is no CPU path")


def clip_guided_diffusion(
    image_size: int = 128, num_cutouts: int = 16, prompts: "list[str]" = [], image_prompts: "list[str]" = [],
    clip_guidance_scale: int = 1000, tv_scale: float = 150, range_scale: float = 50, sat_scale: float = 0, init_scale: float = 0,
    batch_size: int = 1, init_image=None, class_cond: bool = True, cutout_power: float = 1.0, timestep_respacing: str = "1000",
    seed: int = 0, diffusion_steps: int = 1000, skip_timesteps: int = 0, checkpoints_dir: str = CACHE_PATH,
    clip_model_name: "str | list[str]" = "ViT-B/32", randomize_class: bool = True, prefix_path=Path("./outputs"), save_frequency: int = 25,
    noise_schedule: str = "linear", dropout: float = 0.0, device: str = "", wandb_project: str = None, wandb_entity: str = None,
    use_augs: bool = False, use_magnitude: bool = False, height_offset: int = 0, width_offset: int = 0, progress: bool = True,
    reduce_clip: bool = False, progressive_cutout: bool = False, cached_cutouts: bool = False,
    # --- additions of this framework (all optional)
    unet_state_dict: dict = None, clip_state_dict: dict = None, target_embeds: th.Tensor = None, weights: th.Tensor = None,
    lpips_state_dict: dict = None, cutout_resize: str = "pool",
    rank: int = 0, world_size: int = 1, text_encoder: str = "auto", bpe_path: str = None,
):
    if len(device) == 0:
        device = "cuda"
    _require_cuda(device)
    names, clip_sds = _tower_list(clip_model_name, clip_state_dict)
    T = len(names)
    check_tower_options(T, use_augs, cutout_resize)
    if target_embeds is not None:
        if isinstance(target_embeds, th.Tensor):
            if T > 1:
                raise ValueError(f"{T} CLIP towers: target_embeds= must be a sequence of {T} [P, D_m] tensors, one per tower")
            target_embeds = [target_embeds]
        target_embeds = list(target_embeds)
        if len(target_embeds) != T or len({int(e.shape[0]) for e in target_embeds}) != 1:
            raise ValueError(f"target_embeds=: one [P, D_m] tensor per CLIP tower ({T}), the same P each")
    if image_prompts and target_embeds is not None:
        raise NotImplementedError("target_embeds= is the complete target set: with image prompts, encode them with encode_image_prompt() "
                                  "and append the embeddings and weights to target_embeds= / weights= instead of passing image_prompts=")
    image_prompts = [parse_prompt(p) for p in image_prompts]  # "path:weight" (cgd/cgd.py:93)
    for path, _ in image_prompts:
        check_local(path)
    if wandb_project is not None:
        raise NotImplementedError("W&B logging is outside the hot path (SURVEY section 2)")
    if text_encoder not in ("auto", "clip", "device"):
        raise ValueError(f"text_encoder={text_encoder!r}: expected 'auto', 'clip' or 'device'")
    open_clip = [open_clip_arch(n) is not None for n in names]  # also refuses an unknown open_clip: architecture, before any file is read
    if text_encoder == "clip" and any(open_clip):
        raise ValueError("text_encoder='clip' cannot encode for an open_clip: tower (the clip package does not build them): use "
                         "text_encoder='device' or 'auto'")
    th.manual_seed(seed)
    if not use_magnitude and image_size == 64:  # cgd/cgd.py:72-74
        use_magnitude = True
    Path(prefix_path).mkdir(parents=True, exist_ok=True)

    towers = [_clip_tower(n, sd, checkpoints_dir) for n, sd in zip(names, clip_sds)]  # [(state_dict, visual config)] in tower order
    if target_embeds is None:
        # text prompts first, then every image prompt's cutn embeddings (cgd/cgd.py:86-98); an image-only run needs no text tower.
        # Every tower encodes the same prompts with its own text half / visual tower; the weights are the same for every tower.
        embeds, weights = [[] for _ in towers], []
        if prompts or not image_prompts:
            vocab = _text_encoder_choice(text_encoder, bpe_path, checkpoints_dir) if prompts else None
            # an OpenCLIP tower always encodes on the device text tower (same BPE vocabulary); OpenAI towers keep the choice above
            oc_vocab = find_vocab(bpe_path, checkpoints_dir) if prompts and any(open_clip) else None
            for m, (name, (clip_sd, cfg)) in enumerate(zip(names, towers)):
                if open_clip[m]:
                    e, w = _encode_text_device(prompts, clip_sd, oc_vocab, device, act=cfg.act)
                elif vocab is not None:  # one forward-only text tower from the visual tower's state_dict, released here
                    e, w = _encode_text_device(prompts, clip_sd, vocab, device)
                else:
                    e, w = _encode_text(prompts, name, device)
                embeds[m].append(e)
            weights += [float(v) for v in w]
        if image_prompts:
            # tower-major: one forward-only tower for every image prompt, released before the next tower's (and before the engine)
            # is built; the cutout windows come from the CPU generator after the seed and before cache_coordinates / the loop, where
            # the reference draws them
            for m, (clip_sd, vit_cfg) in enumerate(towers):
                encoder = ImagePromptEncoder(vit_cfg, clip_sd, num_cutouts, device)
                for path, w in image_prompts:
                    e, ws = encoder.encode(path, w, image_size)
                    embeds[m].append(e)
                    if m == 0:
                        weights += ws
                del encoder
        target_embeds, weights = [th.cat([e.to(device) for e in em]) for em in embeds], th.tensor(weights)
    if weights is None:  # target_embeds= given without weights=: every prompt weighs 1 (parse_prompt's default)
        weights = th.ones(target_embeds[0].shape[0])
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
    cfgs, sds = [cfg for _, cfg in towers], [sd for sd, _ in towers]
    engine = GuidedStepB200(unet_cfg, unet_sd, cfgs[0] if T == 1 else cfgs, sds[0] if T == 1 else sds, batch=local_b, height=H, width=W,
                            num_cutouts=max(counts), max_prompts=target_embeds[0].shape[0], clip_guidance_scale=clip_guidance_scale, tv_scale=tv_scale,
                            range_scale=range_scale, sat_scale=sat_scale, use_magnitude=use_magnitude, device=device, rank=rank,
                            world_size=world_size,
                            cutn_variants=tuple(c for c in counts if c != max(counts)),
                            lpips_sd=_lpips_sd(lpips_state_dict) if (init_image is not None and init_scale != 0) else None,
                            init_scale=init_scale, cutout_resize=cutout_resize, use_augs=use_augs)
    engine.set_targets(target_embeds[0] if T == 1 else target_embeds, weights)
    make_cutouts = [MakeCutouts(cut_size=cfg.input_resolution, num_cutouts=num_cutouts, cutout_size_power=cutout_power, use_augs=use_augs)
                    for cfg in cfgs]
    if cached_cutouts:
        for mk in make_cutouts:  # cgd/cgd.py:113, once per tower in tower order
            mk.cache_coordinates(W, H)
    cond_fn = CondFnB200(engine, diffusion, make_cutouts[0] if T == 1 else make_cutouts, cached_cutouts=cached_cutouts, reduce_clip=reduce_clip,
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
