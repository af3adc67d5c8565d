"""Image prompts: the intent of the reference's ``encode_image_prompt`` (cgd/clip_util.py:90-101), on the device.

The reference's function crashes before it encodes anything (it hands a PIL image to ResizeRight, quirk B5); what it means to do
is unambiguous and runs here, once per image prompt and run, outside the sampling loop:

1. ``Image.open(path).convert("RGB")`` scaled to [0, 1] like ``tvf.to_tensor``;
2. resize so that the short side becomes ``s = min(diffusion_size, W, H)`` (cgd/clip_util.py:94) and the long side
   ``int(s * long / short)`` (torchvision's ``resize(img, int)`` rule), each axis with ResizeRight's antialiased lanczos3
   (zero outside the image, axes in increasing order of scale factor, an axis with scale 1 untouched, no clamping) -- two
   ``RESIZE_AXIS`` launches over host-built tables (resize_right.py ``tables(S, O, t_max=None)``: any tap count);
3. ``MakeCutouts(cut_size=tower input resolution, num_cutouts)`` with the reference's defaults (cut_pow 1, no augmentations,
   adaptive-avg-pool): the windows are 3 draws per cutout from the CPU default generator, (H, W) passed as (side_x, side_y)
   (quirk B3); ``CUTOUTS_FWD`` writes the normalised cutouts straight into the CLIP tower's patch buffer;
4. ``CLIP_NORMALIZE`` (not the literal ``tf.normalize`` of cgd/clip_util.py:99, a name collision with the notebook's CLIP
   ``Normalize``), then the forward-only tower: ``cutn`` embeddings, each weighing ``weight / cutn``.
"""
from __future__ import annotations

import numpy as np
import torch as th

from . import _lib
from .guidance import CLIP_MEAN, CLIP_STD, MakeCutouts, clip_tower


def check_local(path: str):
    """image prompts are local files: the reference's ``script_util.fetch`` would download a URL, which is out of scope here"""
    if str(path).startswith(("http://", "https://")):
        raise ValueError(f"image prompt {path!r}: URLs are not fetched (downloads are outside this framework's scope); "
                         "save the image and pass its path")


def load_image(path: str) -> th.Tensor:
    """-> fp32 [1, 3, H, W] in [0, 1] (``Image.open(path).convert("RGB")`` and ``tvf.to_tensor``); local files only"""
    check_local(path)
    from PIL import Image
    with Image.open(path) as im:
        arr = np.asarray(im.convert("RGB"), dtype=np.uint8)
    return th.from_numpy(arr.copy()).permute(2, 0, 1).unsqueeze(0).float().div(255)


def resized_shape(height: int, width: int, diffusion_size: int) -> "tuple[int, int]":
    """(H', W'): the short side becomes s = min(diffusion_size, W, H), the long side int(s * long / short)"""
    s = min(int(diffusion_size), width, height)
    if width <= height:
        return int(s * height / width), s
    return s, int(s * width / height)


def _run_op(code: str, i, f=(), p=()):
    _lib.run_op(code, i=i, f=f, p=p)


def resize_lanczos3(x: th.Tensor, out_hw: "tuple[int, int]") -> th.Tensor:
    """fp32 CUDA [N, C, H, W] -> [N, C, out_hw[0], out_hw[1]]: ResizeRight lanczos3 with antialiasing, one ``RESIZE_AXIS`` launch per
    axis whose scale factor is not 1, the axes in increasing order of scale factor (ties: H first), like
    cgd/ResizeRight/resize_right.py:31-122"""
    from . import resize_right as rr
    if not x.is_cuda:
        raise _lib.CgdError("resize_lanczos3 runs on the GPU only (no CPU fallback)")
    x = x.detach().float().contiguous()
    N, C, H, W = x.shape
    dims = sorted([(0, int(out_hw[0])), (1, int(out_hw[1]))], key=lambda d: d[1] / (H, W)[d[0]])
    for axis, O in dims:
        S = x.shape[2 + axis]
        if O == S:
            continue
        left, wt, T = rr.tables(S, O, t_max=None)
        left, wt = left.to(x.device), wt.to(x.device)
        shape = (N, C, O, x.shape[3]) if axis == 0 else (N, C, x.shape[2], O)
        out = th.empty(shape, dtype=th.float32, device=x.device)
        _run_op("RESIZE_AXIS", [N * C, x.shape[2], x.shape[3], axis, O, T], p=[x, out, left, wt])
        x = out
    return x


class ImagePromptEncoder:
    """Encodes image prompts with one forward-only CLIP tower for ``num_cutouts`` cutouts (``ViTB200`` / ``RNB200`` with
    ``build_backward=False``); build it once per run and reuse it for every image prompt, then drop it."""

    def __init__(self, tower_cfg, clip_sd: dict, num_cutouts: int, device="cuda"):
        self.cfg, self.cutn, self.device = tower_cfg, int(num_cutouts), th.device(device)
        self.tower = clip_tower(tower_cfg, clip_sd, n_images=self.cutn, device=device, build_backward=False)
        self.make_cutouts = MakeCutouts(cut_size=tower_cfg.input_resolution, num_cutouts=self.cutn)
        self.last = {}  # resized image and cutout windows of the last call (inspection / tests)

    def encode(self, image: str, weight: float, diffusion_size: int):
        """-> (embeds fp32 [cutn, D], [weight / cutn] * cutn)"""
        x = load_image(image)
        H, W = resized_shape(x.shape[2], x.shape[3], diffusion_size)
        x = resize_lanczos3(x.to(self.device), (H, W))
        coords = self.make_cutouts.coords_for(H, W)  # sic: (H, W) as (side_x, side_y), cgd/modules.py:52 (quirk B3)
        for ox, oy, size in coords:
            if not (ox < W and oy < H):
                raise ValueError(f"image prompt {image!r}: the cutout window (x={ox}, y={oy}, size={size}) lies outside the {H}x{W} resized "
                                 "image (the reference's MakeCutouts draws the x offset over the height: images about twice as tall as "
                                 "wide or taller can leave empty windows, on which its adaptive_avg_pool2d raises)")
        cfg = self.cfg
        patches = self.tower.plan.view(self.tower.patches)
        cdev = th.tensor(coords, dtype=th.int32).to(self.device)
        # the image is in [0, 1], not [-1, 1]: mean (1 + m) / 2 and std s / 2 fold the kernel's (x + 1) / 2 away
        _run_op("CUTOUTS_FWD", [1, H, W, self.cutn, cfg.input_resolution, cfg.patch_size, cfg.kpad],
                f=[(1 + m) / 2 for m in CLIP_MEAN] + [s / 2 for s in CLIP_STD], p=[x, cdev, patches])
        emb = self.tower.encode_patches().float().clone()
        self.last = {"image": x, "coords": coords}
        return emb, [weight / self.cutn] * self.cutn


__all__ = ["ImagePromptEncoder", "check_local", "load_image", "resize_lanczos3", "resized_shape"]
