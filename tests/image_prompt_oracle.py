"""fp32 oracle of image-prompt encoding (test infrastructure): the intent of the reference's ``encode_image_prompt``
(cgd/clip_util.py:90-101) assembled from the oracle's pinned pieces -- ``oracle.resize_right.resize_lanczos3`` (ResizeRight,
tests/golden/resize_right_golden.npz), ``oracle.guidance.MakeCutouts`` (cgd/modules.py) and ``clip_normalize`` -- with any fp32
CLIP visual tower.  Pinned against the reference's own ResizeRight and MakeCutouts on tests/golden/image_prompt_golden.npz."""
from __future__ import annotations

import numpy as np
import torch as th
import torchvision.transforms.functional as tvf

from oracle.guidance import MakeCutouts, clip_normalize
from oracle.resize_right import resize_lanczos3


def load_image(path) -> th.Tensor:
    """Image.open(path).convert("RGB") -> tvf.to_tensor -> [1, 3, H, W]"""
    from PIL import Image
    with Image.open(path) as im:
        return tvf.to_tensor(im.convert("RGB")).unsqueeze(0)


def resized_shape(H, W, diffusion_size):
    """torchvision's resize(img, s) output size for s = min(diffusion_size, W, H) (cgd/clip_util.py:94)"""
    s = min(diffusion_size, W, H)
    return tuple(tvf._compute_resized_output_size((H, W), [s]))


def resize(x: th.Tensor, diffusion_size: int) -> th.Tensor:
    return resize_lanczos3(x, resized_shape(x.shape[2], x.shape[3], diffusion_size))


def encode_image_prompt(x: th.Tensor, weight: float, diffusion_size: int, num_cutouts: int, clip_model, cut_size: int):
    """x [1, 3, H, W] in [0, 1]; ``clip_model(images) -> [n, D]`` an fp32 tower.  Draws the windows from the CPU default generator.
    -> (embeds [cutn, D], [weight / cutn] * cutn, {"image": resized, "coords": windows, "cutouts": pooled cutouts})"""
    y = resize(x.float(), diffusion_size)
    mc = MakeCutouts(cut_size, num_cutouts)
    coords = mc._generate_coords(y.shape[2], y.shape[3], num_cutouts)  # (H, W) as (side_x, side_y): quirk B3
    cuts = mc(y, coords=coords)
    with th.no_grad():
        emb = clip_model(clip_normalize(cuts)).float()
    return emb, [weight / num_cutouts] * num_cutouts, {"image": y, "coords": coords, "cutouts": cuts}


def write_png(path, H, W, seed):
    """a seeded uint8 RGB image -> PNG; returns the array"""
    from PIL import Image
    arr = th.randint(0, 256, (H, W, 3), generator=th.Generator().manual_seed(seed), dtype=th.uint8).numpy()
    Image.fromarray(np.ascontiguousarray(arr)).save(path)
    return arr
