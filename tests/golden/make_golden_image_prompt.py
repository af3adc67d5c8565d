"""Writes tests/golden/image_prompt_golden.npz: what the reference's own pieces of ``encode_image_prompt`` (cgd/clip_util.py:90-101)
return for seeded uint8 images -- its vendored ``ResizeRight.resize`` (tensor path, lanczos3, antialiasing, ``out_shape=[H', W']``:
the short side becomes s = min(image_size, W, H), the long side int(s * long / short)) and ``cgd.modules.MakeCutouts`` under
``manual_seed``: the resized image, the cutout windows, the pooled cutouts and the CPU generator state afterwards.

    python tests/golden/make_golden_image_prompt.py <path of a checkout of the reference>

Cases: a landscape image, a portrait image (the windows' x offset is drawn over the height and clipped at the right border, quirk
B3), a heavy downscale needing more than 16 taps per output (the two axes' scale factors differ, so their order matters), and an
image smaller than image_size (the identity path).
"""
import os
import sys

import numpy as np
import torch as th

CASES = {  # name: (H, W, image_size, cut_size, num_cutouts, seed)
    "landscape": (72, 108, 64, 32, 4, 1),
    "portrait": (150, 100, 64, 32, 6, 2),
    "heavy": (180, 240, 64, 32, 4, 3),
    "small": (40, 52, 64, 32, 4, 4),
}


def resized_shape(H, W, image_size):  # torchvision's resize(img, int) rule for the short side s
    s = min(image_size, W, H)
    return (int(s * H / W), s) if W <= H else (s, int(s * W / H))


def main(ref_root):
    sys.path.insert(0, ref_root)
    from cgd.modules import MakeCutouts
    from cgd.ResizeRight import resize_right
    from cgd.ResizeRight.interp_methods import lanczos3

    out = {}
    g = th.Generator().manual_seed(2024)
    for name, (H, W, image_size, cut_size, cutn, seed) in CASES.items():
        img = th.randint(0, 256, (H, W, 3), generator=g, dtype=th.uint8)
        x = img.permute(2, 0, 1).unsqueeze(0).float().div(255)  # tvf.to_tensor
        Ho, Wo = resized_shape(H, W, image_size)
        y = resize_right.resize(x, out_shape=[Ho, Wo], interp_method=lanczos3, support_sz=None, antialiasing=True, by_convs=False,
                                scale_tolerance=None)
        mc = MakeCutouts(cut_size=cut_size, num_cutouts=cutn)
        th.manual_seed(seed)
        coords = mc._generate_coords(*y.shape[2:4], cutn)  # the draws forward() makes (side_x, side_y = H, W)
        th.manual_seed(seed)
        cuts = mc(y)
        out[name + "_image"] = img.numpy()
        out[name + "_resized"] = y.numpy().astype(np.float32)
        out[name + "_coords"] = np.array(coords, dtype=np.int64)
        out[name + "_cutouts"] = cuts.numpy().astype(np.float32)
        out[name + "_rng"] = th.get_rng_state().numpy()
        out[name + "_cfg"] = np.array([H, W, image_size, cut_size, cutn, seed])
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "image_prompt_golden.npz"), **out)
    print({k: v.shape for k, v in out.items() if k.endswith(("_resized", "_coords"))})


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])
