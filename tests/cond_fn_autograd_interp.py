"""TEST-ONLY: a CPU stand-in for ``_lib.run_op`` covering what the package's MakeCutouts and losses launch (CUTOUTS_FWD flags 1,
CUTOUTS_AUG_FWD, CUTOUTS_BWD flags 4 / 6, CUTOUTS_AUG_BWD flags 4, IMG_LOSS_FWD / _BWD, SPH_DIST_FWD / _BWD), in plain fp32 PyTorch on the
operands' own tensors, with one fp16 rounding where the kernels store fp16; and ``reference_style_cond_fn``, a cond_fn written like the
reference's closure (cgd/cgd.py:176-232) over whichever cutouts / normalisation / losses / CLIP / LPIPS modules it is given."""
from __future__ import annotations

import types

import torch as th
import torch.nn.functional as F

from oracle.guidance import apply_augs


def _coords(t):
    return [tuple(int(v) for v in r) for r in t.tolist()]


def _pool_cuts(x, coords, cs):
    return th.cat([F.adaptive_avg_pool2d(x[:, :, oy:oy + s, ox:ox + s], cs) for ox, oy, s in coords])


def _aug_cuts(x, coords, cs, prm, noise):
    out = []
    for k, (ox, oy, s) in enumerate(coords):
        cut = x[:, :, oy:oy + s, ox:ox + s]
        nz = None if noise is None else noise[k][..., :cut.shape[-2], :cut.shape[-1]]
        out.append(F.adaptive_avg_pool2d(apply_augs(cut, prm[k], nz), cs))
    return th.cat(out)


def _img_loss(x, kind):
    if kind == 1:
        p = F.pad(x, (0, 1, 0, 1), "replicate")
        return ((p[..., :-1, 1:] - p[..., :-1, :-1]) ** 2 + (p[..., 1:, :-1] - p[..., :-1, :-1]) ** 2).mean([1, 2, 3])
    return (x - x.clamp(-1, 1)).pow(2).mean([1, 2, 3])


def _sph(xr, yr):
    return (F.normalize(xr, dim=-1) - F.normalize(yr, dim=-1)).norm(dim=-1).div(2).clamp(max=1).arcsin().pow(2).mul(2)


def run_op(code, *, flags=0, i=(), f=(), p=(), what=None):
    i, f = [int(v) for v in i], [float(v) for v in f]
    if code in ("CUTOUTS_FWD", "CUTOUTS_AUG_FWD"):
        B, H, W, n, cs, P, kpad = i[:7]
        assert P == cs and kpad == 3 * cs * cs
        x, coords = p[0], _coords(p[1])
        mean, std = th.tensor(f[0:3]).view(1, 3, 1, 1), th.tensor(f[3:6]).view(1, 3, 1, 1)
        if code == "CUTOUTS_FWD":
            assert flags == 1
            p[2].copy_((((_pool_cuts(x, coords, cs) + 1) * 0.5 - mean) / std).view_as(p[2]))
        else:
            img = (_aug_cuts((x + 1) * 0.5, coords, cs, p[3], p[4]) - mean) / std
            p[2].copy_(img.reshape(p[2].shape).half())
    elif code in ("CUTOUTS_BWD", "CUTOUTS_AUG_BWD"):
        B, H, W, n, cs, P, kpad = i[:7]
        assert flags & 4 and P == cs and kpad == 3 * cs * cs
        d, coords = p[0].view(n * B, 3, cs, cs), _coords(p[1])
        std = th.tensor(f[3:6]).view(1, 3, 1, 1)
        x = th.zeros(B, 3, H, W, requires_grad=True)
        with th.enable_grad():
            cuts = _pool_cuts(x, coords, cs) if code == "CUTOUTS_BWD" else _aug_cuts((x + 1) * 0.5, coords, cs, p[3], None)
            (gx,) = th.autograd.grad(((cuts + 1) * 0.5 / std * d).sum() if code == "CUTOUTS_BWD" else (cuts / std * d).sum(), x)
        gx = gx * f[6]
        if code == "CUTOUTS_AUG_BWD" or flags & 2:
            p[2].add_(gx)
        else:
            p[2].copy_(gx)
    elif code == "IMG_LOSS_FWD":
        B, C, H, W, nblk = i[:5]
        p[2].copy_(_img_loss(p[0].view(B, C, H, W), flags))
    elif code == "IMG_LOSS_BWD":
        B, C, H, W = i[:4]
        x = p[0].view(B, C, H, W).clone().requires_grad_()
        with th.enable_grad():
            (g,) = th.autograd.grad(_img_loss(x, flags), x, p[1])
        p[2].copy_(g)
    elif code == "SPH_DIST_FWD":
        pairs = p[2].long()
        p[3].copy_(_sph(p[0][pairs[:, 0]], p[1][pairs[:, 1]]))
    elif code == "SPH_DIST_BWD":
        pairs = p[2].long()
        x, y = p[0].clone().requires_grad_(), p[1].clone().requires_grad_()
        with th.enable_grad():
            gx, gy = th.autograd.grad(_sph(x[pairs[:, 0]], y[pairs[:, 1]]), (x, y), p[3])
        if flags & 1:
            p[4].copy_(gx)
        if flags & 2:
            p[5].copy_(gy)
    else:
        raise AssertionError(f"no CPU interpreter for {code}")


def reference_style_cond_fn(ns: types.SimpleNamespace):
    """cgd/cgd.py:176-232 written over ``ns``: diffusion, current_timestep, make_cutouts, clip_util (CLIP_NORMALIZE), losses, clip_model,
    target_embeds, weights, num_cutouts, clip_guidance_scale, tv_scale, range_scale, sat_scale, use_magnitude, lpips_vgg, init_tensor,
    init_scale.  ``ns.terms`` receives the loss terms of the last call."""
    def cond_fn(x, t, out, y=None):
        n = x.shape[0]
        fac = ns.diffusion.sqrt_one_minus_alphas_cumprod[ns.current_timestep]
        x_in = out["pred_xstart"] * fac + x * (1 - fac)
        clip_in = ns.clip_util.CLIP_NORMALIZE(ns.make_cutouts(x_in.add(1).div(2), num_cutouts_override=ns.num_cutouts))
        cutout_embeds = ns.clip_model.encode_image(clip_in).float().view([ns.num_cutouts, n, -1])
        dists = ns.losses.spherical_dist_loss(cutout_embeds.unsqueeze(0), ns.target_embeds.unsqueeze(0)).view([ns.num_cutouts, n, -1])
        clip_losses = dists.mul(ns.weights).sum(2).mean(0).sum() * ns.clip_guidance_scale
        range_losses = ns.losses.range_loss(out["pred_xstart"]).sum() * ns.range_scale
        tv_losses = ns.losses.tv_loss(x_in).sum() * ns.tv_scale
        loss = clip_losses + tv_losses + range_losses
        ns.terms = {"clip": clip_losses.detach(), "range": range_losses.detach(), "tv": tv_losses.detach()}
        if ns.sat_scale:
            loss = loss + th.abs(x_in - x_in.clamp(min=-1, max=1)).mean() * ns.sat_scale
        if getattr(ns, "lpips_vgg", None) is not None and ns.init_scale:
            init_losses = ns.lpips_vgg(x_in, ns.init_tensor).sum() * ns.init_scale
            ns.terms["init"] = init_losses.detach()
            loss = loss + init_losses
        g = -th.autograd.grad(loss, x)[0]
        if ns.use_magnitude:
            magnitude = g.square().mean().sqrt()
            g = g * magnitude.clamp(max=0.05) / magnitude
        return g
    return cond_fn
