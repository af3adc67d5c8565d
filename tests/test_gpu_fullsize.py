"""GPU, BASELINE.json full sizes.
cfg1 (64x64 checkpoint architecture, respace 25, batch 1, cutn 4, ViT-B/32, use_magnitude auto-on): teacher-forced step vs the
fp32 oracle on the host CPU.  cfg2 (256x256, cutn 16): too slow for the CPU oracle inside a test, so it is checked through
size-independent properties: wgmma path == SIMT verification twin on the full UNet, graph replay == eager (bitwise),
linearity of the input-gradient backward in its seed."""
import pytest
import torch as th

from clip_guided_diffusion_b200 import gaussian_diffusion as pgd
from clip_guided_diffusion_b200 import guidance as pg
from clip_guided_diffusion_b200 import unet as pu
from clip_guided_diffusion_b200 import vit as pv
from clip_guided_diffusion_b200 import weights as pw
from tests.step_parity import compare, cos, rel

pytestmark = pytest.mark.gpu


def test_cfg1_step_vs_oracle():
    from oracle import diffusion as od
    from oracle import guidance as og
    from oracle.clip_vit import VIT_CONFIGS, CLIPVisualOnly
    from oracle.unet import UNetModel, config_for
    ucfg, vcfg = pu.config_for(64, True), pv.VIT_CONFIGS["ViT-B/32"]
    usd = pw.seeded_state_dict(pw.unet_param_shapes(ucfg), 1234)
    vsd = pw.seeded_state_dict(pw.vit_param_shapes(vcfg), 1235)
    ounet = UNetModel(config_for(64, True)).eval()
    ounet.load_state_dict(usd)
    oclip = CLIPVisualOnly(VIT_CONFIGS["ViT-B/32"]).eval()
    oclip.load_state_dict(vsd)
    for p in list(ounet.parameters()) + list(oclip.parameters()):
        p.requires_grad_(False)
    odiff = od.create_gaussian_diffusion(1000, "linear", "25")  # CLI default schedule overrides the cosine flag (quirk B8)
    pdiff = pgd.create_gaussian_diffusion(1000, "linear", "25")
    th.manual_seed(0)
    tgt = th.randn(1, 512)
    eng = pg.GuidedStepB200(ucfg, usd, vcfg, vsd, batch=1, num_cutouts=4, use_magnitude=True, device="cuda")
    eng.set_targets(tgt, th.ones(1))
    x = th.randn(1, 3, 64, 64)
    y = th.tensor([207])
    coords = [(0, 0, 64)] * 4  # 64^2: min == max == 64 -> whole-image windows (SURVEY App. E)
    t_index = 20
    cond = og.OracleCondFn(odiff, oclip, tgt, th.ones(1), cut_size=224, num_cutouts=4, use_magnitude=True)
    cond.current_timestep = t_index
    grabbed = {}

    def cond_fn(xx, tt, out, y=None):
        grabbed["g"] = cond(xx, tt, out, y=y, coords=coords).detach().clone()
        return grabbed["g"]

    th.manual_seed(5)
    o = odiff.p_sample_with_grad(ounet, x, th.tensor([t_index]), clip_denoised=False, cond_fn=cond_fn, model_kwargs={"y": y})
    th.manual_seed(5)
    noise = th.randn_like(x)
    eng.stage_step(pdiff.scalar_table(t_index, t_index, 0.0), coords, pdiff.model_timestep(t_index), y)
    eng.img(eng.unet.x_in).copy_(x)
    eng.img(eng.noise).copy_(noise)
    eng.replay("ancestral")
    th.cuda.synchronize()
    e = dict(sample=eng.img(eng.sample).cpu(), pred_xstart=eng.img(eng.x0).cpu(), g=eng.img(eng.g).cpu())
    res = compare(dict(sample=o["sample"], pred_xstart=o["pred_xstart"], g=grabbed["g"]), e)
    assert res["cos_g"] > 0.99 and res["rel_x0"] < 2e-2 and res["rel_sample"] < 2e-2, res


def test_cfg2_unet_properties():
    ucfg = pu.config_for(256, True)
    usd = pw.seeded_state_dict(pw.unet_param_shapes(ucfg), 1234)
    nets = [pu.UNetB200(ucfg, usd, batch=1, device="cuda", conv_impl=impl, seed_scale=16.0) for impl in (0, 1)]
    th.manual_seed(0)
    x = th.randn(1, 3, 256, 256, device="cuda")
    t = th.tensor([601.0], device="cuda")
    y = th.tensor([3], device="cuda")
    d_out = th.zeros(1, 6, 256, 256, device="cuda")
    d_out[:, :3] = th.randn(1, 3, 256, 256, device="cuda") * 0.05
    outs, grads = [], []
    for net in nets:
        outs.append(net(x, t, y).clone())
        grads.append(net.backward_input(d_out).clone() / net.seed_scale)
    assert th.isfinite(outs[0]).all() and th.isfinite(grads[0]).all()
    # tensor-core path vs the CUDA-core verification twin over all 106 convs + 16 attention blocks, both directions
    assert rel(outs[0], outs[1]) < 5e-3, rel(outs[0], outs[1])
    assert cos(grads[0], grads[1]) > 0.999 and rel(grads[0], grads[1]) < 3e-2, (cos(grads[0], grads[1]), rel(grads[0], grads[1]))
    # the backward is linear in its seed
    g2 = nets[0].backward_input(2 * d_out).clone() / nets[0].seed_scale
    assert rel(g2, 2 * grads[0]) < 2e-2, rel(g2, 2 * grads[0])
    # replay determinism (bitwise)
    again = nets[0](x, t, y).clone()
    assert th.equal(again, outs[0])
