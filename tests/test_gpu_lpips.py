"""GPU: the LPIPS-VGG16 init loss (clip_guided_diffusion_b200/lpips.py + csrc/lpips.cu + the wgmma conv kernel): every op against
the PyTorch interpreter on identical inputs, loss value and x_in-gradient against the fp32 oracle restatement of
``lpips.LPIPS(net='vgg')`` ([3P], cgd/cgd.py:147-148, 220-224; SURVEY.md A.4)."""
import pytest
import torch as th

from tests.gpu_harness import compare_ops
from tests.test_lpips_cpu import build, reference

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("shape", [(2, 32, 48), (1, 256, 256)], ids=["b2_32x48", "b1_256x256"])
def test_lpips_value_and_gradient_vs_oracle(shape):
    B, H, W = shape
    scale = 1000.0
    sd, plan, lp, x_src, g_dst = build("cuda", B, H, W, scale)
    th.manual_seed(0)
    init = th.rand(1, 3, H, W) * 2 - 1
    x = (th.rand(B, 3, H, W) * 2 - 1) * 0.9
    lp.set_init_image(init.cuda())
    plan.view(x_src, (B, 3, H, W)).copy_(x)
    plan.view(g_dst, (B, 3, H, W)).fill_(0.25)
    plan.run_range("lpips", "lpips_end")
    th.cuda.synchronize()
    val, g = reference(sd, x, init, scale)
    got_val = lp.loss_value().cpu()
    got_g = plan.view(g_dst, (B, 3, H, W)).cpu() - 0.25
    assert th.isfinite(got_g).all()
    assert th.allclose(got_val, val, rtol=3e-2, atol=1e-4), (got_val, val)
    cosg = float(th.nn.functional.cosine_similarity(got_g.flatten(), g.flatten(), dim=0))
    relg = float((got_g - g).norm() / g.norm())
    assert cosg > 0.998 and relg < 6e-2, (cosg, relg)  # fp16 activations / weights through 13 conv + ReLU layers, both directions


def test_lpips_ops_match_interpreter():
    B, H, W = 2, 32, 48
    sd, plan, lp, x_src, g_dst = build("cuda", B, H, W, 1000.0)
    th.manual_seed(1)
    lp.set_init_image((th.rand(1, 3, H, W) * 2 - 1).cuda())
    plan.view(x_src, (B, 3, H, W)).copy_((th.rand(B, 3, H, W) * 2 - 1))
    th.cuda.synchronize()
    n, failures = compare_ops(plan, [("lpips", "lpips_end")])
    assert not failures, f"{len(failures)} of {n} ops differ from the interpreter:\n" + "\n".join(str(f) for f in failures[:20])
