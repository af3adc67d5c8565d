"""Where do non-finite values first appear in a cfg2 chain with random weights?  Prints max|.| of key buffers per segment."""
import os, sys
import torch as th
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench

th.cuda.set_device(0)
eng, diff, cond = bench.build_engine(th.device("cuda", 0), 0, 1)
eng.use_graph = False
th.manual_seed(0)
img = eng.draw_initial_noise()
i = diff.num_timesteps - 1
p = eng.plan
vt = eng.towers[0].by_count[eng.cutn]  # the (only) CLIP tower at the default cutout count


def stat(name, t):
    t = t.float()
    print(f"   {name:12s} max|.|={float(t.abs().max()):.4e} finite={bool(th.isfinite(t).all())} mean|.|={float(t.abs().mean()):.4e}")


segs = [("unet_emb", "unet_bwd"), ("pmv", "cond"), ("cut_fwd", "sph"), ("vit_fwd", "vit_bwd"), ("sph", "cut_bwd"), ("vit_bwd", "vit_end"),
        ("cut_bwd", "guide"), ("guide", "final"), ("unet_bwd", "unet_end"), ("final", "upd_anc_g"), ("upd_ddim_g", "upd_ddim")]
for step in range(6):
    y = eng.draw_classes()
    coords = cond.next_coords(eng.H, eng.W)
    eng.stage_step(diff.scalar_table(i, cond.current_timestep, 0.0), coords, diff.model_timestep(i), y)
    eng.img(eng.unet.x_in).copy_(img)
    eng.draw_noise()
    print(f"step {step} t={i}")
    stat("x_t", eng.img(eng.unet.x_in))
    for a, b in segs:
        p.run_range(a, b)
        th.cuda.synchronize()
        if a == "unet_emb":
            stat("model_out", eng.unet.out_view)
        elif a == "pmv":
            stat("pred_xstart", eng.img(eng.x0)); stat("x_in", eng.img(eng.x_inb))
        elif a == "cut_fwd":
            stat("patches", p.view(vt.patches))
        elif a == "vit_fwd":
            stat("embeds", p.view(vt.embeds))
        elif a == "sph":
            stat("d_embeds", p.view(vt.d_embeds))
        elif a == "vit_bwd":
            stat("d_patches", p.view(vt.d_patches))
        elif a == "cut_bwd":
            stat("g_clip", eng.img(eng.g_clip))
        elif a == "guide":
            stat("seed", eng.unet.seed_view[:, :, :6]); stat("dx_direct", eng.img(eng.dx_direct))
        elif a == "unet_bwd":
            stat("dx_unet", eng.unet.dx_view)
        elif a == "final":
            stat("g", eng.img(eng.g))
        else:
            stat("sample", eng.img(eng.sample))
    print("   losses", {k: v.tolist() for k, v in eng.losses().items()})
    img = eng.img(eng.sample).clone()
    cond.step_done()
    i -= 1
