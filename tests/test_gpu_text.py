"""GPU: text prompts on the device -- causal ATTN_FWD (small and flash kernels) against fp32 ``scaled_dot_product_attention``,
TOKEN_EMBED / ROW_GATHER against torch indexing, the text towers of widths 512 / 640 / 768 against the fp32 oracle, and
``clip_guided_diffusion(prompts=..., text_encoder="device")`` end to end.  Optional checks against the published vocabulary file and
the ``clip`` package run when those are present."""
import os

import pytest
import torch as th
import torch.nn.functional as F

from clip_guided_diffusion_b200 import _lib
from clip_guided_diffusion_b200 import cgd
from clip_guided_diffusion_b200 import guidance as pg
from clip_guided_diffusion_b200 import text as ptx
from clip_guided_diffusion_b200 import tokenizer as ptok
from clip_guided_diffusion_b200 import unet as pu
from clip_guided_diffusion_b200 import vit as pv
from clip_guided_diffusion_b200 import weights as pw
from tests import clip_text_oracle as oct
from tests import gpu_harness

pytestmark = pytest.mark.gpu

gpu_harness.OUT_PTRS.update({"TOKEN_EMBED": [3], "ROW_GATHER": [2]})


# ---------------------------------------------------------------- causal attention
def _causal(B, heads, T, d, seed):
    C = heads * d
    g = th.Generator().manual_seed(seed)
    qkv = th.randn(B, T, 3 * C, generator=g).half().cuda()
    out = th.full((B, T, C), float("nan"), dtype=th.float16, device="cuda")
    lse = th.empty(B, heads, T, device="cuda")
    _lib.run_op("ATTN_FWD", i=[B, heads, T, d, T * 3 * C, 3 * C, d, T * C, C, d], p=[qkv, qkv[..., C:], qkv[..., 2 * C:], out, lse], f=[d ** -0.5],
            flags=1)
    q, k, v = (t.float().view(B, T, heads, d).transpose(1, 2) for t in qkv.split(C, dim=-1))
    ref = F.scaled_dot_product_attention(q, k, v, is_causal=True).transpose(1, 2).reshape(B, T, C)
    s = (q @ k.transpose(-1, -2)) * d ** -0.5
    ref_lse = th.logsumexp(s.masked_fill(th.ones(T, T, dtype=th.bool, device="cuda").triu(1), float("-inf")), dim=-1)
    return out.float(), ref, lse, ref_lse


@pytest.mark.parametrize("heads", [8, 10, 12])
@pytest.mark.parametrize("T", [1, 17, 64, 65, 77, 128, 300])
def test_causal_attention_matches_sdpa(T, heads):
    """T <= 64 runs the single-tile kernel, larger T the flash kernel (which stops at the diagonal key tile)"""
    out, ref, lse, ref_lse = _causal(2, heads, T, 64, seed=T * 100 + heads)
    assert th.isfinite(out).all()
    assert float((out - ref).abs().max()) <= 4e-3 * float(ref.abs().max())
    assert float((lse - ref_lse).abs().max()) < 1e-3


@pytest.mark.parametrize("d,T", [(128, 150), (192, 77), (256, 100)])
def test_causal_attention_wide_heads(d, T):
    out, ref, lse, ref_lse = _causal(2, 4, T, d, seed=d + T)
    assert float((out - ref).abs().max()) <= 4e-3 * float(ref.abs().max())
    assert float((lse - ref_lse).abs().max()) < 1e-3


def test_non_causal_attention_is_unchanged_by_the_flag_path():
    """flags 0 still attends to every key"""
    B, heads, T, d = 1, 8, 77, 64
    C = heads * d
    qkv = th.randn(B, T, 3 * C, generator=th.Generator().manual_seed(1)).half().cuda()
    out = th.empty(B, T, C, dtype=th.float16, device="cuda")
    lse = th.empty(B, heads, T, device="cuda")
    _lib.run_op("ATTN_FWD", i=[B, heads, T, d, T * 3 * C, 3 * C, d, T * C, C, d], p=[qkv, qkv[..., C:], qkv[..., 2 * C:], out, lse], f=[d ** -0.5])
    q, k, v = (t.float().view(B, T, heads, d).transpose(1, 2) for t in qkv.split(C, dim=-1))
    ref = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B, T, C)
    assert float((out.float() - ref).abs().max()) <= 4e-3 * float(ref.abs().max())


# ---------------------------------------------------------------- gathers
@pytest.mark.parametrize("n,T,w,V", [(3, 77, 512, 49408), (1, 5, 768, 1000), (5, 77, 640, 300)])
def test_token_embed_is_exact(n, T, w, V):
    g = th.Generator().manual_seed(n + T + w)
    ids = th.randint(0, V, (n, T), generator=g, dtype=th.int32)
    table = th.randn(V, w, generator=g).half()
    pos = th.randn(T, w, generator=g) * 0.1
    x = th.empty(n, T, w, dtype=th.float16, device="cuda")
    _lib.run_op("TOKEN_EMBED", i=[n, T, w, V], p=[ids.cuda(), table.cuda(), pos.cuda(), x])
    assert th.equal(x.cpu(), (table.float()[ids.long()] + pos).half())
    ids[0, 1], ids[-1, -1] = V, -3  # outside the table: NaN rows, nothing read outside it
    _lib.run_op("TOKEN_EMBED", i=[n, T, w, V], p=[ids.cuda(), table.cuda(), pos.cuda(), x])
    got = x.cpu()
    assert got[0, 1].isnan().all() and got[-1, -1].isnan().all() and th.isfinite(got[0, 0]).all()


@pytest.mark.parametrize("rows,w,ldx,ldy,n_src", [(4, 512, 512, 512, 4 * 77), (3, 768, 1024, 776, 50), (1, 8, 8, 8, 1)])
def test_row_gather_is_exact(rows, w, ldx, ldy, n_src):
    g = th.Generator().manual_seed(rows * w)
    x = th.randn(n_src, ldx, generator=g).half()
    idx = th.randint(0, n_src, (rows,), generator=g, dtype=th.int32)
    y = th.zeros(rows, ldy, dtype=th.float16, device="cuda")
    _lib.run_op("ROW_GATHER", i=[rows, w, ldx, ldy, n_src], p=[x.cuda(), idx.cuda(), y])
    assert th.equal(y.cpu()[:, :w], x[idx.long(), :w]) and not y.cpu()[:, w:].any()
    idx[0] = n_src
    _lib.run_op("ROW_GATHER", i=[rows, w, ldx, ldy, n_src], p=[x.cuda(), idx.cuda(), y])
    assert y.cpu()[0, :w].isnan().all()


# ---------------------------------------------------------------- text towers
def _ids(cfg, lengths, seed=0):
    g = th.Generator().manual_seed(seed)
    ids = th.zeros(len(lengths), cfg.context_length, dtype=th.int32)
    for i, n in enumerate(lengths):
        ids[i, 0] = cfg.vocab_size - 2
        ids[i, 1:n - 1] = th.randint(1, cfg.vocab_size - 2, (n - 2,), generator=g)
        ids[i, n - 1] = cfg.vocab_size - 1
    return ids


@pytest.mark.parametrize("width", [512, 640, 768])
def test_text_tower_matches_the_oracle(width):
    """the B/32, RN50x4 and L/14 text towers' shapes (12 layers, 77 tokens, full vocabulary) with seeded weights"""
    cfg = ptx.TextConfig(width=width, layers=12, output_dim=width)
    sd = pw.seeded_state_dict(pw.text_param_shapes(cfg), width)
    ids = _ids(cfg, [2, 7, 33, 77, 50], seed=width)
    tower = ptx.TextB200(cfg, sd, 5)
    got = tower.encode(ids).cpu()
    ref = oct.encode_text(sd, ids)
    cos = F.cosine_similarity(got.double(), ref.double(), dim=-1)
    rel = (got - ref).norm(dim=-1) / ref.norm(dim=-1)
    assert float(cos.min()) > 0.999 and float(rel.max()) < 1e-2, (cos, rel)


def test_text_tower_ops_match_the_interpreter(monkeypatch):
    """every op of a two-layer tower against the interpreter on identical inputs"""
    cfg = ptx.TextConfig(width=512, layers=2, output_dim=512)
    sd = pw.seeded_state_dict(pw.text_param_shapes(cfg), 3)
    tower = ptx.TextB200(cfg, sd, 3)
    tower.encode(_ids(cfg, [5, 77, 20]))
    monkeypatch.setattr(gpu_harness, "Interp", oct.TextInterp)
    n, failures = gpu_harness.compare_ops(tower.plan, [("text_fwd", "text_end")])
    assert n == len(tower.plan.ops) and not failures, failures[:3]


# ---------------------------------------------------------------- the entry
@pytest.fixture(scope="module")
def synthetic_vocab(tmp_path_factory):
    d = tmp_path_factory.mktemp("vocab")
    path = str(d / ptok.VOCAB_FILE)
    return path, oct.write_vocab(path, oct.synthetic_merges(400))


def test_clip_guided_diffusion_with_device_text_prompts(tmp_path, monkeypatch, synthetic_vocab):
    monkeypatch.chdir(tmp_path)
    path, V = synthetic_vocab
    ucfg, vcfg = pu.config_for(64, True), pv.VIT_CONFIGS["ViT-B/32"]
    tcfg = ptx.TextConfig(width=512, layers=12, vocab_size=V, output_dim=512)
    usd = pw.seeded_state_dict(pw.unet_param_shapes(ucfg), 1234)
    csd = {**pw.seeded_state_dict(pw.vit_param_shapes(vcfg), 1235), **pw.seeded_state_dict(pw.text_param_shapes(tcfg), 1236)}
    seen = []

    class Engine(pg.GuidedStepB200):
        def set_targets(self, target_embeds, weights):
            seen.append((target_embeds.detach().float().cpu().clone(), th.as_tensor(weights).clone()))
            super().set_targets(target_embeds, weights)

    monkeypatch.setattr(cgd, "GuidedStepB200", Engine)
    monkeypatch.setattr(cgd, "_encode_text", lambda *a, **k: pytest.fail("text_encoder='device' must not use the clip package"))
    prompts = ["a lighthouse on a rocky coast:2", "oil painting of a fox", "sunset:-0.5"]
    got = list(cgd.clip_guided_diffusion(image_size=64, num_cutouts=4, prompts=prompts, batch_size=1, timestep_respacing="25",
                                         skip_timesteps=22, save_frequency=2, prefix_path=tmp_path / "out", progress=False, seed=0,
                                         unet_state_dict=usd, clip_state_dict=csd, text_encoder="device", bpe_path=path))
    assert [b for b, _ in got] == [0, 0] and all(os.path.exists(p) for _, p in got)
    (targets, weights), = seen
    ids = ptok.tokenize(["a lighthouse on a rocky coast", "oil painting of a fox", "sunset"], bpe_path=path)
    ref = oct.encode_text(csd, ids)
    assert targets.shape == (3, 512) and float(F.cosine_similarity(targets.double(), ref.double(), dim=-1).min()) > 0.999
    assert th.allclose(weights.float(), th.tensor([2.0, 1.0, -0.5]) / 2.5, atol=1e-7)
    emb, w = cgd.encode_text_prompt("oil painting of a fox", 0.7, clip_state_dict=csd, bpe_path=path)
    assert w == 0.7 and emb.shape == (1, 512) and emb.is_cuda
    assert float(F.cosine_similarity(emb.cpu().double(), ref[1:2].double(), dim=-1)) > 0.999


# ---------------------------------------------------------------- optional: the published vocabulary, the clip package
def _published_vocab():
    try:
        return ptok.find_vocab(None, cgd.CACHE_PATH)
    except FileNotFoundError:
        try:
            import clip
            p = os.path.join(os.path.dirname(clip.__file__), ptok.VOCAB_FILE)
            return p if os.path.exists(p) else None
        except ImportError:
            return None


def test_published_vocabulary():
    path = _published_vocab()
    if path is None:
        pytest.skip("CLIP's bpe_simple_vocab_16e6.txt.gz is not present")
    tok = ptok.Tokenizer(path)
    assert len(tok) == 49408 and (tok.sot, tok.eot) == (49406, 49407)


def test_matches_the_clip_package():
    clip = pytest.importorskip("clip")
    texts = ["a lighthouse on a rocky coast", "It's 3 o'clock &amp; the sky is   RED!"]
    path = os.path.join(os.path.dirname(clip.__file__), ptok.VOCAB_FILE)
    assert th.equal(ptok.tokenize(texts, bpe_path=path), clip.tokenize(texts).to(th.int32))
    ckpt = os.path.expanduser("~/.cache/clip/ViT-B-32.pt")  # a local file only: clip.load(name) would download
    if not os.path.exists(ckpt):
        pytest.skip("no local ViT-B/32 checkpoint")
    model = clip.load(ckpt, jit=False, device="cuda")[0].eval()
    sd = {k: v.float().cpu() for k, v in model.state_dict().items()}
    with th.no_grad():
        ref = model.encode_text(clip.tokenize(texts).cuda()).float().cpu()
    got = ptx.TextB200(ptx.text_config_from_state_dict(sd), sd, 2).encode(ptok.tokenize(texts, bpe_path=path)).cpu()
    assert float(F.cosine_similarity(got.double(), ref.double(), dim=-1).min()) > 0.999
