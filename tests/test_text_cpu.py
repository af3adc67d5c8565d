"""CPU: text prompts on this package's own text tower -- the BPE tokenizer against ``transformers.CLIPTokenizer``, the fp32 oracle
against ``CLIPTextModelWithProjection``, the ``TextB200`` op list on the plan interpreter against the oracle, how the entry chooses
between the device tower and the ``clip`` package, and the argument checks of TOKEN_EMBED, ROW_GATHER and the causal flag."""
import os
import subprocess
import sys

import pytest
import torch as th

from clip_guided_diffusion_b200 import cgd
from clip_guided_diffusion_b200 import guidance as pg
from clip_guided_diffusion_b200 import text as ptx
from clip_guided_diffusion_b200 import tokenizer as ptok
from clip_guided_diffusion_b200 import unet as pu
from clip_guided_diffusion_b200 import vit as pv
from clip_guided_diffusion_b200 import weights as pw
from clip_guided_diffusion_b200._lib import OP
from clip_guided_diffusion_b200.plan import Plan
from tests import clip_text_oracle as oct
from tests.plan_interp import Interp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MERGES = oct.synthetic_merges(400)


@pytest.fixture(scope="module")
def vocab(tmp_path_factory):
    d = tmp_path_factory.mktemp("vocab")
    path = str(d / ptok.VOCAB_FILE)
    V = oct.write_vocab(path, MERGES)
    return path, V, d


# ---------------------------------------------------------------- tokenizer
PROMPTS = ["A lighthouse on a rocky coast", "it's the painter's 2nd  work;   3 boats", "12 BIRDS!! at sunset, oil-painting",
           "they're sure we've seen (the) red FOX... i'm told you'll find it", "Trending on ArtStation, 4k: highly-detailed #matte", "x",
           "   leading and trailing blanks   ", "numbers 2024 and 3.14159; percent 100%"]


def test_tokenizer_matches_transformers(vocab):
    from transformers import CLIPTokenizer
    path, V, d = vocab
    hf = CLIPTokenizer(*oct.write_hf_vocab(str(d), MERGES))
    tok = ptok.Tokenizer(path)
    assert len(tok) == V == len(MERGES) + 514 and (tok.sot, tok.eot) == (V - 2, V - 1)
    out = tok.tokenize(PROMPTS)
    assert out.dtype == th.int32 and out.shape == (len(PROMPTS), 77)
    for row, p in zip(out, PROMPTS):
        n = int((row != 0).sum())
        assert row[:n].tolist() == hf(p)["input_ids"], p
        assert row[0] == tok.sot and row[n - 1] == tok.eot and not row[n:].any()
    # transformers' CLIP tokenizer does not unescape HTML; CLIP's cleaning unescapes twice
    for p in ("a &amp; b", "a &amp;amp; b"):
        assert tok.encode(p) == hf("a & b")["input_ids"][1:-1]


def test_byte_symbols_have_the_published_ids(vocab):
    """the 512 byte-level ids are laid out in GPT-2's published byte order, not in byte order: `!` is 0, `a</w>` 320, chr(256) 188"""
    tok = ptok.Tokenizer(vocab[0])
    assert tok.byte_encoder == oct.BYTE_SYMBOL
    assert {k: tok.encoder[k] for k in oct.PUBLISHED_IDS} == oct.PUBLISHED_IDS
    assert [tok.encoder[s] for s in oct.SYMBOLS] == list(range(256))
    assert tok.encode("a , . 1 !") == [320, 267, 269, 272, 256]  # single-byte words: no merge applies


def test_tokenize_lengths_padding_and_truncation(vocab):
    path, _, _ = vocab
    tok = ptok.Tokenizer(path)
    ids = tok.encode("a lighthouse")
    out = ptok.tokenize(["a lighthouse", ""], context_length=8, bpe_path=path)
    assert out[0].tolist() == [tok.sot] + ids + [tok.eot] + [0] * (6 - len(ids))
    assert out[1].tolist() == [tok.sot, tok.eot] + [0] * 6
    long = " ".join(["lighthouse"] * 100)
    with pytest.raises(RuntimeError, match="too long for context length 77"):
        tok.tokenize([long])
    cut = tok.tokenize([long], truncate=True)[0]
    full = [tok.sot] + tok.encode(long) + [tok.eot]
    assert cut[:76].tolist() == full[:76] and cut[76] == tok.eot
    exact = tok.tokenize(["a"], context_length=len(tok.encode("a")) + 2)  # SOT + tokens + EOT fill the context exactly
    assert exact[0, -1] == tok.eot


def test_vocabulary_lookup_order(vocab, tmp_path, monkeypatch):
    path, _, _ = vocab
    monkeypatch.setattr(cgd, "CACHE_PATH", str(tmp_path / "cache"))
    ck = tmp_path / "ckpt"
    with pytest.raises(FileNotFoundError) as e:
        ptok.find_vocab(None, str(ck))
    assert str(ck / "clip" / ptok.VOCAB_FILE) in str(e.value) and str(tmp_path / "cache" / "clip" / ptok.VOCAB_FILE) in str(e.value)
    (tmp_path / "cache" / "clip").mkdir(parents=True)
    oct.write_vocab(tmp_path / "cache" / "clip" / ptok.VOCAB_FILE, MERGES[:10])
    assert ptok.find_vocab(None, str(ck)) == str(tmp_path / "cache" / "clip" / ptok.VOCAB_FILE)
    (ck / "clip").mkdir(parents=True)
    oct.write_vocab(ck / "clip" / ptok.VOCAB_FILE, MERGES[:20])
    assert ptok.find_vocab(None, str(ck)) == str(ck / "clip" / ptok.VOCAB_FILE)
    assert ptok.find_vocab(path, str(ck)) == path
    with pytest.raises(FileNotFoundError, match="bpe_path"):
        ptok.find_vocab(str(tmp_path / "nope.txt.gz"), str(ck))


def test_tokenizer_needs_regex(vocab, monkeypatch):
    monkeypatch.setitem(sys.modules, "regex", None)
    with pytest.raises(RuntimeError, match="`regex` module"):
        ptok.Tokenizer(vocab[0])


def test_published_vocabulary_layout(tmp_path):
    """more merges than CLIP uses: the vocabulary stops at 48 894 merges, SOT = 49406, EOT = 49407"""
    merges = [(f"a{i}", f"b{i}") for i in range(ptok.N_MERGES + 50)]
    oct.write_vocab(tmp_path / "v.txt.gz", merges)
    tok = ptok.Tokenizer(str(tmp_path / "v.txt.gz"))
    assert len(tok) == 49408 and (tok.sot, tok.eot) == (49406, 49407)


# ---------------------------------------------------------------- oracle vs transformers
def _text_sd(width, layers, D=32, T=77, V=None, seed=5):
    cfg = ptx.TextConfig(width=width, layers=layers, context_length=T, vocab_size=V or len(MERGES) + 514, output_dim=D)
    return cfg, pw.seeded_state_dict(pw.text_param_shapes(cfg), seed)


def _ids(cfg, lengths, seed=0):
    g = th.Generator().manual_seed(seed)
    ids = th.zeros(len(lengths), cfg.context_length, dtype=th.int32)
    for i, n in enumerate(lengths):
        ids[i, 0] = cfg.vocab_size - 2
        ids[i, 1:n - 1] = th.randint(1, cfg.vocab_size - 2, (n - 2,), generator=g)
        ids[i, n - 1] = cfg.vocab_size - 1
    return ids


@pytest.mark.parametrize("width,layers,T", [(64, 2, 16), (512, 12, 77)])
def test_oracle_matches_transformers(width, layers, T):
    cfg, sd = _text_sd(width, layers, D=48, T=T, V=600)
    ids = _ids(cfg, [2, 5, T])
    m = oct.hf_text_model(sd, T, cfg.vocab_size)
    with th.no_grad():
        ref = m(input_ids=ids.long()).text_embeds.double()
    got = oct.encode_text(sd, ids).double()
    assert float((got - ref).norm() / ref.norm()) < 1e-5


# ---------------------------------------------------------------- the tower's op list on the interpreter
def _interp_tower(cfg, sd, n):
    tower = ptx.TextB200(cfg, sd, n, device="cpu")
    it = oct.TextInterp(tower.plan)
    tower.plan.run = lambda first=0, count=None, stream=None: it.run(first, count)
    return tower


def _cos(a, b):
    return th.nn.functional.cosine_similarity(a.double(), b.double(), dim=-1)


@pytest.mark.parametrize("width,layers", [(64, 2), (640, 1)])
def test_text_tower_on_the_interpreter_matches_the_oracle(width, layers):
    cfg, sd = _text_sd(width, layers, D=40)
    ids = _ids(cfg, [2, 9, 40, 77], seed=3)
    tower = _interp_tower(cfg, sd, 4)
    codes = [op.code for op in tower.plan.ops]
    attn = [op for op in tower.plan.ops if op.code == OP["ATTN_FWD"]]
    assert len(attn) == layers and all(op.flags == 1 for op in attn)
    assert codes.count(OP["TOKEN_EMBED"]) == 1 and codes.count(OP["ROW_GATHER"]) == 1 and OP["ATTN_BWD"] not in codes
    got = tower.encode(ids)
    ref = oct.encode_text(sd, ids)
    assert got.shape == ref.shape == (4, 40)
    assert float(_cos(got, ref).min()) > 0.999
    assert float((got - ref).norm() / ref.norm()) < 1e-2


def test_text_configs_of_the_published_towers():
    """B/32, RN50x4 and L/14 text towers (widths 512 / 640 / 768), read back from their shapes next to a visual tower's keys"""
    vis = {k: th.zeros(v) for k, v in pw.vit_param_shapes(pv.ViTConfig(224, 32, 768, 2, 512)).items()}
    for width, D in ((512, 512), (640, 640), (768, 768)):
        cfg = ptx.TextConfig(width=width, layers=12, output_dim=D)
        sd = {**vis, **{k: th.zeros(v) for k, v in pw.text_param_shapes(cfg).items()}}
        assert ptx.text_config_from_state_dict(sd) == cfg and cfg.heads == width // 64


def test_token_ids_are_checked_on_the_host():
    cfg, sd = _text_sd(64, 1, T=16)
    tower = _interp_tower(cfg, sd, 2)
    bad = _ids(cfg, [3, 4])
    bad[1, 2] = cfg.vocab_size
    with pytest.raises(ValueError, match=r"token ids must lie in \[0, %d\)" % cfg.vocab_size):
        tower.encode(bad)
    bad[1, 2] = -1
    with pytest.raises(ValueError, match="token ids must lie"):
        tower.encode(bad)
    with pytest.raises(ValueError, match="this tower encodes"):
        tower.encode(_ids(cfg, [3]))


def test_visual_only_state_dict_has_no_text_tower():
    vsd = pw.seeded_state_dict(pw.vit_param_shapes(pv.ViTConfig(32, 16, 64, 1, 32)), 1)
    with pytest.raises(ValueError, match="no text tower"):
        ptx.text_config_from_state_dict(vsd)


def test_causal_attention_has_no_backward():
    p = Plan()
    x = p.act(1, 1, 8, 3 * 64)
    out = p.attention(x, 1, 8, 1, legacy_order=False, causal=True)
    p._grads[out.key()] = p.act(1, 1, 8, 64)
    with pytest.raises(NotImplementedError, match="causal attention has no backward"):
        p.backward()


# ---------------------------------------------------------------- the entry on the interpreter
VCFG = pv.ViTConfig(32, 16, 64, 1, 32)  # a one-layer CLIP tower (as tests/test_entry_cpu.py)
_REAL_CLIP_IMPORTABLE = cgd._clip_importable


class _RecordingEngine(pg.GuidedStepB200):
    seen = []

    def __init__(self, *a, **k):
        k["device"] = "cpu"
        self.seen.append({"P": k["max_prompts"]})
        super().__init__(*a, **k)
        it = Interp(self.plan)
        self.plan.run_range = lambda a, b, stream=None: it.run_range(a, b)
        self.plan.run = lambda first=0, count=None, stream=None: it.run(first, len(self.plan.ops) - first if count is None else count)

    def set_targets(self, target_embeds, weights):
        self.seen[-1].update(targets=target_embeds.clone(), weights=weights.clone())
        super().set_targets(target_embeds, weights)


class _InterpTower(ptx.TextB200):
    """stand-in for cgd.TextB200 (the device tower): the same op list, run by the interpreter"""
    built = []

    def __init__(self, cfg, sd, n_prompts, device="cuda"):
        super().__init__(cfg, sd, n_prompts, device="cpu")
        type(self).built.append(n_prompts)
        it = oct.TextInterp(self.plan)
        self.plan.run = lambda first=0, count=None, stream=None: it.run(first, count)


@pytest.fixture
def entry(tmp_path, monkeypatch, vocab):
    monkeypatch.setattr(cgd, "_require_cuda", lambda device: None)
    monkeypatch.setattr(cgd, "GuidedStepB200", _RecordingEngine)
    monkeypatch.setattr(cgd, "TextB200", _InterpTower)
    monkeypatch.setattr(cgd, "_clip_importable", lambda: False)
    monkeypatch.setattr(cgd, "CACHE_PATH", str(tmp_path / "cache"))
    monkeypatch.chdir(tmp_path)
    _RecordingEngine.seen.clear()
    _InterpTower.built.clear()
    usd = pw.seeded_state_dict(pw.unet_param_shapes(pu.config_for(64, True)), 1234)
    tcfg = ptx.TextConfig(width=64, layers=1, context_length=24, vocab_size=vocab[1], output_dim=32)
    csd = {**pw.seeded_state_dict(pw.vit_param_shapes(VCFG), 1235), **pw.seeded_state_dict(pw.text_param_shapes(tcfg), 1236)}
    return dict(usd=usd, csd=csd, tmp=tmp_path, vocab=vocab[0])


def _run(e, **kw):
    args = dict(image_size=64, num_cutouts=2, batch_size=1, timestep_respacing="25", skip_timesteps=24, save_frequency=1,
                prefix_path=e["tmp"] / "out", progress=False, seed=3, device="cpu", unet_state_dict=e["usd"], clip_state_dict=e["csd"],
                checkpoints_dir=str(e["tmp"] / "ckpt"))
    args.update(kw)
    return list(cgd.clip_guided_diffusion(**args))


def _no_clip(*a, **k):
    raise AssertionError("the device tower was chosen: the clip path must not run")


def test_entry_device_text_encoder(entry, monkeypatch):
    """P, prompt order and normalised weights as the clip path would give them: one tower for all prompts"""
    monkeypatch.setattr(cgd, "_encode_text", _no_clip)
    prompts = ["a lighthouse:2", "oil painting of a fox:-0.5", "rocky coast"]
    got = _run(entry, prompts=prompts, text_encoder="device", bpe_path=entry["vocab"])
    assert len(got) == 1 and os.path.exists(got[0][1])
    seen = _RecordingEngine.seen[-1]
    assert seen["P"] == 3 and _InterpTower.built == [3]
    ids = ptok.tokenize(["a lighthouse", "oil painting of a fox", "rocky coast"], context_length=24, bpe_path=entry["vocab"])
    ref = oct.encode_text(entry["csd"], ids)
    assert float(_cos(seen["targets"], ref).min()) > 0.999
    assert th.allclose(seen["weights"], th.tensor([2.0, -0.5, 1.0]) / 2.5, rtol=0, atol=1e-7)


def test_entry_auto_without_clip_or_vocabulary_calls_encode_text(entry, monkeypatch):
    calls = []

    def fake(prompts, name, device):
        calls.append((list(prompts), name, device))
        return th.randn(len(prompts), 32, generator=th.Generator().manual_seed(1)), th.ones(len(prompts))

    monkeypatch.setattr(cgd, "_encode_text", fake)
    _run(entry, prompts=["a", "b"])
    assert calls == [(["a", "b"], "ViT-B/32", "cpu")] and _InterpTower.built == []
    with pytest.raises(FileNotFoundError, match=ptok.VOCAB_FILE):
        _run(entry, prompts=["a"], text_encoder="device")
    calls.clear()
    _run(entry, prompts=["a"], text_encoder="clip", bpe_path=entry["vocab"])  # forced: the vocabulary is not used
    assert calls == [(["a"], "ViT-B/32", "cpu")] and _InterpTower.built == []
    with pytest.raises(ValueError, match="text_encoder"):
        _run(entry, prompts=["a"], text_encoder="gpu")


def test_entry_auto_finds_the_vocabulary_under_checkpoints_dir(entry, monkeypatch):
    monkeypatch.setattr(cgd, "_encode_text", _no_clip)
    (entry["tmp"] / "ckpt" / "clip").mkdir(parents=True)
    oct.write_vocab(entry["tmp"] / "ckpt" / "clip" / ptok.VOCAB_FILE, MERGES)
    _run(entry, prompts=["a lighthouse"])
    assert _InterpTower.built == [1] and _RecordingEngine.seen[-1]["P"] == 1
    # with the clip package importable, "auto" prefers it
    monkeypatch.setattr(cgd, "_clip_importable", lambda: True)
    monkeypatch.setattr(cgd, "_encode_text", lambda prompts, name, device: (th.ones(len(prompts), 32), th.ones(len(prompts))))
    _run(entry, prompts=["a lighthouse"])
    assert _InterpTower.built == [1]


def test_auto_treats_a_clip_package_that_fails_to_import_as_absent(entry, monkeypatch):
    """an installed `clip` whose import raises: "auto" falls back to the device tower instead of choosing the clip path"""
    pkg = entry["tmp"] / "site" / "clip"
    pkg.mkdir(parents=True)
    (pkg / "__init__.py").write_text("raise OSError('broken install')\n")
    monkeypatch.syspath_prepend(str(entry["tmp"] / "site"))
    monkeypatch.delitem(sys.modules, "clip", raising=False)
    monkeypatch.setattr(cgd, "_clip_importable", _REAL_CLIP_IMPORTABLE)  # the real predicate, not the fixture's stand-in
    assert not cgd._clip_importable()
    monkeypatch.setattr(cgd, "_encode_text", _no_clip)
    _run(entry, prompts=["a lighthouse"], bpe_path=entry["vocab"])
    assert _InterpTower.built == [1]


def test_entry_image_only_builds_no_text_tower(entry, monkeypatch):
    from tests import image_prompt_oracle as oip
    monkeypatch.setattr(cgd, "_encode_text", _no_clip)

    class _Enc:
        def __init__(self, cfg, sd, cutn, device="cuda"):
            self.cutn = cutn

        def encode(self, image, weight, size):
            return th.ones(self.cutn, 32), [weight / self.cutn] * self.cutn

    monkeypatch.setattr(cgd, "ImagePromptEncoder", _Enc)
    oip.write_png(entry["tmp"] / "a.png", 40, 50, seed=1)
    _run(entry, prompts=[], image_prompts=[str(entry["tmp"] / "a.png")], text_encoder="device", bpe_path=entry["vocab"])
    assert _InterpTower.built == [] and _RecordingEngine.seen[-1]["P"] == 2


# ---------------------------------------------------------------- argument checks without a device
ARGS_CHILD = r"""
import ctypes, sys
sys.path.insert(0, sys.argv[1])
from clip_guided_diffusion_b200 import _lib
lib = _lib.load()
good = 1 << 40
def run(code, i, p, flags=0):
    op = _lib.CgdOp()
    op.code, op.flags = _lib.OP[code], flags
    for k, x in enumerate(i):
        op.i[k] = x
    for k, x in enumerate(p):
        op.p[k] = x
    rc = lib.cgd_run_op(ctypes.byref(op), None)
    print("CASE", code, flags, i, [x - good if x else 0 for x in p], rc, lib.cgd_last_error().decode().replace(" ", "_"), flush=True)
P4 = [good, good + 4096, good + 8192, good + 12288]
base = {"TOKEN_EMBED": [3, 77, 512, 49408], "ROW_GATHER": [3, 512, 512, 512, 231]}
for code, ii in base.items():
    for j in range(len(ii)):
        for v in (0, -1, 1 << 31, 1 << 40):
            vals = list(ii); vals[j] = v; run(code, vals, P4)
    np = 4 if code == "TOKEN_EMBED" else 3
    for j in range(np):
        for v in (0, 8):
            ptrs = list(P4[:np]); ptrs[j] = 0 if v == 0 else ptrs[j] + v
            if code == "ROW_GATHER" and j == 1 and v:
                ptrs[j] = P4[1] + 2  # idx is an int32 array: 4-byte alignment is enough, 2 is not
            run(code, ii, ptrs)
    vals = list(ii); vals[2 if code == "TOKEN_EMBED" else 1] = 500; run(code, vals, P4)  # w % 8 != 0
    if code == "ROW_GATHER":
        run(code, [3, 512, 504, 512, 231], P4)  # ldx < w
        run(code, [3, 512, 512, 516, 231], P4)  # ldy % 8 != 0
    print("OK", code, flush=True); run(code, ii, P4[:np])
attn = [2, 8, 77, 64, 77 * 1536, 1536, 64, 77 * 512, 512, 64]
print("OK ATTN_FWD", flush=True); run("ATTN_FWD", attn, [good, good + 1024, good + 2048, good + 4096, good + 8192], flags=1)
run("ATTN_FWD", attn, [good, good + 1024, good + 2048, good + 4096, good + 8192], flags=2)
run("ATTN_BWD", attn, [good + 1024 * k for k in range(10)], flags=1)
print("DONE", flush=True)
"""


@pytest.mark.skipif(th.cuda.is_available(), reason="needs a box WITHOUT a GPU: only the argument checks may run")
def test_text_ops_reject_malformed_operands_without_a_device():
    """bad dims, V <= 0, w % 8, null or misaligned pointers, strides below w, a causal ATTN_BWD or an unknown ATTN_FWD flag: a negative
    return before any CUDA call.  Well-formed ops (after each "OK") reach the launch, which fails for lack of a device."""
    r = subprocess.run([sys.executable, "-c", ARGS_CHILD, ROOT], capture_output=True, text=True, timeout=120)
    lines = r.stdout.splitlines()
    assert r.returncode == 0 and lines and lines[-1] == "DONE", r.stderr[-400:]
    ok_next, n_bad = False, 0
    for l in lines[:-1]:
        if l.startswith("OK"):
            ok_next = True
            continue
        rc, msg = int(l.split(" ")[-2]), l.split(" ")[-1]
        if ok_next:
            assert rc > 0, l
            ok_next = False
        else:
            n_bad += 1
            assert rc == -1 and ("token_embed" in msg or "row_gather" in msg or "attention" in msg), l
    assert n_bad == 56
    assert any("no_causal_backward" in l for l in lines) and any("flags_2_unsupported" in l for l in lines)
