"""GPU tests of the native CLIP text encoder (pytest -m gpu): the causal attention and the two new GEMM epilogues
against float64 at the kernel suite's 5e-6 (scaled with K above 1024 for the wgmma GEMM), the whole tower against the float64 oracle and the transformers
golden, kernel selection, the host-side savings, and text -> joints end to end against the oracle chain."""
import pytest
import torch
import torch.nn.functional as F

from conftest import golden
from mld_b200 import synth
from oracle import mld_oracle as O
from oracle.clip_text import ClipTextCfg, clip_text_forward
from oracle.make_golden_clip import WEIGHT_SEED, golden_ids

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / b.abs().max())


def _tc_tol(K):
    """The CUDA-core kernel meets 5e-6 at every K.  The wgmma kernel's fp32 accumulator adds an error that grows
    with K (measured 7.7e-6 at K = 2304 and 1.2e-5 at K = 3072 on an H100): 5e-6 per 1024 of K, never below 5e-6."""
    return 5e-6 * max(1.0, K / 1024)


def _rel_rows(a, b):
    """Worst per-sequence relative-to-max error (a, b: [n, ...])."""
    return max(_rel(a[i], b[i]) for i in range(a.shape[0]))


@pytest.fixture(scope="module")
def eng(built_lib):
    from mld_b200.engine import Engine, make_config
    return Engine(make_config(num_layers=0, vae="none"), 0)


@pytest.fixture(scope="module")
def tower(built_lib):
    """A text-only engine with the full CLIP-L/14 tower (synthetic weights) and the float64 weights on the GPU."""
    from mld_b200 import _lib
    from mld_b200.engine import Engine, make_config
    sd = synth.clip_text_state_dict(WEIGHT_SEED)
    e = Engine(make_config(num_layers=0, vae="none"), 0)
    e.text_configure(_lib.default_text_config())
    e.load_state_dict(sd, "text_encoder.")
    e.finalize()
    sd64 = {k: v.double().cuda() for k, v in sd.items()}
    return e, sd, sd64


def _causal_ref(qkv, nseq, L, heads):
    d = qkv.shape[1] // 3
    hd = d // heads
    q, k, v = (t.reshape(nseq, L, heads, hd).transpose(1, 2) for t in qkv.double().split(d, dim=1))
    s = q @ k.transpose(-1, -2) / hd ** 0.5 + torch.full((L, L), float("-inf"), dtype=torch.float64).triu(1)
    return (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(nseq * L, d)


@pytest.mark.parametrize("L,heads,hd", [pytest.param(L, 12, 64, id=str(L)) for L in (1, 20, 77, 130)] + [
    # head_dim 128 around the 64-row query tiles and key blocks, up to the wgmma core's 256 keys; power-of-two and
    # other head counts take the two head-decode branches of the wgmma kernel
    pytest.param(L, heads, 128, id=f"hd128-h{heads}-{L}") for L, heads in
    ((64, 8), (65, 12), (128, 16), (129, 8), (256, 12), (256, 16))])
def test_causal_attention(eng, L, heads, hd):
    nseq = 5
    g = torch.Generator().manual_seed(L * heads + hd)
    qkv = torch.randn(nseq * L, 3 * heads * hd, generator=g)
    ref = _causal_ref(qkv, nseq, L, heads)
    for mode in (0, 2):
        y = eng.debug_attention(qkv, nseq, L, heads, mode=mode, causal=True)
        assert torch.isfinite(y).all()
        assert _rel(y, ref) < 5e-6, f"mode {mode}"
    with pytest.raises(RuntimeError):           # the mma.sync kernel has no causal mask: refused, not ignored
        eng.debug_attention(qkv, nseq, L, heads, mode=1, causal=True)


@pytest.mark.parametrize("M,N,K", [(385, 768, 768), (333, 768, 3072), (1000, 768, 2304),
                                   (200, 512, 4096), (129, 1024, 4096)])     # CLIP-B fc2 width, CLIP-H fc2 (K = 4096)
def test_residual_add_epilogue(eng, M, N, K):
    g = torch.Generator().manual_seed(M + N + K)
    A, R = torch.randn(M, K, generator=g), torch.randn(M, N, generator=g)
    W, b = torch.randn(N, K, generator=g) / K ** 0.5, 0.1 * torch.randn(N, generator=g)
    ref = F.linear(A.double(), W.double(), b.double()) + R.double()
    for tc in (True, False):
        for in_place in (False, True):
            y = eng.debug_gemm(A, W, b, R=R, use_tc=tc, in_place=in_place)
            assert _rel(y, ref) < (_tc_tol(K) if tc else 5e-6), (tc, in_place)


@pytest.mark.parametrize("M,N,K", [(385, 3072, 768), (1000, 2304, 768), (129, 768, 3072),
                                   (300, 1000, 256)])                         # N not a whole number of tiles
def test_quick_gelu_epilogue(eng, M, N, K):
    g = torch.Generator().manual_seed(M * 3 + N)
    A = torch.randn(M, K, generator=g)
    W, b = torch.randn(N, K, generator=g) / K ** 0.5, 0.1 * torch.randn(N, generator=g)
    h = F.linear(A.double(), W.double(), b.double())
    ref = h * torch.sigmoid(1.702 * h)
    for tc in (True, False):
        assert _rel(eng.debug_gemm(A, W, b, act=4, use_tc=tc), ref) < (_tc_tol(K) if tc else 5e-6), tc
    assert _rel(eng.debug_gemm(A, W, b, act=4, use_tc=True, split_out=True), ref) < _tc_tol(K)   # fast split16 epilogue


def test_tower_vs_oracle_and_golden(tower):
    from mld_b200 import _lib
    e, _, sd64 = tower
    ids, g = golden_ids(), golden("clip_text.npz")
    cfg = ClipTextCfg()
    e.kernel_stats(reset=True)
    hid = e.text_encode(ids, _lib.TEXT_HIDDEN)
    pooled = e.text_encode(ids, _lib.TEXT_POOLED)
    torch.cuda.synchronize()
    st = e.kernel_stats()
    assert st["gemm_simt"] == 0 and st["attn_simt"] == 0 and st["attn_mma"] == 0, st
    assert st["gemm_tc"] == 2 * (12 * 4) + 1 and st["attn_tc"] == 2 * 12 and st["text_ln"] == 2 * (1 + 12 * 2), st
    ref_h = clip_text_forward(sd64, ids.cuda(), "clip_hidden", cfg)
    ref_p = clip_text_forward(sd64, ids.cuda(), "clip", cfg)[:, 0]
    assert _rel_rows(hid, ref_h) < 1e-4 and _rel_rows(pooled, ref_p) < 1e-4
    assert _rel_rows(hid[:, torch.from_numpy(g["hidden_pos"]).cuda()], torch.from_numpy(g["hidden"])) < 1e-4
    assert _rel_rows(pooled, torch.from_numpy(g["pooled"])) < 1e-4
    print(f"\n[text] golden ids: hidden {_rel_rows(hid, ref_h):.2e}, pooled {_rel_rows(pooled, ref_p):.2e} vs float64")


def test_tower_legacy_eos_rule(built_lib):
    from mld_b200 import _lib
    from mld_b200.engine import Engine, make_config
    e = Engine(make_config(num_layers=0, vae="none"), 0)
    tc = _lib.default_text_config()
    tc.eos_token_id = 2
    e.text_configure(tc)
    e.load_state_dict(synth.clip_text_state_dict(WEIGHT_SEED), "text_encoder.")
    e.finalize()
    ids = golden_ids()
    assert _rel_rows(e.text_encode(ids, _lib.TEXT_POOLED), torch.from_numpy(golden("clip_text.npz")["pooled_legacy"])) < 1e-4


def test_tower_512_prompts_vs_float64(tower):
    from mld_b200 import _lib
    e, _, sd64 = tower
    ids = synth.clip_text_ids(512, 77, seed=17)
    cfg = ClipTextCfg()
    hid = e.text_encode(ids, _lib.TEXT_HIDDEN)
    pooled = e.text_encode(ids, _lib.TEXT_POOLED)
    err_h = err_p = 0.0
    for c in range(0, 512, 128):
        sl = slice(c, c + 128)
        err_h = max(err_h, _rel_rows(hid[sl], clip_text_forward(sd64, ids[sl].cuda(), "clip_hidden", cfg)))
        err_p = max(err_p, _rel_rows(pooled[sl], clip_text_forward(sd64, ids[sl].cuda(), "clip", cfg)[:, 0]))
    print(f"\n[text] 512 prompts: hidden {err_h:.2e}, pooled {err_p:.2e} vs float64")
    assert err_h < 1e-4 and err_p < 1e-4


def test_savings_are_exact_and_rows_independent(tower):
    from mld_b200 import _lib
    from mld_b200.text import B200TextEncoder
    e, sd, _ = tower
    enc = B200TextEncoder.from_state_dict(sd).cuda()
    enc._engine, enc._engine_epoch = e, enc._weights_epoch            # reuse the module-scoped engine
    ids = torch.cat([torch.tensor([[49406] + [49407] * 76] * 8), synth.clip_text_ids(24, 77, seed=23)])
    plain_p = e.text_encode(ids, _lib.TEXT_POOLED).clone()
    plain_h = e.text_encode(ids, _lib.TEXT_HIDDEN).clone()
    assert _rel(enc.encode_ids(ids)[:, 0], plain_p) < 1e-6
    enc.name = "clip_hidden"
    assert _rel(enc.encode_ids(ids), plain_h) < 1e-6
    enc.name = "clip"
    for i in (0, 9, 31):                       # a row alone gives what it gives inside the batch
        assert torch.equal(e.text_encode(ids[i:i + 1], _lib.TEXT_HIDDEN)[0], plain_h[i])
        assert _rel(e.text_encode(ids[i:i + 1], _lib.TEXT_POOLED)[0], plain_p[i]) < 1e-6


class _FakeTokenizer:
    """The Hugging Face tokenizer call MldTextEncoder makes (mld_clip.py:56-62): bos, one id per word, eos, eos padding."""

    def __call__(self, texts, padding, truncation, max_length, return_tensors):
        assert padding == "max_length" and truncation and return_tensors == "pt"
        rows = []
        for t in texts:
            words = [sum(map(ord, w)) * 131 % 49000 for w in t.split()][:max_length - 2]
            r = [49406] + words + [49407]
            rows.append(r + [49407] * (max_length - len(r)))
        from types import SimpleNamespace
        return SimpleNamespace(input_ids=torch.tensor(rows, dtype=torch.long))


@pytest.mark.parametrize("hidden_state", [False, True])
def test_text_to_joints_end_to_end(tower, hidden_state):
    """B200MLD(text_encoder=B200TextEncoder) against the oracle chain (float64 CLIP -> oracle.mld_forward)."""
    from mld_b200.pipeline import B200MLD
    from mld_b200.text import B200TextEncoder
    _, sd, sd64 = tower
    tok = _FakeTokenizer()
    enc = B200TextEncoder.from_state_dict(sd, tokenizer=tok, last_hidden_state=hidden_state).cuda()
    dsd, vsd = synth.denoiser_state_dict(1234), synth.mld_vae_state_dict(4321)
    mean, std = synth.mean_std()
    model = B200MLD(dsd, vsd, mean=mean, std=std, text_encoder=enc)
    texts = ["a person walks forward and turns left", "jump", "someone waves with both hands then sits down"]
    lengths = [196, 64, 120]
    noise = synth.init_noise(3, seed=5)
    joints = model({"text": texts, "length": lengths, "init_noise": noise})
    ids = tok([""] * 3 + texts, padding="max_length", truncation=True, max_length=77, return_tensors="pt").input_ids
    ctx = clip_text_forward(sd64, ids.cuda(), "clip_hidden" if hidden_state else "clip", ClipTextCfg()).float().cpu()
    assert ctx.shape[1] == (77 if hidden_state else 1)
    jo, _, _ = O.mld_forward(dsd, O.DenoiserCfg(), vsd, O.VaeCfg(), O.DDIMScheduler(), 50, ctx, noise, lengths,
                             mean, std)
    err = max(float((a - r).abs().max() / r.abs().max()) for a, r in zip(joints, jo))
    print(f"\n[text] text -> joints, S_ctx {ctx.shape[1]}: {err:.2e} vs the oracle chain")
    assert err < 1e-3
