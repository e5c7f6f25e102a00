"""GPU tests of the native T2M evaluator (pytest -m gpu): the LeakyReLU epilogue, the movement, motion and text
encoders against the float64 restatement (with fp32 torch on the same GPU, TF32 off, reported beside it), the
renorm4t2m -> movement -> motion chain against the reference golden, per-sequence isolation and bit-identity, kernel
selection, and the drop-in modules."""
import pytest
import torch

from conftest import golden
from mld_b200 import _lib, synth
from mld_b200.engine import Engine, make_config
from oracle import t2m_eval as O
from oracle.make_golden_t2m import MOTION_LENS, MOVE_HEAD, TEXT_LENS, WEIGHT_SEED, golden_inputs

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
PREFIX = {"text_encoder": "t2m_textencoder.", "movement_encoder": "t2m_moveencoder.",
          "motion_encoder": "t2m_motionencoder."}
MOTION_GATE, TEXT_GATE = 5e-5, 2e-5


def _tc_tol(K):
    return 5e-6 * max(1.0, K / 1024)


def _rel_rows(a, b):
    """Worst per-sequence relative-to-max error (a, b: [n, ...])."""
    a, b = a.double().cpu().flatten(1), b.double().cpu().flatten(1)
    return float(((a - b).abs().max(1).values / b.abs().max(1).values).max())


@pytest.fixture(scope="module")
def sds():
    return synth.t2m_state_dicts(WEIGHT_SEED)


@pytest.fixture(scope="module")
def sd64(sds):
    return {k: {kk: vv.double().cuda() for kk, vv in v.items()} for k, v in sds.items()}


def _engine(sds, parts=7):
    eng = Engine(make_config(num_layers=0, vae="none"), 0)
    cfg = _lib.default_t2m_config()
    cfg.parts = parts
    eng.t2m_configure(cfg)
    for k, bit in (("text_encoder", 1), ("movement_encoder", 2), ("motion_encoder", 4)):
        if parts & bit:
            eng.load_state_dict(sds[k], PREFIX[k])
    eng.finalize()
    return eng


@pytest.fixture(scope="module")
def eng(built_lib, sds):
    return _engine(sds)


@pytest.fixture(scope="module")
def nets(sds):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return O.TorchNets(sds, "cuda")


@pytest.mark.parametrize("split_out", [False, True])
@pytest.mark.parametrize("use_tc", [True, False])
@pytest.mark.parametrize("M,N,K", [(37, 512, 1088), (300, 1024, 2048), (5, 96, 64)])
def test_leaky_relu_epilogue(eng, use_tc, split_out, M, N, K):
    """act = 5 through the generic (fp32 out) and the fast (split16 out) wgmma epilogues and the CUDA-core GEMM."""
    g = torch.Generator().manual_seed(M + N)
    A, W, b = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g) / K ** 0.5, torch.randn(N, generator=g)
    out = eng.debug_gemm(A.cuda(), W, b, act=5, use_tc=use_tc, split_out=split_out)
    y = A.double() @ W.double().T + b.double()
    ref = torch.where(y > 0, y, 0.2 * y)
    assert float((out.double().cpu() - ref).abs().max() / ref.abs().max()) < _tc_tol(K)


@pytest.mark.parametrize("B", [1, 3, 300])
@pytest.mark.parametrize("T", [4, 5, 40, 196, 199])
def test_movement_encoder(eng, nets, sd64, B, T):
    x = torch.randn(B, T, 263, generator=torch.Generator().manual_seed(T * 7 + B)).cuda()   # every frame non-zero
    out = eng.t2m_movement(x[..., :-4])                     # strided view: ld = 263, no copy
    ref = O.movement(sd64["movement_encoder"], x[..., :-4].double())
    assert out.shape == (B, T // 2 // 2, 512)
    err = _rel_rows(out, ref)
    fp32 = _rel_rows(nets.movement(x[..., :-4].contiguous()), ref)
    print(f"movement B={B} T={T}: {err:.2e} (fp32 torch {fp32:.2e})")
    assert err < 2e-5
    assert torch.equal(out, eng.t2m_movement(x[..., :-4].contiguous()))


def _ragged(B, L, seed):
    g = torch.Generator().manual_seed(seed)
    ln = torch.randint(1, L + 1, (B,), generator=g)
    ln[0], ln[-1] = L, 1
    return ln


@pytest.mark.parametrize("order", ["sorted", "unsorted"])
@pytest.mark.parametrize("B", [1, 5, 300])
def test_motion_encoder(eng, nets, sd64, B, order):
    L = 49
    x = (torch.randn(B, L, 512, generator=torch.Generator().manual_seed(B)) * 0.5).cuda()
    ln = torch.tensor([L]) if B == 1 else _ragged(B, L, B)
    if order == "sorted":
        ln = ln.sort(descending=True).values
    out = eng.t2m_motion(x, ln)
    ref = O.motion(sd64["motion_encoder"], x.double(), ln.tolist())
    err, fp32 = _rel_rows(out, ref), _rel_rows(nets.motion(x, ln), ref)
    print(f"motion B={B} {order}: {err:.2e} (fp32 torch {fp32:.2e})")
    assert err < MOTION_GATE


@pytest.mark.parametrize("order", ["sorted", "unsorted"])
@pytest.mark.parametrize("L", [1, 3, 22])
def test_text_encoder(eng, nets, sd64, L, order):
    B = 37
    w, p = synth.t2m_text_inputs(B, L, seed=L)
    w, p = w.cuda(), p.cuda()
    ln = _ragged(B, L, L + 1) if L > 1 else torch.ones(B, dtype=torch.int64)
    if order == "sorted":
        ln = ln.sort(descending=True).values
    out = eng.t2m_text(w, p, ln)
    ref = O.text(sd64["text_encoder"], w.double(), p.double(), ln.tolist())
    err, fp32 = _rel_rows(out, ref), _rel_rows(nets.text(w, p, ln), ref)
    print(f"text L={L} {order}: {err:.2e} (fp32 torch {fp32:.2e})")
    assert err < TEXT_GATE


def test_chain_matches_oracle_and_reference_golden(eng, sd64):
    g = golden("t2m_eval.npz")
    word, pos, motions = golden_inputs()
    mov = eng.t2m_movement(motions.cuda()[..., :-4])
    emb = eng.t2m_motion(mov, torch.tensor(MOTION_LENS) // 4)
    mov64 = O.movement(sd64["movement_encoder"], motions.cuda().double()[..., :-4])
    emb64 = O.motion(sd64["motion_encoder"], mov64, [n // 4 for n in MOTION_LENS])
    assert _rel_rows(mov, mov64) < 2e-5 and _rel_rows(emb, emb64) < MOTION_GATE
    assert _rel_rows(mov[:, :MOVE_HEAD], torch.from_numpy(g["movement_head"])) < 2e-5
    assert _rel_rows(emb, torch.from_numpy(g["motion_emb"])) < MOTION_GATE
    text = eng.t2m_text(word.cuda(), pos.cuda(), torch.tensor(TEXT_LENS))
    assert _rel_rows(text, torch.from_numpy(g["text_emb"])) < TEXT_GATE


# ---------------------------------------------------------------------------------------------- isolation
POISONS = [float("nan"), float("inf"), 1e5]


@pytest.mark.parametrize("victim", [0, 3, 6])
@pytest.mark.parametrize("value", POISONS)
def test_poisoned_member_does_not_reach_others(eng, victim, value):
    B, T = 7, 196
    x = torch.randn(B, T, 259, generator=torch.Generator().manual_seed(1)).cuda()
    ln = torch.tensor([49, 30, 1, 49, 12, 7, 40])
    w, p = synth.t2m_text_inputs(B, 22, seed=3)
    w, p = w.cuda(), p.cuda()
    tl = torch.tensor([22, 5, 1, 13, 22, 9, 2])
    clean_mov = eng.t2m_movement(x)
    clean = (eng.t2m_motion(clean_mov, ln), eng.t2m_text(w, p, tl))
    xp, wp = x.clone(), w.clone()
    xp[victim, 17, 5] = value
    wp[victim, 0, 9] = value
    mov = eng.t2m_movement(xp)
    got = (eng.t2m_motion(mov, ln), eng.t2m_text(wp, p, tl))
    keep = [b for b in range(B) if b != victim]
    assert torch.equal(mov[keep], clean_mov[keep])
    for a, c in zip(got, clean):
        assert torch.equal(a[keep], c[keep])


@pytest.mark.parametrize("value", POISONS)
def test_gru_inputs_past_length_are_never_read(eng, value):
    B, L = 6, 49
    x = torch.randn(B, L, 512, generator=torch.Generator().manual_seed(2)).cuda()
    ln = torch.tensor([49, 1, 30, 2, 48, 17])
    w, p = synth.t2m_text_inputs(B, 22, seed=4)
    w, p = w.cuda(), p.cuda()
    tl = torch.tensor([22, 1, 3, 21, 10, 5])
    clean = (eng.t2m_motion(x, ln), eng.t2m_text(w, p, tl))
    xp, wp, pp = x.clone(), w.clone(), p.clone()
    for b in range(B):
        xp[b, int(ln[b]):] = value
        wp[b, int(tl[b]):] = value
        pp[b, int(tl[b]):] = value
    assert torch.equal(eng.t2m_motion(xp, ln), clean[0])
    assert torch.equal(eng.t2m_text(wp, pp, tl), clean[1])


def test_bit_identity_across_batch_position_and_chunk(sds, eng):
    B, L = 300, 49
    x = torch.randn(B, L, 512, generator=torch.Generator().manual_seed(5)).cuda()
    ln = _ragged(B, L, 6)
    w, p = synth.t2m_text_inputs(B, 22, seed=7)
    w, p = w.cuda(), p.cuda()
    tl = _ragged(B, 22, 8)
    f = torch.randn(B, 60, 259, generator=torch.Generator().manual_seed(9)).cuda()
    full = (eng.t2m_motion(x, ln), eng.t2m_text(w, p, tl), eng.t2m_movement(f))
    again = (eng.t2m_motion(x, ln), eng.t2m_text(w, p, tl), eng.t2m_movement(f))
    for a, b in zip(full, again):
        assert torch.equal(a, b)                                        # repeated runs
    for i in (0, 131, 299):                                              # alone
        assert torch.equal(eng.t2m_motion(x[i:i + 1], ln[i:i + 1])[0], full[0][i])
        assert torch.equal(eng.t2m_text(w[i:i + 1], p[i:i + 1], tl[i:i + 1])[0], full[1][i])
        assert torch.equal(eng.t2m_movement(f[i:i + 1])[0], full[2][i])
    perm = torch.randperm(B, generator=torch.Generator().manual_seed(10))   # other positions, other tiles
    assert torch.equal(eng.t2m_motion(x[perm], ln[perm]), full[0][perm])
    assert torch.equal(eng.t2m_text(w[perm], p[perm], tl[perm]), full[1][perm])
    assert torch.equal(eng.t2m_movement(f[perm]), full[2][perm])
    for chunk in (1, 7, 128):                                            # batch chunks
        eng.set_option("t2m_chunk", str(chunk))
        try:
            got = (eng.t2m_motion(x, ln), eng.t2m_text(w, p, tl), eng.t2m_movement(f))
        finally:
            eng.set_option("t2m_chunk", "0")
        for a, b in zip(got, full):
            assert torch.equal(a, b)


# ---------------------------------------------------------------------------------------------- kernel choice
def test_kernel_stats_and_cuda_core_path(sds, sd64):
    e = _engine(sds)
    x = torch.randn(9, 196, 259, generator=torch.Generator().manual_seed(11)).cuda()
    ln = _ragged(9, 49, 12)
    w, p = synth.t2m_text_inputs(9, 22, seed=13)
    w, p = w.cuda(), p.cuda()
    tl = _ragged(9, 22, 14)

    def run():
        mov = e.t2m_movement(x)
        return mov, e.t2m_motion(mov, ln), e.t2m_text(w, p, tl)

    e.kernel_stats(reset=True)
    tc = run()
    st = e.kernel_stats()
    assert st["gru_tc"] == 49 + 22 and st["gemm_simt"] == 0 and st["gemm_tc"] > 0, st
    e.set_option("gemm", "simt")
    e.kernel_stats(reset=True)
    simt = run()
    st = e.kernel_stats()
    assert st["gru_tc"] == 0 and st["gemm_tc"] == 0 and st["gemm_simt"] > 0, st
    mov64 = O.movement(sd64["movement_encoder"], x.double())
    assert _rel_rows(simt[0], mov64) < 2e-5
    assert _rel_rows(simt[1], O.motion(sd64["motion_encoder"], simt[0].double(), ln.tolist())) < MOTION_GATE
    assert _rel_rows(simt[2], O.text(sd64["text_encoder"], w.double(), p.double(), tl.tolist())) < TEXT_GATE
    assert _rel_rows(simt[1], tc[1]) < 2 * MOTION_GATE


def test_missing_part_and_bad_shapes_are_refused(sds):
    e = _engine(sds, parts=_lib.T2M_MOVEMENT)
    with pytest.raises(RuntimeError, match="not configured"):
        e.t2m_motion(torch.zeros(2, 5, 512).cuda(), [5, 1])
    with pytest.raises(ValueError):
        e.t2m_movement(torch.zeros(2, 3, 259).cuda())                  # T < 4
    eng = _engine(sds)
    with pytest.raises(ValueError):
        eng.t2m_motion(torch.zeros(2, 5, 512).cuda(), [6, 1])          # length > L
    with pytest.raises(ValueError):
        eng.t2m_text(torch.zeros(2, 5, 300).cuda(), torch.zeros(2, 5, 14).cuda(), [5, 1])


# ---------------------------------------------------------------------------------------------- drop-in modules
def test_drop_in_modules(sds, eng):
    from mld_b200.evaluator import B200MotionEncoderBiGRUCo, B200MovementConvEncoder, B200TextEncoderBiGRUCo
    te = B200TextEncoderBiGRUCo(word_size=300, pos_size=15, hidden_size=512, output_size=512)
    mv = B200MovementConvEncoder(input_size=259, hidden_size=512, output_size=512)
    mo = B200MotionEncoderBiGRUCo(input_size=512, hidden_size=1024, output_size=512)
    te.load_state_dict(sds["text_encoder"], strict=True)
    mv.load_state_dict(sds["movement_encoder"], strict=True)
    mo.load_state_dict(sds["motion_encoder"], strict=True)
    te, mv, mo = te.cuda().eval(), mv.cuda().eval(), mo.cuda().eval()
    word, pos, motions = golden_inputs()
    feats = motions.cuda()
    m_lens = torch.tensor(MOTION_LENS, device="cuda") // 4
    mov = mv(feats[..., :-4])
    emb = mo(mov, m_lens)
    text = te(word.cuda(), pos.cuda(), torch.tensor(TEXT_LENS, device="cuda"))
    assert mov.shape == (4, 49, 512) and emb.shape == (4, 512) and text.shape == (4, 512)
    assert torch.equal(mov, eng.t2m_movement(feats[..., :-4]))
    assert torch.equal(emb, eng.t2m_motion(mov, m_lens))
    assert torch.equal(text, eng.t2m_text(word.cuda(), pos.cuda(), torch.tensor(TEXT_LENS)))
    with pytest.raises(RuntimeError, match="decreasing"):
        mo(mov, m_lens.flip(0))
