"""GPU tests (pytest -m gpu) of the GEMM's row-mapped epilogues, of every k_gemm_tc instantiation, of the CUDA-core
LayerNorm kernels and of the token placement (rows_to_split), through the C ABI's debug hooks.

The float64 references are written here as plain index operations of the documented maps:
  GEMM:          row r -> (r / in_group) * out_group + out_off + r % in_group, columns [out_col0, out_col0 + N),
                 y = act(A W^T + b + tab[out_off + r % in_group]), 0 when r % in_group >= zero_lengths[r / in_group]
  LayerNorm:     input row of r = (r / sel_group) * in_group + r % sel_group; rowvec row = input row / rv_group
  rows_to_split: the GEMM's row map, relu?(src[r or r % in_group]) + tab[out_off + r % in_group]
Output buffers start filled with a sentinel that survives the split16 round trip (-777.5 has 11 significant bits),
so every cell an op must leave alone is checked bit for bit."""
import re

import pytest
import torch
import torch.nn.functional as F
from torch.profiler import ProfilerActivity, profile

import kernel_matrix as KM

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

SENTINEL = -777.5
CC_TOL = 5e-6                     # CUDA cores, relative to the largest element
ACTS = {0: lambda x: x, 1: F.gelu, 2: F.relu, 3: F.silu, 4: lambda x: x * torch.sigmoid(1.702 * x),
        5: lambda x: torch.where(x > 0, x, 0.2 * x)}


@pytest.fixture(scope="module")
def eng(built_lib):
    from mld_b200.engine import Engine, make_config
    return Engine(make_config(num_layers=0, vae="none"), 0)


@pytest.fixture(scope="module")
def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _tc_tol(K):
    return 5e-6 * max(1.0, K / 1024)


def _rel(a, ref):
    a, ref = a.double(), ref.double()
    return float((a - ref).abs().max() / ref.abs().max())


def _kernels(fn):
    """The device kernels fn launched, in order.  Now and then the profiler records no device activity at all for a
    run; such a run is repeated (every fn here writes the same bits when it runs again)."""
    for _ in range(3):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        if names:
            break
    return names


def _bits(t):
    return t.contiguous().view(torch.int32)


def _sentinel(rows, cols):
    return torch.full((rows, cols), SENTINEL, dtype=torch.float32, device="cuda")


def _data(M, N, K, seed, tab_rows=0):
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(M, K, generator=g)
    W = torch.randn(N, K, generator=g) / K ** 0.5
    b = 0.1 * torch.randn(N, generator=g)
    tab = 0.5 * torch.randn(tab_rows, N, generator=g) if tab_rows else None
    return A.cuda(), W, b, tab


def _map(M, in_group, out_group, out_off):
    r = torch.arange(M, device="cuda")
    seq, pos = r // in_group, r % in_group
    return seq * out_group + out_off + pos, seq, pos


def _gemm_ref(A, W, b, act, pos, tab=None, out_off=0, zero=None, a_relu=False):
    x = A.double()
    if a_relu:
        x = x.clamp_min(0)
    y = x @ W.double().cuda().T + b.double().cuda()
    if tab is not None:
        y = y + tab.double().cuda()[out_off + pos]
    y = ACTS[act](y)
    if zero is not None:
        y[zero] = 0.0
    return y


def _check_placement(out, init, orow, col0, ref, zero, tol, what):
    """1. mapped cells match float64; 2. every other cell keeps its bits; 3. zeroed rows are +0.0 bit for bit."""
    N = ref.shape[1]
    cols = torch.arange(col0, col0 + N, device="cuda")
    mapped = torch.zeros(out.shape, dtype=torch.bool, device="cuda")
    mapped[orow[:, None], cols[None, :]] = True
    got = out[orow][:, col0:col0 + N]
    keep = torch.ones(orow.numel(), dtype=torch.bool, device="cuda") if zero is None else ~zero
    if keep.any():
        assert torch.isfinite(got[keep]).all(), what
        assert _rel(got[keep], ref[keep]) < tol, what
    assert torch.equal(_bits(out[~mapped]), _bits(init[~mapped])), f"{what}: a cell outside the map changed"
    if zero is not None and zero.any():
        assert (_bits(got[zero]) == 0).all(), f"{what}: a zeroed row is not +0.0"
    return got


# ----------------------------------------------------------------------------- every k_gemm_tc instantiation
def _matrix_case(eng, key, kw, K, K1):
    M, N = 333, kw["N"]
    A, W, b, _ = _data(M, N, K, seed=K * 1000 + N * 10 + key[1] * 3 + key[2])
    g = torch.Generator().manual_seed(N + K)
    args = dict(act=kw.get("act", 0), K1=K1, use_tc=True)
    ref = _gemm_ref(A, W, b, args["act"], None)
    if kw.get("layer_norm") or kw.get("residual"):
        R = torch.randn(M, N, generator=g).cuda()
        ref = ref + R.double()
        args["R"] = R
    if kw.get("layer_norm"):
        gamma, beta = 1 + 0.1 * torch.randn(N, generator=g), 0.1 * torch.randn(N, generator=g)
        ref = F.layer_norm(ref, (N,), gamma.double().cuda(), beta.double().cuda(), 1e-5)
        args.update(gamma=gamma, beta=beta)
    out_cols = kw.get("out_cols", N)
    out = _sentinel(M, out_cols)
    init = out.clone()
    names = _kernels(lambda: eng.debug_gemm_rows(A, W, b, out=out, split_out=kw.get("split_out", False),
                                                 vec_f32=kw.get("vec_f32", False), **args))
    return names, out, init, ref


@pytest.mark.parametrize("K", KM.GEMM_KS)
@pytest.mark.parametrize("key,kw", KM.GEMM_TC, ids=[KM.gemm_tc_name(k) for k, _ in KM.GEMM_TC])
def test_every_gemm_tc_instantiation(eng, key, kw, K):
    """Each row of the matrix launches exactly its instantiation (from one A source and from two) and matches
    float64."""
    for K1 in (0, 64 * (K // 128)) if K > 64 else (0,):
        names, out, init, ref = _matrix_case(eng, key, kw, K, K1)
        launched = [m.group(0) for n in names for m in [re.search(r"k_gemm_tc<\d+, \d+, \d+>", n)] if m]
        assert launched == [KM.gemm_tc_name(key)], (K1, names)
        assert not any("k_proj_tc" in n or "k_gemm_simt" in n for n in names), names
        N = ref.shape[1]
        assert torch.isfinite(out[:, :N]).all()
        assert _rel(out[:, :N], ref) < _tc_tol(K), (K1, _rel(out[:, :N], ref))
        assert torch.equal(_bits(out[:, N:]), _bits(init[:, N:]))


# ----------------------------------------------------------------------------- row maps on both GEMM paths
# (in_group, out_group, out_off) as the call sites use them
MAPS = [
    (1, 1, 0),          # the time MLP (engine.cu): one row per sequence
    (24, 24, 0),        # the ST-GCN's per-joint table
    (77, 79, 2),        # CLIP tokens after the latent and time tokens (denoiser.cu)
    (128, 128, 0),      # sequences on m-tile boundaries
    (129, 129, 0),      # sequences straddling m-tiles
    (196, 198, 2),      # VAE encoder frames after the two distribution tokens (vae.cu)
    (196, 196, 0),      # no-VAE pose embedding / padded frames zeroed (denoiser.cu, vae.cu)
]
OUTS = {
    # split16 planes at column 16 of a wider buffer; fp32 at column N of a [rows, 2N] buffer (op_gru's gate layout)
    "split": dict(N=263, out_col0=16, out_cols=288, split_out=True),
    "f32": dict(N=192, out_col0=192, out_cols=384, split_out=False),
}
K_MAP = 320


def _nseq(size, in_group, N, sm_count):
    if size == "one":
        return 1
    if size == "few":
        return 3
    n_tiles = -(-N // (256 if N % 256 == 0 else 128))
    rows = 128 * (sm_count // n_tiles + 2)          # more tiles than SMs: some CTAs take a second tile
    return -(-rows // in_group)


def _zero_lengths(nseq, in_group):
    return [(0, 1, in_group - 1, in_group)[s % 4] for s in range(nseq)]


def _run_map(eng, A, W, b, o, init, use_tc, **kw):
    out = init.clone()
    eng.kernel_stats(reset=True)
    eng.debug_gemm_rows(A, W, b, out=out, out_col0=o["out_col0"], split_out=o["split_out"], use_tc=use_tc,
                        K1=0, **kw)
    st = eng.kernel_stats(reset=True)
    assert (st["gemm_tc"], st["gemm_simt"]) == ((1, 0) if use_tc else (0, 1)), st
    return out


@pytest.mark.parametrize("size", ["one", "few", "many"])
@pytest.mark.parametrize("outk", sorted(OUTS))
@pytest.mark.parametrize("zeroing", [False, True])
@pytest.mark.parametrize("with_tab", [False, True])
@pytest.mark.parametrize("in_group,out_group,out_off", MAPS)
def test_gemm_row_map(eng, sm_count, in_group, out_group, out_off, with_tab, zeroing, outk, size):
    o = OUTS[outk]
    N = o["N"]
    nseq = _nseq(size, in_group, N, sm_count)
    M = nseq * in_group
    orow, seq, pos = _map(M, in_group, out_group, out_off)
    out_rows = int(orow.max()) + 3
    A, W, b, tab = _data(M, N, K_MAP, seed=in_group * 31 + M, tab_rows=(out_off + in_group) if with_tab else 0)
    kw = dict(in_group=in_group, out_group=out_group, out_off=out_off, addtab=tab, act=0)
    zero = None
    if zeroing:
        zl = _zero_lengths(nseq, in_group)
        kw["zero_lengths"] = zl
        zero = pos >= torch.tensor(zl, device="cuda")[seq]
        A[zero, 0] = float("nan")                          # a zeroed row is +0.0 whatever its A row holds
        A[zero, 1] = float("inf")
    ref = _gemm_ref(A, W, b, 0, pos, tab, out_off, zero)
    init = _sentinel(out_rows, o["out_cols"])
    what = f"M={M}"
    tc = _run_map(eng, A, W, b, o, init, True, **kw)
    got_tc = _check_placement(tc, init, orow, o["out_col0"], ref, zero, _tc_tol(K_MAP), f"wgmma {what}")
    cc = _run_map(eng, A, W, b, o, init, False, **kw)
    got_cc = _check_placement(cc, init, orow, o["out_col0"], ref, zero, CC_TOL, f"CUDA cores {what}")
    keep = torch.ones(M, dtype=torch.bool, device="cuda") if zero is None else ~zero
    if keep.any():
        assert _rel(got_tc[keep], got_cc[keep].double()) < CC_TOL, "the wgmma and CUDA-core paths disagree"
    if not with_tab and not zeroing:
        # 4. the map only moves rows: each mapped row has the bits of the identity-mapped run's row
        for use_tc, got in ((True, got_tc), (False, got_cc)):
            ident = _sentinel(M, o["out_cols"])
            eng.debug_gemm_rows(A, W, b, out=ident, out_col0=o["out_col0"], split_out=o["split_out"], use_tc=use_tc)
            assert torch.equal(_bits(got), _bits(ident[:, o["out_col0"]:o["out_col0"] + N])), use_tc


@pytest.mark.parametrize("act", sorted(ACTS))
@pytest.mark.parametrize("outk", sorted(OUTS))
def test_gemm_row_map_activations(eng, sm_count, act, outk):
    """Every runtime activation through the generic epilogue with the table (the ST-GCN's ReLU + per-joint table)
    and zeroed rows."""
    o = OUTS[outk]
    N, in_group = o["N"], 24
    nseq = _nseq("many", in_group, N, sm_count)
    M = nseq * in_group
    orow, seq, pos = _map(M, in_group, in_group, 0)
    A, W, b, tab = _data(M, N, K_MAP, seed=act + 7, tab_rows=in_group)
    zl = _zero_lengths(nseq, in_group)
    zero = pos >= torch.tensor(zl, device="cuda")[seq]
    kw = dict(in_group=in_group, out_group=in_group, out_off=0, addtab=tab, zero_lengths=zl, act=act)
    ref = _gemm_ref(A, W, b, act, pos, tab, 0, zero)
    init = _sentinel(M + 1, o["out_cols"])
    names = _kernels(lambda: _run_map(eng, A, W, b, o, init, True, **kw))
    assert sum("k_gemm_tc<128, 2, 0>" in n for n in names) == 1, names
    tc = _run_map(eng, A, W, b, o, init, True, **kw)
    got_tc = _check_placement(tc, init, orow, o["out_col0"], ref, zero, _tc_tol(K_MAP), f"wgmma act {act}")
    cc = _run_map(eng, A, W, b, o, init, False, **kw)
    got_cc = _check_placement(cc, init, orow, o["out_col0"], ref, zero, CC_TOL, f"CUDA cores act {act}")
    assert _rel(got_tc[~zero], got_cc[~zero].double()) < CC_TOL


@pytest.mark.parametrize("with_tab", [False, True])
@pytest.mark.parametrize("M", [77, 300])
def test_gemm_one_sequence_at_an_offset(eng, M, with_tab):
    """in_group >= M with out_group == 0: both paths place the rows at out_off + r (the CUDA-core kernel used to
    write them at r while reading the table at out_off + r)."""
    o = OUTS["split"]
    N, out_off = o["N"], 3
    orow, _, pos = _map(M, M, 0, out_off)
    A, W, b, tab = _data(M, N, K_MAP, seed=M + with_tab, tab_rows=(out_off + M) if with_tab else 0)
    ref = _gemm_ref(A, W, b, 0, pos, tab, out_off)
    init = _sentinel(M + out_off + 2, o["out_cols"])
    for use_tc, tol in ((True, _tc_tol(K_MAP)), (False, CC_TOL)):
        out = _run_map(eng, A, W, b, o, init, use_tc, in_group=M, out_group=0, out_off=out_off, addtab=tab)
        _check_placement(out, init, orow, o["out_col0"], ref, None, tol, f"use_tc={use_tc}")


@pytest.mark.parametrize("a_kind", [1, 2])
def test_gemm_fp32_a_on_the_cuda_cores(eng, a_kind):
    """An fp32 A (the motion features, the CLIP context), through ReLU for a_kind 2, with a row map and table."""
    in_group, out_group, out_off, nseq, N, K = 77, 79, 2, 5, 256, 263
    M = nseq * in_group
    orow, seq, pos = _map(M, in_group, out_group, out_off)
    A, W, b, tab = _data(M, N, K, seed=a_kind, tab_rows=out_off + in_group)
    ref = _gemm_ref(A, W, b, 0, pos, tab, out_off, a_relu=a_kind == 2)
    init = _sentinel(nseq * out_group + 1, N)
    for split_out in (False, True):
        out = init.clone()
        eng.debug_gemm_rows(A, W, b, out=out, split_out=split_out, use_tc=False, a_kind=a_kind, in_group=in_group,
                            out_group=out_group, out_off=out_off, addtab=tab)
        _check_placement(out, init, orow, 0, ref, None, CC_TOL, f"split_out={split_out}")
    with pytest.raises(RuntimeError, match="status 4"):
        eng.debug_gemm_rows(A, W, b, out=init.clone(), use_tc=True, a_kind=a_kind)


def test_gemm_rows_refuses_maps_outside_the_buffer(eng):
    A, W, b, tab = _data(100, 64, 64, seed=3, tab_rows=10)
    for kw in (dict(out=_sentinel(99, 64)),                                        # identity: 100 rows
               dict(out=_sentinel(110, 64), in_group=50, out_group=60, out_off=1),  # last row 60 + 1 + 49
               dict(out=_sentinel(100, 64), out_col0=1),
               dict(out=_sentinel(200, 64), in_group=10, out_group=10, addtab=tab, out_off=1)):
        with pytest.raises(RuntimeError, match="status 1"):
            eng.debug_gemm_rows(A, W, b, use_tc=False, **kw)


# ----------------------------------------------------------------------------- LayerNorm (simt_ln)
def _ln_ref(d, M, c=None, res=None, rowvec=None, rv_group=1, gamma=None, beta=None, irow=None, act=0):
    x = 0
    if c is not None:
        x = x + c[:, :d].double()[irow]
    if res is not None:
        x = x + res.double()[irow]
    if rowvec is not None:
        x = x + rowvec.double().cuda()[irow // rv_group]
    y = F.layer_norm(x, (d,), gamma.double().cuda(), beta.double().cuda(), 1e-5)
    return ACTS[act](y)


def _ln_inputs(d, M_in, seed, rv_rows=0):
    g = torch.Generator().manual_seed(seed)
    c = (torch.randn(M_in, d, generator=g) * 2 + 0.5).cuda()
    res = torch.randn(M_in, d, generator=g).cuda()
    rowvec = torch.randn(rv_rows, d, generator=g) if rv_rows else None
    gamma, beta = 1 + 0.1 * torch.randn(d, generator=g), 0.1 * torch.randn(d, generator=g)
    return c, res, rowvec, gamma, beta


def _ln_run(eng, kernel, init, **kw):
    out = init.clone()
    names = _kernels(lambda: eng.debug_ln(out=out, **kw))
    launched = [m.group(0) for n in names for m in [re.search(r"k_ln(_vec)?<\d+>", n)] if m]
    assert launched == [kernel], names
    return out


@pytest.mark.parametrize("act", [0, 5])
@pytest.mark.parametrize("inputs", ["c", "res", "c+res", "rowvec1", "rowvec79", "rowvec198"])
@pytest.mark.parametrize("d,aligned,kernel", KM.LN_CASES)
def test_layer_norm_inputs(eng, d, aligned, kernel, inputs, act):
    M = 2 * 198 + 37
    rv_group = int(inputs[6:]) if inputs.startswith("rowvec") else 1
    c, res, rowvec, gamma, beta = _ln_inputs(d, M, seed=d + len(inputs) + act, rv_rows=-(-M // rv_group))
    kw = dict(gamma=gamma, beta=beta, act=act)
    if "c" in inputs.split("+"):
        kw["c"] = c
    if "res" in inputs or inputs.startswith("rowvec"):
        kw["res"] = res
    if inputs.startswith("rowvec"):
        kw.update(rowvec=rowvec, rv_group=rv_group)
    kw["M_in"] = M
    ld_out = d if aligned else d + 1
    for split_out in (False, True):
        init = _sentinel(M, ld_out)
        out = _ln_run(eng, kernel, init, split_out=split_out, **kw)
        ref = _ln_ref(d, M, irow=torch.arange(M, device="cuda"), **{k: v for k, v in kw.items() if k != "M_in"})
        assert torch.isfinite(out[:, :d]).all()
        assert _rel(out[:, :d], ref) < CC_TOL, (split_out, _rel(out[:, :d], ref))
        assert torch.equal(_bits(out[:, d:]), _bits(init[:, d:]))


@pytest.mark.parametrize("split_out", [False, True])
@pytest.mark.parametrize("act", [0, 5])
@pytest.mark.parametrize("sel_group,in_group", [(1, 79), (2, 198), (2, 62)])
@pytest.mark.parametrize("d,aligned,kernel", KM.LN_CASES)
def test_layer_norm_row_gather(eng, d, aligned, kernel, sel_group, in_group, act, split_out):
    """The kept tokens of each sequence (the denoiser's latent tokens, the VAE encoder's distribution tokens), with a
    per-sequence row vector; the rows the gather skips hold NaN and change nothing."""
    nseq = 5
    M_in, M = nseq * in_group, nseq * sel_group
    c, res, rowvec, gamma, beta = _ln_inputs(d, M_in, seed=d * 7 + in_group + act, rv_rows=nseq)
    r = torch.arange(M, device="cuda")
    irow = (r // sel_group) * in_group + r % sel_group
    skipped = torch.ones(M_in, dtype=torch.bool, device="cuda")
    skipped[irow] = False
    ld_out = d if aligned else d + 1
    init = _sentinel(M, ld_out)
    kw = dict(gamma=gamma, beta=beta, act=act, rowvec=rowvec, rv_group=in_group, sel_group=sel_group,
              in_group=in_group, split_out=split_out)
    c0, r0 = c.clone(), res.clone()
    c0[skipped], r0[skipped] = 0.0, 0.0
    clean = _ln_run(eng, kernel, init, c=c0, res=r0, **kw)
    c[skipped], res[skipped] = float("nan"), float("nan")
    out = _ln_run(eng, kernel, init, c=c, res=res, **kw)
    ref = _ln_ref(d, M, c=c0, res=r0, rowvec=rowvec, rv_group=in_group, gamma=gamma, beta=beta, irow=irow, act=act)
    assert torch.isfinite(out[:, :d]).all()
    assert _rel(out[:, :d], ref) < CC_TOL
    assert torch.equal(_bits(out), _bits(clean))
    assert torch.equal(_bits(out[:, d:]), _bits(init[:, d:]))


def test_layer_norm_refuses_rows_wider_than_its_kernels(eng):
    d = 1025
    c, _, _, gamma, beta = _ln_inputs(d, 8, seed=1)
    with pytest.raises(RuntimeError, match="status 4"):
        eng.debug_ln(gamma, beta, out=_sentinel(8, d), c=c)


# ----------------------------------------------------------------------------- rows_to_split
R2S_MAPS = [
    # (in_group, out_group, out_off, src, tab)
    (77, 79, 2, True, True),          # condition tokens with the query PE (text_dim == latent_dim)
    (77, 78, 1, True, True),          # the decoder's memory tokens after the time token, with their PE
    (196, 196, 0, False, True),       # the VAE decoder's queries: the PE table alone
    (1 << 30, 0, 0, True, False),     # the CLIP context as it is
    (24, 26, 2, True, False),
]


@pytest.mark.parametrize("src_bcast", [False, True])
@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("in_group,out_group,out_off,with_src,with_tab", R2S_MAPS)
def test_rows_to_split(eng, in_group, out_group, out_off, with_src, with_tab, relu, src_bcast):
    d, nseq = 256, 3
    g_eff = min(in_group, 200)
    M = nseq * g_eff if in_group < (1 << 30) else 200
    if src_bcast and (not with_src or in_group >= M):
        pytest.skip("src_bcast broadcasts one sequence of a source")
    orow, seq, pos = _map(M, in_group, out_group, out_off)
    g = torch.Generator().manual_seed(in_group + out_off + 2 * relu + src_bcast)
    src = torch.randn(in_group if src_bcast else M, d, generator=g).cuda() if with_src else None
    tab = torch.randn(out_off + min(in_group, M), d, generator=g) if with_tab else None
    x = torch.zeros(M, d, dtype=torch.float64, device="cuda")
    if src is not None:
        x = src.double()[pos if src_bcast else torch.arange(M, device="cuda")]
    if relu:
        x = x.clamp_min(0)
    if tab is not None:
        x = x + tab.double().cuda()[out_off + pos]
    init = _sentinel(int(orow.max()) + 3, d + 8)
    outs = []
    for kernel, kw in KM.ROWS_TO_SPLIT:
        out = init.clone()
        names = _kernels(lambda: eng.debug_rows_to_split(src, M, d, out=out, in_group=in_group, out_group=out_group,
                                                         out_off=out_off, src_bcast=src_bcast, tab=tab, relu=relu,
                                                         **kw))
        launched = [m.group(1) for n in names for m in [re.search(r"\b(k_rows_to_split8?)\(", n)] if m]
        # the hook fills the split16 buffer from out with the scalar kernel first
        assert launched[1:] == [kernel], names
        _check_placement(out, init, orow, 0, x, None, CC_TOL, kernel)
        outs.append(out)
    assert torch.equal(_bits(outs[0]), _bits(outs[1])), "the two kernels disagree"
