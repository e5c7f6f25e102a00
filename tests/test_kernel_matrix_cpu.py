"""CPU: tests/kernel_matrix.py lists exactly the kernels the sources instantiate and launch - every k_gemm_tc
instantiation tc_create opts in (and tc_gemm launches), every LayerNorm kernel simt_ln launches and both
rows_to_split kernels - so that a new kernel without a GPU test row fails here."""
import os
import re

from conftest import ROOT
import kernel_matrix as KM

CSRC = os.path.join(ROOT, "mld_b200", "csrc")


def _src(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _body(text, signature):
    """The brace-balanced body of the function whose definition starts with `signature`."""
    i = text.index(signature)
    i = text.index("{", i)
    depth = 0
    for j in range(i, len(text)):
        depth += {"{": 1, "}": -1}.get(text[j], 0)
        if depth == 0:
            return text[i:j + 1]
    raise AssertionError(f"unbalanced body of {signature}")


def _enum(text, pattern):
    body = re.search(pattern, text, re.S).group(1)
    return {k: int(v) for k, v in re.findall(r"(\w+)\s*=\s*(\d+)", body)}


def test_enums_match_the_sources():
    assert _enum(_src("gemm_tc.cu"), r"enum\s*\{([^}]*EPI_FAST[^}]*)\}") == KM.EPI
    assert _enum(_src("common.cuh"), r"enum ActKind\s*\{([^}]*)\}") == KM.ACT


def _key(bn, epi, act):
    return int(bn), KM.EPI[epi], KM.ACT[act or "ACT_NONE"]


def test_gemm_tc_table_is_every_instantiation():
    src = _src("gemm_tc.cu")
    opted = [_key(*m) for m in re.findall(r"opt_in\(k_gemm_tc<(\d+),\s*(EPI_\w+)(?:,\s*(ACT_\w+))?>", src)]
    assert len(opted) == len(set(opted)) == 17, opted
    table = [key for key, _ in KM.GEMM_TC]
    assert len(table) == len(set(table)), "a kernel listed twice"
    assert set(table) == set(opted)
    # every launch in tc_gemm is of an opted-in instantiation, and every instantiation is launched
    launch = _body(src, "bool tc_gemm(TcCtx* c")
    launched = {_key(bn, e, a) for bn, e, a in re.findall(r"MLDB_LAUNCH\((\d+),\s*(EPI_\w+)(?:,\s*(ACT_\w+))?\)", launch)}
    for e, a in re.findall(r"MLDB_LAUNCH_SHAPE\((EPI_\w+)(?:,\s*(ACT_\w+))?\)", launch):
        launched |= {_key(256, e, a), _key(128, e, a)}
    assert launched == set(opted)


def test_gemm_tc_rows_follow_the_selection():
    """The structural rules of tc_gemm's choice that each row relies on."""
    for (bn, epi, act), kw in KM.GEMM_TC:
        assert bn == (256 if kw["N"] % 256 == 0 else 128), (bn, epi, act)
        assert kw.get("act", 0) == act or epi in (KM.GENERIC,), (bn, epi, act)
        if epi == KM.FAST:
            assert kw["N"] % bn == 0 and kw.get("split_out") and act in (KM.NONE, KM.GELU, KM.QUICKGELU, KM.LEAKY)
        if epi == KM.F32:
            assert kw.get("vec_f32") and not kw.get("split_out") and kw["N"] % 2 == 0 and act in (KM.NONE, KM.LEAKY)
        if epi == KM.RES:
            assert kw.get("residual") and kw["N"] % 2 == 0
        if epi == KM.LN:
            assert kw.get("layer_norm") and kw["N"] == 256
        if epi == KM.GENERIC:
            assert kw.get("split_out") and (kw["N"] % bn or kw["act"] not in (KM.NONE, KM.GELU, KM.QUICKGELU, KM.LEAKY))
    assert 256 not in KM.GEMM_KS and min(KM.GEMM_KS) == 64 and max(KM.GEMM_KS) >= 1024
    assert all(k % 64 == 0 for k in KM.GEMM_KS)
    assert {(bn, epi) for (bn, epi, _), kw in KM.GEMM_TC if kw["N"] % 128} == {(128, KM.GENERIC), (128, KM.RES)}


def test_layer_norm_table_is_every_kernel():
    launch = _body(_src("simt.cu"), "void simt_ln(const LnArgs& a")
    launched = re.findall(r"launch_pdl\((k_ln(?:_vec)?<\d+>)", launch)
    assert len(launched) == len(set(launched)) == 5, launched
    assert set(KM.LN_KERNELS) == set(launched)
    assert {d for d, _, _ in KM.LN_CASES} == {64, 256, 263, 384, 512, 768, 1024}


def test_rows_to_split_table_is_every_kernel():
    launch = _body(_src("stack.cu"), "void rows_to_split(mldb_handle* h")
    launched = re.findall(r"(k_rows_to_split8?)<<<", launch)
    assert sorted(launched) == sorted(k for k, _ in KM.ROWS_TO_SPLIT)
