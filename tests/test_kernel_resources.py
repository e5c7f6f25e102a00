"""ptxas resource report of the wgmma GEMM and attention kernels (CPU only: nvcc cross-compiles for sm_90a).

A consumer warpgroup of a three-warpgroup CTA gets 168 registers. Past that, ptxas spills to local
memory and serialises the wgmma instructions (C7512: every MMA waits for the one before it), which
costs far more than the spill traffic itself. These tests compile the kernels with the library's own
flags and pin, per instantiation, the spill bytes and the absence of C7512.
"""
import os
import re
import shutil
import subprocess

import pytest

import __graft_entry__ as G

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

# spill-store bytes that an instantiation may not exceed, and whether its MMAs may be serialised
GEMM_LIMIT = (0, False)                       # every k_gemm_tc instantiation, the LayerNorm epilogue included
ATTN_LIMITS = {                               # (head_dim, causal, key blocks) -> limit
    (64, False, 2): (0, False), (64, True, 2): (0, False),        # the denoiser (79 tokens), the CLIP tower (77)
    (128, False, 2): (256, True), (128, True, 2): (256, True),
    (64, False, 4): (1012, True), (64, True, 4): (1044, True),    # up to 256 keys (the VAE's 196 / 198 frames)
    (128, False, 4): (1364, True), (128, True, 4): (1444, True),
}


def _report(src, tmp_path):
    if not shutil.which(NVCC) and not os.path.exists(NVCC):
        pytest.skip("nvcc not found")
    flags = [f for f in G.NVCC_FLAGS if f != "-shared"]
    r = subprocess.run([NVCC, *flags, "-Xptxas", "-v", "-c", os.path.join(G.CSRC, src),
                        "-o", str(tmp_path / (src + ".o"))], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    spills, serial = {}, set()
    cur = None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores", line)
        if m and cur:
            spills[cur] = int(m.group(1))
        m = re.search(r"C7512\).*function '(\w+)'", line)
        if m:
            serial.add(m.group(1))
    assert spills, r.stderr[-4000:]
    return spills, serial


def _check(name, limit, spills, serial):
    max_spill, may_serialise = limit
    assert spills[name] <= max_spill, f"{name}: {spills[name]} bytes spill stores (limit {max_spill})"
    assert may_serialise or name not in serial, f"{name}: wgmma serialised (C7512)"


def test_gemm_resources(tmp_path):
    spills, serial = _report("gemm_tc.cu", tmp_path)
    gemm = [n for n in spills if re.search(r"k_gemm_tcILi\d+E", n)]
    assert len(gemm) >= 11, sorted(spills)
    assert any("k_gemm_tcILi256ELi1E" in n for n in gemm), "k_gemm_tc<256, EPI_LN> not compiled"
    for n in gemm:
        _check(n, GEMM_LIMIT, spills, serial)


def test_attention_resources(tmp_path):
    spills, serial = _report("attn_tc.cu", tmp_path)
    seen = set()
    for n in spills:
        m = re.search(r"k_attn_tcILi(\d+)ELb([01])ELi(\d+)E", n)
        if not m:
            continue
        key = (int(m.group(1)), m.group(2) == "1", int(m.group(3)))
        assert key in ATTN_LIMITS, f"unexpected instantiation {key}"
        _check(n, ATTN_LIMITS[key], spills, serial)
        seen.add(key)
    assert seen == set(ATTN_LIMITS), sorted(seen)
