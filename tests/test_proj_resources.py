"""ptxas resource report of the K = 256 projection kernel (CPU only; see tests/test_kernel_resources.py). k_proj_tc
holds two 64 x 128 accumulators per thread in a 256-thread CTA, which ptxas compiles under 255 registers; every
activation's instantiation must fit them with no spills and unserialised wgmma."""
import re

from test_kernel_resources import _check, _report


def test_proj_resources(tmp_path):
    spills, serial = _report("gemm_tc.cu", tmp_path)
    names = [n for n in spills if "k_proj_tc" in n]
    acts = sorted(int(re.search(r"k_proj_tcILi(\d+)E", n).group(1)) for n in names)
    assert acts == [0, 1, 4, 5], sorted(spills)                # NONE, GELU, QUICKGELU, LEAKY
    for n in names:
        _check(n, (0, False), spills, serial)
