"""ptxas resource report of the fused FFN kernel (CPU only; see tests/test_kernel_resources.py). k_ffn_tc runs as
two warpgroups with no producer warpgroup, so ptxas may give it 255 registers per thread instead of the 168 of a
384-thread CTA; its body must fit them with no spills and unserialised wgmma."""
from test_kernel_resources import _check, _report


def test_ffn_resources(tmp_path):
    spills, serial = _report("gemm_tc.cu", tmp_path)
    names = [n for n in spills if "k_ffn_tc" in n]
    assert len(names) == 1, sorted(spills)
    _check(names[0], (0, False), spills, serial)
