"""ptxas resource report of k_tconv_tc (CPU only; see tests/test_kernel_resources.py): every channel width keeps its
accumulators in registers with no spills and unserialised wgmma."""
from test_kernel_resources import _check, _report


def test_tconv_resources(tmp_path):
    spills, serial = _report("tconv_tc.cu", tmp_path)
    names = [n for n in spills if "k_tconv_tc" in n]
    assert len(names) == 3, sorted(spills)
    for n in names:
        _check(n, (0, False), spills, serial)
