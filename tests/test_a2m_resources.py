"""ptxas resource report of k_gru_seq_tc (CPU only; see tests/test_kernel_resources.py): both hidden sizes keep the
layer's state, A fragments, accumulators and gi prefetch in registers with no spills and unserialised wgmma."""
from test_kernel_resources import _check, _report


def test_gru_seq_resources(tmp_path):
    spills, serial = _report("gru_tc.cu", tmp_path)
    names = [n for n in spills if "k_gru_seq_tc" in n]
    assert len(names) == 2, sorted(spills)
    for n in names:
        _check(n, (0, False), spills, serial)
