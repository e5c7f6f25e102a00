"""ptxas resource report of the GRU step kernel (CPU only; see tests/test_kernel_resources.py): its two consumer
warpgroups must fit the 168 registers of a 384-thread CTA with no spills and unserialised wgmma."""
from test_kernel_resources import _check, _report


def test_gru_step_resources(tmp_path):
    spills, serial = _report("gru_tc.cu", tmp_path)
    names = [n for n in spills if "k_gru_step_tc" in n]
    assert len(names) == 1, sorted(spills)
    _check(names[0], (0, False), spills, serial)
