"""ptxas resource report of the APE / AVE kernels (CPU only; see tests/test_kernel_resources.py): no spills."""
from test_kernel_resources import _check, _report


def test_metrics_resources(tmp_path):
    spills, serial = _report("metrics.cu", tmp_path)
    names = [n for n in spills if "k_ape_ave" in n]
    assert len(names) == 2, sorted(spills)
    for n in names:
        _check(n, (0, False), spills, serial)
