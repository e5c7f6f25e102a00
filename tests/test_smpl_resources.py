"""ptxas resource report of the SMPL layer's kernels (CPU only; see tests/test_kernel_resources.py): the LBS kernel
keeps its accumulators and skinning sums in registers with no spills and unserialised wgmma, and the FK kernel does
not spill."""
from test_kernel_resources import _check, _report


def test_smpl_resources(tmp_path):
    spills, serial = _report("smpl.cu", tmp_path)
    names = [n for n in spills if "k_smpl_lbs" in n or "k_smpl_fk" in n]
    assert len(names) == 2, sorted(spills)
    for n in names:
        _check(n, (0, False), spills, serial)
