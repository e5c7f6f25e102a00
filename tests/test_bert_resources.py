"""ptxas resource report of the text towers' row LayerNorm kernel (CPU only; see tests/test_kernel_resources.py): every
width of k_text_ln, whose BERT embedding and post-norm modes keep the row in registers, compiles without spills."""
from test_kernel_resources import _check, _report


def test_text_ln_resources(tmp_path):
    spills, serial = _report("text_ln.cu", tmp_path)
    names = [n for n in spills if "k_text_ln" in n]
    assert len(names) == 8, sorted(spills)                 # d = 128 .. 1024
    for n in names:
        _check(n, (0, False), spills, serial)
