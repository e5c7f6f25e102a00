"""CPU tests of the APE / AVE metric: the float64 oracle against the reference's own ComputeMetrics.update, the
fixture's coverage (a zero `across` frame, padding that moves the floor), and the refusals of ape_ave_update, which
all happen before any GPU work."""
import numpy as np
import pytest
import torch

from conftest import golden
from oracle import ape_ave as O
from oracle.make_golden_ape_ave import LENGTHS, ZERO_ACROSS, case_inputs


@pytest.mark.parametrize("jointstype", ["humanml3d", "mmm"])
@pytest.mark.parametrize("force_in_meter", [True, False])
def test_oracle_matches_reference(jointstype, force_in_meter):
    g = golden("ape_ave.npz")
    text, ref = torch.from_numpy(g[f"{jointstype}/text"]), torch.from_numpy(g[f"{jointstype}/ref"])
    out = O.ape_ave_update(text, ref, LENGTHS, jointstype, force_in_meter)
    for k in O.NAMES:
        want = g[f"{jointstype}/{int(force_in_meter)}/float64/{k}"]
        assert out[k].shape == want.shape, k
        np.testing.assert_allclose(out[k].numpy(), want, rtol=1e-12, atol=1e-12 * np.abs(want).max(), err_msg=k)


@pytest.mark.parametrize("jointstype", ["humanml3d", "mmm"])
def test_fixture_inputs(jointstype):
    g = golden("ape_ave.npz")
    text, ref = case_inputs(jointstype)
    assert torch.equal(text, torch.from_numpy(g[f"{jointstype}/text"]))
    assert torch.equal(ref, torch.from_numpy(g[f"{jointstype}/ref"]))
    assert min(LENGTHS) == 2 and max(LENGTHS) == text.shape[1]
    tab = O.TABLES[jointstype]
    (ls, rs), (lh, rh) = tab["shoulders"], tab["hips"]
    for b, t in ZERO_ACROSS:
        assert t < LENGTHS[b]
        p = text[b, t, 1:].double() - text[b, t, 0].double()
        across = p[rh] - p[lh] + p[rs] - p[ls]
        assert across[0] == 0 and across[2] == 0
    # padding reaches the result through the floor: it differs from the valid frames and lowers the feet
    feet = list(tab["feet"])
    for b, n in enumerate(LENGTHS):
        if n < text.shape[1]:
            assert text[b, n:, feet, 1].min() < text[b, :n, feet, 1].min()


def test_refusals_before_gpu_work():
    from mld_b200.metrics import ape_ave_update
    x = torch.zeros(2, 5, 22, 3)                  # a CPU tensor: refused before any device is touched
    with pytest.raises(NotImplementedError):
        ape_ave_update(x, x, [5, 5], jointstype="smplh")
    with pytest.raises(ValueError, match="CUDA"):
        ape_ave_update(x, x, [5, 5])
    with pytest.raises(ValueError, match="CUDA"):
        ape_ave_update(x.double(), x.double(), [5, 5])
