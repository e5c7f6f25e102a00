"""GPU tests of the native APE / AVE metric (pytest -m gpu): the reference's own ComputeMetrics.update in the fixture,
float64 parity at the HumanML3D eval batch and at a long sequence, the floor's dependence on padded frames, the batch
as the sum of its sequences, bit-identity, the launches per update and the refusals."""
import pytest
import torch

from conftest import golden
from mld_b200 import metrics as M
from oracle import ape_ave as O
from oracle.make_golden_ape_ave import LENGTHS

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
GATE = 1e-6                       # of each output's largest absolute element, against float64


def _rel(out, ref):
    worst = 0.0
    for k in O.NAMES:
        a, r = out[k].double().cpu(), ref[k].double().cpu()
        assert a.shape == r.shape, k
        worst = max(worst, float((a - r).abs().max() / r.abs().max().clamp_min(1e-300)))
    return worst


def _batch(B, T, jointstype, seed, lengths, device="cuda"):
    text = O.synth_joints(B, T, jointstype, seed, lengths, [(0, 1)]).to(device)
    ref = O.synth_joints(B, T, jointstype, seed + 1, lengths).to(device)
    return text, ref


def _ragged(B, T, seed):
    g = torch.Generator().manual_seed(seed)
    ln = torch.randint(40, T + 1, (B,), generator=g)
    ln[0] = T
    return ln.tolist()


@pytest.mark.parametrize("jointstype", ["humanml3d", "mmm"])
@pytest.mark.parametrize("force_in_meter", [True, False])
def test_fixture(jointstype, force_in_meter):
    g = golden("ape_ave.npz")
    text = torch.from_numpy(g[f"{jointstype}/text"]).cuda()
    ref = torch.from_numpy(g[f"{jointstype}/ref"]).cuda()
    out = M.ape_ave_update(text, ref, list(LENGTHS), jointstype=jointstype, force_in_meter=force_in_meter)
    want = {k: torch.from_numpy(g[f"{jointstype}/{int(force_in_meter)}/float64/{k}"]) for k in O.NAMES}
    for k, v in out.items():
        assert v.dtype == torch.float32 and v.device == text.device, k
    assert _rel(out, want) < GATE


@pytest.mark.parametrize("jointstype", ["humanml3d", "mmm"])
def test_eval_batch_against_float64(jointstype):
    B, T = 32, 196
    lengths = _ragged(B, T, 5)
    text, ref = _batch(B, T, jointstype, 7, lengths)
    out = M.ape_ave_update(text, ref, lengths, jointstype=jointstype)
    assert _rel(out, O.ape_ave_update(text, ref, lengths, jointstype)) < GATE


def test_long_sequence_tiles():
    T = 1237                                          # ten frame tiles, the last one partial
    for lengths in ([T], [1000]):
        text, ref = _batch(1, T, "humanml3d", 9, lengths)
        out = M.ape_ave_update(text, ref, lengths)
        assert _rel(out, O.ape_ave_update(text, ref, lengths)) < GATE


def test_padding_moves_the_floor():
    B, T = 4, 60
    lengths = [60, 30, 45, 2]
    text, ref = _batch(B, T, "humanml3d", 13, lengths)
    before = M.ape_ave_update(text, ref, lengths)
    text2 = text.clone()
    text2[1, 30:, :, 1] -= 0.5                        # only padded frames change: the lowest foot goes down
    after = M.ape_ave_update(text2, ref, lengths)
    want = O.ape_ave_update(text2, ref, lengths)
    assert _rel(after, want) < GATE
    assert not torch.equal(before["APE_joints"], after["APE_joints"])
    # the floor shifts heights only: the trajectory terms keep their bits
    assert torch.equal(before["APE_traj"], after["APE_traj"]) and torch.equal(before["AVE_traj"], after["AVE_traj"])
    d_nat = (after["APE_joints"] - before["APE_joints"]).double().cpu()
    d_ref = (want["APE_joints"] - O.ape_ave_update(text, ref, lengths)["APE_joints"]).cpu()
    assert float((d_nat - d_ref).abs().max()) < GATE * float(want["APE_joints"].abs().max())
    assert float(d_ref.abs().max()) > 100 * GATE * float(want["APE_joints"].abs().max())


def test_batch_is_sum_of_sequences():
    B, T = 12, 80
    lengths = _ragged(B, T, 3)
    text, ref = _batch(B, T, "mmm", 17, lengths)
    whole = M.ape_ave_update(text, ref, lengths, jointstype="mmm")
    parts = [M.ape_ave_update(text[i:i + 1], ref[i:i + 1], lengths[i:i + 1], jointstype="mmm") for i in range(B)]
    summed = {k: sum(p[k].double() for p in parts) for k in O.NAMES}
    assert _rel(whole, summed) < GATE


def test_bitwise_repeatable_and_inputs():
    B, T = 40, 196
    lengths = _ragged(B, T, 8)
    text, ref = _batch(B, T, "humanml3d", 21, lengths)
    a = M.ape_ave_update(text, ref, lengths)
    b = M.ape_ave_update(text, ref, lengths)
    for k in O.NAMES:
        assert torch.equal(a[k], b[k]), k
    # lengths as a CPU or CUDA tensor, and non-contiguous joints, give the same bits
    nc_text = text.transpose(1, 2).contiguous().transpose(1, 2)
    assert not nc_text.is_contiguous()
    for ln in (torch.tensor(lengths), torch.tensor(lengths, device="cuda", dtype=torch.int32)):
        c = M.ape_ave_update(nc_text, ref, ln)
        for k in O.NAMES:
            assert torch.equal(a[k], c[k]), k


def _launches():
    return M._engine(torch.device("cuda", torch.cuda.current_device())).launch_count


def test_launches_per_update():
    B, T = 32, 196
    lengths = _ragged(B, T, 4)
    text, ref = _batch(B, T, "humanml3d", 1, lengths)
    M.ape_ave_update(text, ref, lengths)
    n0 = _launches()
    M.ape_ave_update(text, ref, lengths)
    assert 1 <= _launches() - n0 <= 2
    torch.cuda.synchronize()


@pytest.mark.parametrize("case", ["len1", "len_over", "len_count", "J", "jointstype", "f64", "cpu", "shape"])
def test_refusals_before_any_launch(case):
    B, T = 3, 20
    lengths = [20, 10, 5]
    text, ref = _batch(B, T, "humanml3d", 2, lengths)
    M.ape_ave_update(text, ref, lengths)
    n0 = _launches()
    kw, args = {}, [text, ref, lengths]
    err = ValueError
    if case == "len1":
        args[2] = [20, 1, 5]
    elif case == "len_over":
        args[2] = [21, 10, 5]
    elif case == "len_count":
        args[2] = [20, 10]
    elif case == "J":
        kw["jointstype"] = "mmm"
    elif case == "jointstype":
        kw["jointstype"] = "smpl"
        err = NotImplementedError
    elif case == "f64":
        args[0] = text.double()
    elif case == "cpu":
        args[1] = ref.cpu()
    elif case == "shape":
        args[1] = ref[:, :19]
    with pytest.raises(err):
        M.ape_ave_update(*args, **kw)
    assert _launches() == n0
