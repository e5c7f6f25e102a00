"""CPU: the scheduler settings beyond the shipped one (beta_schedule, clip_sample, DDIM eta > 0).

The library's host tables must equal torch's for every beta schedule, the configuration surface must refuse
what the library does not implement, and the per-step noise must shard with the batch."""
import ctypes as C
import os
import re

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import stochastic_ref as R
from conftest import ROOT
from mld_b200 import _lib
from mld_b200.distributed import sample_sharded
from oracle import mld_oracle as O

SCHEDULES = ("scaled_linear", "linear", "squaredcos_cap_v2")


def _table(lib, cfg):
    ac = torch.empty(cfg.num_train_timesteps, dtype=torch.float32)
    rc = lib.mldb_scheduler_table(C.byref(cfg), C.c_void_p(ac.data_ptr()))
    return rc, ac


@pytest.mark.parametrize("schedule", SCHEDULES)
def test_library_table_bit_exact_per_schedule(built_lib, schedule):
    from mld_b200.engine import make_config
    for T, b0, b1 in ((1000, 0.00085, 0.012), (1000, 0.0001, 0.02), (500, 0.00085, 0.012)):
        cfg = make_config(beta_schedule=schedule, num_train_timesteps=T, beta_start=b0, beta_end=b1)
        rc, ac = _table(built_lib, cfg)
        assert rc == 0
        ref = R.DDIMScheduler(T, b0, b1, beta_schedule=schedule)
        assert torch.equal(ac, ref.alphas_cumprod), (schedule, T, b0, b1)
        assert torch.equal(ac, R.DDPMScheduler(T, b0, b1, beta_schedule=schedule).alphas_cumprod)


def test_squaredcos_betas_are_capped():
    b = R.make_betas("squaredcos_cap_v2", 1000, 0.0, 0.0)
    assert b.dtype == torch.float32 and float(b.max()) == float(torch.tensor(0.999))
    assert float(b[0]) > 0 and bool((b[1:] >= b[:-1]).all())


def test_reference_restatement_matches_oracle_on_the_shipped_setting():
    """eta == 0, scaled_linear, no clipping: the extended schedulers are the oracle's, bit for bit."""
    g = torch.Generator().manual_seed(5)
    x, e, nz = (torch.randn(3, 1, 256, generator=g) for _ in range(3))
    a, b = R.DDIMScheduler(), O.DDIMScheduler()
    a.set_timesteps(50)
    b.set_timesteps(50)
    for t in (981, 501, 1):
        assert torch.equal(a.step(e, t, x), b.step(e, t, x))
    a, b = R.DDPMScheduler(), O.DDPMScheduler()
    a.set_timesteps(20)
    b.set_timesteps(20)
    for t in (950, 500, 0):
        assert torch.equal(a.step(e, t, x, noise=nz), b.step(e, t, x, noise=nz))


@pytest.mark.parametrize("schedule", SCHEDULES)
def test_ddim_eta1_full_length_std_equals_ddpm_fixed_small(schedule):
    """DDIM with eta = 1 run over all training timesteps (steps_offset 0) is the ancestral DDPM sampler: its
    per-step std equals DDPM's fixed_small sigma (float64).  At t = 0 DDPM adds no noise, and DDIM's std is 0
    when the final alpha_cumprod is one."""
    T = 1000
    ddim = R.DDIMScheduler(T, beta_schedule=schedule, steps_offset=0, set_alpha_to_one=True)
    ddpm = R.DDPMScheduler(T, beta_schedule=schedule)
    ddim.set_timesteps(T)
    ddpm.set_timesteps(T)
    assert torch.equal(ddim.timesteps, ddpm.timesteps)
    for t in ddpm.timesteps.tolist():
        s_ddim = 1.0 * ddim.variance(t, torch.float64) ** 0.5
        if t == 0:
            assert float(s_ddim) == 0.0
            continue
        s_ddpm = ddpm.variance(t, torch.float64) ** 0.5
        assert abs(float(s_ddim - s_ddpm)) <= 1e-12, t


def test_make_config_validates_scheduler_settings(built_lib):
    from mld_b200.engine import make_config
    with pytest.raises(ValueError, match="beta_schedule"):
        make_config(beta_schedule="cosine")
    for eta in (-0.1, 1.5, float("nan")):
        with pytest.raises(ValueError, match="eta"):
            make_config(eta=eta)
    cfg = make_config(eta=1.0, beta_schedule="linear", clip_sample=True)
    assert (cfg.eta, cfg.beta_schedule, cfg.clip_sample) == (1.0, _lib.BETA_SCHEDULES["linear"], 1)
    d = _lib.default_config()
    assert (d.eta, d.beta_schedule, d.clip_sample) == (0.0, 0, 0)          # the shipped scheduler.yaml


def test_library_refuses_unknown_schedule_and_eta(built_lib):
    """The C side checks the same settings (mldb_create runs the same check as the table helper)."""
    cfg = _lib.default_config()
    cfg.beta_schedule = 3
    rc, _ = _table(built_lib, cfg)
    assert rc == 1 and b"beta_schedule" in built_lib.mldb_last_error()
    cfg = _lib.default_config()
    cfg.eta = 1.25
    rc, _ = _table(built_lib, cfg)
    assert rc == 1 and b"eta" in built_lib.mldb_last_error()


def test_header_and_binding_agree_on_abi_4(built_lib):
    text = open(os.path.join(ROOT, "include", "mldb.h")).read()
    assert int(re.search(r"#define MLDB_ABI_VERSION (\d+)", text).group(1)) == 4 == _lib.MLDB_ABI_VERSION
    assert built_lib.mldb_abi_version() == 4
    for name, v in (("SCALED_LINEAR", "scaled_linear"), ("LINEAR", "linear"),
                    ("SQUAREDCOS_CAP_V2", "squaredcos_cap_v2")):
        assert int(re.search(rf"#define MLDB_BETA_{name} (\d+)", text).group(1)) == _lib.BETA_SCHEDULES[v]
    # the two new fields close the struct, after njoints
    body = re.search(r"typedef struct mldb_config \{(.*?)\} mldb_config;", text, re.S).group(1)
    fields = re.findall(r"^\s*\w+\s+(\w+);", body, re.M)
    assert fields == [f for f, _ in _lib.MldbConfig._fields_]
    assert fields[-3:] == ["njoints", "beta_schedule", "clip_sample"]


# ------------------------------------------------------------------ sharding of the per-step draws
def _fake_sampler(cond, noise, lengths, step_noise):
    b = noise.shape[0]
    out = torch.zeros(b, max(lengths), 2)
    for i in range(b):
        out[i, : lengths[i]] = cond[i].sum() + cond[b + i].sum() + noise[i].sum() + step_noise[:, i].sum()
    return out


def _inputs(B):
    g = torch.Generator().manual_seed(1)
    cond = torch.randn(2 * B, 3, 8, generator=g)
    noise = torch.randn(B, 1, 16, generator=g)
    step_noise = torch.randn(5, B, 1, 16, generator=g)
    lengths = torch.randint(3, 9, (B,), generator=g).tolist()
    return cond, noise, step_noise, lengths


def _worker(rank, world, port, B, out_path):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    cond, noise, step_noise, lengths = _inputs(B)
    out = sample_sharded(_fake_sampler, cond, noise, lengths, cfg_on=True, step_noise=step_noise)
    if rank == 0:
        torch.save(out, out_path)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("B", [8, 7])
def test_two_rank_gather_slices_step_noise(tmp_path, B):
    import socket
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    out_path = str(tmp_path / "gathered.pt")
    procs = [ctx.Process(target=_worker, args=(r, 2, port, B, out_path)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(120)
        assert p.exitcode == 0
    cond, noise, step_noise, lengths = _inputs(B)
    assert torch.equal(torch.load(out_path), _fake_sampler(cond, noise, lengths, step_noise))
