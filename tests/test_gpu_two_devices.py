"""Handles on two devices in one process (pytest -m gpu, skipped with fewer than 2 GPUs).

A kernel's shared-memory opt-in holds for one device, and the attention kernels size their grid from the device's SM
count, so each handle sets up the kernels on its own device. The same seeded sample then gives the same motion on both
devices, and neither falls back to the CUDA-core attention."""
import pytest
import torch

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

B, S, STEPS = 2, 77, 2
LENGTHS = [196, 64]


def _engine(device):
    from mld_b200 import synth
    from mld_b200.engine import Engine, make_config
    eng = Engine(make_config(), device)
    eng.load_state_dict(synth.denoiser_state_dict(1234), "denoiser.")
    eng.load_state_dict(synth.mld_vae_state_dict(4321), "vae.")
    eng.finalize()
    eng.set_mean_std(*synth.mean_std())
    eng.set_timesteps(STEPS)
    return eng


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_same_sample_on_two_devices_in_one_process(built_lib):
    from mld_b200 import synth
    engines = [_engine(0), _engine(1)]   # both handles exist before either samples
    ctx, noise = synth.text_context(B, S, seed=11), synth.init_noise(B, seed=12)
    joints = []
    for dev, eng in enumerate(engines):
        eng.kernel_stats(reset=True)
        joints.append(eng.sample(ctx, noise, LENGTHS, want=("joints",))["joints"].cpu())
        st = eng.kernel_stats()
        assert st["attn_tc"] > 0 and st["attn_simt"] == 0, (dev, st)
    assert torch.equal(joints[0], joints[1])
