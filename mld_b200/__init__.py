"""mld_b200: H100-native (sm_90a) latent-diffusion sampling path for Motion Latent Diffusion.

The math lives in ``libmldb200.so`` (hand-written CUDA, C ABI in ``include/mldb.h``); this
package is the torch-side mirror of the reference's interfaces for that path:
``modules`` (YAML ``target:`` drop-ins), ``pipeline.B200MLD`` (``MLD.forward`` /
``_diffusion_reverse`` surface), ``engine.Engine`` (raw C-ABI wrapper), ``distributed``
(batch sharding + the single all-gather).  There is no CPU or PyTorch fallback.
"""
__all__ = ["synth", "engine", "modules", "pipeline", "distributed"]
