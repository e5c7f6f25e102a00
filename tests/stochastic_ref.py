"""Reference restatement of the scheduler settings beyond the shipped one, for the stochastic-sampling tests.

``oracle.mld_oracle`` restates diffusers' ``DDIMScheduler`` / ``DDPMScheduler`` for the shipped configs only
(scaled_linear, no clipping, DDIM eta == 0).  The schedulers here extend them with what the yaml may also set
(configs/modules*/scheduler.yaml): the ``linear`` and ``squaredcos_cap_v2`` beta schedules, ``clip_sample``
(clip_sample_range 1.0) and DDIM's ``eta > 0`` variance noise, in diffusers' fp32 operation order.  They stay
subclasses of the oracle's, so ``mld_oracle.diffusion_reverse`` / ``mld_forward`` drive them unchanged; a DDIM
scheduler built with ``step_noise`` [n_steps, ...] takes slice i as the variance noise of step i."""
import math
from typing import Optional

import torch
from torch import Tensor

from oracle import mld_oracle as O


def betas_for_alpha_bar(num_diffusion_timesteps: int, max_beta: float = 0.999) -> Tensor:
    """diffusers' betas_for_alpha_bar (alpha_transform_type "cosine"): double math, then float32."""
    def alpha_bar_fn(t):
        return math.cos((t + 0.008) / 1.008 * math.pi / 2) ** 2
    betas = []
    for i in range(num_diffusion_timesteps):
        t1 = i / num_diffusion_timesteps
        t2 = (i + 1) / num_diffusion_timesteps
        betas.append(min(1 - alpha_bar_fn(t2) / alpha_bar_fn(t1), max_beta))
    return torch.tensor(betas, dtype=torch.float32)


def make_betas(beta_schedule: str, num_train_timesteps: int, beta_start: float, beta_end: float) -> Tensor:
    """The ``betas`` of diffusers' DDIMScheduler / DDPMScheduler __init__ for each beta_schedule."""
    if beta_schedule == "linear":
        return torch.linspace(beta_start, beta_end, num_train_timesteps, dtype=torch.float32)
    if beta_schedule == "scaled_linear":
        return torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
    if beta_schedule == "squaredcos_cap_v2":
        return betas_for_alpha_bar(num_train_timesteps)
    raise NotImplementedError(beta_schedule)


def _set_tables(s, beta_schedule, num_train_timesteps, beta_start, beta_end):
    s.betas = make_betas(beta_schedule, num_train_timesteps, beta_start, beta_end)
    s.alphas = 1.0 - s.betas
    s.alphas_cumprod = torch.cumprod(s.alphas, dim=0)


class DDIMScheduler(O.DDIMScheduler):
    """diffusers.DDIMScheduler with any beta_schedule, clip_sample and eta (epsilon prediction)."""

    def __init__(self, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012,
                 beta_schedule="scaled_linear", clip_sample=False, set_alpha_to_one=False, steps_offset=1,
                 step_noise: Optional[Tensor] = None):
        super().__init__(num_train_timesteps, beta_start, beta_end, set_alpha_to_one=set_alpha_to_one,
                         steps_offset=steps_offset)
        _set_tables(self, beta_schedule, num_train_timesteps, beta_start, beta_end)
        self.final_alpha_cumprod = torch.tensor(1.0) if set_alpha_to_one else self.alphas_cumprod[0]
        self.clip_sample = clip_sample
        self.step_noise = step_noise

    def variance(self, t: int, dtype=torch.float32) -> Tensor:
        """DDIMScheduler._get_variance(t, prev_t)."""
        prev_t = t - self.num_train_timesteps // self.num_inference_steps
        ac = self.alphas_cumprod.to(dtype)
        a_t = ac[t]
        a_prev = ac[prev_t] if prev_t >= 0 else self.final_alpha_cumprod.to(dtype)
        return (1 - a_prev) / (1 - a_t) * (1 - a_t / a_prev)

    def step(self, model_output: Tensor, timestep, sample: Tensor, eta: float = 0.0,
             noise: Optional[Tensor] = None) -> Tensor:
        t = int(timestep)
        prev_t = t - self.num_train_timesteps // self.num_inference_steps
        a_t = self.alphas_cumprod[t]
        a_prev = self.alphas_cumprod[prev_t] if prev_t >= 0 else self.final_alpha_cumprod
        beta_prod_t = 1 - a_t
        pred_x0 = (sample - beta_prod_t ** 0.5 * model_output) / a_t ** 0.5
        if self.clip_sample:
            pred_x0 = pred_x0.clamp(-1.0, 1.0)
        std_dev_t = eta * self.variance(t) ** 0.5
        direction = (1 - a_prev - std_dev_t ** 2) ** 0.5 * model_output
        prev = a_prev ** 0.5 * pred_x0 + direction
        if eta > 0:
            if noise is None:
                i = int((self.timesteps == t).nonzero()[0, 0])
                noise = self.step_noise[i].to(prev.device)
            prev = prev + std_dev_t * noise
        return prev


class DDPMScheduler(O.DDPMScheduler):
    """diffusers.DDPMScheduler (fixed_small variance, epsilon prediction) with any beta_schedule and clip_sample."""

    def __init__(self, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012,
                 beta_schedule="scaled_linear", variance_type="fixed_small", clip_sample=False):
        assert variance_type == "fixed_small"
        super().__init__(num_train_timesteps, beta_start, beta_end)
        _set_tables(self, beta_schedule, num_train_timesteps, beta_start, beta_end)
        self.clip_sample = clip_sample

    def variance(self, t: int, dtype=torch.float32) -> Tensor:
        """DDPMScheduler._get_variance(t) for fixed_small, before the clamp."""
        n = self.num_inference_steps or self.num_train_timesteps
        prev_t = t - self.num_train_timesteps // n
        ac = self.alphas_cumprod.to(dtype)
        a_t = ac[t]
        a_prev = ac[prev_t] if prev_t >= 0 else torch.tensor(1.0, dtype=dtype)
        return (1 - a_prev) / (1 - a_t) * (1 - a_t / a_prev)

    def step(self, model_output: Tensor, timestep, sample: Tensor, noise: Optional[Tensor] = None) -> Tensor:
        t = int(timestep)
        n = self.num_inference_steps or self.num_train_timesteps
        prev_t = t - self.num_train_timesteps // n
        a_t = self.alphas_cumprod[t]
        a_prev = self.alphas_cumprod[prev_t] if prev_t >= 0 else self.one
        beta_prod_t = 1 - a_t
        beta_prod_prev = 1 - a_prev
        cur_alpha = a_t / a_prev
        cur_beta = 1 - cur_alpha
        pred_x0 = (sample - beta_prod_t ** 0.5 * model_output) / a_t ** 0.5
        if self.clip_sample:
            pred_x0 = pred_x0.clamp(-1.0, 1.0)
        c0 = (a_prev ** 0.5 * cur_beta) / beta_prod_t
        c1 = cur_alpha ** 0.5 * beta_prod_prev / beta_prod_t
        prev = c0 * pred_x0 + c1 * sample
        if t > 0:
            var = torch.clamp(beta_prod_prev / beta_prod_t * cur_beta, min=1e-20)
            prev = prev + var ** 0.5 * noise
        return prev
