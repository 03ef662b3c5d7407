"""Noise schedulers for the denoise loop, with the ``set_timesteps / scale_model_input / step`` interface the patched
pipeline drives (utils/monkey_patch/sd_pipeline_monkey_patch.py:153-154, 190, 216-218).

The reference holds a diffusers ``DDPMScheduler`` built from the SD-2.1-base ``scheduler/`` config
(decoders/sd.py:48-50) and hands it to the pipeline (sd.py:154-159), so image generation is DDPM ancestral sampling
on a ``leading``-spaced timestep grid.  diffusers (pinned 0.20.0, requirements.txt:9) is a third-party dependency that is
neither under /root/reference nor in this image: ``DDPMScheduler`` below restates its published arithmetic (Ho et
al. 2020, eq. 7 posterior mean + ``fixed_small`` posterior variance; ``scheduling_ddpm.py`` ``set_timesteps`` /
``step`` / ``_get_variance``) -- **parity unpinned**, checked against the independent restatement in
``oracle/scheduler.py``.  Any object with the same three methods (e.g. a real diffusers scheduler) can be passed to
``denoise_loop`` instead.  ``DDIMScheduler`` (eta = 0) is the deterministic variant round 1 used.
"""
from __future__ import annotations

import torch

# SD-2.1-base ``scheduler/scheduler_config.json`` fields DDPMScheduler.from_pretrained picks up (sd.py:48-50)
SD21_BASE_SCHEDULER = dict(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                           prediction_type="epsilon", steps_offset=1, clip_sample=False, variance_type="fixed_small",
                           timestep_spacing="leading")


def _betas(num_train_timesteps, beta_start, beta_end, beta_schedule):
    if beta_schedule == "scaled_linear":      # the latent-diffusion schedule
        return torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
    if beta_schedule == "linear":
        return torch.linspace(beta_start, beta_end, num_train_timesteps, dtype=torch.float32)
    raise NotImplementedError(f"beta_schedule {beta_schedule!r}")


class _SchedulerBase:
    order = 1
    init_noise_sigma = 1.0

    def __init__(self, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                 prediction_type="epsilon", steps_offset=0, timestep_spacing="leading", **extra):
        self.num_train_timesteps = num_train_timesteps
        self.prediction_type = prediction_type
        self.steps_offset = steps_offset
        self.timestep_spacing = timestep_spacing
        self.betas = _betas(num_train_timesteps, beta_start, beta_end, beta_schedule)
        self.alphas_cumprod = torch.cumprod(1.0 - self.betas, dim=0)           # fp32, like diffusers
        self.num_inference_steps = None
        self.timesteps = torch.arange(num_train_timesteps - 1, -1, -1)
        self._acp_dev = None

    def set_timesteps(self, num_inference_steps: int, device=None):
        if num_inference_steps > self.num_train_timesteps:
            raise ValueError("num_inference_steps exceeds num_train_timesteps")
        n, N = num_inference_steps, self.num_train_timesteps
        self.num_inference_steps = n
        if self.timestep_spacing == "leading":
            ts = (torch.arange(0, n, dtype=torch.float64) * (N // n)).round().flip(0).long() + self.steps_offset
        elif self.timestep_spacing == "linspace":
            ts = torch.linspace(0, N - 1, n, dtype=torch.float64).round().flip(0).long()
        elif self.timestep_spacing == "trailing":
            ts = (torch.arange(N, 0, -N / n, dtype=torch.float64)).round().long() - 1
        else:
            raise NotImplementedError(self.timestep_spacing)
        self.timesteps = ts.to(device) if device is not None else ts
        self._host_timesteps = ts.tolist()       # so that step() never reads a device scalar

    def scale_model_input(self, sample, timestep=None):
        return sample

    def _acp(self, device):
        if self._acp_dev is None or self._acp_dev.device != device:
            self._acp_dev = self.alphas_cumprod.to(device)
        return self._acp_dev

    def _prev(self, t: int) -> int:
        return t - self.num_train_timesteps // self.num_inference_steps

    def _noise_coefficients(self, timesteps, sample):
        """(sqrt(abar_t), sqrt(1 - abar_t)) per sample, shaped to broadcast over (C, H, W); ``alphas_cumprod`` is moved
        to the sample's device AND dtype first, as in diffusers 0.20 (a 16-bit sample rounds abar_t to 16 bit)."""
        acp = self.alphas_cumprod.to(device=sample.device, dtype=sample.dtype)[timesteps.to(sample.device)]
        shape = (-1,) + (1,) * (sample.dim() - 1)
        return (acp ** 0.5).flatten().view(shape), ((1 - acp) ** 0.5).flatten().view(shape)

    def add_noise(self, original_samples, noise, timesteps):
        """Forward diffusion ``sqrt(abar_t) x + sqrt(1 - abar_t) eps``, one timestep per sample (diffusers 0.20's
        ``add_noise``)."""
        a, b = self._noise_coefficients(timesteps, original_samples)
        return a * original_samples + b * noise

    def get_velocity(self, sample, noise, timesteps):
        """The v-prediction target ``sqrt(abar_t) eps - sqrt(1 - abar_t) x``, one timestep per sample."""
        a, b = self._noise_coefficients(timesteps, sample)
        return a * noise - b * sample

    def _x0(self, model_output, sample, a_t):
        if self.prediction_type == "epsilon":
            return (sample - (1 - a_t) ** 0.5 * model_output) / a_t ** 0.5
        if self.prediction_type == "v_prediction":
            return a_t ** 0.5 * sample - (1 - a_t) ** 0.5 * model_output
        if self.prediction_type == "sample":
            return model_output
        raise NotImplementedError(self.prediction_type)


class DDPMScheduler(_SchedulerBase):
    """Ancestral sampling step: ``x_{t-1} = c0 * x0_pred + ct * x_t + sigma_t * z`` with
    ``c0 = sqrt(abar_prev) * beta_t / (1 - abar_t)``, ``ct = sqrt(alpha_t) * (1 - abar_prev) / (1 - abar_t)``,
    ``alpha_t = abar_t / abar_prev`` (so strided grids are handled), ``sigma_t^2 = clamp((1 - abar_prev) / (1 - abar_t)
    * beta_t, 1e-20)`` (``fixed_small``) and no noise at the last step (t == 0)."""

    def __init__(self, clip_sample=False, clip_sample_range=1.0, variance_type="fixed_small", **kw):
        super().__init__(**kw)
        if variance_type not in ("fixed_small", "fixed_large"):
            raise NotImplementedError(f"variance_type {variance_type!r}")
        self.clip_sample, self.clip_sample_range, self.variance_type = clip_sample, clip_sample_range, variance_type

    def step(self, model_output, timestep, sample, generator=None, noise=None):
        """``timestep`` may be a Python int or a 0-d tensor; ``noise`` (extension) supplies z explicitly."""
        t = int(timestep)
        prev_t = self._prev(t)
        acp = self._acp(sample.device)
        a_t = acp[t]
        a_prev = acp[prev_t] if prev_t >= 0 else torch.ones((), device=sample.device)
        alpha_t = a_t / a_prev
        beta_t = 1 - alpha_t
        x = sample.float()
        eps = model_output.float()
        x0 = self._x0(eps, x, a_t)
        if self.clip_sample:
            x0 = x0.clamp(-self.clip_sample_range, self.clip_sample_range)
        c0 = a_prev ** 0.5 * beta_t / (1 - a_t)
        ct = alpha_t ** 0.5 * (1 - a_prev) / (1 - a_t)
        prev = c0 * x0 + ct * x
        if t > 0:
            var = beta_t if self.variance_type == "fixed_large" else (1 - a_prev) / (1 - a_t) * beta_t
            var = var.clamp(min=1e-20)
            if noise is None:
                noise = torch.randn(model_output.shape, generator=generator, device=model_output.device,
                                    dtype=model_output.dtype)
            prev = prev + var ** 0.5 * noise.float()
        return prev.to(sample.dtype)


class DDIMScheduler(_SchedulerBase):
    """Deterministic DDIM (eta = 0): ``x_prev = sqrt(abar_prev) x0 + sqrt(1 - abar_prev) eps`` with abar_prev = 1 after
    the last step (``set_alpha_to_one``)."""

    def __init__(self, timestep_spacing="linspace", **kw):
        super().__init__(timestep_spacing=timestep_spacing, **kw)

    def _prev(self, t):
        i = self._host_timesteps.index(t)
        return self._host_timesteps[i + 1] if i + 1 < len(self._host_timesteps) else -1

    def step(self, model_output, timestep, sample, generator=None, noise=None):
        t = int(timestep)
        prev_t = self._prev(t)
        acp = self._acp(sample.device)
        a_t = acp[t]
        a_prev = acp[prev_t] if prev_t >= 0 else torch.ones((), device=sample.device)
        x, out = sample.float(), model_output.float()
        x0 = self._x0(out, x, a_t)
        eps = out if self.prediction_type == "epsilon" else (x - a_t ** 0.5 * x0) / (1 - a_t) ** 0.5
        return (a_prev ** 0.5 * x0 + (1 - a_prev) ** 0.5 * eps).to(sample.dtype)
