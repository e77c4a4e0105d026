"""minicomfy -- a small stand-in for the slice of ComfyUI the LanPaint nodes touch.

NOT ComfyUI and not part of the product: ComfyUI is an un-vendored, unpinned
third-party dependency of the reference (SURVEY Appendix A) and is absent from
this image.  Tests and bench.py need *something* to drive the node layer end to
end (`nodes.common_ksampler -> CFGGuider.sample -> outer_sample -> inner_sample
-> KSAMPLER.sample -> k-diffusion sampler -> model(x, sigma)`), so this package
re-creates that call chain with the member names listed in SURVEY Appendix A,
written from the documented behaviour of those calls, nothing more.

    import minicomfy; minicomfy.install()      # registers comfy.*, nodes, latent_preview, comfyui_version

`install()` refuses to shadow a real ComfyUI.
"""
from __future__ import annotations

import math
import sys
import types
from typing import Callable

import torch

from . import deis  # noqa: F401  sample_deis reads its coefficients through this attribute, as ComfyUI's does


# ------------------------------------------------------------------ model side
class ModelType:
    EPS = "EPS"
    V_PREDICTION = "V_PREDICTION"
    FLUX = "FLUX"
    FLOW = "FLOW"


class ModelSamplingEPS:
    """VE (x_t = x_0 + sigma*noise) parameterisation, SDXL-like sigma range."""

    sigma_min, sigma_max = 0.0292, 14.6146

    def noise_scaling(self, sigma, noise, latent_image, max_denoise=False):
        sigma = sigma.view(sigma.shape[:1] + (1,) * (noise.ndim - 1)) if sigma.ndim <= 1 else sigma
        if max_denoise:
            noise = noise * torch.sqrt(1.0 + sigma ** 2.0)
        else:
            noise = noise * sigma
        return noise + latent_image

    def inverse_noise_scaling(self, sigma, latent):
        return latent


class ModelSamplingCONST:
    """Rectified-flow parameterisation (x_t = sigma*noise + (1-sigma)*x_0) with ComfyUI's time shift:
    sigma(t) = shift*t / (1 + (shift-1)*t), tabulated at t = 1/1000 .. 1 (ModelSamplingDiscreteFlow)."""

    noise_scale = 1.0

    def __init__(self, shift: float = 1.0, timesteps: int = 1000):
        self.shift = float(shift)
        t = torch.arange(1, timesteps + 1, dtype=torch.float32) / timesteps
        self.sigmas = self.shift * t / (1 + (self.shift - 1) * t)

    @property
    def sigma_min(self):
        return self.sigmas[0]

    @property
    def sigma_max(self):
        return self.sigmas[-1]

    def noise_scaling(self, sigma, noise, latent_image, max_denoise=False):
        sigma = sigma.view(sigma.shape[:1] + (1,) * (noise.ndim - 1)) if sigma.ndim <= 1 else sigma
        return sigma * (self.noise_scale * noise) + (1.0 - sigma) * latent_image

    def inverse_noise_scaling(self, sigma, latent):
        sigma = sigma.view(sigma.shape[:1] + (1,) * (latent.ndim - 1)) if sigma.ndim <= 1 else sigma
        return latent / (1.0 - sigma)


class BaseModel:
    """`denoiser(x, sigma, cond) -> x0 prediction` wrapped with ComfyUI's BaseModel members."""

    def __init__(self, denoiser: Callable, model_type=ModelType.EPS, latent_channels: int = 4, shift: float = 1.0):
        self.diffusion_model = denoiser
        self.model_type = model_type
        self.model_sampling = (ModelSamplingCONST(shift) if model_type in (ModelType.FLUX, ModelType.FLOW)
                               else ModelSamplingEPS())
        self.latent_channels = latent_channels

    def apply_model(self, x, t, c=None, **kwargs):
        return self.diffusion_model(x, t, c)

    def process_latent_out(self, latent):
        return latent

    def extra_conds(self, **kwargs):
        return {}


class WAN22(BaseModel):
    pass


class ModelPatcher:
    def __init__(self, model: BaseModel, load_device):
        self.model = model
        self.load_device = torch.device(load_device)
        self.model_options = {"transformer_options": {}}
        self.pre_runs = 0
        self.cleanups = 0

    def model_dtype(self):
        return torch.float32

    def pre_run(self):
        self.pre_runs += 1

    def cleanup(self):
        self.cleanups += 1

    def get_model_object(self, name):
        return getattr(self.model, name)


# ------------------------------------------------------------------ comfy.utils / model_management
PROGRESS_BAR_ENABLED = False


def repeat_to_batch_size(tensor, batch_size, dim=0):
    if tensor.shape[dim] > batch_size:
        return tensor.narrow(dim, 0, batch_size)
    if tensor.shape[dim] < batch_size:
        reps = [1] * tensor.ndim
        reps[dim] = math.ceil(batch_size / tensor.shape[dim])
        return tensor.repeat(reps).narrow(dim, 0, batch_size)
    return tensor


def intermediate_device():
    return torch.device("cpu")


# ------------------------------------------------------------------ comfy.sampler_helpers
def prepare_mask(noise_mask, shape, device):
    m = torch.nn.functional.interpolate(noise_mask.reshape((-1, 1, noise_mask.shape[-2], noise_mask.shape[-1])),
                                        size=(shape[-2], shape[-1]), mode="bilinear")
    m = torch.cat([m] * shape[1], dim=1)
    return repeat_to_batch_size(m, shape[0]).to(device)


def prepare_sampling(model_patcher, noise_shape, conds, model_options=None):
    return model_patcher.model, conds, []


def cleanup_models(conds, models):
    return None


# ------------------------------------------------------------------ comfy.samplers
def cast_to_load_options(model_options, device=None, dtype=None):
    return None


def calc_cond_batch(model, conds, x_in, timestep, model_options):
    """One denoiser evaluation per non-None cond; returns the list of x0 predictions."""
    out = []
    for c in conds:
        out.append(None if c is None else model.apply_model(x_in, timestep, c))
    return out


def cfg_function(model, cond_pred, uncond_pred, cond_scale, x, timestep, model_options={}, cond=None, uncond=None):
    if uncond_pred is None:
        uncond_pred = cond_pred
    if "sampler_cfg_function" in model_options:
        args = {"cond": x - cond_pred, "uncond": x - uncond_pred, "cond_scale": cond_scale, "timestep": timestep,
                "input": x, "sigma": timestep, "cond_denoised": cond_pred, "uncond_denoised": uncond_pred,
                "model": model, "model_options": model_options}
        cfg_result = x - model_options["sampler_cfg_function"](args)
    else:
        cfg_result = uncond_pred + (cond_pred - uncond_pred) * cond_scale
    for fn in model_options.get("sampler_post_cfg_function", []):
        cfg_result = fn({"denoised": cfg_result, "cond": cond, "uncond": uncond, "cond_scale": cond_scale,
                         "model": model, "uncond_denoised": uncond_pred, "cond_denoised": cond_pred,
                         "sigma": timestep, "model_options": model_options, "input": x})
    return cfg_result


def sampling_function(model, x, timestep, uncond, cond, cond_scale, model_options={}, seed=None):
    if math.isclose(cond_scale, 1.0) and not model_options.get("disable_cfg1_optimization", False):
        uncond_ = None
    else:
        uncond_ = uncond
    out = calc_cond_batch(model, [cond, uncond_], x, timestep, model_options)
    return cfg_function(model, out[0], out[1], cond_scale, x, timestep, model_options=model_options, cond=cond,
                        uncond=uncond_)


class KSamplerX0Inpaint:
    """Stock (non-LanPaint) masked denoise wrapper."""

    def __init__(self, model, sigmas):
        self.inner_model = model
        self.sigmas = sigmas

    def __call__(self, x, sigma, denoise_mask, model_options={}, seed=None):
        if denoise_mask is not None:
            latent_mask = 1.0 - denoise_mask
            x = x * denoise_mask + self.inner_model.inner_model.model_sampling.noise_scaling(
                sigma.reshape([sigma.shape[0]] + [1] * (x.ndim - 1)), self.noise, self.latent_image) * latent_mask
        out = self.inner_model(x, sigma, model_options=model_options, seed=seed)
        if denoise_mask is not None:
            out = out * denoise_mask + self.latent_image * latent_mask
        return out


def _append_dims(s, ndim):
    return s.reshape(s.shape + (1,) * (ndim - s.ndim))


@torch.no_grad()
def sample_euler(model, x, sigmas, extra_args=None, callback=None, disable=None):
    extra_args = extra_args or {}
    s_in = x.new_ones([x.shape[0]])
    for i in range(len(sigmas) - 1):
        sigma = sigmas[i]
        denoised = model(x, sigma * s_in, **extra_args)
        d = (x - denoised) / _append_dims(sigma * s_in, x.ndim)
        if callback is not None:
            callback({"x": x, "i": i, "sigma": sigmas[i], "sigma_hat": sigma, "denoised": denoised})
        x = x + d * (sigmas[i + 1] - sigma)
    return x


@torch.no_grad()
def sample_heun(model, x, sigmas, extra_args=None, callback=None, disable=None):
    extra_args = extra_args or {}
    s_in = x.new_ones([x.shape[0]])
    for i in range(len(sigmas) - 1):
        sigma = sigmas[i]
        denoised = model(x, sigma * s_in, **extra_args)
        d = (x - denoised) / _append_dims(sigma * s_in, x.ndim)
        if callback is not None:
            callback({"x": x, "i": i, "sigma": sigmas[i], "sigma_hat": sigma, "denoised": denoised})
        dt = sigmas[i + 1] - sigma
        if sigmas[i + 1] == 0:
            x = x + d * dt
        else:
            x_2 = x + d * dt
            denoised_2 = model(x_2, sigmas[i + 1] * s_in, **extra_args)
            d_2 = (x_2 - denoised_2) / _append_dims(sigmas[i + 1] * s_in, x.ndim)
            x = x + (d + d_2) / 2 * dt
    return x


@torch.no_grad()
def sample_euler_ancestral(model, x, sigmas, extra_args=None, callback=None, disable=None, eta=1.0, s_noise=1.0):
    """k-diffusion's ancestral Euler with its default noise sampler (torch.randn_like on the global generator)."""
    extra_args = extra_args or {}
    s_in = x.new_ones([x.shape[0]])
    for i in range(len(sigmas) - 1):
        denoised = model(x, sigmas[i] * s_in, **extra_args)
        s_from, s_to = float(sigmas[i]), float(sigmas[i + 1])
        s_up = min(s_to, eta * (s_to ** 2 * (s_from ** 2 - s_to ** 2) / s_from ** 2) ** 0.5) if s_to > 0 else 0.0
        s_down = (s_to ** 2 - s_up ** 2) ** 0.5
        if callback is not None:
            callback({"x": x, "i": i, "sigma": sigmas[i], "sigma_hat": sigmas[i], "denoised": denoised})
        d = (x - denoised) / _append_dims(sigmas[i] * s_in, x.ndim)
        x = x + d * (s_down - s_from)
        if s_to > 0:
            x = x + torch.randn_like(x) * s_noise * s_up
    return x


@torch.no_grad()
def sample_dpmpp_2m(model, x, sigmas, extra_args=None, callback=None, disable=None):
    """k-diffusion's DPM-Solver++(2M): a second-order multistep update from this step's and the previous step's
    denoised latents, first order on the first step and on the step to sigma = 0."""
    extra_args = extra_args or {}
    s_in = x.new_ones([x.shape[0]])
    sigma_fn = lambda t: t.neg().exp()     # noqa: E731
    t_fn = lambda sigma: sigma.log().neg()  # noqa: E731
    old_denoised = None
    for i in range(len(sigmas) - 1):
        denoised = model(x, sigmas[i] * s_in, **extra_args)
        if callback is not None:
            callback({"x": x, "i": i, "sigma": sigmas[i], "sigma_hat": sigmas[i], "denoised": denoised})
        t, t_next = t_fn(sigmas[i]), t_fn(sigmas[i + 1])
        h = t_next - t
        if old_denoised is None or sigmas[i + 1] == 0:
            x = (sigma_fn(t_next) / sigma_fn(t)) * x - (-h).expm1() * denoised
        else:
            h_last = t - t_fn(sigmas[i - 1])
            r = h_last / h
            denoised_d = (1 + 1 / (2 * r)) * denoised - (1 / (2 * r)) * old_denoised
            x = (sigma_fn(t_next) / sigma_fn(t)) * x - (-h).expm1() * denoised_d
        old_denoised = denoised
    return x


@torch.no_grad()
def sample_dpm_2(model, x, sigmas, extra_args=None, callback=None, disable=None):
    """k-diffusion's DPM-Solver-2 without churn: an Euler step to the log-midpoint of sigma and sigma_next, a second
    model call there, and the step from sigma to sigma_next with that call's derivative; plain Euler to sigma = 0."""
    extra_args = extra_args or {}
    s_in = x.new_ones([x.shape[0]])
    for i in range(len(sigmas) - 1):
        sigma_hat = sigmas[i] * (0.0 + 1)
        denoised = model(x, sigma_hat * s_in, **extra_args)
        d = (x - denoised) / _append_dims(sigma_hat, x.ndim)
        if callback is not None:
            callback({"x": x, "i": i, "sigma": sigmas[i], "sigma_hat": sigma_hat, "denoised": denoised})
        if sigmas[i + 1] == 0:
            dt = sigmas[i + 1] - sigma_hat
            x = x + d * dt
        else:
            sigma_mid = sigma_hat.log().lerp(sigmas[i + 1].log(), 0.5).exp()
            dt_1 = sigma_mid - sigma_hat
            dt_2 = sigmas[i + 1] - sigma_hat
            x_2 = x + d * dt_1
            denoised_2 = model(x_2, sigma_mid * s_in, **extra_args)
            d_2 = (x_2 - denoised_2) / _append_dims(sigma_mid, x.ndim)
            x = x + d_2 * dt_2
    return x


@torch.no_grad()
def sample_deis(model, x, sigmas, extra_args=None, callback=None, disable=None, max_order=3, deis_mode="tab"):
    """ComfyUI's DEIS sampler: a multistep update from this step's derivative and the last max_order - 1 ones, with
    the coefficients of `deis.get_deis_coeff_list`; first order on the first step and on the step to sigma = 0.
    As ComfyUI's, its callback sees the sampler's initial x."""
    extra_args = extra_args or {}
    s_in = x.new_ones([x.shape[0]])
    x_next = x
    coeff_list = deis.get_deis_coeff_list(sigmas, max_order, deis_mode=deis_mode)
    buffer_model = []
    for i in range(len(sigmas) - 1):
        t_cur, t_next = sigmas[i], sigmas[i + 1]
        x_cur = x_next
        denoised = model(x_cur, t_cur * s_in, **extra_args)
        if callback is not None:
            callback({"x": x, "i": i, "sigma": sigmas[i], "sigma_hat": sigmas[i], "denoised": denoised})
        d_cur = (x_cur - denoised) / t_cur
        order = min(max_order, i + 1)
        if t_next <= 0:
            order = 1
        if order == 1:
            x_next = x_cur + (t_next - t_cur) * d_cur
        elif order == 2:
            coeff_cur, coeff_prev1 = coeff_list[i]
            x_next = x_cur + coeff_cur * d_cur + coeff_prev1 * buffer_model[-1]
        elif order == 3:
            coeff_cur, coeff_prev1, coeff_prev2 = coeff_list[i]
            x_next = x_cur + coeff_cur * d_cur + coeff_prev1 * buffer_model[-1] + coeff_prev2 * buffer_model[-2]
        else:
            coeff_cur, coeff_prev1, coeff_prev2, coeff_prev3 = coeff_list[i]
            x_next = (x_cur + coeff_cur * d_cur + coeff_prev1 * buffer_model[-1] + coeff_prev2 * buffer_model[-2]
                      + coeff_prev3 * buffer_model[-3])
        if len(buffer_model) == max_order - 1:
            for k in range(max_order - 2):
                buffer_model[k] = buffer_model[k + 1]
            buffer_model[-1] = d_cur.detach()
        else:
            buffer_model.append(d_cur.detach())
    return x_next


def get_ancestral_step(sigma_from, sigma_to, eta=1.0):
    """k-diffusion's get_ancestral_step: (sigma_down, sigma_up) of an ancestral step; (sigma_to, 0.) when eta is 0."""
    if not eta:
        return sigma_to, 0.0
    sigma_up = min(sigma_to, eta * (sigma_to ** 2 * (sigma_from ** 2 - sigma_to ** 2) / sigma_from ** 2) ** 0.5)
    sigma_down = (sigma_to ** 2 - sigma_up ** 2) ** 0.5
    return sigma_down, sigma_up


def default_noise_sampler(x, seed=None):
    """ComfyUI's default_noise_sampler: randn of x's shape from a private generator on x's device, seeded once, when a
    seed is given; from the global generator otherwise."""
    if seed is not None:
        generator = torch.Generator(device=x.device)
        generator.manual_seed(seed)
    else:
        generator = None
    return lambda sigma, sigma_next: torch.randn(x.size(), dtype=x.dtype, layout=x.layout, device=x.device,
                                                 generator=generator)


@torch.no_grad()
def res_multistep(model, x, sigmas, extra_args=None, callback=None, disable=None, s_noise=1.0, noise_sampler=None,
                  eta=1.0):
    """ComfyUI's res_multistep without its cfg_pp branch: RES (arXiv 2308.02157), a second-order exponential multistep
    update from this step's and the previous step's denoised latents, Euler on the first step and on the step to
    sigma_down = 0, and an ancestral draw scaled by sigma_up.

    Written from ComfyUI's comfy/k_diffusion/sampling.py as its author knows it, and not compared with ComfyUI itself,
    which is not a dependency of this project."""
    extra_args = {} if extra_args is None else extra_args
    seed = extra_args.get("seed", None)
    noise_sampler = default_noise_sampler(x, seed=seed) if noise_sampler is None else noise_sampler
    s_in = x.new_ones([x.shape[0]])
    sigma_fn = lambda t: t.neg().exp()              # noqa: E731
    t_fn = lambda sigma: sigma.log().neg()          # noqa: E731
    phi1_fn = lambda t: torch.expm1(t) / t          # noqa: E731
    phi2_fn = lambda t: (phi1_fn(t) - 1.0) / t      # noqa: E731
    old_sigma_down = None
    old_denoised = None
    for i in range(len(sigmas) - 1):
        denoised = model(x, sigmas[i] * s_in, **extra_args)
        sigma_down, sigma_up = get_ancestral_step(sigmas[i], sigmas[i + 1], eta=eta)
        if callback is not None:
            callback({"x": x, "i": i, "sigma": sigmas[i], "sigma_hat": sigmas[i], "denoised": denoised})
        if sigma_down == 0 or old_denoised is None:
            d = (x - denoised) / _append_dims(sigmas[i], x.ndim)
            x = x + d * (sigma_down - sigmas[i])
        else:
            t, t_old, t_next, t_prev = t_fn(sigmas[i]), t_fn(old_sigma_down), t_fn(sigma_down), t_fn(sigmas[i - 1])
            h = t_next - t
            c2 = (t_prev - t_old) / h
            phi1_val, phi2_val = phi1_fn(-h), phi2_fn(-h)
            b1 = torch.nan_to_num(phi1_val - phi2_val / c2, nan=0.0)
            b2 = torch.nan_to_num(phi2_val / c2, nan=0.0)
            x = sigma_fn(h) * x + h * (b1 * denoised + b2 * old_denoised)
        if sigmas[i + 1] > 0:
            x = x + noise_sampler(sigmas[i], sigmas[i + 1]) * s_noise * sigma_up
        old_denoised = denoised
        old_sigma_down = sigma_down
    return x


@torch.no_grad()
def sample_res_multistep(model, x, sigmas, extra_args=None, callback=None, disable=None, s_noise=1.0,
                         noise_sampler=None):
    """ComfyUI's sample_res_multistep: res_multistep with eta = 0 (its draw is multiplied by sigma_up = 0)."""
    return res_multistep(model, x, sigmas, extra_args=extra_args, callback=callback, disable=disable, s_noise=s_noise,
                         noise_sampler=noise_sampler, eta=0.0)


@torch.no_grad()
def sample_gradient_estimation(model, x, sigmas, extra_args=None, callback=None, disable=None, ge_gamma=2.0):
    """ComfyUI's gradient-estimation sampler without its cfg_pp branch: an Euler step corrected, from the second step
    on, by (ge_gamma - 1) times the change of the derivative; the step to sigma = 0 returns the denoised latent.

    Written from ComfyUI's comfy/k_diffusion/sampling.py as its author knows it, and not compared with ComfyUI itself,
    which is not a dependency of this project.  ComfyUI has also shipped an older form (x + (ge_gamma d + (1 - ge_gamma)
    old_d) dt, no x = denoised at sigma = 0); this is the newer one."""
    extra_args = {} if extra_args is None else extra_args
    s_in = x.new_ones([x.shape[0]])
    old_d = None
    for i in range(len(sigmas) - 1):
        denoised = model(x, sigmas[i] * s_in, **extra_args)
        d = (x - denoised) / _append_dims(sigmas[i], x.ndim)
        if callback is not None:
            callback({"x": x, "i": i, "sigma": sigmas[i], "sigma_hat": sigmas[i], "denoised": denoised})
        dt = sigmas[i + 1] - sigmas[i]
        if sigmas[i + 1] == 0:
            x = denoised
        else:
            x = x + d * dt
            if i >= 1:
                d_bar = (ge_gamma - 1) * (d - old_d)
                x = x + d_bar * dt
        old_d = d
    return x


_SAMPLER_FUNCTIONS = {"euler": sample_euler, "heun": sample_heun, "euler_ancestral": sample_euler_ancestral,
                      "dpmpp_2m": sample_dpmpp_2m, "dpm_2": sample_dpm_2, "deis": sample_deis,
                      "res_multistep": sample_res_multistep, "gradient_estimation": sample_gradient_estimation}
# ComfyUI's KSampler takes one step more for these and drops the penultimate sigma (the samplers minicomfy has)
DISCARD_PENULTIMATE_SIGMA_SAMPLERS = {"dpm_2"}


class KSAMPLER:
    def __init__(self, sampler_function, extra_options=None, inpaint_options=None):
        self.sampler_function = sampler_function
        self.extra_options = extra_options or {}
        self.inpaint_options = inpaint_options or {}

    def max_denoise(self, model_wrap, sigmas):
        max_sigma = float(model_wrap.inner_model.model_sampling.sigma_max)
        sigma = float(sigmas[0])
        return math.isclose(max_sigma, sigma, rel_tol=1e-05) or sigma > max_sigma

    def sample(self, model_wrap, sigmas, extra_args, callback, noise, latent_image=None, denoise_mask=None,
               disable_pbar=False):
        extra_args["denoise_mask"] = denoise_mask
        model_k = KSamplerX0Inpaint(model_wrap, sigmas)
        model_k.latent_image = latent_image
        model_k.noise = noise
        noise = model_wrap.inner_model.model_sampling.noise_scaling(sigmas[0], noise, latent_image,
                                                                    self.max_denoise(model_wrap, sigmas))
        k_callback = None
        total_steps = len(sigmas) - 1
        if callback is not None:
            k_callback = lambda x: callback(x["i"], x["denoised"], x["x"], total_steps)
        samples = self.sampler_function(model_k, noise, sigmas, extra_args=extra_args, callback=k_callback,
                                        disable=disable_pbar, **self.extra_options)
        return model_wrap.inner_model.model_sampling.inverse_noise_scaling(sigmas[-1], samples)


def ksampler(sampler_name, extra_options=None, inpaint_options=None):
    fn = _SAMPLER_FUNCTIONS.get(sampler_name)
    if fn is None:
        raise NotImplementedError(f"minicomfy has no sampler {sampler_name!r} (only {sorted(_SAMPLER_FUNCTIONS)})")
    return KSAMPLER(fn, extra_options, inpaint_options)


def sampler_object(name):
    return ksampler(name)


class CFGGuider:
    def __init__(self, model_patcher):
        self.model_patcher = model_patcher
        self.model_options = model_patcher.model_options
        self.original_conds = {}
        self.conds = {}
        self.cfg = 1.0

    def set_conds(self, positive, negative):
        self.conds = {"positive": positive, "negative": negative}
        self.original_conds = dict(self.conds)

    def set_cfg(self, cfg):
        self.cfg = cfg

    def __call__(self, *args, **kwargs):
        return self.predict_noise(*args, **kwargs)

    def predict_noise(self, x, timestep, model_options={}, seed=None):
        return sampling_function(self.inner_model, x, timestep, self.conds.get("negative"), self.conds.get("positive"),
                                 self.cfg, model_options=model_options, seed=seed)

    def inner_sample(self, noise, latent_image, device, sampler, sigmas, denoise_mask, callback, disable_pbar, seed,
                     latent_shapes=None):
        extra_args = {"model_options": dict(self.model_options), "seed": seed}
        return sampler.sample(self, sigmas, extra_args, callback, noise, latent_image, denoise_mask, disable_pbar)

    def outer_sample(self, noise, latent_image, sampler, sigmas, denoise_mask=None, callback=None, disable_pbar=False,
                     seed=None, latent_shapes=None):
        self.inner_model, self.conds, self.loaded_models = prepare_sampling(self.model_patcher, noise.shape, self.conds,
                                                                            self.model_options)
        device = self.model_patcher.load_device
        if denoise_mask is not None:
            denoise_mask = sys.modules["comfy.sampler_helpers"].prepare_mask(denoise_mask, noise.shape, device)
        noise, latent_image, sigmas = noise.to(device), latent_image.to(device), sigmas.to(device)
        try:
            self.model_patcher.pre_run()
            output = self.inner_sample(noise, latent_image, device, sampler, sigmas, denoise_mask, callback,
                                       disable_pbar, seed)
        finally:
            self.model_patcher.cleanup()
        del self.inner_model
        del self.loaded_models
        return output

    def sample(self, noise, latent_image, sampler, sigmas, denoise_mask=None, callback=None, disable_pbar=False,
               seed=None):
        if sigmas.shape[-1] == 0:
            return latent_image
        self.conds = dict(self.original_conds)
        # class-level lookup so that a patched CFGGuider.outer_sample is honoured
        output = type(self).outer_sample(self, noise, latent_image, sampler, sigmas, denoise_mask, callback,
                                         disable_pbar, seed)
        return output.to(intermediate_device())


def get_sigmas_karras(n, sigma_min, sigma_max, rho=7.0, device="cpu"):
    ramp = torch.linspace(0, 1, n, device=device)
    lo, hi = sigma_min ** (1 / rho), sigma_max ** (1 / rho)
    s = (hi + ramp * (lo - hi)) ** rho
    return torch.cat([s, s.new_zeros([1])])


def simple_scheduler(model_sampling, steps):
    """comfy.samplers.simple_scheduler: every (len/steps)-th entry of the model's sigma table, from the top."""
    table = getattr(model_sampling, "sigmas", None)
    if table is None:   # EPS stand-in has no table: log-spaced between its extremes
        hi, lo = float(model_sampling.sigma_max), max(float(model_sampling.sigma_min), 1e-3)
        s = torch.exp(torch.linspace(math.log(hi), math.log(lo), steps))
        return torch.cat([s, s.new_zeros([1])])
    ss = len(table) / steps
    sigs = [float(table[-(1 + int(x * ss))]) for x in range(steps)] + [0.0]
    return torch.FloatTensor(sigs)


class KSampler:
    SCHEDULERS = ["simple", "sgm_uniform", "karras", "exponential", "ddim_uniform", "beta", "normal",
                  "linear_quadratic", "kl_optimal"]
    SAMPLERS = sorted(_SAMPLER_FUNCTIONS)

    def __init__(self, model, steps, device, sampler=None, scheduler=None, denoise=None, model_options={}):
        self.model = model
        self.device = device
        self.scheduler = scheduler
        self.sampler = sampler
        self.model_options = model_options
        ms = model.model.model_sampling
        discard = sampler in DISCARD_PENULTIMATE_SIGMA_SAMPLERS
        n = steps + 1 if discard else steps
        if scheduler == "karras":
            self.sigmas = get_sigmas_karras(n, float(ms.sigma_min), float(ms.sigma_max))
        else:
            self.sigmas = simple_scheduler(ms, n)
        if discard:
            self.sigmas = torch.cat([self.sigmas[:-2], self.sigmas[-1:]])
        if denoise is not None and denoise < 0.9999 and denoise > 0.0:
            new_steps = int(steps / denoise)
            full = KSampler(model, new_steps, device, sampler, scheduler, None, model_options).sigmas
            self.sigmas = full[-(steps + 1):]

    def sample(self, noise, positive, negative, cfg, latent_image=None, start_step=None, last_step=None,
               force_full_denoise=False, denoise_mask=None, sigmas=None, callback=None, disable_pbar=False, seed=None):
        sigmas = self.sigmas if sigmas is None else sigmas
        if last_step is not None and last_step < (len(sigmas) - 1):
            sigmas = sigmas[:last_step + 1]
            if force_full_denoise:
                sigmas = sigmas.clone()
                sigmas[-1] = 0
        if start_step is not None:
            if start_step < (len(sigmas) - 1):
                sigmas = sigmas[start_step:]
            else:
                return latent_image if latent_image is not None else torch.zeros_like(noise)
        guider = CFGGuider(self.model)
        guider.set_conds(positive, negative)
        guider.set_cfg(cfg)
        return guider.sample(noise, latent_image, ksampler(self.sampler), sigmas, denoise_mask, callback, disable_pbar,
                             seed)


# ------------------------------------------------------------------ comfy.sample / nodes / latent_preview
def prepare_noise(latent_image, seed, noise_inds=None):
    generator = torch.manual_seed(seed)
    return torch.randn(latent_image.size(), dtype=latent_image.dtype, layout=latent_image.layout,
                       generator=generator, device="cpu")


def fix_empty_latent_channels(model, latent_image):
    return latent_image


def sample(model, noise, steps, cfg, sampler_name, scheduler, positive, negative, latent_image, denoise=1.0,
           disable_noise=False, start_step=None, last_step=None, force_full_denoise=False, noise_mask=None,
           sigmas=None, callback=None, disable_pbar=False, seed=None):
    sampler = KSampler(model, steps=steps, device=model.load_device, sampler=sampler_name, scheduler=scheduler,
                       denoise=denoise, model_options=model.model_options)
    samples = sampler.sample(noise, positive, negative, cfg=cfg, latent_image=latent_image, start_step=start_step,
                             last_step=last_step, force_full_denoise=force_full_denoise, denoise_mask=noise_mask,
                             sigmas=sigmas, callback=callback, disable_pbar=disable_pbar, seed=seed)
    return samples.to(intermediate_device())


def sample_custom(model, noise, cfg, sampler, sigmas, positive, negative, latent_image, noise_mask=None, callback=None,
                  disable_pbar=False, seed=None):
    guider = CFGGuider(model)
    guider.set_conds(positive, negative)
    guider.set_cfg(cfg)
    return guider.sample(noise, latent_image, sampler, sigmas, noise_mask, callback, disable_pbar, seed).to(
        intermediate_device())


def common_ksampler(model, seed, steps, cfg, sampler_name, scheduler, positive, negative, latent, denoise=1.0,
                    disable_noise=False, start_step=None, last_step=None, force_full_denoise=False):
    latent_image = latent["samples"]
    if disable_noise:
        noise = torch.zeros(latent_image.size(), dtype=latent_image.dtype, layout=latent_image.layout, device="cpu")
    else:
        # through the module, like ComfyUI's nodes.py (`comfy.sample.prepare_noise(...)`): a patched one is honoured
        noise = sys.modules["comfy.sample"].prepare_noise(latent_image, seed, latent.get("batch_index"))
    noise_mask = latent.get("noise_mask")
    # like ComfyUI: there is always a callback (progress bar; a preview only when a previewer is configured)
    callback = sys.modules["latent_preview"].prepare_callback(model, steps)
    samples = sample(model, noise, steps, cfg, sampler_name, scheduler, positive, negative, latent_image,
                     denoise=denoise, disable_noise=disable_noise, start_step=start_step, last_step=last_step,
                     force_full_denoise=force_full_denoise, noise_mask=noise_mask, callback=callback,
                     disable_pbar=not PROGRESS_BAR_ENABLED, seed=seed)
    out = latent.copy()
    out["samples"] = samples
    return (out,)


PROGRESS = {"calls": 0, "last": None}
PREVIEW = {"previewer": None}     # what get_previewer returns (ComfyUI: per the --preview-method setting)


class Latent2RGBPreviewer:
    """ComfyUI's latent-to-RGB previewer, as far as a caller can observe it: it decodes the first request's latent,
    x0[:1], here kept as a device copy per call."""

    def __init__(self):
        self.seen = []

    def decode_latent_to_preview_image(self, preview_format, x0):
        self.seen.append(x0[:1].clone())
        return None


def get_previewer(device=None, latent_format=None):
    return PREVIEW["previewer"]


def prepare_callback(model, steps, x0_output_dict=None):
    """ComfyUI's latent_preview.prepare_callback: keeps the latest x0 for the custom-sampler nodes, hands it to the
    previewer when one is configured (none by default) and advances the progress bar."""
    previewer = get_previewer()

    def callback(step, x0, x, total_steps):
        if x0_output_dict is not None:
            x0_output_dict["x0"] = x0
        if previewer:
            previewer.decode_latent_to_preview_image("JPEG", x0)
        PROGRESS["calls"] += 1
        PROGRESS["last"] = (step + 1, total_steps)
    return callback


# ------------------------------------------------------------------ registration
_MODULES = ("comfy", "comfy.utils", "comfy.samplers", "comfy.sampler_helpers", "comfy.model_base", "comfy.sample",
            "comfy.model_management", "nodes", "latent_preview", "comfyui_version")


def is_installed() -> bool:
    m = sys.modules.get("comfy")
    return bool(m is not None and getattr(m, "__minicomfy__", False))


def install(version: str = "0.6.0") -> None:
    """Register the stand-in modules.  Idempotent; never shadows a real ComfyUI."""
    if is_installed():
        return
    existing = sys.modules.get("comfy")
    if existing is not None and getattr(existing, "__file__", None):
        raise RuntimeError("a real ComfyUI is importable; minicomfy will not shadow it")
    me = sys.modules[__name__]

    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__minicomfy__ = True
        for k, v in attrs.items():
            setattr(m, k, v)
        sys.modules[name] = m
        return m

    comfy = mod("comfy")
    comfy.__path__ = []
    comfy.utils = mod("comfy.utils", repeat_to_batch_size=repeat_to_batch_size, PROGRESS_BAR_ENABLED=False)
    samplers_all = ["calc_cond_batch", "cfg_function", "cast_to_load_options", "sampling_function", "CFGGuider",
                    "KSAMPLER", "KSampler", "ksampler", "sampler_object", "KSamplerX0Inpaint", "sample_euler", "sample_heun",
                    "sample_euler_ancestral"]
    comfy.samplers = mod("comfy.samplers", **{k: getattr(me, k) for k in samplers_all}, __all__=samplers_all)
    comfy.sampler_helpers = mod("comfy.sampler_helpers", prepare_mask=prepare_mask, prepare_sampling=prepare_sampling,
                                cleanup_models=cleanup_models)
    comfy.model_base = mod("comfy.model_base", ModelType=ModelType, BaseModel=BaseModel, WAN22=WAN22)
    comfy.sample = mod("comfy.sample", sample=sample, sample_custom=sample_custom, prepare_noise=prepare_noise,
                       fix_empty_latent_channels=fix_empty_latent_channels)
    comfy.model_management = mod("comfy.model_management", intermediate_device=intermediate_device)
    mod("nodes", common_ksampler=common_ksampler)
    mod("latent_preview", prepare_callback=prepare_callback, get_previewer=get_previewer,
        Latent2RGBPreviewer=Latent2RGBPreviewer)
    mod("comfyui_version", __version__=version)


def uninstall() -> None:
    if is_installed():
        for n in _MODULES:
            sys.modules.pop(n, None)
