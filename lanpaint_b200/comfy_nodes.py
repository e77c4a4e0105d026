"""ComfyUI node surface of LanPaint, backed by the H100 (sm_90a) engine.

What is kept byte-identical to the reference (SURVEY 8b/b1, checked by
tests/test_nodes_api.py against a dump of the reference's own classes):
node class names, INPUT_TYPES (order, types, defaults, ranges, tooltips,
hidden retired widgets), RETURN_TYPES / RETURN_NAMES / FUNCTION / CATEGORY,
NODE_CLASS_MAPPINGS keys and display names of the four sampler nodes
(src/LanPaint/nodes.py:452-589,659-808,1347-1378), the hyper-parameter
attributes hung on the ModelPatcher (nodes.py:492-504), the four functions
patched for the duration of one sample call and their restore-on-exception
(nodes.py:384-421), the LATENT dict contract.

What is different: the per-sigma wrapper computes the schedule on the host
from ONE read-back of sigma (the reference syncs twice per outer step plus
once per sub-step), caches the packed mask across outer steps, and calls the
fused engine (`lanpaint_b200.engine.LanPaint`).  Around the sampler loop, two
costs that dwarf it at large batches are taken over as well: the result goes
back to the host through pinned memory (`_host_result`), and -- when this
host's torch.randn was verified to draw the same bits -- ComfyUI's CPU noise
image (`comfy.sample.prepare_noise`) is drawn on the device (`hostnoise.py`; a
fifth, optional swap in `override_sample_function`).  Only the four sampler
nodes exist here: mask/video/audio tooling is outside the hot path (SURVEY 2).
"""
from __future__ import annotations

import math
import sys
from contextlib import contextmanager

import torch

import comfy  # noqa: F401  (ComfyUI, or minicomfy in tests)
import comfy.samplers
import comfy.utils
import latent_preview
import nodes as comfy_nodes_module
from comfy.model_base import ModelType

# Used only while a node samples (as `comfy.<module>.<function>`, like the reference does).  Tooling that merely
# introspects the node classes (ComfyUI's node-diff CI, the reference's own tests) stubs just the modules above
# (reference __init__.py:14-87), so their absence must not break the import.
for _name in ("comfy.model_management", "comfy.sample", "comfy.sampler_helpers"):
    try:
        __import__(_name)
    except ImportError:
        pass

try:  # WAN22 exists only in recent ComfyUI builds
    from comfy.model_base import WAN22
except Exception:  # pragma: no cover
    WAN22 = None

try:  # MiniMax-H3 schedule helpers: present only in ComfyUI builds that ship the model
    from comfy.ldm.minimax.model import time_shift_sigma, time_shift_slope
except Exception:
    time_shift_sigma = None
    time_shift_slope = None

from .engine import CfgPair, LanPaint, _IdentityCache, pack_mask
from .schedule import effective_inner_steps, min_step_frac_effective_steps, times_from_sigma  # noqa: F401

FLOW_MODEL_TYPES = (ModelType.FLOW, getattr(ModelType, "FLOW_AV", None))

IMAGE_MODE, VIDEO_MODE = "🖼️ Image Inpainting", "🎬 Video Inpainting"
PROMPT_MODES = ("Image First", "Prompt First")
_STAR = ("For more info, visit https://github.com/scraed/LanPaint. "
         "If you find it useful, please give a star ⭐️!")

KSAMPLER_NAMES = ["euler", "euler_ancestral", "heun", "heunpp2", "dpm_2", "dpm_2_ancestral",
                  "dpm_fast", "dpmpp_sde", "dpmpp_sde_gpu",
                  "dpmpp_2m", "dpmpp_2m_sde", "dpmpp_2m_sde_gpu", "dpmpp_3m_sde", "dpmpp_3m_sde_gpu", "ddpm",
                  "deis", "res_multistep", "res_multistep_ancestral",
                  "gradient_estimation", "er_sde", "seeds_2", "seeds_3"]

# retired widgets old workflows still send; accepted and ignored (nodes.py:472-477,538-548)
_RETIRED_ALL = ("LanPaint_Beta", "LanPaint_Friction", "LanPaint_EarlyStop", "LanPaint_InnerThreshold",
                "LanPaint_InnerPatience", "LanPaint_MinStepFrac")


def _detect_minimax_h3_audio(model_patcher, model_options, latent_shapes):
    """A MiniMax-H3 AV pack is a nested (video, audio) latent whose diffusion model carries
    sigma_shift_video / sigma_shift_audio (nodes.py:34-52).  Returns (latent_shapes, shift_v, shift_a) or None;
    `transformer_options` may override the shifts."""
    if latent_shapes is None or len(latent_shapes) < 2:
        return None
    diff_model = getattr(getattr(model_patcher, "model", None), "diffusion_model", None)
    shift_v = getattr(diff_model, "sigma_shift_video", None)
    shift_a = getattr(diff_model, "sigma_shift_audio", None)
    if shift_v is None or shift_a is None:
        return None
    topts = model_options.get("transformer_options", {}) if isinstance(model_options, dict) else {}
    shift_v = topts.get("minimax_h3_sigma_shift_video", shift_v)
    shift_a = topts.get("minimax_h3_sigma_shift_audio", shift_a)
    return (latent_shapes, float(shift_v), float(shift_a))


def _hidden(names):
    return {n: "DEFAULT" for n in names}


# ---- widget specs shared between nodes ------------------------------------------------------
def _w_num_steps(tip):
    return ("INT", {"default": 5, "min": 0, "max": 100, "tooltip": tip})


def _w_prompt_mode(tip):
    return (list(PROMPT_MODES), {"tooltip": tip})


def _w_info(default):
    return ("STRING", {"default": default, "tooltip": _STAR})


def _w_mode():
    return ([IMAGE_MODE, VIDEO_MODE], {"default": IMAGE_MODE, "tooltip": "Choose Image mode for photos or Video mode for video frames with temporal consistency"})


_TIP_STEPS_K = "The number of steps for the Langevin dynamics, representing the turns of thinking per step."
_TIP_STEPS_C = "Number of steps for Langevin dynamics, representing turns of thinking per step."
_TIP_MODE_K = "Image First: emphasis image quality, Prompt First: emphasis prompt following"
_TIP_MODE_C = "Image First: prioritizes image quality; Prompt First: prioritizes prompt adherence."


def _sanitize_param(value, default, allowed=None):
    """Bad widget values fall back to the default instead of raising (nodes.py:146-157)."""
    if allowed is not None:
        return value if value in allowed else default
    if isinstance(value, bool) or not isinstance(value, (int, float)):
        return default
    return value


def _set_hyper(patcher, *, num_steps, cfg, prompt_mode, lam=5.0, step_size=0.2):
    """The attribute protocol between the nodes and KSAMPLER.sample (nodes.py:492-504 -> :351-364)."""
    patcher.LanPaint_StepSize = step_size
    patcher.LanPaint_Lambda = lam
    patcher.LanPaint_Beta = 1.0
    patcher.LanPaint_NumSteps = num_steps
    patcher.LanPaint_MinStepFrac = 1.0
    patcher.LanPaint_Friction = 15.0
    patcher.LanPaint_EarlyStop = 1
    patcher.LanPaint_InnerThreshold = 0.0
    patcher.LanPaint_InnerPatience = 1
    patcher.LanPaint_cfg_BIG = cfg if prompt_mode == "Image First" else 0 * cfg - 0.5


# =============================================================================================
# mask preparation (runs once per sample; plain torch)
# =============================================================================================
def reshape_mask(input_mask, output_shape, video_inpainting=False):
    """noise_mask of any accepted rank -> latent shape (nodes.py:59-133): nearest-exact resize;
    video masks additionally take the union over a 5-slice temporal window."""
    import torch.nn.functional as F
    spatial_rank = len(output_shape) - 2
    m = input_mask
    if video_inpainting:
        if m.ndim == 2:
            m = m[None, None, None]
        elif m.ndim == 3:
            m = m[None, None]
        elif m.ndim == 4:
            m = m.permute(1, 0, 2, 3)[None]
    elif m.ndim == 1 and len(output_shape) == 4:
        t = output_shape[-1]
        m = F.interpolate(m.float()[None, None], size=(t,), mode="nearest-exact").expand(1, 1, output_shape[-2], t)
    elif m.ndim == 4 and len(output_shape) == 4 and m.shape[1] == 1 and m.shape[3] == 1:
        t = output_shape[-1]
        m = F.interpolate(m, size=(t, 1), mode="nearest-exact").permute(0, 1, 3, 2).expand(1, 1, output_shape[-2], t)
    elif m.ndim == 2:
        m = m[None, None]
    elif m.ndim == 3:
        m = m[:, None]
    if len(output_shape) == 5 and m.ndim == 4:
        m = m.unsqueeze(2)

    if video_inpainting:
        m = F.interpolate(m, size=(output_shape[2], output_shape[-2], output_shape[-1]), mode="nearest-exact")
        m = F.max_pool3d(m, kernel_size=(5, 1, 1), stride=(1, 1, 1), padding=(2, 0, 0))
        if m.shape[1] < output_shape[1]:
            m = m.repeat(1, output_shape[1], 1, 1, 1)[:, :output_shape[1]]
        return comfy.utils.repeat_to_batch_size(m, output_shape[0])
    m = F.interpolate(m, size=tuple(output_shape[2:]), mode="nearest-exact")
    if m.shape[1] < output_shape[1]:
        m = m.repeat((1, output_shape[1]) + (1,) * spatial_rank)[:, :output_shape[1]]
    return comfy.utils.repeat_to_batch_size(m, output_shape[0])


def prepare_mask(noise_mask, shape, device, video_inpainting=False):
    """Same values and shape as the reference's prepare_mask (nodes.py:119-130).  Two savings on the way to the
    device: a mask with a single channel stays single-channel across PCIe and is *expanded* (stride 0) over the
    latent's channels instead of repeated (1/C of the bytes; `_latent_mask` then sees without a device read-back
    that one uint8 per spatial site is enough), and a mask that already has the latent's spatial size (nothing to
    resample) travels in its own dtype -- uint8 / bool masks as one byte per site -- and is widened on the device."""
    m = noise_mask
    one_channel = m.ndim <= 3 or m.shape[1] == 1
    no_resample = (not video_inpainting) and m.ndim >= 2 and tuple(m.shape[-(len(shape) - 2):]) == tuple(shape[2:]) \
        and m.ndim in (len(shape) - 2, len(shape) - 1, len(shape))
    if no_resample:
        m = m.to(device)
        if not m.is_floating_point():
            m = m.float()
    if one_channel and len(shape) >= 3 and shape[1] > 1:
        compact = reshape_mask(m, (shape[0], 1) + tuple(shape[2:]), video_inpainting).to(device)
        return compact.expand(tuple(shape))
    return reshape_mask(m, shape, video_inpainting).to(device)


# =============================================================================================
# patch layer (nodes.py:161-421)
# =============================================================================================
def sampling_function_LanPaint(model, x, timestep, uncond, cond, cond_scale, cond_scale_BIG, model_options={},
                               seed=None):
    """One batched cond/uncond evaluation, two CFG combines -> (x0 at cfg, x0 at cfg_BIG)."""
    skip_uncond = math.isclose(cond_scale, 1.0) and not model_options.get("disable_cfg1_optimization", False)
    uncond_ = None if skip_uncond else uncond
    conds = [cond, uncond_]
    out = comfy.samplers.calc_cond_batch(model, conds, x, timestep, model_options)
    for fn in model_options.get("sampler_pre_cfg_function", []):
        out = fn({"conds": conds, "conds_out": out, "cond_scale": cond_scale, "timestep": timestep, "input": x,
                  "sigma": timestep, "model": model, "model_options": model_options})
    opts = model_options.get("lanpaint_b200", {}) if isinstance(model_options, dict) else {}
    plain_cfg = ("sampler_cfg_function" not in model_options and not model_options.get("sampler_post_cfg_function")
                 and uncond_ is not None and isinstance(out[0], torch.Tensor) and isinstance(out[1], torch.Tensor))
    if plain_cfg and opts.get("fused_cfg", True):
        # nothing needs the combined tensors materialised: hand cond/uncond to the fused kernel (SURVEY 8f rank 1)
        return CfgPair(out[0], out[1], cond_scale, cond_scale_BIG)
    combine = comfy.samplers.cfg_function
    return (combine(model, out[0], out[1], cond_scale, x, timestep, model_options=model_options, cond=cond, uncond=uncond_),
            combine(model, out[0], out[1], cond_scale_BIG, x, timestep, model_options=model_options, cond=cond, uncond=uncond_))


def _host_result(t, opts=None):
    """Device -> host copy of a sampler result into a PINNED tensor from PyTorch's caching host allocator.

    ComfyUI ends every sample call with `samples.to(intermediate_device())`: a copy into a freshly allocated pageable
    tensor, whose first-touch page faults and staged DMA make it several times slower than a copy into pinned memory
    (for a 33.5 MB latent batch, longer than the whole sampler loop).  A pinned destination takes the same bytes at the
    link's rate, and the allocator recycles the block once the caller drops the result, so steady state allocates nothing.  The
    tensor handed back is an ordinary CPU tensor: ComfyUI's own `.to(cpu)` on it is then a no-op.  Left alone: results
    that are not on a CUDA device, hosts whose intermediate device is not the CPU (--gpu-only), sizes outside
    [64 KiB, 1 GiB], `{"pinned_result": False}`."""
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.is_nested:
        return t
    if opts is not None and not opts.get("pinned_result", True):
        return t
    try:
        if comfy.model_management.intermediate_device().type != "cpu":
            return t
    except AttributeError:      # a partial ComfyUI (tooling stubs): nothing to decide with
        return t
    nbytes = t.numel() * t.element_size()
    if nbytes < (64 << 10) or nbytes > (1 << 30):
        return t
    src = t if t.is_contiguous() else t.contiguous()
    try:
        host = torch.empty(src.shape, dtype=src.dtype, device="cpu", pin_memory=True)
    except RuntimeError:        # pinned memory exhausted / not permitted: ComfyUI's own copy still works
        return t
    host.copy_(src, non_blocking=True)
    torch.cuda.current_stream(src.device).synchronize()
    return host


class CFGGuider_LanPaint:
    """Methods grafted onto comfy.samplers.CFGGuider while a LanPaint node samples."""

    def outer_sample(self, noise, latent_image, sampler, sigmas, denoise_mask=None, callback=None, disable_pbar=False,
                     seed=None, **kwargs):
        self.inner_model, self.conds, self.loaded_models = comfy.sampler_helpers.prepare_sampling(
            self.model_patcher, noise.shape, self.conds, self.model_options)
        device = self.model_patcher.load_device
        if WAN22 is not None and isinstance(self.inner_model, WAN22):
            self.inner_model.extra_conds = super(WAN22, self.inner_model).extra_conds
        # MiniMax-H3 AV packs carry an audio stream on a shifted sigma schedule (nodes.py:188-191)
        self.minimax_h3_audio = _detect_minimax_h3_audio(self.model_patcher, self.model_options,
                                                         kwargs.get("latent_shapes", None))
        if denoise_mask is not None and tuple(denoise_mask.shape) != tuple(noise.shape):
            denoise_mask = prepare_mask(denoise_mask, noise.shape, device,
                                        self.model_options.get("video_inpainting", False))
        noise = noise.to(device)
        latent_image = latent_image.to(device)
        sigmas_host = sigmas.detach().to("cpu", torch.float32)  # schedule stays host-visible: no argmin sync later
        sigmas = sigmas.to(device)
        sigmas._lanpaint_host = sigmas_host
        comfy.samplers.cast_to_load_options(self.model_options, device=device, dtype=self.model_patcher.model_dtype())
        try:
            self.model_patcher.pre_run()
            output = self.inner_sample(noise, latent_image, device, sampler, sigmas, denoise_mask, callback,
                                       disable_pbar, seed, **kwargs)
        finally:
            self.model_patcher.cleanup()
        comfy.sampler_helpers.cleanup_models(self.conds, self.loaded_models)
        del self.inner_model
        del self.loaded_models
        # what ComfyUI does next with `output` is a device -> host copy: do it here through pinned memory
        return _host_result(output, (self.model_options or {}).get("lanpaint_b200"))

    def predict_noise(self, x, timestep, model_options={}, seed=None):
        return sampling_function_LanPaint(self.inner_model, x, timestep, self.conds.get("negative", None),
                                          self.conds.get("positive", None), self.cfg, self.cfg_BIG,
                                          model_options=model_options, seed=seed)


class KSamplerX0Inpaint:
    """Per-sigma wrapper the k-diffusion sampler calls once per model evaluation
    (nodes.py:221-315): returns the denoised latent, rewrites x in place."""

    def __init__(self, model, sigmas):
        self.inner_model = model
        self.sigmas = sigmas
        host = getattr(sigmas, "_lanpaint_host", None)
        self.sigmas_host = [float(v) for v in (host if host is not None else sigmas.detach().cpu())]
        self.audio_indicator = None
        self.audio_shifts = None
        self._mask_cache = _IdentityCache()
        self.trace = None          # list: record (sigma, times, n_eff) of every call (runner.SamplerGraphJob)
        self.planned_call = None   # set while a whole sampler loop is being captured: serves the recorded calls
        self.rng_delta = 0         # CUDA generator offset consumed by the engine calls (vs. by the sampler itself)

    def _latent_mask(self, denoise_mask, like):
        """1 - (denoise_mask > 0.5), packed once per distinct mask tensor (nodes.py:281-283)."""
        packed = self._mask_cache.get(denoise_mask)
        if packed is None:
            m = denoise_mask
            if m.ndim == like.ndim and m.shape[1] > 1 and m.stride(1) == 0:
                m = m[:, :1]          # our prepare_mask: one spatial mask expanded over the channels
            known = m <= 0.5
            # a mask some other node materialised per channel: check once whether the channels agree (one
            # read-back per distinct mask tensor, not per outer step) and keep 1/C byte per latent element
            if known.ndim == like.ndim and known.shape[1] > 1 and bool((known == known[:, :1]).all()):
                known = known[:, :1]
            packed = pack_mask(known, like)
            self._mask_cache.put(denoise_mask, packed)
        return packed

    def __call__(self, x, sigma, denoise_mask, model_options={}, seed=None, **kwargs):
        mtype = self.inner_model.inner_model.model_type
        is_flux = mtype == ModelType.FLUX
        is_flow = mtype in FLOW_MODEL_TYPES
        if denoise_mask is not None and self.planned_call is not None:
            return self.planned_call(x, model_options, seed)     # capture of the whole sampler loop: nothing is read back
        if denoise_mask is None:
            out, _ = self.PaintMethod.unpack_model_output(
                self.inner_model(x, sigma, model_options=model_options, seed=seed))
        else:
            if "denoise_mask_function" in model_options:
                denoise_mask = model_options["denoise_mask_function"](
                    sigma, denoise_mask, extra_options={"model": self.inner_model, "sigmas": self.sigmas})
            sigma_host = sigma.detach().to("cpu", torch.float32)  # the one read-back of this outer step
            times = times_from_sigma(sigma_host, is_flux or is_flow)  # reference op order, fp32 (nodes.py:242-252)
            n_eff = effective_inner_steps(self.PaintMethod.n_steps, self.sigmas_host, float(sigma_host.mean()),
                                          float((1.0 - times[1]).mean()), self.LanPaint_early_stop,
                                          getattr(self, "LanPaint_min_step_frac", 1.0))
            audio = {}
            if self.audio_indicator is not None and self.audio_shifts is not None and time_shift_sigma is not None:
                # the audio rows run on sigma_audio = time_shift_sigma(sigma_video, shift_v, shift_a) and the
                # flat-grid target overshoots them by sigma_v*slope/sigma_a (nodes.py:254-275)
                shift_v, shift_a = self.audio_shifts
                flow_v = times[2]
                flow_a = time_shift_sigma(flow_v, shift_v, shift_a)
                abt_a = (1 - flow_a) ** 2 / ((1 - flow_a) ** 2 + flow_a ** 2)
                c = 1.0
                ft = float(flow_v)
                if ft > 1e-4 and time_shift_slope is not None:
                    c = float(flow_a) / (ft * float(time_shift_slope(flow_v, shift_v, shift_a)))
                audio = dict(current_times_audio=(flow_a / (1 - flow_a), abt_a, flow_a),
                             audio_indicator=self.audio_indicator,
                             audio_correction=(1.0 - self.audio_indicator) + c * self.audio_indicator)
            if self.trace is not None:
                self.trace.append((sigma_host.clone(), tuple(t.clone() for t in times), n_eff))
            gen = torch.cuda.default_generators[x.device.index if x.device.index is not None else torch.cuda.current_device()]
            before = gen.get_offset()
            out = self.PaintMethod(x, self.latent_image, self.noise, sigma_host,
                                   self._latent_mask(denoise_mask, x), times, model_options, seed, n_steps=n_eff,
                                   **audio)
            self.rng_delta += gen.get_offset() - before
        step = model_options.get("i", kwargs.get("i", 0))
        if step % 2 == 0:  # preview every other step (nodes.py:304-313)
            callback = model_options.get("callback", None)
            if callback is not None:
                callback({"i": step, "denoised": out, "x": x})
        return out


class KSAMPLER(comfy.samplers.KSAMPLER):
    """KSAMPLER.sample replacement (nodes.py:318-379): builds the per-sigma wrapper and the engine.

    Three launch strategies behind the same call:
      * the sampler is plain Euler (what the node recommends) and nothing needs host code inside an outer
        step: the whole sampler loop is run by `runner.GraphedJob` -- host-computed schedule, Euler update and
        next replace step fused into the step-boundary kernel, CUDA graphs (one per job, or one per outer step
        with ComfyUI's callback between them when the job is long enough to watch) cached across sample() calls;
        with the option "fused_ancestral" the same holds for euler_ancestral, whose step and randn_like draw
        run inside lp_boundary_ancestral; dpmpp_2m runs there too (on by default), its update and the previous
        step's denoised latent inside lp_boundary_multistep, and so does dpm_2 (on by default), both of its wrapper
        calls per step in the loop and both of its updates inside lp_boundary_midpoint, deis (on by default),
        its third-order update and the derivatives of the two previous steps inside lp_boundary_deis,
        res_multistep (on by default when extra_args has a seed), its second-order step inside lp_boundary_multistep
        and its Euler steps inside lp_boundary_midpoint, and gradient_estimation (on by default), its update and
        the previous step's derivative inside lp_boundary_gradient_estimation; each of the last two only when a
        check of the sampler function on a tiny CPU problem shows the form the loop restates; with the option
        "fused_heun" (and the same check) heun runs there too, both of its wrapper calls per step in the loop, its
        predictor inside lp_boundary_midpoint and its corrector inside lp_boundary_heun;
      * any other deterministic sampler: the first job records which sigmas the sampler hands the wrapper, then
        k-diffusion's sampler function itself is captured into ONE graph (`runner.SamplerGraphJob`);
      * anything else (samplers that draw their own noise, early stop, AV packs, mask schedules): k-diffusion's own
        loop calls the per-sigma wrapper, which replays one CUDA graph per outer step.
    In every case the first job of a configuration launches eagerly and the graphs are captured when the same
    configuration comes back, so no model evaluation is ever spent on a warm-up pass."""

    def sample(self, model_wrap, sigmas, extra_args, callback, noise, latent_image=None, denoise_mask=None,
               disable_pbar=False):
        # NB: while the patch is active this function is installed on comfy.samplers.KSAMPLER itself, so `self`
        # is ComfyUI's class, not this subclass: helpers are reached through the class, never through `self`
        extra_args["denoise_mask"] = denoise_mask
        LAST_RUN.update(mode=None, fused=False, job=None, events=None, events_call=None)
        model_k = KSamplerX0Inpaint(model_wrap, sigmas)
        model_k.latent_image = latent_image
        if self.inpaint_options.get("random", False):
            generator = torch.manual_seed(extra_args.get("seed", 41) + 1)
            model_k.noise = torch.randn(noise.shape, generator=generator, device="cpu").to(noise.dtype).to(noise.device)
        else:
            model_k.noise = noise
        base = model_wrap.inner_model
        is_flux = base.model_type == ModelType.FLUX
        is_flow = base.model_type in FLOW_MODEL_TYPES
        patcher = model_wrap.model_patcher
        model_wrap.cfg_BIG = 1.0 if is_flux else patcher.LanPaint_cfg_BIG
        max_denoise = self.max_denoise(model_wrap, sigmas)
        x_init = base.model_sampling.noise_scaling(sigmas[0], noise, latent_image, max_denoise)
        layout = getattr(model_wrap, "minimax_h3_audio", None)
        if layout is not None and time_shift_sigma is not None:  # mark the audio rows of the flat pack (nodes.py:340-349)
            latent_shapes, shift_v, shift_a = layout
            video_n = math.prod(latent_shapes[0][1:])
            indicator = torch.zeros(x_init.shape, dtype=torch.float32, device=x_init.device)
            indicator[..., video_n:] = 1.0
            model_k.audio_indicator = indicator
            model_k.audio_shifts = (shift_v, shift_a)
        model_options = extra_args.get("model_options", {}) or {}
        opts = model_options.get("lanpaint_b200", {}) or {}
        hyper = dict(NSteps=patcher.LanPaint_NumSteps, Friction=patcher.LanPaint_Friction,
                     Lambda=patcher.LanPaint_Lambda, Beta=patcher.LanPaint_Beta, StepSize=patcher.LanPaint_StepSize,
                     IS_FLUX=is_flux, IS_FLOW=is_flow,
                     EarlyStopThreshold=getattr(patcher, "LanPaint_InnerThreshold", 0.0),
                     EarlyStopPatience=getattr(patcher, "LanPaint_InnerPatience", 1),
                     MinStepFrac=getattr(patcher, "LanPaint_MinStepFrac", 1.0))
        early_stop = patcher.LanPaint_EarlyStop
        use_graph = _graphs_enabled(opts)
        eo = self.extra_options or {}
        sampler_key = (getattr(self.sampler_function, "__name__", ""), float(eo.get("eta", 1.0)),
                       float(eo.get("s_noise", 1.0)))
        entry = _ENGINES.lookup(model_wrap, x_init, model_k.sigmas_host, hyper, early_stop, max_denoise, opts,
                                model_options, callback is not None, sampler=sampler_key) if use_graph else None
        engine = entry.engine if entry is not None else None
        if engine is None:
            engine = LanPaint(model_k.inner_model, EarlyStopHook=model_options.get("lanpaint_semantic_hook", None),
                              rng=opts.get("rng", "torch"), batched_replace=opts.get("batched_replace", "reference"),
                              cuda_graph=use_graph, graph_after=int(opts.get("graph_after", 1)), **hyper)
            if entry is not None:
                entry.engine = engine
                engine.graph_model_token = "node-cache"   # the entry's key already pins model, conds and scales
        else:  # a configuration seen before: same engine (and its graphs), this call's guider and hook
            engine.inner_model = model_k.inner_model
            engine.early_stop_hook = model_options.get("lanpaint_semantic_hook", None)
            engine.reset_counters()
        model_k.PaintMethod = engine
        model_k.LanPaint_early_stop = early_stop
        model_k.LanPaint_min_step_frac = hyper["MinStepFrac"]
        total_steps = len(sigmas) - 1
        timing = None
        if opts.get("timing"):   # bench/profiling: device time of the sampler loop, inputs already on the device
            timing = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            timing[0].record()

        samples = None
        fused = None      # the runner.GraphedJob sampler kwargs of the host-owned loop this sampler maps onto
        if opts.get("fused_ancestral", False) and KSAMPLER._fused_ancestral_ok(self, model_k, denoise_mask, model_options,
                                                                                engine):
            fused = dict(sampler="euler_ancestral", eta=sampler_key[1], s_noise=sampler_key[2])
        elif KSAMPLER._fused_dpmpp_2m_ok(self, model_k, denoise_mask, model_options, engine):
            fused = dict(sampler="dpmpp_2m")
        elif KSAMPLER._fused_dpm_2_ok(self, model_k, denoise_mask, model_options, engine):
            fused = dict(sampler="dpm_2")
        elif KSAMPLER._fused_deis_ok(self, model_k, denoise_mask, model_options, engine):
            fused = dict(sampler="deis", sampler_fn=self.sampler_function)
        elif KSAMPLER._fused_res_multistep_ok(self, model_k, denoise_mask, model_options, engine, extra_args):
            fused = dict(sampler="res_multistep")
        elif KSAMPLER._fused_gradient_estimation_ok(self, model_k, denoise_mask, model_options, engine):
            fused = dict(sampler="gradient_estimation")
        elif opts.get("fused_heun", False) and KSAMPLER._fused_heun_ok(self, model_k, denoise_mask, model_options,
                                                                        engine):
            fused = dict(sampler="heun", sampler_fn=self.sampler_function)
        elif KSAMPLER._fused_euler_ok(self, model_k, denoise_mask, model_options, engine):
            fused = {}
        if opts.get("fused_sampler", True) and fused is not None:
            samples = KSAMPLER._fused_euler(self, model_k, entry, engine, x_init, latent_image, denoise_mask, model_options,
                                        extra_args.get("seed"), is_flux or is_flow, early_stop, callback, total_steps,
                                        use_graph, opts, fused)
        sg_ok = False
        if samples is None and use_graph and entry is not None and opts.get("sampler_graph", True):
            sg_ok = KSAMPLER._sampler_graph_ok(self, model_k, denoise_mask, model_options, engine, entry)
            if sg_ok and isinstance(entry.trace, list):
                samples = KSAMPLER._sampler_graph(self, model_k, entry, engine, x_init, latent_image, denoise_mask,
                                                  model_options, extra_args, callback, opts)
                sg_ok = sg_ok and entry.trace is not False
        if samples is None:
            k_callback = None
            if callback is not None:
                k_callback = lambda d: callback(d["i"], d["denoised"], d["x"], total_steps)  # noqa: E731
            recording = sg_ok and entry.trace is None
            if recording:       # first job of this configuration: plain launches, and remember what the sampler asked for
                model_k.trace = []
                engine.cuda_graph = False
                gen = torch.cuda.default_generators[x_init.device.index if x_init.device.index is not None
                                                    else torch.cuda.current_device()]
                off0 = gen.get_offset()
                t_ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
                t_ev[0].record()
            try:
                samples = self.sampler_function(model_k, x_init, sigmas, extra_args=extra_args, callback=k_callback,
                                                disable=disable_pbar, **self.extra_options)
            finally:
                if recording:
                    engine.cuda_graph = use_graph
            if recording:
                t_ev[1].record()
                own_draws = (gen.get_offset() - off0) != model_k.rng_delta     # the sampler drew noise itself
                entry.trace = False if (own_draws or not model_k.trace) else model_k.trace
                entry.eager_events = t_ev
                model_k.trace = None
        self.last_engine = engine
        if timing is not None:
            timing[1].record()
            job = LAST_RUN.get("job")
            # fused loop: the events GraphedJob recorded around the loop itself (inputs resident in its buffers)
            LAST_RUN["events"] = job.last_events if (job is not None and job.last_events is not None) else timing
            LAST_RUN["events_call"] = timing    # whole KSAMPLER.sample body, host-side preparation included
        return base.model_sampling.inverse_noise_scaling(sigmas[-1], samples)

    # ---- plain Euler: the sampler loop as one launch sequence ---------------------------------------
    @staticmethod
    def _fused_loop_ok(model_k, denoise_mask, model_options, engine) -> bool:
        """What every host-owned loop of runner.GraphedJob needs: an inpainting mask, nothing that runs host code or
        changes the mask inside an outer step, an in-kernel RNG, every sigma but the last > 0."""
        if denoise_mask is None or model_k.audio_indicator is not None:
            return False
        if "denoise_mask_function" in model_options or model_options.get("callback") is not None:
            return False
        if float(engine.early_stop_threshold or 0.0) > 0.0 or isinstance(model_options.get("lanpaint_semantic_stop"), dict):
            return False
        if engine.rng not in ("torch", "philox"):
            return False
        sig = model_k.sigmas_host
        return len(sig) >= 2 and all(v > 0.0 for v in sig[:-1])

    def _fused_euler_ok(self, model_k, denoise_mask, model_options, engine) -> bool:
        """True when k-diffusion's sample_euler around the per-sigma wrapper is exactly the host-owned loop of
        runner.GraphedJob: default Euler (no churn), an inpainting mask, nothing that runs host code or changes
        the mask inside an outer step."""
        fn = self.sampler_function
        if getattr(fn, "__name__", "") != "sample_euler":
            return False
        eo = self.extra_options or {}
        if float(eo.get("s_churn", 0.0) or 0.0) != 0.0 or float(eo.get("s_noise", 1.0) or 1.0) != 1.0:
            return False
        return KSAMPLER._fused_loop_ok(model_k, denoise_mask, model_options, engine)

    def _fused_ancestral_ok(self, model_k, denoise_mask, model_options, engine) -> bool:
        """True when k-diffusion's sample_euler_ancestral around the per-sigma wrapper is the host-owned loop of
        runner.GraphedJob(sampler="euler_ancestral"): the exclusions of `_fused_euler_ok`, and the sampler's noise
        drawn from the global generator (the default noise sampler of the stand-in and of the reference fixtures)."""
        if getattr(self.sampler_function, "__name__", "") != "sample_euler_ancestral":
            return False
        if set(self.extra_options or {}) - {"eta", "s_noise"}:
            return False
        return KSAMPLER._fused_loop_ok(model_k, denoise_mask, model_options, engine)

    def _fused_dpmpp_2m_ok(self, model_k, denoise_mask, model_options, engine) -> bool:
        """True when k-diffusion's sample_dpmpp_2m around the per-sigma wrapper is the host-owned loop of
        runner.GraphedJob(sampler="dpmpp_2m"): the sampler without extra options, and the exclusions of
        `_fused_euler_ok`."""
        if getattr(self.sampler_function, "__name__", "") != "sample_dpmpp_2m" or self.extra_options:
            return False
        return KSAMPLER._fused_loop_ok(model_k, denoise_mask, model_options, engine)

    def _fused_dpm_2_ok(self, model_k, denoise_mask, model_options, engine) -> bool:
        """True when k-diffusion's sample_dpm_2 around the per-sigma wrapper is the host-owned loop of
        runner.GraphedJob(sampler="dpm_2"): the sampler without extra options (no churn), and the exclusions of
        `_fused_euler_ok`."""
        if getattr(self.sampler_function, "__name__", "") != "sample_dpm_2" or self.extra_options:
            return False
        return KSAMPLER._fused_loop_ok(model_k, denoise_mask, model_options, engine)

    def _fused_deis_ok(self, model_k, denoise_mask, model_options, engine) -> bool:
        """True when ComfyUI's sample_deis around the per-sigma wrapper is the host-owned loop of
        runner.GraphedJob(sampler="deis"): the sampler without extra options (max_order 3, 'tab' mode), its module's
        `deis.get_deis_coeff_list` to take the coefficients from, and the exclusions of `_fused_euler_ok`."""
        fn = self.sampler_function
        if getattr(fn, "__name__", "") != "sample_deis" or self.extra_options:
            return False
        deis = getattr(sys.modules.get(getattr(fn, "__module__", None) or ""), "deis", None)
        if not callable(getattr(deis, "get_deis_coeff_list", None)):
            return False
        return KSAMPLER._fused_loop_ok(model_k, denoise_mask, model_options, engine)

    def _fused_res_multistep_ok(self, model_k, denoise_mask, model_options, engine, extra_args) -> bool:
        """True when ComfyUI's sample_res_multistep around the per-sigma wrapper is the host-owned loop of
        runner.GraphedJob(sampler="res_multistep"): the sampler without extra options (eta = 0), a seed in extra_args
        (its draw, multiplied by sigma_up = 0, then comes from a private generator, so skipping it leaves every
        generator as the sampler leaves it), the exclusions of `_fused_euler_ok`, and the form check of
        `_restates`."""
        fn = self.sampler_function
        if getattr(fn, "__name__", "") != "sample_res_multistep" or self.extra_options:
            return False
        if (extra_args or {}).get("seed") is None:
            return False
        return KSAMPLER._fused_loop_ok(model_k, denoise_mask, model_options, engine) and _restates(fn, "res_multistep")

    def _fused_gradient_estimation_ok(self, model_k, denoise_mask, model_options, engine) -> bool:
        """True when ComfyUI's sample_gradient_estimation around the per-sigma wrapper is the host-owned loop of
        runner.GraphedJob(sampler="gradient_estimation"): the sampler without extra options (ge_gamma = 2), the
        exclusions of `_fused_euler_ok`, and the form check of `_restates` (ComfyUI has shipped an older form that
        the loop does not restate)."""
        fn = self.sampler_function
        if getattr(fn, "__name__", "") != "sample_gradient_estimation" or self.extra_options:
            return False
        return (KSAMPLER._fused_loop_ok(model_k, denoise_mask, model_options, engine)
                and _restates(fn, "gradient_estimation"))

    def _fused_heun_ok(self, model_k, denoise_mask, model_options, engine) -> bool:
        """True when k-diffusion's sample_heun around the per-sigma wrapper is the host-owned loop of
        runner.GraphedJob(sampler="heun"): the sampler without extra options (no churn), the exclusions of
        `_fused_euler_ok`, and the form check of `_restates`, which also turns away a sample_heun that draws from the
        global generator without churn (k-diffusion's original)."""
        fn = self.sampler_function
        if getattr(fn, "__name__", "") != "sample_heun" or self.extra_options:
            return False
        return KSAMPLER._fused_loop_ok(model_k, denoise_mask, model_options, engine) and _restates(fn, "heun")

    def _fused_euler(self, model_k, entry, engine, x_init, latent_image, denoise_mask, model_options, seed, flow,
                     early_stop, callback, total_steps, use_graph, opts, sampler=None):
        """sampler: the GraphedJob sampler kwargs (None or {}: plain Euler)."""
        from .runner import GraphedJob, HostSchedule
        if not x_init.is_cuda:
            raise RuntimeError("lanpaint_b200 needs the latent on a CUDA device: there is no CPU or eager fallback")
        if engine._noise_is_zero(model_k.noise):   # add_noise disabled: fresh noise every outer step (lanpaint.py:51-52)
            return None
        B = x_init.shape[0]
        job = entry.job if entry is not None else None
        if job is None:
            sched = HostSchedule(model_k.sigmas_host, B, engine.n_steps, flow, early_stop, engine.min_step_frac)
            try:
                job = GraphedJob(engine, sched, tuple(x_init.shape), x_init.device, flow=flow, external_init=True,
                                 first_replace_noop=False, **(sampler or {}))
            except ValueError:     # noise_scaling is not a linear form: the per-sigma wrapper calls it instead
                return None
            if entry is not None:
                entry.job = job
        job.model_options, job.seed = model_options, seed
        job.timing = bool(opts.get("timing"))
        pm = model_k._latent_mask(denoise_mask, x_init)
        runs = entry.runs if entry is not None else 0
        after = int(opts.get("graph_after", 1))
        captures = job.captures
        if not use_graph or entry is None or entry.graph_failed or runs < after:
            mode = "eager"
        elif callback is None:
            mode = "job"
        else:
            # ComfyUI always passes a callback (progress bar / preview / interrupt check).  One graph per outer step
            # keeps it live -- right for a real network, where a step takes long enough to watch.  When the eager
            # job of this configuration took only a few (< 50) milliseconds nobody can watch anything: the whole job runs
            # as ONE graph, each outer step keeps its denoised latent, and the callbacks run in order right after.
            dev_ms = None      # device time of this configuration's previous job
            if entry.eager_events is not None:
                dev_ms = entry.eager_events[0].elapsed_time(entry.eager_events[1]) * entry.eager_scale
            deferred = (opts.get("deferred_callbacks", True) and dev_ms is not None
                        and dev_ms <= float(opts.get("deferred_max_ms", 50.0))
                        and job.per_step_bytes() <= int(opts.get("deferred_max_bytes", 4 << 30)))
            mode = "job" if deferred else "steps"
        observe = _deferred_outputs(callback, opts)
        timing = None
        if entry is not None:
            timing = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            timing[0].record()
        try:
            out = job.run(latent_image, model_k.noise, pm, x_init=x_init, callback=callback, mode=mode,
                          warm=after <= 0, observe=observe)
            if timing is not None and job.captures == captures:   # a run that captured graphs also timed the capture
                timing[1].record()
                entry.eager_events, entry.eager_scale = timing, 1.0
                n = len(job.sched.steps)
                if mode == "eager" and n > 1:
                    # the first outer step of the first job of a process also loads every kernel the job launches
                    # (CUDA's lazy module loading), which can take as long as the job: time the other steps
                    entry.eager_events, entry.eager_scale = (job.first_step_end, timing[1]), n / (n - 1)
        except Exception as e:
            if mode == "eager":
                raise
            import warnings
            from .engine import _repair_generator_after_failed_capture
            warnings.warn(f"lanpaint_b200: CUDA-graph capture of the sampler loop failed ({type(e).__name__}: {e}); "
                          "running eagerly")
            _repair_generator_after_failed_capture(x_init.device)
            entry.graph_failed = True
            job._graphs = {}
            engine.reset_counters()
            out = job.run(latent_image, model_k.noise, pm, x_init=x_init, callback=callback, mode="eager")
        if entry is not None:
            entry.runs += 1
            entry.last_mode = mode
            if job.captures != captures:   # graphs captured during this call read through this call's guider
                entry.pinned.append((model_k.inner_model, model_options))
        LAST_RUN.update(mode=mode, fused=True, job=job)
        return out if out.dtype == x_init.dtype else out.to(x_init.dtype)


    # ---- any other deterministic sampler: the whole k-diffusion loop as one graph ------------------------------
    def _sampler_graph_ok(self, model_k, denoise_mask, model_options, engine, entry) -> bool:
        if entry.trace is False or entry.graph_failed:
            return False
        if denoise_mask is None or model_k.audio_indicator is not None:
            return False
        if "denoise_mask_function" in model_options or model_options.get("callback") is not None:
            return False
        if float(engine.early_stop_threshold or 0.0) > 0.0 or isinstance(model_options.get("lanpaint_semantic_stop"), dict):
            return False
        if engine.rng not in ("torch", "philox") or engine._noise_is_zero(model_k.noise):
            return False
        return True

    def _sampler_graph(self, model_k, entry, engine, x_init, latent_image, denoise_mask, model_options, extra_args,
                       callback, opts):
        from .engine import _repair_generator_after_failed_capture
        from .runner import SamplerGraphJob
        job = entry.sampler_job
        if job is None:
            if callback is not None:     # callbacks can only be delivered after the replay: short jobs only
                dev_ms = entry.eager_events[0].elapsed_time(entry.eager_events[1]) if entry.eager_events else None
                # the recorded callbacks keep (denoised, x) of every step alive inside the graph's memory pool
                nbytes = 2 * (len(model_k.sigmas_host) - 1) * x_init.numel() * 4
                if not opts.get("deferred_callbacks", True) or nbytes > int(opts.get("deferred_max_bytes", 4 << 30)):
                    entry.trace = False
                    return None
                if dev_ms is None or dev_ms > float(opts.get("deferred_max_ms", 50.0)):
                    # too long to be sure nobody watches the progress bar -- or the first job of the process, which
                    # also paid CUDA's lazy module loading: record and time one more eager job before giving up
                    entry.sg_retries += 1
                    entry.trace = None if entry.sg_retries < 3 else False
                    return None
            job = entry.sampler_job = SamplerGraphJob(engine, self.sampler_function, self.extra_options,
                                                      torch.tensor(model_k.sigmas_host), entry.trace,
                                                      tuple(x_init.shape), x_init.device)
        job.timing = bool(opts.get("timing"))
        pm = model_k._latent_mask(denoise_mask, x_init)
        captures = job.captures
        try:
            out = job.run(model_k, extra_args, latent_image, model_k.noise, pm, x_init, callback=callback)
        except Exception as e:
            import warnings
            warnings.warn(f"lanpaint_b200: capturing the sampler loop failed ({type(e).__name__}: {e}); "
                          "using one graph per wrapper call instead")
            _repair_generator_after_failed_capture(x_init.device)
            entry.trace, entry.sampler_job = False, None
            engine.reset_counters()
            return None
        if job.captures != captures:
            entry.pinned.append((model_k.inner_model, model_options))
        entry.runs += 1
        LAST_RUN.update(mode="sampler-graph", fused=False, job=job)
        return out if out.dtype == x_init.dtype else out.to(x_init.dtype)


# =============================================================================================
# the form check of the res_multistep and gradient_estimation gates
# =============================================================================================
def _res_multistep_form(model, x, sigmas):
    """runner.GraphedJob(sampler="res_multistep")'s update from `res_multistep_step`'s scalars, in x's dtype."""
    from .schedule import res_multistep_step
    old = None
    for i, (second, a, b, c, e) in enumerate(res_multistep_step(sigmas.to(torch.float32))):
        den = model(x, sigmas[i])
        x = a * x - b * (c * den - e * old) if second else x + ((x - den) / a) * b
        old = den
    return x


def _gradient_estimation_form(model, x, sigmas):
    """runner.GraphedJob(sampler="gradient_estimation")'s update from `gradient_estimation_step`'s scalars, in x's
    dtype."""
    from .schedule import gradient_estimation_step
    old = None
    for i, (sigma, dt, gm1, reads, final, _) in enumerate(gradient_estimation_step(sigmas.to(torch.float32))):
        den = model(x, sigmas[i])
        d = (x - den) / sigma
        if final:
            x = den
        else:
            x = x + d * dt
            if reads:
                x = x + gm1 * (d - old) * dt
        old = d
    return x


def _heun_form(model, x, sigmas):
    """runner.GraphedJob(sampler="heun")'s update from `heun_step`'s scalars, in x's dtype."""
    from .schedule import heun_step
    for i, (sigma, dt, sigma_next, corrector) in enumerate(heun_step(sigmas.to(torch.float32))):
        d = (x - model(x, sigmas[i])) / sigma
        if not corrector:
            x = x + d * dt
            continue
        x_2 = x + d * dt
        d_2 = (x_2 - model(x_2, sigmas[i + 1])) / sigma_next
        x = x + (d + d_2) / 2 * dt
    return x


_FORMS = {"res_multistep": _res_multistep_form, "gradient_estimation": _gradient_estimation_form,
          "heun": _heun_form}
_FORM_OK = {}     # (sampler function, sampler) -> whether the function computes the form of that fused loop


def _restates(fn, sampler: str) -> bool:
    """Whether the sampler function `fn` computes what the fused loop of `sampler` restates: `fn` runs once, in fp64
    on the CPU, around an affine stand-in network, on a 5-step schedule that ends at 0 and on a window that ends above
    it, and its results must match the loop's update from its own fp32 scalars to 1e-5.  The function must also leave
    the global generator where it found it: the fused loops take no draw from it (k-diffusion's original sample_heun
    draws a randn_like every step even without churn, which on the device would shift every later Langevin draw).  The
    generator's state is put back afterwards, so the check consumes nothing.  Cached per function."""
    key = (fn, sampler)
    ok = _FORM_OK.get(key)
    if ok is None:
        g = torch.Generator().manual_seed(0)
        x0 = torch.randn(2, 3, 4, 4, generator=g, dtype=torch.float64) * 5
        bias = torch.randn(2, 3, 4, 4, generator=g, dtype=torch.float64)
        model = lambda x, sigma, **kw: 0.75 * x + 0.25 * bias   # noqa: E731
        ok = True
        state = torch.default_generator.get_state()
        try:
            for sig in ([5.0, 2.5, 1.1, 0.4, 0.1, 0.0], [5.0, 2.5, 1.1, 0.4]):
                sigmas = torch.tensor(sig, dtype=torch.float64)
                try:
                    got = fn(model, x0.clone(), sigmas, extra_args={"seed": 0}, callback=None, disable=True)
                except Exception:
                    ok = False
                    break
                want = _FORMS[sampler](model, x0.clone(), sigmas)
                if not float((got - want).abs().max()) <= 1e-5 * float(want.abs().max()):
                    ok = False
                    break
            ok = ok and torch.equal(torch.default_generator.get_state(), state)
        finally:
            torch.default_generator.set_state(state)
        _FORM_OK[key] = ok
    return ok


# =============================================================================================
# engines (and their CUDA graphs) kept across sample() calls
# =============================================================================================
# ComfyUI's own previewers (latent_preview.py): each decodes the first request's latent, x0[:1], and nothing else
_STOCK_PREVIEWERS = ("Latent2RGBPreviewer", "TAESDPreviewerImpl")


def _deferred_outputs(callback, opts) -> str:
    """What of each outer step's denoised latent a deferred fused job keeps for `callback` (GraphedJob.run's observe).

    ComfyUI's stock callback, the closure `latent_preview.prepare_callback` returns, stores x0 into its output dict
    (each step overwriting the last), hands it to the previewer, if one is configured, and advances the progress bar.
    So before the last step it reads only what the previewer decodes, the first request's latent: "final" without a
    previewer, "preview" with one of ComfyUI's own.  Any other callback -- a user's, one from a patched or replaced
    prepare_callback, one whose previewer is not ComfyUI's -- gets "full", every step's whole latent, as does the model
    option {"lanpaint_b200": {"deferred_outputs": "full"}}.  The stock closure is told by its code object: one of the
    functions compiled into the current prepare_callback, itself ComfyUI's (minicomfy's in tests) by name and module."""
    setting = opts.get("deferred_outputs", "auto")
    if setting not in ("auto", "full"):
        raise ValueError(f"lanpaint_b200 option deferred_outputs: 'auto' or 'full', not {setting!r}")
    prepare = getattr(latent_preview, "prepare_callback", None)
    code = getattr(callback, "__code__", None)
    if setting == "full" or code is None or not (getattr(prepare, "__qualname__", "") == "prepare_callback" and
                                                 getattr(prepare, "__module__", "") in ("latent_preview", "minicomfy")):
        return "full"
    if code not in prepare.__code__.co_consts:
        return "full"
    cells = dict(zip(code.co_freevars, callback.__closure__ or ()))
    if not set(cells) <= {"x0_output_dict", "previewer", "pbar", "preview_format"}:
        return "full"
    previewer = cells["previewer"].cell_contents if "previewer" in cells else None
    if not previewer:
        return "final"
    kind = type(previewer)
    if kind.__name__ in _STOCK_PREVIEWERS and kind.__module__ in ("latent_preview", "minicomfy"):
        return "preview"
    return "full"


def _graphs_enabled(opts) -> bool:
    import os
    if os.environ.get("LANPAINT_B200_GRAPH", "1") == "0":
        return False
    return bool(opts.get("cuda_graph", True))


def _weights_fingerprint(model_wrap):
    """Where the network's parameters live right now.  A captured graph holds raw pointers into them: if
    ComfyUI off-loaded and re-loaded the model (new addresses) the cached graphs must be dropped."""
    net = getattr(getattr(model_wrap, "inner_model", None), "diffusion_model", None)
    if isinstance(net, torch.nn.Module):
        return tuple(p.data_ptr() for p in net.parameters())
    return id(net)


def _cond_fingerprint(c, depth: int = 0):
    """Identity of a CONDITIONING value as a captured graph sees it.  ComfyUI's CFGGuider.set_conds runs
    `convert_cond` on every call: a NEW list of NEW dicts (each with a fresh `uuid`) around the SAME tensors -- the
    text-encoder outputs ComfyUI's node cache keeps alive while the prompt is unchanged.  So containers are compared
    structurally, tensors and other leaves by object identity (the cache entry pins them, an id cannot be recycled),
    thin wrapper objects (comfy.conds.CONDRegular & co.: one `.cond` attribute) by what they wrap, `uuid` not at all."""
    if isinstance(c, (str, int, float, bool, type(None))):
        return c
    if depth < 5:
        if isinstance(c, dict):
            return tuple((str(k), _cond_fingerprint(v, depth + 1)) for k, v in sorted(c.items(), key=lambda kv: str(kv[0]))
                         if k != "uuid")
        if isinstance(c, (list, tuple)):
            return tuple(_cond_fingerprint(v, depth + 1) for v in c)
        inner = getattr(c, "cond", None)
        if inner is not None and not isinstance(c, torch.Tensor):
            return (type(c).__name__, _cond_fingerprint(inner, depth + 1))
    if isinstance(c, torch.Tensor):
        return ("tensor", id(c), tuple(c.shape), str(c.dtype), str(c.device))
    return ("object", id(c))


class _EngineEntry:
    __slots__ = ("engine", "job", "runs", "graph_failed", "last_mode", "weights", "keep", "pinned", "eager_events",
                 "eager_scale", "trace", "sampler_job", "sg_retries")

    def __init__(self):
        self.engine = self.job = None
        self.trace = None           # None: not recorded yet; list: the wrapper calls of one job; False: not capturable
        self.sampler_job = None
        self.sg_retries = 0
        self.pinned = []
        self.eager_events = None   # CUDA events around the previous job: how long this configuration takes
        self.eager_scale = 1.0     # ... times this (the events span only part of it)
        self.runs = 0
        self.graph_failed = False
        self.last_mode = None
        self.weights = None
        self.keep = None


class _EngineCache:
    """A few recently used (engine, GraphedJob) pairs keyed by everything a captured graph bakes in: the
    ModelPatcher, the conditioning objects, both guidance scales, latent shape and device, the sigma schedule,
    every hyper-parameter, the model_options the network reads, whether a callback wants the denoised latent,
    the sampler function with its eta / s_noise.
    The entry keeps the objects named by id() alive, so an id in the key can never be recycled."""

    def __init__(self, capacity: int = 4):
        self.capacity = capacity
        self.entries = {}

    def lookup(self, model_wrap, x, sigmas_host, hyper, early_stop, max_denoise, opts, model_options, has_callback,
               sampler=None):
        from .engine import options_fingerprint
        conds = getattr(model_wrap, "original_conds", None) or getattr(model_wrap, "conds", {}) or {}
        pos, neg = conds.get("positive"), conds.get("negative")
        net_opts = {k: v for k, v in model_options.items() if k != "lanpaint_b200"}
        key = (id(model_wrap.model_patcher), _cond_fingerprint(pos), _cond_fingerprint(neg), float(model_wrap.cfg),
               float(model_wrap.cfg_BIG),
               str(x.device), tuple(x.shape), str(x.dtype), tuple(sigmas_host), tuple(sorted(hyper.items())),
               early_stop, bool(max_denoise), options_fingerprint(opts), options_fingerprint(net_opts),
               bool(has_callback), sampler)   # sampler: (function name, eta, s_noise): entry.job runs that loop only
        entry = self.entries.pop(key, None)
        weights = _weights_fingerprint(model_wrap)
        if entry is not None and entry.weights != weights:
            entry = None                       # the model moved: graphs captured against it are dead
        if entry is None:
            entry = _EngineEntry()
            entry.weights = weights
        entry.keep = (model_wrap, model_wrap.model_patcher, pos, neg, model_options)
        self.entries[key] = entry              # most recently used last
        while len(self.entries) > self.capacity:
            self.entries.pop(next(iter(self.entries)))
        return entry

    def clear(self):
        self.entries.clear()


_ENGINES = _EngineCache()
LAST_RUN = {"mode": None, "fused": False, "job": None, "events": None, "events_call": None}   # how the most recent sample call was launched


_override_active = False
LAST_ENGINE = {"engine": None}  # the engine of the most recent sample call (bench/test introspection)


def _noise_device(model, opts=None):
    """The CUDA device a node's noise image may be drawn on instead of ComfyUI's CPU, or None: the model's load
    device, unless `{"device_noise": False}` or this host's torch draws other bits than the kernel (hostnoise.verified)."""
    if opts is None:
        opts = (getattr(model, "model_options", None) or {}).get("lanpaint_b200") or {}
    if not opts.get("device_noise", True):
        return None
    dev = getattr(model, "load_device", None)
    if dev is None or torch.device(dev).type != "cuda":
        return None
    from . import hostnoise
    return torch.device(dev) if hostnoise.verified(dev) else None


def _device_randn_ok(latent_image, noise_inds=None) -> bool:
    """What lp_torch_cpu_randn_f32 reproduces: one `torch.randn(size, fp32, strided)` of at least 16 values."""
    return (noise_inds is None and isinstance(latent_image, torch.Tensor) and not latent_image.is_nested
            and latent_image.dtype == torch.float32 and latent_image.layout == torch.strided and latent_image.numel() >= 16)


@contextmanager
def override_sample_function(noise_device=None):
    """Swap CFGGuider.outer_sample / .predict_noise, KSAMPLER.sample and sampler_helpers.prepare_mask for
    the duration of one sample call; always restore; nested entry is a no-op (nodes.py:384-421).

    With `noise_device` (a CUDA device whose stream was verified against this host's torch.randn) a fifth function
    is swapped as well: `comfy.sample.prepare_noise`, ComfyUI's single-threaded CPU draw of the noise image, by
    `hostnoise.torch_cpu_randn` -- the same bits, the same effect on torch's generators, drawn on the device."""
    global _override_active
    if _override_active:
        yield
        return
    _override_active = True
    guider_cls, ksampler_cls, helpers = comfy.samplers.CFGGuider, comfy.samplers.KSAMPLER, comfy.sampler_helpers
    saved = (guider_cls.outer_sample, guider_cls.predict_noise, ksampler_cls.sample, helpers.prepare_mask)
    sample_mod = getattr(comfy, "sample", None) if noise_device is not None else None
    saved_noise = getattr(sample_mod, "prepare_noise", None)
    if not (getattr(saved_noise, "__name__", "") == "prepare_noise"
            and getattr(saved_noise, "__module__", "") in ("comfy.sample", "minicomfy")):
        saved_noise = None      # some extension installed its own noise source: that is what the user asked for

    def prepare_noise_on_device(latent_image, seed, noise_inds=None):
        if not _device_randn_ok(latent_image, noise_inds):
            return saved_noise(latent_image, seed, noise_inds)
        from . import hostnoise
        return hostnoise.torch_cpu_randn(latent_image.size(), seed, noise_device)

    def sample_and_remember(self, *a, **k):
        out = KSAMPLER.sample(self, *a, **k)
        LAST_ENGINE["engine"] = getattr(self, "last_engine", None)
        return out

    try:
        guider_cls.outer_sample = CFGGuider_LanPaint.outer_sample
        guider_cls.predict_noise = CFGGuider_LanPaint.predict_noise
        ksampler_cls.sample = sample_and_remember
        helpers.prepare_mask = lambda noise_mask, shape, device: prepare_mask(
            noise_mask, shape, device, video_inpainting=(len(shape) == 5))
        if saved_noise is not None:
            sample_mod.prepare_noise = prepare_noise_on_device
        yield
    finally:
        guider_cls.outer_sample, guider_cls.predict_noise, ksampler_cls.sample, helpers.prepare_mask = saved
        if saved_noise is not None:
            sample_mod.prepare_noise = saved_noise
        _override_active = False


def _ensure_model_options(model, video_inpainting):
    if not hasattr(model, "model_options") or model.model_options is None:
        model.model_options = {}
    model.model_options["video_inpainting"] = video_inpainting


# =============================================================================================
# nodes (nodes.py:452-589, 659-808)
# =============================================================================================
class LanPaint_KSampler:
    @classmethod
    def INPUT_TYPES(s):
        return {
            "required": {
                "model": ("MODEL", {"tooltip": "The model used for denoising the input latent."}),
                "seed": ("INT", {"default": 0, "min": 0, "max": 0xffffffffffffffff, "tooltip": "The random seed used for creating the noise."}),
                "steps": ("INT", {"default": 30, "min": 1, "max": 10000, "tooltip": "The number of steps used in the denoising process."}),
                "cfg": ("FLOAT", {"default": 5.0, "min": 0.0, "max": 100.0, "step": 0.1, "round": 0.01, "tooltip": "The Classifier-Free Guidance scale balances creativity and adherence to the prompt. Higher values result in images more closely matching the prompt however too high values will negatively impact quality."}),
                "sampler_name": (KSAMPLER_NAMES, {"tooltip": "Recommended: euler."}),
                "scheduler": (comfy.samplers.KSampler.SCHEDULERS, {"default": "karras", "tooltip": "The scheduler controls how noise is gradually removed to form the image."}),
                "positive": ("CONDITIONING", {"tooltip": "The conditioning describing the attributes you want to include in the image."}),
                "negative": ("CONDITIONING", {"tooltip": "The conditioning describing the attributes you want to exclude from the image."}),
                "latent_image": ("LATENT", {"tooltip": "The latent image to denoise."}),
                "denoise": ("FLOAT", {"default": 1.0, "min": 0.0, "max": 1.0, "step": 0.01, "tooltip": "The amount of denoising applied, lower values will maintain the structure of the initial image allowing for image to image sampling."}),
                "LanPaint_NumSteps": _w_num_steps(_TIP_STEPS_K),
                "LanPaint_PromptMode": _w_prompt_mode(_TIP_MODE_K),
                "LanPaint_Info": _w_info("LanPaint KSampler."),
                "Inpainting_mode": _w_mode(),
            },
            "hidden": _hidden(("LanPaint_MinStepFrac",)),
        }

    RETURN_TYPES = ("LATENT",)
    OUTPUT_TOOLTIPS = ("The denoised latent.",)
    FUNCTION = "sample"
    CATEGORY = "sampling"
    DESCRIPTION = "Uses the provided model, positive and negative conditioning to denoise the latent image."

    def sample(self, model, seed, steps, cfg, sampler_name, scheduler, positive, negative, latent_image, denoise=1.0,
               LanPaint_NumSteps=5, LanPaint_PromptMode="Image First", LanPaint_Info="", Inpainting_mode=IMAGE_MODE,
               **kwargs):
        n = _sanitize_param(LanPaint_NumSteps, 5)
        mode = _sanitize_param(LanPaint_PromptMode, "Image First", allowed=PROMPT_MODES)
        imode = _sanitize_param(Inpainting_mode, IMAGE_MODE, allowed=(IMAGE_MODE, VIDEO_MODE))
        _set_hyper(model, num_steps=n, cfg=cfg, prompt_mode=mode)
        _ensure_model_options(model, imode == VIDEO_MODE)
        with override_sample_function(_noise_device(model)):
            return comfy_nodes_module.common_ksampler(model, seed, steps, cfg, sampler_name, scheduler, positive,
                                                      negative, latent_image, denoise=denoise)


class LanPaint_KSamplerAdvanced:
    @classmethod
    def INPUT_TYPES(s):
        return {
            "required": {
                "model": ("MODEL",),
                "add_noise": (["enable", "disable"],),
                "noise_seed": ("INT", {"default": 0, "min": 0, "max": 0xffffffffffffffff}),
                "steps": ("INT", {"default": 30, "min": 1, "max": 10000}),
                "cfg": ("FLOAT", {"default": 5.0, "min": 0.0, "max": 100.0, "step": 0.1, "round": 0.01}),
                "sampler_name": (KSAMPLER_NAMES,),
                "scheduler": (comfy.samplers.KSampler.SCHEDULERS,),
                "positive": ("CONDITIONING",),
                "negative": ("CONDITIONING",),
                "latent_image": ("LATENT",),
                "start_at_step": ("INT", {"default": 0, "min": 0, "max": 10000}),
                "end_at_step": ("INT", {"default": 10000, "min": 0, "max": 10000}),
                "return_with_leftover_noise": (["disable", "enable"],),
                "LanPaint_NumSteps": _w_num_steps(_TIP_STEPS_K),
                "LanPaint_Lambda": ("FLOAT", {"default": 5.0, "min": 0.1, "max": 50.0, "step": 0.1, "round": 0.1, "tooltip": "The bidirectional guidance scale. Higher values align with known regions more closely, but may result in instability."}),
                "LanPaint_StepSize": ("FLOAT", {"default": 0.2, "min": 0.0001, "max": 1., "step": 0.01, "round": 0.001, "tooltip": "The step size for the Langevin dynamics. Higher values result in faster convergence but may be unstable."}),
                "LanPaint_PromptMode": _w_prompt_mode(_TIP_MODE_K),
                "LanPaint_Info": _w_info("LanPaint KSampler Adv."),
                "Inpainting_mode": _w_mode(),
            },
            "hidden": _hidden(_RETIRED_ALL),
        }

    RETURN_TYPES = ("LATENT",)
    FUNCTION = "sample"
    CATEGORY = "sampling"

    def sample(self, model, add_noise, noise_seed, steps, cfg, sampler_name, scheduler, positive, negative,
               latent_image, start_at_step, end_at_step, return_with_leftover_noise, LanPaint_NumSteps=5,
               LanPaint_Lambda=5.0, LanPaint_StepSize=0.2, LanPaint_PromptMode="Image First", LanPaint_Info="",
               Inpainting_mode=IMAGE_MODE, **kwargs):
        n = _sanitize_param(LanPaint_NumSteps, 5)
        lam = _sanitize_param(LanPaint_Lambda, 5.0)
        step = _sanitize_param(LanPaint_StepSize, 0.2)
        mode = _sanitize_param(LanPaint_PromptMode, "Image First", allowed=PROMPT_MODES)
        imode = _sanitize_param(Inpainting_mode, IMAGE_MODE, allowed=(IMAGE_MODE, VIDEO_MODE))
        _set_hyper(model, num_steps=n, cfg=cfg, prompt_mode=mode, lam=lam, step_size=step)
        _ensure_model_options(model, imode == VIDEO_MODE)
        with override_sample_function(_noise_device(model)):
            return comfy_nodes_module.common_ksampler(
                model, noise_seed, steps, cfg, sampler_name, scheduler, positive, negative, latent_image, denoise=1.0,
                disable_noise=(add_noise == "disable"), start_step=start_at_step, last_step=end_at_step,
                force_full_denoise=(return_with_leftover_noise != "enable"))


class Noise_EmptyNoise:
    def generate_noise(self, latent):
        return torch.zeros_like(latent["samples"])


class Noise_RandomNoise:
    def __init__(self, seed, device=None):
        self.seed = seed
        self.device = device       # a verified CUDA device (see _noise_device): same bits, drawn there

    def generate_noise(self, latent):
        samples = latent["samples"]
        if self.device is not None and _device_randn_ok(samples) and samples.device.type == "cpu":
            from . import hostnoise
            return hostnoise.torch_cpu_randn(samples.size(), self.seed, self.device)
        torch.manual_seed(self.seed)
        return torch.randn_like(samples)


def _finish_custom(model_for_preview, latent, samples, x0_output):
    out = latent.copy()
    out["samples"] = samples
    if "x0" in x0_output:
        den = latent.copy()
        den["samples"] = model_for_preview.model.process_latent_out(_host_result(x0_output["x0"]).cpu())
        return out, den
    return out, out


class LanPaint_SamplerCustom:
    @classmethod
    def INPUT_TYPES(s):
        return {"required": {
            "model": ("MODEL",),
            "add_noise": ("BOOLEAN", {"default": True}),
            "noise_seed": ("INT", {"default": 0, "min": 0, "max": 0xffffffffffffffff, "control_after_generate": True}),
            "cfg": ("FLOAT", {"default": 8.0, "min": 0.0, "max": 100.0, "step": 0.1, "round": 0.01}),
            "positive": ("CONDITIONING",),
            "negative": ("CONDITIONING",),
            "sampler": ("SAMPLER",),
            "sigmas": ("SIGMAS",),
            "latent_image": ("LATENT",),
            "LanPaint_NumSteps": _w_num_steps(_TIP_STEPS_C),
            "LanPaint_PromptMode": _w_prompt_mode(_TIP_MODE_C),
            "LanPaint_Info": _w_info("LanPaint Custom Sampler."),
        }}

    RETURN_TYPES = ("LATENT", "LATENT")
    RETURN_NAMES = ("output", "denoised_output")
    FUNCTION = "sample"
    CATEGORY = "sampling/custom_sampling"

    def sample(self, model, sampler, sigmas, add_noise, noise_seed, cfg, positive, negative, latent_image,
               LanPaint_NumSteps, LanPaint_PromptMode, LanPaint_Info=""):
        n = _sanitize_param(LanPaint_NumSteps, 5)
        mode = _sanitize_param(LanPaint_PromptMode, "Image First", allowed=PROMPT_MODES)
        _set_hyper(model, num_steps=n, cfg=cfg, prompt_mode=mode)
        noise_device = _noise_device(model)
        with override_sample_function(noise_device):
            latent = latent_image.copy()
            latent["samples"] = comfy.sample.fix_empty_latent_channels(model, latent["samples"])
            noise = (Noise_RandomNoise(noise_seed, noise_device) if add_noise else Noise_EmptyNoise()).generate_noise(latent)
            x0_output = {}
            callback = latent_preview.prepare_callback(model, sigmas.shape[-1] - 1, x0_output)
            samples = comfy.sample.sample_custom(model, noise, cfg, sampler, sigmas, positive, negative,
                                                 latent["samples"], noise_mask=latent.get("noise_mask"),
                                                 callback=callback, disable_pbar=not comfy.utils.PROGRESS_BAR_ENABLED,
                                                 seed=noise_seed)
            return _finish_custom(model, latent, samples, x0_output)


class LanPaint_SamplerCustomAdvanced:
    @classmethod
    def INPUT_TYPES(s):
        return {
            "required": {
                "noise": ("NOISE",),
                "guider": ("GUIDER",),
                "sampler": ("SAMPLER",),
                "sigmas": ("SIGMAS",),
                "latent_image": ("LATENT",),
                "LanPaint_NumSteps": _w_num_steps(_TIP_STEPS_C),
                "LanPaint_Lambda": ("FLOAT", {"default": 5.0, "min": 0.1, "max": 50.0, "step": 0.1, "tooltip": "Bidirectional guidance scale. Higher values align with known regions but may cause instability."}),
                "LanPaint_StepSize": ("FLOAT", {"default": 0.2, "min": 0.0001, "max": 1.0, "step": 0.01, "tooltip": "Step size for Langevin dynamics. Higher values speed convergence but may be unstable."}),
                "LanPaint_PromptMode": _w_prompt_mode(_TIP_MODE_C),
                "LanPaint_Info": _w_info("LanPaint Custom Sampler Adv."),
            },
            "hidden": _hidden(_RETIRED_ALL),
        }

    RETURN_TYPES = ("LATENT", "LATENT")
    RETURN_NAMES = ("output", "denoised_output")
    FUNCTION = "sample"
    CATEGORY = "sampling/custom_sampling"

    def sample(self, noise, guider, sampler, sigmas, latent_image, LanPaint_NumSteps, LanPaint_Lambda,
               LanPaint_StepSize, LanPaint_PromptMode, LanPaint_Info="", **kwargs):
        n = _sanitize_param(LanPaint_NumSteps, 5)
        lam = _sanitize_param(LanPaint_Lambda, 5.0)
        step = _sanitize_param(LanPaint_StepSize, 0.2)
        mode = _sanitize_param(LanPaint_PromptMode, "Image First", allowed=PROMPT_MODES)
        patcher = guider.model_patcher
        _set_hyper(patcher, num_steps=n, cfg=guider.cfg, prompt_mode=mode, lam=lam, step_size=step)
        with override_sample_function(_noise_device(patcher)):      # ComfyUI's RandomNoise calls comfy.sample.prepare_noise
            latent = latent_image.copy()
            latent["samples"] = comfy.sample.fix_empty_latent_channels(patcher, latent_image["samples"])
            x0_output = {}
            callback = latent_preview.prepare_callback(patcher, sigmas.shape[-1] - 1, x0_output)
            samples = guider.sample(noise.generate_noise(latent), latent["samples"], sampler, sigmas,
                                    denoise_mask=latent.get("noise_mask"), callback=callback,
                                    disable_pbar=not comfy.utils.PROGRESS_BAR_ENABLED, seed=noise.seed)
            samples = samples.to(comfy.model_management.intermediate_device())
            return _finish_custom(patcher, latent, samples, x0_output)


NODE_CLASS_MAPPINGS = {
    "LanPaint_KSampler": LanPaint_KSampler,
    "LanPaint_KSamplerAdvanced": LanPaint_KSamplerAdvanced,
    "LanPaint_SamplerCustom": LanPaint_SamplerCustom,
    "LanPaint_SamplerCustomAdvanced": LanPaint_SamplerCustomAdvanced,
}

NODE_DISPLAY_NAME_MAPPINGS = {
    "LanPaint_KSampler": "LanPaint KSampler",
    "LanPaint_KSamplerAdvanced": "LanPaint KSampler (Advanced)",
    "LanPaint_SamplerCustom": "LanPaint Sampler Custom",
    "LanPaint_SamplerCustomAdvanced": "LanPaint Sampler Custom (Advanced)",
}
