"""A whole LanPaint sampling job restated over the oracle, in any float dtype (test infrastructure).

`job` is what one sampler node call computes between the LATENT dict in and the LATENT dict out: the initial
noise_scaling (max_denoise as the sampler decides it), a k-diffusion sampler (minicomfy's sample_euler / sample_heun /
sample_euler_ancestral, the same Python the node path runs) around the per-sigma wrapper, and inverse_noise_scaling.
The wrapper is `O.outer_step`, which the oracle tests pin to the reference bit for bit in fp32.  Everything the node
layer derives on the host stays in fp32 exactly as the node computes it -- the sigma schedule (`ksampler_sigmas`),
the (VE, abt, flow t) triple from `O.times_from_sigma`, the inner-step count from `O.inner_steps_for`, the audio
stream's times of an AV pack (`av_audio`) -- and is then cast to the job's dtype; the state, the network, every
sub-step, the sampler's updates and the noise scaling run in that dtype.

The routes a node call can take are inputs, not code paths: a step window or `denoise < 1` is the schedule the
caller passes, `add_noise = disable` is a zero noise image (`O.outer_step` then regenerates it through `draw` at
every outer step, before that step's Langevin draws), an ancestral sampler takes its own draws from `draw` too, an
AV pack is `audio`, and an inner early stop is `on_substep`.  In fp64 this is the reference the GPU job tests compare
with; in fp32 it reproduces the reference's node layer on the node fixtures' tapes (tests/test_oracle_node_golden.py).
"""
from __future__ import annotations

import functools
import math
from unittest import mock

import torch

import minicomfy
from _node_cases import NEG, POS, av_shift_sigma, av_shift_slope
from oracle import langevin_oracle as O


class Guider:
    """What the node's patched CFGGuider hands the engine: (x0 at cfg, x0 at cfg_BIG) of `net` between the POS and
    NEG conditionings (nodes.py:161-175); at cfg == 1 the uncond evaluation is skipped and both heads are cond."""

    def __init__(self, net, sampling, cfg, cfg_big):
        self.inner_model, self.model_sampling = self, sampling
        self.net, self.cfg, self.cfg_big = net, cfg, cfg_big
        self.calls = 0

    def __call__(self, x, sigma, model_options=None, seed=None):
        c = self.net(x, sigma, POS)
        self.calls += 1
        if math.isclose(self.cfg, 1.0):
            u = c
        else:
            u = self.net(x, sigma, NEG)
            self.calls += 1
        return u + (c - u) * self.cfg, u + (c - u) * self.cfg_big


def cuda_draw(like):
    """The engine's torch stream: `torch.randn(shape, float32)` on the device's default generator, in the job's
    dtype (fp64: exactly the same normals, upcast).  An ancestral sampler's `torch.randn_like(x)` on the fp32 latent
    draws the same values from the same generator."""
    return torch.randn(like.shape, dtype=torch.float32, device=like.device).to(like.dtype)


def max_denoise(sampling, sigma0) -> bool:
    """KSAMPLER.max_denoise (minicomfy / ComfyUI) for a ModelSampling with sigma_max."""
    hi = float(sampling.sigma_max)
    return math.isclose(hi, float(sigma0), rel_tol=1e-05) or float(sigma0) > hi


def ksampler_sigmas(patcher, steps, sampler, scheduler, denoise=1.0, start_step=None, last_step=None,
                    force_full_denoise=False):
    """The schedule `common_ksampler` hands the sampler: minicomfy.KSampler's (truncated for denoise < 1), then the
    start / last step window of KSampler.sample (a leftover-noise window keeps its last sigma > 0)."""
    sigmas = minicomfy.KSampler(patcher, steps, "cpu", sampler, scheduler, denoise).sigmas
    if last_step is not None and last_step < len(sigmas) - 1:
        sigmas = sigmas[:last_step + 1]
        if force_full_denoise:
            sigmas = sigmas.clone()
            sigmas[-1] = 0
    if start_step is not None:
        assert start_step < len(sigmas) - 1, "an empty window returns the latent unchanged"
        sigmas = sigmas[start_step:]
    return sigmas


def av_audio(n_video, shift_video, shift_audio):
    """The MiniMax-H3 flat pack's audio rows (nodes.py:254-275, 340-349), per outer step: (indicator, the audio
    stream's (VE, abt, flow t) in fp32, the target correction c on audio rows), with `_node_cases`' time-shift
    stand-ins."""
    def audio(times, like):
        fv = times.flow_t
        fa = av_shift_sigma(fv, shift_video, shift_audio)
        abt_a = (1 - fa) ** 2 / ((1 - fa) ** 2 + fa ** 2)
        c = 1.0
        if float(fv) > 1e-4:
            c = float(fa) / (float(fv) * float(av_shift_slope(fv, shift_video, shift_audio)))
        ind = torch.zeros(like.shape, dtype=like.dtype, device=like.device)
        ind[..., n_video:] = 1.0
        return ind, O.Times(fa / (1 - fa), abt_a, fa), c
    return audio


def _plain(fn):
    def sampler(model, x, sigmas, callback=None, draw=None):
        return fn(model, x, sigmas, callback=callback)
    return sampler


def _euler_ancestral(model, x, sigmas, callback=None, draw=None):
    """minicomfy.sample_euler_ancestral with its `torch.randn_like(x)` taken from the job's `draw`, interleaved with
    the wrapper's draws in call order."""
    with mock.patch.object(torch, "randn_like", lambda like, **kw: draw(like)):
        return minicomfy.sample_euler_ancestral(model, x, sigmas, callback=callback)


def job(sampler, model, y, noise, denoise_mask, sigmas, hp: O.Hyper, draw=cuda_draw, max_denoise=False,
        callback=None, early_stop=1, min_frac=1.0, audio=None, on_substep=None):
    """One job in y.dtype.  sampler: a `SAMPLERS` entry.  denoise_mask: 1 = regenerate, of y's shape (or
    broadcastable).  sigmas: the fp32 schedule.  callback(i, denoised) per sampler step.  The model is called as
    model(x, sigma) and returns (x0 at cfg, x0 at cfg_BIG); model.inner_model.model_sampling has noise_scaling /
    inverse_noise_scaling.  audio: `av_audio(...)` for an AV pack.  on_substep(k): the `O.outer_step` hook for the
    k-th wrapper call (or None)."""
    dt, dev = y.dtype, y.device
    sig32 = sigmas.detach().to("cpu", torch.float32)
    sig = sig32.to(device=dev, dtype=dt)
    sampling = model.inner_model.model_sampling
    mask = O.binarise_mask(denoise_mask).to(dt)
    calls = [0]

    def cast(times):
        return O.Times(*(t.to(device=dev, dtype=dt) for t in times))

    def wrapper(x, sigma, **kwargs):
        s32 = sigma.detach().to("cpu", torch.float32)
        tm = O.times_from_sigma(s32, hp.flow)
        n_eff = O.inner_steps_for(s32, sig32, tm.abt, hp.n_steps, early_stop, min_frac)
        aud = None
        if audio is not None:
            ind, tm_a, c = audio(tm, x)
            aud = O.Audio(ind, cast(tm_a), (1.0 - ind) + c * ind)
        hook = None if on_substep is None else on_substep(calls[0])
        calls[0] += 1
        denoised, x_new = O.outer_step(model, x, y, noise, sigma, mask, cast(tm), hp, n_eff, draw, audio=aud,
                                       on_substep=hook)
        x.copy_(x_new)      # the per-sigma wrapper rewrites the sampler's x in place (nodes.py:300)
        return denoised

    x = sampling.noise_scaling(sig[0], noise, y, max_denoise)
    cb = None if callback is None else (lambda d: callback(d["i"], d["denoised"]))
    with torch.no_grad():
        x = sampler(wrapper, x, sig, callback=cb, draw=draw)
    return sampling.inverse_noise_scaling(sig[-1], x)


SAMPLERS = {"euler": _plain(minicomfy.sample_euler), "heun": _plain(minicomfy.sample_heun),
            "euler_ancestral": _euler_ancestral, "dpmpp_2m": _plain(minicomfy.sample_dpmpp_2m),
            "dpm_2": _plain(minicomfy.sample_dpm_2), "deis": _plain(minicomfy.sample_deis),
            # its noise sampler is seeded from extra_args, and its draws are multiplied by sigma_up = 0 (eta = 0)
            "res_multistep": _plain(functools.partial(minicomfy.sample_res_multistep, extra_args={"seed": 0})),
            "gradient_estimation": _plain(minicomfy.sample_gradient_estimation)}
