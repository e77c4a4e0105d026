"""A whole LanPaint sampling job restated over the oracle, in any float dtype (test infrastructure).

`job` is what one `LanPaint_KSampler` call computes between the LATENT dict in and the LATENT dict out: the initial
noise_scaling (max_denoise as the sampler decides it), a k-diffusion sampler (minicomfy's sample_euler / sample_heun,
the same Python the node path runs) around the per-sigma wrapper, and inverse_noise_scaling.  The wrapper is
`O.outer_step`, which the oracle tests pin to the reference bit for bit in fp32.  Everything the node layer derives
on the host stays in fp32 exactly as the node computes it -- the sigma schedule, the (VE, abt, flow t) triple from
`O.times_from_sigma`, the inner-step count from `O.inner_steps_for` -- and is then cast to the job's dtype; the
state, the network, every sub-step, the Euler / Heun updates and the noise scaling run in that dtype.  In fp64 this
is the reference the GPU job tests compare with; in fp32 it equals `O.euler_inpaint` (tests/test_job_ref_host.py).
"""
from __future__ import annotations

import math

import torch

import minicomfy
from _node_cases import NEG, POS
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
    dtype (fp64: exactly the same normals, upcast)."""
    return torch.randn(like.shape, dtype=torch.float32, device=like.device).to(like.dtype)


def max_denoise(sampling, sigma0) -> bool:
    """KSAMPLER.max_denoise (minicomfy / ComfyUI) for a ModelSampling with sigma_max."""
    hi = float(sampling.sigma_max)
    return math.isclose(hi, float(sigma0), rel_tol=1e-05) or float(sigma0) > hi


def job(sampler, model, y, noise, denoise_mask, sigmas, hp: O.Hyper, draw=cuda_draw, max_denoise=False,
        callback=None, early_stop=1, min_frac=1.0):
    """One job in y.dtype.  sampler: minicomfy.sample_euler / sample_heun.  denoise_mask: 1 = regenerate, of y's
    shape (or broadcastable).  sigmas: the fp32 schedule.  callback(i, denoised) per sampler step.  The model is
    called as model(x, sigma) and returns (x0 at cfg, x0 at cfg_BIG); model.inner_model.model_sampling has
    noise_scaling / inverse_noise_scaling."""
    dt, dev = y.dtype, y.device
    sig32 = sigmas.detach().to("cpu", torch.float32)
    sig = sig32.to(device=dev, dtype=dt)
    sampling = model.inner_model.model_sampling
    mask = O.binarise_mask(denoise_mask).to(dt)

    def wrapper(x, sigma, **kwargs):
        s32 = sigma.detach().to("cpu", torch.float32)
        tm = O.times_from_sigma(s32, hp.flow)
        n_eff = O.inner_steps_for(s32, sig32, tm.abt, hp.n_steps, early_stop, min_frac)
        tm = O.Times(*(t.to(device=dev, dtype=dt) for t in tm))
        denoised, x_new = O.outer_step(model, x, y, noise, sigma, mask, tm, hp, n_eff, draw)
        x.copy_(x_new)      # the per-sigma wrapper rewrites the sampler's x in place (nodes.py:300)
        return denoised

    x = sampling.noise_scaling(sig[0], noise, y, max_denoise)
    cb = None if callback is None else (lambda d: callback(d["i"], d["denoised"]))
    with torch.no_grad():
        x = sampler(wrapper, x, sig, callback=cb)
    return sampling.inverse_noise_scaling(sig[-1], x)


SAMPLERS = {"euler": minicomfy.sample_euler, "heun": minicomfy.sample_heun}
