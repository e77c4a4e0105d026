"""Host-scheduled sampling runs over the engine (SURVEY 8f rank 3).

`HostSchedule` does on the host, once per run, what the reference's per-sigma
wrapper recomputes on the device every outer step with two syncs
(src/LanPaint/nodes.py:242-252,286-299): the (VE sigma, abt, flow t) triple and
the effective inner-step count for every sigma of the schedule.
`euler_inpaint` is then the reference's `LanPaint_KSampler` run with sampler
"euler" (nodes.py:338,376-378 around k-diffusion's sample_euler) expressed as a
sync-free launch sequence.

`SynthDenoiser` is the SURVEY 8d pointwise two-head stand-in for the UNet/DiT,
running as one CUDA kernel (lp_synth_denoiser_f32); bench.py and the tests use it.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import List, Optional, Sequence

import torch

from . import _native
from .schedule import (ancestral_step, deis_step, dpm_2_step, dpmpp_2m_step, effective_inner_steps,
                       gradient_estimation_step, heun_step, res_multistep_step, times_from_sigma)


class VESampling:
    """EPS-type model_sampling: noise_scaling = y + sigma*noise (what nodes.py:338 relies on)."""

    def noise_scaling(self, sigma, noise, latent_image, max_denoise=False):
        if max_denoise:
            return noise * torch.sqrt(1.0 + sigma ** 2.0) + latent_image
        return latent_image + noise * sigma

    def inverse_noise_scaling(self, sigma, latent):
        return latent


class FlowSampling:
    """CONST-type (rectified flow) model_sampling."""

    noise_scale = 1.0

    def noise_scaling(self, sigma, noise, latent_image, max_denoise=False):
        return sigma * (self.noise_scale * noise) + (1.0 - sigma) * latent_image

    def inverse_noise_scaling(self, sigma, latent):
        return latent / (1.0 - sigma)


class SynthDenoiser:
    """x -> (a0 x + b0 tanh x + c0, a1 x + c1) as ONE kernel writing both heads.

    Follows the model protocol of the engine seam (`inner_model.model_sampling`,
    `__call__(x, t, model_options=, seed=)`).  Output buffers are reused, which is
    what a CUDA-graph-captured network does too."""

    def __init__(self, sampling=None, coef=(0.7, 0.1, 0.0, 0.6, -0.05), two_heads: bool = True,
                 dtype: torch.dtype = torch.float32):
        self.inner_model = self
        self.model_sampling = sampling or VESampling()
        self.coef = tuple(float(c) for c in coef)
        self._coef_c = (C.c_float * 5)(*self.coef)
        self.two_heads = two_heads
        self.dtype = dtype     # element type of the returned heads (a network computing in bf16 returns bf16)
        self._dtype_code = {torch.float32: _native.DTYPE_F32, torch.bfloat16: _native.DTYPE_BF16,
                            torch.float16: _native.DTYPE_F16}[dtype]
        self.calls = 0
        self._h0: Optional[torch.Tensor] = None
        self._h1: Optional[torch.Tensor] = None
        self._lib = _native.load()

    def set_coef(self, coef: Sequence[float]):
        self.coef = tuple(float(c) for c in coef)
        self._coef_c = (C.c_float * 5)(*self.coef)

    def __call__(self, x, t, model_options=None, seed=None):
        if self._h0 is None or self._h0.shape != x.shape or self._h0.device != x.device:
            self._h0 = torch.empty_like(x, dtype=self.dtype)
            self._h1 = torch.empty_like(x, dtype=self.dtype) if self.two_heads else None
        rc = self._lib.lp_synth_denoiser(C.c_void_p(x.data_ptr()), C.c_void_p(self._h0.data_ptr()),
                                         C.c_void_p(self._h1.data_ptr()) if self._h1 is not None else None,
                                         self._dtype_code, x.numel(), self._coef_c,
                                         C.c_void_p(torch.cuda.current_stream(x.device).cuda_stream))
        _native.check(rc, "lp_synth_denoiser")
        self.calls += 1
        return (self._h0, self._h1) if self.two_heads else self._h0


class SynthCondNet:
    """`denoiser(x, sigma, cond) -> x0` for a ComfyUI-style BaseModel (bench / tests): the same pointwise
    kernel as SynthDenoiser, one head per call, `cond` (a float standing in for CONDITIONING) shifts the
    output.  One output buffer per distinct cond, reused across calls like a captured network's."""

    def __init__(self, coef=(0.7, 0.1, 0.0)):
        self.coef = tuple(float(c) for c in coef)
        self._out = {}
        self._lib = _native.load()
        self.calls = 0

    def __call__(self, x, sigma, cond):
        c = float(cond)
        key = (c, tuple(x.shape), x.device)
        out = self._out.get(key)
        if out is None:
            out = self._out[key] = (torch.empty_like(x), (C.c_float * 5)(self.coef[0], self.coef[1], self.coef[2] + c, 0.0, 0.0))
        rc = self._lib.lp_synth_denoiser_f32(C.c_void_p(x.data_ptr()), C.c_void_p(out[0].data_ptr()), None, x.numel(),
                                             out[1], C.c_void_p(torch.cuda.current_stream(x.device).cuda_stream))
        _native.check(rc, "lp_synth_denoiser_f32")
        self.calls += 1
        return out[0]


@dataclass
class OuterStep:
    sigma: float
    sigma_next: float
    n_inner: int
    sigma_t: torch.Tensor    # CPU [B] fp32, what the sampler would pass as `sigma`
    times: tuple             # CPU (VE_Sigma, abt, Flow_t), reference op order (nodes.py:242-252)


class HostSchedule:
    """All per-sigma scalars of a run, computed once on the host."""

    def __init__(self, sigmas: Sequence[float], batch: int, n_inner: int, flow: bool = False,
                 early_stop: int = 1, min_step_frac: float = 1.0):
        sig = torch.as_tensor(list(sigmas), dtype=torch.float32)
        self.sigmas = sig
        host = [float(v) for v in sig]
        self._call = (batch, n_inner, flow, early_stop, min_step_frac)
        self.steps: List[OuterStep] = []
        ones = torch.ones(batch, dtype=torch.float32)
        for i in range(len(host) - 1):
            s = sig[i] * ones
            tm = times_from_sigma(s, flow)
            n_eff = effective_inner_steps(n_inner, host, float(torch.mean(s)), float((1.0 - tm[1]).mean()),
                                          early_stop, min_step_frac)
            self.steps.append(OuterStep(host[i], host[i + 1], n_eff, s, tm))
        self.substeps = sum(st.n_inner for st in self.steps)
        self.model_calls = self.substeps + len(self.steps)

    def call_at(self, sigma: float, sigma_next: float) -> OuterStep:
        """The row of a wrapper call at a sigma that need not be in the schedule (sample_dpm_2's midpoint): what the
        per-sigma wrapper derives from it -- sigma * ones[B], the times, and n_eff by its nearest-sigma rule."""
        batch, n_inner, flow, early_stop, min_step_frac = self._call
        s = torch.tensor(sigma, dtype=torch.float32) * torch.ones(batch, dtype=torch.float32)
        tm = times_from_sigma(s, flow)
        n_eff = effective_inner_steps(n_inner, [float(v) for v in self.sigmas], float(torch.mean(s)),
                                      float((1.0 - tm[1]).mean()), early_stop, min_step_frac)
        return OuterStep(float(s[0]), sigma_next, n_eff, s, tm)


def karras_sigmas(n: int, sigma_min: float = 0.0292, sigma_max: float = 14.6146, rho: float = 7.0) -> List[float]:
    """SDXL's karras schedule (SURVEY 8d), trailing 0 included."""
    ramp = torch.linspace(0, 1, n, dtype=torch.float32)
    lo, hi = sigma_min ** (1 / rho), sigma_max ** (1 / rho)
    s = (hi + ramp * (lo - hi)) ** rho
    return [float(v) for v in s] + [0.0]


def euler_inpaint(engine, latent_image: torch.Tensor, noise: torch.Tensor, mask, sched: HostSchedule,
                  x_out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """One full inpaint job on device-resident inputs; returns the final latent.

    mask: latent_mask (1 = known) tensor or an engine PackedMask."""
    sampling = engine.inner_model.inner_model.model_sampling
    x = sampling.noise_scaling(sched.sigmas[0].to(latent_image.device), noise, latent_image)
    for st in sched.steps:
        denoised = engine(x, latent_image, noise, st.sigma_t, mask, st.times, None, 0, n_steps=st.n_inner)
        # k-diffusion sample_euler: d = (x - denoised)/sigma ; x = x + d*(sigma_next - sigma)
        x = torch.add(x, x - denoised, alpha=(st.sigma_next - st.sigma) / st.sigma)
    if x_out is not None:
        x_out.copy_(x, non_blocking=True)
        return x_out
    return x


def _sampler_draw(engine, x: torch.Tensor) -> torch.Tensor:
    """The sampler's own `torch.randn_like(x)` on the engine's stream: the global generator itself for "torch", the
    next whole-tensor draw index of the same generator for "philox" (lp_fill_normal_f32)."""
    if engine.rng == "torch":
        return torch.randn_like(x)
    from .engine import _DrawPlan
    plan = _DrawPlan(engine.rng, x, 1)
    xi = torch.empty_like(x)
    r = plan.rng_struct(1)
    rc = _native.load().lp_fill_normal_f32(C.c_void_p(xi.data_ptr()), xi.numel(), C.byref(r),
                                           C.c_void_p(torch.cuda.current_stream(x.device).cuda_stream))
    _native.check(rc, "lp_fill_normal_f32")
    plan.finish()
    return xi


def euler_ancestral_inpaint(engine, latent_image: torch.Tensor, noise: torch.Tensor, mask, sched: HostSchedule,
                            eta: float = 1.0, s_noise: float = 1.0) -> torch.Tensor:
    """`euler_inpaint` with k-diffusion's sample_euler_ancestral as the sampler: the un-fused definition of
    GraphedJob(sampler="euler_ancestral"), eager torch ops and the sampler's own draw after every wrapper call."""
    sampling = engine.inner_model.inner_model.model_sampling
    x = sampling.noise_scaling(sched.sigmas[0].to(latent_image.device), noise, latent_image)
    for st in sched.steps:
        denoised = engine(x, latent_image, noise, st.sigma_t, mask, st.times, None, 0, n_steps=st.n_inner)
        s_down, s_up = ancestral_step(st.sigma, st.sigma_next, eta)
        d = (x - denoised) / st.sigma_t.to(x.device).reshape((-1,) + (1,) * (x.ndim - 1))
        x = x + d * (s_down - st.sigma)
        if st.sigma_next > 0:
            x = x + _sampler_draw(engine, x) * s_noise * s_up
    return x


def dpmpp_2m_inpaint(engine, latent_image: torch.Tensor, noise: torch.Tensor, mask, sched: HostSchedule) -> torch.Tensor:
    """`euler_inpaint` with k-diffusion's sample_dpmpp_2m as the sampler: the un-fused definition of
    GraphedJob(sampler="dpmpp_2m"), eager torch ops around every wrapper call with the sampler's own scalars
    (`dpmpp_2m_step` on the schedule, on the latent's device)."""
    sampling = engine.inner_model.inner_model.model_sampling
    x = sampling.noise_scaling(sched.sigmas[0].to(latent_image.device), noise, latent_image)
    old = None
    for st, (ratio, em1, c_cur, c_old, second) in zip(sched.steps, dpmpp_2m_step(sched.sigmas.to(latent_image.device))):
        denoised = engine(x, latent_image, noise, st.sigma_t, mask, st.times, None, 0, n_steps=st.n_inner)
        d = c_cur * denoised - c_old * old if second else denoised
        x = ratio * x - em1 * d
        old = denoised
    return x


def dpm_2_inpaint(engine, latent_image: torch.Tensor, noise: torch.Tensor, mask, sched: HostSchedule) -> torch.Tensor:
    """`euler_inpaint` with k-diffusion's sample_dpm_2 (no churn) as the sampler: the un-fused definition of
    GraphedJob(sampler="dpm_2"), eager torch ops around both wrapper calls of a step with the sampler's own scalars
    (`dpm_2_step` on the schedule, on the latent's device); the midpoint call's row is `HostSchedule.call_at`."""
    dev = latent_image.device
    sampling = engine.inner_model.inner_model.model_sampling
    sig = sched.sigmas.to(dev)
    x = sampling.noise_scaling(sig[0], noise, latent_image)
    for i, (st, (s_mid, dt_1, dt_2, mid)) in enumerate(zip(sched.steps, dpm_2_step(sig))):
        sigma_hat = sig[i] * (0.0 + 1)
        denoised = engine(x, latent_image, noise, st.sigma_t, mask, st.times, None, 0, n_steps=st.n_inner)
        d = (x - denoised) / sigma_hat
        if not mid:
            x = x + d * torch.tensor(dt_2, device=dev)
            continue
        x_2 = x + d * torch.tensor(dt_1, device=dev)
        ms = sched.call_at(s_mid, st.sigma_next)
        denoised_2 = engine(x_2, latent_image, noise, ms.sigma_t, mask, ms.times, None, 0, n_steps=ms.n_inner)
        x = x + ((x_2 - denoised_2) / torch.tensor(s_mid, device=dev)) * torch.tensor(dt_2, device=dev)
    return x


def heun_inpaint(engine, latent_image: torch.Tensor, noise: torch.Tensor, mask, sched: HostSchedule) -> torch.Tensor:
    """`euler_inpaint` with k-diffusion's sample_heun (no churn) as the sampler: the un-fused definition of
    GraphedJob(sampler="heun"), eager torch ops around both wrapper calls of a step with the sampler's own scalars
    (`heun_step` on the schedule, on the latent's device); the second call's row is `HostSchedule.call_at`."""
    dev = latent_image.device
    sampling = engine.inner_model.inner_model.model_sampling
    sig = sched.sigmas.to(dev)
    x = sampling.noise_scaling(sig[0], noise, latent_image)
    t = lambda v: torch.tensor(v, dtype=torch.float32, device=dev)   # noqa: E731
    for st, (sigma_hat, dt, sigma_next, corrector) in zip(sched.steps, heun_step(sig)):
        denoised = engine(x, latent_image, noise, st.sigma_t, mask, st.times, None, 0, n_steps=st.n_inner)
        d = (x - denoised) / t(sigma_hat)
        if not corrector:
            x = x + d * t(dt)
            continue
        x_2 = x + d * t(dt)
        ms = sched.call_at(sigma_next, st.sigma_next)
        denoised_2 = engine(x_2, latent_image, noise, ms.sigma_t, mask, ms.times, None, 0, n_steps=ms.n_inner)
        d_2 = (x_2 - denoised_2) / t(sigma_next)
        x = x + (d + d_2) / 2 * t(dt)
    return x


def deis_inpaint(engine, latent_image: torch.Tensor, noise: torch.Tensor, mask, sched: HostSchedule,
                 sampler_fn) -> torch.Tensor:
    """`euler_inpaint` with ComfyUI's sample_deis (max_order 3, 'tab') as the sampler: the un-fused definition of
    GraphedJob(sampler="deis"), eager torch ops around every wrapper call with the coefficients of `sampler_fn`'s own
    module (`deis_step`) and the derivative d = (x - denoised) / sigma divided by the device schedule's sigma."""
    dev = latent_image.device
    sampling = engine.inner_model.inner_model.model_sampling
    sig = sched.sigmas.to(dev)
    x = sampling.noise_scaling(sig[0], noise, latent_image)
    hist = []
    for i, (st, (_, c_cur, c_prev1, c_prev2, order)) in enumerate(zip(sched.steps, deis_step(sampler_fn, sig))):
        denoised = engine(x, latent_image, noise, st.sigma_t, mask, st.times, None, 0, n_steps=st.n_inner)
        d = (x - denoised) / sig[i]
        t = lambda v: torch.tensor(v, dtype=torch.float32, device=dev)   # noqa: E731
        x = x + t(c_cur) * d
        if order >= 2:
            x = x + t(c_prev1) * hist[-1]
        if order >= 3:
            x = x + t(c_prev2) * hist[-2]
        hist = (hist + [d])[-2:]
    return x


def res_multistep_inpaint(engine, latent_image: torch.Tensor, noise: torch.Tensor, mask,
                          sched: HostSchedule) -> torch.Tensor:
    """`euler_inpaint` with ComfyUI's sample_res_multistep (eta = 0) as the sampler: the un-fused definition of
    GraphedJob(sampler="res_multistep"), eager torch ops around every wrapper call with the sampler's own scalars
    (`res_multistep_step` on the schedule, on the latent's device).  The sampler's draw, multiplied by sigma_up = 0,
    adds a signed zero to every element and is not taken."""
    dev = latent_image.device
    sampling = engine.inner_model.inner_model.model_sampling
    x = sampling.noise_scaling(sched.sigmas[0].to(dev), noise, latent_image)
    t = lambda v: torch.tensor(v, dtype=torch.float32, device=dev)   # noqa: E731
    old = None
    for st, (second, a, b, c, e) in zip(sched.steps, res_multistep_step(sched.sigmas.to(dev))):
        denoised = engine(x, latent_image, noise, st.sigma_t, mask, st.times, None, 0, n_steps=st.n_inner)
        if second:     # a, b, c, e = sigma_fn(h), -h, b1, -b2
            x = t(a) * x + t(-b) * (t(c) * denoised + t(-e) * old)
        else:          # a, b = sigma_i, sigma_next - sigma_i
            x = x + ((x - denoised) / t(a)) * t(b)
        old = denoised
    return x


def gradient_estimation_inpaint(engine, latent_image: torch.Tensor, noise: torch.Tensor, mask,
                                sched: HostSchedule) -> torch.Tensor:
    """`euler_inpaint` with ComfyUI's sample_gradient_estimation (ge_gamma = 2) as the sampler: the un-fused definition
    of GraphedJob(sampler="gradient_estimation"), eager torch ops around every wrapper call with the sampler's own
    scalars (`gradient_estimation_step` on the schedule, on the latent's device)."""
    dev = latent_image.device
    sampling = engine.inner_model.inner_model.model_sampling
    x = sampling.noise_scaling(sched.sigmas[0].to(dev), noise, latent_image)
    t = lambda v: torch.tensor(v, dtype=torch.float32, device=dev)   # noqa: E731
    old_d = None
    for st, (sigma, dt, gm1, reads, final, _) in zip(sched.steps, gradient_estimation_step(sched.sigmas.to(dev))):
        denoised = engine(x, latent_image, noise, st.sigma_t, mask, st.times, None, 0, n_steps=st.n_inner)
        d = (x - denoised) / t(sigma)
        if final:
            x = denoised
        else:
            x = x + d * t(dt)
            if reads:
                x = x + (gm1 * (d - old_d)) * t(dt)
        old_d = d
    return x


def time_steady_substep(engine, latent_image: torch.Tensor, mask, sigma: float, launches: int = 53,
                        repeats: int = 20, flow: bool = False, rotate: int = 3):
    """Roofline probe: `launches` steady fused sub-step launches (flags = FUSE_NEXT, the kernel that
    dominates a job) back to back on job-shaped operands, between two CUDA events on the launching
    stream, `repeats` times.  Returns the list of per-launch durations in microseconds (one per repeat).

    `rotate` independent operand sets (x, x0, x0_BIG, y, C, mask) are cycled, so a launch's operands were
    last touched `rotate - 1` launches ago: with 176 MB per set at the bench's default size that is far more
    than the 50 MB L2 of an H100 can hold, i.e. every launch really streams from HBM (rotate=1 re-uses one set and lets
    the L2 keep part of it -- reported separately as the L2-assisted figure).  The launches are identical to
    those `LanPaint._launch_sequence` issues, minus the model call between them."""
    import numpy as np
    from .engine import PackedMask, _DrawPlan, pack_mask
    from .schedule import Hyper, build_table
    lib = _native.load()
    dev = latent_image.device
    B = latent_image.shape[0]
    pm0 = mask if isinstance(mask, PackedMask) else pack_mask(mask, latent_image)
    sets = []
    for r in range(max(1, rotate)):
        x = torch.randn_like(latent_image)
        heads = engine.inner_model(x, torch.full((B,), sigma, device=dev))
        x0, x0b = engine.unpack_model_output(heads)
        sets.append(dict(x=x, x0=x0.clone(), x0b=x0b.clone(), y=latent_image if r == 0 else latent_image.clone(),
                         c=torch.randn_like(x), m=pm0.data if r == 0 else pm0.data.clone()))
    s = torch.full((B,), sigma, dtype=torch.float32)
    ve, abt, _ = times_from_sigma(s, flow)
    hp = Hyper(engine.step_size, engine.chara_lamb, engine.chara_beta, engine.min_step_frac, flow)
    tab = torch.from_numpy(build_table(abt.numpy(), ve.numpy(), hp)).to(dev)
    per_row = latent_image.numel() // B
    spatial = int(np.prod(latent_image.shape[2:]))
    dims = _native.Dims(B, per_row, spatial, pm0.row_stride, pm0.channel_stride)
    plan = _DrawPlan(engine.rng, latent_image, launches + 1)
    merge = plan.mode == _native.RNG_PHILOX and engine.merge_noise
    flags = _native.SUBSTEP_FUSE_NEXT | (_native.SUBSTEP_MERGE_NOISE if merge else 0)
    P = C.c_void_p
    stream = P(torch.cuda.current_stream(dev).cuda_stream)

    from .engine import _heads
    for o in sets:   # heads in whatever dtype the model returns (fp32 / bf16 / fp16)
        o["heads"], o["keep"] = _heads(o["x0"], o["x0b"], o["x"])

    def burst():
        for k in range(launches):
            o = sets[k % len(sets)]
            r = plan.rng_struct(1 if merge else 2)
            rc = lib.lp_substep(P(o["x"].data_ptr()), C.byref(o["heads"]), P(o["y"].data_ptr()), P(o["m"].data_ptr()),
                                P(o["c"].data_ptr()), None, None, P(tab.data_ptr()), C.byref(dims), C.byref(r), flags,
                                stream)
            _native.check(rc, "lp_substep")

    for _ in range(3):
        burst()
    torch.cuda.synchronize(dev)
    out = []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        burst()
        e1.record()
        e1.synchronize()
        out.append(1e3 * e0.elapsed_time(e1) / launches)
    return out


class GraphedJob:
    """A whole inpaint job -- initial noise_scaling, every outer step (prologue, model calls, fused
    sub-steps, epilogue) and the Euler updates between them -- on static buffers, launched in one of
    three ways that share ONE body (`_step`):

      mode "job"    the whole job is ONE CUDA graph (captured once, replayed per batch of requests); with a callback
                    every outer step writes its denoised latent to its own buffer and the callbacks run, in order,
                    after the replay (for jobs so short that nobody can watch a progress bar move);
      mode "steps"  one CUDA graph per outer step, replayed in order with a host callback between them
                    (ComfyUI's progress / preview callback wants the denoised latent of every step);
      mode "eager"  plain launches (the first job of a configuration: nothing is wasted on warm-up).

    Everything sigma-dependent is a device constant computed at construction (one coefficient table per
    outer step), so a replay costs one 16-byte H2D copy (the RNG position) plus the copies of the
    request's own inputs.  Used directly by hosts that own the sampler loop (serving: fixed schedule,
    fixed batch shape, a stream of request batches) and by the node path (`comfy_nodes.KSAMPLER.sample`)
    whenever the ComfyUI sampler is plain Euler, the configuration the reference recommends
    (src/LanPaint/nodes.py:459 "Recommended: euler").

    Semantics are exactly `euler_inpaint(engine, ...)`, i.e. k-diffusion's sample_euler around the
    per-sigma wrapper (asserted bit-for-bit by the tests); sampler="euler_ancestral", "dpmpp_2m", "dpm_2" and "deis" are
    `euler_ancestral_inpaint`, `dpmpp_2m_inpaint`, `dpm_2_inpaint` and `deis_inpaint`.  dpm_2 makes two wrapper calls
    per outer step: call A at sigma_i on x, call B at the midpoint sigma on a second state buffer x2; both are in the
    step's graph.  sampler="heun" (with `sampler_fn`, the sample_heun the loop stands in for) is `heun_inpaint` and has
    the same two calls, call B at sigma_next; its corrector (lp_boundary_heun) also reads call A's denoised latent, which
    call A therefore always writes.  deis takes its
    coefficients from the sampler function `sampler_fn` (ComfyUI's sample_deis or a stand-in with a `deis` module
    beside it).  sampler="res_multistep" (eta = 0) and "gradient_estimation" (ge_gamma = 2) are `res_multistep_inpaint`
    and `gradient_estimation_inpaint`."""

    def __init__(self, engine, sched: HostSchedule, shape, device, flow: bool = False, fused_euler: bool = True,
                 l2_persist: bool = False, model_options=None, seed=0, external_init: bool = False,
                 first_replace_noop=None, sampler: str = "euler", eta: float = 1.0, s_noise: float = 1.0,
                 sampler_fn=None):
        import numpy as np
        from .engine import _DrawPlan
        if sampler not in ("euler", "euler_ancestral", "dpmpp_2m", "dpm_2", "heun", "deis", "res_multistep",
                           "gradient_estimation"):
            raise ValueError("GraphedJob owns the loops of 'euler', 'euler_ancestral', 'dpmpp_2m', 'dpm_2', 'heun', "
                             f"'deis', 'res_multistep' and 'gradient_estimation', not {sampler!r}")
        if sampler == "deis" and sampler_fn is None:
            raise ValueError("GraphedJob(sampler='deis') needs the sampler function (sampler_fn): the coefficients are "
                             "its module's")
        if sampler == "heun" and getattr(sampler_fn, "__name__", "") != "sample_heun":
            # the loop restates one sampler function, sample_heun without churn and without draws of its own; the caller
            # names the function it checked (the node gate's `_restates`), and another one -- heunpp2, say -- is refused
            raise ValueError("GraphedJob(sampler='heun') needs the sample_heun it restates (sampler_fn), run without "
                             "churn and checked to draw nothing of its own")
        self.sampler = sampler
        self.fused_euler = fused_euler   # the sampler's update inside the step-boundary kernel instead of torch kernels
        # optional persisting-L2 window over the clean latent (re-read by every launch).  Off by default: the
        # set-aside takes L2 away from absorbing the sub-step's writes, which can cost more than the y hits give back
        self.l2_persist = l2_persist
        self.l2_window = 0
        from .schedule import Hyper, build_table, mean_half_dt
        if engine.rng not in ("philox", "torch"):
            raise ValueError("GraphedJob needs an in-kernel RNG mode ('philox' or 'torch')")
        self.engine, self.sched, self.flow = engine, sched, flow
        self.model_options, self.seed = model_options, seed
        self.external_init = external_init   # run(x_init=...) supplies the initial state (node path: max_denoise etc.)
        self.device = torch.device(device)
        self.shape = tuple(shape)
        B = self.shape[0]
        dev = self.device
        mk = lambda: torch.empty(self.shape, dtype=torch.float32, device=dev)
        self.x, self.y, self.noise, self.c, self.out = mk(), mk(), mk(), mk(), mk()
        # dpmpp_2m writes every step's denoised latent and reads it back at the next step: two buffers taken in turn
        self.out_pair = (self.out, mk()) if sampler in ("dpmpp_2m", "res_multistep") else None
        # dpm_2 and heun: the state of the step's second call (x_2 of the sampler)
        self.x2 = mk() if sampler in ("dpm_2", "heun") else None
        self.mask = None
        hyper = Hyper(engine.step_size, engine.chara_lamb, engine.chara_beta, engine.min_step_frac, flow)

        def call_row(st):
            """(table, model time, sigma, active sub-steps) of one wrapper call"""
            ve, abt, flow_t = (t.numpy() for t in st.times)
            sig = st.sigma_t.numpy()
            form = engine._replace_form(sig, st.sigma_t.numel() == 1, B, engine.replace_mode, engine.batched_replace)
            if form is None:
                raise ValueError("model_sampling.noise_scaling is not a linear form; GraphedJob cannot precompute it")
            return (build_table(abt, ve, hyper, form[0], form[1]), flow_t if flow else ve, sig,
                    st.n_inner if mean_half_dt(abt, hyper) > 0.0 else 0)

        tabs, tms, sgs, self.active = [], [], [], []
        for st in sched.steps:
            tab, tm, sig, active = call_row(st)
            tabs.append(tab)
            tms.append(tm)
            sgs.append(sig)
            self.active.append(active)
        # draws consumed before outer step i (1 for sub-step 0, 2 for each later one): lets every outer step be
        # captured on its own against ONE {seed, base} block that is refreshed once per job
        merged = engine.rng == "philox" and engine.merge_noise   # a fused launch then draws ONE normal, not two
        # euler_ancestral: one lp_ancestral per outer step, and the sampler's randn_like -- taken whenever
        # sigma_next > 0, whatever eta makes of sigma_up -- as one more draw after the step's Langevin draws
        self.ancestral = None
        if sampler == "euler_ancestral":
            self.ancestral = []
            for st in sched.steps:
                s_down, s_up = ancestral_step(st.sigma, st.sigma_next, eta)
                self.ancestral.append((_native.Ancestral(st.sigma, s_down - st.sigma, s_noise, s_up),
                                       st.sigma_next > 0))
        # dpmpp_2m: one lp_multistep per outer step (the sampler's scalars from its own expressions on this device),
        # and whether the step is second order, i.e. reads the previous step's denoised latent.  No draw of its own
        self.multistep = None
        if sampler == "dpmpp_2m":
            self.multistep = [(_native.Multistep(ratio, em1, c_cur, c_old), second)
                              for ratio, em1, c_cur, c_old, second in dpmpp_2m_step(sched.sigmas.to(dev))]
        # res_multistep: the same, its second-order steps as lp_multistep and its Euler steps (the first one, the step
        # to sigma = 0) as lp_midpoint on x alone; the scalars also as device tensors for the un-fused update.  Its draw
        # is multiplied by sigma_up = 0 and not taken
        if sampler == "res_multistep":
            rows = res_multistep_step(sched.sigmas.to(dev))
            self.multistep = [(_native.Multistep(*v) if second else _native.Midpoint(v[0], v[1]), second)
                              for second, *v in rows]
            self.res_scalars = torch.tensor([v for _, *v in rows], dtype=torch.float32, device=dev)
        # dpm_2 and heun: per outer step (lp_midpoint of call A's update, call B's update -- lp_midpoint for dpm_2,
        # lp_heun for heun -- or None, the index of call B's row), the rows of the second calls (their own tables, model
        # times, sigmas and active counts), and the sampler's scalars (call A's sigma and dt, call B's) as device tensors
        # for the un-fused update.  No draw of their own
        self.midpoint = None
        self.substeps = sched.substeps
        if sampler in ("dpm_2", "heun"):
            sig_dev = sched.sigmas.to(dev)
            if sampler == "dpm_2":
                calls = [(_native.Midpoint(st.sigma, dt_1 if mid else dt_2), s_mid if mid else None,
                          _native.Midpoint(s_mid, dt_2), (s_mid, dt_2))
                         for st, (s_mid, dt_1, dt_2, mid) in zip(sched.steps, dpm_2_step(sig_dev))]
            else:      # call B at sigma_next, the next outer step's row whenever there is one
                calls = [(_native.Midpoint(s, dt), s_next if corr else None, _native.Heun(s, s_next, dt), (s_next, dt))
                         for s, dt, s_next, corr in heun_step(sig_dev)]
            self.midpoint, mrows, scalars = [], [], []
            for st, (pred, s_b, corr, sc_b) in zip(sched.steps, calls):
                scalars.append([pred.sigma, pred.dt] + (list(sc_b) if s_b is not None else [0.0, 0.0]))
                if s_b is None:
                    self.midpoint.append((pred, None, None))
                    continue
                ms = sched.call_at(s_b, st.sigma_next)
                self.substeps += ms.n_inner
                self.midpoint.append((pred, corr, len(mrows)))
                mrows.append(call_row(ms))
            col = lambda j: (torch.from_numpy(np.stack([r[j] for r in mrows]).astype(np.float32)).to(dev)  # noqa: E731
                             if mrows else None)
            self.mid_tables, self.mid_t_model, self.mid_sigma = col(0), col(1), col(2)
            self.mid_active = [r[3] for r in mrows]
            self.call_scalars = torch.tensor(scalars, dtype=torch.float32, device=dev)
            self.out_mid = mk() if not fused_euler else None   # call B's denoised latent (un-fused update)
        # deis: per outer step (lp_deis, order, whether a later step reads its derivative), the coefficients read back
        # once here, and a ring of three derivative buffers: step i writes d_ring[i % 3] and reads the two before it,
        # so every per-step graph bakes in a fixed triple.  No draw of its own
        self.deis = self.d_ring = None
        if sampler == "deis":
            rows = deis_step(sampler_fn, sched.sigmas)
            self.deis = [(_native.Deis(sigma, c_cur, c_prev1, c_prev2), order, i + 1 < len(rows) and rows[i + 1][4] >= 2)
                         for i, (sigma, c_cur, c_prev1, c_prev2, order) in enumerate(rows)]
            self.d_ring = (mk(), mk(), mk())
            self.deis_scalars = torch.tensor([r[:4] for r in rows], dtype=torch.float32, device=dev)
        # gradient_estimation: per outer step (lp_gradient_estimation, whether it reads the previous step's d, whether a
        # later step reads its own), and a ring of two derivative buffers: step i writes d_ring[i % 2] and reads
        # d_ring[(i - 1) % 2], so every per-step graph bakes in a fixed pair.  No draw of its own
        self.ge = None
        if sampler == "gradient_estimation":
            rows = gradient_estimation_step(sched.sigmas.to(dev))
            self.ge = [(_native.GradientEstimation(sigma, dt, gm1, int(final)), reads, keep)
                       for sigma, dt, gm1, reads, final, keep in rows]
            self.d_ring = (mk(), mk())
            self.ge_scalars = torch.tensor([r[:2] for r in rows], dtype=torch.float32, device=dev)
        draws = lambda n: 0 if n <= 0 else (n if merged else 2 * n - 1)   # noqa: E731  one wrapper call's draws
        self._call_draws = draws
        self.draws_before = [0]
        for i, n in enumerate(self.active):
            own = 1 if (self.ancestral is not None and self.ancestral[i][1]) else 0
            if self.midpoint is not None and self.midpoint[i][2] is not None:
                own = draws(self.mid_active[self.midpoint[i][2]])     # call B's Langevin draws
            self.draws_before.append(self.draws_before[-1] + draws(n) + own)
        self.tables = torch.from_numpy(np.stack(tabs)).to(dev)
        self.t_model = torch.from_numpy(np.stack(tms).astype(np.float32)).to(dev)
        self.sigma = torch.from_numpy(np.stack(sgs).astype(np.float32)).to(dev)
        self.sigma0 = torch.tensor(float(sched.sigmas[0]), device=dev)
        self.rng_state = torch.zeros(2, dtype=torch.int64, device=dev)
        if first_replace_noop is None:
            # the first replace step is a no-op when the replace form is noise_scaling's own form at sigmas[0]
            # (every known position of x already holds it); the reference's batched flow-form quirk differs
            first_replace_noop = (not external_init) and (B == 1 or engine.batched_replace == "per_sample")
        self.first_replace_noop = bool(first_replace_noop) and fused_euler
        self._graphs = {}
        self._dims = None
        self.timing, self.last_events = False, None
        self.first_step_end = None   # mode "eager": an event recorded after the first outer step
        self.outs = None     # per-outer-step denoised latents (mode "job" with a callback: callbacks run after the replay)
        self._outs = {}      # observe setting -> its `outs`, kept as long as the graphs that write them
        self.launches = 0
        self.model_calls = 0
        self.captures = 0
        self._plan_cls = _DrawPlan

    @property
    def draws(self) -> int:
        return self.draws_before[-1]

    @property
    def graph(self):
        """The whole-job graph (None until the first mode="job" run)."""
        return self._graphs.get(("job", False, "full"))

    def per_step_bytes(self) -> int:
        return len(self.sched.steps) * self.x.numel() * 4

    def denoised_buffer(self, i: int, want_out) -> torch.Tensor:
        """Where outer step i writes its denoised latent (mode "job" with a callback: its own buffer, see `_observed`)."""
        if want_out == "each":
            return self.outs[i]
        return self.out_pair[i % 2] if self.out_pair is not None else self.out

    def _out_whole(self, i: int) -> bool:
        """Whether outer step i stores its whole denoised latent whatever the callback reads: a later launch reads it
        (the un-fused update, the multistep samplers' next step, heun's corrector), or its boundary,
        lp_boundary_multistep, has no row-bounded form."""
        if not self.fused_euler:
            return True
        if self.multistep is not None:
            read = i + 1 < len(self.sched.steps) and self.multistep[i + 1][1]
            return read or not isinstance(self.multistep[i][0], _native.Midpoint)
        return self.sampler == "heun" and self.midpoint[i][2] is not None

    def _observed(self, observe: str):
        """`outs` of mode "job" with a callback: per outer step, the buffer its denoised latent goes to.  "full": every
        step's whole latent.  "preview": before the last step, only row 0 -- all a latent preview decodes -- into a
        [1, ...] buffer; "final": nothing.  The last step, and every step `_out_whole` names, keep the whole latent."""
        if observe not in ("full", "preview", "final"):
            raise ValueError(f"unknown observe setting {observe!r}")
        outs = self._outs.get(observe)
        if outs is None:
            n = len(self.sched.steps)
            outs = []
            for i in range(n):
                if observe == "full" or i + 1 == n or self._out_whole(i):
                    outs.append(torch.empty_like(self.x))
                elif observe == "preview":
                    outs.append(torch.empty((1,) + self.shape[1:], dtype=torch.float32, device=self.device))
                else:
                    outs.append(None)
            self._outs[observe] = outs
        return outs

    def _out_rows(self, out):
        """The out_rows argument of a boundary that writes `out`: None (every row) unless `out` holds fewer rows."""
        return out.shape[0] if out is not None and out.shape[0] < self.shape[0] else None

    # ---- the body ------------------------------------------------------------------------------
    def _init_state(self):
        sampling = self.engine.inner_model.inner_model.model_sampling
        self.x.copy_(sampling.noise_scaling(self.sigma0, self.noise, self.y))

    def _step(self, i, plan, want_out):
        if self.midpoint is not None:
            return self._two_call_step(i, plan, want_out)
        eng = self.engine
        st = self.sched.steps[i]
        coef = (st.sigma_next - st.sigma) / st.sigma
        anc = self.ancestral[i] if self.ancestral is not None else None
        ms, old, dz, ge = None, None, None, None
        if self.multistep is not None:
            ms = self.multistep[i]
            old = self.denoised_buffer(i - 1, want_out) if ms[1] else None
        euler_mp = ms is not None and isinstance(ms[0], _native.Midpoint)   # a res_multistep Euler step
        if self.deis is not None:     # (lp_deis, d_out, d_prev1, d_prev2)
            step, order, keep = self.deis[i]
            ring = self.d_ring
            dz = (step, ring[i % 3] if keep else None, ring[(i - 1) % 3] if order >= 2 else None,
                  ring[(i - 2) % 3] if order >= 3 else None)
        if self.ge is not None:       # (lp_gradient_estimation, d_out, d_prev)
            step, reads, keep = self.ge[i]
            ge = (step, self.d_ring[i % 2] if keep else None, self.d_ring[(i - 1) % 2] if reads else None)
        last = i + 1 == len(self.sched.steps)
        plan.used = self.draws_before[i]
        out = self.out if (want_out or not self.fused_euler) else None
        if want_out == "each" or ms is not None:      # every outer step keeps its own denoised latent
            out = self.denoised_buffer(i, want_out)
        from .engine import heads_discardable
        # the job owns every network call it makes, and the next one overwrites what the last update read
        eng._launch_sequence(self.x, self.y, self.noise, self.mask, self._dims, self.tables[i], self.t_model[i],
                             self.sigma[i], self.c, out, self.active[i], plan, False, self.model_options, self.seed,
                             None, self.rng_state.data_ptr(), discard_heads=heads_discardable(self.model_options),
                             euler_coef=coef if (self.fused_euler and anc is None and ms is None and dz is None
                                                 and ge is None) else None,
                             skip_prologue=(self.fused_euler and i > 0) or (i == 0 and self.first_replace_noop),
                             next_table=self.tables[i + 1] if (self.fused_euler and not last) else None,
                             ancestral=anc if self.fused_euler else None,
                             multistep=(ms[0], old) if (self.fused_euler and ms is not None and not euler_mp) else None,
                             midpoint=(ms[0], self.x, self.x) if (self.fused_euler and euler_mp) else None,
                             deis=dz if self.fused_euler else None, ge=ge if self.fused_euler else None,
                             out_rows=self._out_rows(out))
        if self.fused_euler:
            return
        if self.sampler == "res_multistep":     # sample_res_multistep's tensor ops, in its order
            sc = self.res_scalars[i]
            if euler_mp:
                self.x.copy_(self.x + ((self.x - out) / sc[0]) * sc[1])
            else:     # sigma_fn(h) * x + h * (b1 * denoised + b2 * old_denoised), h = -em1, b2 = -c_old
                self.x.copy_(sc[0] * self.x + (-sc[1]) * (sc[2] * out + (-sc[3]) * old))
            return
        if ge is not None:     # sample_gradient_estimation's tensor ops, in its order
            step, d_out, d_prev = ge
            sc = self.ge_scalars[i]
            d = (self.x - out) / sc[0]
            if step.final:
                self.x.copy_(out)
            else:
                x = self.x + d * sc[1]
                if d_prev is not None:
                    x = x + (step.gm1 * (d - d_prev)) * sc[1]
                self.x.copy_(x)
            if d_out is not None:
                d_out.copy_(d)
            return
        if dz is not None:     # sample_deis's tensor ops, in its order
            sc = self.deis_scalars[i]
            d = (self.x - out) / sc[0]
            x = self.x + sc[1] * d
            if dz[2] is not None:
                x = x + sc[2] * dz[2]
            if dz[3] is not None:
                x = x + sc[3] * dz[3]
            self.x.copy_(x)
            if dz[1] is not None:
                dz[1].copy_(d)
            return
        # un-fused: from this step's denoised latent, wherever it was written
        if ms is not None:     # sample_dpmpp_2m's tensor ops, in its order
            step = ms[0]
            d = out * step.c_cur - old * step.c_old if old is not None else out
            self.x.mul_(step.ratio).sub_(d * step.em1)
            return
        if anc is None:
            self.x.add_(self.x - out, alpha=coef)
            return
        step, draws = anc
        d = (self.x - out) / self.sigma[i].reshape((-1,) + (1,) * (self.x.ndim - 1))
        self.x.add_(d * step.down)
        if draws:   # torch.randn_like's values at the plan's position, by a capturable launch
            xi = torch.empty_like(self.x)
            r = plan.rng_struct(1, self.rng_state.data_ptr())
            rc = _native.load().lp_fill_normal_f32(C.c_void_p(xi.data_ptr()), xi.numel(), C.byref(r),
                                                   C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream))
            _native.check(rc, "lp_fill_normal_f32")
            self.x.add_(xi * step.s_noise * step.sigma_up)

    def _two_call_step(self, i, plan, want_out):
        """Outer step i of sample_dpm_2 or sample_heun: call A at sigma_i on x, then (sigma_next > 0) call B on x2 --
        at sigma_mid for dpm_2, at sigma_next for heun.  Fused, call A's boundary is the predictor (x -> x2) with call
        B's replace step (its row) folded in, and call B's boundary is the corrector (x2, x -> x; heun's also reads call
        A's denoised latent) with the next outer step's replace step; the step to sigma = 0 is one Euler boundary on
        x."""
        from .engine import heads_discardable
        eng = self.engine
        pred, corr, k = self.midpoint[i]
        heun = self.sampler == "heun"
        last = i + 1 == len(self.sched.steps)
        fused = self.fused_euler
        after = self.tables[i + 1] if not last else None     # the next outer step's replace step
        plan.used = self.draws_before[i]
        # heun's corrector reads call A's denoised latent, so call A writes it whenever there is a call B
        out = self.out if (want_out or not fused or (heun and k is not None)) else None
        if want_out == "each":
            out = self.outs[i]
        dead = heads_discardable(self.model_options)
        common = (self.y, self.noise, self.mask, self._dims)
        x_a = self.x2 if k is not None else self.x
        eng._launch_sequence(self.x, *common, self.tables[i], self.t_model[i], self.sigma[i], self.c, out,
                             self.active[i], plan, False, self.model_options, self.seed, None,
                             self.rng_state.data_ptr(), discard_heads=dead,
                             skip_prologue=(fused and i > 0) or (i == 0 and self.first_replace_noop),
                             next_table=(self.mid_tables[k] if k is not None else after) if fused else None,
                             midpoint=(pred, self.x, x_a) if fused else None, out_rows=self._out_rows(out))
        sc = self.call_scalars[i]
        if not fused:   # the sampler's tensor ops, in its order
            d = (self.x - out) / sc[0]
            if k is None:
                self.x.add_(d * sc[1])
                return
            torch.add(self.x, d * sc[1], out=self.x2)
        if k is None:
            return
        plan.used = self.draws_before[i] + self._call_draws(self.active[i])
        update = dict(heun=(corr, self.x, out)) if heun else dict(midpoint=(corr, self.x, self.x))
        eng._launch_sequence(self.x2, *common, self.mid_tables[k], self.mid_t_model[k], self.mid_sigma[k], self.c,
                             None if fused else self.out_mid, self.mid_active[k], plan, False, self.model_options,
                             self.seed, None, self.rng_state.data_ptr(), discard_heads=dead, skip_prologue=fused,
                             next_table=after if fused else None, **(update if fused else {}))
        if fused:
            return
        d_2 = (self.x2 - self.out_mid) / sc[2]
        if heun:
            self.x.copy_(self.x + (d + d_2) / 2 * sc[3])
        else:
            self.x.add_(d_2 * sc[3])

    def _body(self, plan, want_out):
        if not self.external_init:
            self._init_state()
        for i in range(len(self.sched.steps)):
            self._step(i, plan, want_out)

    def _relative_plan(self):
        return self._plan_cls(self.engine.rng, self.x, 1).relative()

    def _capture(self, fn, warm: bool):
        """Capture `fn(plan)` into a CUDA graph.  warm=True first runs it once on a side stream (lazy
        initialisation of whatever the model uses); the node path passes warm=False because the same body has
        already run eagerly as the previous job."""
        eng = self.engine
        counts = (eng.launches, eng.model_calls, eng.substeps_done)
        timer, eng.kernel_timer = eng.kernel_timer, None
        plan = self._relative_plan()   # built BEFORE capture begins: reading the generator's offset is not capturable
        try:
            if warm:
                # the warm-up pass really runs the captured steps: put the sampler state back afterwards, or an outer
                # step captured on its own (mode "steps"), or a job whose initial state was loaded from x_init, would
                # then be applied twice
                state = self.x.clone()
                side = torch.cuda.Stream(device=self.device)
                side.wait_stream(torch.cuda.current_stream(self.device))
                with torch.cuda.stream(side):
                    fn(plan)
                torch.cuda.current_stream(self.device).wait_stream(side)
                self.x.copy_(state)
                eng.launches, eng.model_calls, eng.substeps_done = counts
            graph = torch.cuda.CUDAGraph()
            lib = _native.load()
            cap_stream = torch.cuda.Stream(device=self.device)
            cap = C.c_void_p(cap_stream.cuda_stream)
            if self.l2_persist:   # configured before capture begins; the window then rides on every captured kernel node
                nbytes = self.y.numel() * 4
                if lib.lp_l2_persist_set(C.c_void_p(self.y.data_ptr()), nbytes, cap) == 0:
                    self.l2_window = nbytes
            cap_stream.wait_stream(torch.cuda.current_stream(self.device))
            with torch.cuda.graph(graph, stream=cap_stream):
                fn(plan)
            if self.l2_window:
                lib.lp_l2_persist_clear(cap)
        finally:
            eng.kernel_timer = timer
        stats = (eng.launches - counts[0], eng.model_calls - counts[1])
        eng.launches, eng.model_calls, eng.substeps_done = counts
        self.captures += 1
        return graph, stats

    def _graph_for(self, key, fn, warm):
        g = self._graphs.get(key)
        if g is None:
            g = self._graphs[key] = self._capture(fn, warm)
        return g

    # ---- one job ---------------------------------------------------------------------------------
    def load_inputs(self, latent_image: torch.Tensor, noise: torch.Tensor, mask, x_init=None):
        """Copies of the request's own inputs into the static buffers (H2D when they are host tensors)."""
        import numpy as np
        from .engine import PackedMask, pack_known, pack_mask
        self.y.copy_(latent_image, non_blocking=True)
        if noise is None:   # serving hosts that do not need ComfyUI's CPU noise image: draw it on the device
            self.noise.normal_()
        else:
            self.noise.copy_(noise, non_blocking=True)
        if x_init is not None:
            self.x.copy_(x_init, non_blocking=True)
        pm = mask if isinstance(mask, PackedMask) else pack_mask(mask, self.x)
        if self.mask is None or self.mask.data.shape != pm.data.shape or (
                self.mask.row_stride, self.mask.channel_stride) != (pm.row_stride, pm.channel_stride):
            self.mask = PackedMask(torch.empty_like(pm.data), pm.row_stride, pm.channel_stride)
            self._graphs = {}
        self.mask.data.copy_(pm.data, non_blocking=True)
        B = self.shape[0]
        self._dims = _native.Dims(B, self.x.numel() // B, int(np.prod(self.shape[2:])), self.mask.row_stride,
                                  self.mask.channel_stride)
        # y and the noise image at known positions only, for the kernels that stream them (same buffers every job)
        self.mask.known = pack_known(self.mask, self._dims, self.y, self.noise, out=self.mask.known)

    def run(self, latent_image: torch.Tensor, noise: torch.Tensor, mask, x_out: Optional[torch.Tensor] = None,
            x_init: Optional[torch.Tensor] = None, callback=None, mode: Optional[str] = None, warm: bool = True,
            observe: str = "full"):
        """callback(i, denoised, x, total_steps) is called on the host after outer step i has been ENQUEUED
        (it sees device tensors in stream order; a callback that only counts steps never synchronises).

        observe (mode "job" with a callback): what of each step's denoised latent the callback is handed, see
        `_observed` -- "full", "preview" (before the last step, the [1, ...] latent of the first request) or "final"
        (before the last step, an empty [0, ...] tensor).  The last step's is always whole."""
        import numpy as np
        eng = self.engine
        if self.external_init != (x_init is not None):
            raise ValueError("x_init must be given exactly when the job was built with external_init=True")
        if mode is None:
            mode = "steps" if callback is not None else "job"
        if mode not in ("job", "steps", "eager"):
            raise ValueError(f"unknown mode {mode!r}")
        with torch.cuda.device(self.device):
            before = (eng.launches, eng.model_calls)
            self.load_inputs(latent_image, noise, mask, x_init)
            plan = self._plan_cls(eng.rng, self.x, 1)
            self.rng_state.copy_(torch.from_numpy(plan.state_words().view(np.int64)))
            if self.timing:   # device time of the sampler loop proper: inputs resident, first kernel -> last kernel
                self.last_events = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
                self.last_events[0].record()
            n_steps = len(self.sched.steps)
            want_out = callback is not None
            if mode == "job":
                if want_out:
                    self.outs = self._observed(observe)
                else:
                    observe = "full"
                each = "each" if want_out else False
                graph, stats = self._graph_for(("job", each, observe), lambda p: self._body(p, each), warm)
                graph.replay()
                eng.launches += stats[0]
                eng.model_calls += stats[1]
                if callback is not None:
                    for i in range(n_steps):
                        out = self.outs[i]
                        callback(i, out if out is not None else self.outs[-1][:0], self.x, n_steps)
            elif mode == "steps":
                if not self.external_init:
                    self._init_state()
                for i in range(n_steps):
                    graph, stats = self._graph_for(("step", i, want_out), lambda p, i=i: self._step(i, p, want_out), warm)
                    graph.replay()
                    eng.launches += stats[0]
                    eng.model_calls += stats[1]
                    if callback is not None:
                        callback(i, self.denoised_buffer(i, want_out), self.x, n_steps)
            elif mode == "eager":
                rel = self._relative_plan()
                if not self.external_init:
                    self._init_state()
                for i in range(n_steps):
                    self._step(i, rel, want_out)
                    if callback is not None:
                        callback(i, self.denoised_buffer(i, want_out), self.x, n_steps)
                    if i == 0:   # the first outer step also pays the process's first launches (CUDA's lazy loading)
                        self.first_step_end = torch.cuda.Event(enable_timing=True)
                        self.first_step_end.record()
            else:
                raise ValueError(f"unknown mode {mode!r}")
            if self.timing:
                self.last_events[1].record()
            plan.consume(self.draws)
            plan.finish()
            eng.substeps_done += self.substeps
            self.launches, self.model_calls = eng.launches - before[0], eng.model_calls - before[1]
            if x_out is not None:
                x_out.copy_(self.x, non_blocking=True)
                return x_out
            return self.x.clone()


class SamplerGraphJob:
    """ANY deterministic k-diffusion sampler around the per-sigma wrapper as ONE CUDA graph per job.

    `runner.GraphedJob` owns the sampler loop, so it only serves the samplers it restates (euler, euler_ancestral,
    dpmpp_2m, dpm_2, heun, deis, res_multistep, gradient_estimation).  For the other samplers (heunpp2, ..., and heun
    unless the node's option "fused_heun" routes it to the fused loop) the loop is
    third-party Python that calls the wrapper with sigma values only it knows.  But for a fixed schedule that sequence is deterministic: the node layer records it during the first,
    eager job of a configuration (`KSamplerX0Inpaint.trace`), this class turns every recorded call into device
    constants (`engine.plan_item`) and then runs the sampler function ITSELF under stream capture -- its Python runs
    once, at capture -- with the wrapper serving the planned calls (`engine.run_planned`: no read-back, no copies).
    The sampler gets the schedule as a CPU tensor so that its own scalar tests (`sigmas[i + 1] == 0`) stay on the host.
    Falls back (exception -> the node layer uses the per-sigma graphs) when the sampler syncs, allocates host
    memory in a way capture forbids, draws its own noise, or calls the model a different number of times.

    Callbacks: the sampler's per-step callback runs at capture time only, so it is recorded there (step index,
    denoised tensor, x tensor -- graph-owned buffers that stay valid) and delivered in order after every replay, the
    same deferred form GraphedJob uses for short jobs."""

    def __init__(self, engine, sampler_function, extra_options, sigmas_cpu: torch.Tensor, trace, shape, device):
        from .engine import _DrawPlan
        self.engine, self.fn, self.extra_options = engine, sampler_function, dict(extra_options or {})
        self.sigmas = sigmas_cpu.detach().to("cpu", torch.float32)
        self.trace = list(trace)            # [(sigma_host [B] CPU tensor, times tuple, n_eff)]
        self.device, self.shape = torch.device(device), tuple(shape)
        mk = lambda: torch.empty(self.shape, dtype=torch.float32, device=self.device)
        self.x0, self.y, self.noise, self.c = mk(), mk(), mk(), mk()
        self.mask = None
        self.rng_state = torch.zeros(2, dtype=torch.int64, device=self.device)
        self.items = None
        self.graph = None
        self.result = None
        self.recorded = []                  # callbacks seen at capture: (i, denoised, x)
        self.draws = 0
        self.launches = self.model_calls = self.substeps = 0
        self.captures = 0
        self._plan_cls = _DrawPlan
        self.timing, self.last_events = False, None

    def _load(self, latent_image, noise, pm, x_init):
        import numpy as np
        from .engine import PackedMask, pack_known
        self.y.copy_(latent_image, non_blocking=True)
        self.noise.copy_(noise, non_blocking=True)
        self.x0.copy_(x_init, non_blocking=True)
        if self.mask is None or self.mask.data.shape != pm.data.shape or (
                self.mask.row_stride, self.mask.channel_stride) != (pm.row_stride, pm.channel_stride):
            self.mask = PackedMask(torch.empty_like(pm.data), pm.row_stride, pm.channel_stride)
            self.graph = None
        self.mask.data.copy_(pm.data, non_blocking=True)
        B = self.shape[0]
        self.dims = _native.Dims(B, self.x0.numel() // B, int(np.prod(self.shape[2:])), self.mask.row_stride,
                                 self.mask.channel_stride)
        self.mask.known = pack_known(self.mask, self.dims, self.y, self.noise, out=self.mask.known)

    def _capture(self, model_k, extra_args, want_callbacks):
        from .engine import heads_discardable
        eng = self.engine
        B = self.shape[0]
        self.items = []
        for sigma_host, times, n_eff in self.trace:
            item = eng.plan_item(B, sigma_host, times, n_eff, self.device)
            if item is None:
                raise RuntimeError("noise_scaling is not a linear form")
            self.items.append(item)
        plan = self._plan_cls(eng.rng, self.x0, 1).relative()   # before capture: reads the generator once
        counts = (eng.launches, eng.model_calls, eng.substeps_done)
        state = {"pos": 0}
        job = self

        def planned(x, model_options, seed):
            if state["pos"] >= len(job.items):
                raise RuntimeError("the sampler called the model more often than in its recorded job")
            item = job.items[state["pos"]]
            state["pos"] += 1
            return eng.run_planned(x, item, job.y, job.noise, job.mask, job.dims, job.c, plan, job.rng_state.data_ptr(),
                                   model_options, seed, discard_heads=heads_discardable(model_options))
        model_k.planned_call = planned
        self.recorded = []
        k_callback = None
        if want_callbacks:
            k_callback = lambda d: job.recorded.append((d["i"], d["denoised"], d["x"]))  # noqa: E731
        graph = torch.cuda.CUDAGraph()
        cap_stream = torch.cuda.Stream(device=self.device)
        cap_stream.wait_stream(torch.cuda.current_stream(self.device))
        try:
            with torch.cuda.graph(graph, stream=cap_stream):
                self.result = self.fn(model_k, self.x0, self.sigmas, extra_args=extra_args, callback=k_callback,
                                      disable=True, **self.extra_options)
        finally:
            model_k.planned_call = None
        if state["pos"] != len(self.items):
            raise RuntimeError("the sampler called the model less often than in its recorded job")
        self.graph, self.draws = graph, plan.used
        self.launches, self.model_calls = eng.launches - counts[0], eng.model_calls - counts[1]
        self.substeps = eng.substeps_done - counts[2]
        eng.launches, eng.model_calls, eng.substeps_done = counts
        self.captures += 1

    def run(self, model_k, extra_args, latent_image, noise, pm, x_init, callback=None):
        """callback(i, denoised, x, total_steps): ComfyUI's; delivered after the replay, in the sampler's order."""
        import numpy as np
        eng = self.engine
        with torch.cuda.device(self.device):
            self._load(latent_image, noise, pm, x_init)
            if self.graph is None:
                self._capture(model_k, extra_args, callback is not None)
            plan = self._plan_cls(eng.rng, self.x0, 1)
            self.rng_state.copy_(torch.from_numpy(plan.state_words().view(np.int64)))
            if self.timing:
                self.last_events = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
                self.last_events[0].record()
            self.graph.replay()
            if self.timing:
                self.last_events[1].record()
            plan.consume(self.draws)
            plan.finish()
            eng.launches += self.launches
            eng.model_calls += self.model_calls
            eng.substeps_done += self.substeps
            if callback is not None:
                total = len(self.sigmas) - 1
                for i, den, xx in self.recorded:
                    callback(i, den, xx, total)
            return self.result.clone()
