"""Host-side schedule logic of the Langevin hot path.

Everything the reference computes per outer step as device scalars-with-syncs
(src/LanPaint/nodes.py:242-252,286-299; src/LanPaint/lanpaint.py:81,205,
295-328) happens here once, on the host, from the per-sample sigma values:
the (VE sigma, alpha-bar, flow t) triple, the effective inner-step count and
the coefficient table the kernels read.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Optional, Sequence

import numpy as np
import torch

from . import _native

TABLE_STRIDE = _native.TABLE_STRIDE


def times_from_sigma(sigma: torch.Tensor, flow: bool):
    """sigma -> (VE_Sigma, abt, Flow_t) with the reference's own fp32 op order
    (nodes.py:242-252), so the alpha-bar the table is built from is bit-identical."""
    if flow:
        flow_t = sigma
        abt = (1 - flow_t) ** 2 / ((1 - flow_t) ** 2 + flow_t ** 2)
        ve = flow_t / (1 - flow_t)
    else:
        ve = sigma
        abt = 1 / (1 + ve ** 2)
        flow_t = (1 - abt) ** 0.5 / ((1 - abt) ** 0.5 + abt ** 0.5)
    return ve, abt, flow_t


def min_step_frac_effective_steps(n_steps, frac, min_frac):
    """Inner-step count under the MinStepFrac tail ramp (nodes.py:134-144).

    Above the fraction (or with the feature off) the count is unchanged; below
    it the count ramps down as round(n * frac / min_frac) with Python's
    half-to-even rounding, never below zero."""
    if min_frac <= 0 or frac >= min_frac or n_steps <= 0:
        return n_steps
    return max(0, round(n_steps * frac / min_frac))


def effective_inner_steps(n_steps: int, sigmas_host: Sequence[float], sigma_mean: float, abt_frac: float,
                          early_stop: int = 1, min_frac: float = 1.0) -> int:
    """n_eff of nodes.py:286-299 from host values.

    `abt_frac` must be float(float32 mean(1 - abt)) so the banker's rounding sees
    the same number the reference does."""
    diffs = [abs(s - sigma_mean) for s in sigmas_host]
    current = diffs.index(min(diffs))  # torch.argmin returns the first minimum, so does index()
    total = len(sigmas_host) - 1
    if total - current <= early_stop:
        return 0
    return min_step_frac_effective_steps(n_steps, abt_frac, min_frac)


def ancestral_step(sigma_from: float, sigma_to: float, eta: float = 1.0):
    """(sigma_down, sigma_up) of one step of k-diffusion's sample_euler_ancestral (get_ancestral_step), in Python
    doubles with the sampler's own expression, operation for operation: the fused loop rounds what the sampler
    rounds."""
    s_from, s_to = float(sigma_from), float(sigma_to)
    s_up = min(s_to, eta * (s_to ** 2 * (s_from ** 2 - s_to ** 2) / s_from ** 2) ** 0.5) if s_to > 0 else 0.0
    s_down = (s_to ** 2 - s_up ** 2) ** 0.5
    return s_down, s_up


def dpmpp_2m_step(sigmas: torch.Tensor):
    """[(ratio, em1, c_cur, c_old, second_order)] for every outer step of k-diffusion's sample_dpmpp_2m on `sigmas`.

    The sampler's own torch expressions on its own 0-d fp32 tensors, evaluated where `sigmas` lives (the node hands
    the sampler a device schedule, so its scalars come from the device's logf / expf / expm1f), then read back once:
    ratio = sigma_fn(t_next) / sigma_fn(t), em1 = expm1(-h), c_cur = 1 + 1/(2r), c_old = 1/(2r), with t = -log(sigma),
    h = t_next - t, r = h_last / h.  A step is second order when the sampler has a previous denoised latent and
    sigma_next != 0; a first-order step has c_cur = c_old = 0 (unused).  The step to sigma = 0 comes out as the sampler
    computes it: t_next = inf, ratio = 0, em1 = -1."""
    sigma_fn = lambda t: t.neg().exp()     # noqa: E731
    t_fn = lambda sigma: sigma.log().neg()  # noqa: E731
    host = [float(v) for v in sigmas.detach().cpu()]
    rows = []
    for i in range(len(host) - 1):
        t, t_next = t_fn(sigmas[i]), t_fn(sigmas[i + 1])
        h = t_next - t
        ratio, em1 = sigma_fn(t_next) / sigma_fn(t), (-h).expm1()
        second = i > 0 and host[i + 1] != 0.0
        if second:
            h_last = t - t_fn(sigmas[i - 1])
            r = h_last / h
            c_cur, c_old = 1 + 1 / (2 * r), 1 / (2 * r)
        else:
            c_cur = c_old = torch.zeros_like(ratio)
        rows.append(torch.stack([ratio, em1, c_cur, c_old]))
    vals = torch.stack(rows).cpu().tolist() if rows else []
    return [(v[0], v[1], v[2], v[3], i > 0 and host[i + 1] != 0.0) for i, v in enumerate(vals)]


def dpm_2_step(sigmas: torch.Tensor):
    """[(sigma_mid, dt_1, dt_2, midpoint)] for every outer step of k-diffusion's sample_dpm_2 (no churn) on `sigmas`.

    As `dpmpp_2m_step`: the sampler's own torch expressions on its own 0-d fp32 tensors where `sigmas` lives, read back
    once.  With sigma_hat = sigma_i: sigma_mid = exp(lerp(log sigma_hat, log sigma_next, 1/2)), dt_1 = sigma_mid -
    sigma_hat, dt_2 = sigma_next - sigma_hat.  A step makes its midpoint call when sigma_next != 0; the step to
    sigma = 0 is one Euler update with dt_2 = sigma_next - sigma_hat, and sigma_mid = dt_1 = 0 (unused)."""
    host = [float(v) for v in sigmas.detach().cpu()]
    rows = []
    for i in range(len(host) - 1):
        sigma_hat = sigmas[i] * (0.0 + 1)
        dt_2 = sigmas[i + 1] - sigma_hat
        if host[i + 1] != 0.0:
            sigma_mid = sigma_hat.log().lerp(sigmas[i + 1].log(), 0.5).exp()
            rows.append(torch.stack([sigma_mid, sigma_mid - sigma_hat, dt_2]))
        else:
            rows.append(torch.stack([torch.zeros_like(dt_2), torch.zeros_like(dt_2), dt_2]))
    vals = torch.stack(rows).cpu().tolist() if rows else []
    return [(v[0], v[1], v[2], host[i + 1] != 0.0) for i, v in enumerate(vals)]


def heun_step(sigmas: torch.Tensor):
    """[(sigma_hat, dt, sigma_next, corrector)] for every outer step of k-diffusion's sample_heun (no churn) on `sigmas`.

    As `dpm_2_step`: the sampler's own torch expressions on its own 0-d fp32 tensors where `sigmas` lives, read back
    once.  sigma_hat = sigma_i * (0 + 1) (= sigma_i), dt = sigma_next - sigma_hat.  A step makes its corrector call at
    sigma_next when sigma_next != 0; the step to sigma = 0 is one Euler update with the same dt."""
    host = [float(v) for v in sigmas.detach().cpu()]
    rows = []
    for i in range(len(host) - 1):
        sigma_hat = sigmas[i] * (0.0 + 1)
        rows.append(torch.stack([sigma_hat, sigmas[i + 1] - sigma_hat, sigmas[i + 1]]))
    vals = torch.stack(rows).to(torch.float32).cpu().tolist() if rows else []
    return [(v[0], v[1], v[2], host[i + 1] != 0.0) for i, v in enumerate(vals)]


def deis_step(sampler_fn, sigmas: torch.Tensor):
    """[(sigma, c_cur, c_prev1, c_prev2, order)] for every outer step of ComfyUI's sample_deis (max_order = 3,
    deis_mode = 'tab') on `sigmas`: x = x + c_cur d [+ c_prev1 d_{i-1} [+ c_prev2 d_{i-2}]], d = (x - denoised) / sigma.

    The coefficients are the sampler's own: `get_deis_coeff_list` of the `deis` module next to `sampler_fn` (ComfyUI's
    k_diffusion.sampling, or the stand-in), 0-d fp32 CPU tensors, called once here (it runs autograd on the CPU).
    order = min(3, i + 1), and 1 on the step to sigma <= 0; a first-order step's c_cur is the sampler's fp32
    difference sigma_next - sigma of schedule entries, evaluated where `sigmas` lives.  Unused coefficients are 0."""
    import sys
    deis = sys.modules[sampler_fn.__module__].deis
    with torch.no_grad():
        coeff = deis.get_deis_coeff_list(sigmas, 3, deis_mode="tab")
        host = [float(v) for v in sigmas.detach().cpu()]
        first = (sigmas[1:] - sigmas[:-1]).to(torch.float32).cpu().tolist()
    rows = []
    for i in range(len(host) - 1):
        order = 1 if host[i + 1] <= 0 else min(3, i + 1)
        c = [first[i]] if order == 1 else [float(v.to(torch.float32)) for v in coeff[i][:order]]
        c += [0.0] * (3 - len(c))
        rows.append((host[i], c[0], c[1], c[2], order))
    return rows


def res_multistep_step(sigmas: torch.Tensor):
    """[(second, a, b, c, d)] for every outer step of ComfyUI's sample_res_multistep (res_multistep, eta = 0) on
    `sigmas`: an Euler step (False, sigma_i, dt, 0, 0), x = x + ((x - denoised) / sigma_i) * dt with dt = sigma_next -
    sigma_i, or a second-order step (True, ratio, em1, c_cur, c_old) in lp_multistep's form, x = ratio*x -
    em1*(c_cur*denoised - c_old*old_denoised), with ratio = sigma_fn(h), em1 = -h, c_cur = b1 and c_old = -b2.

    As `dpmpp_2m_step`: the sampler's own torch expressions (get_ancestral_step with eta = 0, the phi functions,
    nan_to_num) on its own 0-d fp32 tensors where `sigmas` lives, read back once.  The sampler takes the Euler step on
    its first step and where sigma_down = sigma_next is 0."""
    sigma_fn = lambda t: t.neg().exp()              # noqa: E731
    t_fn = lambda sigma: sigma.log().neg()          # noqa: E731
    phi1_fn = lambda t: torch.expm1(t) / t          # noqa: E731
    phi2_fn = lambda t: (phi1_fn(t) - 1.0) / t      # noqa: E731
    host = [float(v) for v in sigmas.detach().cpu()]
    rows = []
    for i in range(len(host) - 1):
        sigma_down = sigmas[i + 1]              # get_ancestral_step(sigma_i, sigma_next, eta=0)
        if i == 0 or host[i + 1] == 0.0:
            z = torch.zeros_like(sigma_down)
            rows.append(torch.stack([sigmas[i], sigma_down - sigmas[i], z, z]))
            continue
        t, t_old, t_next, t_prev = t_fn(sigmas[i]), t_fn(sigmas[i]), t_fn(sigma_down), t_fn(sigmas[i - 1])
        h = t_next - t
        c2 = (t_prev - t_old) / h
        phi1_val, phi2_val = phi1_fn(-h), phi2_fn(-h)
        b1 = torch.nan_to_num(phi1_val - phi2_val / c2, nan=0.0)
        b2 = torch.nan_to_num(phi2_val / c2, nan=0.0)
        rows.append(torch.stack([sigma_fn(h), -h, b1, -b2]))
    vals = torch.stack(rows).cpu().tolist() if rows else []
    return [(i > 0 and host[i + 1] != 0.0, *v) for i, v in enumerate(vals)]


def gradient_estimation_step(sigmas: torch.Tensor, ge_gamma: float = 2.0):
    """[(sigma, dt, gm1, reads_old, final, keep)] for every outer step of ComfyUI's sample_gradient_estimation on
    `sigmas`: d = (x - denoised) / sigma; x = denoised on the step to sigma = 0 (final), else x = x + d*dt and, when the
    step reads the previous step's d (i >= 1), x = x + (gm1*(d - old_d))*dt.  keep: a later step reads this step's d.

    sigma and dt = sigma_next - sigma are the sampler's 0-d fp32 tensors where `sigmas` lives, read back once; gm1 is
    the fp32 value of the Python float ge_gamma - 1, which torch rounds to the tensor's type before it multiplies."""
    host = [float(v) for v in sigmas.detach().cpu()]
    n = len(host) - 1
    vals = torch.stack([sigmas[:-1], sigmas[1:] - sigmas[:-1]], 1).cpu().tolist() if n > 0 else []
    gm1 = float(torch.tensor(ge_gamma - 1, dtype=torch.float32))
    final = [host[i + 1] == 0.0 for i in range(n)]
    reads = [i >= 1 and not final[i] for i in range(n)]
    return [(v[0], v[1], gm1, reads[i], final[i], i + 1 < n and reads[i + 1]) for i, v in enumerate(vals)]


@dataclass
class Hyper:
    step_size: float
    lam: float
    beta: float
    min_step_frac: float
    flow: bool

    def to_c(self) -> _native.Hyper:
        return _native.Hyper(float(self.step_size), float(self.lam), float(self.beta),
                             float(self.min_step_frac), 1 if self.flow else 0, 0)


def build_table(abt: Sequence[float], ve_sigma: Sequence[float], hyper: Hyper,
                rep_noise: Optional[Sequence[float]] = None, rep_y: Optional[Sequence[float]] = None,
                corr: Optional[Sequence[float]] = None, out: Optional[np.ndarray] = None) -> np.ndarray:
    """Coefficient table [rows, 24] fp32 (host) via the library's lp_build_coef_table."""
    lib = _native.load()
    a = np.ascontiguousarray(abt, dtype=np.float64)
    v = np.ascontiguousarray(ve_sigma, dtype=np.float64)
    n = a.shape[0]
    assert v.shape[0] == n
    if out is None:
        out = np.empty((n, TABLE_STRIDE), dtype=np.float32)
    assert out.dtype == np.float32 and out.size >= n * TABLE_STRIDE and out.flags["C_CONTIGUOUS"]

    def opt(x):
        if x is None:
            return None, None
        arr = np.ascontiguousarray(x, dtype=np.float64)
        assert arr.shape[0] == n
        return arr, arr.ctypes.data_as(C.c_void_p)

    rn, rn_p = opt(rep_noise)
    ry, ry_p = opt(rep_y)
    cc, cc_p = opt(corr)
    hc = hyper.to_c()
    rc = lib.lp_build_coef_table(a.ctypes.data_as(C.c_void_p), v.ctypes.data_as(C.c_void_p), rn_p, ry_p, cc_p,
                                 n, C.byref(hc), out.ctypes.data_as(C.c_void_p))
    _native.check(rc, "lp_build_coef_table")
    return out


def mean_half_dt(abt: Sequence[float], hyper: Hyper) -> float:
    """mean over the batch of dtx/2 = StepSize*clamp(1-abt, MinStepFrac); the reference
    skips the whole sub-step when it is <= 0 (lanpaint.py:205)."""
    vals = [hyper.step_size * max(1.0 - float(a), hyper.min_step_frac) for a in abt]
    return sum(vals) / max(1, len(vals))
