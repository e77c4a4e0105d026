"""The coefficients of DEIS (Zhang & Chen, "Fast Sampling of Diffusion Models with Exponential Integrator"), 'tab'
mode: the stand-in for ComfyUI's `comfy/k_diffusion/deis.py`, which `sample_deis` reads through the `deis` attribute
of its own module.

Written from ComfyUI's source as its author knows it, and not compared with ComfyUI itself, which is not a dependency
of this project.  The EDM sigmas are mapped to the time t of a VP SDE (`edm2t`); for each step of order k the coefficient of
the j-th latest derivative is the integral over [t_cur, t_next] of d sigma / d t times the j-th Lagrange basis
polynomial through the last k times, by an N-point Riemann sum on a uniform grid.
"""
from __future__ import annotations

import torch


def edm2t(edm_steps, epsilon_s=1e-3, sigma_min=0.002, sigma_max=80):
    """EDM sigmas -> the VP time t with sigma(t) = sqrt(exp(beta_d t^2 / 2 + beta_min t) - 1); also beta_min and
    beta_min + beta_d (fp32 CPU tensors)."""
    vp_sigma_inv = lambda beta_d, beta_min: lambda sigma: (   # noqa: E731
        ((beta_min ** 2 + 2 * beta_d * (sigma ** 2 + 1).log()).sqrt() - beta_min) / beta_d)
    smin2 = torch.log(torch.tensor(sigma_min) ** 2 + 1)
    smax2 = torch.log(torch.tensor(sigma_max) ** 2 + 1)
    vp_beta_d = 2 * (smin2 / epsilon_s - smax2) / (epsilon_s - 1)
    vp_beta_min = smax2 - 0.5 * vp_beta_d
    t_steps = vp_sigma_inv(vp_beta_d, vp_beta_min)(edm_steps.clone().detach().cpu())
    return t_steps, vp_beta_min, vp_beta_d + vp_beta_min


def cal_poly(prev_t, j, taus):
    """The j-th Lagrange basis polynomial through the times prev_t, at taus."""
    poly = 1
    for k in range(prev_t.shape[0]):
        if k == j:
            continue
        poly *= (taus - prev_t[k]) / (prev_t[j] - prev_t[k])
    return poly


def t2alpha_fn(beta_0, beta_1, t):
    """alpha_t of the VP SDE with a linear beta schedule from beta_0 to beta_1."""
    return torch.exp(-0.5 * t ** 2 * (beta_1 - beta_0) - t * beta_0)


def cal_intergrand(beta_0, beta_1, taus):
    """-1/2 d log(alpha)/d tau / sqrt(alpha (1 - alpha)), i.e. d sigma / d tau, the derivative by autograd (so the
    caller may hold inference mode or no_grad)."""
    with torch.inference_mode(mode=False):
        taus = taus.clone()
        beta_0 = beta_0.clone()
        beta_1 = beta_1.clone()
        with torch.enable_grad():
            taus.requires_grad_(True)
            alpha = t2alpha_fn(beta_0, beta_1, taus)
            log_alpha = alpha.log()
            log_alpha.sum().backward()
            d_log_alpha_dtau = taus.grad
    integrand = -0.5 * d_log_alpha_dtau / torch.sqrt(alpha * (1 - alpha))
    return integrand


def get_deis_coeff_list(t_steps, max_order, N=10000, deis_mode="tab"):
    """Per step i: [] for a first-order step, else the order coefficients [c_cur, c_prev1, ...] (0-d fp32 CPU
    tensors) of x_next = x + c_cur d_i + c_prev1 d_{i-1} + ...; order = min(i + 1, max_order)."""
    if deis_mode != "tab":
        raise NotImplementedError("minicomfy's DEIS has the 'tab' mode only")
    t_steps, beta_0, beta_1 = edm2t(t_steps)
    C = []
    for i, (t_cur, t_next) in enumerate(zip(t_steps[:-1], t_steps[1:])):
        order = min(i + 1, max_order)
        if order == 1:
            C.append([])
        else:
            taus = torch.linspace(t_cur, t_next, N)   # the interval, split for the Riemann sum
            dtau = (t_next - t_cur) / N
            prev_t = t_steps[[i - k for k in range(order)]]
            coeff_temp = []
            integrand = cal_intergrand(beta_0, beta_1, taus)
            for j in range(order):
                poly = cal_poly(prev_t, j, taus)
                coeff_temp.append(torch.sum(integrand * poly) * dtau)
            C.append(coeff_temp)
    return C
