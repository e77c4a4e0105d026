"""CPU: why the whole-job tests run a network that couples positions, and the job restatement they compare with.

With the pointwise test network (`_node_cases.denoiser`) a free element's trajectory never reads a known element, so
the known region reaches the final latent only through the paste `out = y`: changing cfg_BIG (the prompt mode),
lambda or the noise image at known positions leaves the job's result bit for bit unchanged, and a job-level test
cannot see what a kernel does there.  With `_node_cases.mixing_denoiser` each of them moves the result well above
round-off.  Both facts are asserted on the fp32 oracle job (`O.euler_inpaint`), which the node goldens pin to the
reference.  Then `_job_ref.job`, the loop tests/test_gpu_job_ref.py runs in fp64, is checked against
`O.euler_inpaint` in fp32 on the same draws."""
import pytest
import torch

import _job_ref as J
from _node_cases import denoiser, mixing_denoiser
from oracle import langevin_oracle as O

SHAPE = (2, 4, 32, 32)
NETS = {"pointwise": denoiser, "mixing": mixing_denoiser}


def _inputs(seed=0):
    g = torch.Generator().manual_seed(seed)
    y = torch.randn(SHAPE, generator=g)
    noise = torch.randn(SHAPE, generator=g)
    dm = (torch.rand((SHAPE[0], 1) + SHAPE[2:], generator=g) < 0.5).float().expand(SHAPE)   # 1 = regenerate
    other = torch.randn(SHAPE, generator=g)
    return y, noise, dm, other


def _oracle_job(net, y, noise, dm, cfg_big=5.0, lam=5.0, draw_seed=7):
    model = J.Guider(net, O.VESampling(), 5.0, cfg_big)
    draw = O.NoiseTape(generator=torch.Generator().manual_seed(draw_seed))
    with torch.no_grad():
        return O.euler_inpaint(model, y, noise, dm, O.karras_sigmas(20), O.Hyper(n_steps=5, lam=lam, min_step_frac=1.0),
                               draw=draw, max_denoise=True)


@pytest.mark.parametrize("change", ["cfg_big", "lambda", "known_noise"])
def test_known_region_settings_reach_the_latent_only_through_a_mixing_network(change):
    """With the pointwise network the free positions of the result are bit for bit unchanged.  So is the whole
    latent for cfg_BIG and lambda; the noise image still reaches the known positions through one rounding: the last
    outer step runs no sub-step, so x there is its replace-step value s*noise + (1-s)*y, and the final Euler step
    x + (x - y)/s * (0 - s) returns y only up to round-off."""
    y, noise, dm, other = _inputs()
    known = dm < 0.5
    moved = {}
    for name, net in NETS.items():
        base = _oracle_job(net, y, noise, dm)
        if change == "cfg_big":                 # "Image First" (cfg_BIG = cfg) vs "Prompt First" (cfg_BIG = -0.5)
            alt = _oracle_job(net, y, noise, dm, cfg_big=-0.5)
        elif change == "lambda":
            alt = _oracle_job(net, y, noise, dm, lam=0.5)
        else:                                   # the noise image changed where the mask keeps the latent only
            alt = _oracle_job(net, y, torch.where(known, other, noise), dm)
        moved[name] = float((alt - base).abs().max() / base.abs().max())
        if name == "pointwise":
            assert torch.equal(alt[~known], base[~known]), (change, moved)
            if change == "known_noise":
                assert moved[name] <= 1e-6, (change, moved)
            else:
                assert torch.equal(alt, base), (change, moved)
    assert moved["mixing"] > 1e-2, (change, moved)


@pytest.mark.parametrize("flow", [False, True])
def test_job_loop_in_fp32_equals_the_oracle_euler_run(flow):
    y, noise, dm, _ = _inputs(1)
    sampling = O.FlowSampling() if flow else O.VESampling()
    sig = O.flow_simple_sigmas(12, 3.0) if flow else O.karras_sigmas(20)
    hp = O.Hyper(n_steps=5, min_step_frac=1.0, flow=flow)
    cfg, cfg_big = (3.5, 1.0) if flow else (5.0, -0.5)
    m_want, m_got = J.Guider(mixing_denoiser, sampling, cfg, cfg_big), J.Guider(mixing_denoiser, sampling, cfg, cfg_big)
    t_want = O.NoiseTape(generator=torch.Generator().manual_seed(3))
    t_got = O.NoiseTape(generator=torch.Generator().manual_seed(3))
    steps = []
    with torch.no_grad():
        want = O.euler_inpaint(m_want, y, noise, dm, sig, hp, draw=t_want, max_denoise=not flow)
    want = sampling.inverse_noise_scaling(sig[-1], want)
    got = J.job(J.SAMPLERS["euler"], m_got, y, noise, dm, sig, hp, draw=t_got, max_denoise=not flow,
                callback=lambda i, d: steps.append(i))
    assert t_got.pos == t_want.pos and m_got.calls == m_want.calls
    assert steps == list(range(len(sig) - 1))
    err = float((got - want).abs().max() / want.abs().max())
    assert err <= 1e-6, err


def test_fp64_job_is_within_fp32_round_off_of_the_fp32_job():
    """The fp64 loop on the fp32 oracle's draws: how far fp32 arithmetic lands from it on the CPU (the scale the
    GPU tolerance is set against)."""
    y, noise, dm, _ = _inputs(2)
    hp = O.Hyper(n_steps=5, min_step_frac=1.0)
    runs = {}
    for dt in (torch.float32, torch.float64):
        tape = O.NoiseTape(generator=torch.Generator().manual_seed(5))
        model = J.Guider(mixing_denoiser, O.VESampling(), 5.0, -0.5)
        runs[dt] = J.job(J.SAMPLERS["euler"], model, y.to(dt), noise.to(dt), dm.to(dt), O.karras_sigmas(20), hp,
                         draw=tape, max_denoise=True)
    err = float((runs[torch.float32].double() - runs[torch.float64]).abs().max() / runs[torch.float64].abs().max())
    print(f"fp32 job vs fp64 job, max|d| / max|x|: {err:.3g}")
    assert 0.0 < err <= 5e-6, err
