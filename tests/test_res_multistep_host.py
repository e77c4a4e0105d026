"""Host side of the fused res_multistep loop: minicomfy's sample_res_multistep, the per-step scalars
`schedule.res_multistep_step` reads back, the identity that lets lp_boundary_multistep compute the RES step bit for bit,
the buffers and draw accounting of `runner.GraphedJob(sampler="res_multistep")`, the node gate and its form check, and
minicomfy's sampler inside the fp32 job against fp64 and the reference node layer's fixtures."""
import functools
import json
import os

import numpy as np
import pytest
import torch

import _job_ref as J
import minicomfy
import test_oracle_node_golden as NG
from _node_cases import NEG, POS
from conftest import GOLDEN_DIR
from lanpaint_b200.schedule import res_multistep_step
from oracle import langevin_oracle as O

SEEDED = J._plain(functools.partial(minicomfy.sample_res_multistep, extra_args={"seed": 0}))


def _schedules():
    eps = minicomfy.ModelPatcher(minicomfy.BaseModel(None), "cpu")
    flow = minicomfy.ModelPatcher(minicomfy.BaseModel(None, model_type=minicomfy.ModelType.FLOW, shift=3.0), "cpu")
    return {"karras-20": J.ksampler_sigmas(eps, 20, "res_multistep", "karras"),
            "flow-simple-10": J.ksampler_sigmas(flow, 10, "res_multistep", "simple"),
            "window-leftover": J.ksampler_sigmas(eps, 20, "res_multistep", "karras", start_step=3, last_step=15),
            "one-step": J.ksampler_sigmas(eps, 1, "res_multistep", "karras"),
            "repeated": torch.tensor([6.0, 3.0, 3.0, 1.5, 0.5, 0.0])}


def _sampler_scalars(sig):
    """The sampler's own expressions, per step (second, the four scalars), as sample_res_multistep evaluates them."""
    sigma_fn = lambda t: t.neg().exp()              # noqa: E731
    t_fn = lambda sigma: sigma.log().neg()          # noqa: E731
    phi1_fn = lambda t: torch.expm1(t) / t          # noqa: E731
    phi2_fn = lambda t: (phi1_fn(t) - 1.0) / t      # noqa: E731
    rows, old_sigma_down = [], None
    for i in range(len(sig) - 1):
        sigma_down, sigma_up = minicomfy.get_ancestral_step(sig[i], sig[i + 1], eta=0.0)
        assert sigma_up == 0.0
        if sigma_down == 0 or i == 0:
            rows.append((False, float(sig[i]), float(sigma_down - sig[i])))
        else:
            t, t_old, t_next, t_prev = t_fn(sig[i]), t_fn(old_sigma_down), t_fn(sigma_down), t_fn(sig[i - 1])
            h = t_next - t
            c2 = (t_prev - t_old) / h
            b1 = torch.nan_to_num(phi1_fn(-h) - phi2_fn(-h) / c2, nan=0.0)
            b2 = torch.nan_to_num(phi2_fn(-h) / c2, nan=0.0)
            rows.append((True, float(sigma_fn(h)), float(h), float(b1), float(b2)))
        old_sigma_down = sigma_down
    return rows


def test_minicomfy_registers_res_multistep():
    assert minicomfy.ksampler("res_multistep").sampler_function is minicomfy.sample_res_multistep
    assert "res_multistep" in minicomfy.KSampler.SAMPLERS
    assert "res_multistep" not in minicomfy.DISCARD_PENULTIMATE_SIGMA_SAMPLERS
    patcher = minicomfy.ModelPatcher(minicomfy.BaseModel(None), "cpu")
    assert torch.equal(minicomfy.KSampler(patcher, 8, "cpu", "res_multistep", "karras").sigmas,
                       minicomfy.KSampler(patcher, 8, "cpu", "euler", "karras").sigmas)
    base = minicomfy.BaseModel(lambda x, sigma, c: 0.5 * x, model_type=minicomfy.ModelType.EPS, latent_channels=4,
                               shift=1.0)
    patcher = minicomfy.ModelPatcher(base, "cpu")
    g = torch.Generator().manual_seed(2)
    latent, noise = torch.randn(1, 4, 8, 8, generator=g), torch.randn(1, 4, 8, 8, generator=g)
    seen = []
    out = minicomfy.KSampler(patcher, 6, "cpu", "res_multistep", "karras").sample(
        noise, POS, NEG, 3.0, latent_image=latent, callback=lambda i, x0, x, total: seen.append(i), seed=1)
    assert out.shape == latent.shape and bool(torch.isfinite(out).all()) and seen == list(range(6))


def test_seeded_draw_leaves_the_global_generators_alone():
    """With a seed the sampler's draw (times sigma_up = 0) comes from a private generator: the global stream does not
    move, and the result is the draw-free loop's."""
    g = torch.Generator().manual_seed(4)
    x0 = torch.randn(2, 3, 5, generator=g)
    model = lambda x, s, **kw: torch.tanh(0.7 * x) + 0.1 * x     # noqa: E731
    sig = _schedules()["karras-20"]
    state = torch.get_rng_state()
    got = minicomfy.sample_res_multistep(model, x0.clone(), sig, extra_args={"seed": 3})
    assert torch.equal(torch.get_rng_state(), state)
    silent = minicomfy.res_multistep(model, x0.clone(), sig, extra_args={"seed": 3}, eta=0.0,
                                     noise_sampler=lambda s, t: torch.zeros_like(x0))
    assert torch.equal(got, silent)


@pytest.mark.parametrize("name", ["karras-20", "flow-simple-10", "window-leftover", "one-step", "repeated"])
def test_step_scalars_are_the_samplers(name):
    """res_multistep_step's rows are the sampler's own scalars (Euler: sigma, sigma_next - sigma; second order:
    sigma_fn(h), -h, b1, -b2), Euler exactly on the first step and on the step to sigma = 0; on the repeated sigma
    nan_to_num fires.  The sampler's loop equals the loop on these scalars in the fused launches' operation order."""
    sig = _schedules()[name]
    rows = res_multistep_step(sig)
    want = _sampler_scalars(sig)
    assert len(rows) == len(sig) - 1
    for i, (r, w) in enumerate(zip(rows, want)):
        assert r[0] == w[0] == (i > 0 and float(sig[i + 1]) != 0.0), (name, i)
        if r[0]:
            assert r[1:] == (w[1], -w[2], w[3], -w[4]), (name, i)
        else:
            assert r[1:] == (w[1], w[2], 0.0, 0.0), (name, i)
    if name == "window-leftover":
        assert float(sig[-1]) > 0 and rows[-1][0]
    if name == "one-step":
        assert [r[0] for r in rows] == [False]
    if name == "repeated":       # h = 0: phi1, phi2 are 0/0 and nan_to_num makes b1 = b2 = 0; then c2 = 0: b2 = inf
        assert rows[1][3] == 0.0 and rows[1][4] == 0.0 and rows[1][2] == 0.0
        assert abs(rows[2][4]) == np.finfo(np.float32).max
        return      # the step after it overflows, as the sampler's does

    g = torch.Generator().manual_seed(5)
    x0 = torch.randn(2, 3, 5, generator=g)
    model = lambda x, s, **kw: torch.tanh(0.7 * x) + 0.1 * x + 0.05   # noqa: E731
    want_x = minicomfy.sample_res_multistep(model, x0.clone(), sig, extra_args={"seed": 1})
    t = lambda v: torch.tensor(v, dtype=torch.float32)   # noqa: E731
    x, old = x0.clone(), None
    for second, a, b, c, e in rows:
        den = model(x, None)
        if second:   # lp_boundary_multistep: ratio*x - em1*(c_cur*out - c_old*old)
            x = t(a) * x - t(b) * (t(c) * den - t(e) * old)
        else:        # lp_boundary_midpoint on x alone: x + ((x - out) / sigma) * dt
            x = x + ((x - den) / t(a)) * t(b)
        old = den
    assert torch.equal(x, want_x), name


@pytest.mark.parametrize("name", ["karras-20", "flow-simple-10", "window-leftover"])
def test_multistep_form_is_the_res_step_bit_for_bit(name):
    """ratio*x - em1*(c_cur*out - c_old*old) with em1 = -h and c_old = -b2 equals sigma_fn(h)*x + h*(b1*out +
    b2*old) in fp32: negation is exact and a - b is a + (-b), so every product and sum is the same correctly rounded
    operation.  Random operands, signed zeros and large magnitudes included."""
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    n = 1 << 16
    ops = [torch.randn(n, generator=g) * torch.exp(4 * torch.randn(n, generator=g)) for _ in range(3)]
    for o in ops:
        o[:64] = 0.0
        o[64:128] = -0.0
    x, out, old = ops
    t = lambda v: torch.tensor(v, dtype=torch.float32)   # noqa: E731
    steps = [r for r in res_multistep_step(_schedules()[name]) if r[0]]
    assert steps
    for _, ratio, em1, c_cur, c_old in steps:
        h, b1, b2 = t(-em1), t(c_cur), t(-c_old)
        sampler = t(ratio) * x + h * (b1 * out + b2 * old)
        fused = t(ratio) * x - t(em1) * (t(c_cur) * out - t(c_old) * old)
        assert torch.equal(fused, sampler)
        assert torch.equal(torch.signbit(fused), torch.signbit(sampler))


def _job(sigmas, n_inner, sampler, rng="torch", early_stop=1, **kw):
    from lanpaint_b200.engine import LanPaint
    from lanpaint_b200.runner import GraphedJob, HostSchedule, VESampling
    eng = LanPaint(O.PointwiseDenoiser(VESampling()), NSteps=n_inner, Friction=15.0, Lambda=5.0, Beta=1.0, StepSize=0.2,
                   MinStepFrac=1.0, rng=rng, batched_replace="per_sample")
    sched = HostSchedule([float(v) for v in sigmas], 2, n_inner, early_stop=early_stop)
    return GraphedJob(eng, sched, (2, 4, 8, 8), "cpu", sampler=sampler, **kw), sched


class _Plan:
    used = 0


@pytest.mark.parametrize("rng", ["torch", "philox"])
def test_graphed_job_draws_and_launches(rng):
    """The fused loop takes no draw of its own: the draw plan is Euler's.  Euler steps launch lp_boundary_midpoint
    on x alone, second-order steps lp_boundary_multistep with the previous step's denoised latent, each step writing
    its own into the other buffer of the pair."""
    for name in ("karras-20", "window-leftover", "one-step"):
        sig = _schedules()[name]
        euler, sched = _job(sig, 5, "euler", rng=rng, early_stop=2)
        job, _ = _job(sig, 5, "res_multistep", rng=rng, early_stop=2)
        assert job.draws_before == euler.draws_before and job.substeps == euler.substeps == sched.substeps
        seen = []
        job.engine._launch_sequence = lambda *a, **kw: seen.append((a[9], kw))   # noqa: E731
        job._dims, job.mask = None, None
        rows = res_multistep_step(sched.sigmas)
        for i, (second, a, b, c, e) in enumerate(rows):
            job._step(i, _Plan(), False)
            out, kw = seen[-1]
            assert out is job.out_pair[i % 2] and kw["euler_coef"] is None and kw["deis"] is None
            if second:
                step, old = kw["multistep"]
                assert kw["midpoint"] is None and old is job.out_pair[(i - 1) % 2]
                assert (step.ratio, step.em1, step.c_cur, step.c_old) == tuple(np.float32(v) for v in (a, b, c, e))
            else:
                step, base, x_out = kw["midpoint"]
                assert kw["multistep"] is None and base is job.x and x_out is job.x
                assert (step.sigma, step.dt) == (np.float32(a), np.float32(b))
        assert euler.multistep is None and euler.out_pair is None


@pytest.mark.parametrize("name", ["karras-20", "flow-simple-10", "window-leftover"])
def test_sampler_in_the_fp32_job_matches_fp64(name):
    """minicomfy's sampler around the reference wrapper (tests/_job_ref.py), fp32 against fp64 on one tape."""
    sig = _schedules()[name]
    flow = name.startswith("flow")
    model = J.Guider(lambda x, s, c: 0.4 * torch.tanh(x) + 0.2, O.FlowSampling() if flow else O.VESampling(), 4.0, 4.0)
    hp = O.Hyper(n_steps=2, flow=flow, min_step_frac=1.0)
    g = torch.Generator().manual_seed(8)
    y, noise = torch.randn(1, 4, 8, 8, generator=g), torch.randn(1, 4, 8, 8, generator=g)
    dm = (torch.rand(1, 1, 8, 8, generator=g) < 0.5).float().expand(1, 4, 8, 8)
    runs = {}
    for dt in (torch.float32, torch.float64):
        tape = O.NoiseTape(generator=torch.Generator().manual_seed(9))
        runs[dt] = J.job(SEEDED, model, y.to(dt), noise.to(dt), dm.to(dt), sig, hp, draw=tape)
    rel = float((runs[torch.float32].double() - runs[torch.float64]).abs().max() / runs[torch.float64].abs().max())
    assert rel <= 4e-6, (name, rel)


def test_gate_and_form_check():
    """The gate takes sample_res_multistep without extra options when extra_args carries a seed; the form check turns
    away a function of the same name that computes something else, and caches its verdict per function."""
    minicomfy.install()
    from lanpaint_b200 import comfy_nodes as N
    from lanpaint_b200.engine import LanPaint

    class K:
        audio_indicator = None
        sigmas_host = [3.0, 1.0, 0.0]
    ks = minicomfy.ksampler("res_multistep")
    eng = LanPaint(None, NSteps=3, Friction=15.0, Lambda=5.0, Beta=1.0, StepSize=0.2, rng="torch")
    dm = torch.ones(1)
    ok = lambda s=ks, ea={"seed": 1}, mo={}: N.KSAMPLER._fused_res_multistep_ok(s, K, dm, mo, eng, ea)   # noqa: E731
    assert ok()
    assert not ok(ea={}) and not ok(ea={"seed": None})
    assert not ok(mo={"callback": lambda *a: None})
    assert not ok(s=minicomfy.ksampler("res_multistep", {"s_noise": 0.5}))
    assert not ok(s=minicomfy.ksampler("dpmpp_2m")) and not ok(s=minicomfy.ksampler("euler"))
    assert not N.KSAMPLER._fused_res_multistep_ok(ks, K, None, {}, eng, {"seed": 1})

    def sample_res_multistep(model, x, sigmas, extra_args=None, callback=None, disable=None):   # dpmpp_2m's update
        return minicomfy.sample_dpmpp_2m(model, x, sigmas, extra_args=extra_args, callback=callback)
    assert not ok(s=minicomfy.KSAMPLER(sample_res_multistep))
    assert N._FORM_OK[(sample_res_multistep, "res_multistep")] is False
    assert N._FORM_OK[(minicomfy.sample_res_multistep, "res_multistep")] is True


FIXTURES = ["node_ksampler_res_multistep", "node_ksampler_res_multistep_mix"]


@pytest.mark.parametrize("name", FIXTURES)
def test_job_loop_reproduces_reference_node_run(name, monkeypatch):
    """The fp32 job with minicomfy's sample_res_multistep (seeded) on a fixture's tape == the reference node layer's
    outputs, bit for bit, draw for draw and network call for network call."""
    monkeypatch.setitem(J.SAMPLERS, "res_multistep", SEEDED)
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    c = json.loads(str(z["meta"]))
    assert c["args"]["sampler_name"] == "res_multistep" and c["node"] == "LanPaint_KSampler"
    got, _, tape, model = NG.fixture_job(z)
    assert tape.pos == c["n_draws"], (tape.pos, c["n_draws"])
    assert model.calls == c["network_calls"], (model.calls, c["network_calls"])
    assert torch.equal(got, torch.from_numpy(z["out"])), float((got - torch.from_numpy(z["out"])).abs().max())
