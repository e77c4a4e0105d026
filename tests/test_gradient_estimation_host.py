"""Host side of the fused gradient_estimation loop: minicomfy's sample_gradient_estimation, the per-step scalars
`schedule.gradient_estimation_step` reads back, lp_boundary_gradient_estimation's formula against the sampler's
expressions, its declaration and what it rejects before any CUDA call, the derivative ring of
`runner.GraphedJob(sampler="gradient_estimation")`, the node gate and its form check, and minicomfy's sampler inside
the fp32 job against fp64 and the reference node layer's fixtures."""
import ctypes as C
import json
import os
import re

import numpy as np
import pytest
import torch

import _job_ref as J
import minicomfy
import test_oracle_node_golden as NG
from _node_cases import NEG, POS
from conftest import GOLDEN_DIR
from lanpaint_b200 import _native
from lanpaint_b200.schedule import gradient_estimation_step
from oracle import langevin_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PLAIN = J._plain(minicomfy.sample_gradient_estimation)


def _schedules():
    eps = minicomfy.ModelPatcher(minicomfy.BaseModel(None), "cpu")
    flow = minicomfy.ModelPatcher(minicomfy.BaseModel(None, model_type=minicomfy.ModelType.FLOW, shift=3.0), "cpu")
    return {"karras-20": J.ksampler_sigmas(eps, 20, "gradient_estimation", "karras"),
            "flow-simple-10": J.ksampler_sigmas(flow, 10, "gradient_estimation", "simple"),
            "window-leftover": J.ksampler_sigmas(eps, 20, "gradient_estimation", "karras", start_step=3, last_step=15),
            "one-step": J.ksampler_sigmas(eps, 1, "gradient_estimation", "karras"),
            "repeated": torch.tensor([6.0, 3.0, 3.0, 1.5, 0.5, 0.0])}


def _older_form(model, x, sigmas, extra_args=None, callback=None, disable=None, ge_gamma=2.0):
    """The gradient-estimation form ComfyUI shipped first: Euler on the first step, x + (ge_gamma d + (1 - ge_gamma)
    old_d) dt after it, and no x = denoised at sigma = 0."""
    extra_args = extra_args or {}
    s_in = x.new_ones([x.shape[0]])
    old_d = None
    for i in range(len(sigmas) - 1):
        denoised = model(x, sigmas[i] * s_in, **extra_args)
        d = (x - denoised) / sigmas[i]
        dt = sigmas[i + 1] - sigmas[i]
        x = x + d * dt if i == 0 else x + (ge_gamma * d + (1 - ge_gamma) * old_d) * dt
        old_d = d
    return x


_older_form.__name__ = "sample_gradient_estimation"


def test_minicomfy_registers_gradient_estimation():
    assert minicomfy.ksampler("gradient_estimation").sampler_function is minicomfy.sample_gradient_estimation
    assert "gradient_estimation" in minicomfy.KSampler.SAMPLERS
    assert "gradient_estimation" not in minicomfy.DISCARD_PENULTIMATE_SIGMA_SAMPLERS
    base = minicomfy.BaseModel(lambda x, sigma, c: 0.5 * x, model_type=minicomfy.ModelType.EPS, latent_channels=4,
                               shift=1.0)
    patcher = minicomfy.ModelPatcher(base, "cpu")
    g = torch.Generator().manual_seed(2)
    latent, noise = torch.randn(1, 4, 8, 8, generator=g), torch.randn(1, 4, 8, 8, generator=g)
    seen = []
    out = minicomfy.KSampler(patcher, 6, "cpu", "gradient_estimation", "karras").sample(
        noise, POS, NEG, 3.0, latent_image=latent, callback=lambda i, x0, x, total: seen.append(i), seed=1)
    assert out.shape == latent.shape and bool(torch.isfinite(out).all()) and seen == list(range(6))


def _kernel_form(x, out, dp, sigma, dt, gm1, final):
    """lp_boundary_gradient_estimation's update (header), one fp32 torch op per kernel operation."""
    d = (x - out) / sigma
    if final:
        return out, d
    u = x + d * dt
    if dp is not None:
        u = u + (gm1 * (d - dp)) * dt
    return u, d


@pytest.mark.parametrize("name", ["karras-20", "flow-simple-10", "window-leftover", "one-step", "repeated"])
def test_step_scalars_are_the_samplers(name):
    """gradient_estimation_step's rows are the sampler's sigma and dt (fp32), gm1 = fp32(ge_gamma - 1), the correction
    from the second step on, x = denoised exactly on the step to sigma = 0, and keep exactly when the next step reads
    d.  The sampler's loop equals the kernel's formula on these scalars, bit for bit."""
    sig = _schedules()[name]
    rows = gradient_estimation_step(sig)
    n = len(sig) - 1
    assert len(rows) == n
    for i, (sigma, dt, gm1, reads, final, keep) in enumerate(rows):
        assert sigma == float(sig[i]) and dt == float(sig[i + 1] - sig[i]) and gm1 == 1.0
        assert final == (float(sig[i + 1]) == 0.0) and reads == (i >= 1 and not final)
        assert keep == (i + 1 < n and rows[i + 1][3])
    if name == "window-leftover":
        assert float(sig[-1]) > 0 and not rows[-1][4]
    assert gradient_estimation_step(sig, 1.3)[0][2] == float(np.float32(1.3 - 1))

    g = torch.Generator().manual_seed(5)
    x0 = torch.randn(2, 3, 5, generator=g)
    model = lambda x, s, **kw: torch.tanh(0.7 * x) + 0.1 * x + 0.05   # noqa: E731
    for gamma in (2.0, 1.3):
        want = minicomfy.sample_gradient_estimation(model, x0.clone(), sig, ge_gamma=gamma)
        t = lambda v: torch.tensor(v, dtype=torch.float32)   # noqa: E731
        x, old = x0.clone(), None
        for sigma, dt, gm1, reads, final, _ in gradient_estimation_step(sig, gamma):
            x, old = _kernel_form(x, model(x, None), old if reads else None, t(sigma), t(dt), t(gm1), final)
        assert torch.equal(x, want), (name, gamma)


def test_kernel_formula_is_the_samplers_bit_for_bit():
    """The header's formula in fp32, with the real scalars of a karras schedule, against the sampler's own expressions
    (a Python float ge_gamma - 1), on random operands with signed zeros and large magnitudes."""
    g = torch.Generator().manual_seed(11)
    n = 1 << 16
    ops = [torch.randn(n, generator=g) * torch.exp(4 * torch.randn(n, generator=g)) for _ in range(3)]
    for o in ops:
        o[:64] = 0.0
        o[64:128] = -0.0
    x, out, old_d = ops
    t = lambda v: torch.tensor(v, dtype=torch.float32)   # noqa: E731
    sig = _schedules()["karras-20"]
    for i, (sigma, dt, gm1, reads, final, _) in enumerate(gradient_estimation_step(sig)):
        d = (x - out) / sig[i]
        step = sig[i + 1] - sig[i]
        if final:
            want = out
        else:
            want = x + d * step
            if i >= 1:
                want = want + ((2.0 - 1) * (d - old_d)) * step
        got, gd = _kernel_form(x, out, old_d if reads else None, t(sigma), t(dt), t(gm1), final)
        assert torch.equal(got, want) and torch.equal(torch.signbit(got), torch.signbit(want)), i
        assert torch.equal(gd, d)


def test_entry_point_is_declared_and_bound():
    header = open(os.path.join(ROOT, "include", "lanpaint_b200.h")).read()
    assert re.search(r"\bint lp_boundary_gradient_estimation\(", header)
    assert "typedef struct lp_gradient_estimation" in header
    assert "#define LP_ABI_VERSION 5" in header and "#define LP_ABI_MINOR 2" in header
    assert "lp_boundary_gradient_estimation" in _native.SYMBOLS
    lib = _native.load()
    fn = lib.lp_boundary_gradient_estimation
    assert fn.restype is C.c_int and len(fn.argtypes) == 13
    assert fn.argtypes[9]._type_ is _native.GradientEstimation
    assert C.sizeof(_native.GradientEstimation) == 16


def test_invalid_arguments_are_refused_before_any_launch():
    lib = _native.load()
    P = C.c_void_p
    fake = 0x1000     # never dereferenced: validation fails first
    dims = _native.Dims(2, 64, 16, 16, 0, 0)      # 128 floats
    heads = _native.Heads(fake, None, _native.DTYPE_F32, 0, 0.0, 0.0)
    known = _native.Known(fake, fake, fake)
    step = _native.GradientEstimation(2.0, -0.5, 1.0, 0)
    final = _native.GradientEstimation(2.0, -2.0, 1.0, 1)
    X, OUT, D0, D1 = 0x200000, 0x300000, 0x400000, 0x500000

    def call(heads=heads, y=fake, noise=fake, mask=fake, known=known, x=X, out=OUT, dout=D0, dp=D1, step=step,
             table=fake, dims=dims):
        ref = lambda o: None if o is None else C.byref(o)   # noqa: E731
        return lib.lp_boundary_gradient_estimation(ref(heads), P(y), P(noise), P(mask), ref(known), P(x), P(out),
                                                   P(dout), P(dp), ref(step), P(table), ref(dims), None)

    INVALID = 1
    assert call(step=None) == INVALID and call(x=None) == INVALID
    assert call(step=final) == INVALID                                            # x = out takes no history
    # d_out, d_prev, x and out overlap none of each other
    for k in ("dout", "dp"):
        assert call(**{k: X}) == INVALID and call(**{k: OUT}) == INVALID, k
        assert call(**{k: X + 4 * 100}) == INVALID and call(**{k: OUT - 4 * 127}) == INVALID, k
    assert call(dout=D1) == INVALID and call(dp=D0 + 4) == INVALID and call(dout=D1 - 4 * 127) == INVALID
    assert call(out=X) == INVALID and call(out=X + 4 * 127) == INVALID
    # everything lp_boundary_known rejects
    assert call(heads=None) == INVALID
    assert call(heads=_native.Heads(None, None, 0, 0, 0.0, 0.0)) == INVALID
    assert call(y=None) == INVALID and call(mask=None) == INVALID
    assert call(noise=None) == INVALID                                            # next_table needs the noise image
    assert call(known=_native.Known(None, fake, fake)) == INVALID
    assert call(known=_native.Known(fake, None, fake)) == INVALID
    assert call(known=_native.Known(fake, fake, None)) == INVALID                 # ... and its packed form
    assert call(heads=_native.Heads(fake, None, 9, 0, 0.0, 0.0)) == INVALID
    assert call(heads=_native.Heads(fake, fake + 64, _native.DTYPE_BF16, 1, 2.0, 2.0)) == INVALID   # combine: fp32 only
    assert call(heads=_native.Heads(fake, fake, _native.DTYPE_F32, 1, 2.0, 2.0)) == INVALID
    assert call(dims=None) == INVALID
    assert call(dims=_native.Dims(2, 100, 30, 100, 0, 0)) == INVALID
    assert call(dims=_native.Dims(1 << 20, 4096, 1024, 4096, 1024, 0)) == 4       # LP_ERR_UNSUPPORTED
    # well-formed calls on an empty batch succeed without a launch
    empty = _native.Dims(0, 64, 16, 16, 0, 0)
    assert call(dims=empty) == 0
    assert call(dims=empty, dp=None, dout=None, table=None, noise=None, known=None, out=None) == 0
    assert call(dims=empty, step=final, dp=None, dout=None, table=None) == 0
    assert call(dims=empty, dout=X) == INVALID                                    # d_out is x itself


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
def test_graphed_job_draws_and_derivative_ring(rng):
    """The sampler draws nothing of its own: the draw plan is Euler's.  Step i writes d into ring[i % 2] exactly when
    the next step reads it, and reads ring[(i - 1) % 2], the buffer the previous step wrote."""
    for name in ("karras-20", "window-leftover", "one-step"):
        sig = _schedules()[name]
        euler, sched = _job(sig, 5, "euler", rng=rng, early_stop=2)
        job, _ = _job(sig, 5, "gradient_estimation", rng=rng, early_stop=2)
        assert job.draws_before == euler.draws_before and job.substeps == euler.substeps == sched.substeps
        rows = gradient_estimation_step(sched.sigmas)
        seen = []
        job.engine._launch_sequence = lambda *a, **kw: seen.append(kw)   # noqa: E731
        job._dims, job.mask = None, None
        written = {}
        for i, (sigma, dt, gm1, reads, final, keep) in enumerate(rows):
            step, r, k = job.ge[i]
            assert (r, k) == (reads, keep)
            assert (step.sigma, step.dt, step.gm1, step.final) == (np.float32(sigma), np.float32(dt), 1.0, int(final))
            job._step(i, _Plan(), False)
            kw = seen[-1]
            assert kw["euler_coef"] is None and kw["multistep"] is None and kw["deis"] is None
            st, d_out, d_prev = kw["ge"]
            assert st is step
            assert d_out is (job.d_ring[i % 2] if keep else None)
            assert d_prev is (written[i - 1] if reads else None)
            written[i] = d_out
        assert job.ge[-1][0].final == (name != "window-leftover")
        assert len({b.data_ptr() for b in job.d_ring}) == 2
        assert euler.ge is None


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
        runs[dt] = J.job(PLAIN, model, y.to(dt), noise.to(dt), dm.to(dt), sig, hp, draw=tape)
    rel = float((runs[torch.float32].double() - runs[torch.float64]).abs().max() / runs[torch.float64].abs().max())
    assert rel <= 4e-6, (name, rel)


def test_gate_and_form_check():
    """The gate takes sample_gradient_estimation without extra options; the form check turns away the older form of
    the same name (it differs on the step to sigma = 0), and caches its verdict per function."""
    minicomfy.install()
    from lanpaint_b200 import comfy_nodes as N
    from lanpaint_b200.engine import LanPaint

    class K:
        audio_indicator = None
        sigmas_host = [3.0, 1.0, 0.0]
    ks = minicomfy.ksampler("gradient_estimation")
    eng = LanPaint(None, NSteps=3, Friction=15.0, Lambda=5.0, Beta=1.0, StepSize=0.2, rng="torch")
    dm = torch.ones(1)
    ok = lambda s=ks, mo={}: N.KSAMPLER._fused_gradient_estimation_ok(s, K, dm, mo, eng)   # noqa: E731
    assert ok()
    assert not ok(mo={"denoise_mask_function": lambda *a, **k: None})
    assert not ok(s=minicomfy.ksampler("gradient_estimation", {"ge_gamma": 1.5}))
    assert not ok(s=minicomfy.ksampler("euler")) and not ok(s=minicomfy.ksampler("res_multistep"))
    assert not N.KSAMPLER._fused_gradient_estimation_ok(ks, K, None, {}, eng)
    assert not ok(s=minicomfy.KSAMPLER(_older_form))
    assert N._FORM_OK[(_older_form, "gradient_estimation")] is False
    assert N._FORM_OK[(minicomfy.sample_gradient_estimation, "gradient_estimation")] is True


FIXTURES = ["node_ksampler_gradient_estimation", "node_ksampler_gradient_estimation_mix"]


@pytest.mark.parametrize("name", FIXTURES)
def test_job_loop_reproduces_reference_node_run(name, monkeypatch):
    """The fp32 job with minicomfy's sample_gradient_estimation on a fixture's tape == the reference node layer's
    outputs, bit for bit, draw for draw and network call for network call."""
    monkeypatch.setitem(J.SAMPLERS, "gradient_estimation", PLAIN)
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    c = json.loads(str(z["meta"]))
    assert c["args"]["sampler_name"] == "gradient_estimation" and c["node"] == "LanPaint_KSampler"
    got, _, tape, model = NG.fixture_job(z)
    assert tape.pos == c["n_draws"], (tape.pos, c["n_draws"])
    assert model.calls == c["network_calls"], (model.calls, c["network_calls"])
    assert torch.equal(got, torch.from_numpy(z["out"])), float((got - torch.from_numpy(z["out"])).abs().max())
