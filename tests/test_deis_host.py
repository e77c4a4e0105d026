"""Host side of the fused deis loop: minicomfy's sample_deis and its coefficients, the per-step scalars
`schedule.deis_step` reads back, the derivative ring and draw accounting of `runner.GraphedJob(sampler="deis")`,
what `lp_boundary_deis` rejects before any CUDA call, and minicomfy's sample_deis inside the fp32 job against the
reference node layer's fixtures."""
import ctypes as C
import json
import os
import re
import sys

import numpy as np
import pytest
import torch

import _job_ref as J
import minicomfy
import test_oracle_node_golden as NG
from _node_cases import NEG, POS
from conftest import GOLDEN_DIR
from lanpaint_b200 import _native
from lanpaint_b200.schedule import deis_step
from oracle import langevin_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _schedules():
    patcher = minicomfy.ModelPatcher(minicomfy.BaseModel(None), "cpu")
    return {"karras-20": J.ksampler_sigmas(patcher, 20, "deis", "karras"),
            "simple-10": J.ksampler_sigmas(patcher, 10, "deis", "simple"),
            "window-leftover": J.ksampler_sigmas(patcher, 20, "deis", "karras", start_step=3, last_step=15)}


def test_minicomfy_registers_deis():
    """"deis" is a minicomfy sampler, its module carries the `deis` coefficient module as ComfyUI's
    k_diffusion.sampling does, and KSampler runs it end to end; the other samplers and modules are unchanged."""
    assert minicomfy.ksampler("deis").sampler_function is minicomfy.sample_deis
    assert "deis" in minicomfy.KSampler.SAMPLERS
    assert sys.modules[minicomfy.sample_deis.__module__].deis is minicomfy.deis
    assert callable(minicomfy.deis.get_deis_coeff_list)
    assert {"euler", "heun", "euler_ancestral", "dpmpp_2m", "dpm_2"} < set(minicomfy.KSampler.SAMPLERS)
    patcher = minicomfy.ModelPatcher(minicomfy.BaseModel(None), "cpu")
    assert torch.equal(minicomfy.KSampler(patcher, 8, "cpu", "deis", "karras").sigmas,
                       minicomfy.KSampler(patcher, 8, "cpu", "euler", "karras").sigmas)

    base = minicomfy.BaseModel(lambda x, sigma, c: 0.5 * x, model_type=minicomfy.ModelType.EPS, latent_channels=4,
                               shift=1.0)
    patcher = minicomfy.ModelPatcher(base, "cpu")
    g = torch.Generator().manual_seed(2)
    latent, noise = torch.randn(1, 4, 8, 8, generator=g), torch.randn(1, 4, 8, 8, generator=g)
    seen = []
    out = minicomfy.KSampler(patcher, 6, "cpu", "deis", "karras").sample(
        noise, POS, NEG, 3.0, latent_image=latent, callback=lambda i, x0, x, total: seen.append(i), seed=1)
    assert out.shape == latent.shape and bool(torch.isfinite(out).all()) and seen == list(range(6))


@pytest.mark.parametrize("name", ["karras-20", "simple-10", "window-leftover"])
def test_coefficients_sum_to_the_sigma_step(name):
    """The integrand of `cal_intergrand` is d sigma / d tau and the Lagrange basis sums to 1, so each step's
    coefficients sum to sigma_next - sigma up to the quadrature error; orders are 1, 2, 3, ..., 3 and 1 on the step to
    sigma = 0 (a leftover window ends in order 3)."""
    sig = _schedules()[name]
    rows = deis_step(minicomfy.sample_deis, sig)
    orders = [r[4] for r in rows]
    n = len(sig) - 1
    if name == "window-leftover":
        assert float(sig[-1]) > 0 and orders == [1, 2] + [3] * (n - 2)
    else:
        assert orders == [1, 2] + [3] * (n - 3) + [1]
    for i, (sigma, c_cur, c_prev1, c_prev2, order) in enumerate(rows):
        step = float(sig[i + 1]) - float(sig[i])
        assert sigma == float(sig[i])
        if order == 1:
            assert c_cur == float(sig[i + 1] - sig[i]) and c_prev1 == c_prev2 == 0.0
            continue
        assert (c_prev2 == 0.0) == (order == 2)
        assert abs(c_cur + c_prev1 + c_prev2 - step) <= 1e-3 * abs(step), (name, i)
        assert c_cur < 0 < c_prev1      # the current derivative leads, the previous one pulls back


@pytest.mark.parametrize("name", ["karras-20", "simple-10", "window-leftover"])
def test_step_scalars_are_the_samplers(name):
    """On a CPU fp32 schedule: deis_step's coefficients are get_deis_coeff_list's values, and the sampler's own loop
    equals the same loop written with deis_step's scalars in the kernel's operation order."""
    sig = _schedules()[name]
    rows = deis_step(minicomfy.sample_deis, sig)
    with torch.no_grad():
        coeff = minicomfy.deis.get_deis_coeff_list(sig, 3)
    for i, (_, c_cur, c_prev1, c_prev2, order) in enumerate(rows):
        if order > 1:
            assert [c_cur, c_prev1, c_prev2][:order] == [float(v) for v in coeff[i]]

    g = torch.Generator().manual_seed(5)
    x0 = torch.randn(2, 3, 5, generator=g)
    model = lambda x, s, **kw: torch.tanh(0.7 * x) + 0.1 * x + 0.05   # noqa: E731
    want = minicomfy.sample_deis(model, x0.clone(), sig)
    t = lambda v: torch.tensor(v, dtype=torch.float32)   # noqa: E731
    x, hist = x0.clone(), []
    for sigma, c_cur, c_prev1, c_prev2, order in rows:
        d = (x - model(x, None)) / t(sigma)
        x = x + t(c_cur) * d
        if order >= 2:
            x = x + t(c_prev1) * hist[-1]
        if order >= 3:
            x = x + t(c_prev2) * hist[-2]
        hist = (hist + [d])[-2:]
    assert torch.equal(x, want)


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
    """The sampler draws nothing of its own: the draw plan is Euler's.  Step i writes its derivative into ring[i % 3]
    exactly when a later step reads it, and reads ring[(i-1) % 3] (order >= 2) and ring[(i-2) % 3] (order 3): the
    buffers the two previous steps wrote."""
    for name, sig in _schedules().items():
        euler, sched = _job(sig, 5, "euler", rng=rng, early_stop=2)
        for fused in (True, False):
            job, _ = _job(sig, 5, "deis", rng=rng, early_stop=2, sampler_fn=minicomfy.sample_deis, fused_euler=fused)
            assert job.draws_before == euler.draws_before and job.substeps == euler.substeps == sched.substeps
            rows = deis_step(minicomfy.sample_deis, sched.sigmas)
            seen = []
            job.engine._launch_sequence = lambda *a, **kw: seen.append(kw["deis"])   # noqa: E731
            job._dims, job.mask = None, None
            written = {}
            for i, (sigma, c_cur, c_prev1, c_prev2, order) in enumerate(rows):
                step, o, keep = job.deis[i]
                assert o == order and keep == (i + 1 < len(rows) and rows[i + 1][4] >= 2)
                assert (step.sigma, step.c_cur, step.c_prev1, step.c_prev2) == tuple(
                    np.float32(v) for v in (sigma, c_cur, c_prev1, c_prev2))
                if not fused:
                    continue
                job._step(i, _Plan(), False)
                st, d_out, p1, p2 = seen[-1]
                assert st is step
                assert d_out is (job.d_ring[i % 3] if keep else None)
                assert p1 is (written[i - 1] if order >= 2 else None)
                assert p2 is (written[i - 2] if order >= 3 else None)
                written[i] = d_out
            assert len({b.data_ptr() for b in job.d_ring}) == 3
        assert euler.deis is None and euler.d_ring is None
    with pytest.raises(ValueError):
        _job(_schedules()["karras-20"], 5, "deis")          # the coefficients are the sampler function's own


def test_entry_point_is_declared_and_bound():
    header = open(os.path.join(ROOT, "include", "lanpaint_b200.h")).read()
    assert re.search(r"\bint lp_boundary_deis\(", header) and "typedef struct lp_deis" in header
    assert "#define LP_ABI_VERSION 5" in header and "#define LP_ABI_MINOR 2" in header
    assert "lp_boundary_deis" in _native.SYMBOLS
    lib = _native.load()
    assert lib.lp_boundary_deis.restype is C.c_int and len(lib.lp_boundary_deis.argtypes) == 14
    assert C.sizeof(_native.Deis) == 16


def test_invalid_arguments_are_refused_before_any_launch():
    lib = _native.load()
    P = C.c_void_p
    fake = 0x1000     # never dereferenced: validation fails first
    dims = _native.Dims(2, 64, 16, 16, 0, 0)      # 128 floats
    heads = _native.Heads(fake, None, _native.DTYPE_F32, 0, 0.0, 0.0)
    known = _native.Known(fake, fake, fake)
    step = _native.Deis(2.0, -0.5, 0.25, -0.125)
    X, OUT, D0, D1, D2 = 0x200000, 0x300000, 0x400000, 0x500000, 0x600000

    def call(heads=heads, y=fake, noise=fake, mask=fake, known=known, x=X, out=OUT, dout=D0, p1=D1, p2=D2, step=step,
             table=fake, dims=dims):
        ref = lambda o: None if o is None else C.byref(o)   # noqa: E731
        return lib.lp_boundary_deis(ref(heads), P(y), P(noise), P(mask), ref(known), P(x), P(out), P(dout), P(p1),
                                    P(p2), ref(step), P(table), ref(dims), None)

    INVALID = 1
    assert call(step=None) == INVALID and call(x=None) == INVALID
    assert call(p1=None) == INVALID                                               # d_prev2 without d_prev1
    # the histories overlap neither each other nor x or out
    for k in ("dout", "p1", "p2"):
        assert call(**{k: X}) == INVALID and call(**{k: OUT}) == INVALID, k
        assert call(**{k: X + 4 * 100}) == INVALID and call(**{k: OUT - 4 * 127}) == INVALID, k
    assert call(dout=D1) == INVALID and call(p2=D1) == INVALID and call(dout=D2 + 4) == INVALID
    assert call(p1=D0 - 4 * 64) == INVALID
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
    # well-formed calls on an empty batch succeed without a launch, for every order
    empty = _native.Dims(0, 64, 16, 16, 0, 0)
    assert call(dims=empty) == 0                                                  # third order
    assert call(dims=empty, p2=None) == 0                                         # second order
    assert call(dims=empty, p1=None, p2=None, dout=None, table=None, noise=None, known=None, out=None) == 0
    assert call(dims=empty, dout=X) == INVALID                                    # d_out is x itself


DEIS_FIXTURES = ["node_ksampler_deis", "node_ksampler_deis_mix"]


@pytest.mark.parametrize("name", DEIS_FIXTURES)
def test_job_loop_reproduces_reference_node_run(name, monkeypatch):
    """The fp32 job with minicomfy's sample_deis on a fixture's tape == the reference node layer's outputs, bit for
    bit, draw for draw and network call for network call."""
    monkeypatch.setitem(J.SAMPLERS, "deis", J._plain(minicomfy.sample_deis))
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    c = json.loads(str(z["meta"]))
    assert c["args"]["sampler_name"] == "deis" and c["node"] == "LanPaint_KSampler"
    got, _, tape, model = NG.fixture_job(z)
    assert tape.pos == c["n_draws"], (tape.pos, c["n_draws"])
    assert model.calls == c["network_calls"], (model.calls, c["network_calls"])
    assert torch.equal(got, torch.from_numpy(z["out"])), float((got - torch.from_numpy(z["out"])).abs().max())
