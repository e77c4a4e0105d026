"""Host side of the fused dpm_2 loop: the per-step scalars `schedule.dpm_2_step` reads back, minicomfy's discarded
penultimate sigma, the wrapper-equivalent rows of the midpoint calls, the draw accounting of
`runner.GraphedJob(sampler="dpm_2")`, what `lp_boundary_midpoint` rejects before any CUDA call, and minicomfy's
sample_dpm_2 inside the fp32 job against the reference node layer's fixtures."""
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
from conftest import GOLDEN_DIR
from lanpaint_b200 import _native
from lanpaint_b200.schedule import dpm_2_step
from oracle import langevin_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _schedules():
    patcher = minicomfy.ModelPatcher(minicomfy.BaseModel(None), "cpu")
    return {"karras-20": J.ksampler_sigmas(patcher, 20, "dpm_2", "karras"),
            "simple-10": J.ksampler_sigmas(patcher, 10, "dpm_2", "simple"),
            "window-leftover": J.ksampler_sigmas(patcher, 20, "dpm_2", "karras", start_step=3, last_step=15)}


@pytest.mark.parametrize("name", ["karras-20", "simple-10", "window-leftover"])
def test_step_scalars_are_the_samplers_expressions(name):
    """On a CPU fp32 schedule: dpm_2_step equals sample_dpm_2's scalar expressions bit for bit, and the sampler's own
    loop equals the same loop written with those scalars in the kernel's operation order."""
    sig = _schedules()[name]
    assert sig.dtype == torch.float32
    steps = dpm_2_step(sig)
    assert len(steps) == len(sig) - 1
    f32 = lambda v: float(v.to(torch.float32))   # noqa: E731
    for i, (s_mid, dt_1, dt_2, mid) in enumerate(steps):
        sigma_hat = sig[i] * (0.0 + 1)
        assert mid == (float(sig[i + 1]) != 0.0)
        assert dt_2 == f32(sig[i + 1] - sigma_hat)
        if mid:
            want = sigma_hat.log().lerp(sig[i + 1].log(), 0.5).exp()
            assert s_mid == f32(want) and dt_1 == f32(want - sigma_hat)
            assert float(sig[i + 1]) < s_mid < float(sig[i])
        else:
            assert s_mid == dt_1 == 0.0
    assert steps[-1][3] == (name == "window-leftover")

    g = torch.Generator().manual_seed(5)
    x0 = torch.randn(2, 3, 5, generator=g)
    model = lambda x, s, **kw: torch.tanh(0.7 * x) + 0.1 * x + 0.05   # noqa: E731
    want = minicomfy.sample_dpm_2(model, x0.clone(), sig)
    x = x0.clone()
    for i, (s_mid, dt_1, dt_2, mid) in enumerate(steps):
        t = lambda v: torch.tensor(v, dtype=torch.float32)   # noqa: E731
        d = (x - model(x, None)) / t(float(sig[i]))
        if not mid:
            x = x + d * t(dt_2)
            continue
        x2 = x + d * t(dt_1)
        x = x + ((x2 - model(x2, None)) / t(s_mid)) * t(dt_2)
    assert torch.equal(x, want)


def test_schedule_drops_the_penultimate_sigma():
    """KSampler takes one step more for dpm_2 and drops the penultimate sigma, in the denoise < 1 branch too; the
    other samplers' schedules are unchanged."""
    patcher = minicomfy.ModelPatcher(minicomfy.BaseModel(None), "cpu")
    ms = patcher.model.model_sampling
    for sched in ("karras", "simple"):
        got = minicomfy.KSampler(patcher, 8, "cpu", "dpm_2", sched).sigmas
        full = minicomfy.KSampler(patcher, 9, "cpu", "euler", sched).sigmas
        assert len(got) == 9 and torch.equal(got, torch.cat([full[:-2], full[-1:]]))
        assert torch.equal(minicomfy.KSampler(patcher, 8, "cpu", "heun", sched).sigmas,
                           minicomfy.KSampler(patcher, 8, "cpu", "euler", sched).sigmas)
    want = minicomfy.get_sigmas_karras(9, float(ms.sigma_min), float(ms.sigma_max))
    assert torch.equal(minicomfy.KSampler(patcher, 8, "cpu", "dpm_2", "karras").sigmas,
                       torch.cat([want[:-2], want[-1:]]))
    part = minicomfy.KSampler(patcher, 6, "cpu", "dpm_2", "karras", denoise=0.5).sigmas
    assert torch.equal(part, minicomfy.KSampler(patcher, 12, "cpu", "dpm_2", "karras").sigmas[-7:])


class _StubEngine:
    """What the per-sigma wrapper calls: returns a denoised latent and records nothing itself."""

    def __init__(self, n_steps):
        self.n_steps = n_steps

    def __call__(self, x, latent_image, noise, sigma, mask, times, model_options, seed, n_steps=None, **kw):
        return torch.tanh(0.5 * x) + 0.1 * latent_image


class _Gen:
    def get_offset(self):
        return 0


@pytest.mark.parametrize("early_stop,min_frac", [(1, 1.0), (2, 1.0), (1, 0.6)])
def test_planned_calls_are_what_the_wrapper_records(early_stop, min_frac, monkeypatch):
    """Every wrapper call sample_dpm_2 makes through comfy_nodes.KSamplerX0Inpaint -- sigma, times and n_eff, the
    midpoint calls' by the nearest-sigma rule -- equals the row GraphedJob(sampler="dpm_2") plans for it."""
    minicomfy.install()
    from lanpaint_b200 import comfy_nodes as N
    from lanpaint_b200.runner import HostSchedule
    monkeypatch.setattr(N, "pack_mask", lambda known, like: None)     # the stub engine takes no mask
    monkeypatch.setattr(torch.cuda, "default_generators", (_Gen(),))
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)
    B, n = 2, 4
    for name, sig in _schedules().items():
        base = minicomfy.BaseModel(None)
        model = type("Wrap", (), {"inner_model": base})()
        wk = N.KSamplerX0Inpaint(model, sig)
        wk.latent_image = torch.randn(B, 4, 8, 8, generator=torch.Generator().manual_seed(1))
        wk.noise = torch.zeros_like(wk.latent_image)
        wk.PaintMethod, wk.LanPaint_early_stop, wk.LanPaint_min_step_frac = _StubEngine(n), early_stop, min_frac
        wk.trace = []
        dm = torch.ones(B, 1, 8, 8)
        minicomfy.sample_dpm_2(lambda x, s, **kw: wk(x, s, dm), wk.latent_image.clone(), sig)

        sched = HostSchedule(wk.sigmas_host, B, n, False, early_stop, min_frac)
        planned = []
        for st, (s_mid, _, _, mid) in zip(sched.steps, dpm_2_step(sig)):
            planned.append(st)
            if mid:
                planned.append(sched.call_at(s_mid, st.sigma_next))
        assert len(wk.trace) == len(planned)
        for (s, tm, n_eff), st in zip(wk.trace, planned):
            assert torch.equal(s, st.sigma_t) and n_eff == st.n_inner
            assert all(torch.equal(a, b) for a, b in zip(tm, st.times))
        mids = [st for st in planned if float(st.sigma) not in wk.sigmas_host]
        assert len(mids) == sum(mid for *_, mid in dpm_2_step(sig))
        if early_stop == 2 and name != "window-leftover":
            assert any(st.n_inner == 0 for st in mids), name     # a midpoint call with no Langevin sub-step
        if min_frac < 1.0:
            assert {st.n_inner for st in planned} - {0, n}, name     # ... and one on the MinStepFrac ramp


def _job(sigmas, n_inner, sampler, rng="torch", early_stop=1, **kw):
    from lanpaint_b200.engine import LanPaint
    from lanpaint_b200.runner import GraphedJob, HostSchedule, VESampling
    eng = LanPaint(O.PointwiseDenoiser(VESampling()), NSteps=n_inner, Friction=15.0, Lambda=5.0, Beta=1.0, StepSize=0.2,
                   MinStepFrac=1.0, rng=rng, batched_replace="per_sample")
    sched = HostSchedule([float(v) for v in sigmas], 2, n_inner, early_stop=early_stop)
    return GraphedJob(eng, sched, (2, 4, 8, 8), "cpu", sampler=sampler, **kw), sched


@pytest.mark.parametrize("rng", ["torch", "philox"])
def test_graphed_job_counts_both_calls(rng):
    """The sampler draws nothing of its own: each outer step takes the Langevin draws of call A and call B.  One
    predictor per step, a corrector and a midpoint row where sigma_next > 0; sub-steps cover both calls."""
    for name, sig in _schedules().items():
        euler, sched = _job(sig, 5, "euler", rng=rng, early_stop=2)
        job, _ = _job(sig, 5, "dpm_2", rng=rng, early_stop=2)
        per_call = lambda n: 0 if n <= 0 else (n if rng == "philox" else 2 * n - 1)   # noqa: E731
        steps = dpm_2_step(sched.sigmas)
        want, subs, k = [0], sched.substeps, 0
        for i, (st, (s_mid, dt_1, dt_2, mid)) in enumerate(zip(sched.steps, steps)):
            pred, corr, idx = job.midpoint[i]
            assert (pred.sigma, pred.dt) == (np.float32(st.sigma), np.float32(dt_1 if mid else dt_2))
            own = 0
            if mid:
                ms = sched.call_at(s_mid, st.sigma_next)
                assert idx == k and (corr.sigma, corr.dt) == (np.float32(s_mid), np.float32(dt_2))
                assert job.mid_active[k] == ms.n_inner
                assert torch.equal(job.mid_sigma[k], ms.sigma_t) and torch.equal(job.mid_t_model[k], ms.times[0])
                own, subs, k = per_call(ms.n_inner), subs + ms.n_inner, k + 1
            else:
                assert corr is None and idx is None
            want.append(want[-1] + per_call(job.active[i]) + own)
        assert job.draws_before == want and job.substeps == subs and job.x2 is not None
        assert euler.draws_before[-1] < job.draws_before[-1] and euler.midpoint is None and euler.x2 is None
        assert job.mid_tables.shape == (k,) + tuple(job.tables.shape[1:])
    with pytest.raises(ValueError):
        _job(_schedules()["karras-20"], 5, "dpm_2_ancestral")


def test_entry_point_is_declared_and_bound():
    header = open(os.path.join(ROOT, "include", "lanpaint_b200.h")).read()
    assert re.search(r"\bint lp_boundary_midpoint\(", header) and "typedef struct lp_midpoint" in header
    assert "#define LP_ABI_VERSION 5" in header and "#define LP_ABI_MINOR 2" in header
    assert "lp_boundary_midpoint" in _native.SYMBOLS
    lib = _native.load()
    assert lib.lp_boundary_midpoint.restype is C.c_int and len(lib.lp_boundary_midpoint.argtypes) == 13
    assert C.sizeof(_native.Midpoint) == 8


def test_invalid_arguments_are_refused_before_any_launch():
    lib = _native.load()
    P = C.c_void_p
    fake = 0x1000     # never dereferenced: validation fails first
    dims = _native.Dims(2, 64, 16, 16, 0, 0)      # 128 floats
    heads = _native.Heads(fake, None, _native.DTYPE_F32, 0, 0.0, 0.0)
    known = _native.Known(fake, fake, fake)
    step = _native.Midpoint(2.0, -0.5)
    X, X2, OUT = 0x200000, 0x300000, 0x400000

    def call(heads=heads, y=fake, noise=fake, mask=fake, known=known, xin=X, xbase=X, xout=X2, out=OUT, step=step,
             table=fake, dims=dims):
        ref = lambda o: None if o is None else C.byref(o)   # noqa: E731
        return lib.lp_boundary_midpoint(ref(heads), P(y), P(noise), P(mask), ref(known), P(xin), P(xbase), P(xout),
                                        P(out), ref(step), P(table), ref(dims), None)

    INVALID = 1
    assert call(step=None) == INVALID
    assert call(xin=None) == INVALID and call(xbase=None) == INVALID and call(xout=None) == INVALID
    # x_in, x_base, x_out: each pair one buffer or disjoint
    assert call(xout=X + 4) == INVALID and call(xout=X - 4 * 127) == INVALID
    assert call(xbase=X2 + 4 * 64, xin=X2, xout=X) == INVALID
    assert call(xin=X + 4 * 64, xbase=X, xout=X2) == INVALID
    # out overlaps none of them
    assert call(out=X) == INVALID and call(out=X2) == INVALID and call(out=X + 4 * 100) == INVALID
    assert call(xin=X2, xbase=X, xout=X, out=X2 - 4 * 64) == INVALID
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
    # well-formed calls on an empty batch succeed without a launch, in every aliasing role
    empty = _native.Dims(0, 64, 16, 16, 0, 0)
    assert call(dims=empty) == 0                                                  # predictor
    assert call(dims=empty, xin=X2, xbase=X, xout=X, table=None, noise=None, known=None, out=None) == 0   # corrector
    assert call(dims=empty, xout=X, table=None) == 0                              # the step to sigma = 0
    assert call(dims=empty, out=X) == INVALID                                     # out is x_in itself


DPM_2_FIXTURES = ["node_ksampler_dpm_2", "node_ksampler_dpm_2_mix"]


@pytest.mark.parametrize("name", DPM_2_FIXTURES)
def test_job_loop_reproduces_reference_node_run(name, monkeypatch):
    """The fp32 job with minicomfy's sample_dpm_2 on a fixture's tape == the reference node layer's outputs, bit for
    bit, draw for draw and network call for network call (the wrapper at every midpoint sigma included)."""
    monkeypatch.setitem(J.SAMPLERS, "dpm_2", J._plain(minicomfy.sample_dpm_2))
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    c = json.loads(str(z["meta"]))
    assert c["args"]["sampler_name"] == "dpm_2" and c["node"] == "LanPaint_KSampler"
    got, _, tape, model = NG.fixture_job(z)
    assert tape.pos == c["n_draws"], (tape.pos, c["n_draws"])
    assert model.calls == c["network_calls"], (model.calls, c["network_calls"])
    assert torch.equal(got, torch.from_numpy(z["out"])), float((got - torch.from_numpy(z["out"])).abs().max())
