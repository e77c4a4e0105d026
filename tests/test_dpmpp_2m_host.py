"""Host side of the fused dpmpp_2m loop: the per-step scalars `schedule.dpmpp_2m_step` reads back, the draw accounting
and step table of `runner.GraphedJob(sampler="dpmpp_2m")`, what `lp_boundary_multistep` rejects before any CUDA call,
and minicomfy's sample_dpmpp_2m inside the fp64 job."""
import ctypes as C
import os
import re

import pytest
import torch

import _job_ref as J
import minicomfy
from _node_cases import mixing_denoiser
from lanpaint_b200 import _native
from lanpaint_b200.schedule import dpmpp_2m_step
from oracle import langevin_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _schedules():
    patcher = minicomfy.ModelPatcher(minicomfy.BaseModel(None), "cpu")
    return {"karras-20": J.ksampler_sigmas(patcher, 20, "dpmpp_2m", "karras"),
            "simple-20": J.ksampler_sigmas(patcher, 20, "dpmpp_2m", "simple"),
            "window-leftover": J.ksampler_sigmas(patcher, 20, "dpmpp_2m", "karras", start_step=3, last_step=15)}


@pytest.mark.parametrize("name", ["karras-20", "simple-20", "window-leftover"])
def test_step_scalars_are_the_samplers_expressions(name):
    """On a CPU fp32 schedule: dpmpp_2m_step equals k-diffusion's scalar expressions bit for bit, and the sampler's
    own loop equals the same loop written with those scalars in the kernel's operation order."""
    sig = _schedules()[name]
    assert sig.dtype == torch.float32
    steps = dpmpp_2m_step(sig)
    assert len(steps) == len(sig) - 1
    t_fn = lambda s: s.log().neg()          # noqa: E731
    sigma_fn = lambda t: t.neg().exp()      # noqa: E731
    f32 = lambda v: float(v.to(torch.float32))   # noqa: E731
    for i, (ratio, em1, c_cur, c_old, second) in enumerate(steps):
        t, t_next = t_fn(sig[i]), t_fn(sig[i + 1])
        h = t_next - t
        assert ratio == f32(sigma_fn(t_next) / sigma_fn(t)) and em1 == f32((-h).expm1())
        assert second == (i > 0 and float(sig[i + 1]) != 0.0)
        if second:
            r = (t - t_fn(sig[i - 1])) / h
            assert c_cur == f32(1 + 1 / (2 * r)) and c_old == f32(1 / (2 * r))
        else:
            assert c_cur == c_old == 0.0
    if name == "window-leftover":
        assert float(sig[-1]) > 0 and steps[-1][4]         # its last step is second order, sigma_next > 0
    else:
        assert steps[-1][:2] == (0.0, -1.0) and not steps[-1][4]   # the step to sigma = 0: t_next = inf

    g = torch.Generator().manual_seed(5)
    x0 = torch.randn(2, 3, 5, generator=g)
    model = lambda x, s, **kw: torch.tanh(0.7 * x) + 0.1 * x + 0.05   # noqa: E731
    want = minicomfy.sample_dpmpp_2m(model, x0.clone(), sig)
    x, old = x0.clone(), None
    for ratio, em1, c_cur, c_old, second in steps:
        den = model(x, None)
        d = c_cur * den - c_old * old if second else den
        x = ratio * x - em1 * d
        old = den
    assert torch.equal(x, want)


def _job(sigmas, n_inner, sampler, rng="torch", **kw):
    from lanpaint_b200.engine import LanPaint
    from lanpaint_b200.runner import GraphedJob, HostSchedule, VESampling
    eng = LanPaint(O.PointwiseDenoiser(VESampling()), NSteps=n_inner, Friction=15.0, Lambda=5.0, Beta=1.0, StepSize=0.2,
                   MinStepFrac=1.0, rng=rng, batched_replace="per_sample")
    sched = HostSchedule([float(v) for v in sigmas], 2, n_inner)
    return GraphedJob(eng, sched, (2, 4, 8, 8), "cpu", sampler=sampler, **kw), sched


@pytest.mark.parametrize("rng", ["torch", "philox"])
def test_graphed_job_takes_eulers_draws_and_one_step_per_sigma(rng):
    """The sampler draws nothing: the job's draw plan is the Euler job's.  One lp_multistep per outer step, from
    dpmpp_2m_step on the job's schedule; first step and step to sigma = 0 first order."""
    for name, sig in _schedules().items():
        euler, sched = _job(sig, 5, "euler", rng=rng)
        ms, _ = _job(sig, 5, "dpmpp_2m", rng=rng)
        assert ms.draws_before == euler.draws_before and ms.ancestral is None and euler.multistep is None
        want = dpmpp_2m_step(sched.sigmas)
        assert len(ms.multistep) == len(sched.steps) == len(want)
        for (step, second), w in zip(ms.multistep, want):
            assert (step.ratio, step.em1, step.c_cur, step.c_old, second) == w
        assert not ms.multistep[0][1]
        assert ms.multistep[-1][1] == (name == "window-leftover")
        # two denoised-latent buffers taken in turn; Euler keeps its one
        assert ms.denoised_buffer(0, True) is ms.out and ms.denoised_buffer(1, True) is not ms.out
        assert ms.denoised_buffer(2, False) is ms.out and euler.denoised_buffer(1, True) is euler.out
    with pytest.raises(ValueError):
        _job(_schedules()["karras-20"], 5, "dpmpp_3m_sde")


def test_entry_point_is_declared_and_bound():
    header = open(os.path.join(ROOT, "include", "lanpaint_b200.h")).read()
    assert re.search(r"\bint lp_boundary_multistep\(", header) and "typedef struct lp_multistep" in header
    assert "#define LP_ABI_VERSION 5" in header and "#define LP_ABI_MINOR 2" in header
    assert "lp_boundary_multistep" in _native.SYMBOLS
    lib = _native.load()
    assert lib.lp_boundary_multistep.restype is C.c_int and len(lib.lp_boundary_multistep.argtypes) == 12
    assert C.sizeof(_native.Multistep) == 16


def test_invalid_arguments_are_refused_before_any_launch():
    lib = _native.load()
    P = C.c_void_p
    fake, old_fake = 0x1000, 0x100000    # never dereferenced: validation fails first
    dims = _native.Dims(2, 64, 16, 16, 0, 0)
    heads = _native.Heads(fake, None, _native.DTYPE_F32, 0, 0.0, 0.0)
    known = _native.Known(fake, fake, fake)
    step = _native.Multistep(0.5, -0.5, 1.4, 0.4)
    x_fake, out_fake = 0x200000, 0x300000

    def call(heads=heads, y=fake, noise=fake, mask=fake, known=known, x=x_fake, out=out_fake, old=old_fake, step=step,
             table=fake, dims=dims):
        ref = lambda o: None if o is None else C.byref(o)   # noqa: E731
        return lib.lp_boundary_multistep(ref(heads), P(y), P(noise), P(mask), ref(known), P(x), P(out), P(old),
                                         ref(step), P(table), ref(dims), None)

    INVALID = 1
    assert call(step=None) == INVALID
    assert call(x=None) == INVALID                                                # the state is always updated
    assert call(old=x_fake) == INVALID and call(old=out_fake) == INVALID          # old_out aliases an output
    assert call(old=x_fake + 4 * 64) == INVALID                                   # ... or overlaps one (128 floats)
    assert call(old=out_fake - 4 * 100) == INVALID
    # everything lp_boundary rejects
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
    # well-formed calls on an empty batch succeed without a launch: second order, first order, no next step, no out
    empty = _native.Dims(0, 64, 16, 16, 0, 0)
    assert call(dims=empty) == 0
    assert call(dims=empty, old=None, table=None, noise=None, known=None, out=None) == 0
    assert call(dims=empty, old=old_fake + 4 * 64) == 0       # nothing overlaps an empty launch's outputs


def test_sampler_runs_in_the_fp64_job():
    """minicomfy.sample_dpmpp_2m around the fp64 per-sigma wrapper: finite, and not Euler's result."""
    sampler = J._plain(minicomfy.sample_dpmpp_2m)
    shape = (1, 4, 8, 8)
    g = torch.Generator().manual_seed(11)
    y = torch.randn(shape, generator=g, dtype=torch.float64)
    noise = torch.randn(shape, generator=g, dtype=torch.float64)
    dm = (torch.rand((1, 1, 8, 8), generator=g) < 0.5).to(torch.float64).expand(shape)
    patcher = minicomfy.ModelPatcher(minicomfy.BaseModel(mixing_denoiser), "cpu")
    hp = O.Hyper(n_steps=2, lam=5.0, step_size=0.2, min_step_frac=1.0, flow=False)
    res = {}
    for name, fn in (("dpmpp_2m", sampler), ("euler", J.SAMPLERS["euler"])):
        sig = J.ksampler_sigmas(patcher, 6, name, "karras")
        model = J.Guider(mixing_denoiser, O.VESampling(), 5.0, 5.0)
        steps = []
        res[name] = J.job(fn, model, y, noise, dm, sig, hp, draw=lambda like: torch.zeros_like(like),
                          callback=lambda i, d: steps.append(i))
        assert steps == list(range(len(sig) - 1))
    assert torch.isfinite(res["dpmpp_2m"]).all()
    assert not torch.allclose(res["dpmpp_2m"], res["euler"], rtol=1e-6, atol=1e-9)
