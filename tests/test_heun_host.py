"""Host side of the fused heun loop: the per-step scalars `schedule.heun_step` reads back, lp_boundary_heun's formula
against the sampler's expressions, its declaration and what it rejects before any CUDA call, the wrapper rows, draw
accounting and launch arguments of `runner.GraphedJob(sampler="heun")`, and the node gate with its form check."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import _job_ref as J
import minicomfy
from lanpaint_b200 import _native
from lanpaint_b200.schedule import heun_step
from oracle import langevin_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _schedules():
    eps = minicomfy.ModelPatcher(minicomfy.BaseModel(None), "cpu")
    flow = minicomfy.ModelPatcher(minicomfy.BaseModel(None, model_type=minicomfy.ModelType.FLOW, shift=3.0), "cpu")
    return {"karras-20": J.ksampler_sigmas(eps, 20, "heun", "karras"),
            "flow-simple-10": J.ksampler_sigmas(flow, 10, "heun", "simple"),
            "window-leftover": J.ksampler_sigmas(eps, 20, "heun", "karras", start_step=3, last_step=15),
            "one-step": J.ksampler_sigmas(eps, 1, "heun", "karras")}


def _corrector(x, out_prev, x2, out, sigma, sigma_next, dt, half):
    """lp_boundary_heun's update (header), one fp32 torch op per kernel operation; /2 or *0.5 as `half` says."""
    s = ((x - out_prev) / sigma) + ((x2 - out) / sigma_next)
    return x + (s / 2 if half == "div" else s * 0.5) * dt


@pytest.mark.parametrize("name", ["karras-20", "flow-simple-10", "window-leftover", "one-step"])
def test_step_scalars_are_the_samplers(name):
    """heun_step's rows are the sampler's sigma_hat, dt and sigma_next (fp32), with a corrector exactly where
    sigma_next != 0.  The sampler's loop equals the fused loop's launches on these scalars -- lp_boundary_midpoint's
    predictor and Euler step, lp_boundary_heun's corrector recomputing d -- bit for bit."""
    sig = _schedules()[name]
    assert sig.dtype == torch.float32
    rows = heun_step(sig)
    assert len(rows) == len(sig) - 1
    f32 = lambda v: float(v.to(torch.float32))   # noqa: E731
    for i, (sigma, dt, sigma_next, corrector) in enumerate(rows):
        sigma_hat = sig[i] * (0.0 + 1)
        assert sigma == f32(sigma_hat) == float(sig[i]) and dt == f32(sig[i + 1] - sigma_hat)
        assert sigma_next == float(sig[i + 1]) and corrector == (float(sig[i + 1]) != 0.0)
    assert rows[-1][3] == (name == "window-leftover")

    g = torch.Generator().manual_seed(5)
    x0 = torch.randn(2, 3, 5, generator=g)
    model = lambda x, s, **kw: torch.tanh(0.7 * x) + 0.1 * x + 0.05   # noqa: E731
    want = minicomfy.sample_heun(model, x0.clone(), sig)
    t = lambda v: torch.tensor(v, dtype=torch.float32)   # noqa: E731
    x = x0.clone()
    for sigma, dt, sigma_next, corrector in rows:
        out = model(x, None)
        x2 = x + ((x - out) / t(sigma)) * t(dt)          # lp_boundary_midpoint, x_in = x_base = x
        if not corrector:
            x = x2
            continue
        x = _corrector(x, out, x2, model(x2, None), t(sigma), t(sigma_next), t(dt), "mul")
    assert torch.equal(x, want), name


def test_kernel_formula_is_the_samplers_bit_for_bit():
    """The header's formula in fp32, with /2 and with *0.5, against sample_heun's own expressions (d from the first
    call, d_2 from the second, (d + d_2) / 2 * dt), with the real scalars of a karras schedule, on operands that include
    signed zeros, subnormals and large magnitudes."""
    g = torch.Generator().manual_seed(11)
    n = 1 << 16
    ops = [torch.randn(n, generator=g) * torch.exp(4 * torch.randn(n, generator=g)) for _ in range(4)]
    tiny = torch.finfo(torch.float32).smallest_normal
    for k, o in enumerate(ops):
        o[:64] = 0.0
        o[64:128] = -0.0
        o[128:512] = torch.randint(-64, 64, (384,), generator=g).float() * (tiny / 64) * (k + 1)   # subnormals
        o[512:576] = torch.randn(64, generator=g) * 1e36
    x, den, x_2, den_2 = ops
    assert bool(((x.abs() < tiny) & (x != 0)).any())
    t = lambda v: torch.tensor(v, dtype=torch.float32)   # noqa: E731
    sig = _schedules()["karras-20"]
    for i, (sigma, dt, sigma_next, corrector) in enumerate(heun_step(sig)):
        if not corrector:
            continue
        s_in = torch.ones(1)
        d = (x - den) / (sig[i] * s_in)
        d_2 = (x_2 - den_2) / (sig[i + 1] * s_in)
        want = x + (d + d_2) / 2 * (sig[i + 1] - sig[i])
        for half in ("div", "mul"):
            got = _corrector(x, den, x_2, den_2, t(sigma), t(sigma_next), t(dt), half)
            assert torch.equal(got.view(torch.int32), want.view(torch.int32)), (i, half)   # bits: signed zeros too
    # subnormal sums halved: the multiply by 0.5 and the division by 2 round alike
    s = torch.arange(-300, 300, dtype=torch.float32) * (tiny / 128)
    assert torch.equal(s / 2, s * 0.5) and bool((s / 2 != 0).any())


def test_entry_point_is_declared_and_bound():
    header = open(os.path.join(ROOT, "include", "lanpaint_b200.h")).read()
    assert re.search(r"\bint lp_boundary_heun\(", header) and "typedef struct lp_heun" in header
    assert "#define LP_ABI_VERSION 5" in header and "#define LP_ABI_MINOR 2" in header
    assert "lp_boundary_heun" in _native.SYMBOLS
    lib = _native.load()
    fn = lib.lp_boundary_heun
    assert fn.restype is C.c_int and len(fn.argtypes) == 13
    assert fn.argtypes[9]._type_ is _native.Heun
    assert C.sizeof(_native.Heun) == 12
    assert lib.lp_abi_version() == 5


def test_invalid_arguments_are_refused_before_any_launch():
    lib = _native.load()
    P = C.c_void_p
    fake = 0x1000     # never dereferenced: validation fails first
    dims = _native.Dims(2, 64, 16, 16, 0, 0)      # 128 floats
    heads = _native.Heads(fake, None, _native.DTYPE_F32, 0, 0.0, 0.0)
    known = _native.Known(fake, fake, fake)
    step = _native.Heun(2.0, 1.5, -0.5)
    X, X2, PREV, OUT = 0x200000, 0x300000, 0x400000, 0x500000

    def call(heads=heads, y=fake, noise=fake, mask=fake, known=known, x=X, x2=X2, prev=PREV, out=OUT, step=step,
             table=fake, dims=dims):
        ref = lambda o: None if o is None else C.byref(o)   # noqa: E731
        return lib.lp_boundary_heun(ref(heads), P(y), P(noise), P(mask), ref(known), P(x), P(x2), P(prev), P(out),
                                    ref(step), P(table), ref(dims), None)

    INVALID = 1
    assert call(step=None) == INVALID
    assert call(x=None) == INVALID and call(x2=None) == INVALID and call(prev=None) == INVALID
    # x, x2, out_prev and out overlap none of each other
    bufs = {"x": X, "x2": X2, "prev": PREV, "out": OUT}
    for a in bufs:
        for b, base in bufs.items():
            if a != b:
                assert call(**{a: base}) == INVALID, (a, b)
                assert call(**{a: base + 4 * 100}) == INVALID and call(**{a: base - 4 * 127}) == INVALID, (a, b)
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
    assert call(dims=empty, table=None, noise=None, known=None, out=None) == 0   # the last corrector of a window
    assert call(dims=empty, out=PREV) == INVALID                                  # out is out_prev itself


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
    """Every wrapper call sample_heun makes through comfy_nodes.KSamplerX0Inpaint -- sigma, times and n_eff -- equals
    the row GraphedJob(sampler="heun") plans for it; call B's row is the next outer step's wherever there is one."""
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
        minicomfy.sample_heun(lambda x, s, **kw: wk(x, s, dm), wk.latent_image.clone(), sig)

        sched = HostSchedule(wk.sigmas_host, B, n, False, early_stop, min_frac)
        planned = []
        for i, (st, (_, _, s_next, corrector)) in enumerate(zip(sched.steps, heun_step(sig))):
            planned.append(st)
            if corrector:
                ms = sched.call_at(s_next, st.sigma_next)
                if i + 1 < len(sched.steps):
                    nx = sched.steps[i + 1]
                    assert ms.sigma == nx.sigma and ms.n_inner == nx.n_inner and torch.equal(ms.sigma_t, nx.sigma_t)
                    assert all(torch.equal(a, b) for a, b in zip(ms.times, nx.times))
                planned.append(ms)
        assert len(wk.trace) == len(planned), name
        for (s, tm, n_eff), st in zip(wk.trace, planned):
            assert torch.equal(s, st.sigma_t) and n_eff == st.n_inner
            assert all(torch.equal(a, b) for a, b in zip(tm, st.times))


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
@pytest.mark.parametrize("want_out", [False, True, "each"])
def test_graphed_job_launches_rows_and_draws(rng, want_out):
    """Per outer step: call A on x with the predictor (x -> x2, call B's replace step) or, on the step to sigma = 0,
    the Euler step on x; call B on x2 with lp_boundary_heun, whose out_prev is the buffer call A wrote its denoised
    latent to, and the next outer step's replace step (none after a window that ends above 0).  Call B's row is the
    next step's wherever there is one; the draw plan counts both calls' Langevin draws, as the per-sigma route does."""
    for name in ("karras-20", "window-leftover", "one-step"):
        sig = _schedules()[name]
        job, sched = _job(sig, 5, "heun", rng=rng, early_stop=2, sampler_fn=minicomfy.sample_heun)
        euler, _ = _job(sig, 5, "euler", rng=rng, early_stop=2)
        if want_out == "each":
            job.outs = [torch.empty_like(job.x) for _ in sched.steps]
        per_call = lambda n: 0 if n <= 0 else (n if rng == "philox" else 2 * n - 1)   # noqa: E731
        rows = heun_step(sched.sigmas)
        seen = []
        job.engine._launch_sequence = lambda xm, *a, **kw: seen.append((xm, a, kw))   # noqa: E731
        job._dims, job.mask = None, None
        draws, subs, n_steps = [0], sched.substeps, len(sched.steps)
        for i, (st, (sigma, dt, s_next, corrector)) in enumerate(zip(sched.steps, rows)):
            del seen[:]
            plan = _Plan()
            job._step(i, plan, want_out)
            pred, corr, k = job.midpoint[i]
            assert (pred.sigma, pred.dt) == (np.float32(sigma), np.float32(dt))
            xm, a, kw = seen[0]
            assert xm is job.x and kw["midpoint"][0] is pred and kw["midpoint"][1] is job.x
            out = a[8]
            if want_out == "each":
                assert out is job.outs[i]
            elif corrector or want_out:
                assert out is job.out
            else:
                assert out is None
            after = job.tables[i + 1] if i + 1 < n_steps else None
            own = 0
            if not corrector:
                assert len(seen) == 1 and corr is None and k is None
                assert kw["midpoint"][2] is job.x
                assert (kw["next_table"] is None) == (after is None)
            else:
                assert len(seen) == 2
                assert kw["midpoint"][2] is job.x2
                assert kw["next_table"].data_ptr() == job.mid_tables[k].data_ptr()      # call B's replace step
                ms = sched.call_at(s_next, st.sigma_next)
                assert (corr.sigma, corr.sigma_next, corr.dt) == (np.float32(sigma), np.float32(s_next), np.float32(dt))
                assert job.mid_active[k] == ms.n_inner and torch.equal(job.mid_sigma[k], ms.sigma_t)
                assert torch.equal(job.mid_t_model[k], ms.times[0])
                if i + 1 < n_steps:     # call B's row is the next outer step's
                    assert torch.equal(job.mid_tables[k], job.tables[i + 1])
                    assert torch.equal(job.mid_sigma[k], job.sigma[i + 1])
                    assert torch.equal(job.mid_t_model[k], job.t_model[i + 1])
                    assert job.mid_active[k] == job.active[i + 1]
                xb, ab, kwb = seen[1]
                assert xb is job.x2 and ab[8] is None and kwb.get("midpoint") is None and kwb["skip_prologue"]
                step, x_base, out_prev = kwb["heun"]
                assert step is corr and x_base is job.x and out_prev is out and out is not None
                assert (kwb["next_table"] is None) == (after is None)
                if after is not None:     # the next outer step's replace step
                    assert kwb["next_table"].data_ptr() == after.data_ptr()
                assert plan.used == draws[-1] + per_call(job.active[i])
                own, subs = per_call(ms.n_inner), subs + ms.n_inner
            draws.append(draws[-1] + per_call(job.active[i]) + own)
        assert job.draws_before == draws and job.substeps == subs and job.x2 is not None
        assert (name == "window-leftover") == (job.midpoint[-1][1] is not None)
        assert euler.midpoint is None and euler.x2 is None


def test_graphed_job_takes_heun_only_with_its_sampler_function():
    """GraphedJob(sampler="heun") restates one sampler function: it wants the sample_heun it stands in for, and refuses
    none or another one."""
    sig = _schedules()["karras-20"]
    job, _ = _job(sig, 3, "heun", sampler_fn=minicomfy.sample_heun)
    assert job.sampler == "heun" and job.x2 is not None
    for fn in (None, minicomfy.sample_dpm_2, minicomfy.sample_euler):
        with pytest.raises(ValueError):
            _job(sig, 3, "heun", sampler_fn=fn)


def _restating_heun_that_draws(model, x, sigmas, extra_args=None, callback=None, disable=None, s_churn=0.0,
                               s_noise=1.0):
    """k-diffusion's original sample_heun: eps = randn_like(x) every step, added only with churn."""
    extra_args = extra_args or {}
    s_in = x.new_ones([x.shape[0]])
    for i in range(len(sigmas) - 1):
        gamma = min(s_churn / (len(sigmas) - 1), 2 ** 0.5 - 1)
        eps = torch.randn_like(x) * s_noise
        sigma_hat = sigmas[i] * (gamma + 1)
        if gamma > 0:
            x = x + eps * (sigma_hat ** 2 - sigmas[i] ** 2) ** 0.5
        denoised = model(x, sigma_hat * s_in, **extra_args)
        d = (x - denoised) / sigma_hat
        dt = sigmas[i + 1] - sigma_hat
        if sigmas[i + 1] == 0:
            x = x + d * dt
        else:
            x_2 = x + d * dt
            denoised_2 = model(x_2, sigmas[i + 1] * s_in, **extra_args)
            d_2 = (x_2 - denoised_2) / sigmas[i + 1]
            x = x + (d + d_2) / 2 * dt
    return x


_restating_heun_that_draws.__name__ = "sample_heun"


def test_gate_and_form_check():
    """The gate takes sample_heun without extra options and with a mask; the form check turns away a heun that draws
    from the global generator, leaves that generator where it was, and caches its verdict per function."""
    minicomfy.install()
    from lanpaint_b200 import comfy_nodes as N
    from lanpaint_b200.engine import LanPaint

    class K:
        audio_indicator = None
        sigmas_host = [3.0, 1.0, 0.0]
    ks = minicomfy.ksampler("heun")
    eng = LanPaint(None, NSteps=3, Friction=15.0, Lambda=5.0, Beta=1.0, StepSize=0.2, rng="torch")
    dm = torch.ones(1)
    ok = lambda s=ks, mo={}, m=dm: N.KSAMPLER._fused_heun_ok(s, K, m, mo, eng)   # noqa: E731
    assert ok()
    assert not ok(s=minicomfy.ksampler("heun", {"s_churn": 1.0}))
    assert not ok(mo={"denoise_mask_function": lambda *a, **k: None})
    assert not ok(m=None)
    assert not ok(s=minicomfy.ksampler("euler")) and not ok(s=minicomfy.ksampler("dpm_2"))
    torch.manual_seed(123)
    before = torch.default_generator.get_state()
    assert not ok(s=minicomfy.KSAMPLER(_restating_heun_that_draws))
    assert torch.equal(torch.default_generator.get_state(), before)
    assert N._FORM_OK[(_restating_heun_that_draws, "heun")] is False
    assert N._FORM_OK[(minicomfy.sample_heun, "heun")] is True
    assert not ok(s=minicomfy.KSAMPLER(_restating_heun_that_draws))     # the cached verdict
    assert torch.equal(torch.default_generator.get_state(), before)
