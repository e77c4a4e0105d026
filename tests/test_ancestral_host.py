"""Host side of the fused euler_ancestral loop: the step coefficients, the draw accounting of
`runner.GraphedJob(sampler="euler_ancestral")`, and what `lp_boundary_ancestral` rejects before any CUDA call."""
import ctypes as C
import os
import re
from unittest import mock

import pytest
import torch

import _job_ref as J
import minicomfy
from lanpaint_b200 import _native
from lanpaint_b200.schedule import ancestral_step

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _schedules():
    patcher = minicomfy.ModelPatcher(minicomfy.BaseModel(None), "cpu")
    return {"karras-20": J.ksampler_sigmas(patcher, 20, "euler_ancestral", "karras"),
            "simple-20": J.ksampler_sigmas(patcher, 20, "euler_ancestral", "simple"),
            "window-leftover": J.ksampler_sigmas(patcher, 20, "euler_ancestral", "karras", start_step=3, last_step=15)}


@pytest.mark.parametrize("eta", [0.0, 0.5, 1.0])
@pytest.mark.parametrize("name", ["karras-20", "simple-20", "window-leftover"])
def test_ancestral_step_is_the_samplers_expression(name, eta):
    """minicomfy.sample_euler_ancestral in fp64 (so that its Python-double factors are applied unrounded) equals,
    bit for bit, the same loop written with ancestral_step -- and takes its draws at the same steps."""
    sig = _schedules()[name]
    if name == "window-leftover":
        assert float(sig[-1]) > 0
    g = torch.Generator().manual_seed(5)
    x0 = torch.randn(2, 3, dtype=torch.float64, generator=g)
    tape = [torch.randn(2, 3, dtype=torch.float64, generator=g) for _ in range(len(sig))]
    drawn = []

    def randn_like(like, **kw):
        drawn.append(len(drawn))
        return tape[len(drawn) - 1]

    model = lambda x, s, **kw: 0.3 * x + 0.1      # noqa: E731
    with mock.patch.object(torch, "randn_like", randn_like):
        want = minicomfy.sample_euler_ancestral(model, x0.clone(), sig.double(), eta=eta, s_noise=0.9)
    x, k = x0.clone(), 0
    for i in range(len(sig) - 1):
        s_from, s_to = float(sig[i]), float(sig[i + 1])
        s_down, s_up = ancestral_step(s_from, s_to, eta)
        # the sampler's expression, restated
        up = min(s_to, eta * (s_to ** 2 * (s_from ** 2 - s_to ** 2) / s_from ** 2) ** 0.5) if s_to > 0 else 0.0
        assert (s_down, s_up) == ((s_to ** 2 - up ** 2) ** 0.5, up)
        x = x + (x - model(x, None)) / s_from * (s_down - s_from)
        if s_to > 0:
            x = x + tape[k] * 0.9 * s_up
            k += 1
    assert k == len(drawn) == sum(1 for v in sig[1:] if float(v) > 0)
    assert torch.equal(x, want)
    if eta == 0.0:
        assert all(ancestral_step(float(a), float(b), 0.0) == (float(b), 0.0) for a, b in zip(sig[:-1], sig[1:]))


def _job(sigmas, n_inner, sampler, rng="torch", merge=None, **kw):
    from lanpaint_b200.engine import LanPaint
    from lanpaint_b200.runner import GraphedJob, HostSchedule, VESampling
    from oracle import langevin_oracle as O
    eng = LanPaint(O.PointwiseDenoiser(VESampling()), NSteps=n_inner, Friction=15.0, Lambda=5.0, Beta=1.0, StepSize=0.2,
                   MinStepFrac=1.0, rng=rng, batched_replace="per_sample")
    if merge is not None:
        eng.merge_noise = merge
    sched = HostSchedule([float(v) for v in sigmas], 2, n_inner)
    return GraphedJob(eng, sched, (2, 4, 8, 8), "cpu", sampler=sampler, **kw), sched


@pytest.mark.parametrize("eta", [0.0, 1.0])
def test_draws_before_counts_the_samplers_draw_after_each_steps_langevin_draws(eta):
    """One extra draw per outer step with sigma_next > 0, whatever eta is; none at the last step to 0; a window that
    ends above 0 draws at its last step too."""
    sch = _schedules()
    for name in ("karras-20", "window-leftover"):
        sig = sch[name]
        euler, sched = _job(sig, 5, "euler")
        anc, _ = _job(sig, 5, "euler_ancestral", eta=eta, s_noise=0.8)
        own = [1 if st.sigma_next > 0 else 0 for st in sched.steps]
        assert sum(own) == (len(own) if name == "window-leftover" else len(own) - 1)
        for i in range(len(own)):
            lang = euler.draws_before[i + 1] - euler.draws_before[i]
            assert lang == (2 * sched.steps[i].n_inner - 1 if euler.active[i] > 0 else 0)
            assert anc.draws_before[i + 1] - anc.draws_before[i] == lang + own[i]
            step, draws = anc.ancestral[i]
            assert draws == bool(own[i])
            s_down, s_up = ancestral_step(sched.steps[i].sigma, sched.steps[i].sigma_next, eta)
            assert step.sigma == sched.steps[i].sigma
            assert step.down == C.c_float(s_down - sched.steps[i].sigma).value     # the difference in double, one rounding
            assert step.s_noise == C.c_float(0.8).value and step.sigma_up == C.c_float(s_up).value
            if eta == 0.0:
                assert step.sigma_up == 0.0
        assert anc.draws == euler.draws + sum(own)
    with pytest.raises(ValueError):
        _job(sch["karras-20"], 5, "heun")


def test_merged_philox_draws_still_get_the_samplers_draw():
    sig = _schedules()["karras-20"]
    euler, sched = _job(sig, 5, "euler", rng="philox", merge=True)
    anc, _ = _job(sig, 5, "euler_ancestral", rng="philox", merge=True)
    assert anc.draws == euler.draws + len(sched.steps) - 1


def test_entry_point_is_declared_and_bound():
    header = open(os.path.join(ROOT, "include", "lanpaint_b200.h")).read()
    assert re.search(r"\bint lp_boundary_ancestral\(", header) and "typedef struct lp_ancestral" in header
    assert "#define LP_ABI_VERSION 5" in header
    assert "lp_boundary_ancestral" in _native.SYMBOLS
    lib = _native.load()
    assert lib.lp_boundary_ancestral.restype is C.c_int and len(lib.lp_boundary_ancestral.argtypes) == 12
    assert C.sizeof(_native.Ancestral) == 16


def test_invalid_arguments_are_refused_before_any_launch():
    lib = _native.load()
    P = C.c_void_p
    fake = 0x1000    # never dereferenced: validation fails first
    dims = _native.Dims(2, 64, 16, 16, 0, 0)
    heads = _native.Heads(fake, None, _native.DTYPE_F32, 0, 0.0, 0.0)
    known = _native.Known(fake, fake, fake)
    step = _native.Ancestral(2.0, -0.5, 1.0, 0.3)
    rng = _native.Rng(mode=_native.RNG_TORCH)

    def call(heads=heads, y=fake, noise=fake, mask=fake, known=known, x=fake, out=fake, step=step, rng=rng,
             table=fake, dims=dims):
        ref = lambda o: None if o is None else C.byref(o)   # noqa: E731
        return lib.lp_boundary_ancestral(ref(heads), P(y), P(noise), P(mask), ref(known), P(x), P(out), ref(step),
                                         ref(rng), P(table), ref(dims), None)

    INVALID = 1
    assert call(step=None) == INVALID
    assert call(step=_native.Ancestral(0.0, -0.5, 1.0, 0.3)) == INVALID          # sigma_from must be > 0
    assert call(step=_native.Ancestral(-1.0, -0.5, 1.0, 0.3)) == INVALID
    assert call(step=_native.Ancestral(float("nan"), -0.5, 1.0, 0.3)) == INVALID
    assert call(rng=None) == INVALID                                              # sigma_up != 0 needs the draw
    assert call(rng=_native.Rng(mode=_native.RNG_TAPE)) == INVALID                # a tape stream without its tape
    assert call(rng=_native.Rng(mode=7)) == INVALID
    assert call(x=None) == INVALID                                                # the state is always updated
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
    assert call(dims=_native.Dims(2, 100, 30, 100, 0, 0)) == INVALID
    assert call(dims=_native.Dims(1 << 20, 4096, 1024, 4096, 1024, 0)) == 4       # LP_ERR_UNSUPPORTED
    # well-formed calls on an empty batch succeed without a launch: with a draw, without one, eta == 0 with a draw
    empty = _native.Dims(0, 64, 16, 16, 0, 0)
    assert call(dims=empty) == 0
    assert call(dims=empty, rng=None, step=_native.Ancestral(2.0, -2.0, 1.0, 0.0), table=None, noise=None,
                known=None) == 0
    assert call(dims=empty, step=_native.Ancestral(2.0, -0.5, 1.0, 0.0)) == 0
