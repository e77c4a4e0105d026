"""Host side of what a deferred fused job keeps of each outer step's denoised latent (GraphedJob.run's observe
setting, "full" / "preview" / "final"): the launches of every fused sampler on every kind of schedule, recorded with
the engine's launch stubbed out, and the argument rules of the row-bounded boundary entry points
(lp_boundary_*_rows), checked before any CUDA call.  No device calls here."""
import ctypes as C
import os
import re

import pytest
import torch

import _job_ref as J
import minicomfy
from conftest import ROOT
from lanpaint_b200 import _native
from oracle import langevin_oracle as O

B = 3
SHAPE = (B, 4, 8, 8)
SAMPLERS = ("euler", "euler_ancestral", "dpmpp_2m", "dpm_2", "deis", "res_multistep", "gradient_estimation", "heun")
SAMPLER_FN = {"deis": minicomfy.sample_deis, "heun": minicomfy.sample_heun}
SETTINGS = ("full", "preview", "final")


def _sigmas(sampler, name):
    eps = minicomfy.ModelPatcher(minicomfy.BaseModel(None), "cpu")
    return {"karras-20": lambda: J.ksampler_sigmas(eps, 20, sampler, "karras"),
            "window-leftover": lambda: J.ksampler_sigmas(eps, 20, sampler, "karras", start_step=3, last_step=15),
            "one-step": lambda: J.ksampler_sigmas(eps, 1, sampler, "karras")}[name]()


def _job(sampler, sigmas):
    from lanpaint_b200.engine import LanPaint
    from lanpaint_b200.runner import GraphedJob, HostSchedule, VESampling
    eng = LanPaint(O.PointwiseDenoiser(VESampling()), NSteps=4, Friction=15.0, Lambda=5.0, Beta=1.0, StepSize=0.2,
                   MinStepFrac=1.0, rng="torch", batched_replace="per_sample")
    sched = HostSchedule([float(v) for v in sigmas], B, 4, early_stop=2)
    job = GraphedJob(eng, sched, SHAPE, "cpu", sampler=sampler, sampler_fn=SAMPLER_FN.get(sampler))
    job._dims, job.mask = None, None
    return job


class _Plan:
    used = 0


def _tensors(v):
    """Every tensor inside a launch argument (tuples flattened)."""
    if isinstance(v, torch.Tensor):
        return [v]
    if isinstance(v, (tuple, list)):
        return [t for e in v for t in _tensors(e)]
    return []


def _launches(job, observe):
    """-> [(outer step, out, out_rows, args, kwargs, draws used)] of one mode "job" body with a callback."""
    job.outs = job._observed(observe)
    seen, step = [], [0]

    def stub(xm, *a, **kw):
        seen.append((step[0], a[8], kw.get("out_rows"), (xm,) + a, kw, a[10].used))
    job.engine._launch_sequence = stub
    for i in range(len(job.sched.steps)):
        step[0] = i
        job._step(i, _Plan(), "each")
    return seen


def _canon(v, outs):
    """A launch argument in a form comparable across observe settings: a denoised-latent buffer by its outer step,
    any other tensor by its storage and view, a tuple element by element."""
    if isinstance(v, torch.Tensor):
        for j, o in enumerate(outs):
            if o is v:
                return ("outs", j)
        return ("tensor", v.data_ptr(), tuple(v.shape), tuple(v.stride()))
    if isinstance(v, (tuple, list)):
        return tuple(_canon(e, outs) for e in v)
    if isinstance(v, dict):
        return {k: _canon(e, outs) for k, e in v.items()}
    if isinstance(v, C.Structure):
        return (type(v).__name__, bytes(v))
    if isinstance(v, _Plan):       # a fresh one per step: its draws are compared apart
        return "plan"
    return v


@pytest.mark.parametrize("schedule", ["karras-20", "window-leftover", "one-step"])
@pytest.mark.parametrize("sampler", SAMPLERS)
def test_every_buffer_a_later_launch_reads_is_stored_whole(sampler, schedule):
    """Under each setting, every denoised-latent buffer a launch reads (dpmpp_2m's and res_multistep's previous
    latent, heun's out_prev) was written whole (B rows, out_rows None) by an earlier launch, and no [1, ...] preview
    buffer feeds any launch.  The last step stores a whole latent.  "final" passes out=None exactly where the step's
    latent is neither read later nor the last (where `_out_whole` is false), "preview" a [1, ...] buffer with
    out_rows = 1 there.  The launches, their draws and tables are the same under the three settings apart from
    out / out_rows."""
    job = _job(sampler, _sigmas(sampler, schedule))
    n = len(job.sched.steps)
    runs = {}
    for observe in SETTINGS:
        runs[observe] = seen = _launches(job, observe)
        outs = job.outs
        assert len(outs) == n and outs[-1] is not None and outs[-1].shape == SHAPE, observe
        written = {}
        for k, (i, out, rows, args, kw, _) in enumerate(seen):
            reads = [t for v in list(args[:9]) + list(args[10:]) + list(kw.values()) for t in _tensors(v)]
            for t in reads:
                src = [j for j, o in enumerate(outs) if o is t]
                if not src:
                    continue
                assert t.shape == SHAPE, (observe, i, src, tuple(t.shape))
                assert id(t) in written and written[id(t)] is None, (observe, i, src, "read before a whole store")
            if out is not None:
                assert any(o is out for o in outs), (observe, i)
                assert rows == (1 if out.shape[0] == 1 else None), (observe, i, rows, tuple(out.shape))
                assert out.shape[0] in (1, B)
                written[id(out)] = rows
            else:
                assert rows is None
        last = [out for i, out, *_ in seen if i == n - 1 and out is not None]
        assert last and last[0] is outs[-1], observe

    # which steps' latents a later launch reads (heun's corrector: the same step's), from the "full" run alone
    outs_full, read_later = job._observed("full"), set()
    for k, (i, out, rows, args, kw, _) in enumerate(runs["full"]):
        for t in [t for v in list(args[:9]) + list(args[10:]) + list(kw.values()) for t in _tensors(v)]:
            read_later |= {j for j, o in enumerate(outs_full) if o is t}
    if sampler in ("dpmpp_2m", "heun") and n > 1:
        assert read_later, "the rule's subject: a step whose latent a later launch reads"
    first = {}
    for observe in SETTINGS:
        first[observe] = {}
        for i, out, rows, *_ in runs[observe]:
            first[observe].setdefault(i, (out, rows))
    for i in range(n):
        whole = i + 1 == n or job._out_whole(i)
        assert i not in read_later or whole, (i, "a later launch reads a latent _out_whole lets go")
        out, rows = first["full"][i]
        assert out is not None and out.shape == SHAPE and rows is None, i
        out, rows = first["final"][i]
        assert (out is None) == (not whole), (i, whole)
        out, rows = first["preview"][i]
        if whole:
            assert out.shape == SHAPE and rows is None, i
        else:
            assert out.shape == (1,) + SHAPE[1:] and rows == 1, i
    # the same launches, draws and tables apart from out / out_rows
    for observe in ("preview", "final"):
        a_runs, b_runs = runs["full"], runs[observe]
        assert len(a_runs) == len(b_runs), observe
        outs_a, outs_b = job._observed("full"), job._observed(observe)
        for (ia, _, _, aa, ka, ua), (ib, _, _, ab, kb, ub) in zip(a_runs, b_runs):
            assert ia == ib and ua == ub, observe
            assert _canon(aa[:9] + aa[10:], outs_a) == _canon(ab[:9] + ab[10:], outs_b), (observe, ia)
            drop = lambda kw: {k: v for k, v in kw.items() if k != "out_rows"}   # noqa: E731
            assert _canon(drop(ka), outs_a) == _canon(drop(kb), outs_b), (observe, ia)


@pytest.mark.parametrize("sampler", ["dpmpp_2m", "res_multistep", "heun"])
def test_the_rule_names_the_read_buffers(sampler):
    """The buffers a later launch reads, named step by step: every dpmpp_2m step but the last (its next step is
    second order), the res_multistep steps before a second-order step (its Euler steps included), and every heun step
    with a corrector (its predictor's latent is the corrector's out_prev)."""
    job = _job(sampler, _sigmas(sampler, "karras-20"))
    n = len(job.sched.steps)
    if sampler == "heun":
        want = [job.midpoint[i][2] is not None for i in range(n)]
        assert want[:-1] == [True] * (n - 1) and not want[-1]
    else:
        want = [i + 1 < n and bool(job.multistep[i + 1][1]) for i in range(n)]
        if sampler == "res_multistep":
            assert isinstance(job.multistep[0][0], _native.Midpoint) and want[0]   # the first, Euler, step is read
    for i in range(n):
        if want[i]:
            assert job._out_whole(i), i


# ---- the row-bounded entry points' argument rules -------------------------------------------------------------
P = C.c_void_p
INVALID = 1
ROWS = ("lp_boundary_known", "lp_boundary_ancestral", "lp_boundary_midpoint", "lp_boundary_deis",
        "lp_boundary_gradient_estimation")
_CTYPE = {"float": C.c_float, "int64_t": C.c_int64}
_STRUCT = {"lp_heads": _native.Heads, "lp_known": _native.Known, "lp_ancestral": _native.Ancestral,
           "lp_rng": _native.Rng, "lp_midpoint": _native.Midpoint, "lp_deis": _native.Deis,
           "lp_gradient_estimation": _native.GradientEstimation, "lp_dims": _native.Dims}


def _declared_params(name):
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "lanpaint_b200.h")).read(), flags=re.S)
    m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", src)
    assert m, name
    params = []
    for decl in m.group(1).split(","):
        words = decl.replace("*", " * ").split()
        names = [w for w in words if w not in ("const", "*")]
        params.append((names[0], "*" in words, names[-1]))
    return params


@pytest.mark.parametrize("name", ROWS)
def test_rows_entry_points_are_bound_with_the_headers_argtypes(name):
    """Each lp_boundary_*_rows is its unbounded entry point's parameter list with `int64_t out_rows` right after
    `out`, and _native binds it with ctypes types that match the header's parameter by parameter."""
    lib = _native.load()
    params, base = _declared_params(name + "_rows"), _declared_params(name)
    at = [p for p, (_, _, pname) in enumerate(params) if pname == "out_rows"]
    assert len(at) == 1 and params[at[0] - 1][2] == "out" and params[at[0]][:2] == ("int64_t", False)
    assert params[:at[0]] + params[at[0] + 1:] == base
    fn = getattr(lib, name + "_rows")
    assert name + "_rows" in _native.SYMBOLS and fn.restype is C.c_int
    assert len(fn.argtypes) == len(params)
    for got, (ctype, ptr, pname) in zip(fn.argtypes, params):
        if ptr and ctype in _STRUCT:
            want = C.POINTER(_STRUCT[ctype])
        elif ptr or ctype == "lp_stream_t":
            want = C.c_void_p
        else:
            want = _CTYPE[ctype]
        assert got is want, (name, pname, got, want)


# fake device addresses, never dereferenced: every call below fails validation first
FAKE = 0x1000
X, X2, OUT, D0, D1, D2 = 0x200000, 0x300000, 0x400000, 0x500000, 0x600000, 0x700000
N_ROWS, PER_ROW = 4, 64       # 256 bytes per row
ROW = 4 * PER_ROW


def _call(name, out, out_rows, **states):
    """One lp_boundary_*_rows call on fake operands; `states` overrides the state buffers' addresses."""
    lib = _native.load()
    s = dict(x=X, x2=X2, d_out=D0, p1=D1, p2=D2)
    s.update(states)
    heads = _native.Heads(FAKE, None, _native.DTYPE_F32, 0, 0.0, 0.0)
    known = _native.Known(FAKE, FAKE, FAKE)
    dims = _native.Dims(N_ROWS, PER_ROW, 16, 16, 0, 0)
    common = (C.byref(heads), P(FAKE), P(FAKE), P(FAKE), C.byref(known))
    tail = (P(FAKE), C.byref(dims), None)
    rows = C.c_int64(out_rows)
    if name == "lp_boundary_known":
        return lib.lp_boundary_known_rows(*common, P(s["x"]), P(out), rows, C.c_float(-0.25), *tail)
    if name == "lp_boundary_ancestral":
        return lib.lp_boundary_ancestral_rows(*common, P(s["x"]), P(out), rows,
                                              C.byref(_native.Ancestral(2.0, -0.5, 1.0, 0.0)), None, *tail)
    if name == "lp_boundary_midpoint":       # the predictor: x -> x2
        return lib.lp_boundary_midpoint_rows(*common, P(s["x"]), P(s["x"]), P(s["x2"]), P(out), rows,
                                             C.byref(_native.Midpoint(2.0, -0.5)), *tail)
    if name == "lp_boundary_deis":
        return lib.lp_boundary_deis_rows(*common, P(s["x"]), P(out), rows, P(s["d_out"]), P(s["p1"]), P(s["p2"]),
                                         C.byref(_native.Deis(2.0, -0.5, 0.25, -0.125)), *tail)
    return lib.lp_boundary_gradient_estimation_rows(*common, P(s["x"]), P(out), rows, P(s["d_out"]), P(s["p1"]),
                                                    C.byref(_native.GradientEstimation(2.0, -0.5, 1.0, 0)), *tail)


# the state buffers `out` may share no byte with (lp_boundary_known and lp_boundary_ancestral let out alias x, and so
# does lp_boundary_deis)
STATES = {"lp_boundary_known": (), "lp_boundary_ancestral": (), "lp_boundary_midpoint": ("x", "x2"),
          "lp_boundary_deis": ("d_out", "p1", "p2"), "lp_boundary_gradient_estimation": ("x", "d_out", "p1")}


@pytest.mark.parametrize("name", ROWS)
def test_rows_arguments_are_refused_before_any_launch(name):
    """out_rows < 0 is LP_ERR_INVALID, and so is an `out` that shares a byte with a state buffer inside its first
    min(out_rows, n_rows) rows: one ending a float into the state, one starting at the state's last float."""
    assert _call(name, OUT, -1) == INVALID and _call(name, OUT, -(1 << 40)) == INVALID
    assert _call(name, None, -1) == INVALID
    for state in STATES[name]:
        base = dict(x=X, x2=X2, d_out=D0, p1=D1, p2=D2)[state]
        for out_rows in (1, 2, N_ROWS - 1, N_ROWS, N_ROWS + 3, 1 << 40):
            held = min(out_rows, N_ROWS) * ROW       # bytes of out the launch may write
            assert _call(name, base - held + 4, out_rows) == INVALID, (state, out_rows, "end")
            assert _call(name, base + N_ROWS * ROW - 4, out_rows) == INVALID, (state, out_rows, "start")
            assert _call(name, base, out_rows) == INVALID, (state, out_rows, "same")
