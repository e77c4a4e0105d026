"""GPU: inner-loop early stop (row a13) against traces and outputs recorded from the REFERENCE's
LanPaintEarlyStopper driven through its own LanPaint.__call__ (tests/golden/make_golden.py --earlystop)."""
import glob
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR, load_golden
from _support import make_model, max_rel

pytestmark = pytest.mark.gpu

ES_ALL = sorted(os.path.splitext(os.path.basename(p))[0] for p in glob.glob(os.path.join(GOLDEN_DIR, "aux_es_*.npz")))
ES_CASES = [n for n in ES_ALL if not n.startswith("aux_es_av_")]
ES_AV_CASES = [n for n in ES_ALL if n.startswith("aux_es_av_")]


def _custom_distance(prev, cur, ctx):
    return ((cur - prev) ** 2).mean()


def _close(a, b, rel=2e-4):
    if a is None or b is None:
        return a is None and b is None
    return abs(a - b) <= rel * max(abs(a), abs(b), 1e-12)


@pytest.mark.parametrize("name", ES_CASES)
def test_early_stop_matches_reference_trace(name, cuda_device):
    from lanpaint_b200.engine import LanPaint, NoiseTape
    assert len(ES_CASES) >= 6
    g = load_golden(name)
    meta = g["meta"]
    dev = cuda_device
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    x, y, noise, mask = t(g["x"]), t(g["y"]), t(g["noise"]), t(g["mask_full"])
    sigma = t(g["sigma"])
    times = (t(g["ve"]), t(g["abt"]), t(g["flow_t"]))
    tape = NoiseTape([t(d) for d in g["tape"]])
    model = make_model("two_heads", False)
    eng = LanPaint(model, NSteps=meta["n_steps"], Friction=15.0, Lambda=5.0, Beta=1.0, StepSize=0.2, MinStepFrac=1.0,
                   EarlyStopThreshold=meta["ctor_threshold"], EarlyStopPatience=meta["ctor_patience"], rng=tape)
    trace = []
    mo = {"lanpaint_semantic_trace": trace, "bench_case_id": name, "bench_outer_step": 3, "bench_timestep": 0.5}
    if meta["stop"] is not None:
        stop = dict(meta["stop"])
        if stop.get("distance_fn") == "mean_sq_xt":
            stop["distance_fn"] = _custom_distance
        mo["lanpaint_semantic_stop"] = stop
    out = eng(x, y, noise, sigma, mask, times, mo, 0, n_steps=meta["n_steps"])
    want = meta["trace"]
    assert len(trace) == len(want), (len(trace), len(want))          # stopped after the same sub-step
    assert model.calls == meta["model_calls"] and tape.pos == meta["n_draws"]
    for got, ref in zip(trace, want):
        for k in ("inner_step", "patience_counter", "patience_eff", "custom_dist", "stopped", "case_id", "outer_step"):
            assert got[k] == ref[k], (k, got, ref)
        for k in ("dist", "dist_inpaint", "dist_ring", "dist_drift", "threshold", "threshold_eff", "abt"):
            assert _close(got[k], ref[k]), (k, got[k], ref[k])
    assert max_rel(out, torch.from_numpy(g["out"])) <= 2e-5
    assert max_rel(x, torch.from_numpy(g["x_new"])) <= 2e-5


@pytest.mark.parametrize("name", ES_AV_CASES)
def test_early_stop_on_av_pack_matches_reference_trace(name, cuda_device):
    """The stopper on an AV flat pack (audio suffix on its own schedule, with and without the target correction):
    the reference stops midway, and the engine must stop after the same sub-step with the same distances, draws
    and outputs."""
    from lanpaint_b200.engine import LanPaint, NoiseTape
    assert len(ES_AV_CASES) >= 2
    g = load_golden(name)
    meta = g["meta"]
    dev = cuda_device
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    x, y, noise, mask = t(g["x"]), t(g["y"]), t(g["noise"]), t(g["mask_full"])
    sigma = t(g["sigma"])
    times = (t(g["ve"]), t(g["abt"]), t(g["flow_t"]))
    times_a = (t(g["ve_a"]), t(g["abt_a"]), t(g["flow_a"]))
    ai = torch.zeros((1, 1, x.shape[-1]), device=dev)
    ai[..., meta["video_n"]:] = 1.0
    corr = None if meta["corr"] is None else (1.0 - ai) + meta["corr"] * ai
    tape = NoiseTape([t(d) for d in g["tape"]])
    model = make_model("two_heads", True)
    eng = LanPaint(model, NSteps=meta["n_steps"], Friction=15.0, Lambda=5.0, Beta=1.0, StepSize=0.2, IS_FLOW=True,
                   MinStepFrac=1.0, rng=tape)
    trace = []
    mo = {"lanpaint_semantic_trace": trace, "bench_case_id": name, "bench_outer_step": 3, "bench_timestep": 0.5,
          "lanpaint_semantic_stop": dict(meta["stop"])}
    out = eng(x, y, noise, sigma, mask, times, mo, 0, n_steps=meta["n_steps"], current_times_audio=times_a,
              audio_indicator=ai, audio_correction=corr)
    want = meta["trace"]
    assert 1 < len(want) < meta["n_steps"]
    assert len(trace) == len(want), (len(trace), len(want))
    assert model.calls == meta["model_calls"] and tape.pos == meta["n_draws"]
    for got, ref in zip(trace, want):
        for k in ("inner_step", "patience_counter", "patience_eff", "custom_dist", "stopped", "case_id", "outer_step"):
            assert got[k] == ref[k], (k, got, ref)
        for k in ("dist", "dist_inpaint", "dist_ring", "dist_drift", "threshold", "threshold_eff", "abt"):
            assert _close(got[k], ref[k]), (k, got[k], ref[k])
    assert max_rel(out, torch.from_numpy(g["out"])) <= 2e-5
    assert max_rel(x, torch.from_numpy(g["x_new"])) <= 2e-5


def test_torch_stream_early_stop_equals_its_tape(cuda_device):
    """The early-stop loop under the default torch stream (lp_advance_f32 -> advance_torch_kernel, lp_substep with
    the x0e side output) against the same loop fed a NoiseTape of the torch.randn draws the reference makes from the
    same seed, in its order (1 draw for sub-step 0, then 2 per sub-step).  The tape path is pinned to the
    reference's own stopper by test_early_stop_matches_reference_trace; the stop (min_steps 4 with a threshold
    every distance passes) fires mid-loop whatever the noise.  Same draws, same per-element arithmetic: the stop
    trace, the outputs and the generator's final offset must be identical."""
    from lanpaint_b200.engine import LanPaint, NoiseTape
    g = load_golden("aux_es_min_steps_legacy")
    meta = g["meta"]
    dev = cuda_device
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    y, noise, mask, sigma = t(g["y"]), t(g["noise"]), t(g["mask_full"]), t(g["sigma"])
    times = (t(g["ve"]), t(g["abt"]), t(g["flow_t"]))
    gen = torch.cuda.default_generators[dev.index or 0]
    n = meta["n_steps"]

    def run(rng):
        model = make_model("two_heads", False)
        eng = LanPaint(model, NSteps=n, Friction=15.0, Lambda=5.0, Beta=1.0, StepSize=0.2, MinStepFrac=1.0,
                       EarlyStopThreshold=meta["ctor_threshold"], EarlyStopPatience=meta["ctor_patience"], rng=rng)
        trace = []
        mo = {"lanpaint_semantic_trace": trace, "lanpaint_semantic_stop": dict(meta["stop"])}
        x = t(g["x"])
        out = eng(x, y, noise, sigma, mask, times, mo, 0, n_steps=n)
        return out, x, trace, model.calls

    torch.manual_seed(1234)
    off0 = gen.get_offset()
    draws = [torch.randn_like(y) for _ in range(2 * n - 1)]     # every draw the reference could make, in its order
    inc = (gen.get_offset() - off0) // (2 * n - 1)
    tape = NoiseTape(draws)
    want = run(tape)
    assert 0 < tape.pos < 2 * n - 1, tape.pos                     # stopped mid-loop
    torch.manual_seed(1234)
    got = run("torch")
    assert len(got[2]) == len(want[2]) and got[3] == want[3]
    for a, b in zip(got[2], want[2]):
        for k in ("inner_step", "patience_counter", "patience_eff", "stopped", "dist", "dist_inpaint", "dist_ring",
                  "dist_drift", "threshold", "threshold_eff", "abt"):
            assert a[k] == b[k], (k, a, b)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    assert gen.get_offset() == off0 + tape.pos * inc             # advanced by exactly the draws consumed


def test_stats_kernel_matches_torch(cuda_device):
    import ctypes as C
    from lanpaint_b200 import _native
    from lanpaint_b200.earlystop import boundary_ring
    lib = _native.load()
    dev = cuda_device
    for shape, bcast in (((3, 4, 32, 32), True), ((2, 4, 17, 13), False), ((1, 16, 21, 80, 45), True)):
        a, b = torch.randn(shape, device=dev), torch.randn(shape, device=dev)
        mshape = (shape[0], 1 if bcast else shape[1]) + shape[2:]
        m8 = (torch.rand(mshape, device=dev) < 0.5).to(torch.uint8)
        ring = boundary_ring(m8)
        S = int(np.prod(shape[2:]))
        dims = _native.Dims(shape[0], shape[1] * S, S, S if bcast else shape[1] * S, 0 if bcast else S)
        sums = torch.zeros(2, dtype=torch.float64, device=dev)
        rc = lib.lp_stop_stats_f32(C.c_void_p(a.data_ptr()), C.c_void_p(b.data_ptr()), C.c_void_p(m8.data_ptr()),
                                   C.c_void_p(ring.data_ptr()) if ring is not None else None, None, C.byref(dims),
                                   C.c_void_p(sums.data_ptr()), C.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert rc == 0
        d2 = (a.double() - b.double()) ** 2
        w_in = (m8 == 0).expand(shape).double()
        assert abs(sums[0].item() / (d2 * w_in).sum().item() - 1) < 1e-5
        if ring is not None:
            assert abs(sums[1].item() / (d2 * ring.expand(shape).double()).sum().item() - 1) < 1e-5
        else:
            assert sums[1].item() == 0.0


def test_early_stop_disabled_without_an_inpaint_region(cuda_device):
    """reference tests/test_lanpaint_semantic_stop.py:68-104: with nothing to inpaint the stopper is never
    built and all n sub-steps run; with a region and an easy threshold it stops after patience + 1 checks."""
    from lanpaint_b200.engine import LanPaint
    dev = cuda_device
    x = torch.zeros(1, 4, 8, 8, device=dev)
    y, noise = torch.zeros_like(x), torch.ones_like(x)
    sig = torch.tensor([1.0], device=dev)
    times = (sig, torch.tensor([0.5], device=dev), torch.tensor([0.0], device=dev))
    for mask, patience, want_calls in ((torch.ones_like(x), 1, 10 + 1), (torch.zeros_like(x), 2, 3 + 1)):
        model = make_model("identity", False)
        eng = LanPaint(model, NSteps=10, Friction=15.0, Lambda=1.0, Beta=1.0, StepSize=0.2, rng="philox")
        mo = {"lanpaint_semantic_stop": {"threshold": 1e6, "patience": patience}}
        eng(x.clone(), y, noise, sig, mask, times, mo, 0, n_steps=10)
        assert model.calls == want_calls, (model.calls, want_calls)
