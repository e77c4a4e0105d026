"""GPU: the fused res_multistep loop -- its second-order step on lp_boundary_multistep and its Euler steps on
lp_boundary_midpoint, per launch against fp64, bit for bit against the sampler's own expression and on guarded
operands, and whole jobs (node path, runner.GraphedJob) against the fp64 job of tests/_job_ref.py and, bit for bit,
against the per-sigma route, where ComfyUI's sample_res_multistep (minicomfy's restatement) runs its own eager tensor
ops on the device schedule."""
import functools
import sys

import numpy as np
import pytest
import torch

import _guard as G
import _job_ref as J
import _launch_ref as R
import minicomfy
import test_gpu_sampler_ancestral as A
import test_gpu_sampler_dpm_2 as D2
import test_gpu_sampler_dpmpp_2m as M2
from _node_cases import NEG, POS, mixing_denoiser
from oracle import langevin_oracle as O

pytestmark = pytest.mark.gpu

K = 8            # |got - want| <= K * 2^-24 * magnitude per element, as tests/test_gpu_launch_ref.py
JOB_B = 4e-6     # max|got - want| / max|want| of a whole job, as tests/test_gpu_job_ref.py
F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16


def _native():
    from lanpaint_b200 import _native as n
    return n
SEEDED = J._plain(functools.partial(minicomfy.sample_res_multistep, extra_args={"seed": 0}))


@pytest.fixture(scope="module", autouse=True)
def _process_state(cuda_device):
    """What this file touches of the process, as it found it: the node layer's engine cache and patch, the default
    generators.  (No test here sets a library option.)"""
    minicomfy.install()
    from lanpaint_b200 import comfy_nodes as N
    import comfy.samplers as S
    patched = (S.CFGGuider.outer_sample, S.CFGGuider.predict_noise, S.KSAMPLER.sample)
    engines = dict(N._ENGINES.entries)
    cpu, cuda = torch.get_rng_state(), torch.cuda.get_rng_state(cuda_device)
    yield
    N._ENGINES.entries = engines
    torch.set_rng_state(cpu)
    torch.cuda.set_rng_state(cuda, cuda_device)
    assert (S.CFGGuider.outer_sample, S.CFGGuider.predict_noise, S.KSAMPLER.sample) == patched
    assert not N._override_active


# ---------------------------------------------------------------------------------------------------------------
# 1. one launch against fp64 and against the sampler's expression
# ---------------------------------------------------------------------------------------------------------------
def _res_rows(dev):
    """res_multistep_step of karras-20 on the device: (second-order rows, Euler rows)."""
    from lanpaint_b200.schedule import res_multistep_step
    patcher = minicomfy.ModelPatcher(minicomfy.BaseModel(None), "cpu")
    rows = res_multistep_step(J.ksampler_sigmas(patcher, 20, "res_multistep", "karras").to(dev))
    return [r[1:] for r in rows if r[0]], [r[1:3] for r in rows if not r[0]]


BASE = dict(shape=(8, 4, 128, 128), dtype=F32, combine=False, next=True, out=True, packed=True, seed=1)
BIG = (16, 4, 128, 128)      # 2^20 elements: the smallest launch that walks tail-first with evict-first operands
R128 = (128, 4, 128, 128)
LAUNCHES = {     # kind: "second" (lp_boundary_multistep, row k of the second-order steps) or "euler" (lp_boundary_midpoint)
    "second-f32-cfg-packed": dict(BASE, kind="second", row=0, combine=True),
    "second-f32-dense-last": dict(BASE, kind="second", row=17, packed=False, next=False, seed=2),
    "second-bf16-packed": dict(BASE, kind="second", row=9, dtype=BF16, seed=3),
    "second-all-known": dict(BASE, kind="second", row=4, mask="known", seed=4),
    "second-all-free-f16": dict(BASE, kind="second", row=5, mask="free", dtype=F16, seed=5),
    "euler-first-f32-packed": dict(BASE, kind="euler", row=0, seed=6),
    "euler-final-f32-last": dict(BASE, kind="euler", row=1, next=False, seed=7),
    "big-second-f32-cfg-packed": dict(BASE, kind="second", row=3, shape=BIG, combine=True, seed=8),
    "big-euler-bf16-dense": dict(BASE, kind="euler", row=0, shape=BIG, dtype=BF16, packed=False, seed=9),
    "r128-second-f32-packed": dict(BASE, kind="second", row=8, shape=R128, seed=10),
    "r128-euler-f32-packed": dict(BASE, kind="euler", row=0, shape=R128, seed=11),
    "wan-second-packed": dict(BASE, kind="second", row=12, shape=(1, 16, 21, 80, 45), seed=12),
    "ragged-second-dense": dict(BASE, kind="second", row=2, shape=(2, 3, 7, 9), packed=False, seed=13),
}


def make_case(c, dev):
    """-> (operands dict, dims, step, known bool tensor, the case in the helper module's terms, the helper module)."""
    second, euler = _res_rows(dev)
    if c["kind"] == "second":
        mc = dict(c, old=True)
        ops, dims, _, known = M2.make_case(mc, dev)
        step = M2._native().Multistep(*second[c["row"]])
        return ops, dims, step, known, mc, M2
    mc = dict(c, role="euler")
    ops, dims, _, known = D2.make_case(mc, dev)
    step = D2._native().Midpoint(*euler[c["row"]])
    return ops, dims, step, known, mc, D2


def _call(mod, mc, t, dims, step, dead=False):
    return (M2.call_multistep if mod is M2 else D2.call_midpoint)(mc, t, dims, step, dead=dead)


@pytest.mark.parametrize("case", list(LAUNCHES))
def test_launch_matches_fp64_and_the_samplers_expression(case, cuda_device):
    c = LAUNCHES[case]
    dev = cuda_device
    ops, dims, step, known, mc, mod = make_case(c, dev)
    cfg = 4.5 if c["combine"] else None
    if mod is M2:
        want = M2.ref_multistep(ops["a"], ops.get("b"), ops["y"], ops["noise"], known, ops["x"], ops["old"], step,
                                ops.get("table"), cfg)
    else:
        want = D2.ref_midpoint(ops["a"], ops.get("b"), ops["y"], ops["noise"], known, ops["x"], ops["x"], step,
                               ops.get("table"), cfg)
    fresh = lambda: dict(ops, **{k: ops[k].clone() for k in ("x", "out") if k in ops})   # noqa: E731
    t = fresh()
    kernels = A._launched(lambda: _call(mod, mc, t, dims, step))
    for _ in range(2):      # CUPTI can, rarely, deliver no record of a kernel that ran: launch again, same inputs
        if kernels:
            break
        t = fresh()
        kernels = A._launched(lambda: _call(mod, mc, t, dims, step))
    assert kernels == {mod.expect_kernel(mc, c["shape"])}, (case, kernels)
    worst, bad = R.within(t["x"], want["x"], K)
    assert bad is None, f"{case}: x element {bad}, worst ratio {worst:.3g} > K = {K}"
    if c["out"]:
        assert torch.equal(t["out"][known], ops["y"][known])
    # sample_res_multistep's own tensor ops (fp32 device tensors, one rounding each): bit for bit where no replace
    # step follows
    a = ops["a"].float()
    den = ops["b"].float() + (a - ops["b"].float()) * 4.5 if c["combine"] else a
    out = torch.where(known, ops["y"], den)
    s = lambda v: torch.tensor(v, dtype=torch.float32, device=dev)   # noqa: E731
    if mod is M2:     # sigma_fn(h) * x + h * (b1 * denoised + b2 * old_denoised)
        h, b1, b2 = s(-step.em1), s(step.c_cur), s(-step.c_old)
        eager = s(step.ratio) * ops["x"] + h * (b1 * out + b2 * ops["old"])
    else:             # x + to_d(x, sigma, denoised) * (sigma_down - sigma)
        eager = ops["x"] + ((ops["x"] - out) / s(step.sigma)) * s(step.dt)
    sel = ~known if c["next"] else torch.ones_like(known)
    assert torch.equal(t["x"][sel], eager[sel]), case


@pytest.mark.parametrize("case", ["second-f32-cfg-packed", "big-second-f32-cfg-packed", "big-euler-bf16-dense",
                                  "wan-second-packed"])
def test_results_do_not_depend_on_dead_heads(case, cuda_device):
    """LP_HEADS_DEAD gives the same x and out as the same launch without it, with res_multistep's scalars."""
    c = LAUNCHES[case]
    ops, dims, step, _, mc, mod = make_case(c, cuda_device)
    res = []
    for dead in (False, True):
        t = dict(ops, **{k: ops[k].clone() for k in ("x", "out", "a", "b") if k in ops})
        assert t["a"].data_ptr() % 128 == 0
        assert _call(mod, mc, t, dims, step, dead=dead) == 0
        torch.cuda.synchronize()
        res.append([t[k] for k in ("x", "out") if k in t])
    assert all(torch.equal(u, v) for u, v in zip(*res)), case


GUARDED = {
    "second-f32-cfg-packed": dict(LAUNCHES["second-f32-cfg-packed"], off=0),
    "second-f32-dense-last": dict(LAUNCHES["second-f32-dense-last"], off=0),
    "euler-first-f32-packed": dict(LAUNCHES["euler-first-f32-packed"], off=0),
    "big-euler-bf16-dense": dict(LAUNCHES["big-euler-bf16-dense"], off=0),
    "ragged-second-dense-misaligned": dict(LAUNCHES["ragged-second-dense"], off=4),
}
SLACK = {"y_known": 4, "noise_known": 4}


@pytest.mark.parametrize("case", list(GUARDED))
def test_guarded_operands(case, cuda_device):
    """Every operand between guard bands (tests/_guard.py): x and out bit-identical to the plain call's, the bands
    intact, the previous denoised latent, the heads and every other input unchanged."""
    c = GUARDED[case]
    dev = cuda_device
    ops, dims, step, _, mc, mod = make_case(c, dev)
    if "out" in ops:
        ops["out"] = torch.zeros_like(ops["out"])
    written = {"x"} | ({"out"} if c["out"] else set())
    offs = {k: (c["off"] if k in ("x", "y", "noise", "out", "old") else 0) for k in ops}
    plain = {k: G.plain(v, offs[k], SLACK.get(k, 0)) for k, v in ops.items()}
    arena = G.Arena(dev)
    guarded = {k: arena.place(v, offset_bytes=offs[k], slack=SLACK.get(k, 0), name=k) for k, v in ops.items()}
    arena.snapshot()
    assert _call(mod, mc, plain, dims, step) == 0
    assert _call(mod, mc, guarded, dims, step) == 0
    torch.cuda.synchronize()
    for k in written:
        assert torch.equal(G.bits(guarded[k]), G.bits(plain[k])), (case, k)
    arena.check(case, written=written)


# ---------------------------------------------------------------------------------------------------------------
# 2. whole jobs through the nodes
# ---------------------------------------------------------------------------------------------------------------
NODE = dict(shape=(8, 4, 128, 128), steps=12, n=5, cfg=5.0, window=None, calls=4, deferred=True)
NODE_CASES = {
    "b8-deferred": dict(NODE),
    "b8-steps": dict(NODE, deferred=False),
    "b8-window-leftover": dict(NODE, window=(2, 9, True)),
    "b8-window-leftover-steps": dict(NODE, window=(2, 9, True), deferred=False),
    "r128": dict(NODE, shape=R128, calls=3),
    "r128-window-leftover": dict(NODE, shape=R128, window=(2, 9, True), calls=3, deferred=False),
    "flow-video": dict(NODE, shape=(1, 16, 5, 32, 32), model_type="FLOW", shift=3.0, calls=3),
}


def _node_call(N, patcher, c, latent, seed):
    if c["window"] is None:
        (out,) = N.LanPaint_KSampler().sample(patcher, seed, c["steps"], c["cfg"], "res_multistep", "karras", POS, NEG,
                                              latent, 1.0, c["n"], "Image First", "", N.IMAGE_MODE)
    else:
        start, end, leftover = c["window"]
        (out,) = N.LanPaint_KSamplerAdvanced().sample(
            patcher, "enable", seed, c["steps"], c["cfg"], "res_multistep", "karras", POS, NEG, latent, start, end,
            "enable" if leftover else "disable", c["n"], 5.0, 0.2, "Image First", "", N.IMAGE_MODE)
    return out["samples"]


def _whole_sampler_call(fn, k):
    """A node call with "fused_sampler" off.  The whole-sampler graph hands the sampler the schedule as a CPU tensor,
    and sample_res_multistep seeds a private generator for its draw and divides by append_dims(sigma) -- a [1, 1, 1, 1]
    CPU tensor, not a 0-d one -- so its capture fails on the second call and the configuration falls back to one graph per wrapper call (the per-sigma
    route)."""
    if k != 1:
        return fn()
    with pytest.warns(UserWarning, match="capturing the sampler loop failed"):
        return fn()


@pytest.mark.parametrize("case", list(NODE_CASES))
def test_node_job_matches_fp64_and_the_per_sigma_route(case, cuda_device, monkeypatch):
    """eager -> capture -> replay -> (a new seed and mask on the same graphs): every call within JOB_B of the fp64
    job, per-step denoised latents equal y at known positions, generator offset the per-sigma route's, and the result
    and every step's denoised latent bit-identical to the per-sigma route.  With the option "fused_sampler" off the
    whole-sampler graph cannot take the job (see `_whole_sampler_call`): within JOB_B on its fallback."""
    c = NODE_CASES[case]
    from lanpaint_b200 import comfy_nodes as N
    N._ENGINES.clear()
    dev, shape = cuda_device, c["shape"]
    flow = c.get("model_type", "EPS") == "FLOW"
    base = minicomfy.BaseModel(mixing_denoiser, model_type=getattr(minicomfy.ModelType, c.get("model_type", "EPS")),
                               latent_channels=shape[1], shift=c.get("shift", 1.0))
    fused = minicomfy.ModelPatcher(base, dev)
    fused.model_options["lanpaint_b200"] = {"deferred_callbacks": c["deferred"], "deferred_max_ms": 1e9}
    per_sigma = minicomfy.ModelPatcher(base, dev)
    per_sigma.model_options["lanpaint_b200"] = {"fused_sampler": False, "sampler_graph": False}
    whole = minicomfy.ModelPatcher(base, dev)
    whole.model_options["lanpaint_b200"] = {"fused_sampler": False, "deferred_max_ms": 1e9}
    store = []
    monkeypatch.setattr(sys.modules["latent_preview"], "prepare_callback", A._recorder(store))
    window = {}
    if c["window"] is not None:
        window = dict(start_step=c["window"][0], last_step=c["window"][1], force_full_denoise=not c["window"][2])
    sig = J.ksampler_sigmas(fused, c["steps"], "res_multistep", "karras", 1.0, **window)
    if c["window"] is not None:
        assert float(sig[-1]) > 0
    md = J.max_denoise(base.model_sampling, sig[0])
    hp = O.Hyper(n_steps=c["n"], lam=5.0, step_size=0.2, min_step_frac=1.0, flow=flow)
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    y = torch.randn(shape, generator=g)
    mask = (torch.rand((shape[0], 1) + shape[2:], generator=g) < 0.5).float()
    gen = A._generator(dev)
    modes = []
    for k in range(c["calls"]):
        seed = 40 + k // 3
        if k == 3:
            y = torch.randn(shape, generator=g)
            mask = (torch.rand((shape[0], 1) + shape[2:], generator=g) < 0.5).float()
        latent = {"samples": y, "noise_mask": mask}
        store.clear()
        torch.cuda.manual_seed(900 + k)
        if k in (0, c["calls"] - 1):    # which kernels the eager job and the last replayed job ran
            got, kernels = A._sub_kernels(lambda: _node_call(N, fused, c, latent, seed))
            bnd = {n for n in kernels if n.startswith("boundary")}
            assert bnd == {"boundary_multistep_kernel<4,float,1>", "boundary_midpoint_kernel<4,float,1>"}, bnd
        else:
            got = _node_call(N, fused, c, latent, seed)
        modes.append(N.LAST_RUN["mode"])
        assert N.LAST_RUN["fused"] and N.LAST_RUN["job"].sampler == "res_multistep"
        torch.cuda.synchronize()
        offset, got_steps = gen.get_offset(), list(store)

        # the per-sigma route: the sampler's loop, its updates as eager device ops
        store.clear()
        torch.cuda.manual_seed(900 + k)
        ref = _node_call(N, per_sigma, c, latent, seed)
        assert N.LAST_RUN["mode"] is None and not N.LAST_RUN["fused"]
        torch.cuda.synchronize()
        assert gen.get_offset() == offset
        assert torch.equal(got, ref), f"{case} call {k}: fused and per-sigma results differ, max {float((got - ref).abs().max())}"
        assert len(store) == len(got_steps) == len(sig) - 1
        for (i, d), (j, e) in zip(got_steps, store):
            assert i == j and torch.equal(d, e), f"{case} call {k}: denoised[{i}] differs from the per-sigma route's"

        # fp64
        torch.cuda.manual_seed(900 + k)
        noise = minicomfy.prepare_noise(y, seed)
        yd = y.to(dev, torch.float64)
        dm = minicomfy.repeat_to_batch_size(mask, shape[0]).expand(shape).to(dev, torch.float64)
        want_steps = []
        model = J.Guider(mixing_denoiser, O.FlowSampling() if flow else O.VESampling(), c["cfg"], c["cfg"])
        want = J.job(SEEDED, model, yd, noise.to(dev, torch.float64), dm, sig, hp,
                     max_denoise=md, callback=lambda i, d: want_steps.append(d))
        assert gen.get_offset() == offset, f"{case} call {k}: generator offset differs from the reference's"
        assert A._rel(got, want) <= JOB_B, (case, k, A._rel(got, want))
        known = (dm <= 0.5)
        for (i, d), w in zip(got_steps, want_steps):
            assert A._rel(d, w) <= JOB_B, (case, k, i, A._rel(d, w))
            assert torch.equal(d[known], y.to(dev)[known])

        # the whole-sampler graph's configuration: recorded on the first call, its capture fails on the second
        if k < 2:
            torch.cuda.manual_seed(900 + k)
            sg = _whole_sampler_call(lambda: _node_call(N, whole, c, latent, seed), k)
            assert not N.LAST_RUN["fused"] and N.LAST_RUN["mode"] is None
            assert A._rel(sg, want) <= JOB_B, (case, k, "whole-sampler fallback", A._rel(sg, want))
    assert modes == ["eager"] + ["job" if c["deferred"] else "steps"] * (c["calls"] - 1), modes
    N._ENGINES.clear()


# ---------------------------------------------------------------------------------------------------------------
# 3. runner.GraphedJob directly
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(2, 4, 64, 64), (8, 4, 128, 128)])
@pytest.mark.parametrize("sigmas", ["to-zero", "leftover"])
@pytest.mark.parametrize("rng", ["torch", "philox"])
def test_graphed_job_equals_the_unfused_definition(shape, sigmas, rng, cuda_device):
    """eager / per-step graphs / whole-job graph (with and without per-step outputs), fused and un-fused, each
    bit-equal to res_multistep_inpaint, with the generator left where the definition leaves it.  Per-step graphs
    are also captured last step first."""
    from lanpaint_b200.runner import GraphedJob, HostSchedule, res_multistep_inpaint, karras_sigmas
    dev = cuda_device
    ks = karras_sigmas(8)
    sched = HostSchedule(ks if sigmas == "to-zero" else ks[1:-2], shape[0], 4, early_stop=2)
    g = torch.Generator().manual_seed(9)
    y, noise = torch.randn(shape, generator=g).to(dev), torch.randn(shape, generator=g).to(dev)
    mask = (torch.rand((shape[0], 1) + shape[2:], generator=g) < 0.5).float().to(dev)
    gen = A._generator(dev)
    engine = lambda: A._engine(rng)      # noqa: E731
    torch.cuda.manual_seed(31)
    want = res_multistep_inpaint(engine(), y, noise, mask, sched)
    offset = gen.get_offset()
    n = len(sched.steps)
    for fused in (True, False):
        job = GraphedJob(engine(), sched, shape, dev, fused_euler=fused, sampler="res_multistep")
        euler = [isinstance(st, _native().Midpoint) for st, _ in job.multistep]
        assert euler[0] and not any(euler[1:-1]) and euler[-1] == (sigmas == "to-zero")
        for mode, cb in (("eager", False), ("steps", False), ("job", False), ("job", True), ("steps", True)):
            steps = []
            callback = (lambda i, d, x, total: steps.append((i, d.clone()))) if cb else None
            torch.cuda.manual_seed(31)
            got = job.run(y, noise, mask, mode=mode, callback=callback)
            assert gen.get_offset() == offset, (fused, mode)
            assert torch.equal(got, want), (fused, mode, cb, float((got - want).abs().max()))
            if cb:
                assert [i for i, _ in steps] == list(range(n))
                ref = steps if mode == "job" else ref
                assert all(torch.equal(d, e) for (_, d), (_, e) in zip(steps, ref)), (fused, mode)
    job = GraphedJob(engine(), sched, shape, dev, sampler="res_multistep")
    job.load_inputs(y, noise, mask)
    for i in reversed(range(n)):
        job._graph_for(("step", i, False), lambda p, i=i: job._step(i, p, False), True)
    torch.cuda.manual_seed(31)
    assert torch.equal(job.run(y, noise, mask, mode="steps"), want)


# ---------------------------------------------------------------------------------------------------------------
# 4. routing
# ---------------------------------------------------------------------------------------------------------------
def test_routing_and_cache_separation(cuda_device):
    """res_multistep takes the fused loop by default; {"fused_sampler": False} turns it off; a zero noise image
    (add_noise = disable) stays on its route; euler and res_multistep on one configuration never share a job."""
    from lanpaint_b200 import comfy_nodes as N
    N._ENGINES.clear()
    dev, shape = cuda_device, (2, 4, 64, 64)
    base = minicomfy.BaseModel(mixing_denoiser, model_type=minicomfy.ModelType.EPS, latent_channels=4, shift=1.0)
    g = torch.Generator().manual_seed(3)
    latent = {"samples": torch.randn(shape, generator=g), "noise_mask": (torch.rand((2, 1, 64, 64), generator=g) < 0.5).float()}

    def run(patcher, sampler="res_multistep"):
        torch.cuda.manual_seed(1)
        (out,), kernels = A._sub_kernels(lambda: N.LanPaint_KSampler().sample(
            patcher, 5, 8, 4.0, sampler, "karras", POS, NEG, latent, 1.0, 3, "Image First", "", N.IMAGE_MODE))
        return out["samples"], N.LAST_RUN["mode"], N.LAST_RUN["fused"], N.LAST_RUN["job"], kernels

    patcher = minicomfy.ModelPatcher(base, dev)
    patcher.model_options["lanpaint_b200"] = {"sampler_graph": False}
    seen = []
    for on in (None, False, None, True, False, None):
        opts = {"sampler_graph": False}
        if on is not None:
            opts["fused_sampler"] = on
        patcher.model_options["lanpaint_b200"] = opts
        out, mode, fused, job, kernels = run(patcher)
        seen.append((out, mode, fused, job))
        assert fused == (on is not False)
        assert ("boundary_multistep_kernel<4,float,1>" in kernels) == fused, kernels
        assert ("boundary_midpoint_kernel<4,float,1>" in kernels) == fused, kernels
        if not fused:
            assert not any(k.startswith(("boundary_multistep", "boundary_midpoint")) for k in kernels), kernels
    # None and {"fused_sampler": True} are two configurations: each starts eager; with the option off (and the
    # whole-sampler graph off) the per-sigma route runs
    assert [m for _, m, _, _ in seen] == ["eager", None, "job", "eager", None, "job"]
    # the per-sigma route bit for bit
    assert all(torch.equal(seen[0][0], seen[k][0]) for k in (1, 2, 3, 4, 5))
    assert seen[0][3] is seen[2][3] is seen[5][3] and seen[0][3].sampler == "res_multistep"
    assert seen[3][3] is not seen[0][3] and seen[3][3].sampler == "res_multistep"
    out_e, mode_e, fused_e, job_e, _ = run(patcher, "euler")
    assert fused_e and job_e is not seen[0][3] and job_e.sampler == "euler" and mode_e == "eager"
    assert not torch.equal(out_e, seen[0][0])
    assert run(patcher)[3] is seen[0][3]
    # add_noise = disable: a zero noise image, regenerated at every outer step by the per-sigma route
    torch.cuda.manual_seed(1)
    N.LanPaint_KSamplerAdvanced().sample(patcher, "disable", 5, 8, 4.0, "res_multistep", "karras", POS, NEG, latent, 0,
                                         10000, "disable", 3, 5.0, 0.2, "Image First", "", N.IMAGE_MODE)
    assert not N.LAST_RUN["fused"]
    N._ENGINES.clear()


def test_gate(cuda_device):
    from lanpaint_b200 import comfy_nodes as N
    from lanpaint_b200.engine import LanPaint

    class K:    # what _fused_res_multistep_ok reads of the wrapper
        audio_indicator = None
        sigmas_host = [3.0, 1.0, 0.0]
    ks = minicomfy.ksampler("res_multistep")
    eng = LanPaint(None, NSteps=3, Friction=15.0, Lambda=5.0, Beta=1.0, StepSize=0.2, rng="torch")
    dm = torch.ones(1)
    ok = lambda k=K, e=eng, mo={}, s=ks, ea={"seed": 5}: N.KSAMPLER._fused_res_multistep_ok(s, k, dm, mo, e, ea)  # noqa
    assert ok()
    assert not ok(ea={}) and not ok(ea={"seed": None})
    assert not N.KSAMPLER._fused_res_multistep_ok(ks, K, None, {}, eng, {"seed": 5})
    assert not ok(k=type("AV", (K,), {"audio_indicator": torch.ones(1)}))
    assert not ok(mo={"denoise_mask_function": lambda *a, **k: None})
    assert not ok(mo={"callback": lambda *a: None})
    assert not ok(mo={"lanpaint_semantic_stop": {}})
    assert not ok(e=LanPaint(None, NSteps=3, Friction=15.0, Lambda=5.0, Beta=1.0, StepSize=0.2, rng="torch",
                             EarlyStopThreshold=1e-3))
    assert not ok(s=minicomfy.ksampler("euler")) and not ok(s=minicomfy.ksampler("dpm_2"))
    assert not ok(s=minicomfy.ksampler("res_multistep", {"s_noise": 0.5}))
    assert not ok(k=type("Z", (K,), {"sigmas_host": [3.0, 0.0, 0.0]}))

    def sample_res_multistep(model, x, sigmas, **kw):     # the name, but not the sampler's form
        return x
    assert not ok(s=minicomfy.KSAMPLER(sample_res_multistep))
