"""GPU: the fused heun loop (opt-in, "fused_heun") -- lp_boundary_heun per launch against fp64 and on guarded operands,
and whole jobs (node path, runner.GraphedJob) against the fp64 job of tests/_job_ref.py and, bit for bit, against the
per-sigma route, where k-diffusion's sample_heun runs its own eager tensor ops on the device schedule, and against
the whole-sampler graph, which captures that loop."""
import ctypes as C
import sys

import numpy as np
import pytest
import torch

import _guard as G
import _job_ref as J
import _launch_ref as R
import minicomfy
import test_gpu_sampler_ancestral as A
from _node_cases import NEG, POS, mixing_denoiser
from oracle import langevin_oracle as O

pytestmark = pytest.mark.gpu

K = 8            # |got - want| <= K * 2^-24 * magnitude per element, as tests/test_gpu_launch_ref.py
JOB_B = 4e-6     # max|got - want| / max|want| of a whole job, as tests/test_gpu_job_ref.py
P = C.c_void_p
DTYPES = A.DTYPES
LP_DT = A.LP_DT
F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16
FUSED = {"fused_heun": True}


def _native():
    from lanpaint_b200 import _native as n
    return n


def _lib():
    return _native().load()


def _stream():
    return P(torch.cuda.current_stream().cuda_stream)


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
# 1. one launch against fp64
# ---------------------------------------------------------------------------------------------------------------
STEP = (1.625, 0.875, -0.75)     # sigma, sigma_next, dt


def ref_heun(a, b, y, noise, known, x, x2, prev, step, next_tab, cfg):
    """lp_boundary_heun of the header in fp64 -> dict(out, x) of (value, magnitude) pairs (see _launch_ref)."""
    def expr(m, a, b, y, noise, x, x2, prev):
        A_ = m.abs
        den = b + m.sub(a, b) * A_(cfg) if cfg is not None else a
        out = torch.where(known, y, den)
        d = m.sub(x, prev) / A_(step.sigma)
        d2 = m.sub(x2, out) / A_(step.sigma_next)
        u = x + (d + d2) * 0.5 * A_(step.dt)
        if next_tab is not None:
            rn, ry = A_(R._row(next_tab, R.T_REPN, u.ndim)), A_(R._row(next_tab, R.T_REPY, u.ndim))
            u = torch.where(known, rn * noise + ry * y, u)
        return out, u
    z = torch.zeros((), dtype=torch.float64, device=y.device)
    ops = [R._d(a), z if b is None else R._d(b), R._d(y), R._d(noise), R._d(x), R._d(x2), R._d(prev)]
    val = expr(R._Val, *ops)
    mag = expr(R._Mag, *[None if o is None else o.abs() for o in ops])
    return {"out": (val[0], mag[0]), "x": (val[1], mag[1])}


def expect_kernel(c, shape):
    v4 = int(np.prod(shape[2:])) % 4 == 0
    return f"boundary_heun_kernel<{4 if v4 else 1},{DTYPES[c['dtype']]},{int(c['packed'])}>"


def make_case(c, dev):
    """-> (operands dict, dims, step, known bool tensor) of case c."""
    nat, lib = _native(), _lib()
    shape = c["shape"]
    total, sp = int(np.prod(shape)), int(np.prod(shape[2:]))
    gen = torch.Generator(device=dev).manual_seed(c["seed"])
    bshape = (shape[0], 1) + tuple(shape[2:])
    known1 = {"rand": lambda: torch.rand(bshape, device=dev, generator=gen) < 0.5,
              "known": lambda: torch.ones(bshape, dtype=torch.bool, device=dev),
              "free": lambda: torch.zeros(bshape, dtype=torch.bool, device=dev)}[c.get("mask", "rand")]()
    m8 = known1.to(torch.uint8).contiguous()
    dims = nat.Dims(shape[0], total // shape[0], sp, sp, 0, 0)
    ops = {"x": torch.randn(shape, device=dev, generator=gen) * 3, "y": torch.randn(shape, device=dev, generator=gen),
           "noise": torch.randn(shape, device=dev, generator=gen), "mask": m8,
           "a": (torch.randn(shape, device=dev, generator=gen) * 1.5).to(c["dtype"])}
    ops["x2"] = ops["x"] + 0.5 * torch.randn(shape, device=dev, generator=gen)
    ops["prev"] = torch.where(known1.expand(shape), ops["y"], torch.randn(shape, device=dev, generator=gen))
    if c["combine"]:
        ops["b"] = (ops["a"].float() + 0.3 * torch.randn(shape, device=dev, generator=gen)).to(c["dtype"])
    if c["next"]:
        ops["table"] = A.table_rows(shape[0], dev, c["seed"])
    if c["out"]:
        ops["out"] = torch.full(shape, float("nan"), device=dev)
    if c["packed"]:
        words = torch.zeros(int(lib.lp_known_words(total)), dtype=torch.int32, device=dev)
        yk, nk = torch.zeros(total + 4, device=dev), torch.zeros(total + 4, device=dev)
        assert lib.lp_pack_known(P(m8.data_ptr()), C.byref(dims), P(ops["y"].data_ptr()), P(ops["noise"].data_ptr()),
                                 P(words.data_ptr()), P(yk.data_ptr()), P(nk.data_ptr()), _stream()) == 0
        ops.update(words=words, y_known=yk, noise_known=nk)
    return ops, dims, nat.Heun(*STEP), known1.expand(shape)


def call_heun(c, t, dims, step, dead=False):
    """One lp_boundary_heun call on the operands t (name -> tensor)."""
    nat, lib = _native(), _lib()
    p = lambda k: P(t[k].data_ptr()) if k in t else None   # noqa: E731
    cfg = 4.5 if c["combine"] else 0.0
    hd = nat.Heads(t["a"].data_ptr(), t["b"].data_ptr() if "b" in t else None,
                   LP_DT[c["dtype"]] | (nat.HEADS_DEAD if dead else 0), 1 if c["combine"] else 0, cfg, cfg)
    kn = nat.Known(t["words"].data_ptr(), t["y_known"].data_ptr(), t["noise_known"].data_ptr()) if c["packed"] else None
    return lib.lp_boundary_heun(C.byref(hd), p("y"), p("noise"), p("mask"), C.byref(kn) if kn is not None else None,
                                p("x"), p("x2"), p("prev"), p("out"), C.byref(step), p("table"), C.byref(dims),
                                _stream())


BASE = dict(shape=(8, 4, 128, 128), dtype=F32, combine=False, next=True, out=False, packed=True, seed=1)
BIG = (16, 4, 128, 128)      # 2^20 elements: the smallest launch that walks tail-first with evict-first operands
R128 = (128, 4, 128, 128)
LAUNCHES = {
    "f32-cfg-next-packed": dict(BASE, combine=True),
    "f32-cfg-next-dense-out": dict(BASE, combine=True, packed=False, out=True, seed=2),
    "bf16-last-packed": dict(BASE, dtype=BF16, next=False, seed=3),
    "bf16-next-dense": dict(BASE, dtype=BF16, packed=False, seed=4),
    "f16-last-dense-out": dict(BASE, dtype=F16, next=False, packed=False, out=True, seed=5),
    "all-known-next": dict(BASE, mask="known", seed=6),
    "all-known-last-dense": dict(BASE, mask="known", next=False, packed=False, seed=7),
    "all-free-f16": dict(BASE, mask="free", dtype=F16, seed=8),
    "big-f32-cfg-packed": dict(BASE, shape=BIG, combine=True, seed=9),
    "big-bf16-dense-last": dict(BASE, shape=BIG, dtype=BF16, packed=False, next=False, seed=10),
    "r128-f32-packed": dict(BASE, shape=R128, seed=11),
    "r128-bf16-dense-last": dict(BASE, shape=R128, dtype=BF16, packed=False, next=False, seed=12),
    "wan-packed": dict(BASE, shape=(1, 16, 21, 80, 45), seed=13),
    "small-cfg-dense": dict(BASE, shape=(1, 4, 32, 32), combine=True, packed=False, seed=14),
    "ragged-packed": dict(BASE, shape=(1, 3, 7, 9), seed=15),
    "ragged-dense-f16-last-out": dict(BASE, shape=(2, 3, 7, 9), packed=False, dtype=F16, next=False, out=True,
                                      seed=16),
    "ragged-cfg-dense": dict(BASE, shape=(2, 3, 7, 9), combine=True, packed=False, seed=17),
}


@pytest.mark.parametrize("case", list(LAUNCHES))
def test_launch_matches_fp64(case, cuda_device):
    c = LAUNCHES[case]
    ops, dims, step, known = make_case(c, cuda_device)
    want = ref_heun(ops["a"], ops.get("b"), ops["y"], ops["noise"], known, ops["x"], ops["x2"], ops["prev"], step,
                    ops.get("table"), 4.5 if c["combine"] else None)
    fresh = lambda: dict(ops, **{k: ops[k].clone() for k in ("x", "out") if k in ops})   # noqa: E731
    t = fresh()
    kernels = A._launched(lambda: call_heun(c, t, dims, step))
    for _ in range(2):      # CUPTI can, rarely, deliver no record of a kernel that ran: launch again, same inputs
        if kernels:
            break
        t = fresh()
        kernels = A._launched(lambda: call_heun(c, t, dims, step))
    assert kernels == {expect_kernel(c, c["shape"])}, (case, kernels)
    worst, bad = R.within(t["x"], want["x"], K)
    assert bad is None, f"{case}: x element {bad}, worst ratio {worst:.3g} > K = {K}"
    for k in ("x2", "prev"):
        assert torch.equal(t[k], ops[k]), (case, k)        # an input is never written
    if c["out"]:
        worst, bad = R.within(t["out"], want["out"], K)
        assert bad is None, f"{case}: out element {bad}, worst ratio {worst:.3g}"
        assert torch.equal(t["out"][known], ops["y"][known])
    if c["next"]:     # the replace step rounds as lp_prologue_f32 does
        xp = torch.zeros_like(t["x"])
        assert _lib().lp_prologue_f32(P(xp.data_ptr()), P(ops["y"].data_ptr()), P(ops["noise"].data_ptr()),
                                      P(ops["mask"].data_ptr()), P(xp.data_ptr()), None, P(ops["table"].data_ptr()),
                                      C.byref(dims), _stream()) == 0
        assert torch.equal(t["x"][known], xp[known])
    # the update in sample_heun's own tensor ops (fp32 device tensors, one rounding each, d and d_2 divided by
    # [B, 1, ...] device sigmas, / 2 as torch does it): bit for bit where no replace step follows
    a = ops["a"].float()
    den = a if not c["combine"] else ops["b"].float() + (a - ops["b"].float()) * 4.5
    out = torch.where(known, ops["y"], den)
    B, nd = c["shape"][0], len(c["shape"])
    s = lambda v: torch.full((B,) + (1,) * (nd - 1), v, dtype=torch.float32, device=cuda_device)   # noqa: E731
    dt = torch.tensor(step.dt, dtype=torch.float32, device=cuda_device)
    d = (ops["x"] - ops["prev"]) / s(step.sigma)
    d_2 = (ops["x2"] - out) / s(step.sigma_next)
    eager = ops["x"] + (d + d_2) / 2 * dt
    sel = ~known if c["next"] else torch.ones_like(known)
    assert torch.equal(t["x"][sel], eager[sel]), case


@pytest.mark.parametrize("case", ["f32-cfg-next-packed", "big-f32-cfg-packed", "big-bf16-dense-last",
                                  "r128-bf16-dense-last", "wan-packed"])
def test_results_do_not_depend_on_dead_heads(case, cuda_device):
    """LP_HEADS_DEAD (128-byte aligned heads that no state or output overlaps: the launch drops their L2 lines) gives
    the same x and out as the same launch without it."""
    c = dict(LAUNCHES[case], out=True)
    ops, dims, step, _ = make_case(c, cuda_device)
    res = []
    for dead in (False, True):
        t = dict(ops, **{k: ops[k].clone() for k in ("x", "out", "a", "b") if k in ops})
        assert t["a"].data_ptr() % 128 == 0
        assert call_heun(c, t, dims, step, dead=dead) == 0
        torch.cuda.synchronize()
        res.append((t["x"], t["out"]))
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1]), case


GUARDED = {
    "f32-cfg-next-packed": dict(LAUNCHES["f32-cfg-next-packed"], off=0),
    "f32-cfg-next-dense-out": dict(LAUNCHES["f32-cfg-next-dense-out"], off=0),
    "big-bf16-dense-last": dict(LAUNCHES["big-bf16-dense-last"], off=0),
    "r128-f32-packed": dict(LAUNCHES["r128-f32-packed"], off=0),
    "wan-packed": dict(LAUNCHES["wan-packed"], off=0),
    "ragged-packed-misaligned": dict(LAUNCHES["ragged-packed"], off=4),
    "ragged-dense-f16-last-out-misaligned": dict(LAUNCHES["ragged-dense-f16-last-out"], off=4),
}
SLACK = {"y_known": 4, "noise_known": 4}


@pytest.mark.parametrize("case", list(GUARDED))
def test_guarded_operands(case, cuda_device):
    """Every operand between guard bands (tests/_guard.py): x and out bit-identical to the plain call's, the bands
    intact, x2, out_prev and every other input unchanged."""
    c = GUARDED[case]
    dev = cuda_device
    ops, dims, step, _ = make_case(c, dev)
    if "out" in ops:
        ops["out"] = torch.zeros_like(ops["out"])
    written = {"x"} | ({"out"} if c["out"] else set())
    offs = {k: (c["off"] if k in ("x", "x2", "prev", "y", "noise", "out") else 0) for k in ops}
    plain = {k: G.plain(v, offs[k], SLACK.get(k, 0)) for k, v in ops.items()}
    arena = G.Arena(dev)
    guarded = {k: arena.place(v, offset_bytes=offs[k], slack=SLACK.get(k, 0), name=k) for k, v in ops.items()}
    arena.snapshot()
    assert call_heun(c, plain, dims, step) == 0
    assert call_heun(c, guarded, dims, step) == 0
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
        (out,) = N.LanPaint_KSampler().sample(patcher, seed, c["steps"], c["cfg"], "heun", "karras", POS, NEG,
                                              latent, 1.0, c["n"], "Image First", "", N.IMAGE_MODE)
    else:
        start, end, leftover = c["window"]
        (out,) = N.LanPaint_KSamplerAdvanced().sample(
            patcher, "enable", seed, c["steps"], c["cfg"], "heun", "karras", POS, NEG, latent, start, end,
            "enable" if leftover else "disable", c["n"], 5.0, 0.2, "Image First", "", N.IMAGE_MODE)
    return out["samples"]


HEUN_KERNELS = {"boundary_midpoint_kernel<4,float,1>", "boundary_heun_kernel<4,float,1>"}


@pytest.mark.parametrize("case", list(NODE_CASES))
def test_node_job_matches_fp64_and_the_other_routes(case, cuda_device, monkeypatch):
    """eager -> capture -> replay -> (a new seed and mask on the same graphs): every call within JOB_B of the fp64
    job, per-step denoised latents equal y at known positions, generator offset the per-sigma route's, and the result
    and every step's denoised latent bit-identical to the per-sigma route.  Without the option the configuration
    takes today's routes (the whole-sampler graph, where the job is short enough): bit-identical again."""
    c = NODE_CASES[case]
    from lanpaint_b200 import comfy_nodes as N
    N._ENGINES.clear()
    dev, shape = cuda_device, c["shape"]
    flow = c.get("model_type", "EPS") == "FLOW"
    base = minicomfy.BaseModel(mixing_denoiser, model_type=getattr(minicomfy.ModelType, c.get("model_type", "EPS")),
                               latent_channels=shape[1], shift=c.get("shift", 1.0))
    fused = minicomfy.ModelPatcher(base, dev)
    fused.model_options["lanpaint_b200"] = dict(FUSED, deferred_callbacks=c["deferred"], deferred_max_ms=1e9)
    per_sigma = minicomfy.ModelPatcher(base, dev)
    per_sigma.model_options["lanpaint_b200"] = {"fused_sampler": False, "sampler_graph": False}
    whole = minicomfy.ModelPatcher(base, dev)
    whole.model_options["lanpaint_b200"] = {"deferred_max_ms": 1e9}
    store = []
    monkeypatch.setattr(sys.modules["latent_preview"], "prepare_callback", A._recorder(store))
    window = {}
    if c["window"] is not None:
        window = dict(start_step=c["window"][0], last_step=c["window"][1], force_full_denoise=not c["window"][2])
    sig = J.ksampler_sigmas(fused, c["steps"], "heun", "karras", 1.0, **window)
    if c["window"] is not None:
        assert float(sig[-1]) > 0
    md = J.max_denoise(base.model_sampling, sig[0])
    hp = O.Hyper(n_steps=c["n"], lam=5.0, step_size=0.2, min_step_frac=1.0, flow=flow)
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    y = torch.randn(shape, generator=g)
    mask = (torch.rand((shape[0], 1) + shape[2:], generator=g) < 0.5).float()
    gen = A._generator(dev)
    modes, whole_modes = [], []
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
            assert bnd == HEUN_KERNELS, bnd
        else:
            got = _node_call(N, fused, c, latent, seed)
        modes.append(N.LAST_RUN["mode"])
        assert N.LAST_RUN["fused"] and N.LAST_RUN["job"].sampler == "heun"
        torch.cuda.synchronize()
        offset, got_steps = gen.get_offset(), list(store)

        # the per-sigma route: k-diffusion's loop, its scalars and updates as eager device ops, two wrapper calls a step
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
        want = J.job(J._plain(minicomfy.sample_heun), model, yd, noise.to(dev, torch.float64), dm, sig, hp,
                     max_denoise=md, callback=lambda i, d: want_steps.append(d))
        assert gen.get_offset() == offset, f"{case} call {k}: generator offset differs from the reference's"
        assert A._rel(got, want) <= JOB_B, (case, k, A._rel(got, want))
        known = (dm <= 0.5)
        for (i, d), w in zip(got_steps, want_steps):
            assert A._rel(d, w) <= JOB_B, (case, k, i, A._rel(d, w))
            assert torch.equal(d[known], y.to(dev)[known])

        # the default options: today's routes (recorded on the first call, the whole-sampler graph after it)
        if k < 3:
            torch.cuda.manual_seed(900 + k)
            sg = _node_call(N, whole, c, latent, seed)
            whole_modes.append(N.LAST_RUN["mode"])
            assert not N.LAST_RUN["fused"]
            assert gen.get_offset() == offset
            assert torch.equal(sg, ref), (case, k, whole_modes[-1], float((sg - ref).abs().max()))
    assert modes == ["eager"] + ["job" if c["deferred"] else "steps"] * (c["calls"] - 1), modes
    assert whole_modes[0] is None, whole_modes
    if case in ("b8-deferred", "b8-steps", "r128"):
        assert "sampler-graph" in whole_modes, whole_modes
    N._ENGINES.clear()


# ---------------------------------------------------------------------------------------------------------------
# 3. runner.GraphedJob directly
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(2, 4, 64, 64), (8, 4, 128, 128)])
@pytest.mark.parametrize("sigmas", ["to-zero", "leftover"])
@pytest.mark.parametrize("rng", ["torch", "philox"])
def test_graphed_job_equals_the_unfused_definition(shape, sigmas, rng, cuda_device):
    """eager / per-step graphs / whole-job graph (with and without per-step outputs), fused and un-fused, each
    bit-equal to heun_inpaint, with the generator left where the definition leaves it.  Per-step graphs are also
    captured last step first."""
    from lanpaint_b200.runner import GraphedJob, HostSchedule, heun_inpaint, karras_sigmas
    dev = cuda_device
    ks = karras_sigmas(8)
    sched = HostSchedule(ks if sigmas == "to-zero" else ks[1:-2], shape[0], 4, early_stop=2)
    g = torch.Generator().manual_seed(9)
    y, noise = torch.randn(shape, generator=g).to(dev), torch.randn(shape, generator=g).to(dev)
    mask = (torch.rand((shape[0], 1) + shape[2:], generator=g) < 0.5).float().to(dev)
    gen = A._generator(dev)
    engine = lambda: A._engine(rng)      # noqa: E731
    torch.cuda.manual_seed(31)
    want = heun_inpaint(engine(), y, noise, mask, sched)
    offset = gen.get_offset()
    n = len(sched.steps)
    for fused in (True, False):
        job = GraphedJob(engine(), sched, shape, dev, fused_euler=fused, sampler="heun",
                         sampler_fn=minicomfy.sample_heun)
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
    job = GraphedJob(engine(), sched, shape, dev, sampler="heun", sampler_fn=minicomfy.sample_heun)
    job.load_inputs(y, noise, mask)
    for i in reversed(range(n)):
        job._graph_for(("step", i, False), lambda p, i=i: job._step(i, p, False), True)
    torch.cuda.manual_seed(31)
    assert torch.equal(job.run(y, noise, mask, mode="steps"), want)


# ---------------------------------------------------------------------------------------------------------------
# 4. routing
# ---------------------------------------------------------------------------------------------------------------
def test_routing_and_cache_separation(cuda_device):
    """heun takes the fused loop only with {"fused_heun": True}, and {"fused_sampler": False} turns it off again;
    without the option its modes are today's.  Toggling the option on one patcher gives identical outputs and keeps the
    fused job and the whole-sampler graph's job apart."""
    from lanpaint_b200 import comfy_nodes as N
    N._ENGINES.clear()
    dev, shape = cuda_device, (2, 4, 64, 64)
    base = minicomfy.BaseModel(mixing_denoiser, model_type=minicomfy.ModelType.EPS, latent_channels=4, shift=1.0)
    g = torch.Generator().manual_seed(3)
    latent = {"samples": torch.randn(shape, generator=g), "noise_mask": (torch.rand((2, 1, 64, 64), generator=g) < 0.5).float()}

    def run(patcher):
        torch.cuda.manual_seed(1)
        (out,), kernels = A._sub_kernels(lambda: N.LanPaint_KSampler().sample(
            patcher, 5, 8, 4.0, "heun", "karras", POS, NEG, latent, 1.0, 3, "Image First", "", N.IMAGE_MODE))
        return out["samples"], N.LAST_RUN["mode"], N.LAST_RUN["fused"], N.LAST_RUN["job"], kernels

    patcher = minicomfy.ModelPatcher(base, dev)
    seen = []
    for opt in (None, FUSED, None, FUSED, dict(FUSED, fused_sampler=False), None, FUSED):
        if opt is None:
            patcher.model_options.pop("lanpaint_b200", None)
        else:
            patcher.model_options["lanpaint_b200"] = dict(opt)
        out, mode, fused, job, kernels = run(patcher)
        seen.append((out, mode, fused, job))
        on = opt is not None and opt.get("fused_sampler", True)
        assert fused == on, (opt, mode)
        assert ("boundary_heun_kernel<4,float,1>" in kernels) == on, kernels
        if on:
            assert job.sampler == "heun"
        else:
            assert not any(k.startswith(("boundary_heun", "boundary_midpoint")) for k in kernels), kernels
    modes = [m for _, m, _, _ in seen]
    # without the option: recorded, then the whole-sampler graph; with it: eager, then the fused job's graph
    assert modes[0] is None and modes[2] == modes[5] == "sampler-graph", modes
    assert modes[1] == "eager" and modes[3] == modes[6] == "job", modes
    assert all(torch.equal(seen[0][0], s[0]) for s in seen[1:])
    assert seen[1][3] is seen[3][3] is seen[6][3]
    assert seen[2][3] is not seen[3][3] and getattr(seen[2][3], "sampler", None) != "heun"
    N._ENGINES.clear()
