"""GPU: the fused gradient_estimation loop -- lp_boundary_gradient_estimation per launch against fp64 and on guarded
operands, and whole jobs (node path, runner.GraphedJob) against the fp64 job of tests/_job_ref.py and, bit for bit,
against the per-sigma route, where ComfyUI's sample_gradient_estimation (minicomfy's restatement) runs its own eager
tensor ops on the device schedule."""
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

K = 10           # |got - want| <= K * 2^-24 * magnitude per element: the longest chain (CFG combine, then the
                 # corrected step) rounds 10 times
JOB_B = 4e-6     # max|got - want| / max|want| of a whole job, as tests/test_gpu_job_ref.py
P = C.c_void_p
DTYPES = A.DTYPES
LP_DT = A.LP_DT
F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16


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
STEP = (2.5, -0.875, 1.0)          # sigma, dt, gm1 of a step with sigma_next > 0
STEP_GM = (1.625, -0.5, 0.375)     # ge_gamma = 1.375
FINAL = (0.4375, -0.4375, 1.0)     # the step to sigma = 0


def ref_ge(a, b, y, noise, known, x, dp, step, next_tab, cfg):
    """lp_boundary_gradient_estimation of the header in fp64 -> dict(out, d, x) of (value, magnitude) pairs (see
    _launch_ref)."""
    def expr(m, a, b, y, noise, x, dp):
        A_ = m.abs
        den = b + m.sub(a, b) * A_(cfg) if cfg is not None else a
        out = torch.where(known, y, den)
        d = m.sub(x, out) / A_(step.sigma)
        if step.final:
            xn = out
        else:
            xn = x + d * A_(step.dt)
            if dp is not None:
                xn = xn + (A_(step.gm1) * m.sub(d, dp)) * A_(step.dt)
        if next_tab is not None:
            rn, ry = A_(R._row(next_tab, R.T_REPN, x.ndim)), A_(R._row(next_tab, R.T_REPY, x.ndim))
            xn = torch.where(known, rn * noise + ry * y, xn)
        return out, d, xn
    z = torch.zeros((), dtype=torch.float64, device=y.device)
    ops = [R._d(a), z if b is None else R._d(b), R._d(y), R._d(noise), R._d(x), None if dp is None else R._d(dp)]
    val = expr(R._Val, *ops)
    mag = expr(R._Mag, *[None if o is None else o.abs() for o in ops])
    return {"out": (val[0], mag[0]), "d": (val[1], mag[1]), "x": (val[2], mag[2])}


def expect_kernel(c, shape):
    v4 = int(np.prod(shape[2:])) % 4 == 0
    return f"boundary_ge_kernel<{4 if v4 else 1},{DTYPES[c['dtype']]},{int(c['packed'])}>"


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
    if c["hist"]:
        ops["dp"] = torch.randn(shape, device=dev, generator=gen) * 2
    if c["combine"]:
        ops["b"] = (ops["a"].float() + 0.3 * torch.randn(shape, device=dev, generator=gen)).to(c["dtype"])
    if c["next"]:
        ops["table"] = A.table_rows(shape[0], dev, c["seed"])
    if c["out"]:
        ops["out"] = torch.full(shape, float("nan"), device=dev)
    if c["dout"]:
        ops["dout"] = torch.full(shape, float("nan"), device=dev)
    if c["packed"]:
        words = torch.zeros(int(lib.lp_known_words(total)), dtype=torch.int32, device=dev)
        yk, nk = torch.zeros(total + 4, device=dev), torch.zeros(total + 4, device=dev)
        assert lib.lp_pack_known(P(m8.data_ptr()), C.byref(dims), P(ops["y"].data_ptr()), P(ops["noise"].data_ptr()),
                                 P(words.data_ptr()), P(yk.data_ptr()), P(nk.data_ptr()), _stream()) == 0
        ops.update(words=words, y_known=yk, noise_known=nk)
    vals = FINAL if c["final"] else (STEP_GM if c.get("gamma") else STEP)
    step = nat.GradientEstimation(*vals, int(c["final"]))
    return ops, dims, step, known1.expand(shape)


def call_ge(c, t, dims, step, dead=False):
    """One lp_boundary_gradient_estimation call on the operands t (name -> tensor)."""
    nat, lib = _native(), _lib()
    p = lambda k: P(t[k].data_ptr()) if k in t else None   # noqa: E731
    cfg = 4.5 if c["combine"] else 0.0
    hd = nat.Heads(t["a"].data_ptr(), t["b"].data_ptr() if "b" in t else None,
                   LP_DT[c["dtype"]] | (nat.HEADS_DEAD if dead else 0), 1 if c["combine"] else 0, cfg, cfg)
    kn = nat.Known(t["words"].data_ptr(), t["y_known"].data_ptr(), t["noise_known"].data_ptr()) if c["packed"] else None
    return lib.lp_boundary_gradient_estimation(C.byref(hd), p("y"), p("noise"), p("mask"),
                                               C.byref(kn) if kn is not None else None, p("x"), p("out"), p("dout"),
                                               p("dp"), C.byref(step), p("table"), C.byref(dims), _stream())


BASE = dict(shape=(8, 4, 128, 128), dtype=F32, combine=False, next=True, out=True, dout=True, packed=True, hist=True,
            final=False, seed=1)
BIG = (16, 4, 128, 128)      # 2^20 elements: the smallest launch that walks tail-first with evict-first operands
R128 = (128, 4, 128, 128)
LAUNCHES = {
    "ge-f32-cfg-packed": dict(BASE, combine=True),
    "ge-f32-cfg-dense": dict(BASE, combine=True, packed=False, seed=2),
    "ge-bf16-packed-gamma": dict(BASE, dtype=BF16, gamma=True, seed=3),
    "first-f16-dense": dict(BASE, hist=False, dtype=F16, packed=False, seed=4),
    "final-noout-nod": dict(BASE, final=True, hist=False, next=False, out=False, dout=False, seed=5),
    "final-cfg-packed": dict(BASE, final=True, hist=False, next=False, combine=True, dout=False, seed=6),
    "ge-last-packed": dict(BASE, next=False, seed=7),
    "ge-last-bf16-dense-nod": dict(BASE, next=False, dtype=BF16, packed=False, dout=False, seed=8),
    "ge-f16-noout-dense": dict(BASE, dtype=F16, out=False, packed=False, seed=9),
    "ge-all-known": dict(BASE, mask="known", seed=10),
    "ge-all-known-last-dense": dict(BASE, mask="known", next=False, packed=False, seed=11),
    "ge-all-free-f16": dict(BASE, mask="free", dtype=F16, seed=12),
    "big-ge-f32-cfg-packed": dict(BASE, shape=BIG, combine=True, seed=13),
    "big-ge-bf16-dense": dict(BASE, shape=BIG, dtype=BF16, packed=False, seed=14),
    "big-final-f16-noout": dict(BASE, shape=BIG, final=True, hist=False, dtype=F16, next=False, out=False, dout=False,
                                seed=15),
    "r128-first-f32-packed": dict(BASE, shape=R128, hist=False, seed=16),
    "r128-ge-f32-packed": dict(BASE, shape=R128, seed=17),
    "r128-ge-bf16-dense-last": dict(BASE, shape=R128, dtype=BF16, packed=False, next=False, seed=18),
    "wan-ge-packed": dict(BASE, shape=(1, 16, 21, 80, 45), seed=19),
    "small-ge-cfg-dense": dict(BASE, shape=(1, 4, 32, 32), combine=True, packed=False, seed=20),
    "ragged-ge-packed": dict(BASE, shape=(1, 3, 7, 9), seed=21),
    "ragged-ge-dense-f16-last": dict(BASE, shape=(2, 3, 7, 9), packed=False, dtype=F16, next=False, seed=22),
    "ragged-first-bf16": dict(BASE, shape=(2, 3, 7, 9), hist=False, dtype=BF16, seed=23),
    "ragged-ge-cfg-noout-nod": dict(BASE, shape=(1, 3, 7, 9), combine=True, out=False, dout=False, packed=False,
                                    seed=24),
}


@pytest.mark.parametrize("case", list(LAUNCHES))
def test_launch_matches_fp64(case, cuda_device):
    c = LAUNCHES[case]
    ops, dims, step, known = make_case(c, cuda_device)
    want = ref_ge(ops["a"], ops.get("b"), ops["y"], ops["noise"], known, ops["x"], ops.get("dp"), step,
                  ops.get("table"), 4.5 if c["combine"] else None)
    fresh = lambda: dict(ops, **{k: ops[k].clone() for k in ("x", "out", "dout") if k in ops})   # noqa: E731
    t = fresh()
    kernels = A._launched(lambda: call_ge(c, t, dims, step))
    for _ in range(2):      # CUPTI can, rarely, deliver no record of a kernel that ran: launch again, same inputs
        if kernels:
            break
        t = fresh()
        kernels = A._launched(lambda: call_ge(c, t, dims, step))
    assert kernels == {expect_kernel(c, c["shape"])}, (case, kernels)
    worst, bad = R.within(t["x"], want["x"], K)
    assert bad is None, f"{case}: x element {bad}, worst ratio {worst:.3g} > K = {K}"
    if c["out"]:
        worst, bad = R.within(t["out"], want["out"], K)
        assert bad is None, f"{case}: out element {bad}, worst ratio {worst:.3g}"
        assert torch.equal(t["out"][known], ops["y"][known])
    if c["dout"]:     # every position, known ones included
        worst, bad = R.within(t["dout"], want["d"], K)
        assert bad is None, f"{case}: d_out element {bad}, worst ratio {worst:.3g}"
    if c["next"]:     # the replace step rounds as lp_prologue_f32 does
        xp = torch.zeros_like(t["x"])
        assert _lib().lp_prologue_f32(P(xp.data_ptr()), P(ops["y"].data_ptr()), P(ops["noise"].data_ptr()),
                                      P(ops["mask"].data_ptr()), P(xp.data_ptr()), None, P(ops["table"].data_ptr()),
                                      C.byref(dims), _stream()) == 0
        assert torch.equal(t["x"][known], xp[known])
    # the update in the sampler's own tensor ops (fp32 device tensors, one rounding each; ge_gamma - 1 a Python
    # float): bit for bit where no replace step follows, and d everywhere
    a = ops["a"].float()
    den = ops["b"].float() + (a - ops["b"].float()) * 4.5 if c["combine"] else a
    out = torch.where(known, ops["y"], den)
    s = lambda v: torch.tensor(v, dtype=torch.float32, device=cuda_device)   # noqa: E731
    d = (ops["x"] - out) / s(step.sigma)
    if step.final:
        eager = out
    else:
        eager = ops["x"] + d * s(step.dt)
        if c["hist"]:
            eager = eager + ((1.375 - 1 if c.get("gamma") else 2.0 - 1) * (d - ops["dp"])) * s(step.dt)
    sel = ~known if c["next"] else torch.ones_like(known)
    assert torch.equal(t["x"][sel], eager[sel]), case
    if c["dout"]:
        assert torch.equal(t["dout"], d), case


@pytest.mark.parametrize("case", ["ge-f32-cfg-packed", "big-ge-f32-cfg-packed", "big-ge-bf16-dense",
                                  "r128-ge-bf16-dense-last", "wan-ge-packed"])
def test_results_do_not_depend_on_dead_heads(case, cuda_device):
    """LP_HEADS_DEAD (128-byte aligned heads that no state, history or output overlaps: the launch drops their L2
    lines) gives the same x, out and d_out as the same launch without it."""
    c = LAUNCHES[case]
    ops, dims, step, _ = make_case(c, cuda_device)
    res = []
    for dead in (False, True):
        t = dict(ops, **{k: ops[k].clone() for k in ("x", "out", "dout", "a", "b") if k in ops})
        assert t["a"].data_ptr() % 128 == 0
        assert call_ge(c, t, dims, step, dead=dead) == 0
        torch.cuda.synchronize()
        res.append([t[k] for k in ("x", "out", "dout") if k in t])
    assert all(torch.equal(u, v) for u, v in zip(*res)), case


GUARDED = {
    "ge-f32-cfg-packed": dict(LAUNCHES["ge-f32-cfg-packed"], off=0),
    "ge-f32-cfg-dense": dict(LAUNCHES["ge-f32-cfg-dense"], off=0),
    "ge-last-packed": dict(LAUNCHES["ge-last-packed"], off=0),
    "first-f16-dense": dict(LAUNCHES["first-f16-dense"], off=0),
    "final-cfg-packed": dict(LAUNCHES["final-cfg-packed"], off=0),
    "big-ge-bf16-dense": dict(LAUNCHES["big-ge-bf16-dense"], off=0),
    "big-final-f16-noout": dict(LAUNCHES["big-final-f16-noout"], off=0),
    "r128-ge-f32-packed": dict(LAUNCHES["r128-ge-f32-packed"], off=0),
    "wan-ge-packed": dict(LAUNCHES["wan-ge-packed"], off=0),
    "ragged-ge-packed-misaligned": dict(LAUNCHES["ragged-ge-packed"], off=4),
    "ragged-ge-dense-f16-last-misaligned": dict(LAUNCHES["ragged-ge-dense-f16-last"], off=4),
}
SLACK = {"y_known": 4, "noise_known": 4}


@pytest.mark.parametrize("case", list(GUARDED))
def test_guarded_operands(case, cuda_device):
    """Every operand between guard bands (tests/_guard.py): x, out and d_out bit-identical to the plain call's, the
    bands intact, the history d_prev, the heads and every other input unchanged."""
    c = GUARDED[case]
    dev = cuda_device
    ops, dims, step, _ = make_case(c, dev)
    for k in ("out", "dout"):
        if k in ops:
            ops[k] = torch.zeros_like(ops[k])
    written = {"x"} | ({"out"} if c["out"] else set()) | ({"dout"} if c["dout"] else set())
    offs = {k: (c["off"] if k in ("x", "y", "noise", "out", "dout", "dp") else 0) for k in ops}
    plain = {k: G.plain(v, offs[k], SLACK.get(k, 0)) for k, v in ops.items()}
    arena = G.Arena(dev)
    guarded = {k: arena.place(v, offset_bytes=offs[k], slack=SLACK.get(k, 0), name=k) for k, v in ops.items()}
    arena.snapshot()
    assert call_ge(c, plain, dims, step) == 0
    assert call_ge(c, guarded, dims, step) == 0
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
        (out,) = N.LanPaint_KSampler().sample(patcher, seed, c["steps"], c["cfg"], "gradient_estimation", "karras", POS, NEG,
                                              latent, 1.0, c["n"], "Image First", "", N.IMAGE_MODE)
    else:
        start, end, leftover = c["window"]
        (out,) = N.LanPaint_KSamplerAdvanced().sample(
            patcher, "enable", seed, c["steps"], c["cfg"], "gradient_estimation", "karras", POS, NEG, latent, start, end,
            "enable" if leftover else "disable", c["n"], 5.0, 0.2, "Image First", "", N.IMAGE_MODE)
    return out["samples"]


def _whole_sampler_call(fn, k):
    """A node call with "fused_sampler" off.  The whole-sampler graph hands the sampler the schedule as a CPU tensor,
    and sample_gradient_estimation divides by append_dims(sigma) -- a [1, 1, 1, 1] CPU tensor, not a 0-d one -- so its
    capture fails on the second call and the configuration falls back to one graph per wrapper call (the per-sigma
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
    sig = J.ksampler_sigmas(fused, c["steps"], "gradient_estimation", "karras", 1.0, **window)
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
            assert bnd == {"boundary_ge_kernel<4,float,1>"}, bnd
        else:
            got = _node_call(N, fused, c, latent, seed)
        modes.append(N.LAST_RUN["mode"])
        assert N.LAST_RUN["fused"] and N.LAST_RUN["job"].sampler == "gradient_estimation"
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
        want = J.job(J._plain(minicomfy.sample_gradient_estimation), model, yd, noise.to(dev, torch.float64), dm, sig, hp,
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
    bit-equal to gradient_estimation_inpaint, with the generator left where the definition leaves it.  Per-step graphs
    are also captured last step first."""
    from lanpaint_b200.runner import GraphedJob, HostSchedule, gradient_estimation_inpaint, karras_sigmas
    dev = cuda_device
    ks = karras_sigmas(8)
    sched = HostSchedule(ks if sigmas == "to-zero" else ks[1:-2], shape[0], 4, early_stop=2)
    g = torch.Generator().manual_seed(9)
    y, noise = torch.randn(shape, generator=g).to(dev), torch.randn(shape, generator=g).to(dev)
    mask = (torch.rand((shape[0], 1) + shape[2:], generator=g) < 0.5).float().to(dev)
    gen = A._generator(dev)
    engine = lambda: A._engine(rng)      # noqa: E731
    torch.cuda.manual_seed(31)
    want = gradient_estimation_inpaint(engine(), y, noise, mask, sched)
    offset = gen.get_offset()
    n = len(sched.steps)
    for fused in (True, False):
        job = GraphedJob(engine(), sched, shape, dev, fused_euler=fused, sampler="gradient_estimation")
        assert bool(job.ge[-1][0].final) == (sigmas == "to-zero") and not job.ge[0][1] and job.ge[1][1]
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
    job = GraphedJob(engine(), sched, shape, dev, sampler="gradient_estimation")
    job.load_inputs(y, noise, mask)
    for i in reversed(range(n)):
        job._graph_for(("step", i, False), lambda p, i=i: job._step(i, p, False), True)
    torch.cuda.manual_seed(31)
    assert torch.equal(job.run(y, noise, mask, mode="steps"), want)


# ---------------------------------------------------------------------------------------------------------------
# 4. routing
# ---------------------------------------------------------------------------------------------------------------
def test_routing_and_cache_separation(cuda_device):
    """gradient_estimation takes the fused loop by default; {"fused_sampler": False} turns it off; a zero noise image
    (add_noise = disable) stays on its route; euler and gradient_estimation on one configuration never share a job."""
    from lanpaint_b200 import comfy_nodes as N
    N._ENGINES.clear()
    dev, shape = cuda_device, (2, 4, 64, 64)
    base = minicomfy.BaseModel(mixing_denoiser, model_type=minicomfy.ModelType.EPS, latent_channels=4, shift=1.0)
    g = torch.Generator().manual_seed(3)
    latent = {"samples": torch.randn(shape, generator=g), "noise_mask": (torch.rand((2, 1, 64, 64), generator=g) < 0.5).float()}

    def run(patcher, sampler="gradient_estimation"):
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
        assert ("boundary_ge_kernel<4,float,1>" in kernels) == fused, kernels
        if not fused:
            assert not any(k.startswith("boundary_ge") for k in kernels), kernels
    # None and {"fused_sampler": True} are two configurations: each starts eager; with the option off (and the
    # whole-sampler graph off) the per-sigma route runs
    assert [m for _, m, _, _ in seen] == ["eager", None, "job", "eager", None, "job"]
    # the per-sigma route bit for bit
    assert all(torch.equal(seen[0][0], seen[k][0]) for k in (1, 2, 3, 4, 5))
    assert seen[0][3] is seen[2][3] is seen[5][3] and seen[0][3].sampler == "gradient_estimation"
    assert seen[3][3] is not seen[0][3] and seen[3][3].sampler == "gradient_estimation"
    out_e, mode_e, fused_e, job_e, _ = run(patcher, "euler")
    assert fused_e and job_e is not seen[0][3] and job_e.sampler == "euler" and mode_e == "eager"
    assert not torch.equal(out_e, seen[0][0])
    assert run(patcher)[3] is seen[0][3]
    # add_noise = disable: a zero noise image, regenerated at every outer step by the per-sigma route
    torch.cuda.manual_seed(1)
    N.LanPaint_KSamplerAdvanced().sample(patcher, "disable", 5, 8, 4.0, "gradient_estimation", "karras", POS, NEG, latent, 0,
                                         10000, "disable", 3, 5.0, 0.2, "Image First", "", N.IMAGE_MODE)
    assert not N.LAST_RUN["fused"]
    N._ENGINES.clear()


def test_gate(cuda_device):
    from lanpaint_b200 import comfy_nodes as N
    from lanpaint_b200.engine import LanPaint

    class K:    # what _fused_gradient_estimation_ok reads of the wrapper
        audio_indicator = None
        sigmas_host = [3.0, 1.0, 0.0]
    ks = minicomfy.ksampler("gradient_estimation")
    eng = LanPaint(None, NSteps=3, Friction=15.0, Lambda=5.0, Beta=1.0, StepSize=0.2, rng="torch")
    dm = torch.ones(1)
    ok = lambda k=K, e=eng, mo={}, s=ks: N.KSAMPLER._fused_gradient_estimation_ok(s, k, dm, mo, e)   # noqa: E731
    assert ok()
    assert not N.KSAMPLER._fused_gradient_estimation_ok(ks, K, None, {}, eng)
    assert not ok(k=type("AV", (K,), {"audio_indicator": torch.ones(1)}))
    assert not ok(mo={"denoise_mask_function": lambda *a, **k: None})
    assert not ok(mo={"callback": lambda *a: None})
    assert not ok(mo={"lanpaint_semantic_stop": {}})
    assert not ok(e=LanPaint(None, NSteps=3, Friction=15.0, Lambda=5.0, Beta=1.0, StepSize=0.2, rng="torch",
                             EarlyStopThreshold=1e-3))
    assert not ok(s=minicomfy.ksampler("euler")) and not ok(s=minicomfy.ksampler("dpm_2"))
    assert not ok(s=minicomfy.ksampler("gradient_estimation", {"ge_gamma": 3.0}))
    assert not ok(k=type("Z", (K,), {"sigmas_host": [3.0, 0.0, 0.0]}))

    def sample_gradient_estimation(model, x, sigmas, **kw):     # the name, but not the sampler's form
        return x
    assert not ok(s=minicomfy.KSAMPLER(sample_gradient_estimation))
