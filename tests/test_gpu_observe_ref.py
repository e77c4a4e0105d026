"""GPU: the row-bounded `out` of the step-boundary kernels, and what a deferred fused job keeps of each outer step's
denoised latent, for every fused sampler.

A. One launch of each row-bounded entry point (lp_boundary_{known,ancestral,midpoint,deis,gradient_estimation}_rows)
   against the per-sampler fp64 restatements of tests/test_gpu_sampler_*.py: the rows of `out` below the bound within
   K * 2^-24 * magnitude (out == y bit for bit at known positions), no byte past the bound written (guarded operands),
   every other result bit-identical to the unbounded call's, and the kernel asserted by name.  The cases cross head
   dtype, 4-wide / scalar vectors, dense / packed known operands, the CFG combine, next-step table / last step and the
   ancestral draw streams, on shapes whose row bound falls inside a TMA tile and a warp's span; a coverage test
   requires every instantiation the five entry points dispatch to among the launches with 0 < out_rows < n_rows.
B. Whole LanPaint_KSampler jobs of every fused sampler with ComfyUI's stock callback, run as "final" (no previewer),
   "preview" (the latent-to-RGB previewer) and "full" (the deferred_outputs option): the same samples, within 4e-6 of
   the fp64 job of tests/_job_ref.py, the previewer fed the "full" run's x0[:1] at every step, the last whole latent in
   x0_output and one progress tick per step."""
import ctypes as C

import numpy as np
import pytest
import torch

import _job_ref as J
import _launch_ref as R
import minicomfy
import test_gpu_sampler_ancestral as A
import test_gpu_sampler_deis as D
import test_gpu_sampler_dpm_2 as M
import test_gpu_sampler_gradient_estimation as G
from _guard import Arena, bits
from _node_cases import NEG, POS, mixing_denoiser
from oracle import langevin_oracle as O

pytestmark = pytest.mark.gpu

K = 8            # |out - fp64| <= K * 2^-24 * magnitude per element, as tests/test_gpu_launch_ref.py
JOB_B = 4e-6     # max|got - want| / max|want| of a whole job, as tests/test_gpu_job_ref.py
P = C.c_void_p
F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16
H_NAME = A.DTYPES
BIG = (5, 4, 120, 136)       # 326400 elements: TMA-eligible; rows of 65280 elements end inside a 2048-element tile
RAGGED = (3, 3, 7, 9)        # odd spatial size: the scalar kernels; rows end inside a warp's span
R128 = (128, 4, 128, 128)    # the preview launch itself, out_rows = 1
KIND_K = {"known": 8, "ancestral": A.K, "midpoint": M.K, "deis": D.K, "ge": G.K}   # x against fp64


def _native():
    from lanpaint_b200 import _native as n
    return n


# ---------------------------------------------------------------------------------------------------------------
# A. one launch of each row-bounded entry point
# ---------------------------------------------------------------------------------------------------------------
def _v4(shape):
    return int(np.prod(shape[2:])) % 4 == 0


def expect_kernel(c):
    shape = c["shape"]
    total, sp = int(np.prod(shape)), int(np.prod(shape[2:]))
    H, cb, nx = H_NAME[c["dtype"]], int(c["combine"]), int(c["next"])
    if c["kind"] == "known":     # tests/test_gpu_launch_ref.py's expect_boundary; the known layout is always packed
        if c.get("tma_boundary") and _v4(shape) and sp % 16 == 0 and total >= A.TMA_MIN:
            return f"boundary_tma_kernel<{H},{cb},{nx},2048,2>"
        return f"boundary_kernel<{4 if _v4(shape) else 1},{H},1>"
    if c["kind"] == "ancestral":
        return A.expect_kernel(c, total, sp)
    return {"midpoint": M, "deis": D, "ge": G}[c["kind"]].expect_kernel(c, shape)


def all_kernels():
    """Every instantiation the five entry points can dispatch to (the expect_kernel functions' range)."""
    names = set()
    for H in (F32, BF16, F16):
        h = H_NAME[H]
        for n in (4, 1):
            names.add(f"boundary_kernel<{n},{h},1>")
            for pk in (0, 1):
                for kind in ("midpoint", "deis", "ge"):
                    names.add(f"boundary_{kind}_kernel<{n},{h},{pk}>")
                for rng in (-1, 0, 1, 2):
                    names.add(f"boundary_ancestral_kernel<{n},{h},{pk},{rng}>")
        for cb in ((0, 1) if H == F32 else (0,)):     # the CFG combine takes fp32 heads
            for nx in (0, 1):
                names.add(f"boundary_tma_kernel<{h},{cb},{nx},2048,2>")
                for pk in (0, 1):
                    names.add(f"boundary_ancestral_torch_tma_kernel<{h},{cb},{nx},{pk}>")
    return names


def _cases():
    """Crossings, not the full product: one launch per instantiation with the bound inside the tensor (out_rows
    alternating between 1 and n_rows - 1, the combine and the next-step table alternating), then the bound's edges
    (0, n_rows, n_rows + 3) on one launch per family, then the R = 128 preview launches."""
    cases, k = {}, [0]

    def add(name, **c):
        c.setdefault("seed", 100 + k[0])
        c.setdefault("packed", True)
        R_ = c["shape"][0]
        if "out_rows" not in c:
            c["out_rows"] = 1 if k[0] % 2 == 0 else R_ - 1
        if "combine" not in c:
            c["combine"] = c["dtype"] == F32 and k[0] % 3 != 1
        if "next" not in c:
            c["next"] = k[0] % 4 != 3
        c["out"] = True
        k[0] += 1
        cases[name] = c

    dts = {"f32": F32, "bf16": BF16, "f16": F16}
    for dn, dt in dts.items():
        for vn, shape in (("v4", BIG), ("scalar", RAGGED)):
            add(f"known-{vn}-{dn}", kind="known", shape=shape, dtype=dt)
            for pk in (0, 1):
                pn = "packed" if pk else "dense"
                role = "corrector" if pk else "predictor"
                add(f"midpoint-{role}-{vn}-{dn}-{pn}", kind="midpoint", shape=shape, dtype=dt, packed=bool(pk),
                    role=role)
                add(f"deis-{vn}-{dn}-{pn}", kind="deis", shape=shape, dtype=dt, packed=bool(pk), order=3)
                add(f"ge-{vn}-{dn}-{pn}", kind="ge", shape=shape, dtype=dt, packed=bool(pk), hist=True, final=False)
                for rng in ("none", "tape", "philox", "torch"):
                    add(f"ancestral-ldg-{rng}-{vn}-{dn}-{pn}", kind="ancestral", shape=shape, dtype=dt, packed=bool(pk),
                        rng=rng, tma=0, eta0=rng == "none")
        for cb in ((False, True) if dt == F32 else (False,)):
            for nx in (False, True):
                cn = ("cfg-" if cb else "") + ("next" if nx else "last")
                add(f"known-tma-{cn}-{dn}", kind="known", shape=BIG, dtype=dt, combine=cb, next=nx, tma_boundary=1)
                for pk in (0, 1):
                    add(f"ancestral-torch-tma-{cn}-{dn}-{'packed' if pk else 'dense'}", kind="ancestral", shape=BIG,
                        dtype=dt, combine=cb, next=nx, packed=bool(pk), rng="torch")
    mid = dict(cases)
    edges = {"known-v4-f32": "known-ldg", "known-tma-cfg-next-f32": "known-tma",
             "ancestral-torch-tma-cfg-next-f32-packed": "ancestral-torch-tma",
             "ancestral-ldg-philox-scalar-bf16-dense": "ancestral-philox-scalar",
             "midpoint-corrector-v4-bf16-packed": "midpoint", "deis-scalar-f16-dense": "deis",
             "ge-v4-f32-packed": "ge"}
    for src, name in edges.items():
        c = mid[src]
        for rows in (0, c["shape"][0], c["shape"][0] + 3):
            add(f"edge-{name}-rows{rows}", **dict(c, out_rows=rows, seed=300 + k[0]))
    for name, c in {"known": dict(kind="known"), "ancestral-torch-tma": dict(kind="ancestral", rng="torch"),
                    "midpoint": dict(kind="midpoint", role="predictor"), "deis": dict(kind="deis", order=3),
                    "ge": dict(kind="ge", hist=True, final=False)}.items():
        add(f"preview-r128-{name}", shape=R128, dtype=F32, combine=True, next=True, out_rows=1, **c)
    return cases, set(mid)


CASES, MID = _cases()
RAN, WORST = set(), {}


def _operands(c, dev):
    """-> (operands dict, dims, step, rng struct, known bool tensor, draws xi of the ancestral step or None)."""
    nat, lib = _native(), A._lib()
    shape = c["shape"]
    total, sp = int(np.prod(shape)), int(np.prod(shape[2:]))
    gen = torch.Generator(device=dev).manual_seed(c["seed"])
    known1 = torch.rand((shape[0], 1) + tuple(shape[2:]), device=dev, generator=gen) < 0.5
    m8 = known1.to(torch.uint8).contiguous()
    dims = nat.Dims(shape[0], total // shape[0], sp, sp, 0, 0)
    t = {"x": torch.randn(shape, device=dev, generator=gen) * 3, "y": torch.randn(shape, device=dev, generator=gen),
         "noise": torch.randn(shape, device=dev, generator=gen), "mask": m8,
         "a": (torch.randn(shape, device=dev, generator=gen) * 1.5).to(c["dtype"])}
    if c["combine"]:
        t["b"] = (t["a"].float() + 0.3 * torch.randn(shape, device=dev, generator=gen)).to(c["dtype"])
    if c["next"]:
        t["table"] = A.table_rows(shape[0], dev, c["seed"])
    if c["packed"]:
        words = torch.zeros(int(lib.lp_known_words(total)), dtype=torch.int32, device=dev)
        yk, nk = torch.zeros(total + 4, device=dev), torch.zeros(total + 4, device=dev)
        assert lib.lp_pack_known(P(m8.data_ptr()), C.byref(dims), P(t["y"].data_ptr()), P(t["noise"].data_ptr()),
                                 P(words.data_ptr()), P(yk.data_ptr()), P(nk.data_ptr()), A._stream()) == 0
        t.update(words=words, y_known=yk, noise_known=nk)
    kind, step, r, xi = c["kind"], None, None, None
    if kind == "known":
        step = -0.37                 # the Euler coefficient
    elif kind == "midpoint":
        t["x2"] = (t["x"] + 0.5 * torch.randn(shape, device=dev, generator=gen) if c["role"] == "corrector"
                   else torch.full(shape, float("nan"), device=dev))
        step = nat.Midpoint(*M.STEPS[c["role"]])
    elif kind == "deis":
        t["p1"] = torch.randn(shape, device=dev, generator=gen) * 2
        t["p2"] = torch.randn(shape, device=dev, generator=gen) * 2
        t["d_out"] = torch.full(shape, float("nan"), device=dev)
        step = nat.Deis(*D.STEPS[3])
    elif kind == "ge":
        t["p1"] = torch.randn(shape, device=dev, generator=gen) * 2
        t["d_out"] = torch.full(shape, float("nan"), device=dev)
        step = nat.GradientEstimation(*G.STEP, 0)
    else:
        step = nat.Ancestral(1.7, -0.4375 * 1.1, 0.9, 0.0 if c.get("eta0") else 0.6)
        seed = c["seed"] * 7919 + 3
        if c["rng"] != "none":
            r = nat.Rng()
        if c["rng"] == "tape":
            xi = torch.randn(shape, device=dev, generator=gen)
            t["tape"] = xi
            r.mode, r.tape0 = nat.RNG_TAPE, xi.data_ptr()
        elif c["rng"] == "philox":
            t["state"] = torch.tensor([seed, 11], dtype=torch.int64, device=dev)
            r.mode, r.seed, r.draw0, r.state = nat.RNG_PHILOX, 0, 5, t["state"].data_ptr()
        elif c["rng"] == "torch":
            g = torch.Generator(device=dev).manual_seed(seed)
            g.set_offset(4 * 37)
            xi = torch.randn(shape, device=dev, generator=g)
            t["state"] = torch.tensor([seed, 4 * 37], dtype=torch.int64, device=dev)
            r.mode, r.seed, r.draw0, r.state = nat.RNG_TORCH, 0, 0, t["state"].data_ptr()
    return t, dims, step, r, known1.expand(shape), xi


def _reference(c, t, step, known, xi):
    """The per-sampler fp64 restatement -> dict of (value, magnitude) pairs with "out" and "x" (and "d")."""
    cfg = 4.5 if c["combine"] else None
    a, b, y, nz, x = t["a"], t.get("b"), t["y"], t["noise"], t["x"]
    tab = t.get("table")
    if c["kind"] == "known":
        return R.boundary(a, b, y, nz if c["next"] else None, known, x, step, tab, cfg=cfg)
    if c["kind"] == "ancestral":
        return A.ref_ancestral(a, b, y, nz, known, x, step, xi, tab, cfg)
    if c["kind"] == "midpoint":
        xin, xbase, _ = M.ROLES[c["role"]]
        return M.ref_midpoint(a, b, y, nz, known, t[xin], t[xbase], step, tab, cfg)
    if c["kind"] == "deis":
        return D.ref_deis(a, b, y, nz, known, x, t["p1"], t["p2"], step, 3, tab, cfg)
    return G.ref_ge(a, b, y, nz, known, x, t["p1"], step, tab, cfg)


def _call(c, t, dims, step, r, out, out_rows):
    """One call of case c's entry point on the operands t; out_rows None: the unbounded entry point."""
    nat, lib = _native(), A._lib()
    p = lambda k: P(t[k].data_ptr()) if k in t else None   # noqa: E731
    cfg = 4.5 if c["combine"] else 0.0
    hd = nat.Heads(t["a"].data_ptr(), t["b"].data_ptr() if "b" in t else None, A.LP_DT[c["dtype"]],
                   1 if c["combine"] else 0, cfg, cfg)
    kn = nat.Known(t["words"].data_ptr(), t["y_known"].data_ptr(), t["noise_known"].data_ptr()) if c["packed"] else None
    common = (C.byref(hd), p("y"), p("noise"), p("mask"), C.byref(kn) if kn is not None else None)
    tail = (p("table"), C.byref(dims), A._stream())
    o = P(out.data_ptr()) if out is not None else None
    ex, sfx = ((), "") if out_rows is None else ((C.c_int64(out_rows),), "_rows")
    kind = c["kind"]
    if kind == "known":
        return getattr(lib, "lp_boundary_known" + sfx)(*common, p("x"), o, *ex, C.c_float(step), *tail)
    if kind == "ancestral":
        return getattr(lib, "lp_boundary_ancestral" + sfx)(*common, p("x"), o, *ex, C.byref(step),
                                                          C.byref(r) if r is not None else None, *tail)
    if kind == "midpoint":
        xin, xbase, xout = M.ROLES[c["role"]]
        return getattr(lib, "lp_boundary_midpoint" + sfx)(*common, p(xin), p(xbase), p(xout), o, *ex, C.byref(step),
                                                         *tail)
    if kind == "deis":
        return getattr(lib, "lp_boundary_deis" + sfx)(*common, p("x"), o, *ex, p("d_out"), p("p1"), p("p2"),
                                                     C.byref(step), *tail)
    return getattr(lib, "lp_boundary_gradient_estimation" + sfx)(*common, p("x"), o, *ex, p("d_out"), p("p1"),
                                                                C.byref(step), *tail)


STATES = ("x", "x2", "d_out")    # what a launch writes besides out


@pytest.fixture
def options():
    lib = A._lib()
    yield lib
    lib.lp_set_option(b"tma", 1)
    lib.lp_set_option(b"tma_boundary", 0)


@pytest.mark.parametrize("case", list(CASES))
def test_rows_launch_matches_fp64(case, cuda_device, options):
    c = CASES[case]
    dev, shape = cuda_device, c["shape"]
    n_rows, rows = shape[0], c["out_rows"]
    held = min(rows, n_rows)
    assert options.lp_set_option(b"tma", c.get("tma", 1)) == 0
    assert options.lp_set_option(b"tma_boundary", c.get("tma_boundary", 0)) == 0
    t, dims, step, r, known, xi = _operands(c, dev)
    want = _reference(c, t, step, known, xi)
    init = {k: t[k].clone() for k in STATES if k in t}

    # the unbounded call on plain operands
    tu = dict(t, **{k: v.clone() for k, v in init.items()})
    out_u = torch.full(shape, float("nan"), device=dev)
    assert _call(c, tu, dims, step, r, out_u, None) == 0
    torch.cuda.synchronize()

    # the bounded call: `out` of exactly min(out_rows, n_rows) rows (one when none), the states between guard bands
    arena = Arena(dev)
    tb = dict(t, **{k: arena.place(v, name=k) for k, v in init.items()})
    out_b = arena.place(torch.full((max(held, 1),) + tuple(shape[1:]), float("nan"), device=dev), name="out")
    arena.snapshot()
    kernels = A._launched(lambda: _call(c, tb, dims, step, r, out_b, rows))
    for _ in range(2):      # CUPTI can, rarely, deliver no record of a kernel that ran: launch again, same inputs
        if kernels:
            break
        for k, v in init.items():
            tb[k].copy_(v)
        out_b.fill_(float("nan"))
        arena.snapshot()
        kernels = A._launched(lambda: _call(c, tb, dims, step, r, out_b, rows))
    written = (M.ROLES[c["role"]][2],) if c["kind"] == "midpoint" else tuple(k for k in ("x", "d_out") if k in init)
    arena.check(case, written=written + (("out",) if held else ()))
    assert kernels == {expect_kernel(c)}, (case, kernels, expect_kernel(c))

    # every other result is the unbounded call's, bit for bit
    for k in init:
        assert torch.equal(bits(tb[k]), bits(tu[k])), (case, k)
    # x against fp64 (the draw of the philox stream is the kernel's own: checked bit for bit above only)
    if not (c["kind"] == "ancestral" and c["rng"] == "philox"):
        xk = M.ROLES[c["role"]][2] if c["kind"] == "midpoint" else "x"
        worst, bad = R.within(tb[xk], want["x"], KIND_K[c["kind"]])
        assert bad is None, f"{case}: {xk} element {bad}, worst ratio {worst:.3g}"
    # the rows of out below the bound
    if held:
        val, mag = want["out"]
        worst, bad = R.within(out_b, (val[:held], mag[:held]), K)
        assert bad is None, f"{case}: out element {bad}, worst ratio {worst:.3g} > K = {K}"
        kn = known[:held]
        assert torch.equal(bits(out_b[kn]), bits(t["y"][:held][kn])), f"{case}: out != y at known positions"
        assert torch.equal(bits(out_b), bits(out_u[:held])), f"{case}: out differs from the unbounded call's"
        if case in MID:
            fam = expect_kernel(c).split("<")[0]
            WORST[fam] = max(WORST.get(fam, 0.0), worst)
    if case in MID:
        RAN.add(expect_kernel(c))


@pytest.mark.parametrize("kind", ["known", "ancestral", "midpoint", "deis", "ge"])
def test_out_of_out_rows_rows_next_to_a_state_is_accepted(kind, cuda_device, options):
    """`out` of exactly out_rows rows directly followed by the state the launch writes (x; midpoint's x_out; deis' and
    gradient estimation's d_out): a whole `out` there would overlap the state, which the unbounded entry point refuses
    where the launch does not let the two alias; the bounded call is accepted and computes the unbounded call's
    results."""
    base = [c for c in CASES.values() if c["kind"] == kind and c["shape"] == BIG and not c.get("tma_boundary")][0]
    c = dict(base, out_rows=2, seed=77)
    dev, shape = cuda_device, c["shape"]
    t, dims, step, r, known, xi = _operands(c, dev)
    state = M.ROLES[c["role"]][2] if kind == "midpoint" else {"deis": "d_out", "ge": "d_out"}.get(kind, "x")
    init = {k: t[k].clone() for k in STATES if k in t}
    tu = dict(t, **{k: v.clone() for k, v in init.items()})
    out_u = torch.full(shape, float("nan"), device=dev)
    assert _call(c, tu, dims, step, r, out_u, None) == 0

    per = int(np.prod(shape[1:]))
    buf = torch.full(((2 + shape[0]) * per,), float("nan"), device=dev)
    out = buf[:2 * per].view((2,) + tuple(shape[1:]))
    tb = dict(t, **{k: v.clone() for k, v in init.items()})
    tb[state] = buf[2 * per:].view(shape)
    tb[state].copy_(init[state])
    if kind in ("midpoint", "deis", "ge"):
        assert _call(c, tb, dims, step, r, out, shape[0]) == 1     # LP_ERR_INVALID: a whole out overlaps the state
        assert _call(c, tb, dims, step, r, out, 3) == 1
    assert _call(c, tb, dims, step, r, out, 2) == 0
    torch.cuda.synchronize()
    for k in init:
        assert torch.equal(bits(tb[k]), bits(tu[k])), (kind, k)
    assert torch.equal(bits(out), bits(out_u[:2])), kind


def test_rows_launches_cover_every_instantiation(cuda_device):
    """The launches with 0 < out_rows < n_rows ran every instantiation of the five entry points; the worst out ratio
    per kernel family is printed."""
    assert len(RAN) > 0, "run with the launch cases above"
    for fam, w in sorted(WORST.items()):
        print(f"{fam}: worst out ratio {w:.3g} (K = {K})")
    missing = sorted(all_kernels() - RAN)
    assert not missing, missing
    assert all(w <= K for w in WORST.values()), WORST


# ---------------------------------------------------------------------------------------------------------------
# B. whole node jobs under each setting
# ---------------------------------------------------------------------------------------------------------------
STEPS, N_INNER, CFG = 10, 3, 5.0
OPTIONS = {"euler_ancestral": {"fused_ancestral": True}, "heun": {"fused_heun": True}}
NODE_CASES = {f"{s}-b8": dict(sampler=s, shape=(8, 4, 64, 64), window=None)
              for s in ("euler", "euler_ancestral", "dpmpp_2m", "dpm_2", "deis", "res_multistep",
                        "gradient_estimation", "heun")}
NODE_CASES.update({f"{s}-r128": dict(sampler=s, shape=(128, 4, 64, 64), window=None)
                   for s in ("euler_ancestral", "heun", "res_multistep")})
NODE_CASES.update({f"{s}-window-leftover": dict(sampler=s, shape=(8, 4, 64, 64), window=(2, 8))
                   for s in ("heun", "res_multistep")})


def _node_run(c, dev, monkeypatch, latent, seed, option=None, previewer=None):
    """Two calls of one request (the eager job, then the deferred whole-job graph) with ComfyUI's stock callback:
    the second call's samples, mode, observe setting, x0_output dict, progress ticks and what the previewer saw."""
    from lanpaint_b200 import comfy_nodes as N
    N._ENGINES.clear()
    base = minicomfy.BaseModel(mixing_denoiser, model_type=minicomfy.ModelType.EPS, latent_channels=c["shape"][1])
    patcher = minicomfy.ModelPatcher(base, dev)
    patcher.model_options["lanpaint_b200"] = dict({"deferred_max_ms": 1e9}, **OPTIONS.get(c["sampler"], {}),
                                                  **(option or {}))
    store = {}
    monkeypatch.setitem(minicomfy.PREVIEW, "previewer", previewer)
    monkeypatch.setattr(minicomfy.prepare_callback, "__defaults__", (store,))
    for _ in range(2):
        if previewer is not None:
            previewer.seen = []
        calls0 = minicomfy.PROGRESS["calls"]
        torch.cuda.manual_seed(50)
        if c["window"] is None:
            (out,) = N.LanPaint_KSampler().sample(patcher, seed, STEPS, CFG, c["sampler"], "karras", POS, NEG, latent,
                                                  1.0, N_INNER, "Image First", "", N.IMAGE_MODE)
        else:
            start, end = c["window"]
            (out,) = N.LanPaint_KSamplerAdvanced().sample(
                patcher, "enable", seed, STEPS, CFG, c["sampler"], "karras", POS, NEG, latent, start, end, "enable",
                N_INNER, 5.0, 0.2, "Image First", "", N.IMAGE_MODE)
    torch.cuda.synchronize()
    job = N.LAST_RUN["job"]
    res = dict(samples=out["samples"].clone(), mode=N.LAST_RUN["mode"], fused=N.LAST_RUN["fused"],
               sampler=getattr(job, "sampler", None), observe=[k for k, v in job._outs.items() if v is job.outs],
               x0=store.get("x0"), calls=minicomfy.PROGRESS["calls"] - calls0, n_steps=len(job.sched.steps),
               seen=list(previewer.seen) if previewer is not None else None, patcher=patcher, base=base)
    N._ENGINES.clear()
    return res


@pytest.mark.parametrize("case", list(NODE_CASES))
def test_node_job_under_each_setting_matches_fp64(case, cuda_device, monkeypatch):
    c = NODE_CASES[case]
    dev, shape = cuda_device, c["shape"]
    minicomfy.install()
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    y = torch.randn(shape, generator=g)
    mask = (torch.rand((shape[0], 1) + shape[2:], generator=g) < 0.5).float()
    latent, seed = {"samples": y, "noise_mask": mask}, 7
    full = _node_run(c, dev, monkeypatch, latent, seed, option={"deferred_outputs": "full"},
                     previewer=minicomfy.Latent2RGBPreviewer())
    final = _node_run(c, dev, monkeypatch, latent, seed)
    preview = _node_run(c, dev, monkeypatch, latent, seed, previewer=minicomfy.Latent2RGBPreviewer())
    n = full["n_steps"]
    for name, r in (("full", full), ("final", final), ("preview", preview)):
        assert r["fused"] and r["sampler"] == c["sampler"], (name, r["fused"], r["sampler"])
        assert r["mode"] == "job" and r["observe"] == [name], (name, r["mode"], r["observe"])
        assert r["calls"] == n, (name, r["calls"], n)       # the progress bar: one tick per outer step
        assert torch.isfinite(r["samples"]).all() and torch.equal(r["samples"], full["samples"]), name
        assert r["x0"].shape == shape and torch.equal(r["x0"], full["x0"]), name    # the whole last latent
    assert len(full["seen"]) == len(preview["seen"]) == n
    for i, (a, b) in enumerate(zip(full["seen"], preview["seen"])):
        assert a.shape[0] == 1 and torch.equal(a, b), (case, i)
    assert torch.equal(full["seen"][-1], full["x0"][:1])

    # the fp64 job
    window = {} if c["window"] is None else dict(start_step=c["window"][0], last_step=c["window"][1])
    sig = J.ksampler_sigmas(full["patcher"], STEPS, c["sampler"], "karras", 1.0, **window)
    assert len(sig) - 1 == n
    base = full["base"]
    md = J.max_denoise(base.model_sampling, sig[0])
    hp = O.Hyper(n_steps=N_INNER, lam=5.0, step_size=0.2, min_step_frac=1.0, flow=False)
    torch.cuda.manual_seed(50)
    noise = minicomfy.prepare_noise(y, seed)
    dm = minicomfy.repeat_to_batch_size(mask, shape[0]).expand(shape).to(dev, torch.float64)
    steps = []
    model = J.Guider(mixing_denoiser, O.VESampling(), CFG, CFG)
    want = J.job(J.SAMPLERS[c["sampler"]], model, y.to(dev, torch.float64), noise.to(dev, torch.float64), dm, sig, hp,
                 max_denoise=md, callback=lambda i, d: steps.append(d))
    assert A._rel(full["samples"], want) <= JOB_B, (case, A._rel(full["samples"], want))
    assert A._rel(full["x0"], steps[-1]) <= JOB_B, (case, A._rel(full["x0"], steps[-1]))
    for i, (a, w) in enumerate(zip(full["seen"], steps)):
        assert A._rel(a, w[:1]) <= JOB_B, (case, i, A._rel(a, w[:1]))
