"""Dead heads (LP_HEADS_DEAD): the update kernels may drop the network's outputs from the L2 unwritten once read.

(a) the jobs that set the flag -- runner.GraphedJob, runner.SamplerGraphJob, the node call -- give bit-identical
    results with the flag honoured and ignored, eager -> capture -> replay, at R = 8 and R = 128 (tail-first walk),
    for fp32 (CFG pair) and bf16 heads;
(b) the routes that must not set it -- an eager engine call, the per-sigma graphs -- leave the heads holding exactly
    what the network wrote;
(c) a discard never reaches past a head: both guard bands of every head are rewritten right before the flagged launch
    (so they are dirty in the L2, where a stray discard would drop the new bytes) and must read back the new bytes,
    on aligned and misaligned heads, partial last tiles / warps and aliased heads."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

P = C.c_void_p


def _lib():
    from lanpaint_b200 import _native
    return _native.load()


class _Net:
    """Guider stand-in over the bench's pointwise network: a CFG pair of fp32 outputs, or two heads of `dtype`.
    Remembers its last input and outputs, so that a test can recompute what the last call wrote."""

    def __init__(self, dtype=torch.float32):
        from lanpaint_b200.runner import SynthDenoiser, VESampling
        self.inner_model, self.model_sampling, self.dtype = self, VESampling(), dtype
        if dtype == torch.float32:
            self.nets = [SynthDenoiser(coef=(0.7, 0.1, c, 0.0, 0.0), two_heads=False) for c in (0.05, -0.05)]
        else:
            self.nets = [SynthDenoiser(coef=(0.7, 0.1, 0.02, 0.6, -0.05), dtype=dtype)]
        self.last = None

    def __call__(self, x, t, model_options=None, seed=None):
        from lanpaint_b200.engine import CfgPair
        if len(self.nets) == 2:
            out = CfgPair(self.nets[0](x, t), self.nets[1](x, t), 5.0, 3.0)
            heads = (out.cond, out.uncond)
        else:
            out = self.nets[0](x, t)
            heads = out
        self.last = (x.clone(), heads)
        return out

    def expected(self):
        """What the last call wrote, recomputed from its remembered input."""
        x, heads = self.last
        if len(self.nets) == 2:
            return [self.nets[k].__class__(coef=self.nets[k].coef, two_heads=False)(x, None).clone() for k in (0, 1)], heads
        want = self.nets[0].__class__(coef=self.nets[0].coef, dtype=self.dtype)(x, None)
        return [want[0].clone(), want[1].clone()], heads


def _inputs(shape, seed, dev):
    g = torch.Generator().manual_seed(seed)
    y = torch.randn(shape, generator=g).to(dev)
    noise = torch.randn(shape, generator=g).to(dev)
    known = (torch.rand((shape[0], 1) + shape[2:], generator=g) < 0.5).to(dev)
    return y, noise, known


def _engine(net):
    from lanpaint_b200.engine import LanPaint
    return LanPaint(net, NSteps=3, Friction=15.0, Lambda=5.0, Beta=1.0, StepSize=0.2, MinStepFrac=1.0, rng="torch")


KEEP = {"lanpaint_b200": {"discard_heads": False}}


@pytest.mark.parametrize("R", [8, 128])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32-cfg", "bf16"])
def test_graphed_job_same_with_and_without_discard(R, dtype, cuda_device):
    from lanpaint_b200.engine import heads_discardable, pack_mask
    from lanpaint_b200.runner import GraphedJob, HostSchedule, karras_sigmas
    dev = cuda_device
    shape = (R, 4, 128, 128)
    assert heads_discardable(None) and not heads_discardable(KEEP)
    outs = {}
    for opts in (None, KEEP):
        eng = _engine(_Net(dtype))
        job = GraphedJob(eng, HostSchedule(karras_sigmas(4), R, 3), shape, dev, model_options=opts)
        got = []
        for k, mode in enumerate(("eager", "job", "job")):   # eager, then capture + replay, then replay
            y, noise, known = _inputs(shape, 10 + k, dev)
            torch.cuda.manual_seed(300 + k)
            got.append(job.run(y, noise, pack_mask(known, y), mode=mode))
        torch.cuda.synchronize()
        outs[opts is None] = got
    for k, (a, b) in enumerate(zip(outs[True], outs[False])):
        assert torch.isfinite(a).all() and torch.equal(a, b), (R, dtype, k)


@pytest.mark.parametrize("sampler", ["euler", "heun"], ids=["graphed-job", "sampler-graph-job"])
@pytest.mark.parametrize("R", [8, 128])
def test_node_call_same_with_and_without_discard(R, sampler, cuda_device):
    """LanPaint_KSampler: euler runs as the node layer's GraphedJob, heun (a loop GraphedJob does not own) as its
    SamplerGraphJob; four calls of one request, from the first eager one to replays."""
    import minicomfy
    from _node_cases import NEG, POS, denoiser
    minicomfy.install()
    from lanpaint_b200 import comfy_nodes as N
    shape = (R, 4, 128, 128)
    g = torch.Generator().manual_seed(R)
    latent = {"samples": torch.randn(shape, generator=g),
              "noise_mask": (torch.rand((R, 1) + shape[2:], generator=g) < 0.5).float()}
    res = {}
    for discard in (True, False):
        N._ENGINES.clear()
        base = minicomfy.BaseModel(denoiser, model_type=minicomfy.ModelType.EPS, latent_channels=shape[1])
        patcher = minicomfy.ModelPatcher(base, cuda_device)
        patcher.model_options["lanpaint_b200"] = {"discard_heads": discard, "deferred_max_ms": 1e9}
        got = []
        for k in range(4):
            torch.cuda.manual_seed(50)
            (out,) = N.LanPaint_KSampler().sample(patcher, 7, 4, 5.0, sampler, "karras", POS, NEG, latent, 1.0, 3,
                                                  "Image First", "", N.IMAGE_MODE)
            got.append((out["samples"].clone(), N.LAST_RUN["mode"]))
        res[discard] = got
    N._ENGINES.clear()
    for k, ((a, ma), (b, mb)) in enumerate(zip(res[True], res[False])):
        assert ma == mb and torch.isfinite(a).all() and torch.equal(a, b), (R, sampler, k, ma, mb)
    assert res[True][-1][1] in ("job", "steps", "sampler-graph"), [m for _, m in res[True]]


@pytest.mark.parametrize("route", ["eager", "per-sigma-graphs"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32-cfg", "bf16"])
def test_routes_without_the_flag_keep_the_heads(route, dtype, cuda_device):
    """LanPaint.__call__ at the engine seam, eagerly and through its per-sigma CUDA graphs (eager -> capture ->
    replay): the heads of the last network call hold what the network wrote (R = 128: a discard would leave stale
    lines)."""
    from lanpaint_b200.runner import karras_sigmas, times_from_sigma
    dev = cuda_device
    shape = (128, 4, 128, 128)
    net = _Net(dtype)
    eng = _engine(net)
    eng.cuda_graph = route != "eager"
    y, noise, known = _inputs(shape, 3, dev)
    sig = karras_sigmas(4)
    for k in range(3):
        s = torch.full((shape[0],), sig[k], dtype=torch.float32)
        x = noise * sig[k] + y
        eng(x, y, noise, s, known.expand(shape).float(), times_from_sigma(s, False), None, 0, n_steps=3)
        torch.cuda.synchronize()
        want, heads = net.expected()
        for w, h in zip(want, heads):
            assert torch.equal(w, h), (route, dtype, k)


# ---- (c) guard bands -------------------------------------------------------------------------------------------
FRESH = 0x3C


def _refresh_bands(arena, names):
    """Rewrite both bands of the named operands with FRESH: they are then dirty lines in the L2."""
    for n in names:
        p = arena.ops[n]
        p.buf[:p.start].fill_(FRESH)
        p.buf[p.start + p.nbytes + p.slack_bytes:].fill_(FRESH)


def _bands_fresh(arena, names):
    for n in names:
        p = arena.ops[n]
        end = p.start + p.nbytes + p.slack_bytes
        assert bool((p.buf[:p.start] == FRESH).all()), (n, "front band lost its new bytes")
        assert bool((p.buf[end:] == FRESH).all()), (n, "back band lost its new bytes")


BIG = (5, 4, 120, 136)   # 326400 elements: TMA-staged kernels with partial tiles / a partial last torch group
CASES = {
    "torch-substep-cfg": dict(kernel="torch_substep", shape=BIG, dtype=torch.float32, combine=True),
    "torch-substep-aliased-bf16": dict(kernel="torch_substep", shape=BIG, dtype=torch.bfloat16, alias=True),
    "torch-substep-two-f32-r40": dict(kernel="torch_substep", shape=(40, 4, 128, 128), dtype=torch.float32),
    "philox-substep-cfg": dict(kernel="philox_substep", shape=BIG, dtype=torch.float32, combine=True),
    "philox-substep-aliased-bf16": dict(kernel="philox_substep", shape=BIG, dtype=torch.bfloat16, alias=True),
    "boundary-cfg": dict(kernel="boundary", shape=BIG, dtype=torch.float32, combine=True),
    "boundary-partial-warp-bf16": dict(kernel="boundary", shape=(1, 4, 100, 100), dtype=torch.bfloat16),
    "boundary-scalar-f32": dict(kernel="boundary", shape=(1, 3, 33, 35), dtype=torch.float32),
    "ancestral-cfg": dict(kernel="ancestral", shape=BIG, dtype=torch.float32, combine=True),
    "ancestral-bf16": dict(kernel="ancestral", shape=BIG, dtype=torch.bfloat16),
}


@pytest.mark.parametrize("offset", [0, 64, 16])
@pytest.mark.parametrize("case", list(CASES))
def test_discard_stays_inside_the_heads(case, offset, cuda_device):
    from lanpaint_b200 import _native
    from lanpaint_b200.engine import pack_known, pack_mask
    from lanpaint_b200.schedule import Hyper, build_table, times_from_sigma
    from _guard import Arena
    c = CASES[case]
    dev, shape, H = cuda_device, c["shape"], c["dtype"]
    if offset % torch.empty(0, dtype=H).element_size():
        pytest.skip("offset not a whole element")
    R = shape[0]
    per_row, spatial = shape[1] * shape[2] * shape[3], shape[2] * shape[3]
    g = torch.Generator().manual_seed(11)
    y, nz, x, cst = (torch.randn(shape, generator=g).to(dev) for _ in range(4))
    pm = pack_mask((torch.rand((R, 1) + shape[2:], generator=g) < 0.5).to(dev), y)
    dims = _native.Dims(R, per_row, spatial, pm.row_stride, pm.channel_stride)
    kn = pack_known(pm, dims, y, nz)
    s = torch.linspace(0.5, 3.0, R)
    ve, abt, _ = times_from_sigma(s, False)
    tab = torch.from_numpy(build_table(abt.numpy(), ve.numpy(), Hyper(0.2, 5.0, 1.0, 1.0, False))).to(dev)
    arena = Arena(dev)
    a = arena.place(torch.randn(shape, generator=g).to(dev, H), offset_bytes=offset, name="a")
    names = ["a"]
    b = a
    if not c.get("alias"):
        b = arena.place(torch.randn(shape, generator=g).to(dev, H), offset_bytes=offset, name="b")
        names.append("b")
    dt = {torch.float32: _native.DTYPE_F32, torch.bfloat16: _native.DTYPE_BF16}[H] | _native.HEADS_DEAD
    hd = _native.Heads(a.data_ptr(), b.data_ptr(), dt, 1 if c.get("combine") else 0, 4.5, 2.5)
    out = torch.empty_like(x)
    st = P(torch.cuda.current_stream().cuda_stream)
    r = _native.Rng()
    r.mode = _native.RNG_PHILOX if c["kernel"] == "philox_substep" else _native.RNG_TORCH
    r.seed, r.draw0, r.draw1 = 99, 4096, 8192
    lib = _lib()
    torch.cuda.synchronize()
    _refresh_bands(arena, names)
    if c["kernel"] == "torch_substep":
        rc = lib.lp_substep_known(P(x.data_ptr()), C.byref(hd), P(y.data_ptr()), P(pm.data.data_ptr()),
                                  C.byref(kn.struct), P(cst.data_ptr()), None, None, P(tab.data_ptr()), C.byref(dims),
                                  C.byref(r), _native.SUBSTEP_FUSE_NEXT, st)
    elif c["kernel"] == "philox_substep":
        rc = lib.lp_substep(P(x.data_ptr()), C.byref(hd), P(y.data_ptr()), P(pm.data.data_ptr()), P(cst.data_ptr()),
                            None, None, P(tab.data_ptr()), C.byref(dims), C.byref(r),
                            _native.SUBSTEP_FUSE_NEXT | _native.SUBSTEP_MERGE_NOISE, st)
    elif c["kernel"] == "boundary":
        rc = lib.lp_boundary_known(C.byref(hd), P(y.data_ptr()), P(nz.data_ptr()), P(pm.data.data_ptr()),
                                   C.byref(kn.struct), P(x.data_ptr()), P(out.data_ptr()), C.c_float(-0.2),
                                   P(tab.data_ptr()), C.byref(dims), st)
    else:
        step = _native.Ancestral(2.0, -0.3, 1.0, 0.5)
        rc = lib.lp_boundary_ancestral(C.byref(hd), P(y.data_ptr()), P(nz.data_ptr()), P(pm.data.data_ptr()),
                                       C.byref(kn.struct), P(x.data_ptr()), P(out.data_ptr()), C.byref(step),
                                       C.byref(r), P(tab.data_ptr()), C.byref(dims), st)
    _native.check(rc, case)
    torch.cuda.synchronize()
    _bands_fresh(arena, names)
    assert torch.isfinite(x).all(), case
