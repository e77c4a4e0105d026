"""GPU: no device entry point writes outside its outputs or into its inputs.

Every other GPU file hands the library ordinary torch tensors and looks only at the elements inside them; under
torch's caching allocator a store a few elements before or past an operand lands in a neighbour and fails nothing.
Here each case makes the same library call twice from the same seeded inputs: once on plain tensors, once with EVERY
pointer argument placed through the arena of tests/_guard.py (inputs included: heads, y, noise, mask, ring, tables,
tapes, the {seed, base} block, the known-operand layout, sums), each between two 64 KiB bands of a NaN pattern.  It
asserts
  * status LP_OK both times, the kernel the case was written for (by name, under torch.profiler), and the same
    kernel in both calls;
  * every output of the guarded call bit-identical to the plain call's -- with NaN bands around every input, an
    out-of-range read whose value reaches a result shows here;
  * arena.check with `written` = exactly the operands the header says the call writes for these flags: bands
    intact, every other operand (and the slack of y_known / noise_known) bit-identical to its snapshot.
Values against fp64 belong to test_gpu_launch_ref.py and test_gpu_sampler_ancestral.py, whose case format,
input builders and expected-kernel rules this file reuses.

The matrix is the edges: every kernel family on a FIRST launch that must leave C alone, a steady and a last launch;
the tail-first walk on and off (2^20 elements and below; option l2_handoff); partial work groups (Wan latent, plane
3600); total == tma_min == torch's T, the torch grid cap and one past it; scalar tails ((1, 3, 7, 9), (2, 4, 45, 45));
packed spans of length 0 and total; side outputs; every operand misaligned in turn; row splits; NULL out / x / next
table / rng; and the builders and fillers at sizes around their block, word and quad boundaries.
"""
import collections
import ctypes as C
import time

import numpy as np
import pytest
import torch
from torch.profiler import ProfilerActivity, profile

import _guard as G
import _launch_ref as R
import test_gpu_launch_ref as L
import test_gpu_sampler_ancestral as A
from _support import make_model, synth_inputs
from oracle import langevin_oracle as O

pytestmark = pytest.mark.gpu

P = C.c_void_p
F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16
DTYPES, LP_DT, TMA_MIN = L.DTYPES, L.LP_DT, L.TMA_MIN
WAN = (1, 16, 21, 80, 45)
BIG = (4, 4, 256, 256)        # 2^20 elements: the smallest launch that walks tail-first
SENTINEL = 0x5A5A5A5A         # what an output holds before the call, where the call need not write all of it

SEEN = collections.Counter()  # canonical kernel name -> guarded launches
RAN = set()
STATS = {"peak_bytes": 0, "seconds": 0.0}


@pytest.fixture(scope="module", autouse=True)
def _peak_memory_of_this_file(cuda_device):
    torch.zeros(1, device=cuda_device)      # the allocator's statistics exist once it has served a request
    torch.cuda.reset_peak_memory_stats(cuda_device)


def _nat():
    from lanpaint_b200 import _native
    return _native


def _lib():
    return _nat().load()


def _stream():
    return P(torch.cuda.current_stream().cuda_stream)


@pytest.fixture
def options():
    """The process-wide switches a case may set, restored whatever the case does."""
    lib = _lib()
    try:
        yield lib
    finally:
        lib.lp_set_option(b"tma", 1)
        lib.lp_set_option(b"tma_min", TMA_MIN)
        lib.lp_set_option(b"tma_boundary", 0)
        lib.lp_set_option(b"l2_handoff", 3)


def set_options(lib, c):
    assert lib.lp_set_option(b"tma", c.get("tma", 1)) == 0
    assert lib.lp_set_option(b"tma_min", c.get("tma_min", TMA_MIN)) == 0
    assert lib.lp_set_option(b"tma_boundary", c.get("tma_boundary", 0)) == 0
    assert lib.lp_set_option(b"l2_handoff", c.get("l2_handoff", 3)) == 0


class Op:
    """One pointer argument of a case: its contents before the call, its misalignment and its slack."""

    def __init__(self, t, off=0, slack=0):
        self.t, self.off, self.slack = t.contiguous(), off, slack


def launched(fn):
    """fn() (library calls, returning a status) under torch.profiler -> the set of canonical lp:: kernel names."""
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        time.sleep(0.005)
        rc = fn()
        torch.cuda.synchronize()
        time.sleep(0.005)
    assert rc == 0, f"status {rc}"
    return {R.canon(e.name()) for e in prof.profiler.kineto_results.events() if "lp::" in e.name()}


def run_guarded(cid, dev, ops, call, written, want, same=None):
    """The case's call on plain tensors, then on guarded ones.  ops: name -> Op; call(t) -> status, t: name -> tensor;
    written: the operands the call may write; same: those compared bit for bit with the plain call (default: all of
    written); want: the kernel name, or the set of names, the call launches.  -> (plain tensors, guarded, arena)."""
    t0 = time.perf_counter()
    same = written if same is None else same

    def once(t):
        got = launched(lambda: call(t))
        if not got:    # CUPTI can, rarely, deliver no record of a kernel that ran: once more from the same inputs
            for k in written:
                t[k].copy_(ops[k].t)
            got = launched(lambda: call(t))
        return got
    pl = {k: G.plain(o.t, o.off, o.slack) for k, o in ops.items()}
    k_plain = once(pl)
    arena = G.Arena(dev)
    gd = {k: arena.place(o.t, offset_bytes=o.off, slack=o.slack, name=k) for k, o in ops.items()}
    arena.snapshot()
    k_guard = once(gd)
    for k in sorted(same):
        if not torch.equal(G.bits(gd[k]), G.bits(pl[k])):
            d = int(torch.nonzero(G.bits(gd[k]) != G.bits(pl[k]))[0])
            pytest.fail(f"{cid}: output '{k}' of the guarded call differs from the plain call's at byte {d}")
    arena.check(cid, written=written)
    want = {want} if isinstance(want, str) else set(want)
    assert k_guard == want, (cid, k_guard, want)
    assert k_plain == k_guard, (cid, k_plain, k_guard)
    for n in k_guard:
        SEEN[n] += 1
    RAN.add(cid)
    STATS["peak_bytes"] = max(STATS["peak_bytes"], torch.cuda.max_memory_allocated(dev))
    STATS["seconds"] += time.perf_counter() - t0
    return pl, gd, arena


def _p(t, k):
    return P(t[k].data_ptr()) if k in t else None


def _known_ops(ops, m8, dims, total, with_noise):
    """The known-operand layout of the case's mask, y and noise as three more inputs (y_known / noise_known with the
    4 floats of slack the TMA-staged fetches may reach into)."""
    _, (words, yk, nk) = L.pack_known(m8, dims, ops["y"].t, ops["noise"].t if with_noise else None, total)
    ops["words"], ops["y_known"] = Op(words), Op(yk[:total], slack=4)
    if with_noise:
        ops["noise_known"] = Op(nk[:total], slack=4)


def _known_struct(t):
    return _nat().Known(t["words"].data_ptr(), t["y_known"].data_ptr(),
                        t["noise_known"].data_ptr() if "noise_known" in t else None)


# ---------------------------------------------------------------------------------------------------------------
# lp_substep / lp_substep_known (cases in the format of test_gpu_launch_ref.py)
# ---------------------------------------------------------------------------------------------------------------
def run_substep(c, dev, lib):
    nat = _nat()
    shape, flags, dt = c["shape"], c["flags"], c["dtype"]
    nxt, store, merge = bool(flags & 2), bool(flags & 4), bool(flags & 8)
    total = int(np.prod(shape))
    gen = torch.Generator(device=dev).manual_seed(c["seed"])
    m8, _, rs, cs = L.make_mask(shape, c["mask"], gen, dev)
    dims = L.dims_of(shape, rs, cs, c.get("split"))
    tab, _ = L.case_table(c, shape, dev)
    mis_op, mis_b = c.get("misalign", (None, 0))

    def rnd(scale=1.0):
        return torch.randn(shape, device=dev, generator=gen) * scale

    def off(k):
        return mis_b if mis_op == k else 0
    a32 = rnd(1.5)
    ops = {"x": Op(rnd(2.0), off("x")), "y": Op(rnd(), off("y")), "c": Op(rnd(3.0), off("c")),
           "a": Op(a32.to(dt), off("a")), "mask": Op(m8), "table": Op(tab)}
    if c["heads"] == "sep":
        ops["b"] = Op((a32 + 0.3 * rnd()).to(dt), off("b"))
    for k in ("x_copy", "x0e"):
        if c.get(k):
            ops[k] = Op(torch.zeros(shape, device=dev))
    mode, seed = c["rng"], c["seed"] * 7919 + 3
    if mode == "tape":
        ops["tape0"] = Op(rnd(), off("tape0"))
        if nxt and not merge:
            ops["tape1"] = Op(rnd())
    elif mode.endswith("_state"):
        ops["state"] = Op(torch.tensor([seed, 11 if mode.startswith("philox") else 4 * 37], dtype=torch.int64, device=dev))
    inc = L.torch_T(total)[1] if mode.startswith("torch") else 0
    if c.get("packed"):
        _known_ops(ops, m8, dims, total, False)
    cfg = c.get("cfg")

    def call(t):
        b = None if c["heads"] == "null" else t["b" if c["heads"] == "sep" else "a"].data_ptr()
        hd = nat.Heads(t["a"].data_ptr(), b, LP_DT[dt], 1 if cfg else 0, cfg[0] if cfg else 0.0, cfg[1] if cfg else 0.0)
        r = nat.Rng()
        if mode == "tape":
            r.mode, r.tape0 = nat.RNG_TAPE, t["tape0"].data_ptr()
            r.tape1 = t["tape1"].data_ptr() if "tape1" in t else None
        elif mode.startswith("philox"):
            r.mode, r.seed, r.draw0, r.draw1 = nat.RNG_PHILOX, seed, 5, 6
        else:
            r.mode, r.seed, r.draw0, r.draw1 = nat.RNG_TORCH, seed, 0, inc
        if "state" in t:
            r.seed, r.state = 0, t["state"].data_ptr()
        if c.get("packed"):
            kn = _known_struct(t)
            return lib.lp_substep_known(_p(t, "x"), C.byref(hd), _p(t, "y"), _p(t, "mask"), C.byref(kn), _p(t, "c"),
                                        _p(t, "x_copy"), _p(t, "x0e"), _p(t, "table"), C.byref(dims), C.byref(r),
                                        flags, _stream())
        return lib.lp_substep(_p(t, "x"), C.byref(hd), _p(t, "y"), _p(t, "mask"), _p(t, "c"), _p(t, "x_copy"),
                              _p(t, "x0e"), _p(t, "table"), C.byref(dims), C.byref(r), flags, _stream())
    written = {"x"} | ({"c"} if nxt or store else set()) | {k for k in ("x_copy", "x0e") if c.get(k)}
    want = L.expect_substep(c, shape, rs, cs)
    if "family" in c:
        assert L.family(want) == c["family"], (c["id"], want)
    run_guarded(c["id"], dev, ops, call, written, want)


def _substep_cases():
    S = dict(rng="torch", flags=2, dtype=F32, heads="sep", mask="rand", table="lam12")
    T = (1, 4, 256, 256)      # total == tma_min == torch's T
    dts, heads, masks = (F32, BF16, F16), ("sep", "null", "same"), ("rand", "full", "blob")
    fams = [("ldg4-tape", "tape", (1, 4, 128, 128), {}), ("ldg1-tape", "tape", (2, 4, 45, 45), {}),
            ("ldg4-philox", "philox", (1, 4, 128, 128), {}), ("ldg1-philox", "philox", (2, 4, 45, 45), {}),
            ("tma-philox", "philox", T, {}), ("torch-tma", "torch", T, {}), ("torch-tma-pk", "torch", T, {"packed": True}),
            ("torchvec", "torch", (40, 4, 50, 50), {}), ("torch-scalar", "torch", (2, 4, 45, 45), {})]
    cases, i = [], 0
    for name, rng, shape, extra in fams:
        # FIRST without STORE_C (C untouched), steady FUSE_NEXT, last (C read, not written), FIRST | FUSE_NEXT
        for flags in (1, 2, 0, 3) + ((2 | 8,) if rng == "philox" else ()):
            cases.append(dict(S, id=f"{name}-f{flags}", shape=shape, rng=rng, flags=flags, dtype=dts[i % 3],
                              heads=heads[(i // 3) % 3], mask=masks[i % 3], table=L.TABLES[i % 3], **extra))
            i += 1
    cases += [
        # 2^20 elements: the tail-first walk, on (default) and off
        dict(S, id="big-torch-tma-pk", shape=BIG, packed=True),
        dict(S, id="big-torch-tma-pk-walk-off", shape=BIG, packed=True, l2_handoff=0),
        dict(S, id="big-torch-tma-first-bf16", shape=BIG, flags=1, dtype=BF16, heads="null", table="dt"),
        dict(S, id="big-torch-tma-dense-walk-only", shape=BIG, flags=3, l2_handoff=1),
        dict(S, id="big-tma-philox-merge", shape=BIG, rng="philox", flags=2 | 8),
        dict(S, id="big-tma-philox-first-f16-walk-off", shape=BIG, rng="philox", flags=1, dtype=F16, l2_handoff=0),
        dict(S, id="big-ldg-tape", shape=BIG, rng="tape", flags=0 | 4),
        dict(S, id="flagship-pk", shape=(128, 4, 128, 128), packed=True),
        # partial work groups: the Wan latent (plane 3600, two calls per subsequence)
        dict(S, id="wan-pk", shape=WAN, packed=True),
        dict(S, id="wan-dense-first-f16", shape=WAN, flags=1, dtype=F16, mask="full"),
        dict(S, id="wan-philox-bf16", shape=WAN, rng="philox", flags=2, dtype=BF16, heads="null"),
        dict(S, id="wan-last-pk", shape=WAN, flags=0, packed=True, heads="same"),
        # the torch grid cap and one past it
        dict(S, id="gridcap-pk-state", shape=(1, 4, 264, 256), rng="torch_state", flags=1 | 4, packed=True, mask="full"),
        dict(S, id="gridcap-dense", shape=(1, 4, 264, 256), flags=1),
        dict(S, id="pastcap-pk", shape=(1, 4, 272, 256), flags=3, packed=True, dtype=BF16, heads="null"),
        dict(S, id="pastcap-dense-last", shape=(1, 4, 272, 256), flags=0, mask="blob"),
        # scalar tails
        dict(S, id="ragged-torch", shape=(1, 3, 7, 9), flags=3),
        dict(S, id="ragged-torch-first-f16", shape=(1, 3, 7, 9), flags=1, dtype=F16, heads="null"),
        dict(S, id="ragged-philox-merge", shape=(1, 3, 7, 9), rng="philox", flags=2 | 8),
        dict(S, id="ragged-tape-last-bf16", shape=(1, 3, 7, 9), rng="tape", flags=0, dtype=BF16),
        # packed spans of length 0 and total; a full-shape mask
        dict(S, id="T-allknown-pk", shape=T, mask="known", packed=True),
        dict(S, id="T-allfree-pk", shape=T, mask="free", packed=True, flags=3, heads="null"),
        dict(S, id="big-allknown-pk", shape=BIG, mask="known", packed=True, flags=1),
        dict(S, id="big-allfree-pk", shape=BIG, mask="free", packed=True),
        dict(S, id="T-full-pk-bf16", shape=T, mask="full", packed=True, dtype=BF16, flags=1 | 4),
        dict(S, id="rows-cfg-pk", shape=(5, 4, 120, 136), rng="torch_state", cfg=(7.0, 2.5), packed=True, mask="full"),
        dict(S, id="rows-cfg-philox-state", shape=(5, 4, 120, 136), rng="philox_state", flags=3, cfg=(4.5, -0.5), table="dt"),
        dict(S, id="rows-cfg-tape", shape=(5, 4, 120, 136), rng="tape", cfg=(4.5, -0.5)),
        dict(S, id="cfg-torchvec", shape=(40, 4, 50, 50), flags=1, cfg=(4.5, -0.5)),
        dict(S, id="cfg-ragged", shape=(2, 4, 45, 45), flags=0 | 4, cfg=(3.0, 1.0)),
        # side outputs (the early-stop loop's launches)
        dict(S, id="side-torch", shape=T, flags=1, x_copy=True, x0e=True),
        dict(S, id="side-torch-steady-bf16", shape=(5, 4, 120, 136), flags=0 | 4, dtype=BF16, heads="null", x0e=True),
        dict(S, id="side-philox", shape=(5, 4, 120, 136), rng="philox", flags=1, x0e=True, x_copy=True),
        dict(S, id="side-tape-scalar-f16", shape=(2, 4, 45, 45), rng="tape", flags=2, dtype=F16, mask="full",
             x0e=True, x_copy=True),
        dict(S, id="side-torch-scalar", shape=(1, 3, 7, 9), flags=0, x_copy=True),
    ]
    # each operand 4 bytes off in turn (scalar fallbacks), a 16-bit head by 8 (vec4, not TMA)
    for op in ("x", "y", "a", "b", "c"):
        cases.append(dict(S, id=f"misalign-{op}", shape=(5, 4, 120, 136), misalign=(op, 4), flags=1 if op == "c" else 2))
    cases += [
        dict(S, id="misalign-tape0", shape=(1, 4, 128, 128), rng="tape", flags=1 | 4, misalign=("tape0", 4)),
        dict(S, id="misalign-x-philox", shape=T, rng="philox", misalign=("x", 4)),
        dict(S, id="misalign-y-tape", shape=(1, 4, 128, 128), rng="tape", flags=0, misalign=("y", 4)),
        dict(S, id="misalign8-a-f16", shape=(5, 4, 120, 136), dtype=F16, misalign=("a", 8)),
        dict(S, id="misalign8-b-bf16-philox", shape=(5, 4, 120, 136), rng="philox", flags=3, dtype=BF16, mask="full",
             misalign=("b", 8)),
    ]
    # row splits (the audio-video flat pack): in the middle, not a multiple of 4, split == per_row
    i = 0
    for split in (3072, 3071, 4096):
        for rng in ("torch", "philox", "tape"):
            cases.append(dict(S, id=f"av-split{split}-{rng}", shape=(4, 1, 4096), split=split, rng=rng, tma_min=0,
                              flags=(1, 2, 0)[i % 3], dtype=dts[i % 3], heads=heads[i % 2], packed=rng == "torch"))
            i += 1
    cases += [
        dict(S, id="av-odd-torch", shape=(3, 1, 2049), split=1000, flags=3, tma_min=0),
        dict(S, id="av-one-odd-line-torch", shape=(1, 1, 2049), split=1000, flags=1, tma_min=0),
        dict(S, id="av-one-odd-line-tape", shape=(1, 1, 2049), split=1000, rng="tape", tma_min=0),
        dict(S, id="av-big-torch-pk", shape=(1, 1, 1 << 22), split=1 << 21, packed=True, tma_min=0),
        dict(S, id="av-big-philox-merge", shape=(1, 1, 1 << 22), split=(1 << 21) + 4, rng="philox", flags=2 | 8, tma_min=0),
    ]
    for i, c in enumerate(cases):
        c.setdefault("seed", 1500 + i)
    return cases


SUBSTEP_CASES = _substep_cases()


@pytest.mark.parametrize("c", SUBSTEP_CASES, ids=lambda c: c["id"])
def test_substep(c, cuda_device, options):
    set_options(options, c)
    run_substep(c, cuda_device, options)


# ---------------------------------------------------------------------------------------------------------------
# lp_boundary / lp_boundary_known and their special cases
# ---------------------------------------------------------------------------------------------------------------
def _boundary_cases():
    Bd = dict(dtype=F32, combine=None, next=True, out=True, euler=True, mask="rand", table="lam12")
    T = (1, 4, 256, 256)
    cases, i = [], 0
    for shape, tag in (((1, 4, 128, 128), "b4"), ((2, 4, 45, 45), "b1"), ((1, 3, 7, 9), "ragged")):
        for packed in (False, True):
            for dt in (F32, BF16, F16):
                cases.append(dict(Bd, id=f"{tag}-{'pk' if packed else 'dense'}-{DTYPES[dt]}", shape=shape, dtype=dt,
                                  packed=packed, next=i % 2 == 0, out=i % 3 != 1, mask=("rand", "full", "blob")[i % 3]))
                i += 1
    cases += [
        # both walks at 2^20 elements, LDG and TMA-staged
        dict(Bd, id="big-ldg-pk", shape=BIG, packed=True),
        dict(Bd, id="big-ldg-pk-walk-off", shape=BIG, packed=True, l2_handoff=0),
        dict(Bd, id="big-ldg-dense-bf16-noout", shape=BIG, dtype=BF16, out=False),
        dict(Bd, id="big-ldg-dense-walk-only", shape=BIG, combine=4.5, l2_handoff=1),
        dict(Bd, id="big-tma", shape=BIG, tma_boundary=1),
        dict(Bd, id="big-tma-walk-off-cfg", shape=BIG, tma_boundary=1, combine=4.5, l2_handoff=0, next=False),
        dict(Bd, id="big-tma-f16-noout", shape=BIG, tma_boundary=1, dtype=F16, out=False, mask="full"),
        dict(Bd, id="T-tma-bf16", shape=T, tma_boundary=1, dtype=BF16, next=False, mask="full"),
        dict(Bd, id="rows-tma-cfg-next", shape=(5, 4, 120, 136), tma_boundary=1, combine=4.5),
        dict(Bd, id="wan-tma", shape=WAN, tma_boundary=1),
        dict(Bd, id="wan-ldg-pk-f16", shape=WAN, packed=True, dtype=F16),
        dict(Bd, id="gridcap-tma-noout", shape=(1, 4, 264, 256), tma_boundary=1, out=False),
        dict(Bd, id="pastcap-tma", shape=(1, 4, 272, 256), tma_boundary=1, next=False),
        dict(Bd, id="flagship-pk-cfg", shape=(128, 4, 128, 128), packed=True, combine=5.0),
        dict(Bd, id="allknown-pk", shape=T, packed=True, mask="known"),
        dict(Bd, id="allfree-pk", shape=T, packed=True, mask="free"),
        dict(Bd, id="out-only", shape=(5, 4, 120, 136), combine=3.5, next=False, euler=False, mask="blob"),
        dict(Bd, id="out-only-pk-ragged", shape=(2, 4, 45, 45), packed=True, next=False, euler=False),
        dict(Bd, id="misalign-noise", shape=(1, 4, 128, 128), misalign="noise"),
        dict(Bd, id="av-vec4-dense", shape=(4, 1, 4096), split=3072, tma_boundary=1),
        dict(Bd, id="av-scalar-pk-cfg", shape=(4, 1, 4096), split=3071, packed=True, combine=3.5),
        dict(Bd, id="av-split-nlast-noout", shape=(4, 1, 4096), split=4096, out=False),
        dict(Bd, id="av-odd-f16", shape=(3, 1, 2049), split=1000, dtype=F16),
        dict(Bd, id="av-one-odd-line", shape=(1, 1, 2049), split=1000),
        # the special cases: NULL out, NULL x, NULL next table
        dict(Bd, id="epilogue", api="epilogue", shape=T, next=False, euler=False),
        dict(Bd, id="epilogue-ragged", api="epilogue", shape=(1, 3, 7, 9), next=False, euler=False),
        dict(Bd, id="epilogue-euler", api="epilogue_euler", shape=BIG, next=False),
        dict(Bd, id="epilogue-euler-noout-ragged", api="epilogue_euler", shape=(2, 4, 45, 45), next=False, out=False),
        dict(Bd, id="step-boundary", api="step_boundary", shape=BIG, mask="full"),
        dict(Bd, id="step-boundary-noout-tma", api="step_boundary", shape=T, out=False, tma_boundary=1),
        dict(Bd, id="step-boundary-ragged", api="step_boundary", shape=(1, 3, 7, 9)),
        dict(Bd, id="epilogue-cfg", api="epilogue_cfg", shape=BIG, combine=4.5, next=False),
        dict(Bd, id="epilogue-cfg-nox-ragged", api="epilogue_cfg", shape=(2, 4, 45, 45), combine=-0.5, next=False,
             euler=False),
    ]
    for i, c in enumerate(cases):
        c.setdefault("seed", 2500 + i)
    return cases


BOUNDARY_CASES = _boundary_cases()


@pytest.mark.parametrize("c", BOUNDARY_CASES, ids=lambda c: c["id"])
def test_boundary(c, cuda_device, options):
    nat, lib, dev = _nat(), options, cuda_device
    set_options(lib, c)
    shape, dt, cfg, api = c["shape"], c["dtype"], c["combine"], c.get("api")
    total = int(np.prod(shape))
    gen = torch.Generator(device=dev).manual_seed(c["seed"])
    m8, _, rs, cs = L.make_mask(shape, c["mask"], gen, dev)
    dims = L.dims_of(shape, rs, cs, c.get("split"))
    tab, _ = L.case_table(c, shape, dev)
    a, b, y, nz, x = (torch.randn(shape, device=dev, generator=gen) for _ in range(5))
    ops = {"a": Op(a.to(dt)), "y": Op(y), "mask": Op(m8)}
    if cfg is not None:
        ops["b"] = Op(b.to(dt))
    if c["next"]:
        ops["noise"], ops["table"] = Op(nz, 4 if c.get("misalign") == "noise" else 0), Op(tab)
    if c["euler"]:
        ops["x"] = Op(x)
    if c["out"]:
        ops["out"] = Op(torch.zeros(shape, device=dev))
    if c.get("packed"):
        _known_ops(ops, m8, dims, total, c["next"])
    coef = C.c_float(-0.37)

    def call(t):
        p = lambda k: _p(t, k)   # noqa: E731
        if api == "epilogue":
            return lib.lp_epilogue_f32(p("a"), p("y"), p("mask"), p("out"), C.byref(dims), _stream())
        if api == "epilogue_euler":
            return lib.lp_epilogue_euler_f32(p("a"), p("y"), p("mask"), p("x"), p("out"), coef, C.byref(dims), _stream())
        if api == "step_boundary":
            return lib.lp_step_boundary_f32(p("a"), p("y"), p("noise"), p("mask"), p("x"), p("out"), coef, p("table"),
                                            C.byref(dims), _stream())
        if api == "epilogue_cfg":
            return lib.lp_epilogue_cfg_f32(p("a"), p("b"), C.c_float(cfg), p("y"), p("mask"), p("x"), p("out"), coef,
                                           C.byref(dims), _stream())
        hd = nat.Heads(t["a"].data_ptr(), t["b"].data_ptr() if "b" in t else None, LP_DT[dt], 1 if cfg is not None else 0,
                       cfg or 0.0, cfg or 0.0)
        if c.get("packed"):
            kn = _known_struct(t)
            return lib.lp_boundary_known(C.byref(hd), p("y"), p("noise"), p("mask"), C.byref(kn), p("x"), p("out"), coef,
                                         p("table"), C.byref(dims), _stream())
        return lib.lp_boundary(C.byref(hd), p("y"), p("noise"), p("mask"), p("x"), p("out"), coef, p("table"),
                               C.byref(dims), _stream())
    written = {k for k in ("x", "out") if k in ops}
    run_guarded(c["id"], dev, ops, call, written, L.expect_boundary(c, shape, rs, cs))


# ---------------------------------------------------------------------------------------------------------------
# lp_boundary_ancestral (cases in the format of test_gpu_sampler_ancestral.py)
# ---------------------------------------------------------------------------------------------------------------
AB = dict(A.BASE)
ANCESTRAL_CASES = {
    "tma-pk-cfg-next": dict(AB, combine=True),
    "tma-dense-cfg-last": dict(AB, combine=True, next=False, packed=False),
    "tma-dense-bf16-noout": dict(AB, dtype=BF16, packed=False, out=False),
    "tma-pk-f16-last-noout": dict(AB, dtype=F16, next=False, out=False),
    "tma-pk-allknown": dict(AB, mask="known"),
    "tma-pk-allfree": dict(AB, mask="free", dtype=BF16),
    "tma-r128-pk": dict(AB, shape=(128, 4, 128, 128), combine=True),
    "tma-r128-dense-bf16-noout": dict(AB, shape=(128, 4, 128, 128), dtype=BF16, packed=False, out=False),
    "tma-big-pk-walk-off": dict(AB, shape=BIG, l2_handoff=0),
    "tma-wan-pk": dict(AB, shape=WAN),
    "tma-wan-dense-f16-last": dict(AB, shape=WAN, dtype=F16, packed=False, next=False),
    "tma-min-pk": dict(AB, shape=(1, 4, 256, 256)),
    "tma-min-dense": dict(AB, shape=(1, 4, 256, 256), packed=False),
    "ldg-torch-vec4-pk": dict(AB, shape=(1, 4, 32, 32)),
    "ldg-torch-vec4-dense-cfg": dict(AB, shape=(3, 4, 128, 128), packed=False, combine=True),
    "ldg-torch-vec4-r128-tma-off": dict(AB, shape=(128, 4, 128, 128), tma=0),
    "ldg-torch-ragged-pk": dict(AB, shape=(1, 3, 7, 9)),
    "ldg-torch-ragged-dense-f16-last": dict(AB, shape=(2, 3, 7, 9), packed=False, dtype=F16, next=False),
    "ldg-philox-big-pk": dict(AB, rng="philox", shape=BIG),
    "ldg-philox-ragged-dense": dict(AB, rng="philox", shape=(1, 3, 7, 9), packed=False),
    "ldg-tape-big-cfg-pk": dict(AB, rng="tape", shape=BIG, combine=True),
    "ldg-tape-dense-bf16": dict(AB, rng="tape", shape=(1, 4, 32, 32), packed=False, dtype=BF16),
    "ldg-tape-ragged-last": dict(AB, rng="tape", shape=(1, 3, 7, 9), next=False),
    "ldg-none-pk-last": dict(AB, rng="none", next=False, eta0=True),
    "ldg-none-r128-dense": dict(AB, rng="none", shape=(128, 4, 128, 128), packed=False, eta0=True),
    "ldg-none-ragged-noout": dict(AB, rng="none", shape=(1, 3, 7, 9), eta0=True, out=False),
}


@pytest.mark.parametrize("case", list(ANCESTRAL_CASES))
def test_boundary_ancestral(case, cuda_device, options):
    nat, lib, dev = _nat(), options, cuda_device
    c = dict(ANCESTRAL_CASES[case], seed=3000 + list(ANCESTRAL_CASES).index(case))
    set_options(lib, c)
    shape, dt = c["shape"], c["dtype"]
    total, sp = int(np.prod(shape)), int(np.prod(shape[2:]))
    gen = torch.Generator(device=dev).manual_seed(c["seed"])
    m8, _, rs, cs = L.make_mask(shape, c.get("mask", "rand"), gen, dev)
    dims = nat.Dims(shape[0], total // shape[0], sp, rs, cs, 0)
    a, b, y, nz, x, xi = (torch.randn(shape, device=dev, generator=gen) for _ in range(6))
    ops = {"a": Op(a.to(dt)), "y": Op(y), "noise": Op(nz), "mask": Op(m8), "x": Op(x * 3)}
    if c["combine"]:
        ops["b"] = Op(b.to(dt))
    if c["next"]:
        ops["table"] = Op(A.table_rows(shape[0], dev, c["seed"]))
    if c["out"]:
        ops["out"] = Op(torch.zeros(shape, device=dev))
    seed = c["seed"] * 7919 + 3
    if c["rng"] == "tape":
        ops["tape0"] = Op(xi)
    elif c["rng"] != "none":
        ops["state"] = Op(torch.tensor([seed, 11 if c["rng"] == "philox" else 4 * 37], dtype=torch.int64, device=dev))
    if c["packed"]:
        _known_ops(ops, m8, dims, total, True)
    step = nat.Ancestral(1.7, -0.4375 * 1.1, 0.9, 0.0 if c.get("eta0") else 0.6)

    def call(t):
        p = lambda k: _p(t, k)   # noqa: E731
        hd = nat.Heads(t["a"].data_ptr(), t["b"].data_ptr() if "b" in t else None, LP_DT[dt], 1 if c["combine"] else 0,
                       4.5 if c["combine"] else 0.0, 4.5 if c["combine"] else 0.0)
        r = nat.Rng()
        if c["rng"] == "tape":
            r.mode, r.tape0 = nat.RNG_TAPE, t["tape0"].data_ptr()
        elif c["rng"] != "none":
            r.mode = nat.RNG_PHILOX if c["rng"] == "philox" else nat.RNG_TORCH
            r.seed, r.draw0, r.state = 0, 5 if c["rng"] == "philox" else 0, t["state"].data_ptr()
        kn = _known_struct(t) if c["packed"] else None
        return lib.lp_boundary_ancestral(C.byref(hd), p("y"), p("noise"), p("mask"), C.byref(kn) if kn is not None else None,
                                         p("x"), p("out"), C.byref(step), C.byref(r) if c["rng"] != "none" else None,
                                         p("table"), C.byref(dims), _stream())
    run_guarded(case, dev, ops, call, {k for k in ("x", "out") if k in ops}, A.expect_kernel(c, total, sp))


# ---------------------------------------------------------------------------------------------------------------
# lp_prologue_f32, lp_advance_f32, lp_stop_stats_f32, lp_pack_mask_f32
# ---------------------------------------------------------------------------------------------------------------
def _dense(shape, mask, dev, seed, split=None, n=3):
    """-> mask, dims, table and n random operands of one launch."""
    gen = torch.Generator(device=dev).manual_seed(seed)
    m8, _, rs, cs = L.make_mask(shape, mask, gen, dev)
    tab, _ = L.case_table(dict(table="lam12", seed=seed, split=split), shape, dev)
    return m8, L.dims_of(shape, rs, cs, split), tab, [torch.randn(shape, device=dev, generator=gen) for _ in range(n)], gen


def _v4(shape, split):
    return 4 if int(np.prod(shape[2:])) % 4 == 0 and (split or 0) % 4 == 0 else 1


@pytest.mark.parametrize("shape,split,aliased,copy", [
    (BIG, None, True, False), ((1, 4, 256, 256), None, False, True), (WAN, None, True, True),
    ((2, 4, 45, 45), None, False, False), ((1, 3, 7, 9), None, True, True), ((1, 3, 7, 9), None, False, True),
    ((4, 1, 4096), 3072, False, True), ((4, 1, 4096), 3071, True, False), ((3, 1, 2049), 1000, False, False),
    ((1, 1, 2049), 1000, False, True)])
def test_prologue(shape, split, aliased, copy, cuda_device):
    lib, dev = _lib(), cuda_device
    m8, dims, tab, (x, y, nz), _ = _dense(shape, "rand", dev, 3500, split)
    ops = {"x": Op(x), "y": Op(y), "noise": Op(nz), "mask": Op(m8), "table": Op(tab)}
    if not aliased:
        ops["x_model"] = Op(torch.zeros(shape, device=dev))
    if copy:
        ops["x_copy"] = Op(torch.zeros(shape, device=dev))
    xm = "x" if aliased else "x_model"

    def call(t):
        return lib.lp_prologue_f32(_p(t, "x"), _p(t, "y"), _p(t, "noise"), _p(t, "mask"), _p(t, xm), _p(t, "x_copy"),
                                   _p(t, "table"), C.byref(dims), _stream())
    cid = f"prologue-{shape}-{split}-{aliased}-{copy}"
    _, gd, _ = run_guarded(cid, dev, ops, call, {xm} | ({"x_copy"} if copy else set()), f"prologue_kernel<{_v4(shape, split)}>")
    if copy:
        assert torch.equal(G.bits(gd["x_copy"]), G.bits(gd[xm]))


ADVANCE = [("tape", (1, 4, 128, 128), None, 1), ("tape", (1, 3, 7, 9), None, 0), ("philox", (5, 4, 120, 136), None, 0),
           ("philox_state", (2, 4, 45, 45), None, 1), ("torch", (1, 4, 272, 256), None, 1), ("torch", WAN, None, 0),
           ("torch_state", BIG, None, 1), ("torch", (1, 3, 7, 9), None, 0), ("torch_state", (3, 1, 2049), 1000, 1),
           ("philox", (4, 1, 4096), 3071, 0), ("tape", (4, 1, 4096), 3072, 1)]


@pytest.mark.parametrize("rng,shape,split,half", ADVANCE)
def test_advance(rng, shape, split, half, cuda_device):
    nat, lib, dev = _nat(), _lib(), cuda_device
    m8, dims, tab, (x, cc, xi), _ = _dense(shape, "rand", dev, 3600, split)
    ops = {"x": Op(x * 2), "c": Op(cc * 3), "mask": Op(m8), "table": Op(tab)}
    if rng == "tape":
        ops["tape0"] = Op(xi)
    elif rng.endswith("_state"):
        ops["state"] = Op(torch.tensor([4242, 9 if rng.startswith("philox") else 4 * 1001], dtype=torch.int64, device=dev))

    def call(t):
        r = nat.Rng()
        if rng == "tape":
            r.mode, r.tape0 = nat.RNG_TAPE, t["tape0"].data_ptr()
        else:
            r.mode = nat.RNG_PHILOX if rng.startswith("philox") else nat.RNG_TORCH
            r.seed, r.draw0 = 4242, 3 if rng.startswith("philox") else 0
        if "state" in t:
            r.seed, r.state = 0, t["state"].data_ptr()
        return lib.lp_advance_f32(_p(t, "x"), _p(t, "c"), _p(t, "mask"), _p(t, "table"), C.byref(dims), C.byref(r), half,
                                  _stream())
    want = {"tape": "advance_kernel<0>", "philox": "advance_kernel<1>", "torch": "advance_torch_kernel"}[rng.split("_")[0]]
    run_guarded(f"advance-{rng}-{shape}-{split}-{half}", dev, ops, call, {"x"}, want)


@pytest.mark.parametrize("shape,mask,split,ring,table", [
    ((128, 4, 128, 128), "full", None, True, True), (BIG, "rand", None, False, True), ((2, 4, 45, 45), "rand", None, True, False),
    ((1, 3, 7, 9), "full", None, False, False), ((16, 1, 40960), "rand", 30720, True, True), ((3, 1, 2049), "rand", 1000, True, True)])
def test_stop_stats(shape, mask, split, ring, table, cuda_device):
    """sums is two doubles, zeroed and then accumulated by the call: the band after it starts at byte 16."""
    lib, dev = _lib(), cuda_device
    m8, dims, tab, (a, b), gen = _dense(shape, mask, dev, 3700, split, n=2)
    ops = {"a": Op(a), "b": Op(b), "mask": Op(m8), "sums": Op(torch.tensor([7.0, -9.0], dtype=torch.float64, device=dev))}
    if ring:
        ops["ring"] = Op((torch.rand(m8.shape, device=dev, generator=gen) < 0.2).to(torch.uint8))
    if table:
        ops["table"] = Op(tab)

    def call(t):
        return lib.lp_stop_stats_f32(_p(t, "a"), _p(t, "b"), _p(t, "mask"), _p(t, "ring"), _p(t, "table"), C.byref(dims),
                                     _p(t, "sums"), _stream())
    cid = f"stats-{shape}-{split}-{ring}-{table}"
    pl, gd, arena = run_guarded(cid, dev, ops, call, {"sums"}, f"stop_stats_kernel<{_v4(shape, split)}>", same=())
    assert arena.ops["sums"].nbytes == 16
    # the order of the per-block atomicAdds is not fixed: the two calls agree to the rounding of a double sum
    assert torch.allclose(gd["sums"], pl["sums"], rtol=1e-12, atol=0.0), (gd["sums"], pl["sums"])
    assert float(gd["sums"][0]) > 0 and (float(gd["sums"][1]) > 0) == ring


@pytest.mark.parametrize("n", [1, 3, 255, 257, 1003, 262147])
@pytest.mark.parametrize("invert", [0, 1])
def test_pack_mask(n, invert, cuda_device):
    lib, dev = _lib(), cuda_device
    gen = torch.Generator(device=dev).manual_seed(n)
    ops = {"mask_f32": Op(torch.rand(n, device=dev, generator=gen)),
           "mask_u8": Op(torch.full((n,), 0x5A, dtype=torch.uint8, device=dev))}

    def call(t):
        return lib.lp_pack_mask_f32(_p(t, "mask_f32"), _p(t, "mask_u8"), n, invert, _stream())
    _, gd, _ = run_guarded(f"pack-mask-{n}-{invert}", dev, ops, call, {"mask_u8"}, "pack_mask_kernel")
    assert torch.equal(gd["mask_u8"].bool(), (gd["mask_f32"] > 0.5) != bool(invert))


# ---------------------------------------------------------------------------------------------------------------
# lp_pack_known
# ---------------------------------------------------------------------------------------------------------------
KNOWN_TOTALS = [1, 31, 32, 33, 256 * 32 - 1, 256 * 32, 256 * 32 + 1, 1 << 18, int(np.prod(WAN))]
KNOWN_CASES = [(n, "rand", True) for n in KNOWN_TOTALS] + [(n, "known", True) for n in (1, 33, 256 * 32, 256 * 32 + 1, 1 << 18)] + \
              [(n, "free", True) for n in (1, 32, 256 * 32 + 1, 1 << 18)] + [(n, "rand", False) for n in (33, 256 * 32 - 1, 1 << 18)] + \
              [(int(np.prod(WAN)), "known", False)]


@pytest.mark.parametrize("total,mask,with_noise", KNOWN_CASES)
def test_pack_known(total, mask, with_noise, cuda_device):
    """words holds lp_known_words(total) uint32 and the band after them stays intact; y_known / noise_known hold
    total + 4 floats of which the builder writes exactly the known count: the rest (the + 4 with an all-known mask)
    keeps what it held, an all-free mask writes nothing at all, and noise == NULL leaves noise_known alone."""
    nat, lib, dev = _nat(), _lib(), cuda_device
    gen = torch.Generator(device=dev).manual_seed(total)
    m8 = {"rand": torch.rand(total, device=dev, generator=gen) < 0.5, "known": torch.ones(total, dtype=torch.bool, device=dev),
          "free": torch.zeros(total, dtype=torch.bool, device=dev)}[mask].to(torch.uint8)
    dims = nat.Dims(1, total, total, total, 0, 0)
    n_words = int(lib.lp_known_words(total))
    assert n_words >= 2 * ((total + 31) // 32 + 1)
    held = torch.full((total + 4,), SENTINEL, dtype=torch.int32, device=dev).view(torch.float32)
    ops = {"mask": Op(m8), "y": Op(torch.randn(total, device=dev, generator=gen)),
           "noise": Op(torch.randn(total, device=dev, generator=gen)),
           "words": Op(torch.full((n_words,), SENTINEL, dtype=torch.int32, device=dev)),
           "y_known": Op(held), "noise_known": Op(held)}

    def call(t):
        return lib.lp_pack_known(_p(t, "mask"), C.byref(dims), _p(t, "y"), _p(t, "noise") if with_noise else None,
                                 _p(t, "words"), _p(t, "y_known"), _p(t, "noise_known"), _stream())
    written = {"words"}
    if mask != "free":
        written |= {"y_known"} | ({"noise_known"} if with_noise else set())
    _, gd, _ = run_guarded(f"pack-known-{total}-{mask}-{with_noise}", dev, ops, call, written,
                           {"known_bits_kernel", "known_scan_kernel", "known_scatter_kernel"})
    count = int(gd["mask"].sum())
    W = (total + 31) // 32
    assert int(gd["words"][2 * W]) == 0 and int(gd["words"][2 * W + 1]) == count
    for k, src in (("y_known", "y"), ("noise_known", "noise")):
        if k in written:
            assert torch.equal(gd[k][:count], gd[src][gd["mask"].bool()]), k
            assert bool((gd[k][count:].view(torch.int32) == SENTINEL).all()), f"{k} written past the known count {count}"


# ---------------------------------------------------------------------------------------------------------------
# lp_fill_normal_f32, lp_torch_cpu_randn_f32, lp_synth_denoiser
# ---------------------------------------------------------------------------------------------------------------
def _fill_sizes():
    return [1, 3, 255, 257, "4T-1", "4T+1"]


@pytest.mark.parametrize("n", _fill_sizes())
@pytest.mark.parametrize("rng", ["philox", "torch", "torch_state"])
def test_fill_normal(n, rng, cuda_device):
    nat, lib, dev = _nat(), _lib(), cuda_device
    if isinstance(n, str):     # around one full call of every subsequence of torch's widest grid
        T = L.torch_T(1 << 24)[0]
        n = 4 * T + (1 if n.endswith("+1") else -1)
        assert L.torch_T(n)[0] == T
    ops = {"out": Op(torch.full((n,), SENTINEL, dtype=torch.int32, device=dev).view(torch.float32))}
    if rng.endswith("_state"):
        ops["state"] = Op(torch.tensor([77, 4 * 5], dtype=torch.int64, device=dev))

    def call(t):
        r = nat.Rng(mode=nat.RNG_PHILOX if rng == "philox" else nat.RNG_TORCH, seed=77, draw0=8)
        if "state" in t:
            r.seed, r.state = 0, t["state"].data_ptr()
        return lib.lp_fill_normal_f32(_p(t, "out"), n, C.byref(r), _stream())
    _, gd, _ = run_guarded(f"fill-{rng}-{n}", dev, ops, call, {"out"}, f"fill_normal_{rng.split('_')[0]}_kernel")
    assert bool(torch.isfinite(gd["out"]).all())


@pytest.mark.parametrize("n", [16, 17, 31, 4104, 624 * 227 + 16])
def test_torch_cpu_randn(n, cuda_device):
    """out has room for n + 16 floats (the raw words of a redrawn tail) and state_out is exactly 624 words."""
    lib, dev = _lib(), cuda_device
    ops = {"out": Op(torch.full((n,), SENTINEL, dtype=torch.int32, device=dev).view(torch.float32), slack=16),
           "state": Op(torch.full((624,), SENTINEL, dtype=torch.int32, device=dev))}
    consumed = C.c_int64(0)

    def call(t):
        return lib.lp_torch_cpu_randn_f32(_p(t, "out"), n, C.c_uint64(0x5EED), _p(t, "state"), C.byref(consumed), _stream())
    want = {"mt19937_raw_kernel", "normal_fill16_kernel"}
    _, gd, _ = run_guarded(f"cpu-randn-{n}", dev, ops, call, {"out", "state"}, want)
    assert consumed.value == n + (16 if n % 16 else 0)
    ref = torch.randn(n, generator=torch.Generator().manual_seed(0x5EED), dtype=torch.float32)
    if torch.equal(ref[:16], gd["out"][:16].cpu()):     # this host's torch draws the AVX2 bits (see hostnoise.verified)
        assert torch.equal(ref, gd["out"].cpu())


@pytest.mark.parametrize("dt", [F32, BF16, F16])
@pytest.mark.parametrize("n,two", [(1003, True), (1002, False), (4096, True), (1 << 20, False), (7, True)])
def test_synth_denoiser(dt, n, two, cuda_device):
    lib, dev = _lib(), cuda_device
    gen = torch.Generator(device=dev).manual_seed(n)
    ops = {"x": Op(torch.randn(n, device=dev, generator=gen)), "h0": Op(torch.zeros(n, dtype=dt, device=dev))}
    if two:
        ops["h1"] = Op(torch.zeros(n, dtype=dt, device=dev))
    coef = (C.c_float * 5)(0.9, 0.05, 0.01, 0.8, -0.02)

    def call(t):
        return lib.lp_synth_denoiser(_p(t, "x"), _p(t, "h0"), _p(t, "h1"), LP_DT[dt], n, coef, _stream())
    want = f"synth_denoiser_kernel<{4 if n % 4 == 0 else 1},{DTYPES[dt]}>"
    run_guarded(f"synth-{DTYPES[dt]}-{n}-{two}", dev, ops, call, {"h0"} | ({"h1"} if two else set()), want)


# ---------------------------------------------------------------------------------------------------------------
# one layer up: the engine call, and the sizes the Python side allocates
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(1, 4, 256, 256), (1, 3, 7, 9)])
def test_engine_call_on_guarded_operands(shape, cuda_device):
    """engine.LanPaint(...)(x, ...) eager, with x, the latent image, the noise and the mask placed through the arena:
    x is rewritten in place, nothing else is, and out and x equal the plain call's bit for bit."""
    from lanpaint_b200.engine import LanPaint
    dev = cuda_device
    x, y, noise, m = synth_inputs(shape, seed=3, device=dev)
    sig = torch.tensor([2.0], device=dev)
    times = O.times_from_sigma(sig, False)

    def run(t):
        torch.manual_seed(1234)
        eng = LanPaint(make_model("two_heads", False), NSteps=3, Friction=15.0, Lambda=5.0, Beta=1.0, StepSize=0.2,
                       MinStepFrac=1.0, rng="torch")
        out = eng(t["x"], t["y"], t["noise"], sig, t["mask"], tuple(times), {}, 0, n_steps=3)
        torch.cuda.synchronize()
        return out
    ops = {"x": x, "y": y, "noise": noise, "mask": m}
    pl = {k: v.clone() for k, v in ops.items()}
    out_plain = run(pl)
    arena = G.Arena(dev)
    gd = {k: arena.place(v, name=k) for k, v in ops.items()}
    arena.snapshot()
    out = run(gd)
    assert torch.equal(G.bits(out), G.bits(out_plain)) and torch.equal(G.bits(gd["x"]), G.bits(pl["x"]))
    assert not torch.equal(gd["x"], x)
    arena.check(f"engine-{shape}", written={"x"})


@pytest.mark.parametrize("total", [33, 256 * 32 + 1, int(np.prod(WAN))])
def test_engine_pack_known_allocates_the_layout_the_header_asks_for(total, cuda_device):
    from lanpaint_b200 import engine
    nat, lib, dev = _nat(), _lib(), cuda_device
    gen = torch.Generator(device=dev).manual_seed(total)
    arena = G.Arena(dev)
    m8 = arena.place((torch.rand(total, device=dev, generator=gen) < 0.5).to(torch.uint8), name="mask")
    y = arena.place(torch.randn(total, device=dev, generator=gen), name="y")
    nz = arena.place(torch.randn(total, device=dev, generator=gen), name="noise")
    arena.snapshot()
    ko = engine.pack_known(engine.PackedMask(m8, total, 0), nat.Dims(1, total, total, total, 0, 0), y, nz)
    torch.cuda.synchronize()
    arena.check(f"engine-pack-known-{total}")
    for t, n in ((ko.words, int(lib.lp_known_words(total))), (ko.y, total + 4), (ko.noise, total + 4)):
        assert t.numel() == n and t.untyped_storage().nbytes() >= 4 * n
    assert torch.equal(ko.y[:int(m8.sum())], y[m8.bool()])


@pytest.mark.parametrize("shape", [(1, 4, 2, 2), (1, 3, 7, 9), (2, 4, 64, 64)])
def test_hostnoise_allocates_the_room_the_header_asks_for(shape, cuda_device):
    from lanpaint_b200 import hostnoise
    n = int(np.prod(shape))
    out, state, consumed = hostnoise._draw(n, 5, cuda_device)
    assert out.numel() == n + 16 and state.numel() == 624 and consumed == n + (16 if n % 16 else 0)
    z = hostnoise.torch_cpu_randn(shape, 5, cuda_device, advance_cpu_generator=False)
    assert tuple(z.shape) == shape and z.untyped_storage().nbytes() >= 4 * (n + 16) and torch.equal(z.reshape(-1), out[:n])


# ---------------------------------------------------------------------------------------------------------------
# coverage
# ---------------------------------------------------------------------------------------------------------------
HEAD_FAMILIES = L.HEAD_FAMILIES + ("boundary_ancestral_torch_tma_kernel", "boundary_ancestral_kernel")
KINDS = ("1,0", "0,1", "0,0", "1,1")     # (FIRST, FUSE_NEXT)
# canonical names with the head type taken out; an entry that ends in "," or "<" is a prefix
REQUIRED = (
    # every family expect_substep of test_gpu_launch_ref.py names
    [f"substep_kernel<{n},{r},{k},0>" for n in (4, 1) for r in (0, 1) for k in KINDS] +
    [f"substep_kernel<{n},1,0,1,1>" for n in (4, 1)] + ["substep_tma_kernel<0,1,1,", "substep_tma_kernel<"] +
    [f"{fam}<{k}>" for fam in ("substep_torchvec_kernel", "substep_torch_kernel") for k in KINDS] +
    [f"substep_torch_tma_kernel<{k},{pk}>" for k in KINDS for pk in (0, 1)] +
    # the boundary sweep
    [f"boundary_kernel<{n},{pk}>" for n in (4, 1) for pk in (0, 1)] + ["boundary_tma_kernel<"] +
    # expect_kernel of test_gpu_sampler_ancestral.py: the TMA kernel packed and dense, the LDG kernel <N, packed, rng>
    [f"boundary_ancestral_torch_tma_kernel<{cb},{nx},{pk}>" for cb, nx, pk in ((1, 1, 1), (1, 0, 0), (0, 1, 0), (0, 0, 1))] +
    [f"boundary_ancestral_kernel<{v}>" for v in ("4,1,2", "4,0,2", "1,1,2", "1,0,2", "4,1,1", "1,0,1", "4,1,0", "4,0,0",
                                                "1,1,0", "4,1,-1", "4,0,-1", "1,1,-1")] +
    ["prologue_kernel<4>", "prologue_kernel<1>", "advance_kernel<0>", "advance_kernel<1>", "advance_torch_kernel",
     "stop_stats_kernel<4>", "stop_stats_kernel<1>", "pack_mask_kernel", "known_bits_kernel", "known_scan_kernel",
     "known_scatter_kernel", "fill_normal_philox_kernel", "fill_normal_torch_kernel", "mt19937_raw_kernel",
     "normal_fill16_kernel", "synth_denoiser_kernel<4>", "synth_denoiser_kernel<1>"])


def _headless(name):
    """canonical name -> (the name without its head type, the head type or None)."""
    for h in DTYPES.values():
        for pat in (f"<{h},", f",{h},", f",{h}>"):
            if pat in name:
                return name.replace(pat, pat.replace(h + ",", "").replace("," + h, ""), 1), h
    return name, None


def test_kernels_reached():
    """Every kernel family the launch tests name ran on guarded operands: a family the cases silently stopped
    reaching fails here."""
    n_cases = (len(SUBSTEP_CASES) + len(BOUNDARY_CASES) + len(ANCESTRAL_CASES) + 10 + len(ADVANCE) + 6 + 12 +
               len(KNOWN_CASES) + 18 + 5 + 15)
    if len(RAN) < n_cases:
        pytest.skip(f"only {len(RAN)} of the {n_cases} guarded cases ran in this session")
    print(f"\nguarded cases: {len(RAN)}, {STATS['seconds']:.1f} s in the cases, "
          f"peak device memory {STATS['peak_bytes'] / 2 ** 30:.2f} GiB")
    print("kernels run on guarded operands (launches):")
    for name in sorted(SEEN):
        print(f"  {SEEN[name]:3d}  {name}")
    seen, heads = set(), collections.defaultdict(set)
    for name in SEEN:
        bare, h = _headless(name)
        seen.add(bare)
        heads[L.family(name)].add(h)
    missing = [r for r in REQUIRED if not (any(n.startswith(r) for n in seen) if r[-1] in ",<" else r in seen)]
    assert not missing, missing
    for fam in HEAD_FAMILIES + ("synth_denoiser_kernel",):
        assert heads[fam] == set(DTYPES.values()), (fam, heads[fam])
