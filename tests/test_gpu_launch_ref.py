"""GPU: every dispatched update kernel against an fp64 restatement of its launch (tests/_launch_ref.py), and which
kernel each launch ran.

Each case makes ONE call of a device entry point (lp_substep[_known], lp_boundary[_known], lp_prologue_f32,
lp_advance_f32, lp_stop_stats_f32) under torch.profiler, asserts the kernel it launched by name and template
arguments, and compares every output element with the fp64 restatement:
    |got - want| <= K * 2^-24 * magnitude     (+ |kick| * eps_BM on the philox stream)
where magnitude is the element's chain evaluated on absolute values (see _launch_ref).  K = 8: the longest chain
of fp32 roundings in a launch is about a dozen operations (CFG combine, target, C, drift, two advances, the change
of variables), and the largest ratio observed on an H100 over the whole matrix is about 4 in every family
(test_kernel_coverage prints it per family), so K leaves a factor of two.  Exact properties are checked bit for bit: out == y at known positions, the
replace step leaves free positions alone, c_state is untouched when the flags do not write it (NaN-poisoned), and
x_copy == x.

The matrix is representative crossings, not a cross product:
  * the launch-kind sweep runs every (FIRST, FUSE_NEXT, STORE_C, MERGE_NOISE) combination on every kernel family
    (LDG vec4 / scalar on the tape and philox streams, the philox TMA kernel, the torch-stream TMA kernel dense and
    packed, the torch vec4 and scalar kernels), rotating head dtype (fp32 / bf16 / fp16), head aliasing
    (separate / b = NULL / b == a), mask kind and coefficient table, so each family sees all three dtypes;
  * the edge cases sit on the dispatch boundaries: total == tma_min == torch's T (one call), exactly the torch grid
    cap, past it (partial call), the Wan latent (two calls, plane 3600), sub-tiles spanning rows with distinct table
    rows, vec4-but-not-TMA sizes, the flagship size packed and dense (eight calls per subsequence), full-shape /
    blob / all-known / all-free masks, the CFG combine with cfg != cfg_big and cfg_big < 0, the rng->state block,
    each operand misaligned by 4 bytes in turn (scalar fallback) and a 16-bit head by 8 (vec4, not TMA), and the
    side outputs x_copy / x0e (which force the LDG kernels);
  * the boundary sweep covers vec4 / scalar x dense / packed x the three dtypes, the TMA boundary kernel with and
    without combine and next, out-only launches and a zero Euler coefficient (replace step only);
  * prologue, advance (all three streams, one torch launch with several calls per subsequence and the state
    block) and the early-stop statistics with the inv_S table and a full-shape ring at 8.4 M elements;
  * the audio-video flat pack (lp_dims.row_split, engine._av_call): every launch kind on every family a split can
    reach (LDG vec4 / scalar on tape and philox with merge, torch vec4 and scalar), the boundary dense and packed,
    prologue, advance on all three streams and the statistics, over 2 * lines distinct table rows whose audio rows
    carry corrections != 1; one 4 Mi-element line split in the middle with TMA otherwise enabled, 16 lines split at
    3/4, splits not a multiple of 4, an odd n_last, split == n_last and split == 4.  No TMA kernel may run under a
    split (they find the row without it);
  * the audio correction without a split on the TMA sub-step kernels, the only way to reach the corr code of the
    torch TMA kernel's lane pairs.
Coefficient tables mix VE rows sigma in {0.0292, 0.3, 1, 14.6, 80} and flow rows t in {0.02, 0.5, 0.98, 1}, with
MinStepFrac 0, Lambda 0.1 or 12 and Beta 1.5 (distinct dt per mask class), or come from lp_build_coef_table_dt."""
import collections
import ctypes as C
import functools
import time

import numpy as np
import pytest
import torch
from torch.profiler import ProfilerActivity, profile

import _launch_ref as R

pytestmark = pytest.mark.gpu

K = 8
P = C.c_void_p
DTYPES = {torch.float32: "float", torch.bfloat16: "__nv_bfloat16", torch.float16: "__half"}
LP_DT = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}
TMA_MIN = 1 << 18

SEEN = collections.Counter()          # canonical kernel name -> launches
SEEN_SPLIT = collections.Counter()    # the same, launches of cases with a row split
WORST = collections.defaultdict(float)  # kernel family -> largest |got - want| / (2^-24 magnitude)
RAN = set()


def _lib():
    from lanpaint_b200 import _native
    return _native.load()


def _stream():
    return P(torch.cuda.current_stream().cuda_stream)


# ---------------------------------------------------------------------------------------------------------------
# which kernel ran
# ---------------------------------------------------------------------------------------------------------------
canon = R.canon


class LostRecord(Exception):
    """The launch's results were right but the profiler recorded no kernel for it."""


def rerun_on_lost_record(test):
    """CUPTI can, rarely, deliver no record of a kernel that ran: run such a case once more from its seeded inputs."""
    @functools.wraps(test)
    def wrapper(*args, **kw):
        try:
            return test(*args, **kw)
        except LostRecord:
            return test(*args, **kw)
    return wrapper


def launched(fn, split=None):
    """Run fn() (one library call returning its status) under torch.profiler -> set of canonical lp:: kernel names.
    The library call sits a few milliseconds inside the profiled window: the profiler keeps only device records whose
    timestamps fall inside the window, and a launch of a few microseconds at its very edge can be dropped.
    split: the launch's row split (None: none), to record the kernels of split launches apart."""
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        time.sleep(0.005)
        rc = fn()
        torch.cuda.synchronize()
        time.sleep(0.005)
    assert rc == 0, rc
    names = [e.name() for e in prof.profiler.kineto_results.events() if "lp::" in e.name()]
    got = {canon(n) for n in names}
    for n in got:
        SEEN[n] += 1
        if split is not None:
            SEEN_SPLIT[n] += 1
    return got


def assert_kernel(case_id, got, want):
    """Checked after the outputs, so that a launch that did not happen fails on its values, not here."""
    if not got:
        raise LostRecord(case_id)
    assert got == {want}, (case_id, got, want)


def family(name: str) -> str:
    return name.split("<")[0]


def _check(fam, label, got, want_mag, k=K, slack=0.0):
    worst, bad = R.within(got, want_mag, k, slack)
    WORST[fam] = max(WORST[fam], worst)
    if bad is not None:
        flat = got.reshape(-1)
        pytest.fail(f"{label}: element {bad} = {float(flat[bad])!r}, want {float(want_mag[0].reshape(-1)[bad])!r} "
                    f"(magnitude {float(want_mag[1].reshape(-1)[bad])!r}); worst ratio {worst:.3g} > K = {k}")


def _bits(t):
    return t.contiguous().view(torch.int32 if t.element_size() == 4 else torch.int16)


# ---------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------
ROWS = [("ve", 0.0292), ("ve", 0.3), ("ve", 1.0), ("ve", 14.6), ("ve", 80.0),
        ("flow", 0.02), ("flow", 0.5), ("flow", 0.98), ("flow", 1.0)]
TABLES = ("lam12", "lam01", "dt")


def make_table(n_rows, variant, shift, dev):
    from lanpaint_b200 import _native
    from lanpaint_b200.schedule import Hyper, build_table
    rows = [ROWS[(r + shift) % len(ROWS)] for r in range(n_rows)]
    out = np.zeros((n_rows, 32), dtype=np.float32)
    for r, (kind, v) in enumerate(rows):
        s = torch.tensor([v], dtype=torch.float32)
        if kind == "ve":
            abt = 1 / (1 + s ** 2)
            ve, rn, ry = s, s, torch.ones(1)
        else:
            abt = (1 - s) ** 2 / ((1 - s) ** 2 + s ** 2)
            ve, rn, ry = torch.zeros(1), s, 1 - s
        if variant == "dt":
            a = abt.double().numpy()
            S = np.sqrt(1 + ve.double().numpy() ** 2) if kind == "ve" else 1 / (np.sqrt(a) + np.sqrt(1 - a))
            dtf, dtk = 0.15 * np.maximum(1 - a, 0.05), 0.4 * np.maximum(1 - a, 0.05)
            rc = _native.load().lp_build_coef_table_dt(
                a.ctypes.data_as(P), S.ctypes.data_as(P), dtf.ctypes.data_as(P), dtk.ctypes.data_as(P), 2.0, 0, 1,
                out[r:].ctypes.data_as(P))
            assert rc == 0
        else:
            lam = 12.0 if variant == "lam12" else 0.1
            hp = Hyper(0.2 if variant == "lam12" else 0.35, lam, 1.5, 0.0, kind == "flow")
            out[r] = build_table(abt.numpy(), ve.numpy(), hp, rep_noise=rn.numpy(), rep_y=ry.numpy())[0]
    return torch.from_numpy(out).to(dev)


def make_mask(shape, kind, gen, dev):
    """-> (uint8 mask, full-shape bool known, mask_row_stride, mask_channel_stride)."""
    B, Cc, sp = shape[0], shape[1], int(np.prod(shape[2:]))
    bshape = (B, 1) + tuple(shape[2:])
    if kind == "full":
        m = torch.rand(shape, device=dev, generator=gen) < 0.5
    elif kind == "rand":
        m = torch.rand(bshape, device=dev, generator=gen) < 0.5
    elif kind == "known":
        m = torch.ones(bshape, dtype=torch.bool, device=dev)
    elif kind == "free":
        m = torch.zeros(bshape, dtype=torch.bool, device=dev)
    else:   # blob: an ellipse in the last two dims
        h, w = shape[-2], shape[-1]
        yy, xx = torch.meshgrid(torch.arange(h, device=dev), torch.arange(w, device=dev), indexing="ij")
        e = ((yy - h / 2) / (0.35 * h)) ** 2 + ((xx - w / 2) / (0.3 * w)) ** 2 < 1
        m = e.expand(bshape).clone()
    m8 = m.to(torch.uint8).contiguous()
    full = kind == "full"
    return m8, m.expand(shape), (Cc * sp if full else sp), (sp if full else 0)


def offset_copy(t, nbytes):
    """t's contents in a fresh buffer whose data pointer is nbytes past a 256-byte boundary."""
    if nbytes == 0:
        return t.clone()
    k = nbytes // t.element_size()
    buf = torch.empty(t.numel() + k, dtype=t.dtype, device=t.device)
    v = buf[k:].view(t.shape)
    v.copy_(t)
    return v


def dims_of(shape, rs, cs, split=None):
    from lanpaint_b200 import _native
    sp = int(np.prod(shape[2:]))
    return _native.Dims(shape[0], shape[1] * sp, sp, rs, cs, split or 0)


AV_CORR = (0.625, 1.3, 0.8)


def case_table(c, shape, dev):
    """-> (table, per-element rows or None).  A case with a "split" is an audio-video flat pack (one line per row,
    shape (lines, 1, n_last)): 2 * lines distinct rows, the audio rows lines.. carrying the corrections AV_CORR in
    turn, and every element reads the row split_rows gives it.  A case with "corr" (no split) sets the correction of
    row b to corr[b % len(corr)]."""
    split = c.get("split")
    lines = shape[0]
    tab = make_table(lines * (2 if split is not None else 1), c["table"], c["seed"], dev)
    if split is not None:
        tab[lines:, R.T_CORR] = torch.tensor([AV_CORR[b % 3] for b in range(lines)], device=dev)
        return tab, R.split_rows(shape, split, dev)
    if c.get("corr"):
        tab[:, R.T_CORR] = torch.tensor([c["corr"][b % len(c["corr"])] for b in range(lines)], device=dev)
    return tab, None


def torch_T(n):
    g, inc = C.c_int64(0), C.c_uint64(0)
    assert _lib().lp_torch_randn_geometry(n, torch.cuda.current_device(), C.byref(g), C.byref(inc)) == 0
    return int(g.value) * 256, int(inc.value)


def pack_known(m8, dims, y, noise, total):
    from lanpaint_b200 import _native
    lib = _lib()
    dev = y.device
    words = torch.zeros(int(lib.lp_known_words(total)), dtype=torch.int32, device=dev)
    yk = torch.zeros(total + 4, device=dev)
    nk = torch.zeros(total + 4, device=dev) if noise is not None else None
    rc = lib.lp_pack_known(P(m8.data_ptr()), C.byref(dims), P(y.data_ptr()), P(noise.data_ptr()) if noise is not None else None,
                           P(words.data_ptr()), P(yk.data_ptr()), P(nk.data_ptr()) if nk is not None else None, _stream())
    assert rc == 0
    return _native.Known(words.data_ptr(), yk.data_ptr(), nk.data_ptr() if nk is not None else None), (words, yk, nk)


# ---------------------------------------------------------------------------------------------------------------
# eps_BM: the philox-stream transform, exhaustively over each input word
# ---------------------------------------------------------------------------------------------------------------
SWEEP_SECOND_FIXED = (0x00000000, 0x40000000, 0x80000000, 0xC0000000, 0xFFFFFFFF)   # first word swept
SWEEP_FIRST_FIXED = (0x00000000, 0x80000000, 0xFFFFFF7F, 0xFFFFFFFF)                  # second word swept


@pytest.fixture(scope="module")
def normal_fast(cuda_device):
    lib = _lib()
    bad = torch.zeros(1, dtype=torch.int64, device=cuda_device)
    err = torch.zeros(1, dtype=torch.float64, device=cuda_device)
    total_bad, worst = 0, 0.0
    for sweep_second, fixed in [(0, w) for w in SWEEP_SECOND_FIXED] + [(1, w) for w in SWEEP_FIRST_FIXED]:
        assert lib.lp_selftest_normal_fast(fixed, sweep_second, P(bad.data_ptr()), P(err.data_ptr()), _stream()) == 0
        total_bad += int(bad.item())
        worst = max(worst, float(err.item()))
    return total_bad, worst


def test_philox_transform_is_finite_and_close_to_fp64(normal_fast):
    """box_muller_fast (MUFU lg2 / sqrt.approx / sin / cos) over all 2^32 values of each word for a handful of
    values of the other: never non-finite -- for u just below 1 the documented error of __logf exceeds |log u|,
    so -2 log u could have come out negative -- and within eps_BM of the fp64 transform of the same u and v."""
    nonfinite, eps = normal_fast
    print(f"\nphilox transform: {nonfinite} non-finite results, eps_BM = {eps:.3e}")
    assert nonfinite == 0
    assert 0 < eps < 5e-4     # measured 2.2e-4 on an H100


def test_philox_restatement_matches_torch_randn_stream(cuda_device):
    """The Philox4x32-10 restatement under torch's CUDA stream mapping (counter (offset/4 + call, subsequence),
    cuRAND's Box-Muller in fp64) reproduces torch.randn: two calls per subsequence, two offsets."""
    n = 1_500_000
    T, inc = torch_T(n)
    g = torch.Generator(device=cuda_device).manual_seed(0xC0FFEE)
    for draw in range(2):
        off = g.get_offset()
        z = torch.randn(n, generator=g, device=cuda_device).cpu().double().numpy()
        assert g.get_offset() - off == inc
        want = R.torch_stream_normals(n, 0xC0FFEE, off, T)
        assert np.abs(z - want).max() <= 1e-4, (draw, np.abs(z - want).max())


# ---------------------------------------------------------------------------------------------------------------
# lp_substep: expected kernel
# ---------------------------------------------------------------------------------------------------------------
def expect_substep(c, shape, rs, cs):
    sp, total = int(np.prod(shape[2:])), int(np.prod(shape))
    per_row = total // shape[0]
    H = DTYPES[c["dtype"]]
    f, n, mg = int(bool(c["flags"] & 1)), int(bool(c["flags"] & 2)), int(bool(c["flags"] & 8))
    mis = c.get("misalign", (None, 0))
    side = c.get("x_copy") or c.get("x0e")
    # a 16-bit head needs 8-byte alignment for the vec4 kernels, every other operand 16 bytes; TMA wants 16 everywhere
    head_mis = mis[0] == "a" or (mis[0] == "b" and c["heads"] == "sep")
    head_ok = not head_mis or (c["dtype"] != torch.float32 and mis[1] % 8 == 0)
    split = c.get("split")
    v4 = (per_row % 4 == 0 and sp % 4 == 0 and rs % 4 == 0 and cs % 4 == 0 and (split or 0) % 4 == 0
          and mis[0] not in ("x", "y", "c", "tape0", "tape1") and head_ok)
    tma = (c.get("tma", 1) != 0 and sp % 16 == 0 and rs % 16 == 0 and cs % 16 == 0 and not side
           and total >= c.get("tma_min", TMA_MIN) and mis[0] is None and not split)
    if c["rng"].startswith("torch"):
        T, _ = torch_T(total)
        calls = -(-total // (4 * T))
        if v4 and tma and T % 1024 == 0 and sp >= 64:
            return f"substep_torch_tma_kernel<{H},{f},{n},{int(bool(c.get('packed')))}>"
        if v4 and calls <= 65535:
            return f"substep_torchvec_kernel<{H},{f},{n}>"
        return f"substep_torch_kernel<{H},{f},{n}>"
    if c["rng"] == "tape":
        return f"substep_kernel<{4 if v4 else 1},{H},0,{f},{n},0>"
    if v4 and tma:
        return f"substep_tma_kernel<{H},{f},{n},{mg},2048,2,2>"
    return f"substep_kernel<{4 if v4 else 1},{H},1,{f},{n},{mg}>"


def run_substep(c, dev, eps_bm):
    from lanpaint_b200 import _native
    lib = _lib()
    shape, flags = c["shape"], c["flags"]
    first, nxt, store = bool(flags & 1), bool(flags & 2), bool(flags & 4)
    total = int(np.prod(shape))
    gen = torch.Generator(device=dev).manual_seed(c["seed"])
    m8, known, rs, cs = make_mask(shape, c["mask"], gen, dev)
    dims = dims_of(shape, rs, cs, c.get("split"))
    tab, rows = case_table(c, shape, dev)
    S = R._row(tab, R.T_S, len(shape), rows).float()
    x = (torch.randn(shape, device=dev, generator=gen) * S).contiguous()
    y = torch.randn(shape, device=dev, generator=gen)
    cprev = torch.randn(shape, device=dev, generator=gen) * 3
    a32 = torch.randn(shape, device=dev, generator=gen) * 1.5
    b32 = a32 + 0.3 * torch.randn(shape, device=dev, generator=gen)
    a, b = a32.to(c["dtype"]), b32.to(c["dtype"])
    mis_op, mis_b = c.get("misalign", (None, 0))
    ops = {"x": x, "y": y, "a": a, "b": b}
    for k in ops:
        ops[k] = offset_copy(ops[k], mis_b if mis_op == k else 0)
    x, y, a, b = ops["x"], ops["y"], ops["a"], ops["b"]
    if c["heads"] == "same":
        b = a
    writes_c = nxt or store
    if first and not writes_c:
        cbuf = offset_copy(torch.full(shape, float("nan"), device=dev), 4 if mis_op == "c" else 0)
    else:
        cbuf = offset_copy(cprev, 4 if mis_op == "c" else 0)
    c_before = cbuf.clone()
    x_copy = torch.full(shape, float("nan"), device=dev) if c.get("x_copy") else None
    x0e = torch.full(shape, float("nan"), device=dev) if c.get("x0e") else None
    # noise
    r = _native.Rng()
    seed, noise_err, keep = c["seed"] * 7919 + 3, 0.0, []
    xi1 = xi2 = None
    mode = c["rng"]
    k_draws = 1 if (not nxt or flags & 8) else 2
    if mode == "tape":
        xi1 = offset_copy(torch.randn(shape, device=dev, generator=gen), 4 if mis_op == "tape0" else 0)
        xi2 = torch.randn(shape, device=dev, generator=gen) if k_draws == 2 else None
        r.mode, r.tape0, r.tape1 = _native.RNG_TAPE, xi1.data_ptr(), xi2.data_ptr() if xi2 is not None else None
    elif mode.startswith("philox"):
        base = 11 if mode == "philox_state" else 0
        d0 = 5
        xi1 = torch.from_numpy(R.philox_normals(total, seed, base + d0)).to(dev).view(shape)
        xi2 = torch.from_numpy(R.philox_normals(total, seed, base + d0 + 1)).to(dev).view(shape) if k_draws == 2 else None
        r.mode, r.seed, r.draw0, r.draw1 = _native.RNG_PHILOX, seed, d0, d0 + 1
        if base:
            st = torch.tensor([seed, base], dtype=torch.int64, device=dev)
            keep.append(st)
            r.seed, r.state = 0, st.data_ptr()
        noise_err = eps_bm
    else:   # torch stream: torch.manual_seed(s) + torch.randn in the reference's order
        base = 4 * 37 if mode == "torch_state" else 0
        T, inc = torch_T(total)
        g = torch.Generator(device=dev).manual_seed(seed)
        g.set_offset(base)
        xi1 = torch.randn(shape, device=dev, generator=g)
        xi2 = torch.randn(shape, device=dev, generator=g) if k_draws == 2 else None
        assert g.get_offset() == base + k_draws * inc
        r.mode, r.seed, r.draw0, r.draw1 = _native.RNG_TORCH, seed, 0, inc   # seed s, draw0 = 0, draw1 = increment
        if base:   # {seed, base} read from the device
            st = torch.tensor([seed, base], dtype=torch.int64, device=dev)
            keep.append(st)
            r.seed, r.state = 0, st.data_ptr()
    cfg = c.get("cfg")
    hd = _native.Heads(a.data_ptr(), None if c["heads"] == "null" else b.data_ptr(), LP_DT[c["dtype"]],
                       1 if cfg else 0, cfg[0] if cfg else 0.0, cfg[1] if cfg else 0.0)
    want_name = expect_substep(c, shape, rs, cs)
    if "family" in c:   # the case reaches the family it was written for
        assert family(want_name) == c["family"], (c["id"], want_name)
    y_dense = y
    if c.get("packed"):
        kn, keep_k = pack_known(m8, dims, y, None, total)
        keep.append(keep_k)
        if "torch_tma" in want_name:   # the packed kernel must not read the dense y
            y_dense = torch.full_like(y, float("nan"))

        def call():
            return lib.lp_substep_known(P(x.data_ptr()), C.byref(hd), P(y_dense.data_ptr()), P(m8.data_ptr()), C.byref(kn),
                                        P(cbuf.data_ptr()), P(x_copy.data_ptr()) if x_copy is not None else None,
                                        P(x0e.data_ptr()) if x0e is not None else None, P(tab.data_ptr()),
                                        C.byref(dims), C.byref(r), flags, _stream())
    else:
        def call():
            return lib.lp_substep(P(x.data_ptr()), C.byref(hd), P(y.data_ptr()), P(m8.data_ptr()), P(cbuf.data_ptr()),
                                  P(x_copy.data_ptr()) if x_copy is not None else None,
                                  P(x0e.data_ptr()) if x0e is not None else None, P(tab.data_ptr()), C.byref(dims),
                                  C.byref(r), flags, _stream())
    x_in = x.clone()
    want = R.substep(x_in, a, None if c["heads"] == "null" else b, y, known, cprev, tab, xi1, xi2, flags, cfg=cfg,
                     noise_err=noise_err, rows=rows)
    got = launched(call, c.get("split"))
    fam = family(want_name)
    _check(fam, f"{c['id']} x", x, want["x"], slack=want["x_slack"])
    if writes_c:
        _check(fam, f"{c['id']} c", cbuf, want["c"])
    else:
        assert torch.equal(_bits(cbuf), _bits(c_before)), f"{c['id']}: c_state written although the flags do not"
    if x_copy is not None:
        assert torch.equal(_bits(x_copy), _bits(x)), f"{c['id']}: x_copy != x"
    if x0e is not None:
        _check(fam, f"{c['id']} x0e", x0e, want["x0e"])
        if cfg is None:
            assert torch.equal(x0e[~known], a.float()[~known]), f"{c['id']}: x0e != x0 at free positions"
    assert_kernel(c["id"], got, want_name)
    RAN.add(c["id"])


# ---------------------------------------------------------------------------------------------------------------
# the case matrix of lp_substep
# ---------------------------------------------------------------------------------------------------------------
def _sweep():
    cases = []
    dts = (torch.float32, torch.bfloat16, torch.float16)
    heads = ("sep", "null", "same")
    masks = ("rand", "full", "blob", "rand", "known", "free")
    kinds = (3, 1, 1 | 4, 2, 0, 0 | 4)
    fams = [("ldg4_tape", "tape", (1, 4, 128, 128), {}), ("ldg1_tape", "tape", (2, 4, 45, 45), {}),
            ("ldg4_philox", "philox", (1, 4, 128, 128), {}), ("ldg1_philox", "philox", (2, 4, 45, 45), {}),
            ("tma_philox", "philox", (1, 4, 128, 128), {"tma_min": 0}),
            ("torch_tma", "torch", (1, 4, 128, 128), {"tma_min": 0}),
            ("torch_tma_packed", "torch", (1, 4, 128, 128), {"tma_min": 0, "packed": True}),
            ("torchvec", "torch", (40, 4, 50, 50), {}), ("torch_scalar", "torch", (2, 4, 45, 45), {})]
    i = 0
    for name, rng, shape, extra in fams:
        fl = kinds + ((3 | 8, 2 | 8) if rng == "philox" else ())
        for flags in fl:
            cases.append(dict(id=f"{name}-f{flags}", shape=shape, rng=rng, flags=flags, dtype=dts[i % 3],
                              heads=heads[(i // 3) % 3], mask=masks[i % 6], table=TABLES[i % 3], seed=100 + i, **extra))
            i += 1
    return cases


F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16
EDGE = [
    # total == tma_min == torch's T: one Philox call, full-shape mask, packed and dense
    dict(id="T262144-full", shape=(1, 4, 256, 256), rng="torch", flags=2, dtype=F32, heads="sep", mask="full", table="lam12"),
    dict(id="T262144-packed-bf16", shape=(1, 4, 256, 256), rng="torch", flags=3, dtype=BF16, heads="sep", mask="full",
         table="dt", packed=True),
    dict(id="T262144-allknown", shape=(1, 4, 256, 256), rng="torch", flags=2, dtype=F32, heads="sep", mask="known",
         table="lam01", packed=True),
    dict(id="T262144-allfree", shape=(1, 4, 256, 256), rng="torch", flags=3, dtype=F32, heads="null", mask="free",
         table="lam12", packed=True),
    dict(id="T262144-philox-f16", shape=(1, 4, 256, 256), rng="philox", flags=1, dtype=F16, heads="sep", mask="full",
         table="lam12"),
    # exactly the torch grid cap (1056 x 256 on 132 SMs), packed fp16 heads, the state block
    dict(id="gridcap-state-f16", shape=(1, 4, 264, 256), rng="torch_state", flags=1 | 4, dtype=F16, heads="sep",
         mask="full", table="dt", packed=True),
    dict(id="gridcap-aliased", shape=(1, 4, 264, 256), rng="torch", flags=2, dtype=F32, heads="same", mask="blob",
         table="lam12"),
    # past the cap: a partial call
    dict(id="pastcap-blob", shape=(1, 4, 272, 256), rng="torch", flags=0 | 4, dtype=F32, heads="sep", mask="blob",
         table="lam01"),
    dict(id="pastcap-null-packed", shape=(1, 4, 272, 256), rng="torch", flags=3, dtype=BF16, heads="null", mask="rand",
         table="lam12", packed=True),
    # Wan latent: two calls, plane 3600, channel size not a multiple of the sub-tile
    dict(id="wan-packed", shape=(1, 16, 21, 80, 45), rng="torch", flags=2, dtype=F32, heads="sep", mask="rand",
         table="lam12", packed=True),
    dict(id="wan-philox-full", shape=(1, 16, 21, 80, 45), rng="philox", flags=2 | 8, dtype=BF16, heads="sep",
         mask="full", table="dt"),
    # sub-tiles spanning rows with distinct table rows; CFG combine with cfg != cfg_big, cfg_big < 0
    dict(id="rows-cfg", shape=(5, 4, 120, 136), rng="torch", flags=3, dtype=F32, heads="sep", mask="rand", table="dt",
         cfg=(4.5, -0.5)),
    dict(id="rows-cfg-packed", shape=(5, 4, 120, 136), rng="torch_state", flags=2, dtype=F32, heads="sep",
         mask="full", table="lam12", cfg=(7.0, 2.5), packed=True),
    dict(id="rows-philox-aliased", shape=(5, 4, 120, 136), rng="philox", flags=2, dtype=F32, heads="same", mask="full",
         table="lam12"),
    dict(id="rows-philox-state-cfg", shape=(5, 4, 120, 136), rng="philox_state", flags=3, dtype=F32, heads="sep",
         mask="rand", table="dt", cfg=(4.5, -0.5)),
    dict(id="rows-philox-bf16-null", shape=(5, 4, 120, 136), rng="philox", flags=3 | 8, dtype=BF16, heads="null",
         mask="blob", table="lam01"),
    dict(id="rows-tape-cfg", shape=(5, 4, 120, 136), rng="tape", flags=2, dtype=F32, heads="sep", mask="rand",
         table="lam12", cfg=(4.5, -0.5)),
    # large, spatial % 16 != 0: vec4 LDG whatever the size
    dict(id="vec4-philox-merge", shape=(40, 4, 50, 50), rng="philox", flags=2 | 8, dtype=F32, heads="sep", mask="full",
         table="lam12"),
    dict(id="vec4-torch-null-f16", shape=(40, 4, 50, 50), rng="torch", flags=3, dtype=F16, heads="null", mask="rand",
         table="dt"),
    # the flagship size: packed (the node default) and dense, eight calls per subsequence
    dict(id="flagship-packed", shape=(128, 4, 128, 128), rng="torch", flags=2, dtype=F32, heads="sep", mask="rand",
         table="lam12", packed=True),
    dict(id="flagship-dense-first", shape=(128, 4, 128, 128), rng="torch", flags=3, dtype=F32, heads="sep",
         mask="rand", table="dt"),
    dict(id="flagship-philox-merge", shape=(128, 4, 128, 128), rng="philox", flags=2 | 8, dtype=F32, heads="sep",
         mask="rand", table="lam01"),
    # side outputs force the LDG kernels (the early-stop loop's launches)
    dict(id="side-torch", shape=(1, 4, 256, 256), rng="torch", flags=1 | 4, dtype=F32, heads="sep", mask="rand",
         table="lam12", x_copy=True, x0e=True),
    dict(id="side-torch-steady-bf16", shape=(5, 4, 120, 136), rng="torch", flags=0 | 4, dtype=BF16, heads="null",
         mask="blob", table="dt", x0e=True),
    dict(id="side-philox", shape=(5, 4, 120, 136), rng="philox", flags=1 | 4, dtype=F32, heads="sep", mask="rand",
         table="lam01", x0e=True, x_copy=True),
    dict(id="side-tape-scalar", shape=(2, 4, 45, 45), rng="tape", flags=0 | 4, dtype=F16, heads="sep", mask="full",
         table="lam12", x0e=True, x_copy=True),
]
# each operand 4 bytes off in turn: the scalar fallbacks (an fp16 head 8 bytes off keeps vec4 but loses TMA)
for _op in ("x", "a", "b", "y", "c"):
    EDGE.append(dict(id=f"misalign-{_op}", shape=(5, 4, 120, 136), rng="torch", flags=2, dtype=F32, heads="sep",
                     mask="rand", table="lam12", misalign=(_op, 4)))
EDGE += [
    dict(id="misalign-tape0", shape=(1, 4, 128, 128), rng="tape", flags=1 | 4, dtype=F32, heads="sep", mask="rand",
         table="dt", misalign=("tape0", 4)),
    dict(id="misalign-x-philox", shape=(1, 4, 256, 256), rng="philox", flags=2, dtype=F32, heads="sep", mask="rand",
         table="lam12", misalign=("x", 4)),
    dict(id="misalign8-a-f16", shape=(5, 4, 120, 136), rng="torch", flags=2, dtype=F16, heads="sep", mask="rand",
         table="lam12", misalign=("a", 8)),
    dict(id="misalign8-b-bf16-philox", shape=(5, 4, 120, 136), rng="philox", flags=3, dtype=BF16, heads="sep",
         mask="full", table="lam12", misalign=("b", 8)),
]
# the audio target correction without a split: the only way to reach the corr code of the TMA kernels (the torch
# one in its lane-pair form); rows alternate corrections and 1
EDGE += [
    dict(id="corr-tma-philox-merge", shape=(5, 4, 120, 136), rng="philox", flags=2 | 8, dtype=F32, heads="sep",
         mask="rand", table="lam12", corr=(0.625, 1.3, 1.0, 0.8), family="substep_tma_kernel"),
    dict(id="corr-tma-philox-first-bf16", shape=(5, 4, 120, 136), rng="philox", flags=1, dtype=BF16, heads="null",
         mask="full", table="dt", corr=(1.3, 1.0, 0.625), family="substep_tma_kernel"),
    dict(id="corr-torch-tma-dense", shape=(5, 4, 120, 136), rng="torch", flags=3, dtype=F32, heads="sep", mask="rand",
         table="dt", corr=(0.625, 1.3, 1.0, 0.8), family="substep_torch_tma_kernel"),
    dict(id="corr-torch-tma-packed", shape=(5, 4, 120, 136), rng="torch", flags=2, dtype=BF16, heads="null",
         mask="full", table="lam12", packed=True, corr=(0.8, 1.0, 1.3), family="substep_torch_tma_kernel"),
    dict(id="corr-torch-tma-packed-cfg", shape=(5, 4, 120, 136), rng="torch_state", flags=0 | 4, dtype=F32,
         heads="sep", mask="rand", table="lam01", packed=True, cfg=(4.5, -0.5), corr=(1.3, 0.625),
         family="substep_torch_tma_kernel"),
]
for _i, _c in enumerate(EDGE):
    _c.setdefault("seed", 500 + _i)


# the audio-video flat pack (engine._av_call): shape (lines, 1, n_last), lp_dims (lines, n_last, n_last, n_last, 0,
# split), one uint8 mask element per latent element, 2 * lines table rows (case_table).  tma_min is 0 everywhere, so
# that on the vec4 shapes only the split keeps the TMA kernels away.
def _av_sweep():
    cases = []
    dts = (torch.float32, torch.bfloat16, torch.float16)
    heads = ("sep", "null", "same")
    masks = ("rand", "full", "rand", "known", "rand", "free")
    kinds = (3, 1, 1 | 4, 2, 0, 0 | 4)
    fams = [("av_ldg4_tape", "tape", (4, 1, 4096), 3072), ("av_ldg1_tape", "tape", (3, 1, 2049), 1000),
            ("av_ldg4_philox", "philox", (4, 1, 4096), 3072), ("av_ldg1_philox", "philox", (4, 1, 4096), 3071),
            ("av_torchvec", "torch", (4, 1, 4096), 3072), ("av_torch_scalar", "torch", (3, 1, 2049), 1000)]
    i = 0
    for name, rng, shape, split in fams:
        for flags in kinds + ((3 | 8, 2 | 8) if rng == "philox" else ()):
            cases.append(dict(id=f"{name}-f{flags}", shape=shape, split=split, rng=rng, flags=flags, dtype=dts[i % 3],
                              heads=heads[(i // 3) % 3], mask=masks[i % 6], table=TABLES[i % 3], seed=700 + i,
                              tma_min=0))
            i += 1
    return cases


BIG = 1 << 22
AV_EDGE = [
    # one line of 4 Mi elements split in the middle (the torch stream: four calls per subsequence)
    dict(id="av-big-torch-packed", shape=(1, 1, BIG), split=BIG // 2, rng="torch", flags=2, dtype=F32, heads="sep",
         mask="rand", table="lam12", packed=True),
    dict(id="av-big-torch-first-bf16", shape=(1, 1, BIG), split=BIG // 2, rng="torch", flags=3, dtype=BF16,
         heads="null", mask="rand", table="dt"),
    dict(id="av-big-philox-merge", shape=(1, 1, BIG), split=BIG // 2, rng="philox", flags=2 | 8, dtype=F32,
         heads="sep", mask="rand", table="lam01"),
    dict(id="av-big-tape-f16", shape=(1, 1, BIG), split=BIG // 2, rng="tape", flags=1 | 4, dtype=F16, heads="sep",
         mask="rand", table="lam12"),
    # 16 lines split at 3/4
    dict(id="av-16-torch-packed", shape=(16, 1, 40960), split=30720, rng="torch", flags=3, dtype=F32, heads="sep",
         mask="rand", table="lam12", packed=True),
    dict(id="av-16-philox-cfg", shape=(16, 1, 40960), split=30720, rng="philox", flags=2, dtype=F32, heads="sep",
         mask="full", table="dt", cfg=(4.5, -0.5)),
    dict(id="av-16-tape-aliased-bf16", shape=(16, 1, 40960), split=30720, rng="tape", flags=0 | 4, dtype=BF16,
         heads="same", mask="rand", table="lam01"),
    # a split that is not a multiple of 4 on an n_last that is: the scalar kernels
    dict(id="av-split3071-torch", shape=(4, 1, 4096), split=3071, rng="torch", flags=2, dtype=F32, heads="sep",
         mask="rand", table="lam12"),
    dict(id="av-split3071-philox-merge-bf16", shape=(4, 1, 4096), split=3071, rng="philox", flags=3 | 8, dtype=BF16,
         heads="sep", mask="rand", table="dt"),
    # an odd n_last
    dict(id="av-odd-torch-f16", shape=(3, 1, 2049), split=1000, rng="torch", flags=3, dtype=F16, heads="null",
         mask="rand", table="lam12"),
    dict(id="av-odd-philox-state", shape=(3, 1, 2049), split=1000, rng="philox_state", flags=2, dtype=F32, heads="sep",
         mask="rand", table="lam01"),
    # split == n_last: the audio rows are never read (and the split still keeps TMA away)
    dict(id="av-split-nlast-torch-packed", shape=(4, 1, 4096), split=4096, rng="torch", flags=2, dtype=F32,
         heads="sep", mask="rand", table="lam12", packed=True),
    dict(id="av-split-nlast-philox", shape=(4, 1, 4096), split=4096, rng="philox", flags=3, dtype=F32, heads="sep",
         mask="rand", table="dt"),
    # split == 4
    dict(id="av-split4-torch-state", shape=(4, 1, 4096), split=4, rng="torch_state", flags=3, dtype=F32, heads="sep",
         mask="rand", table="dt"),
    dict(id="av-split4-tape-bf16", shape=(4, 1, 4096), split=4, rng="tape", flags=1, dtype=BF16, heads="sep",
         mask="full", table="lam12"),
    # the torch scalar kernel with two curand_normal4 calls per subsequence
    dict(id="av-odd-torch-calls", shape=(1, 1, 1_200_001), split=600_001, rng="torch", flags=2, dtype=F32, heads="sep",
         mask="rand", table="lam12"),
]
for _i, _c in enumerate(AV_EDGE):
    _c.setdefault("seed", 800 + _i)
    _c.setdefault("tma_min", 0)
AV_CASES = _av_sweep() + AV_EDGE
SUBSTEP_CASES = _sweep() + EDGE + AV_CASES


@pytest.fixture
def options():
    lib = _lib()
    yield lib
    lib.lp_set_option(b"tma", 1)
    lib.lp_set_option(b"tma_min", TMA_MIN)
    lib.lp_set_option(b"tma_boundary", 0)


@pytest.mark.parametrize("c", SUBSTEP_CASES, ids=lambda c: c["id"])
@rerun_on_lost_record
def test_substep_launch(c, cuda_device, options, normal_fast):
    assert options.lp_set_option(b"tma_min", c.get("tma_min", TMA_MIN)) == 0
    assert options.lp_set_option(b"tma", c.get("tma", 1)) == 0
    run_substep(c, cuda_device, normal_fast[1])


# ---------------------------------------------------------------------------------------------------------------
# lp_boundary
# ---------------------------------------------------------------------------------------------------------------
def _boundary_sweep():
    cases, i = [], 0
    dts = (F32, BF16, F16)
    for shape in ((1, 4, 128, 128), (2, 4, 45, 45)):
        for packed in (False, True):
            for dt in dts:
                cases.append(dict(id=f"b{'4' if shape[-1] == 128 else '1'}-{'pk' if packed else 'dense'}-{DTYPES[dt]}",
                                  shape=shape, dtype=dt, packed=packed, combine=None, next=i % 2 == 0, out=True,
                                  euler=True, mask=("rand", "full", "blob")[i % 3], table=TABLES[i % 3], seed=900 + i))
                i += 1
    cases += [
        dict(id="btma-cfg-next", shape=(5, 4, 120, 136), dtype=F32, combine=4.5, next=True, out=True, euler=True,
             tma_boundary=1, mask="rand", table="lam12"),
        dict(id="btma-bf16", shape=(1, 4, 256, 256), dtype=BF16, combine=None, next=False, out=True, euler=True,
             tma_boundary=1, mask="full", table="dt"),
        dict(id="btma-f16-next", shape=(1, 4, 256, 256), dtype=F16, combine=None, next=True, out=False, euler=True,
             tma_boundary=1, mask="blob", table="lam01"),
        dict(id="btma-cfg", shape=(5, 4, 120, 136), dtype=F32, combine=-0.5, next=False, out=False, euler=True,
             tma_boundary=1, mask="full", table="lam12"),
        dict(id="b-replace-only-f16", shape=(40, 4, 50, 50), dtype=F16, combine=None, next=True, out=True, euler=True,
             coef=0.0, mask="full", table="lam12"),
        dict(id="b-out-only", shape=(5, 4, 120, 136), dtype=F32, combine=3.5, next=False, out=True, euler=False,
             mask="blob", table="dt"),
        dict(id="b-flagship-packed-cfg", shape=(128, 4, 128, 128), dtype=F32, combine=5.0, next=True, out=True,
             euler=True, packed=True, mask="rand", table="lam12"),
        dict(id="b-misalign-noise", shape=(1, 4, 128, 128), dtype=F32, combine=None, next=True, out=True, euler=True,
             misalign="noise", mask="rand", table="lam12"),
    ]
    # audio-video flat packs: the next table's rows follow the split; tma_boundary 1, so only the split keeps the
    # TMA boundary kernel away from the vec4 ones
    cases += [
        dict(id="b-av-vec4-dense", shape=(4, 1, 4096), split=3072, dtype=F32, combine=None, next=True, out=True,
             euler=True, tma_boundary=1, mask="rand", table="lam12"),
        dict(id="b-av-vec4-packed-bf16", shape=(16, 1, 40960), split=30720, dtype=BF16, combine=None, next=True,
             out=True, euler=True, packed=True, tma_boundary=1, mask="rand", table="dt"),
        dict(id="b-av-scalar-dense-f16", shape=(3, 1, 2049), split=1000, dtype=F16, combine=None, next=True, out=True,
             euler=True, mask="rand", table="lam01"),
        dict(id="b-av-scalar-packed-cfg", shape=(4, 1, 4096), split=3071, dtype=F32, combine=3.5, next=True,
             out=True, euler=True, packed=True, mask="rand", table="lam12"),
        dict(id="b-av-big-cfg", shape=(1, 1, BIG), split=BIG // 2, dtype=F32, combine=4.5, next=True, out=True,
             euler=True, tma_boundary=1, mask="rand", table="lam12"),
        dict(id="b-av-split-nlast", shape=(4, 1, 4096), split=4096, dtype=F32, combine=None, next=True, out=False,
             euler=True, tma_boundary=1, mask="rand", table="dt"),
    ]
    for j, c in enumerate(cases):
        c.setdefault("seed", 950 + j)
    return cases


def expect_boundary(c, shape, rs, cs):
    sp, total = int(np.prod(shape[2:])), int(np.prod(shape))
    per_row = total // shape[0]
    H = DTYPES[c["dtype"]]
    v4 = (per_row % 4 == 0 and sp % 4 == 0 and rs % 4 == 0 and cs % 4 == 0 and c.get("misalign") is None
          and (c.get("split") or 0) % 4 == 0)
    tma = (v4 and c.get("tma_boundary", 0) and c["euler"] and sp % 16 == 0 and rs % 16 == 0 and cs % 16 == 0
           and total >= TMA_MIN and not c.get("split"))
    if tma:
        return f"boundary_tma_kernel<{H},{int(c['combine'] is not None)},{int(c['next'])},2048,2>"
    return f"boundary_kernel<{4 if v4 else 1},{H},{int(bool(c.get('packed')))}>"


@pytest.mark.parametrize("c", _boundary_sweep(), ids=lambda c: c["id"])
@rerun_on_lost_record
def test_boundary_launch(c, cuda_device, options):
    from lanpaint_b200 import _native
    lib = options
    assert lib.lp_set_option(b"tma_boundary", c.get("tma_boundary", 0)) == 0
    dev, shape = cuda_device, c["shape"]
    total = int(np.prod(shape))
    gen = torch.Generator(device=dev).manual_seed(c["seed"])
    m8, known, rs, cs = make_mask(shape, c["mask"], gen, dev)
    dims = dims_of(shape, rs, cs, c.get("split"))
    tab, rows = case_table(c, shape, dev)
    a32, b32, y, nz, x = (torch.randn(shape, device=dev, generator=gen) for _ in range(5))
    a, b = a32.to(c["dtype"]), b32.to(c["dtype"])
    nz = offset_copy(nz, 4 if c.get("misalign") == "noise" else 0)
    x_in = x.clone()
    coef = c.get("coef", -0.37)
    out = torch.full(shape, float("nan"), device=dev) if c["out"] else None
    cfg = c["combine"]
    hd = _native.Heads(a.data_ptr(), b.data_ptr() if cfg is not None else None, LP_DT[c["dtype"]],
                       1 if cfg is not None else 0, cfg or 0.0, cfg or 0.0)
    want_name = expect_boundary(c, shape, rs, cs)
    xp = P(x.data_ptr()) if c["euler"] else None
    nt = P(tab.data_ptr()) if c["next"] else None
    if c.get("packed"):
        kn, keep = pack_known(m8, dims, y, nz, total)
        yd, nd = torch.full_like(y, float("nan")), torch.full_like(nz, float("nan"))   # must not be read

        def call():
            return lib.lp_boundary_known(C.byref(hd), P(yd.data_ptr()), P(nd.data_ptr()) if c["next"] else None,
                                         P(m8.data_ptr()), C.byref(kn), xp, P(out.data_ptr()) if out is not None else None,
                                         C.c_float(coef), nt, C.byref(dims), _stream())
    else:
        def call():
            return lib.lp_boundary(C.byref(hd), P(y.data_ptr()), P(nz.data_ptr()) if c["next"] else None,
                                   P(m8.data_ptr()), xp, P(out.data_ptr()) if out is not None else None,
                                   C.c_float(coef), nt, C.byref(dims), _stream())
    want = R.boundary(a, b if cfg is not None else None, y, nz if c["next"] else None, known,
                      x_in if c["euler"] else None, coef, tab if c["next"] else None, cfg=cfg, rows=rows)
    got = launched(call, c.get("split"))
    fam = family(want_name)
    if out is not None:
        assert torch.equal(_bits(out[known]), _bits(y[known])), f"{c['id']}: out != y at known positions"
        _check(fam, f"{c['id']} out", out, want["out"])
    if c["euler"]:
        _check(fam, f"{c['id']} x", x, want["x"])
        if c["next"] and coef == 0.0:
            assert torch.equal(_bits(x[~known]), _bits(x_in[~known])), f"{c['id']}: replace step touched free positions"
    else:
        assert torch.equal(_bits(x), _bits(x_in))
    assert_kernel(c["id"], got, want_name)
    RAN.add(c["id"])


# ---------------------------------------------------------------------------------------------------------------
# lp_prologue_f32, lp_advance_f32, lp_stop_stats_f32
# ---------------------------------------------------------------------------------------------------------------
def _prologue(shape, mask, copy, dev, split=None):
    lib = _lib()
    gen = torch.Generator(device=dev).manual_seed(77)
    m8, known, rs, cs = make_mask(shape, mask, gen, dev)
    dims = dims_of(shape, rs, cs, split)
    tab, rows = case_table(dict(table="lam12", seed=3, split=split), shape, dev)
    x, y, nz = (torch.randn(shape, device=dev, generator=gen) for _ in range(3))
    xm = torch.full(shape, float("nan"), device=dev)
    xc = torch.full(shape, float("nan"), device=dev) if copy else None
    got = launched(lambda: lib.lp_prologue_f32(P(x.data_ptr()), P(y.data_ptr()), P(nz.data_ptr()), P(m8.data_ptr()),
                                               P(xm.data_ptr()), P(xc.data_ptr()) if copy else None, P(tab.data_ptr()),
                                               C.byref(dims), _stream()), split)
    assert torch.equal(_bits(xm[~known]), _bits(x[~known])), "the replace step touched free positions"
    _check("prologue_kernel", f"prologue {shape} split {split}", xm, R.prologue(x, y, nz, known, tab, rows=rows))
    if copy:
        assert torch.equal(_bits(xc), _bits(xm))
    v4 = shape[-1] % 4 == 0 and (split or 0) % 4 == 0
    cid = f"prologue{shape}" + (f"-split{split}" if split is not None else "")
    assert_kernel(cid, got, f"prologue_kernel<{4 if v4 else 1}>")
    RAN.add(cid)


@pytest.mark.parametrize("shape,mask,copy", [((1, 4, 128, 128), "full", True), ((2, 4, 45, 45), "rand", False),
                                            ((5, 4, 120, 136), "blob", True)])
@rerun_on_lost_record
def test_prologue_launch(shape, mask, copy, cuda_device):
    _prologue(shape, mask, copy, cuda_device)


AV_PROLOGUE = [((4, 1, 4096), 3072, True), ((3, 1, 2049), 1000, False), ((4, 1, 4096), 3071, False)]


@pytest.mark.parametrize("shape,split,copy", AV_PROLOGUE)
@rerun_on_lost_record
def test_av_prologue_launch(shape, split, copy, cuda_device):
    """The replace step of an audio-video pack: rep_noise / rep_y of each element's own row (audio or video)."""
    _prologue(shape, "rand", copy, cuda_device, split)


ADVANCE = [
    dict(id="adv-tape", shape=(1, 4, 128, 128), rng="tape", half=1, mask="rand"),
    dict(id="adv-philox", shape=(5, 4, 120, 136), rng="philox", half=0, mask="full"),
    dict(id="adv-philox-state", shape=(2, 4, 45, 45), rng="philox_state", half=1, mask="blob"),
    dict(id="adv-torch-pastcap", shape=(1, 4, 272, 256), rng="torch", half=1, mask="rand"),
    dict(id="adv-torch-wan", shape=(1, 16, 21, 80, 45), rng="torch", half=0, mask="full"),
    dict(id="adv-torch-flagship-state", shape=(128, 4, 128, 128), rng="torch_state", half=1, mask="rand"),
    # audio-video flat packs
    dict(id="adv-av-tape", shape=(4, 1, 4096), split=3072, rng="tape", half=1, mask="rand"),
    dict(id="adv-av-philox-odd", shape=(3, 1, 2049), split=1000, rng="philox", half=0, mask="rand"),
    dict(id="adv-av-torch-16", shape=(16, 1, 40960), split=30720, rng="torch", half=1, mask="rand"),
    dict(id="adv-av-torch-state-big", shape=(1, 1, BIG), split=BIG // 2 + 1, rng="torch_state", half=0, mask="rand"),
]


@pytest.mark.parametrize("c", ADVANCE, ids=lambda c: c["id"])
@rerun_on_lost_record
def test_advance_launch(c, cuda_device, normal_fast):
    """lp_advance_f32 on all three streams -- advance_torch_kernel is what the early-stop loop runs under the
    default torch stream -- with the torch draws from torch.randn and the philox ones from the restatement."""
    from lanpaint_b200 import _native
    lib = _lib()
    dev, shape = cuda_device, c["shape"]
    total = int(np.prod(shape))
    gen = torch.Generator(device=dev).manual_seed(len(c["id"]) * 131)
    m8, known, rs, cs = make_mask(shape, c["mask"], gen, dev)
    dims = dims_of(shape, rs, cs, c.get("split"))
    tab, rows = case_table(dict(table="dt" if c["half"] else "lam12", seed=5, split=c.get("split")), shape, dev)
    x, cc = torch.randn(shape, device=dev, generator=gen) * 2, torch.randn(shape, device=dev, generator=gen) * 3
    r, keep, slack, seed = _native.Rng(), [], 0.0, 4242
    if c["rng"] == "tape":
        xi = torch.randn(shape, device=dev, generator=gen)
        r.mode, r.tape0 = _native.RNG_TAPE, xi.data_ptr()
        want_name = "advance_kernel<0>"
    elif c["rng"].startswith("philox"):
        base = 9 if c["rng"] == "philox_state" else 0
        xi = torch.from_numpy(R.philox_normals(total, seed, base + 3)).to(dev).view(shape)
        r.mode, r.seed, r.draw0 = _native.RNG_PHILOX, seed, 3
        if base:
            st = torch.tensor([seed, base], dtype=torch.int64, device=dev)
            keep.append(st)
            r.seed, r.state = 0, st.data_ptr()
        want_name = "advance_kernel<1>"
        nd = len(shape)
        sd = R._cls(tab, known, R.C_SH if c["half"] else R.C_SF, nd, rows).abs() * R._row(tab, R.T_S, nd, rows).abs()
        slack = sd * normal_fast[1]
    else:
        base = 4 * 1001 if c["rng"] == "torch_state" else 0
        g = torch.Generator(device=dev).manual_seed(seed)
        g.set_offset(base)
        xi = torch.randn(shape, device=dev, generator=g)
        r.mode, r.seed, r.draw0 = _native.RNG_TORCH, seed, base
        if base:
            st = torch.tensor([seed, base], dtype=torch.int64, device=dev)
            keep.append(st)
            r.seed, r.state, r.draw0 = 0, st.data_ptr(), 0
        want_name = "advance_torch_kernel"
    want = R.advance(x, cc, known, tab, xi, c["half"], rows=rows)
    got = launched(lambda: lib.lp_advance_f32(P(x.data_ptr()), P(cc.data_ptr()), P(m8.data_ptr()), P(tab.data_ptr()),
                                              C.byref(dims), C.byref(r), c["half"], _stream()), c.get("split"))
    _check(family(want_name), c["id"], x, want, slack=slack)
    assert_kernel(c["id"], got, want_name)
    RAN.add(c["id"])


def _stop_stats(shape, bcast, dev, split=None):
    lib = _lib()
    gen = torch.Generator(device=dev).manual_seed(61)
    m8, known, rs, cs = make_mask(shape, "rand" if bcast else "full", gen, dev)
    ring8 = (torch.rand(m8.shape, device=dev, generator=gen) < 0.2).to(torch.uint8)
    dims = dims_of(shape, rs, cs, split)
    tab, rows = case_table(dict(table="lam12", seed=2, split=split), shape, dev)
    a, b = torch.randn(shape, device=dev, generator=gen), torch.randn(shape, device=dev, generator=gen)
    sums = torch.zeros(2, dtype=torch.float64, device=dev)
    got = launched(lambda: lib.lp_stop_stats_f32(P(a.data_ptr()), P(b.data_ptr()), P(m8.data_ptr()),
                                                 P(ring8.data_ptr()), P(tab.data_ptr()), C.byref(dims),
                                                 P(sums.data_ptr()), _stream()), split)
    want = R.stop_stats(a, b, known, ring8.bool().expand(shape), tab, rows=rows)
    for k in range(2):
        rel = abs(float(sums[k]) - want[k]) / want[k]
        WORST["stop_stats_kernel"] = max(WORST["stop_stats_kernel"], rel / R.U32)
        assert rel <= 48 * R.U32, (k, float(sums[k]), want[k])
    v4 = shape[-1] % 4 == 0 and (split or 0) % 4 == 0
    cid = f"stats{shape}" + (f"-split{split}" if split is not None else "")
    assert_kernel(cid, got, f"stop_stats_kernel<{4 if v4 else 1}>")
    RAN.add(cid)


@pytest.mark.parametrize("shape,bcast", [((128, 4, 128, 128), False), ((2, 4, 45, 45), True)])
@rerun_on_lost_record
def test_stop_stats_launch(shape, bcast, cuda_device):
    """lp_stop_stats_f32 with the inv_S table the engine passes and a full-shape ring, against fp64 sums.  Every
    term is non-negative, so the fp32 partial sums (a grid-stride chain of at most ~40 additions per thread, then
    the warp and block trees) stay within 48 * 2^-24 of the fp64 sum."""
    _stop_stats(shape, bcast, cuda_device)


AV_STATS = [((16, 1, 40960), 30720), ((3, 1, 2049), 1000)]


@pytest.mark.parametrize("shape,split", AV_STATS)
@rerun_on_lost_record
def test_av_stop_stats_launch(shape, split, cuda_device):
    """The early-stop statistics of an audio-video pack: inv_S of each element's own row, with a ring."""
    _stop_stats(shape, True, cuda_device, split)


# ---------------------------------------------------------------------------------------------------------------
# coverage
# ---------------------------------------------------------------------------------------------------------------
KINDS = ((1, 1), (1, 0), (0, 1), (0, 0))


def _required_split():
    """Every instantiation a launch with a row split can reach: the LDG and torch-LDG kernels (no TMA kernel)."""
    req = set()
    for N in (4, 1):
        for f, n in KINDS:
            req.add(("substep_kernel", f"{N},0,{f},{n},0"))
            req.add(("substep_kernel", f"{N},1,{f},{n},0"))
        req.add(("substep_kernel", f"{N},1,1,1,1"))
        req.add(("substep_kernel", f"{N},1,0,1,1"))
    for f, n in KINDS:
        req.add(("substep_torchvec_kernel", f"{f},{n}"))
        req.add(("substep_torch_kernel", f"{f},{n}"))
    for N in (4, 1):
        for pk in (0, 1):
            req.add(("boundary_kernel", f"{N},{pk}"))
    for s in ("prologue_kernel<4>", "prologue_kernel<1>", "advance_kernel<0>", "advance_kernel<1>",
              "advance_torch_kernel", "stop_stats_kernel<4>", "stop_stats_kernel<1>"):
        req.add((s, ""))
    return req


def _required():
    req = _required_split()
    for f, n, mg in ((1, 1, 1), (1, 1, 0), (0, 1, 1), (0, 1, 0), (1, 0, 0), (0, 0, 0)):
        req.add(("substep_tma_kernel", f"{f},{n},{mg},2048,2,2"))
    for f, n in KINDS:
        for pk in (0, 1):
            req.add(("substep_torch_tma_kernel", f"{f},{n},{pk}"))
    req.add(("boundary_tma_kernel", None))
    return req


HEAD_FAMILIES = ("substep_kernel", "substep_tma_kernel", "substep_torch_tma_kernel", "substep_torchvec_kernel",
                 "substep_torch_kernel", "boundary_kernel", "boundary_tma_kernel")


def _split(name):
    """canonical name -> (family, head type or None, the other template arguments)."""
    fam = family(name)
    if "<" not in name or fam not in HEAD_FAMILIES:
        return name, None, ""
    args = name[len(fam) + 1:-1].split(",")
    h = 1 if fam in ("substep_kernel", "boundary_kernel") else 0
    return fam, args[h], ",".join(args[:h] + args[h + 1:])


def _seen(counter):
    seen = set()
    heads = collections.defaultdict(set)
    for name in counter:
        fam, h, rest = _split(name)
        seen.add((fam, rest))
        seen.add((fam, None))
        if h is not None:
            heads[fam].add(h)
    return seen, heads


def test_kernel_coverage():
    """The union of the kernels the cases above ran covers every production-reachable instantiation of the update
    kernels (the measurement-only philox tile geometries, "tma" 2..5, excluded) and every head type per family; the
    cases with a row split ran every instantiation a split can reach, and never a TMA kernel."""
    n_cases = len(SUBSTEP_CASES) + len(_boundary_sweep()) + 3 + len(AV_PROLOGUE) + len(ADVANCE) + 2 + len(AV_STATS)
    if len(RAN) < n_cases:
        pytest.skip(f"only {len(RAN)} of the {n_cases} launch cases ran in this session")
    seen, heads = _seen(SEEN)
    print("\nkernels seen (launches):")
    for name in sorted(SEEN):
        print(f"  {SEEN[name]:3d}  {name}")
    print("largest |got - want| / (2^-24 magnitude) per family:")
    for fam in sorted(WORST):
        print(f"  {fam:28s} {WORST[fam]:.3g}")
    missing = sorted(str(r) for r in _required() if r not in seen)
    assert not missing, missing
    seen_split, _ = _seen(SEEN_SPLIT)
    missing = sorted(str(r) for r in _required_split() if r not in seen_split)
    print(f"row-split launches: {sum(SEEN_SPLIT.values())}, instantiations missing: {missing}")
    assert not missing, missing
    assert not [n for n in SEEN_SPLIT if "tma" in n], sorted(SEEN_SPLIT)
    for fam in HEAD_FAMILIES:
        assert heads[fam] == set(DTYPES.values()), (fam, heads[fam])
