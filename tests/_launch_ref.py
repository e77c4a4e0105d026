"""fp64 restatement of ONE launch of each device entry point of include/lanpaint_b200.h (test infrastructure).

The launch-level tests (tests/test_gpu_launch_ref.py) compare every dispatched kernel with these functions, element
by element.  The restatement follows the header's contract and the oracle's functions (branch_coefficients,
ou_advance, the masked score), in the table form the kernels use:
    C = c_tgt * tgt + g * x_t,    tgt = known ? (1 + lam) y - lam x0_BIG : x0
and it reads every per-element coefficient from the same fp32 table row the kernel reads (LP_T_* / LP_C_*), so it
checks the kernels, not lp_build_coef_table (tests/test_table_properties.py covers the table).

Table rows: by default element b of the leading axis reads row b (the tensors are shaped so that the leading axis is
lp_dims.n_rows).  With a row split (the audio-video flat pack), pass rows = split_rows(shape, row_split): the
per-element row index, n_rows + b at positions >= row_split within row b.  The audio target correction LP_T_CORR
is restated as the kernel and the oracle's masked_score apply it: x0' = x + corr (x0 - x) on the model-space x,
after the CFG combine, on both heads.

Each function returns the fp64 value and, for the fp32 outputs, the magnitude chain: the same expression evaluated
on the absolute values of every operand and coefficient with subtractions turned into additions.  A kernel that
evaluates the expression in fp32 with n roundings on the longest path is within n * 2^-24 * magnitude of the fp64
value, which is the per-element bound the tests apply (`within`).

Noise is produced without the library: the tape tensors as they are, torch.randn for the torch stream, and a
restatement of Philox4x32-10 (numpy, integer arithmetic) with an fp64 Box-Muller of the kernel's own fp32 u and v
for the philox stream.
"""
from __future__ import annotations

import re

import numpy as np
import torch

U32 = 2.0 ** -24   # unit round-off of fp32


def canon(name: str) -> str:
    """A profiler's kernel name -> the canonical spelling the tests assert on:
    'void lp::substep_kernel<(int)4, float, (bool)1, ...>(lp::SubstepArgs)' (or the true/false spelling)
    -> 'substep_kernel<4,float,1,...>'."""
    n = name.split("lp::", 1)[1]
    n = n[: n.index(">") + 1] if "<" in n.split("(")[0] else n.split("(")[0]
    n = n.replace("(bool)", "").replace("(int)", "").replace("true", "1").replace("false", "0").replace(" ", "")
    return re.sub(r"(\d+)u\b", r"\1", n)

# table layout (include/lanpaint_b200.h)
T_CTGT, T_S, T_INVS, T_LAM, T_ONEPLAM, T_REPN, T_REPY, T_CORR = 0, 1, 2, 3, 4, 5, 6, 7
T_CLS0, T_CLS1, T_SDM, T_SDMF = 8, 16, 24, 26
C_G, C_DT, C_EF, C_KF, C_SF, C_EH, C_KH, C_SH = range(8)
FIRST, FUSE_NEXT, STORE_C, MERGE_NOISE = 1, 2, 4, 8


# ---------------------------------------------------------------------------------------------------------------
# Philox4x32-10 and the two Box-Muller transforms
# ---------------------------------------------------------------------------------------------------------------
_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
_LO = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr: np.ndarray, key) -> np.ndarray:
    """Philox4x32-10 (Salmon et al., SC'11) of counters ctr [n, 4] (uint32) under key (k0, k1): [n, 4] uint32."""
    c = [ctr[:, j].astype(np.uint64) for j in range(4)]
    k0, k1 = int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF
    for r in range(10):
        p0, p1 = _M0 * c[0], _M1 * c[2]
        kx, ky = np.uint64((k0 + r * _W0) & 0xFFFFFFFF), np.uint64((k1 + r * _W1) & 0xFFFFFFFF)
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ kx, p1 & _LO, (p0 >> np.uint64(32)) ^ c[3] ^ ky, p0 & _LO]
    return np.stack(c, axis=1).astype(np.uint32)


_KU = np.float32(2.3283064e-10)
_KV = np.float32(np.float32(2.3283064e-10) * np.float32(6.2831855))


def _uv(a: np.ndarray, b: np.ndarray):
    """The fp32 u in (0, 1] and v in (0, 2 pi] both Box-Muller forms start from: one fused multiply-add each."""
    u = (a.astype(np.float32).astype(np.float64) * float(_KU) + float(_KU) / 2).astype(np.float32)
    v = (b.astype(np.float32).astype(np.float64) * float(_KV) + float(_KV) / 2).astype(np.float32)
    return u.astype(np.float64), v.astype(np.float64)


def box_muller64(a: np.ndarray, b: np.ndarray):
    """fp64 Box-Muller of the words (a, b): (s sin v, s cos v), s = sqrt(-2 log u)."""
    u, v = _uv(a, b)
    s = np.sqrt(-2.0 * np.log(u))
    return s * np.sin(v), s * np.cos(v)


def _normals_of(words: np.ndarray) -> np.ndarray:
    """[n, 4] words -> [n, 4] normals in curand_normal4's order: (x, y) -> 0, 1 and (z, w) -> 2, 3."""
    s0, c0 = box_muller64(words[:, 0], words[:, 1])
    s1, c1 = box_muller64(words[:, 2], words[:, 3])
    return np.stack([s0, c0, s1, c1], axis=1)


def philox_normals(n: int, seed: int, draw: int) -> np.ndarray:
    """LP_RNG_PHILOX: element i <- component i & 3 of Philox(counter = (i >> 2, 0, draw lo, draw hi), key = seed)."""
    q = (n + 3) // 4
    ctr = np.zeros((q, 4), dtype=np.uint32)
    ctr[:, 0] = np.arange(q, dtype=np.uint64).astype(np.uint32)
    ctr[:, 2], ctr[:, 3] = draw & 0xFFFFFFFF, (draw >> 32) & 0xFFFFFFFF
    w = philox4x32_10(ctr, (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF))
    return _normals_of(w).reshape(-1)[:n]


def torch_stream_normals(n: int, seed: int, offset: int, T: int) -> np.ndarray:
    """torch.randn's CUDA stream restated: element li belongs to thread t = li mod T, call k = li div 4T, component
    (li div T) mod 4 of curand_normal4 on subsequence t, i.e. Philox(counter = (offset/4 + k lo, hi, t, 0), seed)."""
    li = np.arange(n, dtype=np.int64)
    t, k, comp = li % T, li // (4 * T), (li // T) % 4
    calls = int(k.max()) + 1
    tt, kk = np.meshgrid(np.arange(T, dtype=np.int64), np.arange(calls, dtype=np.int64), indexing="ij")
    ctr64 = offset // 4 + kk.reshape(-1)
    ctr = np.stack([ctr64 & 0xFFFFFFFF, ctr64 >> 32, tt.reshape(-1), np.zeros_like(ctr64)], axis=1).astype(np.uint32)
    z = _normals_of(philox4x32_10(ctr, (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)))   # [(t, k), 4]
    return z[t * calls + k, comp]


# ---------------------------------------------------------------------------------------------------------------
# per-element coefficients out of the fp32 table
# ---------------------------------------------------------------------------------------------------------------
def split_rows(shape, row_split: int, device=None) -> torch.Tensor:
    """The table row of every element of a launch with lp_dims.n_rows = shape[0], per_row = the rest of the shape and
    lp_dims.row_split = row_split: b, or n_rows + b at positions r >= row_split of row b (row_split 0 = off)."""
    n_rows, per_row = shape[0], int(np.prod(shape[1:]))
    b = torch.arange(n_rows, device=device).view(-1, 1)
    r = torch.arange(per_row, device=device).view(1, -1)
    rows = b + (n_rows * (r >= row_split) if row_split else 0 * r)
    return rows.reshape(shape)


def _row(tab: torch.Tensor, col: int, ndim: int, rows=None) -> torch.Tensor:
    if rows is not None:
        return tab[:, col].double()[rows]
    return tab[:, col].double().view((-1,) + (1,) * (ndim - 1))


def _cls(tab, known, col, ndim, rows=None):
    return torch.where(known, _row(tab, T_CLS1 + col, ndim, rows), _row(tab, T_CLS0 + col, ndim, rows))


class _Val:
    """Arithmetic of the value pass."""
    abs = staticmethod(lambda t: t)
    sub = staticmethod(lambda a, b: a - b)


class _Mag:
    """Arithmetic of the magnitude pass: operands enter as absolute values, a - b costs |a| + |b|."""
    abs = staticmethod(lambda t: t.abs() if torch.is_tensor(t) else abs(t))
    sub = staticmethod(lambda a, b: a + b)


def _substep_expr(m, x, a, b, y, cp, xi1, xi2, tab, known, flags, cfg, rows):
    """lp_substep of the header, in the arithmetic m: (x', C', x_t + score)."""
    nd = x.ndim
    A = m.abs
    row = lambda col: A(_row(tab, col, nd, rows))
    cls = lambda col: A(_cls(tab, known, col, nd, rows))
    first, nxt, merge = bool(flags & FIRST), bool(flags & FUSE_NEXT), bool(flags & MERGE_NOISE)
    if cfg is not None:   # x0 = uncond + (cond - uncond) * cfg ; x0_BIG = uncond + (cond - uncond) * cfg_big
        d = m.sub(a, b)
        a, b = b + d * A(cfg[0]), b + d * A(cfg[1])
    if bool(torch.any(tab[:, T_CORR] != 1)):   # audio rows: x0 = x + corr (x0 - x) on both heads, model-space x
        corr = _row(tab, T_CORR, nd, rows)
        on = corr != 1
        a = torch.where(on, x + A(corr) * m.sub(a, x), a)
        b = torch.where(on, x + A(corr) * m.sub(b, x), b)
    lam, opl = row(T_LAM), row(T_ONEPLAM)
    tgt = torch.where(known, m.sub(opl * y, lam * b), a)                      # x_t + score (masked score)
    xt = x * row(T_INVS)                                                       # model space -> x_t
    cn = row(T_CTGT) * tgt + cls(C_G) * xt                                     # Coef_C, table form
    full = first
    e1, k1, s1 = (cls(c) for c in ((C_EF, C_KF, C_SF) if full else (C_EH, C_KH, C_SH)))
    e2, k2, s2 = (cls(c) for c in (C_EH, C_KH, C_SH))
    if not first:                                                              # x += (Cn - C) dt, advance with old C
        xt = xt + m.sub(cn, cp) * cls(C_DT)
    c_adv = cn if first else cp
    if merge:   # both kicks as one Gaussian of the summed variance, after the second advance
        col = T_SDMF if first else T_SDM
        sm = torch.where(known, row(col + 1), row(col))
        xt = e1 * xt + k1 * c_adv
        xt = e2 * xt + k2 * cn + sm * xi1
    else:
        xt = e1 * xt + k1 * c_adv + s1 * xi1                                   # ou_advance
        if nxt:
            xt = e2 * xt + k2 * cn + s2 * xi2
    return xt * row(T_S), cn, tgt


def _d(t):
    return None if t is None else (t.double() if torch.is_tensor(t) else torch.as_tensor(t, dtype=torch.float64))


def substep(x, a, b, y, known, cprev, tab, xi1, xi2, flags, cfg=None, noise_err=0.0, rows=None):
    """One lp_substep launch.  a, b: the heads as the kernel reads them (widened here; b None = aliased);
    cfg = (cfg, cfg_big) when a, b are cond / uncond.  xi1 / xi2: the draws (fp64 or fp32 tensors).
    noise_err: largest error of each kernel draw against xi (the philox transform's).  rows: see split_rows.
    Returns dict(x, c, x0e) of (value, magnitude) pairs and x_slack, the absolute error noise_err can cause in x."""
    b = a if b is None else b
    z = torch.zeros((), dtype=torch.float64, device=x.device)
    cp = z if cprev is None or flags & FIRST else _d(cprev)
    xi2 = z if xi2 is None else _d(xi2)
    ops = [_d(x), _d(a), _d(b), _d(y), cp, _d(xi1), xi2]
    val = _substep_expr(_Val, *ops, tab, known, flags, cfg, rows)
    mag = _substep_expr(_Mag, *[o.abs() for o in ops], tab, known, flags, cfg, rows)
    slack = 0.0
    if noise_err:   # the chain is linear in the draws: its magnitude with every other operand 0
        zx = torch.zeros_like(ops[0])
        ne = torch.full_like(zx, noise_err)
        slack = _substep_expr(_Mag, zx, zx, zx, zx, zx, ne, ne, tab, known, flags, cfg, rows)[0]
    return {"x": (val[0], mag[0]), "c": (val[1], mag[1]), "x0e": (val[2], mag[2]), "x_slack": slack}


def advance(x, c, known, tab, xi, half, rows=None):
    """lp_advance_f32: x_t = x / S ; x_t = e x_t + k C + sd xi ; x = x_t S  (ou_advance over dt or dt/2)."""
    def expr(m, x, c, xi):
        A, nd = m.abs, x.ndim
        cols = (C_EH, C_KH, C_SH) if half else (C_EF, C_KF, C_SF)
        e, k, sd = (A(_cls(tab, known, col, nd, rows)) for col in cols)
        xt = x * A(_row(tab, T_INVS, nd, rows))
        return (e * xt + k * c + sd * xi) * A(_row(tab, T_S, nd, rows))
    ops = [_d(x), _d(c), _d(xi)]
    return expr(_Val, *ops), expr(_Mag, *[o.abs() for o in ops])


def prologue(x, y, noise, known, tab, rows=None):
    """lp_prologue_f32: x_model = known ? rep_noise * noise + rep_y * y : x."""
    nd = x.ndim
    rn, ry = _row(tab, T_REPN, nd, rows), _row(tab, T_REPY, nd, rows)
    val = torch.where(known, rn * _d(noise) + ry * _d(y), _d(x))
    mag = torch.where(known, rn.abs() * _d(noise).abs() + ry.abs() * _d(y).abs(), _d(x).abs())
    return val, mag


def boundary(a, b, y, noise, known, x, coef, next_tab, cfg=None, rows=None):
    """lp_boundary: d = combine ? b + (a - b) cfg : a ; out = known ? y : d ; x = x + (x - out) coef (x given) ;
    x = known ? rep_noise * noise + rep_y * y : x (next_tab given).  -> dict(out, x) of (value, magnitude)."""
    def expr(m, a, b, y, noise, x):
        A = m.abs
        d = b + m.sub(a, b) * A(cfg) if cfg is not None else a
        out = torch.where(known, y, d)
        if x is None:
            return out, None
        x = x + m.sub(x, out) * A(coef)
        if next_tab is not None:
            nd = x.ndim
            rn, ry = A(_row(next_tab, T_REPN, nd, rows)), A(_row(next_tab, T_REPY, nd, rows))
            x = torch.where(known, rn * noise + ry * y, x)
        return out, x
    z = torch.zeros((), dtype=torch.float64, device=y.device)
    ops = [_d(a), z if b is None else _d(b), _d(y), z if noise is None else _d(noise), _d(x)]
    val = expr(_Val, *ops)
    mag = expr(_Mag, *[None if o is None else o.abs() for o in ops])
    return {"out": (val[0], mag[0]), "x": (val[1], mag[1])}


def stop_stats(a, b, known, ring, tab, rows=None):
    """lp_stop_stats_f32: (sum over free elements, sum over ring elements) of (inv_S (a - b))^2, fp64."""
    d2 = ((_d(a) - _d(b)) * (_row(tab, T_INVS, a.ndim, rows) if tab is not None else 1.0)) ** 2
    s_in = float(torch.where(known, torch.zeros_like(d2), d2).sum())
    s_ring = float(torch.where(ring, d2, torch.zeros_like(d2)).sum()) if ring is not None else 0.0
    return s_in, s_ring


def within(got: torch.Tensor, want_mag, k: float, slack=0.0):
    """Largest (|got - want| - slack) / (U32 * magnitude) over the elements (0 where both vanish), and the flat index
    of the first element outside k * U32 * magnitude + slack (None if there is none; a non-finite got is outside)."""
    want, mag = want_mag
    err = (got.double() - want).abs()
    bad = ~(err <= k * U32 * mag + slack)
    over = (err - slack).clamp_min(0.0)
    ratio = torch.where(mag > 0, over / (U32 * mag), torch.where(over > 0, torch.full_like(err, float("inf")), over))
    worst = float(ratio.max()) if ratio.numel() else 0.0
    first_bad = None
    if bool(bad.any()):
        first_bad = int(torch.nonzero(bad.reshape(-1))[0])
    return worst, first_bad
