"""CPU checks of tests/_launch_ref.py, the fp64 per-launch restatement the GPU launch tests compare kernels with:
its Philox4x32-10 against published known-answer vectors, its two noise mappings against direct evaluation, and its
sub-step / advance / boundary against the oracle's fp32 functions on tiny tensors."""
import numpy as np
import pytest
import torch

import _launch_ref as R
from oracle import langevin_oracle as O


def test_philox_known_answers():
    # Random123 kat_vectors, philox4x32 with 10 rounds: (counter, key) -> output
    kat = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
           ((0xffffffff,) * 4, (0xffffffff, 0xffffffff), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
           ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
            (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, want in kat:
        got = R.philox4x32_10(np.array([ctr], dtype=np.uint32), key)[0]
        assert tuple(int(v) for v in got) == want


def test_noise_mappings_follow_their_counters():
    seed = 0x1234_5678_9ABC
    key = (seed & 0xFFFFFFFF, seed >> 32)
    # philox stream: element i <- component i & 3 of counter (i >> 2, 0, draw lo, draw hi)
    draw = (5 << 32) | 7
    z = R.philox_normals(23, seed, draw)
    for i in (0, 1, 2, 3, 4, 13, 22):
        w = R.philox4x32_10(np.array([[i >> 2, 0, 7, 5]], dtype=np.uint32), key)[0]
        s, c = R.box_muller64(w[2 * ((i & 3) >> 1):][:1], w[2 * ((i & 3) >> 1) + 1:][:1])
        assert z[i] == (s if i % 2 == 0 else c)[0]
    # torch stream: element li <- thread li mod T, call li div 4T, component (li div T) mod 4
    T, off, n = 8, 12, 8 * 4 * 2 + 5
    z = R.torch_stream_normals(n, seed, off, T)
    for li in (0, 7, 8, 31, 32, 47, n - 1):
        t, k, q = li % T, li // (4 * T), (li // T) % 4
        ctr = off // 4 + k
        w = R.philox4x32_10(np.array([[ctr & 0xFFFFFFFF, ctr >> 32, t, 0]], dtype=np.uint32), key)[0]
        s, c = R.box_muller64(w[2 * (q >> 1):][:1], w[2 * (q >> 1) + 1:][:1])
        assert z[li] == (s if q % 2 == 0 else c)[0]
    # the transform's range: u in (0, 1] (u == 1 gives an exact 0), |normal| below sqrt(-2 log 2^-33)
    edge = np.array([0, 1, 0x7fffffff, 0xffffff7f, 0xffffff80, 0xffffffff], dtype=np.uint32)
    s, c = R.box_muller64(edge, edge)
    assert np.all(np.isfinite(s)) and np.all(np.abs(np.hypot(s, c)) <= np.sqrt(-2 * np.log(2.0 ** -33)) + 1e-12)
    assert s[-1] == 0.0 and c[-1] == 0.0


def _table(beta=1.5, lam=5.0):
    from lanpaint_b200.schedule import Hyper, build_table
    sig = torch.tensor([0.3, 4.0])
    ve, abt, _ = O.times_from_sigma(sig, False)
    tab = build_table(abt.numpy(), ve.numpy(), Hyper(0.2, lam, beta, 1.0, False), rep_noise=sig.numpy(),
                      rep_y=np.ones(2))
    return torch.from_numpy(tab), sig, ve, abt


def _oracle_coefs(abt, ve, mask, lam, beta):
    abt_b = abt.double().view(-1, 1, 1)
    Sx = (1 + ve.double() ** 2).sqrt().view(-1, 1, 1)
    step = 0.2 * (1 - abt_b).clamp(min=1.0)
    cf = O.branch_coefficients(abt_b, step, torch.ones_like(abt_b), torch.full_like(abt_b, beta), lam)
    A = cf.A_x * (1 - mask) + cf.A_y * mask
    D = cf.D_x * (1 - mask) + cf.D_y * mask
    dt = cf.half_dt_x * (1 - mask) + cf.half_dt_y * mask
    return abt_b, Sx, A, D, dt


def test_substep_restatement_matches_the_oracle():
    """FIRST (one full advance) and a steady post-model half (flags 0), table form against the oracle's
    langevin_substep in its own form, fp32 operands, fp64 arithmetic on both sides."""
    lam, beta = 5.0, 1.5
    tab, sig, ve, abt = _table(beta, lam)
    g = torch.Generator().manual_seed(3)
    B, Cc, S = 2, 3, 10
    x, x0, x0b, y, xi1, xi2, cprev = (torch.randn(B, Cc, S, generator=g) for _ in range(7))
    known = torch.rand(B, 1, S, generator=g) < 0.5
    mf = known.expand(B, Cc, S).double()
    abt_b, Sx, A, D, dt = _oracle_coefs(abt, ve, mf, lam, beta)
    kn = known.expand(B, Cc, S)

    def score(z):
        return torch.where(kn, -(1 + lam) * (z - y.double()) + lam * (z - x0b.double()), -(z - x0.double()))

    def drift(z):
        return (abt_b.sqrt() * (z + score(z)) - z) / (1 - abt_b) + A * z

    xt = x.double() / Sx
    # FIRST: C = Coef_C(x_t); x_t = ou_advance(x_t, dt, C)
    want = O.ou_advance(xt, dt, A, drift(xt), D, lambda _: xi1.double()) * Sx
    got = R.substep(x, x0, x0b, y, kn, None, tab, xi1, None, R.FIRST)
    assert torch.allclose(got["x"][0], want, rtol=1e-5, atol=1e-5)
    assert torch.allclose(got["c"][0], drift(xt), rtol=1e-5, atol=1e-5)
    # steady, no fused next: Cn = Coef_C(x_t); x_t += (Cn - C) dt; x_t = ou_advance(x_t, dt / 2, C_old)
    cn = drift(xt)
    want = O.ou_advance(xt + (cn - cprev.double()) * dt, dt / 2, A, cprev.double(), D, lambda _: xi2.double()) * Sx
    got = R.substep(x, x0, x0b, y, kn, cprev, tab, xi2, None, 0)
    assert torch.allclose(got["x"][0], want, rtol=1e-5, atol=1e-5)
    # fused next: one more ou_advance over dt / 2 with the new C
    want = O.ou_advance(want / Sx, dt / 2, A, cn, D, lambda _: xi1.double()) * Sx
    got = R.substep(x, x0, x0b, y, kn, cprev, tab, xi2, xi1, R.FUSE_NEXT)
    assert torch.allclose(got["x"][0], want, rtol=1e-5, atol=1e-5)
    assert torch.allclose(got["x0e"][0], xt + score(xt), rtol=1e-5, atol=1e-5)
    # every magnitude bounds its value
    for k in ("x", "c", "x0e"):
        assert torch.all(got[k][1] >= got[k][0].abs() * (1 - 1e-12))


def test_advance_boundary_prologue_restatements():
    lam, beta = 5.0, 1.5
    tab, sig, ve, abt = _table(beta, lam)
    g = torch.Generator().manual_seed(4)
    B, Cc, S = 2, 3, 10
    x, c, xi, a, b, y, nz = (torch.randn(B, Cc, S, generator=g) for _ in range(7))
    known = (torch.rand(B, 1, S, generator=g) < 0.5).expand(B, Cc, S)
    abt_b, Sx, A, D, dt = _oracle_coefs(abt, ve, known.double(), lam, beta)
    for half in (0, 1):
        want = O.ou_advance(x.double() / Sx, dt / 2 if half else dt, A, c.double(), D, lambda _: xi.double()) * Sx
        val, mag = R.advance(x, c, known, tab, xi, half)
        assert torch.allclose(val, want, rtol=1e-5, atol=1e-5) and torch.all(mag >= val.abs() * (1 - 1e-12))
    coef, cfg = -0.37, 3.5
    res = R.boundary(a, b, y, nz, known, x, coef, tab, cfg=cfg)
    d = b.double() + (a.double() - b.double()) * cfg
    out = torch.where(known, y.double(), d)
    xe = x.double() + (x.double() - out) * coef
    xe = torch.where(known, sig.double().view(-1, 1, 1) * nz.double() + y.double(), xe)
    assert torch.allclose(res["out"][0], out) and torch.allclose(res["x"][0], xe, rtol=1e-6, atol=1e-6)
    val, _ = R.prologue(x, y, nz, known, tab)
    assert torch.equal(val[~known], x.double()[~known])
    assert torch.allclose(val[known], (sig.double().view(-1, 1, 1) * nz.double() + y.double())[known], rtol=1e-6)


# ---------------------------------------------------------------------------------------------------------------
# the audio-video row split and the audio target correction
# ---------------------------------------------------------------------------------------------------------------
LINES, N_LAST, SPLIT = 3, 10, 6
CORR = (0.625, 1.3, 0.8)


def _av_table(lam=5.0, beta=1.5):
    """2 * LINES distinct VE rows: video rows 0..LINES-1 (corr 1), audio rows LINES.. with CORR."""
    from lanpaint_b200.schedule import Hyper, build_table
    sig = torch.tensor([0.3, 1.0, 4.0, 0.5, 2.0, 9.0])
    ve, abt, _ = O.times_from_sigma(sig, False)
    tab = build_table(abt.numpy(), ve.numpy(), Hyper(0.2, lam, beta, 1.0, False), rep_noise=sig.numpy(),
                      rep_y=np.linspace(0.5, 1.0, 2 * LINES), corr=(1.0,) * LINES + CORR)
    return torch.from_numpy(tab), sig, ve, abt


def test_split_rows():
    rows = R.split_rows((LINES, 1, N_LAST), SPLIT)
    assert rows.shape == (LINES, 1, N_LAST)
    for b in range(LINES):
        assert rows[b, 0].tolist() == [b] * SPLIT + [LINES + b] * (N_LAST - SPLIT)
    assert torch.equal(R.split_rows((LINES, 2, 5), 0), torch.arange(LINES).view(-1, 1, 1).expand(LINES, 2, 5))
    assert torch.equal(R.split_rows((LINES, 1, N_LAST), N_LAST), R.split_rows((LINES, 1, N_LAST), 0))


def test_av_substep_restatement_matches_the_oracle():
    """A row split with distinct rows per line and the audio correction: the table-form restatement against the
    oracle's masked_score(correction=...) and ou_advance with every coefficient taken per element."""
    lam, beta = 5.0, 1.5
    tab, sig, ve, abt = _av_table(lam, beta)
    shape = (LINES, 1, N_LAST)
    rows = R.split_rows(shape, SPLIT)
    g = torch.Generator().manual_seed(11)
    x, x0, x0b, y, xi1, xi2, cprev = (torch.randn(shape, generator=g) for _ in range(7))
    known = torch.rand(shape, generator=g) < 0.5
    mf = known.double()
    abt_e, ve_e = abt.double()[rows], ve.double()[rows]
    corr = torch.tensor((1.0,) * LINES + CORR, dtype=torch.float64)[rows]
    Sx = (1 + ve_e ** 2).sqrt()
    step = 0.2 * (1 - abt_e).clamp(min=1.0)
    cf = O.branch_coefficients(abt_e, step, torch.ones_like(abt_e), torch.full_like(abt_e, beta), lam)
    A = cf.A_x * (1 - mf) + cf.A_y * mf
    D = cf.D_x * (1 - mf) + cf.D_y * mf
    dt = cf.half_dt_x * (1 - mf) + cf.half_dt_y * mf
    hp = O.Hyper(lam=lam, beta=beta, flow=False)
    heads = lambda *_a, **_k: (x0.double(), x0b.double())

    def score(z):
        return O.masked_score(heads, z, y.double(), mf, abt_e, ve_e, abt_e, hp, 3, correction=corr)

    def drift(z):
        return (abt_e.sqrt() * (z + score(z)) - z) / (1 - abt_e) + A * z

    xt = x.double() / Sx
    want = O.ou_advance(xt, dt, A, drift(xt), D, lambda _: xi1.double()) * Sx
    got = R.substep(x, x0, x0b, y, known, None, tab, xi1, None, R.FIRST, rows=rows)
    assert torch.allclose(got["x"][0], want, rtol=1e-5, atol=1e-5)
    assert torch.allclose(got["c"][0], drift(xt), rtol=1e-5, atol=1e-5)
    assert torch.allclose(got["x0e"][0], xt + score(xt), rtol=1e-5, atol=1e-5)
    cn = drift(xt)
    want = O.ou_advance(xt + (cn - cprev.double()) * dt, dt / 2, A, cprev.double(), D, lambda _: xi2.double()) * Sx
    want = O.ou_advance(want / Sx, dt / 2, A, cn, D, lambda _: xi1.double()) * Sx
    got = R.substep(x, x0, x0b, y, known, cprev, tab, xi2, xi1, R.FUSE_NEXT, rows=rows)
    assert torch.allclose(got["x"][0], want, rtol=1e-5, atol=1e-5)
    # the correction moves the audio part: the same launch without it differs there and only there
    tab1 = tab.clone()
    tab1[:, R.T_CORR] = 1.0
    plain = R.substep(x, x0, x0b, y, known, cprev, tab1, xi2, xi1, R.FUSE_NEXT, rows=rows)
    moved = (plain["x"][0] != got["x"][0]).reshape(LINES, N_LAST)
    assert not moved[:, :SPLIT].any() and moved[:, SPLIT:].all()
    for k in ("x", "c", "x0e"):
        assert torch.all(got[k][1] >= got[k][0].abs() * (1 - 1e-12))


def test_av_restatement_equals_a_per_element_loop():
    """Every restated launch with rows = split_rows(...) equals the same launch made one element at a time with
    that element's table row alone: value and magnitude, bit for bit."""
    tab, *_ = _av_table()
    shape = (LINES, 1, N_LAST)
    rows = R.split_rows(shape, SPLIT)
    g = torch.Generator().manual_seed(12)
    x, a, b, y, cp, xi1, xi2, nz = (torch.randn(shape, generator=g) for _ in range(8))
    known = torch.rand(shape, generator=g) < 0.5
    ring = torch.rand(shape, generator=g) < 0.3
    cfg = (4.5, -0.5)
    whole = {
        "sub": R.substep(x, a, b, y, known, cp, tab, xi1, xi2, R.FUSE_NEXT, cfg=cfg, noise_err=1e-4, rows=rows),
        "merge": R.substep(x, a, None, y, known, cp, tab, xi1, None, R.FIRST | R.FUSE_NEXT | R.MERGE_NOISE, rows=rows),
        "adv": R.advance(x, cp, known, tab, xi1, 1, rows=rows),
        "pro": R.prologue(x, y, nz, known, tab, rows=rows),
        "bnd": R.boundary(a, b, y, nz, known, x, -0.37, tab, cfg=3.5, rows=rows),
    }
    for i in range(x.numel()):
        e = np.unravel_index(i, shape)
        one = lambda t: t[e].reshape(1, 1, 1)
        t1 = tab[int(rows[e]):int(rows[e]) + 1]
        k1 = one(known)
        parts = {
            "sub": R.substep(one(x), one(a), one(b), one(y), k1, one(cp), t1, one(xi1), one(xi2), R.FUSE_NEXT,
                             cfg=cfg, noise_err=1e-4),
            "merge": R.substep(one(x), one(a), None, one(y), k1, one(cp), t1, one(xi1), None,
                               R.FIRST | R.FUSE_NEXT | R.MERGE_NOISE),
            "adv": R.advance(one(x), one(cp), k1, t1, one(xi1), 1),
            "pro": R.prologue(one(x), one(y), one(nz), k1, t1),
            "bnd": R.boundary(one(a), one(b), one(y), one(nz), k1, one(x), -0.37, t1, cfg=3.5),
        }
        for name in ("sub", "merge"):
            for k in ("x", "c", "x0e"):
                for j in range(2):
                    assert whole[name][k][j][e] == parts[name][k][j].reshape(()), (name, k, j, e)
        assert whole["sub"]["x_slack"][e] == parts["sub"]["x_slack"].reshape(()), e
        for name in ("adv", "pro"):
            for j in range(2):
                assert whole[name][j][e] == parts[name][j].reshape(()), (name, j, e)
        for k in ("out", "x"):
            for j in range(2):
                assert whole["bnd"][k][j][e] == parts["bnd"][k][j].reshape(()), ("bnd", k, j, e)
    # stop statistics: inv_S of each element's own row
    s_in, s_ring = R.stop_stats(a, b, known, ring, tab, rows=rows)
    inv_s = tab[:, R.T_INVS].double()[rows]
    d2 = ((a.double() - b.double()) * inv_s) ** 2
    assert s_in == pytest.approx(float(d2[~known].sum()), rel=1e-15)
    assert s_ring == pytest.approx(float(d2[ring].sum()), rel=1e-15)
