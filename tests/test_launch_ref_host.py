"""CPU checks of tests/_launch_ref.py, the fp64 per-launch restatement the GPU launch tests compare kernels with:
its Philox4x32-10 against published known-answer vectors, its two noise mappings against direct evaluation, and its
sub-step / advance / boundary against the oracle's fp32 functions on tiny tensors."""
import numpy as np
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
