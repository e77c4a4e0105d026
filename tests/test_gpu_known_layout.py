"""The known-operand layout (lp_known: known bits + y / noise packed to their known elements) against the dense
operands: the layout itself against a numpy restatement, and the kernels that read it -- the TMA-staged torch-stream
sub-step and the LDG step boundary -- bit for bit against the dense LDG kernels.  The dense y / noise handed to the
packed calls are poisoned with NaN, so a launch that read them instead of the packed operands would show."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SHAPES = [(1, 4, 128, 128), (3, 4, 128, 128), (128, 4, 128, 128),   # SDXL batches
          (1, 16, 21, 80, 45),                                        # Wan: plane 80*45 = 3600, not a multiple of 1024
          (5, 4, 120, 136)]                                           # a total that ends inside a sub-tile group
MASKS = ["random", "blob", "all_known", "all_free"]


def _mask(kind, shape, gen, dev):
    mshape = (shape[0], 1) + tuple(shape[2:])
    if kind == "random":
        return (torch.rand(mshape, device=dev, generator=gen) < 0.5).to(torch.uint8)
    if kind == "all_known":
        return torch.ones(mshape, dtype=torch.uint8, device=dev)
    if kind == "all_free":
        return torch.zeros(mshape, dtype=torch.uint8, device=dev)
    m = torch.zeros(mshape, dtype=torch.uint8, device=dev)
    h, w = shape[-2], shape[-1]
    m[..., int(0.2 * h):int(0.7 * h), int(0.3 * w):int(0.9 * w)] = 1
    return 1 - m                                                        # one hole to regenerate, the rest known


def _dims(shape):
    from lanpaint_b200 import _native
    B, Cc = shape[0], shape[1]
    S = int(np.prod(shape[2:]))
    return _native.Dims(B, Cc * S, S, S, 0, 0)


def _packed(m8, dims, y, noise):
    from lanpaint_b200.engine import PackedMask, pack_known
    pm = PackedMask(m8, dims.spatial, 0)
    return pack_known(pm, dims, y, noise)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def test_layout_matches_numpy_restatement(cuda_device):
    """words[2w] = known bits of elements 32w..32w+31, words[2w+1] = known elements before 32w, sentinel at W;
    y / noise at known elements in element order -- on a ragged total and a full-shape (per-channel) mask."""
    from lanpaint_b200 import _native
    from lanpaint_b200.engine import PackedMask, pack_known
    dev = cuda_device
    gen = torch.Generator(device=dev).manual_seed(5)
    for shape, per_channel in (((3, 4, 7, 13), False), ((2, 4, 64, 64), True), ((1, 16, 21, 80, 45), False)):
        B, Cc, S = shape[0], shape[1], int(np.prod(shape[2:]))
        y, noise = (torch.randn(shape, device=dev, generator=gen) for _ in range(2))
        mshape = shape if per_channel else (B, 1) + tuple(shape[2:])
        m8 = (torch.rand(mshape, device=dev, generator=gen) < 0.3).to(torch.uint8)
        dims = _native.Dims(B, Cc * S, S, Cc * S if per_channel else S, S if per_channel else 0, 0)
        kn = pack_known(PackedMask(m8, dims.mask_row_stride, dims.mask_channel_stride), dims, y, noise)
        torch.cuda.synchronize()
        known = np.broadcast_to(m8.cpu().numpy() != 0, shape).reshape(-1)
        n, W = known.size, (known.size + 31) // 32
        padded = np.zeros(32 * W, dtype=bool)
        padded[:n] = known
        bits = (padded.reshape(W, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(1).astype(np.uint32)
        before = np.concatenate([[0], np.cumsum(padded.reshape(W, 32).sum(1))]).astype(np.uint32)
        words = kn.words.cpu().numpy().view(np.uint32)
        assert int(_native.load().lp_known_words(n)) == words.size
        assert np.array_equal(words[0:2 * W:2], bits)
        assert np.array_equal(words[1:2 * W + 2:2], before)          # W + 1 counts, the last one the sentinel's
        assert words[2 * W] == 0
        k = int(known.sum())
        assert np.array_equal(kn.y[:k].cpu().numpy(), y.reshape(-1).cpu().numpy()[known])
        assert np.array_equal(kn.noise[:k].cpu().numpy(), noise.reshape(-1).cpu().numpy()[known])


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("hdtype", [torch.float32, torch.bfloat16])
def test_substep_known_equals_dense_ldg(shape, hdtype, cuda_device):
    """lp_substep_known (TMA-staged kernel on the packed y, every size: tma_min 0) == lp_substep with the LDG kernels
    (tma 0) for all four launch kinds, both RNG streams, every mask kind."""
    from lanpaint_b200 import _native
    from lanpaint_b200.schedule import Hyper, build_table
    from oracle import langevin_oracle as O
    lib = _native.load()
    dev = cuda_device
    gen = torch.Generator(device=dev).manual_seed(11)
    B = shape[0]
    x_in, y, c_in, h0, h1 = (torch.randn(shape, device=dev, generator=gen) for _ in range(5))
    h0, h1 = h0.to(hdtype), h1.to(hdtype)
    sig = torch.linspace(0.4, 3.0, B)
    ve, abt, _ = O.times_from_sigma(sig, False)
    tab = torch.from_numpy(build_table(abt.numpy(), ve.numpy(), Hyper(0.2, 5.0, 1.0, 1.0, False))).to(dev)
    dims = _dims(shape)
    P = C.c_void_p
    poisoned = torch.full_like(y, float("nan"))
    dt = _native.DTYPE_F32 if hdtype == torch.float32 else _native.DTYPE_BF16
    hd = _native.Heads(h0.data_ptr(), h1.data_ptr(), dt, 0, 0.0, 0.0)
    try:
        assert lib.lp_set_option(b"tma_min", 0) == 0
        for kind in MASKS:
            m8 = _mask(kind, shape, gen, dev)
            kn = _packed(m8, dims, y, None)
            for mode in (_native.RNG_TORCH, _native.RNG_PHILOX):
                for flags in (_native.SUBSTEP_FUSE_NEXT, _native.SUBSTEP_FIRST | _native.SUBSTEP_FUSE_NEXT, 0,
                              _native.SUBSTEP_FIRST):
                    r = _native.Rng(mode, 0, None, None, 1234, 8, 8 + 4096, None)
                    res = []
                    for tma, packed in ((0, False), (1, True)):
                        assert lib.lp_set_option(b"tma", tma) == 0
                        x, c = x_in.clone(), c_in.clone()
                        if packed:
                            rc = lib.lp_substep_known(P(x.data_ptr()), C.byref(hd),
                                                      P((poisoned if mode == _native.RNG_TORCH else y).data_ptr()),
                                                      P(m8.data_ptr()), C.byref(kn.struct), P(c.data_ptr()), None,
                                                      None, P(tab.data_ptr()), C.byref(dims), C.byref(r),
                                                      flags | _native.SUBSTEP_STORE_C, _stream())
                        else:
                            rc = lib.lp_substep(P(x.data_ptr()), C.byref(hd), P(y.data_ptr()), P(m8.data_ptr()),
                                                P(c.data_ptr()), None, None, P(tab.data_ptr()), C.byref(dims),
                                                C.byref(r), flags | _native.SUBSTEP_STORE_C, _stream())
                        assert rc == 0
                        res.append((x, c))
                    assert torch.equal(res[0][0], res[1][0]), (kind, mode, flags)
                    assert torch.equal(res[0][1], res[1][1]), (kind, mode, flags)
    finally:
        lib.lp_set_option(b"tma", 1)
        lib.lp_set_option(b"tma_min", 1 << 18)


@pytest.mark.parametrize("shape", SHAPES + [(2, 4, 45, 45)])           # 45 x 45: the scalar (N = 1) kernel
@pytest.mark.parametrize("combine,with_next,with_out,hdtype", [(False, True, False, torch.float32),
                                                               (False, True, True, torch.bfloat16),
                                                               (True, True, True, torch.float32),
                                                               (False, False, True, torch.float32)])
def test_boundary_known_equals_dense_ldg(shape, combine, with_next, with_out, hdtype, cuda_device):
    """lp_boundary_known (LDG kernel on the known bits and packed y / noise) == lp_boundary (LDG, dense)."""
    from lanpaint_b200 import _native
    from lanpaint_b200.schedule import Hyper, build_table
    from oracle import langevin_oracle as O
    lib = _native.load()
    dev = cuda_device
    gen = torch.Generator(device=dev).manual_seed(3)
    B = shape[0]
    a, b, y, nz, x0 = (torch.randn(shape, device=dev, generator=gen) for _ in range(5))
    a = a.to(hdtype)
    sig = torch.linspace(0.5, 3.0, B)
    ve, abt, _ = O.times_from_sigma(sig, False)
    tab = torch.from_numpy(build_table(abt.numpy(), ve.numpy(), Hyper(0.2, 5.0, 1.0, 1.0, False),
                                       rep_noise=sig.numpy(), rep_y=np.ones(B))).to(dev)
    dims = _dims(shape)
    P = C.c_void_p
    nan = torch.full_like(y, float("nan"))
    dt = _native.DTYPE_F32 if hdtype == torch.float32 else _native.DTYPE_BF16
    h = _native.Heads(a.data_ptr(), b.data_ptr() if combine else None, dt, 1 if combine else 0, 3.5, 3.5)
    for kind in MASKS:
        m8 = _mask(kind, shape, gen, dev)
        kn = _packed(m8, dims, y, nz)
        res = []
        for packed in (False, True):
            x, out = x0.clone(), torch.full(shape, float("nan"), device=dev)
            args = (P(x.data_ptr()), P(out.data_ptr()) if with_out else None, C.c_float(-0.37),
                    P(tab.data_ptr()) if with_next else None, C.byref(dims), _stream())
            if packed:
                rc = lib.lp_boundary_known(C.byref(h), P(nan.data_ptr()), P(nan.data_ptr()) if with_next else None,
                                           P(m8.data_ptr()), C.byref(kn.struct), *args)
            else:
                rc = lib.lp_boundary(C.byref(h), P(y.data_ptr()), P(nz.data_ptr()) if with_next else None,
                                     P(m8.data_ptr()), *args)
            assert rc == 0
            res.append((x, out))
        assert torch.equal(res[0][0], res[1][0]), kind
        if with_out:
            assert torch.equal(res[0][1], res[1][1]), kind
