"""The walk order and the L2 policies of the update kernels (option "l2_handoff") change where and how long bytes sit in
L2, never a result: every setting gives bit-identical x, C and denoised outputs, including the last, partial torch
work group and the TMA-staged boundary."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

P = C.c_void_p
SETTINGS = (0, 1, 2, 3)


def _lib():
    from lanpaint_b200 import _native
    return _native.load()


@pytest.fixture(scope="module")
def job(cuda_device):
    from lanpaint_b200 import _native
    from lanpaint_b200.engine import pack_known, pack_mask
    from lanpaint_b200.schedule import Hyper, build_table, times_from_sigma
    dev = cuda_device
    R, shape = 40, (4, 128, 128)       # 2.6 M elements (>= 2^21: the hand-off applies); the torch-stream kernel's last
    #                                    call is a partial one
    g = torch.Generator().manual_seed(5)
    y, nz, x, c, hc, hu = (torch.randn((R,) + shape, generator=g).to(dev) for _ in range(6))
    pm = pack_mask((torch.rand((R, 1) + shape[1:], generator=g) < 0.5).to(dev), y)
    dims = _native.Dims(R, 4 * 128 * 128, 128 * 128, pm.row_stride, pm.channel_stride)
    kn = pack_known(pm, dims, y, nz)
    s = torch.linspace(0.5, 3.0, R)
    ve, abt, _ = times_from_sigma(s, False)
    tab = torch.from_numpy(build_table(abt.numpy(), ve.numpy(), Hyper(0.2, 5.0, 1.0, 1.0, False))).to(dev)
    heads = _native.Heads(hc.data_ptr(), hu.data_ptr(), 0, 1, 5.0, 3.0)
    yield dict(y=y, nz=nz, x=x, c=c, pm=pm, dims=dims, kn=kn, tab=tab, heads=heads)
    lib = _lib()
    lib.lp_set_option(b"l2_handoff", 3)
    lib.lp_set_option(b"tma_boundary", 0)


def _rng(mode):
    from lanpaint_b200 import _native
    r = _native.Rng()
    r.mode = _native.RNG_TORCH if mode == "torch" else _native.RNG_PHILOX
    r.seed, r.draw0, r.draw1 = 1234, 4096, 8192
    return r


def _run(job, kernel, setting):
    from lanpaint_b200 import _native
    lib = _lib()
    assert lib.lp_set_option(b"l2_handoff", setting) == 0
    assert lib.lp_set_option(b"tma_boundary", 1 if kernel == "boundary_tma" else 0) == 0
    x, c, out = job["x"].clone(), job["c"].clone(), torch.empty_like(job["x"])
    st = P(torch.cuda.current_stream().cuda_stream)
    pm, dims, tab, hd = job["pm"], job["dims"], job["tab"], job["heads"]
    if kernel == "torch_substep":
        rc = lib.lp_substep_known(P(x.data_ptr()), C.byref(hd), P(job["y"].data_ptr()), P(pm.data.data_ptr()),
                                  C.byref(job["kn"].struct), P(c.data_ptr()), None, None, P(tab.data_ptr()),
                                  C.byref(dims), C.byref(_rng("torch")), _native.SUBSTEP_FUSE_NEXT, st)
    elif kernel == "philox_substep":
        rc = lib.lp_substep(P(x.data_ptr()), C.byref(hd), P(job["y"].data_ptr()), P(pm.data.data_ptr()),
                            P(c.data_ptr()), None, None, P(tab.data_ptr()), C.byref(dims), C.byref(_rng("philox")),
                            _native.SUBSTEP_FUSE_NEXT | _native.SUBSTEP_MERGE_NOISE, st)
    else:
        rc = lib.lp_boundary_known(C.byref(hd), P(job["y"].data_ptr()), P(job["nz"].data_ptr()), P(pm.data.data_ptr()),
                                   C.byref(job["kn"].struct), P(x.data_ptr()), P(out.data_ptr()), C.c_float(-0.2),
                                   P(tab.data_ptr()), C.byref(dims), st)
    _native.check(rc, kernel)
    torch.cuda.synchronize()
    return x, c, out


@pytest.mark.parametrize("kernel", ["torch_substep", "philox_substep", "boundary_ldg", "boundary_tma"])
def test_results_do_not_depend_on_walk_order_or_l2_policy(job, kernel):
    x0, c0, o0 = _run(job, kernel, SETTINGS[0])
    assert not torch.equal(x0, job["x"])
    for s in SETTINGS[1:]:
        x, c, o = _run(job, kernel, s)
        assert torch.equal(x, x0) and torch.equal(c, c0), (kernel, s)
        if kernel.startswith("boundary"):
            assert torch.equal(o, o0), (kernel, s)
