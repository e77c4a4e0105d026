"""The guarded-operand arena (tests/_guard.py) on CPU tensors: placement, and that each kind of stray store is
reported with the operand, the side and the byte offset."""
import pytest
import torch

from _guard import ALIGN, BAND, Arena, GuardError, bits, plain


def _raw(arena, name):
    """The whole allocation of a placed operand, as elements of its dtype, and the operand's first element in it."""
    p = arena.ops[name]
    es = p.view.element_size()
    assert p.start % es == 0
    return p.buf[:p.buf.numel() // es * es].view(p.view.dtype), p.start // es


@pytest.mark.parametrize("dtype,shape,offset,slack", [
    (torch.float32, (2, 3, 7, 9), 0, 0), (torch.float32, (1, 4, 16, 16), 4, 4), (torch.bfloat16, (5, 33), 8, 0),
    (torch.float16, (64,), 2, 16), (torch.uint8, (3, 1, 7, 9), 0, 0), (torch.uint8, (189,), 1, 0),
    (torch.int32, (70,), 0, 3), (torch.float64, (2,), 0, 0), (torch.int64, (2,), 8, 0)])
def test_placement(dtype, shape, offset, slack):
    g = torch.Generator().manual_seed(1)
    t = (torch.randn(shape, generator=g) * 50).to(dtype)
    a = Arena("cpu")
    v = a.place(t, offset_bytes=offset, slack=slack, name="t")
    assert v.shape == t.shape and v.dtype == t.dtype and v.is_contiguous() and torch.equal(bits(v), bits(t))
    assert (v.data_ptr() - offset) % ALIGN == 0
    p = a.ops["t"]
    assert p.start >= BAND and p.buf.numel() - (p.start + p.nbytes + p.slack_bytes) >= BAND
    assert a.slack_of("t").numel() == slack
    a.snapshot()
    a.check("untouched")
    a.check("untouched", written={"t"})
    u = plain(t, offset, slack)
    assert torch.equal(bits(u), bits(t)) and (u.data_ptr() - offset) % ALIGN == 0


def test_the_pattern_is_a_nan_at_every_width_and_no_mask_value():
    a = Arena("cpu")
    a.place(torch.zeros(8), name="t")
    band = a.ops["t"].buf[:BAND]
    for dt in (torch.float32, torch.bfloat16, torch.float16):
        assert bool(torch.isnan(band.view(dt)).all()), dt
    assert not bool(((band == 0) | (band == 1)).any())
    a.place(torch.zeros(8), slack=4, name="s")
    assert bool(torch.isnan(a.slack_of("s")).all())


def _arena():
    a = Arena("cpu")
    x = a.place(torch.arange(40, dtype=torch.float32).view(2, 20), slack=4, name="x")
    y = a.place(torch.arange(40, dtype=torch.float32).view(2, 20), offset_bytes=4, name="y")
    h = a.place(torch.ones(33, dtype=torch.bfloat16), offset_bytes=8, name="h")
    m = a.place(torch.ones(21, dtype=torch.uint8), name="m")
    a.snapshot()
    return a


def _expect(a, written, operand, where, offset):
    with pytest.raises(GuardError) as e:
        a.check("case-7", written=written)
    err = e.value
    assert (err.case_id, err.operand, err.where, err.offset) == ("case-7", operand, where, offset), str(err)
    assert "case-7" in str(err) and f"'{operand}'" in str(err) and where in str(err) and str(offset) in str(err)


def test_store_one_element_before_the_view():
    a = _arena()
    raw, first = _raw(a, "y")
    raw[first - 1] = 3.0
    _expect(a, {"y"}, "y", "front", 1)       # the last byte of that element is the byte just before the operand
    a = _arena()
    raw, first = _raw(a, "h")
    raw[first - 3] = 1.0
    _expect(a, {"h", "x"}, "h", "front", 5)


def test_store_one_element_after_the_view():
    a = _arena()
    raw, first = _raw(a, "y")
    raw[first + 40] = 3.0
    _expect(a, {"y"}, "y", "back", 0)
    a = _arena()
    raw, first = _raw(a, "m")
    raw[first + 21 + 2] = 1
    _expect(a, {"m"}, "m", "back", 2)


def test_store_after_the_slack_and_inside_it():
    a = _arena()
    raw, first = _raw(a, "x")
    raw[first + 40:first + 44] = 0.0          # the four slack elements of a written operand: allowed
    a.check("case-7", written={"x"})
    _expect(a, {"y"}, "x", "slack", 160)      # ... of an operand the call must not write: reported
    raw[first + 44] = 0.0                     # one element after the slack
    _expect(a, {"x"}, "x", "back", 0)


def test_store_into_an_input():
    a = _arena()
    a.ops["h"].view[17] = 2.0
    a.check("case-7", written={"h"})
    _expect(a, {"x", "y"}, "h", "input", 34)
    a = _arena()
    a.ops["m"].view[20] = 0
    _expect(a, (), "m", "input", 20)


def test_a_rewrite_with_the_same_bits_is_no_store():
    a = _arena()
    a.ops["y"].view.copy_(a.ops["y"].view.clone())
    a.check("case-7")


def test_check_refuses_an_unknown_operand_name():
    a = _arena()
    with pytest.raises(AssertionError):
        a.check("case-7", written={"z"})
