"""Guarded operands (test infrastructure; CPU and CUDA tensors alike).

An Arena places every operand of one library call in the middle of its own, larger torch allocation:

    | front band >= 64 KiB | operand (+ slack) | back band >= 64 KiB |

Both bands hold a fixed pattern.  After the call, check() asserts that every band still holds it (a kernel that
stores before element 0 or past the last element it may touch), that every operand the call does not write is
bit-identical to its snapshot (a kernel that stores through the pointer of one of its inputs), and that the slack of
such an operand is untouched too.  `slack` is the number of trailing elements the header lets the library touch:
4 for y_known / noise_known, 16 for the output of lp_torch_cpu_randn_f32.

The pattern is the 16-bit word 0x7FA5 repeated: a NaN read as fp32, bf16 or fp16, and neither 0 nor 1 read as a mask
byte, so an out-of-range read whose value reaches a result shows in the result.  64 KiB is more than any tile, work
group or grid-stride step a kernel could be off by in one access, so such an access lands in a band, inside the
operand's own allocation.  Nothing here maps, protects or frees memory: a stray store can be seen, never turned into
a fault.
"""
from __future__ import annotations

import torch

BAND = 64 * 1024          # least size of each band, bytes
ALIGN = 256               # operands start at offset_bytes past a multiple of this
PATTERN = (0xA5, 0x7F)    # the bytes of the little-endian 16-bit word 0x7FA5, by parity of the position in the buffer


class GuardError(AssertionError):
    """A stray store.  where: "front" / "back" (a band), "slack" or "input" (an operand the call must not write);
    offset: the first differing byte, counted from the operand's first byte ("input", "slack"), backwards from it
    ("front": 1 = the byte just before the operand) or from the first byte of the back band ("back")."""

    def __init__(self, case_id, operand, where, offset):
        self.case_id, self.operand, self.where, self.offset = case_id, operand, where, offset
        what = {"front": f"{offset} byte(s) before its first byte",
                "back": f"at byte {offset} past the end of what the call may touch",
                "slack": f"at byte {offset} (inside its slack, which this call must not write)",
                "input": f"at byte {offset} (the call must not write this operand)"}[where]
        super().__init__(f"{case_id}: operand '{operand}' [{where}] modified {what}")


def _pattern(n: int, device) -> torch.Tensor:
    return torch.tensor(PATTERN, dtype=torch.uint8, device=device).repeat((n + 1) // 2)[:n]


def _first_diff(a: torch.Tensor, b: torch.Tensor, last: bool = False):
    """Index of the first (or last) differing byte of two uint8 tensors, None when they are equal."""
    if torch.equal(a, b):
        return None
    idx = torch.nonzero(a != b).reshape(-1)
    return int(idx[-1] if last else idx[0])


class _Placed:
    __slots__ = ("name", "buf", "start", "nbytes", "slack_bytes", "view", "snap")


class Arena:
    def __init__(self, device):
        self.device = torch.device(device)
        self.ops = {}

    def place(self, t: torch.Tensor, *, offset_bytes: int = 0, slack: int = 0, name: str) -> torch.Tensor:
        """A view with t's shape, dtype and contents, its data pointer offset_bytes past a 256-byte boundary, followed
        by `slack` pattern-filled elements the call may touch, between two bands."""
        assert name not in self.ops, name
        es = t.element_size()
        assert offset_bytes % es == 0 and 0 <= offset_bytes < ALIGN, (name, offset_bytes)
        nbytes, slack_bytes = t.numel() * es, slack * es
        size = BAND + 2 * ALIGN + nbytes + slack_bytes + BAND
        buf = _pattern(size, self.device)
        start = BAND + (-(buf.data_ptr() + BAND)) % ALIGN + offset_bytes
        view = buf[start:start + nbytes].view(t.dtype).view(t.shape)
        view.copy_(t)
        assert view.data_ptr() == buf.data_ptr() + start and (view.data_ptr() - offset_bytes) % ALIGN == 0
        p = _Placed()
        p.name, p.buf, p.start, p.nbytes, p.slack_bytes, p.view, p.snap = name, buf, start, nbytes, slack_bytes, view, None
        self.ops[name] = p
        return view

    def slack_of(self, name: str) -> torch.Tensor:
        """The slack of an operand, as elements of its dtype."""
        p = self.ops[name]
        lo = p.start + p.nbytes
        return p.buf[lo:lo + p.slack_bytes].view(p.view.dtype)

    def snapshot(self) -> None:
        for p in self.ops.values():
            p.snap = p.buf[p.start:p.start + p.nbytes + p.slack_bytes].clone()

    def check(self, case_id, written=()) -> None:
        """Bands intact; operands not in `written` (and their slack) bit-identical to the snapshot."""
        unknown = set(written) - set(self.ops)
        assert not unknown, (case_id, unknown)
        for p in self.ops.values():
            assert p.snap is not None, "snapshot() comes before the call"
            size = p.buf.numel()
            pat = _pattern(size, p.buf.device)
            d = _first_diff(p.buf[:p.start], pat[:p.start], last=True)
            if d is not None:
                raise GuardError(case_id, p.name, "front", p.start - d)
            end = p.start + p.nbytes + p.slack_bytes
            d = _first_diff(p.buf[end:], pat[end:])
            if d is not None:
                raise GuardError(case_id, p.name, "back", d)
            if p.name not in written:
                d = _first_diff(p.buf[p.start:end], p.snap)
                if d is not None:
                    raise GuardError(case_id, p.name, "slack" if d >= p.nbytes else "input", d)


def bits(t: torch.Tensor) -> torch.Tensor:
    """The bytes of a (contiguous) tensor: NaNs compare by their bits."""
    return t.contiguous().view(-1).view(torch.uint8)


def plain(t: torch.Tensor, offset_bytes: int = 0, slack: int = 0) -> torch.Tensor:
    """t's contents in an ordinary tensor with the same misalignment and room for the same slack: the operand the
    unguarded call of a case receives.  It sits 256 bytes inside its allocation and ends 256 bytes before its end."""
    es = t.element_size()
    k = (ALIGN + offset_bytes) // es
    buf = torch.zeros(t.numel() + k + slack + 2 * ALIGN // es, dtype=t.dtype, device=t.device)
    k += ((-buf.data_ptr()) % ALIGN) // es
    v = buf[k:k + t.numel()].view(t.shape)
    v.copy_(t)
    return v
