"""Poisoned, guarded allocations for the memory tests (tests/test_poisoned_memory_*.py).

`poisoned(pattern)` replaces torch.empty and torch.empty_like, the two spellings the package allocates with, for calls
made from code of the loftr_b200 package.  Each such allocation becomes one uint8 buffer of nbytes + 2 * guard bytes,
filled with the pattern throughout, and the caller gets the middle part as a contiguous tensor of the requested shape,
dtype and device.  A result that depends on memory the call did not write then changes with the pattern, and a write
past the requested size lands in a guard, which the context checks on exit against the allocation site it recorded.
Calls from anywhere else (torch itself, the float64 references of tests/) get ordinary allocations.

Patterns: "0x00" and "0xFF" (every byte; 0xFF makes fp32 / fp16 values NaN and integers -1) and "big" (fp32 1e30, fp16
6e4, every other dtype 0xFF bytes): NaN is hidden by fmaxf and by comparisons such as `key > -1e29f`, a large finite
value is not.  No pattern turns an integer field into a large positive number: the aim is to see unwritten reads as
wrong results, not to provoke faults."""
from __future__ import annotations

import contextlib
import os
import sys

import torch

PATTERNS = ("0x00", "0xFF", "big")
PACKAGE = "loftr_b200"
_BIG = {torch.float32: 1e30, torch.float16: 6e4}
_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# keyword arguments a poisoned allocation honours; any other (out=, layout=, requires_grad=True, a non-contiguous
# memory format, ...) passes the call through unpoisoned
_PLAIN = {"dtype": None, "device": None, "pin_memory": False, "layout": torch.strided, "requires_grad": False,
          "memory_format": torch.contiguous_format}


class GuardError(AssertionError):
    """A poisoned allocation's guard bytes changed: something wrote past (or before) the buffer it was given."""


class _Alloc:
    __slots__ = ("base", "nbytes", "dtype", "shape", "site")

    def __init__(self, base, nbytes, dtype, shape, site):
        self.base, self.nbytes, self.dtype, self.shape, self.site = base, nbytes, dtype, shape, site


class Poison:
    """The state of one `poisoned` context: its pattern, guard size and every allocation it made (kept alive until the
    guards are checked, so that the allocator cannot hand a guarded block to anyone else meanwhile)."""

    def __init__(self, pattern, guard):
        if pattern not in PATTERNS:
            raise ValueError(f"poisoned: pattern must be one of {PATTERNS} (got {pattern!r})")
        if guard <= 0 or guard % 1024:
            raise ValueError(f"poisoned: guard must be a positive multiple of 1024 bytes (got {guard})")
        self.pattern, self.guard, self.allocs = pattern, guard, []

    @property
    def guard_bytes(self):
        """Guard bytes checked on exit."""
        return 2 * self.guard * len(self.allocs)

    def stats(self):
        return {"pattern": self.pattern, "allocations": len(self.allocs), "guard_bytes": self.guard_bytes,
                "poisoned_bytes": sum(a.nbytes for a in self.allocs)}

    def _fill(self, base, dtype):
        if self.pattern == "big" and dtype in _BIG:
            base.view(dtype).fill_(_BIG[dtype])
        else:
            base.fill_(0 if self.pattern == "0x00" else 0xFF)

    def _expected(self, a):
        """The guard's bytes as the fill left them [guard] uint8 on the buffer's device."""
        ref = torch.empty(self.guard, dtype=torch.uint8, device=a.base.device)
        self._fill(ref, a.dtype)
        return ref

    def allocate(self, shape, dtype, device, pin_memory, site):
        shape = torch.Size(shape)
        nbytes = shape.numel() * dtype.itemsize
        g = self.guard
        base = torch.empty(nbytes + 2 * g, dtype=torch.uint8, device=device, pin_memory=pin_memory)
        self._fill(base, dtype)
        self.allocs.append(_Alloc(base, nbytes, dtype, tuple(shape), site))
        return base[g:g + nbytes].view(dtype).view(shape)

    def check(self):
        """Raises GuardError naming the allocation site of every buffer whose guards changed."""
        if any(a.base.is_cuda for a in self.allocs):
            torch.cuda.synchronize()
        g = self.guard
        bad = []
        for a in self.allocs:
            ref = self._expected(a)
            head = (a.base[:g] != ref).nonzero().flatten()
            tail = (a.base[g + a.nbytes:] != ref).nonzero().flatten()
            if head.numel() or tail.numel():
                where = []
                if head.numel():
                    where.append(f"{head.numel()} bytes before it (from offset {int(head[0]) - g})")
                if tail.numel():
                    where.append(f"{tail.numel()} bytes after it (up to offset +{int(tail[-1]) + 1} past its end)")
                bad.append(f"{a.site}: {a.nbytes}-byte buffer {a.dtype} {list(a.shape)}: " + " and ".join(where))
        if bad:
            raise GuardError(f"poisoned({self.pattern!r}): guard bytes changed\n  " + "\n  ".join(bad))


def _package_frame(frame):
    name = frame.f_globals.get("__name__", "")
    return name == PACKAGE or name.startswith(PACKAGE + ".")


def _site(frame):
    return f"{os.path.relpath(frame.f_code.co_filename, _ROOT)}:{frame.f_lineno}"


def _plain(kwargs):
    """The keyword arguments are all ones a poisoned allocation honours."""
    for k, v in kwargs.items():
        if k not in _PLAIN:
            return False
        if k in ("layout", "requires_grad", "memory_format") and v not in (None, _PLAIN[k]) and \
                not (k == "memory_format" and v == torch.preserve_format):
            return False
    return True


@contextlib.contextmanager
def poisoned(pattern, guard=4096):
    """Context manager: package allocations through torch.empty / torch.empty_like are poisoned with `pattern` and
    guarded by `guard` bytes on each side (a multiple of 1024, which keeps the allocator's alignment for TMA maps).
    On a normal exit it synchronises and raises GuardError for every changed guard byte, by allocation site.
    torch.empty and torch.empty_like are restored on every exit, an exception's included.  -> the Poison record."""
    state = Poison(pattern, guard)
    real_empty, real_like = torch.empty, torch.empty_like

    def empty(*args, **kwargs):
        frame = sys._getframe(1)
        if not _package_frame(frame) or not _plain(kwargs) or not args:
            return real_empty(*args, **kwargs)
        shape = args[0] if len(args) == 1 and isinstance(args[0], (tuple, list, torch.Size)) else args
        dtype = kwargs.get("dtype") or torch.get_default_dtype()
        device = torch.device(kwargs.get("device") or torch.get_default_device())
        return state.allocate(shape, dtype, device, kwargs.get("pin_memory", False), _site(frame))

    def empty_like(input, **kwargs):
        frame = sys._getframe(1)
        if not _package_frame(frame) or not _plain(kwargs) or input.layout != torch.strided:
            return real_like(input, **kwargs)
        dtype = kwargs.get("dtype") or input.dtype
        device = torch.device(kwargs.get("device") or input.device)
        return state.allocate(input.shape, dtype, device, kwargs.get("pin_memory", False), _site(frame))

    torch.empty, torch.empty_like = empty, empty_like
    try:
        yield state
    finally:
        torch.empty, torch.empty_like = real_empty, real_like
    state.check()
