"""The poisoning allocator of tests/poison.py on CPU tensors, with a probe module named like a package module standing
in for the library, and a scan of the package for allocation spellings the allocator does not patch."""
import os
import re
import types

import pytest
import torch

import poison
from poison import GuardError, poisoned

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROBE_FILE = os.path.join(ROOT, "loftr_b200", "_poison_probe.py")
PROBE_SRC = '''\
import torch


def alloc(*shape, dtype=torch.float32):
    return torch.empty(*shape, dtype=dtype, device="cpu")  # alloc


def alloc_tuple(shape, dtype):
    return torch.empty(tuple(shape), dtype=dtype)


def like(t, **kw):
    return torch.empty_like(t, **kw)


def half_written(n):
    """Writes only the first half of what it returns."""
    out = torch.empty(n, dtype=torch.float32, device="cpu")
    out[: n // 2] = 1.0
    return out


def overrun(n, extra):
    """Writes `extra` elements past the end of the buffer it allocated (into the guard, through the storage)."""
    out = torch.empty(n, dtype=torch.int32, device="cpu")
    out.as_strided((n + extra,), (1,)).fill_(7)
    return out
'''


def _probe():
    """A module whose __name__ is inside the package, as the library's own modules are."""
    mod = types.ModuleType("loftr_b200._poison_probe")
    mod.__file__ = PROBE_FILE
    exec(compile(PROBE_SRC, PROBE_FILE, "exec"), mod.__dict__)
    return mod


PROBE_ALLOC = '    return torch.empty(*shape, dtype=dtype, device="cpu")  # alloc'


def _line(text):
    return PROBE_SRC.splitlines().index(text) + 1


@pytest.mark.parametrize("pattern", poison.PATTERNS)
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.int64, torch.int32, torch.uint8, torch.bool])
def test_fill_shape_dtype_and_alignment(pattern, dtype):
    probe = _probe()
    with poisoned(pattern) as pz:
        t = probe.alloc(3, 5, dtype=dtype)
        u = probe.alloc_tuple([2, 0, 4], dtype)
    assert t.shape == (3, 5) and t.dtype == dtype and t.device.type == "cpu" and t.is_contiguous()
    assert u.shape == (2, 0, 4) and u.dtype == dtype
    base = pz.allocs[0].base
    assert base.dtype == torch.uint8 and base.numel() == 15 * t.element_size() + 2 * 4096
    assert t.data_ptr() - base.data_ptr() == 4096 and t.data_ptr() % 1024 == base.data_ptr() % 1024
    raw = base.numpy()
    if pattern == "big" and dtype in (torch.float32, torch.float16):
        big = 1e30 if dtype == torch.float32 else 6e4
        assert (t.float() == big).all() and (base.view(dtype) == torch.tensor(big, dtype=dtype)).all()
    else:
        assert (raw == (0 if pattern == "0x00" else 0xFF)).all()
        if pattern == "0xFF" and dtype in (torch.float32, torch.float16):
            assert torch.isnan(t).all()
        if pattern == "0xFF" and dtype in (torch.int64, torch.int32):
            assert (t == -1).all()
    assert pz.stats() == {"pattern": pattern, "allocations": 2, "guard_bytes": 4 * 4096,
                          "poisoned_bytes": 15 * t.element_size()}


def test_empty_like_and_guard_size():
    probe = _probe()
    src = torch.zeros(4, 6, dtype=torch.float16)
    with poisoned("0xFF", guard=2048) as pz:
        a = probe.like(src)
        b = probe.like(src, dtype=torch.int32)
    assert a.shape == b.shape == (4, 6) and a.dtype == torch.float16 and b.dtype == torch.int32
    assert torch.isnan(a).all() and (b == -1).all()
    assert a.data_ptr() - pz.allocs[0].base.data_ptr() == 2048 and pz.guard_bytes == 2 * 2 * 2048
    with pytest.raises(ValueError, match="multiple of 1024"):
        with poisoned("0x00", guard=1000):
            pass
    with pytest.raises(ValueError, match="pattern"):
        with poisoned("0x7F"):
            pass


def test_only_package_frames_are_poisoned():
    probe = _probe()
    with poisoned("0xFF") as pz:
        mine = torch.empty(64, dtype=torch.int32)
        like = torch.empty_like(mine)
        theirs = probe.alloc(64, dtype=torch.int32)
        out = torch.zeros(3)
        passed = torch.empty(3, out=out)       # out= passes through even from here
    assert passed is out and (theirs == -1).all()
    assert [a.site for a in pz.allocs] == [f"loftr_b200/_poison_probe.py:{_line(PROBE_ALLOC)}"]
    assert (mine.data_ptr() != theirs.data_ptr()) and like.shape == mine.shape


def test_guard_write_is_reported_with_its_allocation_site():
    probe = _probe()
    with pytest.raises(GuardError) as err:
        with poisoned("0xFF"):
            probe.overrun(10, 3)
    msg = str(err.value)
    site = f"loftr_b200/_poison_probe.py:{_line('    out = torch.empty(n, dtype=torch.int32, device=\"cpu\")')}"
    assert site in msg, msg
    assert "40-byte buffer torch.int32 [10]: 12 bytes after it (up to offset +12 past its end)" in msg, msg
    with poisoned("0xFF"):      # within its own bytes: nothing to report
        probe.overrun(10, 0)


def test_a_partly_written_buffer_differs_between_patterns():
    probe = _probe()
    outs = {}
    for pattern in ("0x00", "0xFF", "big"):
        with poisoned(pattern):
            outs[pattern] = probe.half_written(8)
    assert (outs["0x00"][:4] == 1).all() and (outs["0xFF"][:4] == 1).all()
    assert (outs["0x00"][4:] == 0).all() and torch.isnan(outs["0xFF"][4:]).all() and (outs["big"][4:] == 1e30).all()
    with poisoned("0x00"):
        full = probe.alloc(8)
        full.fill_(2.0)
    assert (full == 2).all()


def test_patch_is_undone_after_an_exception():
    probe = _probe()
    real_empty, real_like = torch.empty, torch.empty_like
    with pytest.raises(KeyError):
        with poisoned("0xFF"):
            assert torch.empty is not real_empty and torch.empty_like is not real_like
            probe.alloc(4)
            raise KeyError("inside")
    assert torch.empty is real_empty and torch.empty_like is real_like
    with pytest.raises(GuardError):
        with poisoned("0xFF"):
            probe.overrun(4, 1)
    assert torch.empty is real_empty and torch.empty_like is real_like


# Spellings that hand out uninitialised memory without going through torch.empty / torch.empty_like (which `poisoned`
# patches), or that bind those two under another name, where the patch would not see them.
UNPATCHED = [
    (r"\.new_empty\b", "Tensor.new_empty"),
    (r"\bempty_strided\b", "empty_strided"),
    (r"\bempty_permuted\b", "empty_permuted"),
    (r"\btorch\.(?:cuda\.)?(?:\w+)?Tensor\(", "legacy tensor constructor"),
    (r"\bUntypedStorage\b|\bTypedStorage\b|\b\w+Storage\(", "raw storage"),
    (r"\.resize_\(|\.resize_as_\(", "resize_ (grows storage uninitialised)"),
    (r"\bat::empty\b", "ATen empty"),
    (r"from\s+torch\s+import\s+[^\n]*\bempty", "torch.empty imported under its own name"),
    (r"=\s*torch\.empty(?:_like)?\s*(?:$|[,)\n])", "torch.empty bound to another name"),
    (r"\btorch\.empty(?:_like)?\b(?!\()", "torch.empty used without a call"),
]


def _package_sources():
    pkg = os.path.join(ROOT, "loftr_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in sorted(files):
            if f.endswith(".py"):
                yield os.path.relpath(os.path.join(dirpath, f), ROOT), open(os.path.join(dirpath, f)).read()


def test_package_allocates_only_through_patched_spellings():
    hits, n_empty = [], 0
    for rel, text in _package_sources():
        n_empty += len(re.findall(r"\btorch\.empty(?:_like)?\(", text))
        for pattern, what in UNPATCHED:
            for m in re.finditer(pattern, text, re.M):
                hits.append(f"{rel}:{text.count(chr(10), 0, m.start()) + 1}: {what}: {m.group(0).strip()!r}")
    assert not hits, "allocations tests/poison.py does not poison:\n" + "\n".join(hits)
    assert n_empty >= 50, n_empty     # the scan still sees the package's own allocations
