"""CPU: the host side of counting a text column cut into row-range shards — the ctypes mirror of
``lo_value_counts_text_shards``, the SASS of its merge kernels, and ``ShardedText`` with a test double standing in for
the devices."""
import ctypes as C
import re
import subprocess
from pathlib import Path

import pyarrow as pa
import pytest

from learningorchestra_b200 import _native
from learningorchestra_b200.sharding import ShardedText, all_shard_bounds

ROOT = Path(__file__).resolve().parent.parent
HEADER = ROOT / "include" / "loexec.h"


def test_ctypes_mirror_of_the_shards_entry_point_matches_the_header():
    text = re.sub(r"/\*.*?\*/", "", HEADER.read_text(), flags=re.S)
    assert int(re.search(r"#define LO_ABI_VERSION (\d+)", text).group(1)) == _native.LO_ABI_VERSION == 7
    params = [p.strip() for p in re.search(r"lo_value_counts_text_shards\s*\(([^)]*)\)", text).group(1).split(",")]
    assert params == ["lo_ctx *root", "const lo_text *const *shards", "const int64_t *row0", "int32_t nshards",
                      "int64_t *rep_rows_out", "uint64_t *counts_out", "int64_t capacity", "int64_t *ndistinct",
                      "lo_host_timing *timing"]
    res, args = _native.SIGNATURES["lo_value_counts_text_shards"]
    assert res is C.c_int
    assert args == [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.c_int32, C.c_void_p, C.c_void_p,
                    C.c_int64, C.POINTER(C.c_int64), C.POINTER(_native.HostTiming)]


def _sass_functions():
    sass = subprocess.run(["cuobjdump", "-sass", str(_native.LIB_PATH)], capture_output=True, text=True, check=True).stdout
    out, cur = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = out.setdefault(m.group(1), [])
        elif cur is not None:
            m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?);", line)
            if m:
                cur.append(m.group(1).strip())
    return out


def test_merge_kernels_add_64_bit_counts_in_global_memory_and_never_touch_local_memory(built):
    fns = _sass_functions()

    def one(name):
        found = [f for f in fns if re.search(r"\d%s[A-Z]" % name, f)]
        assert len(found) == 1, (name, found)
        return fns[found[0]]

    merge = one("k_hash_sum_str")
    assert any(re.search(r"\b(RED|ATOM)G?\.E\.ADD\.64\b", t) for t in merge)      # the shard's 64-bit count
    assert any("ATOMG.E.CAS.64" in t for t in merge)
    assert not any(re.search(r"\b(MATCH|ATOMS|LDS|STS)\b", t) for t in merge)      # no warp merge, no shared stage
    for name in ("k_hash_sum_str", "k_gather_lens", "k_gather_cells", "k_take_rows"):
        assert not any(re.search(r"\b(LDL|STL)\b", t) for t in one(name)), name


# ---- a test double for the devices ------------------------------------------------------------------------------
class _Piece:
    def __init__(self, owner, arr):
        self.owner, self.arr, self._h = owner, arr, object()
        self.n, self.nulls = len(arr), arr.null_count
        self.nbytes = 8 * (len(arr) + 1) + 3
        owner.live.add(id(self))

    def free(self):
        self.owner.live.discard(id(self))
        self._h = None


class _Device:
    """``Engine.text`` of one member: records the slices it is given, or raises like a full device."""

    def __init__(self, live, full=False):
        self.live, self.full, self.slices = live, full, []

    def text(self, arr, timing=None):
        self.slices.append(arr)
        if self.full:
            raise MemoryError("LO_ERR_NOMEM")
        if timing is not None:
            timing.update(total_ms=1.0 + len(self.slices), kernel_ms=0.5, h2d_bytes=float(len(arr)), d2h_bytes=0.0,
                          launches=0)
        return _Piece(self, arr)


def _column(n):
    return pa.array([None if i % 7 == 3 else "k%d" % (i % 5) for i in range(n)], type=pa.large_string())


@pytest.mark.parametrize("n,world", [(1000, 4), (70, 8), (3, 2), (0, 3), (33, 1)])
def test_pieces_follow_the_bounds_and_add_up(n, world):
    live = set()
    devs = [_Device(live) for _ in range(world)]
    arr = _column(n)
    bounds = all_shard_bounds(n, world)
    timing = {}
    t = ShardedText.upload(devs, bounds, arr, timing)
    assert t.arr is arr and t.offsets == [b for b, _ in bounds]
    for d, (b, e), p in zip(devs, bounds, t.pieces):
        assert len(d.slices) == 1 and d.slices[0].equals(arr.slice(b, e - b)) and p.owner is d
    assert t.n == n and t.nulls == arr.null_count
    assert t.nbytes == sum(p.nbytes for p in t.pieces) == sum(8 * (e - b + 1) + 3 for b, e in bounds)
    assert timing["h2d_bytes"] == n and timing["total_ms"] == 2.0
    assert len(live) == world
    t.free()
    assert not live and all(p._h is None for p in t.pieces)


def test_a_failed_upload_frees_the_pieces_already_made():
    live = set()
    devs = [_Device(live), _Device(live, full=True), _Device(live), _Device(live)]
    with pytest.raises(MemoryError):
        ShardedText.upload(devs, all_shard_bounds(500, 4), _column(500))
    assert all(len(d.slices) == 1 for d in devs)           # every member tried
    assert not live                                        # and nothing is left on any device
