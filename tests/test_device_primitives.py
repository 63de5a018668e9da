"""The generic device primitives on their own, each against a numpy reference of the same operation, exactly, at the
shapes where such kernels go wrong: tile ends, device-side lengths below the grid the host sized, uint32 sums that wrap,
long runs of equal keys across many tiles, empty lists.

  radix sort   radix.cuh   k_rs_ghist + k_rs_pass through yd::rs_sort (the product's LaunchSort sequence)
  scans        radix.cuh   k_scan_u32 (one block), k_scan_rows (one block per row, ticketed rows)
  compaction   filter.cuh  k_keep_count -> k_scan_u32 -> k_keep_scatter, 24- and 16-byte requests
  state merge  state.cuh   k_state_merge of W sorted lease lists (a range-sharded group's export)

The kernels run through tests/kernels/libydprim.so (tests/kernels/primitives.cu, `make primitives`): host wrappers that
launch the product's kernels from its own headers.  Every output buffer starts as 0xFF bytes, so each case also checks
that nothing past the live length was written."""
import ctypes as C

import numpy as np
import pytest

from conftest import ROOT, have_gpu

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not have_gpu(), reason="needs a CUDA device")]

LIB = ROOT / "tests" / "kernels" / "libydprim.so"
TILE = 1024  # yd::kRsTile, and the compaction's tile
DIGIT = 7  # yd::kRsBits
P = C.c_void_p
U32, U64 = C.c_uint32, C.c_ulonglong


@pytest.fixture(scope="module")
def prim():
    assert LIB.exists(), f"{LIB} missing: run build() or `make primitives`"
    lib = C.CDLL(str(LIB))
    lib.yd_prim_sort_u32.argtypes = [P, U64, U32, C.c_int, C.c_int, P, P]
    lib.yd_prim_sort_u64.argtypes = [P, U64, U32, C.c_int, C.c_int, P, P]
    lib.yd_prim_scan_u32.argtypes = [P, U64, U32, C.c_int, U32, U32, U32, P]
    lib.yd_prim_scan_rows.argtypes = [P, U64, U32, U32, U32]
    lib.yd_prim_compact.argtypes = [C.c_int, P, U32, P, P, P, P, P]
    lib.yd_prim_state_merge.argtypes = [P, U64, P, U32, P, U64]
    return lib


def ptr(a):
    return None if a is None else a.ctypes.data


def exclusive_scan_u32(v):
    """Exclusive prefix sums mod 2^32 and the total mod 2^32."""
    cs = np.cumsum(v.astype(np.uint64), dtype=np.uint64) & np.uint64(0xFFFFFFFF)
    ex = np.concatenate([np.zeros(1, np.uint64), cs[:-1]]) if len(v) else cs
    return ex.astype(np.uint32), int(cs[-1]) if len(v) else 0


# ---- radix sort -----------------------------------------------------------------------------------------------------

# key type -> (dtype, entry point, the product's bit range: slots.cuh's narrow codes use bits 3..30, wide ones 0..62)
SORT = {"u32": (np.uint32, "yd_prim_sort_u32", (3, 30)), "u64": (np.uint64, "yd_prim_sort_u64", (0, 62))}


def passes_of(bits):
    return (bits[1] - bits[0]) // DIGIT + 1


def check_sort(prim, kind, keys, nb=None, bits=None):
    dt, fn, product_bits = SORT[kind]
    first, last = bits or product_bits
    keys = np.ascontiguousarray(keys, dtype=dt)
    n = len(keys)
    nb = nb or max(1, -(-n // TILE))
    k_out, v_out = np.empty(nb * TILE, dt), np.empty(nb * TILE, np.uint32)
    assert getattr(prim, fn)(ptr(keys), n, nb, first, last, ptr(k_out), ptr(v_out)) == 0
    # the digits read are bits [first, first + 7 * passes) of the key; everything else must be ignored
    field = (keys.astype(np.uint64) >> np.uint64(first)) & np.uint64((1 << (DIGIT * passes_of((first, last)))) - 1)
    order = np.argsort(field, kind="stable")
    np.testing.assert_array_equal(v_out[:n], order.astype(np.uint32), err_msg="payload (stability)")
    np.testing.assert_array_equal(k_out[:n], keys[order], err_msg="keys")
    assert (v_out[n:] == 0xFFFFFFFF).all() and (k_out[n:] == np.iinfo(dt).max).all(), "written past n"
    return v_out[:n]


def sort_keys(kind, dist, n, rng, bits=None):
    dt, _, product_bits = SORT[kind]
    first, last = bits or product_bits
    width = 32 if kind == "u32" else 64
    span = min(DIGIT * passes_of((first, last)), width - first)  # in-range bits
    full = rng.integers(0, 2**width, n, dtype=np.uint64)
    in_mask = ((1 << span) - 1) << first
    out_mask = (2**width - 1) ^ in_mask
    noise = full & np.uint64(out_mask)  # bits the sort must ignore, bit 63 / 31 among them
    top = np.uint64(1 << (width - 1))
    if dist == "equal":  # identical keys, top bit set: every pass is the identity
        return np.full(n, (2**width - 1) ^ (1 << first), dtype=np.uint64).astype(dt)
    if dist == "equal-in-range":  # one in-range value, random bits around it: payload must stay arange(n)
        return (noise | np.uint64(0x5A5A5A5A5A5A5A5A & in_mask)).astype(dt)
    if dist == "two-alternating":  # the larger first: every tile moves half its keys past the other half
        a, b = np.uint64((5 << first) & in_mask), np.uint64((3 << first) & in_mask)
        return (np.where(np.arange(n) % 2 == 0, a, b) | top).astype(dt)
    if dist == "three-random":  # ties scattered over every tile, some with bits outside the range
        vals = np.array([(x << first) & in_mask for x in (9, 0, 2**span - 1)], dtype=np.uint64)
        return (vals[rng.integers(0, 3, n)] | noise).astype(dt)
    if dist == "descending":
        return ((np.arange(n, dtype=np.uint64)[::-1] << np.uint64(first)) & np.uint64(in_mask) | top).astype(dt)
    if dist == "random":
        return full.astype(dt)
    raise ValueError(dist)


SORT_N = [0, 1, 31, 32, 33, 1023, 1024, 1025, 8 * 1024 - 1, 8 * 1024, 8 * 1024 + 1, 130_000, 1_048_577]
SORT_DISTS = ["equal", "equal-in-range", "two-alternating", "three-random", "descending", "random"]


@pytest.mark.parametrize("dist", SORT_DISTS)
@pytest.mark.parametrize("n", SORT_N)
@pytest.mark.parametrize("kind", ["u32", "u64"])
def test_radix_sort_product_bits(prim, kind, n, dist):
    rng = np.random.default_rng(n * 7 + SORT_DISTS.index(dist))
    v = check_sort(prim, kind, sort_keys(kind, dist, n, rng))
    if dist.startswith("equal"):
        assert (v == np.arange(n, dtype=np.uint32)).all()


@pytest.mark.parametrize("extra", [1, 3, 40])
@pytest.mark.parametrize("n", [0, 1, 1000, 1025, 130_000])
@pytest.mark.parametrize("kind", ["u32", "u64"])
def test_radix_sort_grid_above_n(prim, kind, n, extra):
    """The grid sized for a larger table than the device-side n (the slot count is only known on the device): the
    surplus tiles draw tickets, publish empty counts and write nothing; n = 0 takes a grid of `extra` empty tiles."""
    rng = np.random.default_rng(n + extra)
    check_sort(prim, kind, sort_keys(kind, "three-random", n, rng), nb=max(1, -(-n // TILE)) + extra)


# bit ranges as LaunchSort takes them: 1, 2, an odd and an even number of passes, and the full 9 of 63 bits
BIT_RANGES = {
    "u32": [(5, 5), (0, 7), (4, 18), (3, 30), (0, 28), (25, 25)],
    "u64": [(57, 57), (10, 17), (20, 34), (1, 36), (0, 62), (30, 60)],
}


@pytest.mark.parametrize("n", [8 * 1024 + 1, 130_000])
@pytest.mark.parametrize("kind,bits", [(k, b) for k in BIT_RANGES for b in BIT_RANGES[k]])
def test_radix_sort_bit_ranges(prim, kind, bits, n):
    """Keys with every bit random, bit 63 / 31 included: only bits [first, first + 7 * passes) order them.  (57, 57)
    reads bits 57..63 of a u64: bit 63 is then part of the digit."""
    rng = np.random.default_rng(bits[0] * 100 + bits[1] + n)
    check_sort(prim, kind, sort_keys(kind, "random", n, rng, bits), bits=bits)
    check_sort(prim, kind, sort_keys(kind, "three-random", n, rng, bits), bits=bits)


@pytest.mark.parametrize("kind", ["u32", "u64"])
def test_radix_sort_one_live_digit(prim, kind):
    """Keys that differ in one pass's digit only: that pass scatters, every other pass in-range digit is one value and
    takes the identity shortcut (before and after the scattering pass, so with and without an input payload)."""
    bits = SORT[kind][2]
    rng = np.random.default_rng(3)
    n = 20 * TILE + 17
    for p in range(passes_of(bits)):
        shift = bits[0] + p * DIGIT
        keys = (np.uint64(0x2A) << np.uint64(bits[0])) | (rng.integers(0, 128, n).astype(np.uint64) << np.uint64(shift))
        if kind == "u32":
            keys &= np.uint64(0xFFFFFFFF)
        check_sort(prim, kind, keys)


def slot_codes(wide, n_servants, seed):
    """A static slot table in slots.cuh's format: per servant the codes of r = 0 .. cap - 1, rows in registry order;
    narrow code = tier << 30 | floor(r * 2^27 / cap) << 3, wide code = tier << 62 | the double r / cap."""
    rng = np.random.default_rng(seed)
    rows = []
    for _ in range(n_servants):
        cap = int(rng.choice([1, 2, 3, 4, 8, 12, 16, 48, 64, 96]))
        nproc = int(rng.choice([4, 8, 16, 64]))
        dedicated = rng.random() < 0.5
        r = np.arange(cap, dtype=np.uint64)
        tier = ~(dedicated & (2 * r < nproc))
        if wide:
            rows.append(np.where(tier, np.uint64(1 << 62), np.uint64(0)) | (r / cap).view(np.uint64))
        else:
            rows.append(np.where(tier, np.uint64(1 << 30), np.uint64(0)) | (((r << np.uint64(27)) // np.uint64(cap)) << np.uint64(3)))
    return np.concatenate(rows)


@pytest.mark.parametrize("n_servants", [300, 4000])
@pytest.mark.parametrize("kind", ["u32", "u64"])
def test_radix_sort_slot_codes(prim, kind, n_servants):
    """The sort as the slot-stream solver runs it: equal codes (every idle servant's r = 0, equal fractions) must keep
    registry order, which is the reference's `first minimum wins`."""
    check_sort(prim, kind, slot_codes(kind == "u64", n_servants, n_servants))


# ---- k_scan_u32 -----------------------------------------------------------------------------------------------------

GUARD = 7


def run_scan_u32(prim, data, n_static=0, n_dyn=None, per_dyn=0, dyn_cap=0):
    buf = data.copy()
    total = np.zeros(1, np.uint32)
    assert prim.yd_prim_scan_u32(ptr(buf), len(buf), n_static, n_dyn is not None, n_dyn or 0, per_dyn, dyn_cap,
                                 ptr(total)) == 0
    return buf, int(total[0])


def scan_values(n, rng):
    # large values so that partial sums wrap 2^32 many times; a run of 0xFFFFFFFF wraps at every step
    v = rng.integers(2**31, 2**32, n, dtype=np.uint64).astype(np.uint32)
    v[: min(n, 40)] = 0xFFFFFFFF
    return v


@pytest.mark.parametrize("n", [0, 1, 8191, 8192, 8193, 3 * 8192 + 5])
def test_scan_u32_static(prim, n):
    rng = np.random.default_rng(n)
    data = np.concatenate([scan_values(n, rng), np.full(GUARD, 0xA5A5A5A5, np.uint32)])
    out, total = run_scan_u32(prim, data, n_static=n)
    ex, tot = exclusive_scan_u32(data[:n])
    np.testing.assert_array_equal(out[:n], ex)
    assert total == tot
    assert (out[n:] == 0xA5A5A5A5).all(), "written past n"


@pytest.mark.parametrize("per_dyn", [1, 3, 97])
@pytest.mark.parametrize("n_dyn", [0, 1, 99, 100, 101, 5000])
def test_scan_u32_dynamic(prim, n_dyn, per_dyn):
    """Length min(*n_dyn, dyn_cap) * per_dyn + 1 from the device: below, at and above the cap the host sized for
    (97 * 100 + 1 > 8192 takes two block-wide rounds)."""
    cap = 100
    rng = np.random.default_rng(n_dyn * 1000 + per_dyn)
    sized = cap * per_dyn + 1
    data = np.concatenate([scan_values(sized, rng), np.full(GUARD, 0xA5A5A5A5, np.uint32)])
    out, total = run_scan_u32(prim, data, n_static=12345, n_dyn=n_dyn, per_dyn=per_dyn, dyn_cap=cap)
    n = min(n_dyn, cap) * per_dyn + 1
    ex, tot = exclusive_scan_u32(data[:n])
    np.testing.assert_array_equal(out[:n], ex)
    assert total == tot
    np.testing.assert_array_equal(out[n:], data[n:], err_msg="written past the device-side length")


# ---- k_scan_rows ----------------------------------------------------------------------------------------------------


def check_scan_rows(prim, grid, n_rows, per_row, seed):
    rng = np.random.default_rng(seed)
    rows = min(n_rows, grid)
    size = grid * per_row + 1 + GUARD
    data = scan_values(size, rng)
    data[-GUARD:] = 0xA5A5A5A5
    out = data.copy()
    assert prim.yd_prim_scan_rows(ptr(out), len(out), grid, n_rows, per_row) == 0
    live = rows * per_row
    if rows:
        ex, tot = exclusive_scan_u32(data[:live])
        np.testing.assert_array_equal(out[:live], ex)
        assert int(out[live]) == tot, "end cell"
        live += 1
    np.testing.assert_array_equal(out[live:], data[live:], err_msg="written past the live rows")


@pytest.mark.parametrize("per_row", [1, 8191, 8192, 8193, 20_000])
@pytest.mark.parametrize("rows", [1, 2, 33, 255, 256])
def test_scan_rows(prim, rows, per_row):
    """One exclusive scan of the whole row-major matrix plus the end cell, however the rows split into 8192-item
    rounds and whichever order the blocks draw their row tickets in."""
    check_scan_rows(prim, rows, rows, per_row, rows * 100_000 + per_row)


@pytest.mark.parametrize("grid,n_rows", [(256, 0), (256, 1), (256, 100), (256, 255), (33, 5), (33, 32), (2, 1),
                                         (33, 40)])
@pytest.mark.parametrize("per_row", [1, 8193])
def test_scan_rows_device_row_count(prim, grid, n_rows, per_row):
    """*n_rows_dyn below gridDim.x (the class count is only known on the device): the surplus blocks draw tickets and
    leave; nothing past the last live row's end cell is written.  Above gridDim.x it is clamped to the grid."""
    check_scan_rows(prim, grid, n_rows, per_row, grid * 1000 + n_rows + per_row)


# ---- compaction of the pre-filtered queue ---------------------------------------------------------------------------

REQ24 = np.dtype([("env", "<u4"), ("min_version", "<u4"), ("ip", "<u4"), ("flags", "<u4"), ("expires_ns", "<i8")])
REQ16 = np.dtype([("env", "<u4"), ("min_version", "<u4"), ("ip", "<u4"), ("lease", "<u4")])
LEASE_PREFETCH = 0x80000000
COMPACT_N = [1, 31, 32, 33, 1023, 1024, 1025, 7 * 1024 + 3, 200_003]


def keep_pattern(pattern, n, rng):
    if pattern == "random":
        return rng.random(n) < 0.6
    if pattern == "all":
        return np.ones(n, bool)
    if pattern == "none":
        return np.zeros(n, bool)
    if pattern == "last-lane":  # only lane 31 of each warp: one survivor per warp, every warp's offset counts
        return np.arange(n) % 32 == 31
    raise ValueError(pattern)


def compact_inputs(width, n, keep, bloom, rt, rng):
    if width == 24:
        reqs = np.frombuffer(rng.integers(0, 256, n * 24, dtype=np.uint8).tobytes(), REQ24).copy()
    else:
        reqs = np.zeros(n, REQ16)
        for f in ("env", "min_version", "ip"):
            reqs[f] = rng.integers(0, 2**32, n, dtype=np.uint64)
        ms = np.array([0, 30_000, 2**31 - 1], np.uint64)[rng.integers(0, 3, n)]
        other = rng.random(n) < 0.25
        ms[other] = rng.integers(0, 2**31, int(other.sum()), dtype=np.uint64)
        reqs["lease"] = (ms | np.where(rng.random(n) < 0.5, np.uint64(LEASE_PREFETCH), np.uint64(0))).astype(np.uint32)
    # a dropped request is a cache hit, a joined task or both (the cache is consulted first)
    how = rng.integers(0, 3, n)  # 0 cache, 1 joined, 2 both
    if bloom and not rt:
        how[:] = 0
    if rt and not bloom:
        how[:] = 1
    drop = ~keep
    bloom_hit = rt_hit = None
    if bloom:
        bloom_hit = np.where(drop & (how != 1), rng.integers(1, 256, n), 0).astype(np.uint8)
    if rt:
        rt_hit = rng.integers(0, 2**32, (n, 4), dtype=np.uint64).astype(np.uint32)  # only .w (found) counts
        found = np.array([1, 0x80000000, 0xFFFFFFFF], np.uint32)[rng.integers(0, 3, n)]
        rt_hit[:, 3] = np.where(drop & (how != 0), found, 0)
    return reqs, bloom_hit, rt_hit


def expected_queue(width, reqs):
    if width == 24:
        return reqs
    out = np.zeros(len(reqs), REQ24)
    for f in ("env", "min_version", "ip"):
        out[f] = reqs[f]
    out["flags"] = np.where(reqs["lease"] & LEASE_PREFETCH, 1, 0)
    out["expires_ns"] = (reqs["lease"] & 0x7FFFFFFF).astype(np.int64) * 1_000_000
    return out


# (filter stages given, which requests survive); with no stage (both hit arrays null) every request survives
COMPACT_CASES = [(f, p) for f in ("cache+dedupe", "cache", "dedupe") for p in ("random", "all", "none", "last-lane")]
COMPACT_CASES.append(("none", "all"))


@pytest.mark.parametrize("filters,pattern", COMPACT_CASES)
@pytest.mark.parametrize("n", COMPACT_N)
@pytest.mark.parametrize("width", [24, 16])
def test_compaction(prim, width, n, filters, pattern):
    """verdict = 1 on a cache hit, else 2 on a joined task, else 0; the verdict-0 requests in queue order, 16-byte ones
    unpacked (milliseconds -> nanoseconds, the prefetch bit -> YD_REQ_FLAG_PREFETCH); tile offsets scanned with the
    survivor count behind them."""
    bloom, rt = "cache" in filters, "dedupe" in filters
    rng = np.random.default_rng(n * 31 + width)
    keep = keep_pattern(pattern, n, rng)
    reqs, bloom_hit, rt_hit = compact_inputs(width, n, keep, bloom, rt, rng)
    nt = -(-n // TILE)
    verdict, tile_off = np.empty(n, np.uint8), np.empty(nt + 1, np.uint32)
    out = np.empty(n, REQ24)
    assert prim.yd_prim_compact(width == 16, ptr(reqs), n, ptr(bloom_hit), ptr(rt_hit), ptr(verdict), ptr(tile_off),
                                ptr(out)) == 0
    b = bloom_hit if bloom_hit is not None else np.zeros(n, np.uint8)
    r = rt_hit[:, 3] if rt_hit is not None else np.zeros(n, np.uint32)
    want_verdict = np.where(b != 0, 1, np.where(r != 0, 2, 0)).astype(np.uint8)
    np.testing.assert_array_equal(verdict, want_verdict)
    kept = want_verdict == 0
    per_tile = np.add.reduceat(kept.astype(np.uint32), np.arange(0, n, TILE))
    ex, tot = exclusive_scan_u32(per_tile)
    np.testing.assert_array_equal(tile_off[:nt], ex)
    assert int(tile_off[nt]) == tot == int(kept.sum())
    want = expected_queue(width, reqs[kept])
    assert out[:tot].tobytes() == want.tobytes(), "compacted queue"
    assert set(out[tot:].tobytes()) <= {0xFF}, "written past the survivors"


# ---- k_state_merge --------------------------------------------------------------------------------------------------

LEASE = np.dtype([("id", "<u8"), ("servant", "<u4"), ("flags", "<u4"), ("expires_rel", "<i8")])


def merge_lists(layout, W, base, rng):
    """W lists of lease ids, disjoint (a lease lives on one rank), each ascending."""
    if layout == "random":
        ids = np.sort(rng.choice(5000, 3000, replace=False)).astype(np.uint64) + np.uint64(base)
        owner = rng.integers(0, W, len(ids))
        return [ids[owner == q] for q in range(W)]
    if layout == "some-empty":  # every other rank holds nothing (with W = 1 the only list is empty)
        ids = np.arange(700, dtype=np.uint64) * np.uint64(3) + np.uint64(base)
        live = [q for q in range(W) if q % 2 == 1]
        owner = rng.choice(live, len(ids)) if live else None
        return [ids[owner == q] if live else ids[:0] for q in range(W)]
    if layout == "unequal":  # one long list, the others one or two records, all padded to the long one
        ids = np.arange(5000, dtype=np.uint64) + np.uint64(base)
        short = rng.choice(len(ids), 2 * (W - 1), replace=False)
        lists = [np.sort(ids[short[2 * q: 2 * q + 1 + q % 2]]) for q in range(W - 1)]
        return [np.setdiff1d(ids, ids[short])] + lists
    if layout == "stacked":  # rank q's ids all below rank q + 1's
        return [np.arange(q * 400, q * 400 + 300 + 50 * q, dtype=np.uint64) + np.uint64(base) for q in range(W)]
    if layout == "stacked-reversed":  # rank q's ids all above rank q + 1's
        return [np.arange((W - q) * 400, (W - q) * 400 + 300, dtype=np.uint64) + np.uint64(base) for q in range(W)]
    raise ValueError(layout)


@pytest.mark.parametrize("base", [0, 2**32 - 1500, 2**63 - 1500, 2**64 - 30_000], ids=["0", "2^32", "2^63", "2^64"])
@pytest.mark.parametrize("layout", ["random", "some-empty", "unequal", "stacked", "stacked-reversed"])
@pytest.mark.parametrize("W", [1, 2, 3, 4])
def test_state_merge(prim, W, layout, base):
    """The merged list is the stable sort of the concatenated lists by id; each list's padding (garbage records up to
    `stride`) is never read as a record."""
    rng = np.random.default_rng(W * 10 + len(layout))
    ids = merge_lists(layout, W, base, rng)
    counts = np.array([len(l) for l in ids], np.uint64)
    stride = max(1, int(counts.max()))
    lists = np.zeros(stride * W, LEASE)
    pad = rng.integers(0, 2**64, stride * W, dtype=np.uint64)
    pad[::3] = 0  # padding that would sort first
    lists["id"] = pad
    lists["servant"] = rng.integers(0, 2**32, stride * W, dtype=np.uint64)
    lists["flags"] = rng.integers(0, 4, stride * W)
    lists["expires_rel"] = rng.integers(-2**62, 2**62, stride * W)
    for q in range(W):
        lists["id"][q * stride: q * stride + len(ids[q])] = ids[q]
    live = np.concatenate([lists[q * stride: q * stride + int(counts[q])] for q in range(W)])
    want = live[np.argsort(live["id"], kind="stable")]
    out = np.empty(len(live) + GUARD, LEASE)
    assert prim.yd_prim_state_merge(ptr(lists), stride, ptr(counts), W, ptr(out), len(out)) == 0
    assert out[: len(live)].tobytes() == want.tobytes()
    assert set(out[len(live):].tobytes()) <= {0xFF}, "written past the merged list"


def test_state_merge_many_blocks(prim):
    """300 k leases over four ranks, ids past 2^32: many blocks per list, lists of different lengths."""
    rng = np.random.default_rng(11)
    ids = np.arange(300_000, dtype=np.uint64) + np.uint64(2**32 - 100_000)
    owner = rng.choice(4, len(ids), p=[0.5, 0.3, 0.15, 0.05])
    counts = np.array([(owner == q).sum() for q in range(4)], np.uint64)
    stride = int(counts.max())
    lists = np.zeros(stride * 4, LEASE)
    for q in range(4):
        seg = lists[q * stride: q * stride + int(counts[q])]
        seg["id"] = ids[owner == q]
        seg["servant"] = q
    live = np.concatenate([lists[q * stride: q * stride + int(counts[q])] for q in range(4)])
    want = live[np.argsort(live["id"], kind="stable")]
    out = np.empty(len(live) + GUARD, LEASE)
    assert prim.yd_prim_state_merge(ptr(lists), stride, ptr(counts), 4, ptr(out), len(out)) == 0
    assert out[: len(live)].tobytes() == want.tobytes()
    assert set(out[len(live):].tobytes()) <= {0xFF}
