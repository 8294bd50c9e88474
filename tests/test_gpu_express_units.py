"""The express lane (scan_sum_express_kernel) decodes a page in 4 KB units -- one TMA stage, two 2 KB halves, a 64-byte window per
lane in each -- with the unmasked word on every unit: the bytes in front of the body, behind it and beyond the copied stage reach
the word as zeros, which the terminator count corrects for.  These tests put page bodies and 3-byte varints on both sides of every
edge that geometry has (16-byte piece, 64-byte window, 2 KB half, 4 KB unit), against the oracle and the express-lane counter, on
resident parts and on the cold host path (pageable and pinned).

The interesting blocks sit at the front of a part of ~72k blocks: a warp takes up to 8 blocks per cursor increment only while more
than 16 blocks per warp are left, so they are streamed through the batch ring one after another (a page after a page of long
varints, a page after a 1-row block, a page after a wide page that left the ring)."""
import numpy as np
import pytest

from oracle import oracle as O
from tests.helpers import STEP, T0, assert_parity, build_part, to_gpu_query
from tests.test_gpu_lanes import NARROW3, WIDE, _varint_lengths, assert_lanes, page_class
from tests.test_gpu_masks import host_images

gpu = pytest.mark.gpu

_RANGES = {1: (0, 63), 2: (64, 8191), 3: (8192, NARROW3), 4: (WIDE, WIDE)}   # |delta| -> zig-zag varint of that many bytes


def values_with_lengths(lengths, rng):
    """int64 values of one block whose delta page body holds varints of exactly these lengths (first value 1000; the first two
    deltas have opposite signs, so the writer keeps the delta encoding)."""
    k = len(lengths)
    mag = np.array([rng.integers(max(_RANGES[L][0], 1 if i < 2 else 0), _RANGES[L][1] + 1) for i, L in enumerate(lengths)], np.int64)
    sign = np.where(rng.random(k) < 0.5, -1, 1)
    if k >= 1:
        sign[0] = 1
    if k >= 2:
        sign[1] = -1
    d = mag * sign
    # zig-zag: -64 is a 1-byte varint and -8192 a 2-byte one; move such draws into their class
    d = np.where((np.asarray(lengths) == 2) & (d == -64), -65, d)
    d = np.where((np.asarray(lengths) == 3) & (d == -8192), -8193, d)
    d = np.where(np.asarray(lengths) == 4, WIDE, d)   # -WIDE is a 3-byte varint
    return np.concatenate([[1000], 1000 + np.cumsum(d)]).astype(np.int64)


def body_lengths(body, long_at=None, long_len=3, max_rows=8193):
    """varint lengths of a body of `body` bytes: 1-byte varints, 2-byte ones where the block would need more than max_rows rows,
    and one `long_len`-byte varint starting at body byte `long_at`."""
    lens = []
    pos = 0
    while pos < body:
        left = body - pos
        if long_at is not None and pos == long_at:
            L = long_len
        else:
            rows_left = max_rows - 1 - len(lens)
            L = 2 if left > rows_left and left >= 2 else 1
            if long_at is not None and pos < long_at < pos + L:
                L = 1
        lens.append(L)
        pos += L
    return lens


def _edges():
    """(name, varint lengths) of the boundary blocks."""
    out = []
    for e in (16, 64, 2048, 4096, 6144, 8192, 12288):
        for b in (e - 1, e, e + 1):
            out.append((f"body {b}", body_lengths(b)))
    for b in (1, 2, 15800, 16383):
        out.append((f"body {b}", body_lengths(b)))
    for e in (2048, 4096, 6144, 8192, 10240, 12288):   # a 3-byte varint before, on and after every half / unit edge
        for at in (e - 3, e - 2, e - 1, e, e + 1):
            out.append((f"3-byte at {at}", body_lengths(14000, long_at=at)))
    out.append(("3-byte first", body_lengths(9000, long_at=0)))
    out.append(("3-byte last", body_lengths(9000, long_at=8997)))
    out.append(("3-byte in a short page", body_lengths(40, long_at=20)))
    lens = body_lengths(9000, long_at=2047)                                   # a 4-byte varint after the switch
    lens[3000] = 4
    out.append(("4-byte after the switch", lens))
    lens = body_lengths(9000, long_at=2046)                                   # ... and in a later unit
    lens[-1000] = 4
    out.append(("4-byte in a later unit", lens))
    return out


def _blocks(rng, n_pad=72_000):
    """-> ((name, int64 values) of every block in series order, number of boundary blocks in front of the padding).  The
    pages keep their varints (no dense form, tests/test_gpu_dense_boundaries.py), so these blocks pin the SWAR decode."""
    blocks = []
    for name, lens in _edges():
        blocks.append((name, values_with_lengths(lens, rng)))
        # behind every boundary block: a page of long varints, a narrow page, a 1-row block
        blocks.append(("3-byte page", values_with_lengths([3] * 300, rng)))
        blocks.append(("narrow after long", values_with_lengths(body_lengths(5000), rng)))
        blocks.append(("one row", np.array([int(rng.integers(0, 100))], np.int64)))
    n_lead = len(blocks)
    for _ in range(n_pad):
        blocks.append(("pad", values_with_lengths([1] * 23, rng)))
    return blocks, n_lead


def _part(rng, n_pad=72_000):
    blocks, n_lead = _blocks(rng, n_pad)
    express = slow = 0
    for name, v in blocks[:n_lead]:
        cls = page_class(v, None, True) if v.size > 1 else "const"
        if name.startswith("body"):
            lens = _varint_lengths(O.int64_list_encode(v)[0])
            assert sum(lens) == int(name.split()[1]), name
        express += cls == "delta"
        slow += cls == "wide"
    express += n_pad
    sizes = [v.size for _, v in blocks]
    sids = np.repeat(np.arange(1, len(blocks) + 1, dtype=np.uint64), sizes)
    ts = np.concatenate([T0 + np.arange(n, dtype=np.int64) * STEP for n in sizes])
    m = np.concatenate([v for _, v in blocks])
    part = build_part(sids, ts, np.ones(sids.size, np.int64), [("i", O.VT_INT64, m, None), ("f", O.VT_FLOAT64, m / 100.0, None)])
    return part, np.unique(sids), express, slow


@pytest.fixture(scope="module")
def express_part():
    return _part(np.random.default_rng(4096))


AGGS = [("i", O.AGG_SUM), ("i", O.AGG_COUNT), ("f", O.AGG_SUM), ("f", O.AGG_MEAN)]


@gpu
@pytest.mark.parametrize("host", [None, "pageable", "pinned"], ids=["resident", "cold-pageable", "cold-pinned"])
def test_express_units_at_every_edge(bydb, gpu_ctx, express_part, host):
    part, usid, express, slow = express_part
    oq = O.Query([part], usid, AGGS, groups=(np.arange(usid.size) % 4096).astype(np.int32), n_groups=4096)
    if host is None:
        h = gpu_ctx.register_part(77_000, part.files())
        try:
            got = gpu_ctx.scan_agg(to_gpu_query(bydb, [h], oq))
        finally:
            gpu_ctx.release_part(h)
    else:
        q = to_gpu_query(bydb, [], oq)
        q.flags = bydb.capi.Q_HOST_ZERO_COPY if host == "pinned" else 0
        got = gpu_ctx.scan_agg_host(host_images([part], host == "pinned"), q)
    want = O.run_query(oq)
    assert_parity(got, want, AGGS, f"express units/{host}")
    assert_lanes(got, express, slow, f"express units/{host}")
