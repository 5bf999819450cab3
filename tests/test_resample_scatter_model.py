"""Integer model of resample_scatter_kernel (csrc/resample.cuh): with the systematic comb t_j = offset + j*stride the
slots that select particle i are [ja_i, jb_i) with ja/jb from two integer divisions.  Checked here against the
per-slot definition (smallest i with cdf[i] > t_j, what resample_kernel and the oracle compute), on one shard and
split over ranks, with python integers.  CPU only."""
import numpy as np
import pytest

from beluga_b200.distributed import cdf_offsets, slot_ranges


def comb_slots_before(position, offset, stride, total_slots):
    """Number of slots j with offset + j * stride < position (resample.cuh: comb_slots_before)."""
    if position <= offset:
        return 0
    return min((position - offset + stride - 1) // stride, total_slots)


def scatter_ancestors(cdf, offset, stride, m, cdf_offset=0):
    out = {}
    for i in range(len(cdf)):
        lo = cdf_offset + (int(cdf[i - 1]) if i > 0 else 0)
        hi = cdf_offset + int(cdf[i])
        for j in range(comb_slots_before(lo, offset, stride, m), comb_slots_before(hi, offset, stride, m)):
            assert j not in out
            out[j] = i
    return out


def searched_ancestors(cdf, offset, stride, m):
    positions = [offset + j * stride for j in range(m)]
    return np.searchsorted(np.asarray(cdf, dtype=object), positions, side="right")  # smallest i with cdf[i] > t


@pytest.mark.parametrize("n,m", [(1, 1), (7, 7), (100, 100), (100, 333), (333, 100), (1000, 1000)])
@pytest.mark.parametrize("kind", ["gamma", "collapse", "zeros"])
def test_scatter_equals_search(n, m, kind):
    rng = np.random.default_rng(n * 1000 + m)
    if kind == "gamma":
        q = rng.integers(1, 1 << 40, n)
    elif kind == "collapse":
        q = np.ones(n, dtype=np.int64)
        q[rng.integers(0, n)] = 1 << 50
    else:
        q = rng.integers(0, 1 << 40, n) * rng.integers(0, 2, n)
        q[rng.integers(0, n)] += 1 << 30
    cdf = np.cumsum(q.astype(object))
    total = int(cdf[-1])
    stride = total // m
    for offset in {0, stride // 2, max(stride - 1, 0)}:
        got = scatter_ancestors(cdf, offset, stride, m)
        want = searched_ancestors(cdf, offset, stride, m)
        assert sorted(got) == list(range(m))  # every slot filled exactly once
        assert [got[j] for j in range(m)] == [int(i) for i in want]


@pytest.mark.parametrize("world", [2, 3, 8])
def test_sharded_scatter_covers_every_slot_once(world):
    """Every rank scatters its own particles with positions shifted by the lower ranks' totals; together they fill
    the global slots exactly like one shard would, and each rank's slots are the contiguous range slot_ranges() names."""
    rng = np.random.default_rng(world)
    shard = 200
    m = world * shard
    parts = [rng.integers(0, 1 << 36, shard).astype(object) for _ in range(world)]
    parts[1][:] = 0  # a rank without weight
    parts[1][5] = 3
    totals = [int(p.sum()) for p in parts]
    offsets = cdf_offsets(totals)
    total = offsets[-1]
    stride = total // m
    offset = stride // 3
    whole = searched_ancestors(np.cumsum(np.concatenate(parts)), offset, stride, m)
    ranges = slot_ranges(offsets, stride, offset, m)
    seen = {}
    for r in range(world):
        local = scatter_ancestors(np.cumsum(parts[r]), offset, stride, m, cdf_offset=offsets[r])
        if local:
            assert (min(local), max(local) + 1) == ranges[r]
        else:
            assert ranges[r][0] == ranges[r][1]
        for j, i in local.items():
            assert j not in seen
            seen[j] = r * shard + i
    assert [seen[j] for j in range(m)] == [int(i) for i in whole]


def comb_slots_before_magic(position, offset, stride, magic, total_slots):
    """resample.cuh: comb_slots_before_magic -- the division replaced by __umul64hi with magic = floor((2^64 - 1) / stride) and one
    remainder check.  64-bit wrap-around arithmetic is modelled with masks."""
    mask = (1 << 64) - 1
    if position <= offset:
        return 0
    x = (position - offset + stride - 1) & mask
    j = (x * magic) >> 64
    if ((x - j * stride) & mask) >= stride:
        j += 1
    return min(j, total_slots)


def test_reciprocal_multiply_is_the_division():
    """The high word of x * magic is floor(x / stride) or one below it for every x < 2^64; the remainder check settles which.
    Totals stay below 2^62 (tests/test_quantize_model.py), so x = position - offset + stride - 1 cannot wrap."""
    import random

    rng = random.Random(5)
    mask = (1 << 64) - 1
    strides = [1, 2, 3, 7, 1 << 20, (1 << 20) + 1, (1 << 40) - 1, 1 << 61, (1 << 62) - 1] + [rng.randrange(1, 1 << 62) for _ in range(200)]
    for stride in strides:
        magic = mask // stride
        xs = [0, 1, stride - 1, stride, stride + 1, 2 * stride - 1, 2 * stride, mask, mask - 1, (1 << 63) - 1, (1 << 63)]
        xs += [rng.randrange(0, mask // stride + 1) * stride + d for _ in range(20) for d in (-1, 0, 1)]
        xs += [rng.randrange(0, 1 << 64) for _ in range(50)]
        for x in xs:
            if not (0 <= x <= mask):
                continue
            j = (x * magic) >> 64
            q = x // stride
            assert j in (q, q - 1), (x, stride)
            if ((x - j * stride) & mask) >= stride:
                j += 1
            assert j == q
    # and through the function, against the plain division, at CDF scale
    for _ in range(2000):
        total = rng.randrange(1 << 30, 1 << 62)
        m = rng.randrange(1, 1 << 24)
        stride = max(total // m, 1)
        offset = rng.randrange(0, stride)
        position = rng.randrange(0, total + 1)
        assert comb_slots_before_magic(position, offset, stride, mask // stride, m) == comb_slots_before(position, offset, stride, m)
