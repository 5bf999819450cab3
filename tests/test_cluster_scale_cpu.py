"""A vectorised NumPy restatement of the spatial hash and of the particle-cloud histogram, so that the clusterizer can be
checked at 10^6-10^7 particles (tests/test_gpu_cluster_scale.py) without a per-particle Python loop.

spatial_hash follows the rule of se2_math.cuh and the oracle: floor(v) as an int64, INT64_MIN when floor(v) is NaN or
outside [-2^63, 2^63); the Fibonacci multiply modulo 2^64; rotations by 0, 21 and 42 bits for x, y and the heading.
histogram groups the particles by hash as beluga_ros/particle_cloud.hpp:197-210 does: bins in the order of their first
particle, that particle's index, the count, and the weight added up one particle after another in particle order.

Both are pinned here to the oracle's spatial_hash and to a plain Python loop, on random states and at the edges of the
double range."""
import math

import numpy as np
import pytest

from test_gpu_integer_edges import EDGE
from test_integer_edges_cpu import spatial_hash as py_spatial_hash

FIB = np.uint64(11400714819323198485)
INT64_MIN = np.iinfo(np.int64).min


def floor_to_int64(v):
    f = np.floor(np.asarray(v, dtype=np.float64))
    inside = (f >= -(2.0**63)) & (f < 2.0**63)  # False for NaN
    out = np.where(inside, f, 0.0).astype(np.int64)
    out[~inside] = INT64_MIN
    return out


def fibo_hash(v, shift):
    h = floor_to_int64(v).view(np.uint64) * FIB  # wraps modulo 2^64
    if shift == 0:
        return h
    return (h << np.uint64(shift)) | (h >> np.uint64(64 - shift))


def spatial_hash(states, rx, ry, rtheta):
    """spatial_hash<SE2d>{rx, ry, rtheta} of every row (cos, sin, x, y) -> uint64 array."""
    s = np.asarray(states, dtype=np.float64).reshape(-1, 4)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        return fibo_hash(s[:, 2] / rx, 0) ^ fibo_hash(s[:, 3] / ry, 21) ^ fibo_hash(np.arctan2(s[:, 1], s[:, 0]) / rtheta, 42)


def histogram(states, weights, linear, angular):
    """-> (first index, count, weight) per bin in first-occurrence order, and the bin of every particle.  The weight of a
    bin is 0.0 + w[i0] + w[i1] + ... over its particles in index order: np.add.at applies its updates one by one, in the
    order of the index array."""
    h = spatial_hash(states, linear, linear, angular)
    _, first, inverse, count = np.unique(h, return_index=True, return_inverse=True, return_counts=True)
    order = np.argsort(first, kind="stable")  # sorted-hash rank -> first-occurrence rank
    rank = np.empty_like(order)
    rank[order] = np.arange(len(order))
    bin_of = rank[inverse.reshape(-1)]
    weight = np.zeros(len(order))
    np.add.at(weight, bin_of, np.asarray(weights, dtype=np.float64))
    return first[order], count[order], weight, bin_of


def loop_histogram(states, weights, linear, angular, hash_fn):
    seen, order = {}, []
    for i, st in enumerate(states):
        h = hash_fn(st, linear, linear, angular)
        if h not in seen:
            seen[h] = [i, 0, 0.0]
            order.append(h)
        seen[h][1] += 1
        seen[h][2] += float(weights[i])
    return [seen[h] for h in order]


def random_states(rng, n, extent):
    th = rng.uniform(-math.pi, math.pi, n)
    return np.stack([np.cos(th), np.sin(th), rng.uniform(-extent, extent, n), rng.uniform(-extent, extent, n)], axis=1)


def edge_states():
    """Every EDGE value (NaN, +-inf, +-1e300, +-2^63 and beyond, +-9.3e18) as x, as y, and as the heading's cosine and
    sine, next to the heading's +-pi with a signed zero sine."""
    rows = []
    for v in EDGE:
        rows += [(1.0, 0.0, v, 0.25), (1.0, 0.0, 0.25, v), (v, 0.0, 0.25, 0.25), (-1.0, v, 0.25, 0.25), (1.0, v, -0.25, 0.25)]
    rows += [(-1.0, 0.0, 0.5, 0.5), (-1.0, -0.0, 0.5, 0.5), (0.0, -0.0, -0.5, -0.5)]
    return np.array(rows)


RESOLUTIONS = [(0.2, 0.524), (1e-3, 1e-3), (0.5, 0.17453292519943295), (0.05, 0.1)]


@pytest.mark.parametrize("linear, angular", RESOLUTIONS)
def test_spatial_hash_matches_the_oracle_and_the_loop(orc, linear, angular):
    rng = np.random.default_rng(int(linear * 1000) + 3)
    states = np.concatenate([random_states(rng, 3000, 60.0), random_states(rng, 300, 1e6), edge_states()])
    got = spatial_hash(states, linear, linear, angular)
    assert got.dtype == np.uint64
    for st, h in zip(states, got):
        assert int(h) == orc.spatial_hash(st, linear, linear, angular) == py_spatial_hash(st, linear, linear, angular), st


def test_floor_to_int64_at_the_edges():
    v = np.array([-0.0, 5e-324, -5e-324, 1.0, np.nextafter(1.0, 0.0), -1.0, np.nextafter(-1.0, -2.0), 2.0**63 - 1024,
                  -(2.0**63), 2.0**63, np.nextafter(-(2.0**63), -math.inf), math.nan, math.inf, -math.inf, 1e300, -1e300])
    want = [0, 0, -1, 1, 0, -1, -2, 2**63 - 1024] + [-(2**63)] * 8
    assert floor_to_int64(v).tolist() == want


@pytest.mark.parametrize("linear, angular", RESOLUTIONS[:3])
def test_histogram_matches_a_plain_loop(orc, linear, angular):
    """Bins in first-occurrence order, first index, count and the sequential weight sum (bit for bit) against a Python
    loop over the particles: a resampled-looking cloud (many exact copies), non-unit weights spanning many magnitudes, so
    that the order of the additions shows in the last bits, and the edge states."""
    rng = np.random.default_rng(17)
    base = np.concatenate([random_states(rng, 400, 3.0), edge_states()])
    states = base[rng.integers(0, len(base), 6000)]
    weights = rng.uniform(0.0, 1.0, len(states)) * 10.0 ** rng.integers(-8, 8, len(states))
    first, count, weight, bin_of = histogram(states, weights, linear, angular)
    want = loop_histogram(states, weights, linear, angular, orc.spatial_hash)
    assert first.tolist() == [b[0] for b in want]
    assert count.tolist() == [b[1] for b in want]
    assert weight.tobytes() == np.array([b[2] for b in want]).tobytes()
    assert np.array_equal(first[bin_of], [first[b] for b in bin_of]) and np.array_equal(bin_of[first], np.arange(len(first)))
    assert count.sum() == len(states) and len(first) < len(base)


def test_histogram_of_unit_weights_counts():
    rng = np.random.default_rng(5)
    states = random_states(rng, 20000, 2.0)
    first, count, weight, _ = histogram(states, np.ones(len(states)), 0.2, 0.524)
    assert np.array_equal(weight, count.astype(np.float64)) and np.all(np.diff(first) > 0)
