"""Where a double becomes an integer: the spatial hash's floor to int64 (se2_math.cuh floor_to_int64, the reference's
algorithm/spatial_hash.hpp:45-75) and the oracle's restatement of it, at the edges of the double range.

The reference casts floor(v) to int64; for NaN, +-inf and values outside [-2^63, 2^63) that cast is undefined, and x86-64
returns INT64_MIN.  The project states that result as its rule, on the host and on the device alike.  The model below is
written with Python's unbounded integers, and the header (compiled for the host by tests/cpp/schedule_probe.cu) and the
oracle are both checked against it."""
import math
import struct

import numpy as np
import pytest

from test_models_against_headers import probe_lines  # noqa: F401  (the compiled probe, a fixture)

INT64_MIN = -(2**63)
MASK = 2**64 - 1
FIB = 11400714819323198485


def from_bits(hex_bits):
    return struct.unpack("<d", int(hex_bits, 16).to_bytes(8, "little"))[0]


def floor_to_int64(v):
    """floor(v) as an int64, INT64_MIN when floor(v) is NaN or outside [-2^63, 2^63)."""
    if math.isnan(v) or math.isinf(v):
        return INT64_MIN
    f = math.floor(v)  # exact: a Python int
    return f if INT64_MIN <= f < 2**63 else INT64_MIN


def fibo_hash(v, shift):
    h = (FIB * (floor_to_int64(v) & MASK)) & MASK
    return ((h << shift) | (h >> (64 - shift))) & MASK if shift else h


def spatial_hash(state, rx, ry, rtheta):
    c, s, x, y = (float(t) for t in state)
    return fibo_hash(x / rx, 0) ^ fibo_hash(y / ry, 21) ^ fibo_hash(math.atan2(s, c) / rtheta, 42)


def edge_poses(v):
    """The poses tests/cpp/schedule_probe.cu builds from one edge value: v as x, as y, as the heading's cosine, and as its
    sine with the cosine -1 (heading +-pi for s = +-0) and 1."""
    return [(1.0, 0.0, v, 0.25), (1.0, 0.0, 0.25, v), (v, 0.0, 0.25, 0.25), (-1.0, v, 0.25, 0.25), (1.0, v, 0.25, 0.25)]


N_EDGES = 36  # values in tests/cpp/schedule_probe.cu's edge list
RESOLUTIONS = [(1.0, 1.0, 0.1), (0.5, 0.5, 0.17453292519943295), (0.5, 0.5, 5e-324)]


def test_the_model_follows_x86_64_at_the_edges():
    """The rule's fixed points, stated once more by hand."""
    assert floor_to_int64(-0.0) == 0 and floor_to_int64(5e-324) == 0 and floor_to_int64(-5e-324) == -1
    assert floor_to_int64(np.nextafter(1.0, 0.0)) == 0 and floor_to_int64(1.0) == 1
    assert floor_to_int64(-1.0) == -1 and floor_to_int64(np.nextafter(-1.0, 0.0)) == -1 and floor_to_int64(np.nextafter(-1.0, -2.0)) == -2
    assert floor_to_int64(2.0**53) == 2**53 and floor_to_int64(2.0**63 - 1024) == 2**63 - 1024
    assert floor_to_int64(-(2.0**63)) == INT64_MIN  # in range: the cast is exact
    for v in (2.0**63, np.nextafter(-(2.0**63), -math.inf), 1e300, -1e300, math.inf, -math.inf, math.nan):
        assert floor_to_int64(v) == INT64_MIN
    # consequences the device's saturating conversion would break: far ends of the line share one bucket, and NaN does
    # not share bucket 0 with a particle in [0, 1)
    assert fibo_hash(1e300, 0) == fibo_hash(-1e300, 0) == fibo_hash(math.nan, 0)
    assert fibo_hash(math.nan, 0) != fibo_hash(0.5, 0)


def test_header_floor_and_hash_match_the_model(probe_lines):  # noqa: F811
    rows = [line.split()[1:] for line in probe_lines if line.startswith("floor ")]
    assert len(rows) == N_EDGES  # keep in step with tests/cpp/schedule_probe.cu
    for bits, f, h0, h21 in rows:
        v = from_bits(bits)
        assert int(f) == floor_to_int64(v), bits
        assert int(h0) == fibo_hash(v, 0) and int(h21) == fibo_hash(v, 21), bits


def test_header_spatial_hash_matches_the_model_and_the_oracle(probe_lines, orc):  # noqa: F811
    rows = [line.split()[1:] for line in probe_lines if line.startswith("pose ")]
    assert len(rows) == 5 * N_EDGES
    by_value = {}
    for r in rows:
        by_value.setdefault(r[0], []).append([int(h) for h in r[5:8]])
    for bits, hashes in by_value.items():
        v = from_bits(bits)
        for pose, got in zip(edge_poses(v), hashes):
            state = np.array(pose)
            for (rx, ry, rt), h in zip(RESOLUTIONS, got):
                want = spatial_hash(state, rx, ry, rt)
                assert h == want, (bits, pose, rx, rt)
                assert orc.spatial_hash(state, rx, ry, rt) == want, (bits, pose, rx, rt)


@pytest.mark.parametrize("sign", [1.0, -1.0])
def test_oracle_hash_at_bucket_edges(orc, sign):
    """Exact bucket edges k * r and one ulp either side, negative fractions, and the heading's +-pi with s = +-0, at a
    resolution whose quotients round (0.1)."""
    rng = np.random.default_rng(7 if sign > 0 else 8)
    ks = np.concatenate([np.arange(-4, 5), rng.integers(-(2**40), 2**40, 16)]).astype(np.float64)
    for r in (1.0, 0.5, 0.1, 0.05):
        for k in ks:
            for x in (k * r, np.nextafter(k * r, math.inf), np.nextafter(k * r, -math.inf)):
                state = np.array([1.0, 0.0, sign * x, -sign * x])
                assert orc.spatial_hash(state, r, r, r) == spatial_hash(state, r, r, r)
    for c, s in ((-1.0, 0.0), (-1.0, -0.0), (-0.0, 0.0), (0.0, -0.0), (np.nextafter(-1.0, 0.0), 5e-324)):
        state = np.array([c, s, sign * 0.5, sign * -0.5])
        for rt in (0.1, 0.17453292519943295, math.pi, math.pi / 2, 5e-324):
            assert orc.spatial_hash(state, 1.0, 1.0, rt) == spatial_hash(state, 1.0, 1.0, rt)
