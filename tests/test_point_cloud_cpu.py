"""bb200_point_cloud_to_points, the host half of beluga_ros::Amcl::update(pose, SparsePointCloud3f)
(beluga_ros/src/amcl.cpp:67-81), against a numpy restatement of the reference arithmetic, bit for bit:

    SparsePointCloud3<float, false>::points() (beluga_ros/include/beluga_ros/sparse_point_cloud.hpp:102-125): point i is the three
    consecutive scalars at data + i * point_step + x_offset (PointCloud2ConstIterator + Eigen::Map); float64 clouds are cast to float;
    amcl.cpp:73-78: origin * p.cast<double>(), keep x and y.

Here the origin is a 3x4 row-major [R | t] and rows 0 and 1 of R p + t are summed left to right.  Also the rejections and the
synthetic lidar cloud."""
import ctypes as C
import math

import numpy as np
import pytest


@pytest.fixture(scope="module")
def bb():
    import beluga_b200 as bb
    from beluga_b200 import build as bb_build

    bb_build.build()
    return bb


def restated(raw: bytes, n: int, point_step: int, x_offset: int, datatype: int, origin) -> np.ndarray:
    scalar = np.dtype("<f4") if datatype == 7 else np.dtype("<f8")
    xyz = np.ndarray((n, 3), dtype=scalar, buffer=raw, offset=x_offset, strides=(point_step, scalar.itemsize)) if n else np.zeros((0, 3), scalar)
    p = xyz.astype(np.float32).astype(np.float64)  # SparsePointCloud3f narrows, amcl.cpp:74 widens
    if origin is None:
        return p[:, :2].copy()
    m = np.asarray(origin, dtype=np.float64).reshape(3, 4)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    return np.stack([((m[0, 0] * x + m[0, 1] * y) + m[0, 2] * z) + m[0, 3], ((m[1, 0] * x + m[1, 1] * y) + m[1, 2] * z) + m[1, 3]], axis=1)


def tilted_origin():
    """yaw 0.7 rad, roll 0.02, pitch -0.03, translation with z."""
    from beluga_b200 import synthetic

    return synthetic.sensor_origin(x=0.31, y=-0.17, z=1.25, roll=0.02, pitch=-0.03, yaw=0.7)


ORIGINS = {"none": lambda: None, "identity": lambda: np.concatenate([np.eye(3), np.zeros((3, 1))], axis=1), "tilted": tilted_origin}


def packed(points_xyz, scalar, x_offset: int, point_step: int) -> bytes:
    """Records of point_step bytes with x, y, z at x_offset and 0xAB filler elsewhere."""
    s = np.dtype(scalar).newbyteorder("<")
    buf = bytearray(b"\xab" * (len(points_xyz) * point_step))
    for i, p in enumerate(points_xyz):
        buf[i * point_step + x_offset:i * point_step + x_offset + 3 * s.itemsize] = np.asarray(p, dtype=s).tobytes()
    return bytes(buf)


@pytest.mark.parametrize("origin", list(ORIGINS))
@pytest.mark.parametrize("datatype", [7, 8])
def test_converter_matches_the_reference_arithmetic(bb, datatype, origin):
    o = ORIGINS[origin]()
    rng = np.random.default_rng(11 + datatype)
    n = 3001
    pts = np.concatenate([rng.uniform(-40.0, 40.0, (n - 5, 3)),
                          [[0.1, 0.2, 0.3], [1.0 / 3.0, -2.0 / 3.0, 1e-3], [123.456789012345, -98.7654321098765, 2.5], [1e6 + 0.1, -1e-7, 0.0], [0.0, -0.0, -0.0]]])
    scalar = np.float32 if datatype == 7 else np.float64
    for x_offset, point_step in ((0, 3 * np.dtype(scalar).itemsize), (5, 3 * np.dtype(scalar).itemsize + 11)):  # dense, and unaligned records
        raw = packed(pts, scalar, x_offset, point_step)
        got = bb.point_cloud_to_points(raw, point_step, x_offset, datatype, origin=o)
        assert got.shape == (n, 2)
        assert np.array_equal(got, restated(raw, n, point_step, x_offset, datatype, o))


def test_float64_clouds_are_narrowed_to_float_first(bb):
    """The node wraps every cloud as SparsePointCloud3f (beluga_amcl/src/amcl_node.cpp:553-576); its points() casts float64
    coordinates to float (sparse_point_cloud.hpp:111-116) before amcl.cpp:74 widens them again."""
    pts = np.array([[0.1, 1.0 / 3.0, 0.7], [123.456789012345, 2.0 ** -30 + 1.0, 5.0]])
    got = bb.point_cloud_to_points(pts, 24, 0, 8)
    assert np.array_equal(got, pts[:, :2].astype(np.float32).astype(np.float64))
    assert not np.any(got == pts[:, :2])  # every one of these values changes when narrowed
    same_as_float32 = bb.point_cloud_to_points(pts.astype(np.float32), 12, 0, 7)
    assert np.array_equal(got, same_as_float32)


# Records of beluga_ros/test/include/beluga_ros/test/point_cloud_utils.hpp (addPointField packs the fields without padding):
#   Velodyne  (:257-268)  x y z intensity FLOAT32 at 0 4 8 12, ring UINT16 at 16, time FLOAT32 at 18: point_step 22
#   Robosense (:299-310)  x y z intensity FLOAT32 at 0 4 8 12, ring UINT16 at 16, time FLOAT64 at 18: point_step 26
#   Ouster    (:341-356)  x y z FLOAT32 at 0 4 8, 4 bytes skipped, intensity FLOAT32 at 16, t UINT32 at 20, reflectivity UINT16 at 24,
#                         ring UINT8 at 26, ambient UINT16 at 27, range UINT32 at 29: point_step 33
# filled as make_point_data (:35-44): point i = (i, 2i, 3i), and the constant extra fields of those helpers.
LAYOUTS = {
    "velodyne": (["x", "y", "z", "intensity", "ring", "time"], ["<f4", "<f4", "<f4", "<f4", "<u2", "<f4"], [0, 4, 8, 12, 16, 18], 22,
                 {"intensity": 1.1, "ring": 1, "time": 0.1}),
    "robosense": (["x", "y", "z", "intensity", "ring", "time"], ["<f4", "<f4", "<f4", "<f4", "<u2", "<f8"], [0, 4, 8, 12, 16, 18], 26,
                  {"intensity": 1.1, "ring": 1, "time": 0.1}),
    "ouster": (["x", "y", "z", "intensity", "t", "reflectivity", "ring", "ambient", "range"],
               ["<f4", "<f4", "<f4", "<f4", "<u4", "<u2", "u1", "<u2", "<u4"], [0, 4, 8, 16, 20, 24, 26, 27, 29], 33,
               {"intensity": 1.1, "t": 1, "reflectivity": 10, "ring": 11, "ambient": 20, "range": 21}),
}


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_reference_sensor_layouts(bb, layout):
    """VelodyneLayout, RobosenseLayout, OusterLayout (beluga_ros/test/test_sparse_point_cloud.cpp:192-223): five points
    (kUnorderedWidth, :44), read back in order; then the same records through a tilted origin."""
    names, formats, offsets, step, extra = LAYOUTS[layout]
    rec = np.zeros(5, dtype=np.dtype({"names": names, "formats": formats, "offsets": offsets, "itemsize": step}))
    i = np.arange(5)
    rec["x"], rec["y"], rec["z"] = i, 2 * i, 3 * i
    for k, v in extra.items():
        rec[k] = v
    got = bb.point_cloud_to_points(rec, step, 0, np.float32)
    assert np.array_equal(got, np.stack([i, 2 * i], axis=1).astype(np.float64))
    o = tilted_origin()
    assert np.array_equal(bb.point_cloud_to_points(rec.tobytes(), step, 0, 7, origin=o), restated(rec.tobytes(), 5, step, 0, 7, o))


def test_empty_cloud(bb):
    for data in (b"", np.zeros(0, dtype=np.float32)):
        got = bb.point_cloud_to_points(data, 12, 0, 7, origin=tilted_origin())
        assert got.shape == (0, 2)


def test_nan_points_stay_in_place(bb):
    """The reference does not filter (sparse_point_cloud.hpp:102-125): NaN points reach the sensor model, which reads them as
    out of the grid (INTEGRATION.md)."""
    pts = np.array([[1.0, 2.0, 0.5], [np.nan, 1.0, 0.0], [3.0, np.nan, 0.0], [4.0, 5.0, np.nan], [6.0, 7.0, 0.25]], dtype=np.float32)
    plain = bb.point_cloud_to_points(pts, 12, 0, 7)
    assert plain.shape == (5, 2)
    assert np.array_equal(plain, pts[:, :2].astype(np.float64), equal_nan=True)  # z does not touch (x, y) without an origin
    o = tilted_origin()
    moved = bb.point_cloud_to_points(pts, 12, 0, 7, origin=o)
    assert np.array_equal(moved, restated(pts.tobytes(), 5, 12, 0, 7, o), equal_nan=True)
    assert np.isnan(moved[1:4]).all() and not np.isnan(moved[[0, 4]]).any()  # a NaN coordinate reaches both rows of R p + t


def call_raw(lib, data, n_points, point_step, x_offset, datatype, capacity=64):
    from beluga_b200 import _capi

    cloud = _capi.PointCloud(data, n_points, point_step, x_offset, datatype, None)
    out = np.full((max(capacity, 1), 2), -7.0)
    n = C.c_uint64(12345)
    st = lib.bb200_point_cloud_to_points(C.byref(cloud), out.ctypes.data_as(C.POINTER(C.c_double)), capacity, C.byref(n))
    return st, out, n.value


@pytest.mark.parametrize("case, status", [
    ("datatype_int32", -1), ("datatype_zero", -1), ("datatype_9", -1), ("float32_overruns_record", -1), ("float64_overruns_record", -1),
    ("offset_wraps", -1), ("null_data", -1), ("too_many_points", -5)])
def test_rejections_write_nothing(bb, case, status):
    from beluga_b200 import _capi

    lib = _capi.load()
    buf = np.arange(5 * 32, dtype=np.uint8)
    data = buf.ctypes.data
    args = dict(data=data, n_points=5, point_step=32, x_offset=0, datatype=7)
    args.update({
        "datatype_int32": dict(datatype=5), "datatype_zero": dict(datatype=0), "datatype_9": dict(datatype=9),
        "float32_overruns_record": dict(point_step=12, x_offset=1),  # 1 + 3 * 4 > 12
        "float64_overruns_record": dict(point_step=20, x_offset=0, datatype=8),  # 3 * 8 > 20
        "offset_wraps": dict(x_offset=0xFFFFFFFF),
        "null_data": dict(data=None),
        "too_many_points": dict(),
    }[case])
    st, out, n = call_raw(lib, capacity=4 if case == "too_many_points" else 64, **args)
    assert st == status
    assert np.all(out == -7.0) and n == 12345
    # the boundary cases that are accepted
    assert call_raw(lib, data, 5, 12, 0, 7)[0] == 0  # x, y, z fill the record exactly
    assert call_raw(lib, data, 5, 32, 8, 8)[0] == 0
    assert call_raw(lib, None, 0, 12, 0, 7)[0] == 0  # an empty cloud needs no buffer
    assert call_raw(lib, data, 4, 32, 0, 7, capacity=4)[0] == 0


def test_null_arguments(bb):
    from beluga_b200 import _capi

    lib = _capi.load()
    cloud = _capi.PointCloud(None, 0, 12, 0, 7, None)
    n = C.c_uint64()
    assert lib.bb200_point_cloud_to_points(None, None, 0, C.byref(n)) == -1
    assert lib.bb200_point_cloud_to_points(C.byref(cloud), None, 0, None) == -1
    assert lib.bb200_point_cloud_to_points(C.byref(cloud), None, 0, C.byref(n)) == 0 and n.value == 0
    pose = np.array([1.0, 0.0, 0.0, 0.0])
    res = _capi.UpdateResult()
    assert lib.bb200_amcl_update_point_cloud(None, pose.ctypes.data_as(C.POINTER(C.c_double)), C.byref(cloud), C.byref(res)) == -1


def test_python_view_checks_the_buffer_size(bb):
    with pytest.raises(ValueError):
        bb.point_cloud_to_points(np.zeros(6, dtype=np.float32), 12, 0, 7, n_points=3)
    with pytest.raises(bb.BelugaB200Error) as e:
        bb.point_cloud_to_points(np.zeros(6, dtype=np.int32), 12, 0, np.int32)  # not a coordinate type
    assert e.value.status == -1


# ---- the synthetic lidar cloud --------------------------------------------------------------------------
def test_synthetic_cloud_lands_on_the_map(bb):
    from beluga_b200 import synthetic

    sc = synthetic.make_scenario(grid_size=200, n_beams=181, steps=12)
    pc = synthetic.make_point_cloud(sc, 4, rows=8, azimuths=512)
    assert (pc.point_step, pc.x_offset, pc.datatype, pc.width, pc.height) == (22, 0, 7, 512, 8)
    assert pc.data.dtype.names == synthetic.LIDAR_FIELDS and pc.data.shape == (8 * 512,)
    again = synthetic.make_point_cloud(sc, 4, rows=8, azimuths=512)
    assert pc.data.tobytes() == again.data.tobytes()  # seeded
    ring = pc.data["ring"].reshape(8, 512)
    assert np.array_equal(ring, np.repeat(np.arange(8, dtype=np.uint16)[:, None], 512, axis=1))
    pts = bb.point_cloud_to_points(pc.data, pc.point_step, pc.x_offset, pc.datatype, pc.origin)
    # base-frame z of each ring differs (the sensor is tilted, so compute it with the third row of [R | t])
    xyz = np.stack([pc.data["x"], pc.data["y"], pc.data["z"]], axis=1).astype(np.float64)
    z = (xyz @ pc.origin[2, :3] + pc.origin[2, 3]).reshape(8, 512)
    assert np.all(np.diff(z.mean(axis=1)) > 0.0)
    # the end points, seen from the true pose, hit occupied cells (up to the 2 cm range noise)
    x, y, th = sc.poses[4]
    world = np.stack([x + math.cos(th) * pts[:, 0] - math.sin(th) * pts[:, 1], y + math.sin(th) * pts[:, 0] + math.cos(th) * pts[:, 1]], axis=1)
    cell = np.floor(world / sc.resolution).astype(int)
    near = [sc.cells[max(j - 1, 0):j + 2, max(i - 1, 0):i + 2].any() for i, j in np.clip(cell, 0, 199)]
    assert np.mean(near) > 0.99
    wide = synthetic.make_point_cloud(sc, 4, rows=2, azimuths=16, coordinate_type=np.float64)
    assert (wide.point_step, wide.datatype) == (34, 8)
