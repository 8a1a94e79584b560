"""sensor_msgs/PointCloud2 messages for the PointCloud2 decoding tests — TEST INFRASTRUCTURE.

LAYOUTS are the field layouts drivers publish and the edges of fromROSMsg<PointXYZI>: the Velodyne driver's 32-B
PointXYZIR, a 22-B step with ring and time (every other point's floats 2-byte aligned), FLOAT64 x, y, z, no intensity,
intensity as UINT16 or UINT8 at offset 0 (x at offset 1), every integer datatype, and an organised cloud (height > 1)
with row_step padding.  MALFORMED are messages the host decoder rejects.  The host references are tools/synth/lins_bag.cpp's
lins_bag_index_cloud2_msg and lins_bag_decode_cloud2_msg (csrc/host/rosbag_reader.hpp decode_pointcloud2).
"""
import ctypes as C
import os
import struct
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bag_tool  # noqa: E402

F32, F64, U16, U8, I8, I16, I32, U32 = 7, 8, 4, 2, 1, 3, 5, 6
# name: (fields (name, offset, datatype, count), point_step, height)
LAYOUTS = {
    "velodyne32": (bag_tool.VELODYNE_FIELDS, 32, 1),
    "ring_time22": ([("x", 0, F32, 1), ("y", 4, F32, 1), ("z", 8, F32, 1), ("intensity", 12, F32, 1), ("ring", 16, U16, 1),
                     ("time", 18, F32, 1)], 22, 1),
    "f64_48": ([("x", 0, F64, 1), ("y", 8, F64, 1), ("z", 16, F64, 1), ("intensity", 24, F32, 1), ("ring", 28, U16, 1)], 48, 1),
    "no_intensity": ([("x", 0, F32, 1), ("y", 4, F32, 1), ("z", 8, F32, 1)], 12, 1),
    "intensity_u16": ([("x", 0, F32, 1), ("y", 4, F32, 1), ("z", 8, F32, 1), ("intensity", 12, U16, 1), ("ring", 14, U8, 1)], 15, 1),
    "intensity_u8_first": ([("intensity", 0, U8, 1), ("x", 1, F32, 1), ("y", 5, F32, 1), ("z", 9, F32, 1)], 13, 1),
    "integers": ([("x", 0, I32, 1), ("y", 4, I16, 1), ("z", 6, U32, 1), ("intensity", 10, I8, 1)], 11, 1),
    "organised": (bag_tool.VELODYNE_FIELDS, 32, 4),
}
ROW_PAD = {"organised": 6}


def sweep(rng, n):
    """n points (x, y, z, intensity) in float64 (the encoder casts them per field), a few NaN no-returns."""
    a = np.empty((n, 4))
    a[:, :3] = rng.standard_normal((n, 3)) * 20.0
    a[:, 3] = rng.uniform(0, 200, n)
    if n > 8:
        a[rng.choice(n, n // 8, replace=False), :3] = np.nan
    return a


def message(name, pts, seq=0, stamp=100.0):
    """(PointCloud2 bytes of pts in layout `name`, its ring column)."""
    fields, step, height = LAYOUTS[name]
    pts = np.array(pts, np.float64)
    types = dict((f[0], f[2]) for f in fields)
    if any(types.get(k) not in (F32, F64) for k in "xyz"):  # (integer fields: finite values, scaled)
        pts[:, :3] = np.nan_to_num(pts[:, :3]) * 1000.0
    n = len(pts)
    ring = np.arange(n) % 16
    msg = bag_tool.encode_pointcloud2(seq, stamp, pts[:, :3], pts[:, 3], ring=ring, fields=fields, point_step=step,
                                      height=height if n else 1, row_pad=ROW_PAD.get(name, 0), extra={"time": np.arange(n) * 1e-5})
    return msg, ring


def baglib():
    L = C.CDLL(os.path.join(ROOT, "tools", "synth", "liblins_bag.so"))
    vp = C.c_void_p
    L.lins_bag_index_cloud2_msg.argtypes = [C.c_char_p, C.c_size_t, vp, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_double)]
    L.lins_bag_decode_cloud2_msg.argtypes = [C.c_char_p, C.c_size_t, vp, C.c_int, C.POINTER(C.c_int)]
    return L


def index_cpp(L, msg):
    """lins_bag_index_cloud2_msg as bag_tool.index_pointcloud2's dict, or None."""
    lay = (C.c_uint8 * 40)()
    ds, dl, st = C.c_int64(), C.c_int64(), C.c_double()
    if L.lins_bag_index_cloud2_msg(msg, len(msg), lay, C.byref(ds), C.byref(dl), C.byref(st)) != 0:
        return None
    b = bytes(lay)
    h, w, step, row = struct.unpack_from("<4I", b, 0)
    off = list(struct.unpack_from("<4I", b, 16))
    return dict(stamp=st.value, height=h, width=w, point_step=step, row_step=row, is_bigendian=b[36], offset=off, datatype=list(b[32:36]),
                data_start=ds.value, data_len=dl.value)


def decode_cpp(L, msg):
    """decode_pointcloud2 of one message: (n, 8) float32 lins_point records, or None where it rejects the message."""
    n = C.c_int(0)
    if L.lins_bag_decode_cloud2_msg(msg, len(msg), None, 0, C.byref(n)) != 0:
        return None
    out = np.zeros((max(n.value, 1), 8), np.float32)
    assert L.lins_bag_decode_cloud2_msg(msg, len(msg), out.ctypes.data, n.value, C.byref(n)) == 0
    return out[: n.value]


def layout_of(defs, ix):
    """LinsCloud2Layout of an index dict."""
    lay = defs.LinsCloud2Layout()
    lay.height, lay.width, lay.point_step, lay.row_step, lay.is_bigendian = ix["height"], ix["width"], ix["point_step"], ix["row_step"], ix["is_bigendian"]
    for k in range(4):
        lay.offset[k], lay.datatype[k] = ix["offset"][k], ix["datatype"][k]
    return lay


def as_input(defs, msg):
    """(layout, data field bytes) of a valid message: what LinsGpu.cloud2_desc takes."""
    ix = bag_tool.index_pointcloud2(msg)
    assert ix is not None
    return layout_of(defs, ix), msg[ix["data_start"]: ix["data_start"] + ix["data_len"]]


def host_decode(lay, data):
    """(x, y, z, intensity) float32 of a layout and its data field in numpy: each field read, then (float) of the
    double, as read_scalar + (float) in decode_pointcloud2."""
    h, w, ps, rs = int(lay.height), int(lay.width), int(lay.point_step), int(lay.row_step)
    out = np.zeros((h * w, 4), np.float32)
    at = (np.arange(h)[:, None] * rs + np.arange(w)[None, :] * ps).reshape(-1)
    for k in range(4):
        if lay.datatype[k]:
            t = np.dtype(bag_tool._NPT[lay.datatype[k]]).newbyteorder("<")
            b = np.asarray(data)[at[:, None] + int(lay.offset[k]) + np.arange(t.itemsize)]
            out[:, k] = np.ascontiguousarray(b).view(t).reshape(-1).astype(np.float64).astype(np.float32)
    return out


def edge_vectors():
    """(datatype, 8 little-endian bytes) records covering each datatype's edges."""
    recs = []

    def add(dt, values, np_t):
        for v in np.asarray(values).astype(np_t):
            b = np.asarray(v, np_t).tobytes()
            recs.append(bytes([dt]) + b + bytes(8 - len(b)))

    i8, i16, i32 = np.iinfo(np.int8), np.iinfo(np.int16), np.iinfo(np.int32)
    add(1, [i8.min, -1, 0, 1, i8.max], np.int8)
    add(2, [0, 1, 127, 128, 255], np.uint8)
    add(3, [i16.min, -1, 0, 1, i16.max], np.int16)
    add(4, [0, 1, 2 ** 15, 65535], np.uint16)
    big = [2 ** 24, 2 ** 24 + 1, 2 ** 24 + 3, 2 ** 25 + 2, 2 ** 25 + 6, 2 ** 31 - 1, 123456789, 2 ** 31 - 65, 2 ** 31 - 64]
    add(5, [i32.min, i32.min + 1, -1, 0, 1, i32.max] + big + [-v for v in big[:-3]], np.int32)
    add(6, [0, 1, 2 ** 32 - 1, 2 ** 31, 2 ** 32 - 129, 2 ** 32 - 128, 2 ** 32 - 127] + big + [3000000001, 4000000003], np.uint32)
    f32 = [0.0, -0.0, 1.0, -1.5, np.inf, -np.inf, np.nan, 1e-45, -1e-45, 1.17549421e-38, 1.17549435e-38, 3.4028235e38, 0.1]
    add(7, f32, np.float32)
    recs.append(bytes([7]) + struct.pack("<I", 0x7FA00001) + bytes(4))  # a signalling NaN
    recs.append(bytes([7]) + struct.pack("<I", 0xFFC12345) + bytes(4))  # a negative NaN with payload
    one = 1.0
    ulp = np.spacing(np.float32(one)).astype(np.float64)
    f64 = [0.0, -0.0, 1.0, 0.1, -0.1, np.pi, np.inf, -np.inf, np.nan, 5e-324, -5e-324, 2.2250738585072014e-308,
           one + ulp / 2, one + 3 * ulp / 2, one + ulp / 2 + 1e-16, one + ulp / 2 - 1e-16,  # halfway cases, both sides
           3.4028235677973366e38, 3.4028235677973366e38 * (1 + 2 ** -25), 3.4028235677973366e38 * (1 + 2 ** -23), 1e39, -1e300,
           1.4e-45, 7e-46, 7.006492321624086e-46, 1e-46, 1.1754942e-38, 2.0 ** -149 * 1.5, 2.0 ** -149 * 2.5, 1e-300]
    add(8, f64, np.float64)
    rng = np.random.default_rng(5)
    add(8, rng.standard_normal(200) * 10.0 ** rng.integers(-40, 40, 200), np.float64)
    add(5, rng.integers(i32.min, i32.max, 200), np.int32)
    add(6, rng.integers(0, 2 ** 32 - 1, 200, dtype=np.uint64), np.uint32)
    for dt in (0, 9, 200):  # not a datatype: 0 on both sides
        recs.append(bytes([dt]) + bytes(range(1, 9)))
    return recs


def edge_messages():
    """One PointCloud2 per datatype 1..8 whose x, y, z and intensity all have that datatype, at offsets 1, 1 + s, ...
    of an odd point_step (every field misaligned somewhere), the datatype's edge_vectors() rotated through the four fields:
    the device conversion meets the edges the host conversion is checked on."""
    by_dt = {}
    for r in edge_vectors():
        if 1 <= r[0] <= 8:
            by_dt.setdefault(r[0], []).append(r[1:])
    msgs = []
    for dt, vals in sorted(by_dt.items()):
        size = bag_tool._TSIZE[dt]
        step = 1 + 4 * size + 2
        n = len(vals)
        data = bytearray(n * step)
        for i in range(n):
            for k in range(4):
                o = i * step + 1 + k * size
                data[o: o + size] = vals[(i + k) % n][:size]
        out = bag_tool._hdr(dt, 1.0, "edges") + struct.pack("<III", 1, n, 4)
        for k, name in enumerate(("x", "y", "z", "intensity")):
            out += struct.pack("<I", len(name)) + name.encode() + struct.pack("<IBI", 1 + k * size, dt, 1)
        msgs.append(out + struct.pack("<BII", 0, step, step * n) + struct.pack("<I", len(data)) + bytes(data) + struct.pack("<B", 1))
    return msgs


def _patch(msg, pos, fmt, v):
    b = bytearray(msg)
    struct.pack_into(fmt, b, pos, v)
    return bytes(b)


def _fields_msg(fields, step=32, n=10):
    rng = np.random.default_rng(1)
    p = rng.standard_normal((n, 4))
    return bag_tool.encode_pointcloud2(0, 1.0, p[:, :3], p[:, 3], fields=fields, point_step=step)


MALFORMED = ["bigendian", "no_x", "no_z", "x_datatype_0", "datatype_9", "intensity_datatype_0", "field_past_step", "f64_past_step",
             "row_step_past_data", "point_step_past_data", "truncated", "too_many_fields"]


def malformed(case):
    good, _ = message("velodyne32", sweep(np.random.default_rng(2), 20))
    ds = bag_tool.index_pointcloud2(good)["data_start"]  # big-endian flag, point_step, row_step, data length: ds - 13 .. ds
    v = [("x", 0, F32, 1), ("y", 4, F32, 1), ("z", 8, F32, 1), ("intensity", 16, F32, 1)]
    if case == "bigendian":
        return _patch(good, ds - 13, "<B", 1)
    if case == "no_x":
        return _fields_msg(v[1:])
    if case == "no_z":
        return _fields_msg([v[0], v[1], v[3]])
    if case == "x_datatype_0":
        return _fields_msg([("x", 0, 0, 1)] + v[1:])
    if case == "datatype_9":
        return _fields_msg([v[0], ("y", 4, 9, 1)] + v[2:])
    if case == "intensity_datatype_0":
        return _fields_msg(v[:3] + [("intensity", 16, 0, 1)])
    if case == "field_past_step":
        return _fields_msg(v[:3] + [("intensity", 30, F32, 1)])
    if case == "f64_past_step":
        return _fields_msg([("x", 28, F64, 1)] + v[1:])
    if case == "row_step_past_data":
        msg, _ = message("organised", sweep(np.random.default_rng(3), 16))
        d = bag_tool.index_pointcloud2(msg)["data_start"]
        return _patch(msg, d - 8, "<I", 4 * 32 + 6 + 100)
    if case == "point_step_past_data":
        return _patch(good, ds - 12, "<I", 33)
    if case == "truncated":
        return good[: ds + 32 * 20 - 5]
    if case == "too_many_fields":
        i = 16 + len("velodyne")
        return _patch(good, i + 8, "<I", 65)
    raise KeyError(case)
