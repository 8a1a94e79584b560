#!/usr/bin/env python
"""tools/bag_tool.py — a pure-Python ROS1 bag v2.0 reader / writer (struct + bz2 + an own LZ4 codec; no ROS).

Independent of csrc/host/rosbag_reader.hpp on purpose: the two implementations check each other in
tests/test_rosbag_cpu.py (Python writes -> C++ reads, C++ writes -> Python reads).

  python tools/bag_tool.py info X.bag               topics, types, counts, time span
  python tools/bag_tool.py decompress IN.bag OUT.bag   rewrite with uncompressed chunks (bz2 / lz4 chunks are inflated; the C++
                                                       reader handles "none" and "lz4" itself)
  python tools/bag_tool.py make-fixture OUT.bag     the small synthetic fixture committed as tests/golden/tiny.bag

Format: wiki.ros.org/Bags/Format/2.0 (records = <u32 hlen><header fields><u32 dlen><data>; field = <u32 len>name=value).
"""
import bz2
import struct
import sys

import numpy as np

MAGIC = b"#ROSBAG V2.0\n"
OP_MSG, OP_BAGHDR, OP_INDEX, OP_CHUNK, OP_CHUNKINFO, OP_CONN = 2, 3, 4, 5, 6, 7


# ---- LZ4 (the "lz4" chunk compression of rosbag = one LZ4 frame per chunk, written by ros_comm's roslz4) --------------------
# Public formats: LZ4 frame (magic 0x184D2204, FLG, BD, optional content size / dictionary id, header checksum, blocks
# <u32 size, bit 31 = stored raw>, end mark 0, optional content checksum) and LZ4 block (sequences: token = literal length
# << 4 | match length - 4, 15 = continued in following bytes; literals; u16 offset; match copied byte by byte, may overlap).
LZ4_MAGIC = 0x184D2204


def lz4_block_decompress(src, out):
    """appends the decoded block to bytearray `out` (earlier output stays addressable: linked blocks work too)"""
    i, n = 0, len(src)
    while i < n:
        tok = src[i]; i += 1
        ll = tok >> 4
        if ll == 15:
            while True:
                if i >= n:
                    raise ValueError("lz4: truncated literal length")
                b = src[i]; i += 1; ll += b
                if b != 255:
                    break
        if i + ll > n:
            raise ValueError("lz4: literals run past the block")
        out += src[i:i + ll]; i += ll
        if i >= n:
            break  # the last sequence of a block is literals only
        if i + 2 > n:
            raise ValueError("lz4: truncated offset")
        off = src[i] | (src[i + 1] << 8); i += 2
        if off == 0 or off > len(out):
            raise ValueError("lz4: offset outside the output")
        ml = tok & 15
        if ml == 15:
            while True:
                if i >= n:
                    raise ValueError("lz4: truncated match length")
                b = src[i]; i += 1; ml += b
                if b != 255:
                    break
        ml += 4
        start = len(out) - off
        if off >= ml:
            out += out[start:start + ml]
        else:  # overlapping match: the pattern of `off` bytes repeats
            pat = bytes(out[start:])
            out += (pat * (ml // off + 1))[:ml]


def lz4_frame_decompress(b, expected=None):
    if len(b) < 7 or struct.unpack_from("<I", b, 0)[0] != LZ4_MAGIC:
        raise ValueError("lz4: not an LZ4 frame")
    flg = b[4]
    if flg >> 6 != 1:
        raise ValueError("lz4: unsupported frame version")
    i = 6 + (8 if flg & 0x08 else 0) + (4 if flg & 0x01 else 0) + 1  # FLG, BD, [content size], [dict id], header checksum
    out = bytearray()
    while True:
        if i + 4 > len(b):
            raise ValueError("lz4: frame without end mark")
        (bs,) = struct.unpack_from("<I", b, i); i += 4
        if bs == 0:
            break
        raw, bs = bs >> 31, bs & 0x7FFFFFFF
        if i + bs > len(b):
            raise ValueError("lz4: truncated block")
        if raw:
            out += b[i:i + bs]
        else:
            lz4_block_decompress(b[i:i + bs], out)
        i += bs + (4 if flg & 0x10 else 0)
    if expected is not None and len(out) != expected:
        raise ValueError(f"lz4: chunk inflates to {len(out)} bytes, record says {expected}")
    return bytes(out)


def _xxh32(data, seed=0):
    """XXH32 (public algorithm) — the LZ4 frame header checksum is its second byte"""
    P1, P2, P3, P4, P5, M = 2654435761, 2246822519, 3266489917, 668265263, 374761393, 0xFFFFFFFF
    rotl = lambda x, r: ((x << r) | (x >> (32 - r))) & M
    n, i = len(data), 0
    if n >= 16:
        v = [(seed + P1 + P2) & M, (seed + P2) & M, seed & M, (seed - P1) & M]
        while i + 16 <= n:
            for k in range(4):
                v[k] = (rotl((v[k] + struct.unpack_from("<I", data, i + 4 * k)[0] * P2) & M, 13) * P1) & M
            i += 16
        h = (rotl(v[0], 1) + rotl(v[1], 7) + rotl(v[2], 12) + rotl(v[3], 18)) & M
    else:
        h = (seed + P5) & M
    h = (h + n) & M
    while i + 4 <= n:
        h = (rotl((h + struct.unpack_from("<I", data, i)[0] * P3) & M, 17) * P4) & M; i += 4
    while i < n:
        h = (rotl((h + data[i] * P5) & M, 11) * P1) & M; i += 1
    h ^= h >> 15; h = (h * P2) & M; h ^= h >> 13; h = (h * P3) & M; h ^= h >> 16
    return h


def lz4_block_compress(src):
    """greedy single-probe hash matcher (what the writer and the tests need; ratio is not the point).  Ends the block the
    way the format demands: the last 5 bytes are literals and no match starts within the last 12 bytes."""
    n, out, anchor, i, table = len(src), bytearray(), 0, 0, {}

    def emit(lit, ml, off):
        ll = len(lit)
        out.append((min(ll, 15) << 4) | (min(ml - 4, 15) if ml else 0))
        if ll >= 15:
            r = ll - 15
            while r >= 255:
                out.append(255); r -= 255
            out.append(r)
        out.extend(lit)
        if ml:
            out.extend(struct.pack("<H", off))
            if ml - 4 >= 15:
                r = ml - 4 - 15
                while r >= 255:
                    out.append(255); r -= 255
                out.append(r)

    while i + 12 < n:
        key = src[i:i + 4]
        j = table.get(key, -1)
        table[key] = i
        if j >= 0 and i - j <= 0xFFFF:
            ml = 4
            while i + ml < n - 5 and src[j + ml] == src[i + ml]:
                ml += 1
            emit(src[anchor:i], ml, i - j)
            i += ml; anchor = i
        else:
            i += 1
    emit(src[anchor:], 0, 0)
    return bytes(out)


def lz4_frame_compress(b, block_bytes=1 << 16):
    """an LZ4 frame like roslz4's: version 01, independent blocks, no checksums but the header's"""
    desc = bytes([(1 << 6) | (1 << 5), {1 << 16: 4, 1 << 18: 5, 1 << 20: 6, 1 << 22: 7}[block_bytes] << 4])
    out = bytearray(struct.pack("<I", LZ4_MAGIC) + desc + bytes([(_xxh32(desc) >> 8) & 0xFF]))
    for i in range(0, len(b), block_bytes):
        raw = b[i:i + block_bytes]
        c = lz4_block_compress(raw)
        if len(c) < len(raw):
            out += struct.pack("<I", len(c)) + c
        else:
            out += struct.pack("<I", len(raw) | 0x80000000) + raw
    return bytes(out + struct.pack("<I", 0))


def _fields(b):
    out, i = {}, 0
    while i < len(b):
        (n,) = struct.unpack_from("<I", b, i)
        f = b[i + 4 : i + 4 + n]
        k, v = f.split(b"=", 1)
        out[k.decode()] = v
        i += 4 + n
    return out


def _records(b, start=0):
    i = start
    while i + 8 <= len(b):
        (hl,) = struct.unpack_from("<I", b, i)
        h = b[i + 4 : i + 4 + hl]
        (dl,) = struct.unpack_from("<I", b, i + 4 + hl)
        d = b[i + 8 + hl : i + 8 + hl + dl]
        if len(h) < hl or len(d) < dl:
            return
        yield _fields(h), d
        i += 8 + hl + dl


def read_bag(path):
    """-> (connections {id: dict(topic, type, md5sum)}, messages [(conn_id, time, bytes)]) in file order."""
    b = open(path, "rb").read()
    assert b.startswith(MAGIC), "not a ROS bag v2.0"
    conns, msgs = {}, []

    def walk(recs):
        for h, d in recs:
            op = h["op"][0]
            if op == OP_CHUNK:
                comp = h.get("compression", b"none")
                if comp == b"bz2":
                    d = bz2.decompress(d)
                elif comp == b"lz4":
                    d = lz4_frame_decompress(d, struct.unpack("<I", h["size"])[0] if "size" in h else None)
                elif comp != b"none":
                    raise ValueError(f"unsupported chunk compression {comp!r}")
                walk(_records(d))
            elif op == OP_CONN:
                (cid,) = struct.unpack("<I", h["conn"])
                ch = _fields(d)
                conns[cid] = dict(topic=h["topic"].decode(), type=ch["type"].decode(), md5sum=ch["md5sum"].decode(),
                                  message_definition=ch.get("message_definition", b"").decode())
            elif op == OP_MSG:
                (cid,) = struct.unpack("<I", h["conn"])
                s, ns = struct.unpack("<II", h["time"])
                msgs.append((cid, s + 1e-9 * ns, d))

    walk(_records(b, len(MAGIC)))
    return conns, msgs


# ---- message (de)serialisation -------------------------------------------------------------------------------------------
def _hdr(seq, stamp, frame):
    s = int(stamp)
    ns = min(int(round((stamp - s) * 1e9)), 999999999)
    f = frame.encode()
    return struct.pack("<III", seq, s, ns) + struct.pack("<I", len(f)) + f


def _rd_hdr(b, i):
    seq, s, ns, n = struct.unpack_from("<IIII", b, i)
    return dict(seq=seq, stamp=s + 1e-9 * ns, frame_id=b[i + 16 : i + 16 + n].decode()), i + 16 + n


def encode_imu(seq, stamp, acc, gyr, frame="imu_link"):
    z9 = struct.pack("<9d", *([0.0] * 9))
    return _hdr(seq, stamp, frame) + struct.pack("<4d", 0, 0, 0, 1) + z9 + struct.pack("<3d", *gyr) + z9 + struct.pack("<3d", *acc) + z9


def decode_imu(b):
    h, i = _rd_hdr(b, 0)
    v = struct.unpack_from("<37d", b, i)
    return dict(header=h, orientation=v[0:4], angular_velocity=v[13:16], linear_acceleration=v[25:28])


VELODYNE_FIELDS = [("x", 0, 7, 1), ("y", 4, 7, 1), ("z", 8, 7, 1), ("intensity", 16, 7, 1), ("ring", 20, 4, 1)]  # the velodyne driver's PointXYZIR, 32-byte step


_NPT = {1: np.int8, 2: np.uint8, 3: np.int16, 4: np.uint16, 5: np.int32, 6: np.uint32, 7: np.float32, 8: np.float64}


def encode_pointcloud2(seq, stamp, xyz, intensity, ring=None, frame="velodyne", fields=VELODYNE_FIELDS, point_step=32, height=1,
                       row_pad=0, extra=None):
    """A sensor_msgs/PointCloud2 of len(xyz) points, row-major in `height` rows of row_step = width * point_step + row_pad
    bytes.  fields: (name, offset, datatype, count); x, y, z, intensity, ring and the columns of `extra` ({name: values})
    are written with numpy's casts to the field's datatype, any other field stays zero."""
    n = len(xyz)
    width = n // height if height else 0
    assert width * height == n
    row_step = width * point_step + row_pad
    buf = np.zeros((height, row_step), np.uint8)
    pts = buf[:, : width * point_step].reshape(height, width, point_step)
    cols = {"x": xyz[:, 0], "y": xyz[:, 1], "z": xyz[:, 2], "intensity": intensity, "ring": ring}
    cols.update(extra or {})
    out = _hdr(seq, stamp, frame) + struct.pack("<III", height, width, len(fields))
    for name, off, dt, cnt in fields:
        nb = name.encode()
        out += struct.pack("<I", len(nb)) + nb + struct.pack("<IBI", off, dt, cnt)
        if cols.get(name) is not None and n and dt in _NPT and off + np.dtype(_NPT[dt]).itemsize <= point_step:
            a = np.ascontiguousarray(np.asarray(cols[name]).astype(_NPT[dt]))
            pts[:, :, off : off + a.itemsize] = a.view(np.uint8).reshape(height, width, a.itemsize)
    data = buf.tobytes()
    return out + struct.pack("<BII", 0, point_step, row_step) + struct.pack("<I", len(data)) + data + struct.pack("<B", 1)


_TSIZE = {1: 1, 2: 1, 3: 2, 4: 2, 5: 4, 6: 4, 7: 4, 8: 8}


def index_pointcloud2(b):
    """What fromROSMsg<PointXYZI> reads of a sensor_msgs/PointCloud2 message, without decoding a point: dict(stamp, height,
    width, point_step, row_step, is_bigendian, offset (x, y, z, intensity), datatype (the same; intensity 0 = absent),
    data_start, data_len: the data field's byte range inside the message), or None where the C++ decode_pointcloud2
    (csrc/host/rosbag_reader.hpp) rejects the message.  Field names match as there (the last field of a name wins);
    extents are checked without 32-bit wrap-around."""
    try:
        seq, s, ns, fl = struct.unpack_from("<IIII", b, 0)
        i = 16 + fl
        height, width, nf = struct.unpack_from("<III", b, i)
        i += 12
        if nf > 64:
            return None
        found = {}
        for _ in range(nf):
            (nl,) = struct.unpack_from("<I", b, i)
            name = bytes(b[i + 4 : i + 4 + nl])
            if len(name) < nl:
                return None
            off, dt, cnt = struct.unpack_from("<IBI", b, i + 4 + nl)
            i += 4 + nl + 9
            if name in (b"x", b"y", b"z", b"intensity"):
                found[name.decode()] = (off, dt)
        big, step, row, dlen = struct.unpack_from("<BIII", b, i)
        i += 13
        if i + dlen + 1 > len(b):  # the data field and is_dense
            return None
    except struct.error:
        return None
    if big or not all(k in found for k in "xyz"):
        return None
    for off, dt in found.values():
        if dt < 1 or dt > 8 or off + _TSIZE[dt] > step:
            return None
    if width * height and (height - 1) * row + (width - 1) * step + step > dlen:
        return None
    names = ("x", "y", "z", "intensity")
    return dict(stamp=s + 1e-9 * ns, height=height, width=width, point_step=step, row_step=row, is_bigendian=big,
                offset=[found.get(k, (0, 0))[0] for k in names], datatype=[found.get(k, (0, 0))[1] for k in names],
                data_start=i, data_len=dlen)


def decode_pointcloud2(b):
    h, i = _rd_hdr(b, 0)
    height, width, nf = struct.unpack_from("<III", b, i)
    i += 12
    fields = []
    for _ in range(nf):
        (n,) = struct.unpack_from("<I", b, i)
        name = b[i + 4 : i + 4 + n].decode()
        off, dt, cnt = struct.unpack_from("<IBI", b, i + 4 + n)
        fields.append((name, off, dt, cnt))
        i += 4 + n + 9
    big, step, row = struct.unpack_from("<BII", b, i)
    i += 9
    (dl,) = struct.unpack_from("<I", b, i)
    data = np.frombuffer(b, np.uint8, dl, i + 4).reshape(height * width, step)
    npt = _NPT
    cols = {}
    for name, off, dt, cnt in fields:
        t = np.dtype(npt[dt])
        cols[name] = np.ascontiguousarray(data[:, off : off + t.itemsize]).view(t).reshape(-1)
    return dict(header=h, fields=fields, **cols)


def encode_cloud_info(seq, stamp, start, end, ori, ground, col, rng, frame="base_link"):
    def arr(a, t):
        a = np.ascontiguousarray(np.asarray(a).astype(t))
        return struct.pack("<I", len(a)) + a.tobytes()

    return (_hdr(seq, stamp, frame) + arr(start, np.int32) + arr(end, np.int32) + struct.pack("<3f", *ori) + arr(ground, np.uint8)
            + arr(col, np.uint32) + arr(rng, np.float32))


def decode_cloud_info(b):
    h, i = _rd_hdr(b, 0)

    def arr(t):
        nonlocal i
        (n,) = struct.unpack_from("<I", b, i)
        a = np.frombuffer(b, t, n, i + 4).copy()
        i += 4 + n * np.dtype(t).itemsize
        return a

    start, end = arr(np.int32), arr(np.int32)
    ori = struct.unpack_from("<3f", b, i)
    i += 12
    return dict(header=h, startRingIndex=start, endRingIndex=end, orientation=ori, ground=arr(np.uint8), col=arr(np.uint32), range=arr(np.float32))


# ---- writer ---------------------------------------------------------------------------------------------------------------
def _field(name, value):
    f = name.encode() + b"=" + value
    return struct.pack("<I", len(f)) + f


def _record(hfields, data):
    h = b"".join(_field(k, v) for k, v in hfields)
    return struct.pack("<I", len(h)) + h + struct.pack("<I", len(data)) + data


def _t(t):
    s = int(t)
    return struct.pack("<II", s, min(int(round((t - s) * 1e9)), 999999999))


def write_bag(path, connections, messages, compression="none", chunk_bytes=1 << 20, lz4_compress=None):
    """connections: [(topic, type, md5sum, definition)], messages: [(conn_index, time, bytes)] in recording order.
    lz4_compress: frame compressor to use instead of this module's (tests pass the system liblz4's)."""
    def conn_rec(i):
        topic, typ, md5, dfn = connections[i]
        d = _field("topic", topic.encode()) + _field("type", typ.encode()) + _field("md5sum", md5.encode()) + _field("message_definition", dfn.encode())
        return _record([("op", bytes([OP_CONN])), ("conn", struct.pack("<I", i)), ("topic", topic.encode())], d)

    body, chunk_infos = b"", []
    chunk, index, seen, t0, t1 = b"", {}, set(), None, None

    def flush():
        nonlocal body, chunk, index, seen, t0, t1
        if not chunk:
            return
        pos = len(MAGIC) + 4096 + len(body)
        data = bz2.compress(chunk) if compression == "bz2" else (lz4_compress or lz4_frame_compress)(chunk) if compression == "lz4" else chunk
        rec = _record([("op", bytes([OP_CHUNK])), ("compression", compression.encode()), ("size", struct.pack("<I", len(chunk)))], data)
        for cid, ents in index.items():
            rec += _record([("op", bytes([OP_INDEX])), ("ver", struct.pack("<I", 1)), ("conn", struct.pack("<I", cid)), ("count", struct.pack("<I", len(ents)))],
                           b"".join(_t(t) + struct.pack("<I", off) for t, off in ents))
        chunk_infos.append((pos, t0, t1, {cid: len(e) for cid, e in index.items()}))
        body += rec
        chunk, index, seen, t0, t1 = b"", {}, set(), None, None

    for cid, t, msg in messages:
        if cid not in seen:
            chunk += conn_rec(cid)
            seen.add(cid)
        index.setdefault(cid, []).append((t, len(chunk)))
        chunk += _record([("op", bytes([OP_MSG])), ("conn", struct.pack("<I", cid)), ("time", _t(t))], msg)
        t0 = t if t0 is None else min(t0, t)
        t1 = t if t1 is None else max(t1, t)
        if len(chunk) > chunk_bytes:
            flush()
    flush()
    index_pos = len(MAGIC) + 4096 + len(body)
    tail = b"".join(conn_rec(i) for i in range(len(connections)))
    for pos, a, b_, counts in chunk_infos:
        tail += _record([("op", bytes([OP_CHUNKINFO])), ("ver", struct.pack("<I", 1)), ("chunk_pos", struct.pack("<Q", pos)), ("start_time", _t(a)), ("end_time", _t(b_)),
                         ("count", struct.pack("<I", len(counts)))], b"".join(struct.pack("<II", c, n) for c, n in counts.items()))
    h = b"".join(_field(k, v) for k, v in [("op", bytes([OP_BAGHDR])), ("index_pos", struct.pack("<Q", index_pos)), ("conn_count", struct.pack("<I", len(connections))),
                                           ("chunk_count", struct.pack("<I", len(chunk_infos)))])
    hdr = struct.pack("<I", len(h)) + h
    pad = 4096 - len(hdr) - 4
    hdr += struct.pack("<I", pad) + b" " * pad
    with open(path, "wb") as f:
        f.write(MAGIC + hdr + body + tail)


# ---- the committed fixture ---------------------------------------------------------------------------------------------------
FIXTURE_TOPICS = dict(lidar="/velodyne_points", imu="/imu/data", info="/segmented_cloud_info")


def fixture_contents(seed=7, n_scans=3, cols=60):
    """Deterministic small drive: 16 rings x `cols` columns per scan (velodyne PointXYZIR layout), 10 IMU messages per scan,
    one cloud_info per scan.  Returns (connections, messages, truth) — truth holds the decoded arrays."""
    rng = np.random.default_rng(seed)
    conns = [(FIXTURE_TOPICS["lidar"], "sensor_msgs/PointCloud2", "1158d486dd51d683ce2f1be655c3c181", "(sensor_msgs/PointCloud2)"),
             (FIXTURE_TOPICS["imu"], "sensor_msgs/Imu", "6a62c6daae103f4ff57a132d6f95cec2", "(sensor_msgs/Imu)"),
             (FIXTURE_TOPICS["info"], "cloud_msgs/cloud_info", "00000000000000000000000000000000", "(cloud_msgs/cloud_info)")]
    msgs, truth = [], dict(clouds=[], imu=[], info=[])
    for k in range(n_scans):
        t = 1000.0 + 0.1 * k
        for j in range(10):
            ti = t + 0.01 * (j + 1)
            acc = rng.normal(0, 0.1, 3) + [0, 0, 9.81]
            gyr = rng.normal(0, 0.01, 3)
            msgs.append((1, ti, encode_imu(10 * k + j, ti, acc, gyr)))
            truth["imu"].append(np.r_[ti, acc, gyr])
        ring = np.repeat(np.arange(16), cols)
        az = np.tile(np.linspace(-np.pi, np.pi, cols, endpoint=False), 16)
        el = np.deg2rad(-15.0 + 2.0 * ring)
        r = rng.uniform(2.0, 40.0, len(ring))
        xyz = np.stack([r * np.cos(el) * np.cos(az), -r * np.cos(el) * np.sin(az), r * np.sin(el)], 1).astype(np.float32)
        inten = rng.uniform(0, 255, len(ring)).astype(np.float32)
        msgs.append((0, t + 0.1, encode_pointcloud2(k, t + 0.1, xyz, inten, ring)))
        truth["clouds"].append((t + 0.1, xyz, inten))
        n = 50 + 10 * k
        info = dict(start=np.arange(16) * 3 + k, end=np.arange(16) * 3 + 2, ori=(0.1 * k, 6.2 + 0.1 * k, 6.2), ground=(np.arange(n) % 2).astype(np.uint8),
                    col=(np.arange(n) * 7 % 1800).astype(np.uint32), rng=(1.0 + 0.25 * np.arange(n)).astype(np.float32))
        msgs.append((2, t + 0.1, encode_cloud_info(k, t + 0.1, info["start"], info["end"], info["ori"], info["ground"], info["col"], info["rng"])))
        truth["info"].append((t + 0.1, info))
    return conns, msgs, truth


def main(argv):
    if len(argv) >= 3 and argv[1] == "info":
        conns, msgs = read_bag(argv[2])
        for cid, c in sorted(conns.items()):
            ts = [t for i, t, _ in msgs if i == cid]
            print(f"{c['topic']:32s} {c['type']:28s} {len(ts):6d} msgs  {min(ts) if ts else 0:.6f} .. {max(ts) if ts else 0:.6f}")
    elif len(argv) >= 4 and argv[1] == "decompress":
        conns, msgs = read_bag(argv[2])
        ids = sorted(conns)
        write_bag(argv[3], [(conns[i]["topic"], conns[i]["type"], conns[i]["md5sum"], conns[i]["message_definition"]) for i in ids],
                  [(ids.index(i), t, d) for i, t, d in msgs])
    elif len(argv) >= 3 and argv[1] == "make-fixture":
        conns, msgs, _ = fixture_contents()
        write_bag(argv[2], conns, msgs)
    else:
        print(__doc__)
        return 2
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv))
