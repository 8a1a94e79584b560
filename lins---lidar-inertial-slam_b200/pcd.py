"""Binary PCD v0.7 files of x, y, z, intensity clouds (the layout pcl::io::savePCDFileBinary writes for PointXYZI
without its padding): the global maps tools/run_bag.py and tools/run_bags.py write with --global-map."""
import numpy as np

FIELDS = ("x", "y", "z", "intensity")


def write_pcd(path, cloud):
    """cloud: (n, 4) float32 x, y, z, intensity -> a binary PCD v0.7 file (an unorganised cloud: WIDTH n, HEIGHT 1)."""
    a = np.ascontiguousarray(cloud, "<f4").reshape(-1, 4)
    n = len(a)
    head = ("# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\nFIELDS x y z intensity\nSIZE 4 4 4 4\nTYPE F F F F\n"
            f"COUNT 1 1 1 1\nWIDTH {n}\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS {n}\nDATA binary\n")
    with open(path, "wb") as f:
        f.write(head.encode("ascii"))
        f.write(a.tobytes())


def read_pcd(path):
    """(header dict of str -> list of str, (n, 4) float32) of a binary PCD file write_pcd wrote; ValueError for any other
    layout."""
    with open(path, "rb") as f:
        data = f.read()
    head, pos = {}, 0
    while True:
        end = data.index(b"\n", pos)
        line = data[pos:end].decode("ascii").strip()
        pos = end + 1
        if not line or line.startswith("#"):
            continue
        key, *vals = line.split()
        head[key] = vals
        if key == "DATA":
            break
    want = dict(FIELDS=list(FIELDS), SIZE=["4"] * 4, TYPE=["F"] * 4, COUNT=["1"] * 4, DATA=["binary"])
    for k, v in want.items():
        if head.get(k) != v:
            raise ValueError(f"{path}: {k} {head.get(k)} (this reader takes binary x y z intensity F32 only)")
    n = int(head["POINTS"][0])
    if int(head["WIDTH"][0]) * int(head["HEIGHT"][0]) != n or len(data) - pos != 16 * n:
        raise ValueError(f"{path}: {n} points do not match WIDTH x HEIGHT or the data's {len(data) - pos} bytes")
    return head, np.frombuffer(data, "<f4", 4 * n, pos).reshape(n, 4).copy()
