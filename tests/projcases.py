"""Raw sweeps and range-image scenes for the image-projection tests — TEST INFRASTRUCTURE.

`raw_sweep` simulates one raw sweep (tools/synth lins_synth_raw_sweep); `host_projection` runs the product's host
ImageProjection (csrc/host/image_projection.hpp, through tools/synth lins_projection_host) on a fresh object for any model.
`image_points` turns a range image into raw points at the pixel centres, so hand-built scenes reach the device through
the same projection.  `bfs_owners` restates labelComponents' sequential BFS (as tests/pyfront.py runs it) on a graph of
edge flags, and `min_label_owners` is the order-free model the device runs: the owner of a pixel is the smallest raster
index among the unblocked pixels that reach it.
"""
import ctypes as C

import numpy as np

import featcases as fc

F = np.float32


def raw_sweep(synth, defs, config, seed):
    """(POINT_DTYPE raw points, LinsLidarModel) of one simulated sweep of synth.CONFIGS[config]."""
    L = fc._lib(defs)
    cfg = synth.SynthCfg(**synth.CONFIGS[config])
    model = defs.LinsLidarModel.dense64() if int(synth.CONFIGS[config]["lidar"]) == 1 else defs.LinsLidarModel.vlp16()
    cap = model.line_num * model.scan_num
    raw = np.zeros(cap, defs.POINT_DTYPE)
    n = L.lins_synth_raw_sweep(C.byref(cfg), seed, defs.ptr(raw), cap)
    return raw[:n].copy(), model


def host_projection(defs, raw, model):
    """A fresh ImageProjection::process of the raw points: dict as LinsGpu.project_scans returns it."""
    L = fc._lib(defs)
    if not hasattr(L, "_proj_ready"):
        vp = C.c_void_p
        L.lins_projection_host.argtypes = [vp, C.c_int, C.POINTER(defs.LinsLidarModel)] + [vp] * 9
        L._proj_ready = True
    raw = np.asarray(raw)
    pts = defs.as_points(raw) if raw.dtype == defs.POINT_DTYPE else defs.make_points(np.asarray(raw, F).reshape(len(raw), -1)[:, :3], np.zeros(len(raw), F))
    n = len(pts)
    raw = pts if n else np.zeros(1, defs.POINT_DTYPE)
    m = max(n, 1)
    seg, outl = np.zeros(m, defs.POINT_DTYPE), np.zeros(m, defs.POINT_DTYPE)
    ground, col, rng = np.zeros(m, np.uint8), np.zeros(m, np.uint32), np.zeros(m, F)
    sr, er, ori, cnt = np.zeros(model.line_num, np.int32), np.zeros(model.line_num, np.int32), np.zeros(3, F), np.zeros(2, np.int32)
    L.lins_projection_host(defs.ptr(raw), n, C.byref(model), *[defs.ptr(v) for v in (seg, ground, col, rng, outl, sr, er, ori, cnt)])
    a, b = int(cnt[0]), int(cnt[1])
    return dict(seg=fc._x4(seg, a), ground=ground[:a].copy(), col=col[:a].copy(), range=rng[:a].copy(), start_ring=sr, end_ring=er,
                ori=ori, outlier=fc._x4(outl, b))


def model(defs, line_num, scan_num, ang_res_y=2.0, ang_bottom=15.1, ground_scan_ind=0):
    """A model whose columns cover the full turn (ang_res_x = 360 / scan_num)."""
    return defs.LinsLidarModel(line_num, scan_num, F(360.0) / F(scan_num), F(ang_res_y), F(ang_bottom), ground_scan_ind)


def image_points(m, img):
    """Raw points (n x 3 float32, raster order) at the centres of the pixels of a range image (L x S, NaN = no point)."""
    L, S = img.shape
    rows, cols = np.nonzero(np.isfinite(img))
    v = np.radians((rows + 0.5) * float(m.ang_res_y) - float(m.ang_bottom))
    h = np.radians(90.0 + (S // 2 - cols) * float(m.ang_res_x))
    r = img[rows, cols].astype(np.float64)
    return np.stack([r * np.cos(v) * np.sin(h), r * np.cos(v) * np.cos(h), r * np.sin(v)], 1).astype(F)


# ---- labelling: the sequential BFS and the min-label model on edge flags ------------------------------------------------
# E[k][r, c]: the edge from (r, c) in direction k qualifies (k = 0 right with the wrap, 1 the +255 jump, 2 down); both
# functions ignore edges into blocked pixels themselves.
def targets(L, S):
    r, c = np.indices((L, S))
    right = r * S + np.where(c + 1 < S, c + 1, 0)
    jump = r * S + np.where(c + 255 < S, c + 255, 0)
    down = np.where(r + 1 < L, (r + 1) * S + c, -1)
    return right, jump, down


def bfs_owners(blocked, E):
    """labelComponents' raster-order BFS with the std::pair<uint8_t, uint8_t> neighbours (pyfront.image_projection's loop):
    (owner of every pixel as a raster index, -1 where blocked; feasible flag per owner)."""
    L, S = blocked.shape
    label = np.where(blocked, -1, 0).astype(np.int64)
    owner = np.full((L, S), -1, np.int64)
    feasible = {}
    neigh = [(255, 0, None), (0, 1, 0), (0, 255, 1), (1, 0, 2)]
    count = 1
    for r0 in range(L):
        for c0 in range(S):
            if label[r0, c0] != 0:
                continue
            queue, pushed, line_flag, qs = [(r0, c0)], [(r0, c0)], [False] * L, 0
            while qs < len(queue):
                fr, fc_ = queue[qs]
                qs += 1
                label[fr, fc_] = count
                for dr, dc, k in neigh:
                    tr, tc = fr + dr, fc_ + dc
                    if tr < 0 or tr >= L:
                        continue
                    if tc < 0:
                        tc = S - 1
                    if tc >= S:
                        tc = 0
                    if label[tr, tc] != 0:
                        continue
                    if E[k][fr, fc_]:
                        queue.append((tr, tc))
                        label[tr, tc] = count
                        line_flag[tr] = True
                        pushed.append((tr, tc))
            ok = len(pushed) >= 30 or (len(pushed) >= 5 and sum(line_flag) >= 3)
            for r, c in pushed:
                owner[r, c] = r0 * S + c0
            feasible[r0 * S + c0] = ok
            count += 1
    return owner, feasible


def min_label_owners(blocked, E, max_rounds=100000):
    """The device's formulation: labels start at the raster index, then a segmented prefix minimum along each row's runs
    of right edges and pushes along the wrap, jump and down edges until a round changes nothing.  Returns (owner, feasible
    per owner, rounds)."""
    L, S = blocked.shape
    P = L * S
    BIG = P
    blk = blocked.reshape(-1)
    right, jump, down = (t.reshape(-1) for t in targets(L, S))
    ok = [E[k].reshape(-1) & ~blk for k in range(3)]
    ok[0] = ok[0] & ~blk[right]
    ok[1] = ok[1] & ~blk[jump]
    ok[2] = ok[2] & (down >= 0) & ~blk[np.maximum(down, 0)]
    lab = np.where(blk, BIG, np.arange(P)).astype(np.int64)
    col = np.tile(np.arange(S), L)
    link = np.zeros(P, bool)  # the edge from the left neighbour qualifies
    link[1:] = ok[0][:-1]
    link[col == 0] = False
    seg_id = np.cumsum(~link) - 1
    K = BIG + 1
    wrap = ok[0] & (col == S - 1)
    for rounds in range(1, max_rounds + 1):
        old = lab.copy()
        for m, t in ((wrap, right), (ok[1], jump), (ok[2], down)):
            np.minimum.at(lab, t[m], lab[m])
        lab = np.minimum.accumulate(lab - seg_id * K) + seg_id * K
        if np.array_equal(lab, old):
            break
    lab = np.where(blk, -1, lab)
    owner = lab.reshape(L, S)
    feasible = {}
    mem = np.nonzero(~blk)[0]
    o = lab[mem]
    size = np.bincount(o, minlength=P)
    rows = mem // S
    nonseed = mem != o
    pairs = np.unique(o[nonseed] * 256 + rows[nonseed])
    lines = np.bincount(pairs // 256, minlength=P)
    for s in np.unique(o):
        feasible[int(s)] = bool(size[s] >= 30 or (size[s] >= 5 and lines[s] >= 3))
    return owner, feasible, rounds


def random_graph(rng, L, S, p_block=0.2, p_edge=0.6):
    blocked = rng.random((L, S)) < p_block
    E = [rng.random((L, S)) < p_edge for _ in range(3)]
    return blocked, E


# ---- scenes: range images whose labelling reaches one condition each ------------------------------------------------------
def scene(name):
    """(range image L x S with NaN = empty, ground_scan_ind) of a named scene; equal ranges connect, a 2x range step does
    not (the edge test's angle drops below 60 degrees)."""
    nan = np.nan
    if name == "earlier_seed_blocks":
        # seed (0, 5) goes down to (1, 5) first; the later seed (1, 3) reaches (1, 4) but not (1, 5), which it would
        # reach along the row on its own
        img = np.full((3, 40), nan)
        img[0, 5] = 8.0
        img[1, 3:6] = 8.0
        return img, 0
    if name == "wrap":  # a component from row 0 enters row 1 at column S-1 and wraps to columns 0, 1
        img = np.full((3, 40), nan)
        img[0, 39] = 6.0
        img[1, 39] = 6.0
        img[1, 0:2] = 6.0
        img[1, 5] = 12.0
        return img, 0
    if name == "jump_in_row":  # S = 300: (r, c) -> (r, c + 255) lands inside the row
        img = np.full((4, 300), nan)
        img[1, 10] = 7.0
        img[1, 265] = 7.0
        img[2, 265] = 7.0
        img[2, 266:270] = 7.0
        return img, 0
    if name in ("size30", "size29"):  # one row: feasible from 30 points on
        k = 30 if name == "size30" else 29
        img = np.full((3, 80), nan)
        img[1, 10:10 + k] = 9.0
        return img, 0
    if name == "five_three_rows":  # 5 points, pushed members on rows 0, 1, 2: feasible
        img = np.full((4, 40), nan)
        img[0, 0:2] = 5.0
        img[1, 1] = 5.0
        img[2, 1:3] = 5.0
        return img, 0
    if name == "five_seed_row_only":  # 5 points on 3 rows, but row 0 holds only the seed: 2 rows count, infeasible
        img = np.full((4, 40), nan)
        img[0, 7] = 5.0
        img[1, 7] = 5.0
        img[2, 7:10] = 5.0
        return img, 0
    raise KeyError(name)


SCENES = ["earlier_seed_blocks", "wrap", "jump_in_row", "size30", "size29", "five_three_rows", "five_seed_row_only"]


def scene_graph(img):
    """(blocked, E) of a scene image: empty pixels are blocked (no ground: ground_scan_ind 0), edges join equal ranges."""
    L, S = img.shape
    blocked = ~np.isfinite(img)
    E = []
    for t in targets(L, S):
        ok = t >= 0
        tr = np.where(ok, t, 0)
        other = img.reshape(-1)[tr].reshape(L, S)
        E.append(ok.reshape(L, S) & np.isfinite(img) & np.isfinite(other) & (np.abs(img - other) < 0.5))
    return blocked, E
