"""CPU restatement of the mapping node's publishGlobalMap (lidar_mapping_node.cpp:976-1031) for one node: test
infrastructure, no product code.  From the key poses (cloudKeyPoses6D rows x, y, z, roll, pitch, yaw), each key
frame's body-frame corner, surf and outlier DS clouds and currentRobotPosPoint:
1. no key poses: nothing;
2. globalMapKeyPoses: the poses whose f32 squared distance ((dx^2 + dy^2) + dz^2) to cur is strictly below 500^2 (a
   non-finite pose never: KdTreeFLANN drops it), in ascending key index;
3. globalMapKeyPosesDS: pcl::VoxelGrid at 1 m of (x, y, z, intensity = key index) (mapperref.voxel_grid: f32 sums in
   input order, ascending voxel index), and each voxel's (int) intensity centroid;
4. globalMapKeyFrames: each named key frame's corner, surf and outlier cloud through transformPointCloud with its pose
   (mapperref.transform_cloud), concatenated in DS order;
5. globalMapKeyFramesDS: pcl::VoxelGrid at 0.4 m, or the concatenation itself when it overflows (PCL 1.7 publishes its
   input when the leaf is too small)."""
import numpy as np

import mapperref

F = np.float32
RADIUS_SQ = F(500.0) * F(500.0)
POSE_LEAF, MAP_LEAF = 1.0, 0.4


def select(poses, cur):
    """Step 2: the indices of the key poses within the radius of cur."""
    p = np.asarray(poses, F)[:, :3]
    c = np.asarray(cur, F)
    with np.errstate(all="ignore"):
        e = (p - c).astype(F)
        d2 = (e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1]).astype(F) + e[:, 2] * e[:, 2]
    return np.flatnonzero(d2.astype(F) < RADIUS_SQ)


def key_frames(poses, cur):
    """Steps 2-3: (selected indices, the DS key ids in voxel order)."""
    p = np.asarray(poses, F)
    sel = select(p, cur)
    if len(sel) == 0:
        return sel, np.zeros(0, np.int32)
    rows = np.concatenate([p[sel, :3], sel.astype(F)[:, None]], 1)
    return sel, mapperref.voxel_grid(rows, POSE_LEAF)[:, 3].astype(np.int32)


def global_map(poses, body, cur):
    """Steps 1-5 for one node: poses (k, >= 6), body[i] = (corner, surf, outlier) (n, 4) f32 body-frame clouds of key
    frame i.  Returns dict(n_key_poses, keys, points (the concatenation), map, unfiltered)."""
    poses = np.asarray(poses, np.float64)
    sel, keys = key_frames(poses, cur)
    parts = [mapperref.transform_cloud(np.asarray(body[k][a], F).reshape(-1, 4), poses[k, :6]) for k in keys for a in range(3)]
    cat = np.concatenate(parts).astype(F) if parts else np.zeros((0, 4), F)
    try:
        ds, unf = mapperref.voxel_grid(cat, MAP_LEAF), 0
    except mapperref.TooBig:
        ds, unf = cat, 1
    return dict(n_key_poses=len(sel), keys=keys, points=cat, map=ds, unfiltered=unf)
