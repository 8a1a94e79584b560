"""CPU restatement of transform_fusion_node (transform_fusion_node.cpp): test infrastructure, no product code.

The pose the node publishes on /integrated_to_init for one odometry message: transformSum from the message
(laserOdometryHandler :217-231), transformAssociateToMap (:91-215, tests/mapperref.py's MappingOracle.associate_to_map)
against the (transformAftMapped, transformBefMapped) pair the mapping node published (publishTF of
lidar_mapping_node.cpp:737-777 -> odomAftMappedHandler :256-277), and the published orientation.  f64 is Python's float
(libm through math), f32 is numpy float32 with libm's f32 functions, as in tests/mapperref.py; setRPY is
tests/mapper_drive.py's set_rpy (pinned against scipy in tests/test_transform_fusion_cpu.py)."""
import types

import numpy as np

import mapperref
from mapper_drive import odometry_quat, set_rpy  # noqa: F401  (set_rpy: tf::Quaternion::setRPY, re-exported)

F = np.float32


def odometry_transform(quat, pos):
    """transformSum of a pose message (quat x y z w, pos): getRPY of (z, -x, -y, w), then (-pitch, -yaw, roll) in f32."""
    roll, pitch, yaw = mapperref.get_rpy(float(quat[2]), -float(quat[0]), -float(quat[1]), float(quat[3]))
    return np.array([-pitch, -yaw, roll, float(pos[0]), float(pos[1]), float(pos[2])]).astype(F)


def published_pair(aft, bef):
    """What odomAftMappedHandler stores when the mapping node published (aft, bef): NaN -> 0 in both, aft's angles
    through the published quaternion (odometry_quat) and back through getRPY, positions and bef unchanged."""
    a = np.where(np.isnan(aft), F(0), np.asarray(aft, F)).astype(F)
    b = np.where(np.isnan(bef), F(0), np.asarray(bef, F)).astype(F)
    return odometry_transform(odometry_quat(a), a[3:6]), b


def associate(Sum, Bef, Aft):
    """transformAssociateToMap -> transformMapped (the mapping node's transformTobeMapped algebra)."""
    ns = types.SimpleNamespace(Sum=np.array(Sum, F), Bef=np.array(Bef, F), Aft=np.array(Aft, F), Incre=np.zeros(6, F), Tobe=np.zeros(6, F))
    with np.errstate(all="ignore"):
        mapperref.MappingOracle.associate_to_map(ns)
    return ns.Tobe


def fuse(quat, pos, published, aft=None, bef=None):
    """(transformMapped f32 (6), published position f64 (3), orientation x y z w f64 (4)) for one odometry message.
    published: the mapping node has published (aft, bef); else the node's pair is its initial zeros."""
    A, B = published_pair(aft, bef) if published else (np.zeros(6, F), np.zeros(6, F))
    T = associate(odometry_transform(quat, pos), B, A)
    return T, T[3:6].astype(np.float64), np.array(odometry_quat(T), np.float64)


def fuse_row(quat, pos, published, aft=None, bef=None):
    """fuse() as a bag_replay map_fused row: x y z qx qy qz qw."""
    _, p, q = fuse(quat, pos, published, aft, bef)
    return np.concatenate([p, q])
