"""Data preparation for the examples -- numpy counterparts of the helpers of the reference's examples/utils.py (which need open3d
and transforms3d): same names, same arguments, arrays instead of open3d point clouds (every registration function of
probreg_b200 takes arrays).  Readers and the voxel filter come from probreg_b200.io."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from probreg_b200 import io as pio  # noqa: E402


def euler2mat(ax, ay, az):
    """Rotation for static-frame x-y-z Euler angles (what transforms3d.euler.euler2mat(ax, ay, az) returns): Rz(az) Ry(ay) Rx(ax)."""
    cx, sx, cy, sy, cz, sz = np.cos(ax), np.sin(ax), np.cos(ay), np.sin(ay), np.cos(az), np.sin(az)
    rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return rz.dot(ry).dot(rx)


def prepare_source_and_target_rigid_3d(source_filename, noise_amp=0.001, n_random=500, orientation=np.deg2rad([0.0, 0.0, 30.0]),
                                       translation=np.zeros(3), voxel_size=0.005, normals=False, rng=None):
    """Source: the voxel-filtered cloud of `source_filename`.  Target: a shuffled, noised copy with `n_random` uniform outliers in
    1.5x its bounding box, rotated by `orientation` (x-y-z Euler angles) and shifted by `translation`.  `normals` is accepted
    for signature compatibility and ignored (CPD does not use them); `rng` (a numpy Generator) makes the recipe reproducible."""
    rng = np.random.default_rng() if rng is None else rng
    source = pio.voxel_down_sample(pio.read_points(source_filename), voxel_size)
    print("source: %d points" % source.shape[0])
    pts = source[rng.permutation(source.shape[0])]
    box = 1.5 * (pts.max(axis=0) - pts.min(axis=0))
    outliers = (rng.random((n_random, 3)) - 0.5) * box + pts.mean(axis=0)
    cloud = np.r_[pts + noise_amp * rng.standard_normal(pts.shape), outliers]
    target = cloud.dot(euler2mat(*orientation).T) + np.asarray(translation)
    return source, target


def prepare_source_and_target_nonrigid_2d(source_filename, target_filename):
    return np.loadtxt(source_filename), np.loadtxt(target_filename)


def prepare_source_and_target_nonrigid_3d(source_filename, target_filename, voxel_size=5.0):
    source = pio.voxel_down_sample(np.loadtxt(source_filename), voxel_size)
    target = pio.voxel_down_sample(np.loadtxt(target_filename), voxel_size)
    print("source: %d points, target: %d points" % (source.shape[0], target.shape[0]))
    return source, target


def reference_file(name):
    """Path of one of the reference's example data files (bunny.pcd, fish_source.txt, face-x.txt, ...): next to this script, under
    $PROBREG_EXAMPLES, or among the copies kept for the tests (tests/golden/data); None when it is nowhere."""
    here = os.path.dirname(os.path.abspath(__file__))
    for d in (here, os.environ.get("PROBREG_EXAMPLES", ""), os.path.join(os.path.dirname(here), "tests", "golden", "data")):
        if d and os.path.exists(os.path.join(d, name)):
            return os.path.join(d, name)
    return None
