"""The SE3 arithmetic of lvb_icp_map_optimize_keyframes, restated on the host bit for bit.

The device composes and inverts poses ([qx qy qz qw tx ty tz], Sophus::SE3d::data()) in FP64 with every product and sum rounded on
its own (no fused multiply-add), in the operation order of Sophus and Eigen (icp.cu: kf_se3_mul, kf_se3_inv).  Python floats are IEEE
doubles with the same per-operation rounding, so the functions below return exactly what the device returns: the incoming pose of a
chained keyframe, its transform new * old^-1, and the PoseGraph::ForwardUpdate a caller replays on the host.
"""
import math

import numpy as np


def _rotate(q, p):
    """Eigen QuaternionBase::_transformVector: uv = 2 (q.vec x p); p + w uv + q.vec x uv."""
    uv = [q[1] * p[2] - q[2] * p[1], q[2] * p[0] - q[0] * p[2], q[0] * p[1] - q[1] * p[0]]
    uv = [u + u for u in uv]
    c = [q[1] * uv[2] - q[2] * uv[1], q[2] * uv[0] - q[0] * uv[2], q[0] * uv[1] - q[1] * uv[0]]
    return [(p[k] + q[3] * uv[k]) + c[k] for k in range(3)]


def mul(a, b):
    """Sophus SE3 product a * b: Eigen's quaternion product, renormalised by 2 / (1 + |q|^2) when |q|^2 != 1, t = ta + qa tb."""
    a = [float(x) for x in a]
    b = [float(x) for x in b]
    ax, ay, az, aw = a[:4]
    bx, by, bz, bw = b[:4]
    q = [((aw * bx + ax * bw) + ay * bz) - az * by,
         ((aw * by + ay * bw) + az * bx) - ax * bz,
         ((aw * bz + az * bw) + ax * by) - ay * bx,
         ((aw * bw - ax * bx) - ay * by) - az * bz]
    n2 = ((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3]
    if n2 != 1.0:
        s = 2.0 / (1.0 + n2)
        q = [x * s for x in q]
    t = _rotate(a[:4], b[4:])
    return np.array(q + [a[4 + k] + t[k] for k in range(3)])


def inv(a):
    """Sophus SE3 inverse: the conjugate quaternion normalised (SO3 construction), t = R^-1 (-t)."""
    a = [float(x) for x in a]
    c = [-a[0], -a[1], -a[2], a[3]]
    n = math.sqrt(((c[0] * c[0] + c[1] * c[1]) + c[2] * c[2]) + c[3] * c[3])
    c = [x / n for x in c]
    return np.array(c + _rotate(c, [-a[4], -a[5], -a[6]]))


def transform(new, old):
    """T = new * old^-1 (mapping.cpp:181-182)."""
    return mul(new, inv(old))


def forward_update(transforms, pose):
    """The incoming pose of a chained keyframe: PoseGraph::ForwardUpdate of each earlier transform in order (pose = T * pose)."""
    p = np.asarray(pose, dtype=np.float64)
    for T in transforms:
        p = mul(T, p)
    return p
