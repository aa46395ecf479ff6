// include/lvio_b200/se3.h -- Sophus::SE3d's product and inverse on [qx qy qz qw tx ty tz] arrays, in Sophus' and Eigen's operation
// order, for host code that replays PoseGraph::ForwardUpdate (pose_graph.cpp:245-252) without Sophus: the transforms
// lvb_icp_map_optimize_keyframes returns applied as `pose = T * pose`.  lvio_fusion_b200/se3.py restates the same arithmetic.
#pragma once
#include <cmath>

namespace lvb {
namespace se3 {

// Eigen QuaternionBase::_transformVector: uv = 2 (q.vec x p); p + w uv + q.vec x uv
inline void rotate(const double* q, const double* p, double* out) {
    double uv[3] = {q[1] * p[2] - q[2] * p[1], q[2] * p[0] - q[0] * p[2], q[0] * p[1] - q[1] * p[0]};
    for (int k = 0; k < 3; ++k) uv[k] = uv[k] + uv[k];
    const double c[3] = {q[1] * uv[2] - q[2] * uv[1], q[2] * uv[0] - q[0] * uv[2], q[0] * uv[1] - q[1] * uv[0]};
    for (int k = 0; k < 3; ++k) out[k] = (p[k] + q[3] * uv[k]) + c[k];
}
// a * b: Eigen's quaternion product, renormalised by 2 / (1 + |q|^2) when |q|^2 != 1 (Sophus SO3 operator*); t = ta + qa tb
inline void mul(const double* a, const double* b, double* c) {
    const double ax = a[0], ay = a[1], az = a[2], aw = a[3], bx = b[0], by = b[1], bz = b[2], bw = b[3];
    double q[4] = {((aw * bx + ax * bw) + ay * bz) - az * by, ((aw * by + ay * bw) + az * bx) - ax * bz,
                   ((aw * bz + az * bw) + ax * by) - ay * bx, ((aw * bw - ax * bx) - ay * by) - az * bz};
    const double n2 = ((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3];
    if (n2 != 1.0) { const double s = 2.0 / (1.0 + n2); for (int k = 0; k < 4; ++k) q[k] = q[k] * s; }
    double t[3];
    rotate(a, b + 4, t);
    for (int k = 0; k < 4; ++k) c[k] = q[k];
    for (int k = 0; k < 3; ++k) c[4 + k] = a[4 + k] + t[k];
}
// a^-1: the conjugate quaternion normalised, t = R^-1 (-t)
inline void inv(const double* a, double* c) {
    c[0] = -a[0]; c[1] = -a[1]; c[2] = -a[2]; c[3] = a[3];
    const double n = std::sqrt(((c[0] * c[0] + c[1] * c[1]) + c[2] * c[2]) + c[3] * c[3]);
    for (int k = 0; k < 4; ++k) c[k] = c[k] / n;
    const double mt[3] = {-a[4], -a[5], -a[6]};
    rotate(c, mt, c + 4);
}

}  // namespace se3
}  // namespace lvb
