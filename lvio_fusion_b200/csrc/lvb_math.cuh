// lvb_math.cuh -- per-factor residual / Jacobian arithmetic of the CUDA backend.
//
// Hand-derived closed forms (no autodiff on the hot path).  Everything is
// __host__ __device__ so that tests/hostcheck can compile the very same functions with g++
// and compare them against the CPU oracle without a GPU; the product only ever calls them
// from kernels.
//
// Reference semantics (paths relative to /root/reference/src/lvio_fusion/):
//   include/lvio_fusion/ceres/base.hpp:10-157        SE3 helpers, [qx qy qz qw tx ty tz]
//   include/lvio_fusion/ceres/visual_error.hpp:10-137 the three reprojection factors
//   include/lvio_fusion/ceres/imu_error.hpp:12-122    ImuError (analytic, whitened)
//   src/preintegration.cpp:144-165                    its residual
//   include/lvio_fusion/ceres/lidar_error.hpp:42-110  point-to-plane RPZ / YXY
//   include/lvio_fusion/ceres/pose_error.hpp:10-86    PoseGraphError / PoseError
//
// Pose Jacobians: ceres::QuaternionRotatePoint normalises q, so the ambient 3x4 quaternion
// Jacobian of R(q)v is  -2 [Rv]x E(u) / |q|  with u = q/|q| = (ubar, w) and
// E(u) = [ w I + [ubar]x | -ubar ]  (3x4, columns x y z w), and the tangent Jacobian under
// ceres::EigenQuaternionParameterization (q' = dq (x) q, |delta| used as the half angle) is
// simply  -2 [Rv]x  because E(u) . PlusJacobian(u) = I.  For R(q)^T x it is  +2 R^T [x]x.
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define LVB_HD __host__ __device__ __forceinline__
#else
#define LVB_HD inline
#endif

namespace lvb {

struct V3 { double x, y, z; };
struct M3 { double m[9]; };  // row-major

LVB_HD V3 v3(double x, double y, double z) { V3 r; r.x = x; r.y = y; r.z = z; return r; }
LVB_HD V3 operator+(const V3& a, const V3& b) { return v3(a.x + b.x, a.y + b.y, a.z + b.z); }
LVB_HD V3 operator-(const V3& a, const V3& b) { return v3(a.x - b.x, a.y - b.y, a.z - b.z); }
LVB_HD V3 operator*(const V3& a, double s) { return v3(a.x * s, a.y * s, a.z * s); }
LVB_HD double dot(const V3& a, const V3& b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
LVB_HD V3 cross(const V3& a, const V3& b) { return v3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
LVB_HD V3 mul(const M3& R, const V3& v) {
    return v3(R.m[0] * v.x + R.m[1] * v.y + R.m[2] * v.z, R.m[3] * v.x + R.m[4] * v.y + R.m[5] * v.z, R.m[6] * v.x + R.m[7] * v.y + R.m[8] * v.z);
}
LVB_HD V3 mulT(const M3& R, const V3& v) {
    return v3(R.m[0] * v.x + R.m[3] * v.y + R.m[6] * v.z, R.m[1] * v.x + R.m[4] * v.y + R.m[7] * v.z, R.m[2] * v.x + R.m[5] * v.y + R.m[8] * v.z);
}
LVB_HD M3 mul(const M3& A, const M3& B) {
    M3 C;
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) C.m[3 * i + j] = A.m[3 * i] * B.m[j] + A.m[3 * i + 1] * B.m[3 + j] + A.m[3 * i + 2] * B.m[6 + j];
    return C;
}
LVB_HD M3 transpose(const M3& A) { M3 C; for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) C.m[3 * i + j] = A.m[3 * j + i]; return C; }

// Unit quaternion (xyzw) of a stored pose block and its norm.
struct UQ { double x, y, z, w, norm; };
LVB_HD UQ unit_quat(const double* q) {
    UQ u; u.norm = sqrt(q[3] * q[3] + q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
    const double s = 1.0 / u.norm;
    u.x = q[0] * s; u.y = q[1] * s; u.z = q[2] * s; u.w = q[3] * s; return u;
}
LVB_HD M3 rot_matrix(const UQ& u) {
    const double xx = u.x * u.x, yy = u.y * u.y, zz = u.z * u.z, xy = u.x * u.y, xz = u.x * u.z, yz = u.y * u.z, wx = u.w * u.x, wy = u.w * u.y, wz = u.w * u.z;
    M3 R;
    R.m[0] = 1 - 2 * (yy + zz); R.m[1] = 2 * (xy - wz);     R.m[2] = 2 * (xz + wy);
    R.m[3] = 2 * (xy + wz);     R.m[4] = 1 - 2 * (xx + zz); R.m[5] = 2 * (yz - wx);
    R.m[6] = 2 * (xz - wy);     R.m[7] = 2 * (yz + wx);     R.m[8] = 1 - 2 * (xx + yy);
    return R;
}

// row (1x3 tangent rotation part)  ->  row (1x4 ambient quaternion part):  out = a . E(u) / |q|
LVB_HD void tangent_to_ambient(const UQ& u, const double a[3], double out[4]) {
    const double s = 1.0 / u.norm;
    // E = [ w I + [ubar]x | -ubar ],  [ubar]x = [[0,-z,y],[z,0,-x],[-y,x,0]]
    out[0] = (a[0] * u.w + a[1] * u.z - a[2] * u.y) * s;
    out[1] = (-a[0] * u.z + a[1] * u.w + a[2] * u.x) * s;
    out[2] = (a[0] * u.y - a[1] * u.x + a[2] * u.w) * s;
    out[3] = -(a[0] * u.x + a[1] * u.y + a[2] * u.z) * s;
}
// row a (1x3) times [v]x :  (a [v]x)_j ;  [v]x = [[0,-vz,vy],[vz,0,-vx],[-vy,vx,0]]
LVB_HD void row_times_skew(const double a[3], const V3& v, double out[3]) {
    out[0] = a[1] * v.z - a[2] * v.y;
    out[1] = -a[0] * v.z + a[2] * v.x;
    out[2] = a[0] * v.y - a[1] * v.x;
}

// Camera constants, precomputed once per problem on the host (extrinsic quaternion normalised).
struct Cam {
    double fx, fy, cx, cy;
    M3 R;      // R_body_cam
    V3 t;      // t_body_cam
};
struct Cams { Cam c0, c1; };

LVB_HD Cam make_cam(const double* c11) {
    Cam k; k.fx = c11[0]; k.fy = c11[1]; k.cx = c11[2]; k.cy = c11[3];
    k.R = rot_matrix(unit_quat(c11 + 4)); k.t = v3(c11[8], c11[9], c11[10]); return k;
}

// Projection of a body-frame point into `cam`:  residual rows and d(pixel)/d(p_body) (2x3), times w.
struct Proj { double u, v; double Jb[6]; };  // Jb row-major 2x3 = w * Dpi(pc) * Rc^T
LVB_HD Proj project_body(const Cam& cam, const V3& p_body, double w) {
    const V3 pc = mulT(cam.R, p_body - cam.t);
    const double iz = 1.0 / pc.z;
    Proj o; o.u = cam.fx * (pc.x * iz) + cam.cx; o.v = cam.fy * (pc.y * iz) + cam.cy;
    const double a0 = w * cam.fx * iz, a2 = -w * cam.fx * pc.x * iz * iz;   // row u: [a0, 0, a2]
    const double b1 = w * cam.fy * iz, b2 = -w * cam.fy * pc.y * iz * iz;   // row v: [0, b1, b2]
    // times Rc^T : (row . Rc^T)_j = sum_k row_k Rc[j][k]
    for (int j = 0; j < 3; ++j) {
        o.Jb[j] = a0 * cam.R.m[3 * j] + a2 * cam.R.m[3 * j + 2];
        o.Jb[3 + j] = b1 * cam.R.m[3 * j + 1] + b2 * cam.R.m[3 * j + 2];
    }
    return o;
}

// ---------------------------------------------------------------------------------------
// a1 TwoFrameReprojectionError (visual_error.hpp:84-96).
// In:  c = first_ob.xy ob.xy weight ; rho ; T1 (first keyframe) ; T2 (this keyframe)
// Out: r[2]; Jrho[2]; J1t[12], J2t[12] = tangent 2x6 blocks [rot(3) | trans(3)] row-major.
// ---------------------------------------------------------------------------------------
struct TwoFrameLin { double r[2], Jrho[2], J1[12], J2[12]; };

LVB_HD void two_frame_lin(const Cams& K, double fo_x, double fo_y, double ob_x, double ob_y, double w,
                          double rho, const double* T1, const double* T2, TwoFrameLin& o,
                          UQ* u1_out, UQ* u2_out) {
    const double d = 1.0 / rho;
    const V3 dir = v3((fo_x - K.c1.cx) / K.c1.fx, (fo_y - K.c1.cy) / K.c1.fy, 1.0);
    const V3 Rdir = mul(K.c1.R, dir);
    const V3 pb = Rdir * d + K.c1.t;                        // Pixel2Robot, :25-33
    const UQ u1 = unit_quat(T1), u2 = unit_quat(T2);
    const M3 R1 = rot_matrix(u1), R2 = rot_matrix(u2);
    const V3 R1pb = mul(R1, pb);
    const V3 pw = R1pb + v3(T1[4], T1[5], T1[6]);           // SE3TransformPoint(Twc1, pb)
    const V3 x = pw - v3(T2[4], T2[5], T2[6]);
    const V3 pb2 = mulT(R2, x);                             // Twc2^-1 * pw
    const Proj P = project_body(K.c0, pb2, w);
    o.r[0] = w * (P.u - ob_x); o.r[1] = w * (P.v - ob_y);
    const V3 dpw_drho = mul(R1, Rdir) * (-d * d);
    for (int row = 0; row < 2; ++row) {
        const double* jb = P.Jb + 3 * row;
        double jw[3];                                       // jb . R2^T
        for (int j = 0; j < 3; ++j) jw[j] = jb[0] * R2.m[3 * j] + jb[1] * R2.m[3 * j + 1] + jb[2] * R2.m[3 * j + 2];
        o.Jrho[row] = jw[0] * dpw_drho.x + jw[1] * dpw_drho.y + jw[2] * dpw_drho.z;
        double t[3];
        row_times_skew(jw, R1pb, t);                        // d/dphi1 = -2 jw [R1 pb]x
        o.J1[6 * row + 0] = -2 * t[0]; o.J1[6 * row + 1] = -2 * t[1]; o.J1[6 * row + 2] = -2 * t[2];
        o.J1[6 * row + 3] = jw[0]; o.J1[6 * row + 4] = jw[1]; o.J1[6 * row + 5] = jw[2];
        row_times_skew(jw, x, t);                           // d/dphi2 = +2 jw [x]x
        o.J2[6 * row + 0] = 2 * t[0]; o.J2[6 * row + 1] = 2 * t[1]; o.J2[6 * row + 2] = 2 * t[2];
        o.J2[6 * row + 3] = -jw[0]; o.J2[6 * row + 4] = -jw[1]; o.J2[6 * row + 5] = -jw[2];
    }
    if (u1_out) *u1_out = u1;
    if (u2_out) *u2_out = u2;
}

// a2 PoseOnlyReprojectionError (visual_error.hpp:54-64): c = ob.xy pw.xyz weight
struct PoseOnlyLin { double r[2], J[12]; };
LVB_HD void pose_only_lin(const Cams& K, double ob_x, double ob_y, const V3& pw, double w, const double* T, PoseOnlyLin& o, UQ* u_out) {
    const UQ u = unit_quat(T);
    const M3 R = rot_matrix(u);
    const V3 x = pw - v3(T[4], T[5], T[6]);
    const V3 pb = mulT(R, x);
    const Proj P = project_body(K.c0, pb, w);
    o.r[0] = w * (P.u - ob_x); o.r[1] = w * (P.v - ob_y);
    for (int row = 0; row < 2; ++row) {
        const double* jb = P.Jb + 3 * row;
        double jw[3], t[3];
        for (int j = 0; j < 3; ++j) jw[j] = jb[0] * R.m[3 * j] + jb[1] * R.m[3 * j + 1] + jb[2] * R.m[3 * j + 2];
        row_times_skew(jw, x, t);
        o.J[6 * row + 0] = 2 * t[0]; o.J[6 * row + 1] = 2 * t[1]; o.J[6 * row + 2] = 2 * t[2];
        o.J[6 * row + 3] = -jw[0]; o.J[6 * row + 4] = -jw[1]; o.J[6 * row + 5] = -jw[2];
    }
    if (u_out) *u_out = u;
}

// a3 TwoCameraReprojectionError (visual_error.hpp:115-126): c = left_ob.xy right_ob.xy weight
struct TwoCameraLin { double r[2], Jrho[2]; };
LVB_HD void two_camera_lin(const Cams& K, double lo_x, double lo_y, double ro_x, double ro_y, double w, double rho, TwoCameraLin& o) {
    const double d = 1.0 / rho;
    const V3 dir = v3((ro_x - K.c1.cx) / K.c1.fx, (ro_y - K.c1.cy) / K.c1.fy, 1.0);
    const V3 Rdir = mul(K.c1.R, dir);
    const V3 pb = Rdir * d + K.c1.t;
    const Proj P = project_body(K.c0, pb, w);
    o.r[0] = w * (P.u - lo_x); o.r[1] = w * (P.v - lo_y);
    const V3 dpb = Rdir * (-d * d);
    o.Jrho[0] = P.Jb[0] * dpb.x + P.Jb[1] * dpb.y + P.Jb[2] * dpb.z;
    o.Jrho[1] = P.Jb[3] * dpb.x + P.Jb[4] * dpb.y + P.Jb[5] * dpb.z;
}

// Expand a tangent 2x6 pose block to the ambient 2x7 block Ceres' Evaluate returns.
LVB_HD void pose_block_to_ambient(const UQ& u, const double* Jt /*rows x 6*/, int rows, double* Ja /*rows x ld*/, int ld) {
    for (int r = 0; r < rows; ++r) {
        double q4[4];
        tangent_to_ambient(u, Jt + 6 * r, q4);
        Ja[r * ld + 0] = q4[0]; Ja[r * ld + 1] = q4[1]; Ja[r * ld + 2] = q4[2]; Ja[r * ld + 3] = q4[3];
        Ja[r * ld + 4] = Jt[6 * r + 3]; Ja[r * ld + 5] = Jt[6 * r + 4]; Ja[r * ld + 6] = Jt[6 * r + 5];
    }
}

// [upstream] ceres::EigenQuaternionParameterization::ComputeJacobian (4x3 row-major) at the stored q
LVB_HD void quat_plus_jacobian(const double* q, double* j) {
    j[0] = q[3];  j[1] = q[2];   j[2] = -q[1];
    j[3] = -q[2]; j[4] = q[3];   j[5] = q[0];
    j[6] = q[1];  j[7] = -q[0];  j[8] = q[3];
    j[9] = -q[0]; j[10] = -q[1]; j[11] = -q[2];
}
// ambient row (7) -> tangent row (6) through the ProductParameterization Jacobian (backend.cpp:99-101)
LVB_HD void ambient_row_to_tangent(const double* q, const double* a7, double* t6) {
    double pj[12]; quat_plus_jacobian(q, pj);
    for (int c = 0; c < 3; ++c) t6[c] = a7[0] * pj[c] + a7[1] * pj[3 + c] + a7[2] * pj[6 + c] + a7[3] * pj[9 + c];
    t6[3] = a7[4]; t6[4] = a7[5]; t6[5] = a7[6];
}

// [upstream] EigenQuaternionParameterization::Plus + Identity(3):  q' = dq (x) q
LVB_HD void pose_plus(const double* x, const double* d, double* out) {
    const double n = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    if (n > 0.0) {
        const double k = sin(n) / n, cw = cos(n);
        const double ax = k * d[0], ay = k * d[1], az = k * d[2];
        const double bx = x[0], by = x[1], bz = x[2], bw = x[3];
        out[0] = cw * bx + ax * bw + ay * bz - az * by;
        out[1] = cw * by - ax * bz + ay * bw + az * bx;
        out[2] = cw * bz + ax * by - ay * bx + az * bw;
        out[3] = cw * bw - ax * bx - ay * by - az * bz;
    } else { out[0] = x[0]; out[1] = x[1]; out[2] = x[2]; out[3] = x[3]; }
    out[4] = x[4] + d[3]; out[5] = x[5] + d[4]; out[6] = x[6] + d[5];
}

// Ceres HuberLoss(a) + Corrector [upstream]: rho''<=0 => r,J scaled by sqrt(rho'); a<=0: none.
LVB_HD void huber(double a, double s, double* rho, double* sqrt_rho1) {
    if (a > 0.0 && s > a * a) {
        const double r = sqrt(s);
        *rho = 2.0 * a * r - a * a;
        *sqrt_rho1 = sqrt(fmax(2.2250738585072014e-308, a / r));
    } else { *rho = s; *sqrt_rho1 = 1.0; }
}

// ---------------------------------------------------------------------------------------
// Minimal forward-mode dual for the two rare prior kinds (<= one block per keyframe): the
// Euler-angle chain (atan2/asin of a quaternion product) is not worth a hand derivation.
// ---------------------------------------------------------------------------------------
template <int N> struct Du { double v; double d[N]; };
template <int N> LVB_HD Du<N> du_const(double s) { Du<N> r; r.v = s; for (int i = 0; i < N; ++i) r.d[i] = 0; return r; }
template <int N> LVB_HD Du<N> du_seed(double s, int k) { Du<N> r = du_const<N>(s); r.d[k] = 1.0; return r; }
template <int N> LVB_HD Du<N> operator+(const Du<N>& a, const Du<N>& b) { Du<N> r; r.v = a.v + b.v; for (int i = 0; i < N; ++i) r.d[i] = a.d[i] + b.d[i]; return r; }
template <int N> LVB_HD Du<N> operator-(const Du<N>& a, const Du<N>& b) { Du<N> r; r.v = a.v - b.v; for (int i = 0; i < N; ++i) r.d[i] = a.d[i] - b.d[i]; return r; }
template <int N> LVB_HD Du<N> operator-(const Du<N>& a) { Du<N> r; r.v = -a.v; for (int i = 0; i < N; ++i) r.d[i] = -a.d[i]; return r; }
template <int N> LVB_HD Du<N> operator*(const Du<N>& a, const Du<N>& b) { Du<N> r; r.v = a.v * b.v; for (int i = 0; i < N; ++i) r.d[i] = a.d[i] * b.v + a.v * b.d[i]; return r; }
template <int N> LVB_HD Du<N> operator*(const Du<N>& a, double b) { Du<N> r; r.v = a.v * b; for (int i = 0; i < N; ++i) r.d[i] = a.d[i] * b; return r; }
template <int N> LVB_HD Du<N> operator*(double b, const Du<N>& a) { return a * b; }
template <int N> LVB_HD Du<N> operator+(const Du<N>& a, double b) { Du<N> r = a; r.v += b; return r; }
template <int N> LVB_HD Du<N> operator-(double b, const Du<N>& a) { Du<N> r = -a; r.v += b; return r; }
template <int N> LVB_HD Du<N> operator/(const Du<N>& a, const Du<N>& b) { Du<N> r; const double inv = 1.0 / b.v; r.v = a.v * inv; for (int i = 0; i < N; ++i) r.d[i] = (a.d[i] - r.v * b.d[i]) * inv; return r; }
template <int N> LVB_HD Du<N> du_sqrt(const Du<N>& a) { Du<N> r; r.v = sqrt(a.v); const double k = 0.5 / r.v; for (int i = 0; i < N; ++i) r.d[i] = a.d[i] * k; return r; }
template <int N> LVB_HD Du<N> du_asin(const Du<N>& a) { Du<N> r; r.v = asin(a.v); const double k = 1.0 / sqrt(1.0 - a.v * a.v); for (int i = 0; i < N; ++i) r.d[i] = a.d[i] * k; return r; }
template <int N> LVB_HD Du<N> du_atan2(const Du<N>& y, const Du<N>& x) { Du<N> r; r.v = atan2(y.v, x.v); const double k = 1.0 / (x.v * x.v + y.v * y.v); for (int i = 0; i < N; ++i) r.d[i] = (x.v * y.d[i] - y.v * x.d[i]) * k; return r; }

template <int N> struct DQ { Du<N> x, y, z, w; };
template <int N> struct DV { Du<N> x, y, z; };
template <int N> struct DT { DQ<N> q; DV<N> t; };

template <int N> LVB_HD DV<N> du_rotate(const DQ<N>& q, const DV<N>& p) {      // normalising rotate (base.hpp:26-31)
    const Du<N> one = du_const<N>(1.0);
    const Du<N> s = one / du_sqrt(q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z);
    const Du<N> ux = s * q.x, uy = s * q.y, uz = s * q.z, uw = s * q.w;
    Du<N> a = uy * p.z - uz * p.y, b = uz * p.x - ux * p.z, c = ux * p.y - uy * p.x;
    a = a + a; b = b + b; c = c + c;
    DV<N> r;
    r.x = p.x + uw * a + (uy * c - uz * b);
    r.y = p.y + uw * b + (uz * a - ux * c);
    r.z = p.z + uw * c + (ux * b - uy * a);
    return r;
}
template <int N> LVB_HD DQ<N> du_qmul(const DQ<N>& z, const DQ<N>& w) {
    DQ<N> r;
    r.w = z.w * w.w - z.x * w.x - z.y * w.y - z.z * w.z;
    r.x = z.w * w.x + z.x * w.w + z.y * w.z - z.z * w.y;
    r.y = z.w * w.y - z.x * w.z + z.y * w.w + z.z * w.x;
    r.z = z.w * w.z + z.x * w.y - z.y * w.x + z.z * w.w;
    return r;
}
template <int N> LVB_HD DT<N> du_inverse(const DT<N>& a) {                     // base.hpp:49-55
    DT<N> r; r.q.x = -a.q.x; r.q.y = -a.q.y; r.q.z = -a.q.z; r.q.w = a.q.w;
    DV<N> nt; nt.x = -a.t.x; nt.y = -a.t.y; nt.z = -a.t.z;
    r.t = du_rotate(r.q, nt); return r;
}
template <int N> LVB_HD DT<N> du_compose(const DT<N>& a, const DT<N>& b) {     // base.hpp:70-77
    DT<N> r; r.q = du_qmul(a.q, b.q);
    const DV<N> t = du_rotate(a.q, b.t);
    r.t.x = a.t.x + t.x; r.t.y = a.t.y + t.y; r.t.z = a.t.z + t.z; return r;
}
template <int N> LVB_HD void du_rpyxyz(const DT<N>& a, Du<N>* e) {             // base.hpp:94-141
    const Du<N>& q0 = a.q.w; const Du<N>& q1 = a.q.x; const Du<N>& q2 = a.q.y; const Du<N>& q3 = a.q.z;
    const Du<N> one = du_const<N>(1.0);
    e[0] = du_atan2(2.0 * (q1 * q2 + q0 * q3), one - 2.0 * (q2 * q2 + q3 * q3));
    e[1] = du_asin(2.0 * (q0 * q2 - q1 * q3));
    e[2] = du_atan2(2.0 * (q2 * q3 + q0 * q1), one - 2.0 * (q1 * q1 + q2 * q2));
    e[3] = a.t.x; e[4] = a.t.y; e[5] = a.t.z;
}
template <int N> LVB_HD DT<N> du_load(const double* p, int seed0) {            // seed0 < 0: constant
    DT<N> r;
    Du<N>* f[7] = {&r.q.x, &r.q.y, &r.q.z, &r.q.w, &r.t.x, &r.t.y, &r.t.z};
    for (int i = 0; i < 7; ++i) *f[i] = (seed0 >= 0) ? du_seed<N>(p[i], seed0 + i) : du_const<N>(p[i]);
    return r;
}

// PoseGraphError (pose_error.hpp:25-39): c = rpyxyz_[6] weight v.  r[6], J[6x14] ambient row-major.
LVB_HD void pose_graph_eval(const double* c, const double* T1, const double* T2, double* r, double* J) {
    const DT<14> a = du_load<14>(T1, 0), b = du_load<14>(T2, 7);
    Du<14> e[6];
    du_rpyxyz(du_compose(du_inverse(a), b), e);
    const double w = c[6], v = c[7];
    const double k[6] = {v * w, v * w, v * w, w, 10 * w, 10 * w};
    for (int i = 0; i < 6; ++i) { r[i] = k[i] * (c[i] - e[i].v); if (J) for (int j = 0; j < 14; ++j) J[14 * i + j] = -k[i] * e[i].d[j]; }
}
// PoseError (pose_error.hpp:60-76): c = pose_[7] weight v.  r[6], J[6x7].
LVB_HD void pose_prior_eval(const double* c, const double* T, double* r, double* J) {
    const DT<7> o = du_load<7>(c, -1), p = du_load<7>(T, 0);
    Du<7> e[6];
    du_rpyxyz(du_compose(du_inverse(o), p), e);
    const double w = c[7], v = c[8];
    const double k[6] = {v * w, v * w, v * w, w, w, w};
    for (int i = 0; i < 6; ++i) { r[i] = k[i] * e[i].v; if (J) for (int j = 0; j < 7; ++j) J[7 * i + j] = k[i] * e[i].d[j]; }
}

// ---------------------------------------------------------------------------------------
// a4 ImuError.  Eigen semantics restated: Quaternion::inverse = conj/|q|^2, q*v through the
// unit-quaternion formula, toRotationMatrix (unit formula).  U = sqrt information (upper),
// precomputed once per solve (covariance is constant during a solve).
// ---------------------------------------------------------------------------------------
struct Q4 { double x, y, z, w; };
LVB_HD Q4 q4(double x, double y, double z, double w) { Q4 q; q.x = x; q.y = y; q.z = z; q.w = w; return q; }
LVB_HD Q4 qmul(const Q4& a, const Q4& b) {
    return q4(a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y, a.w * b.y - a.x * b.z + a.y * b.w + a.z * b.x,
              a.w * b.z + a.x * b.y - a.y * b.x + a.z * b.w, a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z);
}
LVB_HD Q4 qinv(const Q4& q) { const double n2 = q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w; return q4(-q.x / n2, -q.y / n2, -q.z / n2, q.w / n2); }
LVB_HD V3 qrot(const Q4& q, const V3& v) { const V3 qv = v3(q.x, q.y, q.z); V3 uv = cross(qv, v); uv = uv + uv; return v + uv * q.w + cross(qv, uv); }
LVB_HD M3 qmat(const Q4& q) {
    const double tx = 2 * q.x, ty = 2 * q.y, tz = 2 * q.z, twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
    const double txx = tx * q.x, txy = ty * q.x, txz = tz * q.x, tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
    M3 R;
    R.m[0] = 1 - (tyy + tzz); R.m[1] = txy - twz;       R.m[2] = txz + twy;
    R.m[3] = txy + twz;       R.m[4] = 1 - (txx + tzz); R.m[5] = tyz - twx;
    R.m[6] = txz - twy;       R.m[7] = tyz + twx;       R.m[8] = 1 - (txx + tyy);
    return R;
}
LVB_HD M3 skew(const V3& v) { M3 r; r.m[0] = 0; r.m[1] = -v.z; r.m[2] = v.y; r.m[3] = v.z; r.m[4] = 0; r.m[5] = -v.x; r.m[6] = -v.y; r.m[7] = v.x; r.m[8] = 0; return r; }
// bottom-right 3x3 of q_left(a) * q_right(b)  (utility.h:124-140, imu_error.hpp:49)
LVB_HD M3 left_right_br(const Q4& a, const Q4& b) {
    const V3 av = v3(a.x, a.y, a.z), bv = v3(b.x, b.y, b.z);
    const M3 sa = skew(av), sb = skew(bv);
    M3 La, Rb, out;
    for (int i = 0; i < 9; ++i) { La.m[i] = sa.m[i]; Rb.m[i] = -sb.m[i]; }
    La.m[0] += a.w; La.m[4] += a.w; La.m[8] += a.w; Rb.m[0] += b.w; Rb.m[4] += b.w; Rb.m[8] += b.w;
    out = mul(La, Rb);
    const double avv[3] = {av.x, av.y, av.z}, bvv[3] = {bv.x, bv.y, bv.z};
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) out.m[3 * i + j] -= avv[i] * bvv[j];
    return out;
}
LVB_HD M3 left_br(const Q4& a) { M3 s = skew(v3(a.x, a.y, a.z)); s.m[0] += a.w; s.m[4] += a.w; s.m[8] += a.w; return s; }

// IMU constants as kept on the device per factor: 17 scalars + the five 3x3 Jacobian sub-blocks
// (dp_dba dp_dbg dq_dbg dv_dba dv_dbg, 45) + U (225, upper, row-major).
struct ImuConst {
    V3 dp, dv, lin_ba, lin_bg; Q4 dq; double sum_dt;
    M3 dp_dba, dp_dbg, dq_dbg, dv_dba, dv_dbg;
};

// raw (un-whitened) residual, preintegration.cpp:144-165; gravity (0,0,9.81007) :13
LVB_HD void imu_raw_residual(const ImuConst& c, const double* Ti, const double* Vi, const double* Bai, const double* Bgi,
                             const double* Tj, const double* Vj, const double* Baj, const double* Bgj, double* r) {
    const V3 g = v3(0.0, 0.0, 9.81007);
    const Q4 Qi = q4(Ti[0], Ti[1], Ti[2], Ti[3]), Qj = q4(Tj[0], Tj[1], Tj[2], Tj[3]);
    const V3 Pi = v3(Ti[4], Ti[5], Ti[6]), Pj = v3(Tj[4], Tj[5], Tj[6]);
    const V3 vi = v3(Vi[0], Vi[1], Vi[2]), vj = v3(Vj[0], Vj[1], Vj[2]);
    const V3 dba = v3(Bai[0], Bai[1], Bai[2]) - c.lin_ba, dbg = v3(Bgi[0], Bgi[1], Bgi[2]) - c.lin_bg;
    const V3 th = mul(c.dq_dbg, dbg);
    const Q4 cq = qmul(c.dq, q4(th.x / 2, th.y / 2, th.z / 2, 1.0));
    const V3 cv = c.dv + mul(c.dv_dba, dba) + mul(c.dv_dbg, dbg);
    const V3 cp = c.dp + mul(c.dp_dba, dba) + mul(c.dp_dbg, dbg);
    const Q4 Qi_inv = qinv(Qi);
    const double dt = c.sum_dt;
    const V3 rp = qrot(Qi_inv, ((g * 0.5) * dt) * dt + Pj - Pi - vi * dt) - cp;
    const Q4 qe = qmul(qinv(cq), qmul(Qi_inv, Qj));
    const V3 rv = qrot(Qi_inv, g * dt + vj - vi) - cv;
    r[0] = rp.x; r[1] = rp.y; r[2] = rp.z; r[3] = 2 * qe.x; r[4] = 2 * qe.y; r[5] = 2 * qe.z;
    r[6] = rv.x; r[7] = rv.y; r[8] = rv.z;
    r[9] = Baj[0] - Bai[0]; r[10] = Baj[1] - Bai[1]; r[11] = Baj[2] - Bai[2];
    r[12] = Bgj[0] - Bgi[0]; r[13] = Bgj[1] - Bgi[1]; r[14] = Bgj[2] - Bgi[2];
}

// raw ambient Jacobian, row-major 15 x 32, columns: pose_i(7) v_i(3) ba_i(3) bg_i(3) pose_j(7) v_j(3) ba_j(3) bg_j(3)
// (imu_error.hpp:43-110; rotation columns at 0..2, column 3 == 0, translation at 4..6)
LVB_HD void put3(double* J, int r0, int c0, const M3& b, double s) { for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) J[(r0 + i) * 32 + c0 + j] = s * b.m[3 * i + j]; }
// One parameter block of the raw Jacobian (blk = 0..7 in AddResidualBlock order); the eight blocks touch disjoint
// columns, so eight lanes of a warp fill the 15x32 matrix concurrently.
LVB_HD void imu_raw_jacobian_block(const ImuConst& c, int blk, const double* Ti, const double* Vi, const double* Bgi,
                                   const double* Tj, const double* Vj, double* J /*15x32, pre-zeroed*/) {
    const V3 g = v3(0.0, 0.0, 9.81007);
    const Q4 Qi = q4(Ti[0], Ti[1], Ti[2], Ti[3]), Qj = q4(Tj[0], Tj[1], Tj[2], Tj[3]);
    const double dt = c.sum_dt;
    const Q4 Qi_inv = qinv(Qi);
    M3 I; for (int i = 0; i < 9; ++i) I.m[i] = 0; I.m[0] = I.m[4] = I.m[8] = 1.0;
    if (blk == 0) {            // pose_i  (:43-53)
        const V3 Pi = v3(Ti[4], Ti[5], Ti[6]), Pj = v3(Tj[4], Tj[5], Tj[6]);
        const V3 vi = v3(Vi[0], Vi[1], Vi[2]), vj = v3(Vj[0], Vj[1], Vj[2]);
        const V3 th = mul(c.dq_dbg, v3(Bgi[0], Bgi[1], Bgi[2]) - c.lin_bg);
        const Q4 cq = qmul(c.dq, q4(th.x / 2, th.y / 2, th.z / 2, 1.0));
        put3(J, 0, 4, qmat(Qi_inv), -1.0);
        put3(J, 0, 0, skew(qrot(Qi_inv, ((g * 0.5) * dt) * dt + Pj - Pi - vi * dt)), 1.0);
        put3(J, 3, 0, left_right_br(qmul(qinv(Qj), Qi), cq), -1.0);
        put3(J, 6, 0, skew(qrot(Qi_inv, g * dt + vj - vi)), 1.0);
    } else if (blk == 1) {     // v_i (:54-61)
        const M3 Ri_inv = qmat(Qi_inv);
        put3(J, 0, 7, Ri_inv, -dt); put3(J, 6, 7, Ri_inv, -1.0);
    } else if (blk == 2) {     // ba_i (:62-70)
        put3(J, 0, 10, c.dp_dba, -1.0); put3(J, 6, 10, c.dv_dba, -1.0); put3(J, 9, 10, I, -1.0);
    } else if (blk == 3) {     // bg_i (:71-80)
        put3(J, 0, 13, c.dp_dbg, -1.0);
        put3(J, 3, 13, mul(left_br(qmul(qmul(qinv(Qj), Qi), c.dq)), c.dq_dbg), -1.0);
        put3(J, 6, 13, c.dv_dbg, -1.0); put3(J, 12, 13, I, -1.0);
    } else if (blk == 4) {     // pose_j (:81-89)
        const V3 th = mul(c.dq_dbg, v3(Bgi[0], Bgi[1], Bgi[2]) - c.lin_bg);
        const Q4 cq = qmul(c.dq, q4(th.x / 2, th.y / 2, th.z / 2, 1.0));
        put3(J, 0, 20, qmat(Qi_inv), 1.0);
        put3(J, 3, 16, left_br(qmul(qmul(qinv(cq), Qi_inv), Qj)), 1.0);
    } else if (blk == 5) {     // v_j (:90-96)
        put3(J, 6, 23, qmat(Qi_inv), 1.0);
    } else if (blk == 6) {     // ba_j (:97-103)
        put3(J, 9, 26, I, 1.0);
    } else {                   // bg_j (:104-110)
        put3(J, 12, 29, I, 1.0);
    }
}
LVB_HD void imu_raw_jacobian(const ImuConst& c, const double* Ti, const double* Vi, const double* Bgi,
                             const double* Tj, const double* Vj, double* J /*15x32, pre-zeroed*/) {
    for (int blk = 0; blk < 8; ++blk) imu_raw_jacobian_block(c, blk, Ti, Vi, Bgi, Tj, Vj, J);
}

// sqrt_info = LLT(cov^-1).matrixL()^T (imu_error.hpp:32): partial-pivot LU inverse, then Cholesky.
// Same operation order as the oracle so that the two agree to rounding.  Returns 0 on success.
LVB_HD int sqrt_information(const double* cov /*225*/, double* U /*225*/, double* a /*225 scratch*/, double* inv /*225 scratch*/, double prior_a = -1.0, double prior_g = -1.0) {
    const int n = 15;
    int piv[15];
    for (int i = 0; i < 225; ++i) a[i] = cov[i];
    for (int i = 0; i < n; ++i) piv[i] = i;
    for (int k = 0; k < n; ++k) {
        int best = k; double bv = fabs(a[k * n + k]);
        for (int i = k + 1; i < n; ++i) if (fabs(a[i * n + k]) > bv) { bv = fabs(a[i * n + k]); best = i; }
        if (bv == 0.0) return 1;
        if (best != k) { for (int j = 0; j < n; ++j) { const double t = a[k * n + j]; a[k * n + j] = a[best * n + j]; a[best * n + j] = t; } const int t = piv[k]; piv[k] = piv[best]; piv[best] = t; }
        for (int i = k + 1; i < n; ++i) { a[i * n + k] /= a[k * n + k]; const double f = a[i * n + k]; for (int j = k + 1; j < n; ++j) a[i * n + j] -= f * a[k * n + j]; }
    }
    for (int c = 0; c < n; ++c) {
        double y[15];
        for (int i = 0; i < n; ++i) { double s = (piv[i] == c) ? 1.0 : 0.0; for (int k = 0; k < i; ++k) s -= a[i * n + k] * y[k]; y[i] = s; }
        for (int i = n - 1; i >= 0; --i) { double s = y[i]; for (int k = i + 1; k < n; ++k) s -= a[i * n + k] * inv[k * n + c]; inv[i * n + c] = s / a[i * n + i]; }
    }
    if (prior_a >= 0.0 && prior_g >= 0.0)      // ImuInitError (imu_error.hpp:147-149): bias blocks of cov^-1 replaced by the priors
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { inv[(9 + i) * n + 9 + j] = (i == j) ? prior_a : 0.0; inv[(12 + i) * n + 12 + j] = (i == j) ? prior_g : 0.0; }
    for (int i = 0; i < 225; ++i) a[i] = 0.0;   // a := L
    for (int j = 0; j < n; ++j) {
        double d = inv[j * n + j];
        for (int k = 0; k < j; ++k) d -= a[j * n + k] * a[j * n + k];
        if (d != d) return 2;
        if (d <= 0.0) {      // Eigen's LLT stops here and matrixL() shows the untouched lower triangle from this column on (oracle/imu.h)
            for (int c = j; c < n; ++c) for (int i = c; i < n; ++i) a[i * n + c] = inv[i * n + c];
            break;
        }
        a[j * n + j] = sqrt(d);
        for (int i = j + 1; i < n; ++i) { double s = inv[i * n + j]; for (int k = 0; k < j; ++k) s -= a[i * n + k] * a[j * n + k]; a[i * n + j] = s / a[j * n + j]; }
    }
    for (int i = 0; i < n; ++i) for (int j = 0; j < n; ++j) U[i * n + j] = a[j * n + i];
    return 0;
}

// ---------------------------------------------------------------------------------------
// a5 LidarPlaneErrorRPZ / YXY (lidar_error.hpp:48-63, 83-98), hoisted form.
// Per solve iteration the point-independent part is computed once (IcpFrame); per point the
// residual is w n.(R2 p + t2 - pa) and the three Jacobian entries are dot products.
// rpyxyz = [yaw pitch roll x y z]; R_rel = Rz(yaw) Ry(pitch) Rx(roll) (base.hpp:110-121).
// ---------------------------------------------------------------------------------------
struct IcpFrame {
    M3 R2; V3 t2;       // Twc2 = Twc1 * se3(rpyxyz)
    M3 dR[3];           // d(R2)/d(free angle k) (zero matrix for translation parameters)
    V3 dt[3];           // d(t2)/d(free translation k) (zero for angles)
};
LVB_HD M3 rz(double a) { M3 r; const double c = cos(a), s = sin(a); r.m[0] = c; r.m[1] = -s; r.m[2] = 0; r.m[3] = s; r.m[4] = c; r.m[5] = 0; r.m[6] = 0; r.m[7] = 0; r.m[8] = 1; return r; }
LVB_HD M3 ry(double a) { M3 r; const double c = cos(a), s = sin(a); r.m[0] = c; r.m[1] = 0; r.m[2] = s; r.m[3] = 0; r.m[4] = 1; r.m[5] = 0; r.m[6] = -s; r.m[7] = 0; r.m[8] = c; return r; }
LVB_HD M3 rx(double a) { M3 r; const double c = cos(a), s = sin(a); r.m[0] = 1; r.m[1] = 0; r.m[2] = 0; r.m[3] = 0; r.m[4] = c; r.m[5] = -s; r.m[6] = 0; r.m[7] = s; r.m[8] = c; return r; }
LVB_HD M3 drz(double a) { M3 r; const double c = cos(a), s = sin(a); r.m[0] = -s; r.m[1] = -c; r.m[2] = 0; r.m[3] = c; r.m[4] = -s; r.m[5] = 0; r.m[6] = 0; r.m[7] = 0; r.m[8] = 0; return r; }
LVB_HD M3 dry(double a) { M3 r; const double c = cos(a), s = sin(a); r.m[0] = -s; r.m[1] = 0; r.m[2] = c; r.m[3] = 0; r.m[4] = 0; r.m[5] = 0; r.m[6] = -c; r.m[7] = 0; r.m[8] = -s; return r; }
LVB_HD M3 drx(double a) { M3 r; const double c = cos(a), s = sin(a); r.m[0] = 0; r.m[1] = 0; r.m[2] = 0; r.m[3] = 0; r.m[4] = -s; r.m[5] = -c; r.m[6] = 0; r.m[7] = c; r.m[8] = -s; return r; }

LVB_HD IcpFrame icp_frame(int mode, const double* Twc1, const double* e /*rpyxyz with free entries substituted*/) {
    const M3 R1 = rot_matrix(unit_quat(Twc1));
    const M3 Z = rz(e[0]), Y = ry(e[1]), X = rx(e[2]);
    const M3 Rrel = mul(Z, mul(Y, X));
    IcpFrame f;
    f.R2 = mul(R1, Rrel);
    f.t2 = mul(R1, v3(e[3], e[4], e[5])) + v3(Twc1[4], Twc1[5], Twc1[6]);
    M3 zero; for (int i = 0; i < 9; ++i) zero.m[i] = 0;
    const V3 z3 = v3(0, 0, 0);
    const V3 c0 = v3(R1.m[0], R1.m[3], R1.m[6]), c1 = v3(R1.m[1], R1.m[4], R1.m[7]), c2 = v3(R1.m[2], R1.m[5], R1.m[8]);
    if (mode == 0) {      // free = pitch, roll, z
        f.dR[0] = mul(R1, mul(Z, mul(dry(e[1]), X))); f.dt[0] = z3;
        f.dR[1] = mul(R1, mul(Z, mul(Y, drx(e[2])))); f.dt[1] = z3;
        f.dR[2] = zero; f.dt[2] = c2;
    } else {              // free = yaw, x, y
        f.dR[0] = mul(R1, mul(drz(e[0]), mul(Y, X))); f.dt[0] = z3;
        f.dR[1] = zero; f.dt[1] = c0;
        f.dR[2] = zero; f.dt[2] = c1;
    }
    return f;
}
LVB_HD double icp_point(const IcpFrame& f, const V3& p, const V3& pa, const V3& n, double w, double* J /*3 or null*/) {
    const V3 lp = mul(f.R2, p) + f.t2;
    const double r = w * dot(lp - pa, n);
    if (J) for (int k = 0; k < 3; ++k) J[k] = w * (dot(mul(f.dR[k], p), n) + dot(f.dt[k], n));
    return r;
}
// LidarPlaneError ctor (lidar_error.hpp:13-18): n = normalize((pa-pb) x (pa-pc)), unguarded
LVB_HD V3 plane_normal(const V3& pa, const V3& pb, const V3& pc) {
    const V3 n = cross(pa - pb, pa - pc);
    const double len = sqrt(n.x * n.x + n.y * n.y + n.z * n.z);
    return v3(n.x / len, n.y / len, n.z / len);
}

}  // namespace lvb
