"""Seeded synthetic KITTI-shaped inputs for the hot path (SURVEY.md section 8d).

All constants come from /root/reference/src/lvio_fusion_node/config/kitti.yaml (camera
intrinsics :23-32, body_to_cam0/1 :55-72, lidar resolution :45, imu noise :48-52) and
src/frame.cpp:11-16 (default weights).  numpy only -- this module builds *inputs*; it never
evaluates a factor.
"""
import numpy as np

SEED = 0x4C56494F
FX = FY = 718.856
CX, CY = 607.1928, 185.2157
IMG_W, IMG_H = 1241.0, 376.0
W_VISUAL = FX / 10.0          # frame.cpp:13
W_LIDAR_GROUND = 1.0          # frame.cpp:14
W_LIDAR_SURF = 0.01           # frame.cpp:15
LIDAR_RESOLUTION = 0.2        # kitti.yaml:45
IMU_NOISE = np.array([0.1, 0.01, 0.001, 1.0e-4])  # ACC_N GYR_N ACC_W GYR_W kitti.yaml:48-51
GRAVITY = np.array([0.0, 0.0, 9.81007])           # preintegration.cpp:13

_B2C0 = np.array([[0.00875117, -0.00479608, 0.99995, 1.10224],
                  [-0.999865, -0.0140025, 0.00868325, -0.319072],
                  [0.0139602, -0.999891, -0.00491796, 0.746066]])
_B2C1 = np.array([[0.00875117, -0.00479608, 0.99995, 1.10695],
                  [-0.999865, -0.0140025, 0.00868325, -0.856165],
                  [0.0139602, -0.999891, -0.00491796, 0.753565]])


# ------------------------------------------------------------------ quaternion helpers (xyzw)
def quat_from_matrix(R):
    R = np.asarray(R, dtype=np.float64)
    t = np.trace(R)
    if t > 0:
        s = np.sqrt(t + 1.0) * 2
        q = np.array([(R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s, 0.25 * s])
    else:
        i = int(np.argmax(np.diag(R)))
        j, k = (i + 1) % 3, (i + 2) % 3
        s = np.sqrt(1.0 + R[i, i] - R[j, j] - R[k, k]) * 2
        q = np.zeros(4)
        q[i] = 0.25 * s
        q[j] = (R[j, i] + R[i, j]) / s
        q[k] = (R[k, i] + R[i, k]) / s
        q[3] = (R[k, j] - R[j, k]) / s
    return q / np.linalg.norm(q)


def quat_to_matrix(q):
    q = np.asarray(q, dtype=np.float64)
    x, y, z, w = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    R = np.empty(q.shape[:-1] + (3, 3))
    R[..., 0, 0] = 1 - 2 * (y * y + z * z); R[..., 0, 1] = 2 * (x * y - z * w); R[..., 0, 2] = 2 * (x * z + y * w)
    R[..., 1, 0] = 2 * (x * y + z * w); R[..., 1, 1] = 1 - 2 * (x * x + z * z); R[..., 1, 2] = 2 * (y * z - x * w)
    R[..., 2, 0] = 2 * (x * z - y * w); R[..., 2, 1] = 2 * (y * z + x * w); R[..., 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def quat_mul(a, b):
    ax, ay, az, aw = a[..., 0], a[..., 1], a[..., 2], a[..., 3]
    bx, by, bz, bw = b[..., 0], b[..., 1], b[..., 2], b[..., 3]
    return np.stack([aw * bx + ax * bw + ay * bz - az * by,
                     aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw,
                     aw * bw - ax * bx - ay * by - az * bz], axis=-1)


def quat_from_rotvec(v):
    v = np.asarray(v, dtype=np.float64)
    ang = np.linalg.norm(v, axis=-1, keepdims=True)
    half = 0.5 * ang
    k = np.where(ang > 1e-12, np.sin(half) / np.maximum(ang, 1e-300), 0.5)
    return np.concatenate([k * v, np.cos(half)], axis=-1)


def quat_from_yaw(yaw):
    yaw = np.asarray(yaw, dtype=np.float64)
    z = np.zeros_like(yaw)
    return np.stack([z, z, np.sin(yaw / 2), np.cos(yaw / 2)], axis=-1)


def se3_apply(T, p):
    """T: [...,7] pose(s), p: [...,3]."""
    return np.einsum("...ij,...j->...i", quat_to_matrix(T[..., :4]), p) + T[..., 4:]


def se3_inv_apply(T, p):
    return np.einsum("...ji,...j->...i", quat_to_matrix(T[..., :4]), p - T[..., 4:])


def kitti_cameras():
    """cam[22] = 2 x {fx fy cx cy, T_body_cam[7]} (lvb_ba_set_cameras)."""
    out = []
    for M in (_B2C0, _B2C1):
        q = quat_from_matrix(M[:, :3])
        out += [FX, FY, CX, CY] + list(q) + list(M[:, 3])
    return np.array(out, dtype=np.float64)


def _rng(seed, stream):
    return np.random.Generator(np.random.PCG64([int(seed), int(stream)]))


# ------------------------------------------------------------------ trajectory
class Trajectory:
    """Planar clothoid-like path: speed 10 m/s, curvature kmax*sin(2 pi s / period), z = 0,
    body x forward / z up.  Sampled at 1 kHz; keyframes every 1.0 m (0.1 s)."""

    def __init__(self, n_kf, speed=10.0, spacing=1.0, kmax=0.02, period=200.0):
        self.speed, self.dt_kf = speed, spacing / speed
        self.n_kf = n_kf
        self.h = 1e-3
        n = int(round((n_kf - 1) * self.dt_kf / self.h)) + 1
        t = np.arange(n + 20) * self.h
        s = speed * t
        w = 2 * np.pi / period
        self.t = t
        self.kappa = kmax * np.sin(w * s)
        self.psi = kmax / w * (1 - np.cos(w * s))
        vel = speed * np.stack([np.cos(self.psi), np.sin(self.psi), np.zeros_like(s)], axis=1)
        pos = np.zeros_like(vel)
        pos[1:] = np.cumsum(0.5 * (vel[1:] + vel[:-1]) * self.h, axis=0)
        self.pos, self.vel = pos, vel
        self.acc = speed * speed * self.kappa[:, None] * np.stack([-np.sin(self.psi), np.cos(self.psi), np.zeros_like(s)], axis=1)
        self.gyr_z = speed * self.kappa
        self.kf_step = int(round(self.dt_kf / self.h))

    def kf_index(self, k):
        return k * self.kf_step

    def poses(self):
        i = np.arange(self.n_kf) * self.kf_step
        return np.concatenate([quat_from_yaw(self.psi[i]), self.pos[i]], axis=1)

    def velocities(self):
        return self.vel[np.arange(self.n_kf) * self.kf_step].copy()

    def imu_samples(self, k, rate_hz=100.0):
        """IMU samples (dt, acc[3], gyr[3]) covering (kf k-1, kf k], plus the sample at kf k-1."""
        step = int(round(1.0 / rate_hz / self.h))
        i0 = self.kf_index(k - 1)
        idx = i0 + step * np.arange(0, self.kf_step // step + 1)
        R = quat_to_matrix(quat_from_yaw(self.psi[idx]))
        acc = np.einsum("nji,nj->ni", R, self.acc[idx] + GRAVITY)
        gyr = np.stack([np.zeros(len(idx)), np.zeros(len(idx)), self.gyr_z[idx]], axis=1)
        return step * self.h, acc, gyr


# ------------------------------------------------------------------ IMU preintegration (producer)
def _skew(v):
    z = np.zeros(v.shape[:-1])
    return np.stack([np.stack([z, -v[..., 2], v[..., 1]], -1),
                     np.stack([v[..., 2], z, -v[..., 0]], -1),
                     np.stack([-v[..., 1], v[..., 0], z], -1)], -2)


def preintegrate_batch(dt, acc, gyr, ba, bg, noise4=IMU_NOISE):
    """Midpoint preintegration of F factors at once (preintegration.cpp:30-127 semantics).

    acc, gyr: [F, S+1, 3] (sample 0 is the seed acc0/gyr0); ba, bg: [F,3].
    Returns the LVB_IMU const records [F, 469] (prior_a = prior_g = -1: plain ImuError).
    """
    F, S1, _ = acc.shape
    dp = np.zeros((F, 3)); dv = np.zeros((F, 3)); dq = np.tile(np.array([0, 0, 0, 1.0]), (F, 1))
    jac = np.tile(np.eye(15), (F, 1, 1)); cov = np.zeros((F, 15, 15))
    nz = np.concatenate([np.full(3, noise4[0] ** 2), np.full(3, noise4[1] ** 2), np.full(3, noise4[0] ** 2),
                         np.full(3, noise4[1] ** 2), np.full(3, noise4[2] ** 2), np.full(3, noise4[3] ** 2)])
    I3 = np.tile(np.eye(3), (F, 1, 1))
    sum_dt = 0.0
    for s in range(1, S1):
        a0, g0, a1, g1 = acc[:, s - 1], gyr[:, s - 1], acc[:, s], gyr[:, s]
        Rd = quat_to_matrix(dq)
        un_acc_0 = np.einsum("fij,fj->fi", Rd, a0 - ba)
        un_gyr = 0.5 * (g0 + g1) - bg
        rq = quat_mul(dq, np.concatenate([un_gyr * dt / 2, np.ones((F, 1))], axis=1))
        Rr = quat_to_matrix(rq / np.linalg.norm(rq, axis=1, keepdims=True))
        # the reference rotates with the un-normalised result_delta_q through Eigen's unit-quaternion
        # formula; the difference is O(|un_gyr dt|^2/4) ~ 1e-9 and irrelevant for an input producer.
        un_acc_1 = np.einsum("fij,fj->fi", Rr, a1 - ba)
        un_acc = 0.5 * (un_acc_0 + un_acc_1)
        ndp = dp + dv * dt + 0.5 * un_acc * dt * dt
        ndv = dv + un_acc * dt
        Rw, Ra0, Ra1 = _skew(un_gyr), _skew(a0 - ba), _skew(a1 - ba)
        ImW = I3 - Rw * dt
        Fm = np.zeros((F, 15, 15)); V = np.zeros((F, 15, 18))
        Fm[:, 0:3, 0:3] = I3
        Fm[:, 0:3, 3:6] = -0.25 * Rd @ Ra0 * dt * dt - 0.25 * Rr @ Ra1 @ ImW * dt * dt
        Fm[:, 0:3, 6:9] = I3 * dt
        Fm[:, 0:3, 9:12] = -0.25 * (Rd + Rr) * dt * dt
        Fm[:, 0:3, 12:15] = 0.25 * Rr @ Ra1 * dt * dt * dt
        Fm[:, 3:6, 3:6] = ImW
        Fm[:, 3:6, 12:15] = -I3 * dt
        Fm[:, 6:9, 3:6] = -0.5 * Rd @ Ra0 * dt - 0.5 * Rr @ Ra1 @ ImW * dt
        Fm[:, 6:9, 6:9] = I3
        Fm[:, 6:9, 9:12] = -0.5 * (Rd + Rr) * dt
        Fm[:, 6:9, 12:15] = 0.5 * Rr @ Ra1 * dt * dt
        Fm[:, 9:12, 9:12] = I3
        Fm[:, 12:15, 12:15] = I3
        V[:, 0:3, 0:3] = 0.25 * Rd * dt * dt
        V[:, 0:3, 3:6] = -0.125 * Rr @ Ra1 * dt ** 3
        V[:, 0:3, 6:9] = 0.25 * Rr * dt * dt
        V[:, 0:3, 9:12] = V[:, 0:3, 3:6]
        V[:, 3:6, 3:6] = 0.5 * I3 * dt
        V[:, 3:6, 9:12] = 0.5 * I3 * dt
        V[:, 6:9, 0:3] = 0.5 * Rd * dt
        V[:, 6:9, 3:6] = -0.25 * Rr @ Ra1 * dt * dt
        V[:, 6:9, 6:9] = 0.5 * Rr * dt
        V[:, 6:9, 9:12] = V[:, 6:9, 3:6]
        V[:, 9:12, 12:15] = I3 * dt
        V[:, 12:15, 15:18] = I3 * dt
        jac = Fm @ jac
        cov = Fm @ cov @ np.transpose(Fm, (0, 2, 1)) + (V * nz) @ np.transpose(V, (0, 2, 1))
        dp, dv = ndp, ndv
        dq = rq / np.linalg.norm(rq, axis=1, keepdims=True)
        sum_dt += dt
    out = np.zeros((F, 469))
    out[:, 467:] = -1.0
    out[:, 0:3] = dp; out[:, 3:7] = dq; out[:, 7:10] = dv; out[:, 10:13] = ba; out[:, 13:16] = bg; out[:, 16] = sum_dt
    out[:, 17:242] = jac.reshape(F, 225); out[:, 242:467] = cov.reshape(F, 225)
    return out


# ------------------------------------------------------------------ BA problem
def _project(cam, T_wb, pw):
    """pixel + depth of world points pw [n,3] seen from body poses T_wb [n,7] through camera cam[11]."""
    pb = se3_inv_apply(T_wb, pw)
    pc = se3_inv_apply(np.broadcast_to(cam[4:11], pb.shape[:-1] + (7,)), pb)
    z = pc[..., 2]
    return np.stack([cam[0] * pc[..., 0] / z + cam[2], cam[1] * pc[..., 1] / z + cam[3]], axis=-1), z


def make_ba_problem(n_kf, n_landmarks, with_imu=True, seed=SEED, track_len=4, pose_only_frac=0.15,
                    pixel_sigma=0.5, outlier_frac=0.05, sigma_t=0.05, sigma_theta_deg=0.5, with_priors=False):
    """The factor mix Backend::BuildProblem assembles (backend.cpp:96-183) on a synthetic window.

    Returns a dict: cameras[22], poses[N,7] (noisy initial guess), poses_true, vec3[3N,3]
    (v, ba, bg per keyframe; empty without IMU), rho[M], rho_true, factors {kind: (consts, idx)},
    loss {kind: huber_a}.
    """
    rng = _rng(seed, 1)
    cams = kitti_cameras()
    cam0, cam1 = cams[:11], cams[11:]
    traj = Trajectory(n_kf)
    P_true = traj.poses()
    N, M = n_kf, n_landmarks

    # -- landmarks: uniform in the cam0 frustum of the birth keyframe, depth U(5,60)
    birth = rng.integers(0, N, size=M)
    birth.sort()
    u = rng.uniform(20, IMG_W - 20, M); v = rng.uniform(20, IMG_H - 20, M); z = rng.uniform(5, 60, M)
    pc0 = np.stack([(u - CX) / FX * z, (v - CY) / FY * z, z], axis=1)
    pb = se3_apply(np.broadcast_to(cam0[4:11], (M, 7)), pc0)
    pw = se3_apply(P_true[birth], pb)
    pc1 = se3_inv_apply(np.broadcast_to(cam1[4:11], (M, 7)), pb)
    rho_true = 1.0 / pc1[:, 2]
    right_px = np.stack([FX * pc1[:, 0] / pc1[:, 2] + CX, FY * pc1[:, 1] / pc1[:, 2] + CY], axis=1)
    left_px = np.stack([u, v], axis=1)
    right_ob = right_px + rng.normal(0, pixel_sigma, (M, 2))
    left_ob = left_px + rng.normal(0, pixel_sigma, (M, 2))

    # a3 TwoCamera: one per landmark in its birth keyframe, weight 5 * w_visual (backend.cpp:123)
    tc_consts = np.concatenate([left_ob, right_ob, np.full((M, 1), 5 * W_VISUAL)], axis=1)
    tc_idx = np.arange(M, dtype=np.int32)[:, None]

    # a1 TwoFrame: observations in the following track_len-1 keyframes that stay in the image
    lm, kf = [], []
    for d in range(1, track_len):
        k = birth + d
        ok = k < N
        lm.append(np.nonzero(ok)[0]); kf.append(k[ok])
    lm = np.concatenate(lm); kf = np.concatenate(kf)
    px, zc = _project(cam0, P_true[kf], pw[lm])
    ok = (zc > 1.0) & (px[:, 0] > 0) & (px[:, 0] < IMG_W) & (px[:, 1] > 0) & (px[:, 1] < IMG_H)
    lm, kf, px = lm[ok], kf[ok], px[ok]
    ob = px + rng.normal(0, pixel_sigma, px.shape)
    out = rng.random(len(ob)) < outlier_frac
    ob[out] += rng.choice([-20.0, 20.0], size=(int(out.sum()), 2))
    order = np.lexsort((kf, lm))          # landmark-major, the order BuildProblem's map walk is not -- any order is legal
    lm, kf, ob = lm[order], kf[order], ob[order]
    tf_consts = np.concatenate([right_ob[lm], ob, np.full((len(lm), 1), W_VISUAL)], axis=1)
    tf_idx = np.stack([lm, birth[lm], kf], axis=1).astype(np.int32)

    # a2 PoseOnly: older, fixed world points
    n_po = int(round(pose_only_frac / (1 - pose_only_frac) * len(lm)))
    kf2 = rng.integers(0, N, size=n_po)
    u2 = rng.uniform(20, IMG_W - 20, n_po); v2 = rng.uniform(20, IMG_H - 20, n_po); z2 = rng.uniform(5, 60, n_po)
    pc = np.stack([(u2 - CX) / FX * z2, (v2 - CY) / FY * z2, z2], axis=1)
    pw2 = se3_apply(P_true[kf2], se3_apply(np.broadcast_to(cam0[4:11], (n_po, 7)), pc))
    pw2 += rng.normal(0, 0.02, pw2.shape)
    ob2 = np.stack([u2, v2], axis=1) + rng.normal(0, pixel_sigma, (n_po, 2))
    out2 = rng.random(n_po) < outlier_frac
    ob2[out2] += rng.choice([-20.0, 20.0], size=(int(out2.sum()), 2))
    po_consts = np.concatenate([ob2, pw2, np.full((n_po, 1), W_VISUAL)], axis=1)
    po_idx = kf2.astype(np.int32)[:, None]

    # -- initial guess
    P0 = P_true.copy()
    dth = rng.normal(0, np.deg2rad(sigma_theta_deg), (N, 3))
    P0[:, :4] = quat_mul(quat_from_rotvec(dth), P_true[:, :4])
    P0[:, 4:] += rng.normal(0, sigma_t, (N, 3))
    rho0 = np.maximum(rho_true + rng.normal(0, 0.5 / (FX * 0.537), M), 1.0 / 200.0)

    factors = {0: (tf_consts, tf_idx), 1: (po_consts, po_idx), 2: (tc_consts, tc_idx)}
    loss = {0: 1.0, 1: 1.0, 2: 1.0}       # HuberLoss(1.0) on the visual kinds (backend.cpp:98)
    vec3 = np.zeros((0, 3)); vec3_true = np.zeros((0, 3))
    if with_imu and N > 1:
        vel = traj.velocities()
        vec3_true = np.zeros((3 * N, 3)); vec3_true[0::3] = vel
        vec3 = vec3_true.copy()
        vec3[0::3] += rng.normal(0, 0.05, (N, 3))
        vec3[1::3] += rng.normal(0, 0.01, (N, 3))      # ba guess
        vec3[2::3] += rng.normal(0, 0.001, (N, 3))     # bg guess
        accs, gyrs = [], []
        for k in range(1, N):
            dt, a, g = traj.imu_samples(k)
            accs.append(a + rng.normal(0, IMU_NOISE[0] * 0.1, a.shape)); gyrs.append(g + rng.normal(0, IMU_NOISE[1] * 0.1, g.shape))
        accs = np.stack(accs); gyrs = np.stack(gyrs)
        imu_consts = preintegrate_batch(dt, accs, gyrs, np.zeros((N - 1, 3)), np.zeros((N - 1, 3)))
        i = np.arange(N - 1); j = i + 1
        imu_idx = np.stack([i, 3 * i, 3 * i + 1, 3 * i + 2, j, 3 * j, 3 * j + 1, 3 * j + 2], axis=1).astype(np.int32)
        factors[3] = (imu_consts, imu_idx)
    if with_priors:
        # weak-constraint priors (backend.cpp:165-178): PoseError on kf 0, PoseGraphError(100,0) chain
        factors[5] = (np.concatenate([P0[0], [100.0, 0.0]])[None, :], np.zeros((1, 1), dtype=np.int32))
    return dict(cameras=cams, poses=P0, poses_true=P_true, vec3=vec3, vec3_true=vec3_true, rho=rho0, rho_true=rho_true,
                factors=factors, loss=loss, n_kf=N, n_landmarks=M)


def make_fullba_problem(n_kf, n_landmarks, prior_a=1e8, prior_g=1e8, seed=SEED):
    """imu::FullBA (tools.cpp:92-171): the visual factor mix of the window plus ImuInitError factors
    (imu_error.hpp:124-229) that all share ONE accelerometer-bias and ONE gyroscope-bias block.

    The reference calls it with prior_a = 1e4, prior_g = 1e2 (initializer.cpp:62); with the kitti.yaml IMU noise
    those values make the patched cov^-1 indefinite and Eigen's LLT returns early (DESIGN.md section 7; the
    backend reproduces that factor).  The default here keeps the matrix positive definite; pass the reference's
    values to exercise the other path."""
    d = make_ba_problem(n_kf, n_landmarks, with_imu=True, seed=seed)
    N = n_kf
    consts, _ = d["factors"][3]
    consts = consts.copy()
    consts[:, 467] = prior_a
    consts[:, 468] = prior_g
    vel = d["vec3"][0::3]
    vec3 = np.concatenate([vel, d["vec3"][1:3]], axis=0)            # v_0..v_{N-1}, ba, bg
    i = np.arange(N - 1); j = i + 1
    idx = np.stack([i, i, np.full(N - 1, N), np.full(N - 1, N + 1), j, j, np.full(N - 1, -1), np.full(N - 1, -1)], axis=1).astype(np.int32)
    d = dict(d)
    d["factors"] = dict(d["factors"])
    d["factors"][3] = (consts, idx)
    d["vec3"] = vec3
    d["vec3_true"] = np.concatenate([d["vec3_true"][0::3], d["vec3_true"][1:3]], axis=0)
    return d


def count_rows(d):
    res = [2, 2, 2, 15, 6, 6]
    return sum(len(f[0]) * res[k] for k, f in d["factors"].items())


def count_blocks(d):
    return sum(len(f[0]) for f in d["factors"].values())


def shard_ba_problem(d, rank, world):
    """Partition by landmark (SURVEY 8e): every block touching rho_l lives on rank l % world;
    pose-only / IMU / prior blocks are dealt round-robin.  Parameter blocks stay replicated."""
    out = dict(d)
    fac = {}
    for kind, (c, ix) in d["factors"].items():
        if kind in (0, 2):
            keep = (ix[:, 0] % world) == rank
        else:
            keep = (np.arange(len(c)) % world) == rank
        fac[kind] = (c[keep], ix[keep])
    out["factors"] = fac
    return out


# ------------------------------------------------------------------ lidar scene
def _sample_surfaces(rng, n, center, radius, ground_frac, wall_every=20.0, z_max=6.0):
    """Points on the ground plane z=0 and on axis-aligned walls every wall_every metres."""
    ng = int(n * ground_frac)
    nw = n - ng
    g = np.stack([rng.uniform(-radius, radius, ng) + center[0], rng.uniform(-radius, radius, ng) + center[1], np.zeros(ng)], axis=1)
    along = rng.uniform(-radius, radius, nw)
    height = rng.uniform(0.0, z_max, nw)
    which = rng.integers(0, 2, nw)
    lines = np.round((center[which] + rng.uniform(-radius, radius, nw)) / wall_every) * wall_every
    w = np.where(which[:, None] == 0,
                 np.stack([lines, center[1] + along, height], axis=1),
                 np.stack([center[0] + along, lines, height], axis=1))
    return g, w


def make_icp_problem(n_scan, n_map, seed=SEED, radius=30.0, min_range=5.0, sigma=0.02, kind="surf", stride_floats=4):
    """One ScanToMapWith{Ground,Segmented} call (association.cpp:270-384) on a synthetic scene:
    ground plane + walls every 20 m; map cloud in the world frame, scan in the robot frame with an
    initial pose error (yaw 1 deg, xy 0.2 m, z 0.05 m, roll/pitch 0.3 deg).

    kind = 'ground' (mode 0: pitch/roll/z, gate d2 < 100 res^2, TrivialLoss, weight 1) or
    'surf' (mode 1: yaw/x/y, gate d2 < 25 res^2, Huber 0.1, weight 0.01).
    """
    rng = _rng(seed, 7 if kind == "surf" else 8)
    center = np.array([3.0, -2.0])
    gmap, wmap = _sample_surfaces(rng, n_map, center, radius, 1.0 if kind == "ground" else 0.0)
    map_pts = gmap if kind == "ground" else wmap
    map_pts = map_pts + rng.normal(0, sigma, map_pts.shape)
    if kind == "ground":
        map_pts[:, 2] = rng.normal(0, sigma, len(map_pts))
    # true robot pose (lidar frame folded into body for the synthetic case)
    true_pose = np.concatenate([quat_from_yaw(np.array(0.3)), [center[0], center[1], 1.7]])
    gs, ws = _sample_surfaces(rng, int(n_scan * 1.6) + 64, center, radius, 1.0 if kind == "ground" else 0.0)
    scan_w = gs if kind == "ground" else ws
    rng_xy = np.linalg.norm(scan_w[:, :2] - center, axis=1)
    scan_w = scan_w[(rng_xy > min_range) & (rng_xy < radius)][:n_scan]
    assert len(scan_w) == n_scan, "not enough scan points in range"
    scan_w = scan_w + rng.normal(0, sigma, scan_w.shape)
    scan_b = se3_inv_apply(np.broadcast_to(true_pose, (n_scan, 7)), scan_w)
    # map frame pose (newest of the merged frames, mapping.cpp:131-133): one metre behind
    map_pose = np.concatenate([quat_from_yaw(np.array(0.28)), [center[0] - 1.0, center[1] - 0.3, 1.7]])
    # initial guess = true pose perturbed
    dq = quat_from_rotvec(np.deg2rad(np.array([0.3, -0.3, 1.0])))
    guess = np.concatenate([quat_mul(dq, true_pose[:4]), true_pose[4:] + np.array([0.2, -0.2, 0.05])])
    res2 = LIDAR_RESOLUTION * LIDAR_RESOLUTION
    cfg = dict(mode=0, thr=res2 * 100, huber_a=0.0, weight=W_LIDAR_GROUND) if kind == "ground" else \
        dict(mode=1, thr=res2 * 25, huber_a=0.1, weight=W_LIDAR_SURF)

    def pack(p):
        out = np.zeros((len(p), stride_floats), dtype=np.float32)
        out[:, :3] = p.astype(np.float32)
        return out
    return dict(map=pack(map_pts), scan=pack(scan_b), true_pose=true_pose, map_pose=map_pose, frame_pose=guess,
                cell_size=float(np.float32(np.sqrt(cfg["thr"])) * np.float32(1.0001)), n_features_left=150, **cfg)


def relative_rpyxyz(map_pose, frame_pose):
    """se32rpyxyz(map_pose^-1 * frame_pose) (mapping.cpp:154, utility.cpp:27-33), numpy float64."""
    Rm = quat_to_matrix(map_pose[:4]); Rf = quat_to_matrix(frame_pose[:4])
    R = Rm.T @ Rf
    t = Rm.T @ (frame_pose[4:] - map_pose[4:])
    q = quat_from_matrix(R)
    q1, q2, q3, q0 = q
    yaw = np.arctan2(2 * (q1 * q2 + q0 * q3), 1 - 2 * (q2 * q2 + q3 * q3))
    pitch = np.arcsin(2 * (q0 * q2 - q1 * q3))
    roll = np.arctan2(2 * (q2 * q3 + q0 * q1), 1 - 2 * (q1 * q1 + q2 * q2))
    return np.array([yaw, pitch, roll, t[0], t[1], t[2]])


def rpyxyz2se3(e):
    """rpyxyz2se3 (utility.cpp:35-40): RPYToEigenQuaternion (ceres/base.hpp:110-132), normalised as Sophus stores it."""
    cz, sz = np.cos(e[0] / 2), np.sin(e[0] / 2)
    cy, sy = np.cos(e[1] / 2), np.sin(e[1] / 2)
    cx, sx = np.cos(e[2] / 2), np.sin(e[2] / 2)
    q = np.array([cz * cy * sx - sz * sy * cx, cz * sy * cx + sz * cy * sx, sz * cy * cx - cz * sy * sx, cz * cy * cx + sz * sy * sx])
    return np.concatenate([q / np.linalg.norm(q), e[3:6]])


def se3_mul(a, b):
    """Sophus SE3 product a * b of two poses [qx qy qz qw tx ty tz]."""
    q = quat_mul(a[:4], b[:4])
    return np.concatenate([q / np.linalg.norm(q), se3_apply(a, b[4:])])


def se3_inv(a):
    """Sophus SE3 inverse of a pose [qx qy qz qw tx ty tz]."""
    q = np.array([-a[0], -a[1], -a[2], a[3]]) / np.linalg.norm(a[:4])
    return np.concatenate([q, se3_inv_apply(a, np.zeros(3))])


def make_lidar_scan(seed=SEED, num_scans=64, horizon_scan=1800, ang_res_y=0.427, ang_bottom=24.9, sensor_height=1.73,
                    sigma=0.01, dropout=0.02, n_boxes=14):
    """One revolution of a KITTI-like 64-beam spinning lidar (kitti.yaml:35-42) in the sensor frame (z up).

    Scene: ground plane, a 44 m x 26 m walled yard, axis-aligned boxes (cars / poles) on the ground.  Rays are fired column by
    column (all beams of one azimuth, azimuth decreasing so that the reference's orientation -atan2(y, x) increases through
    the sweep), range noise sigma, a fraction of returns dropped (NaN, as the driver reports no-returns) and everything
    outside the walls missing.  Returns float32 [n, 4] (x, y, z, 0) = pcl::PointXYZ records with a 16-byte stride.
    """
    rng = _rng(seed, 7)
    az0 = rng.uniform(-np.pi, np.pi)
    az = az0 - 2 * np.pi * (np.arange(horizon_scan) + rng.uniform(-0.2, 0.2, horizon_scan)) / horizon_scan
    el = np.deg2rad(-ang_bottom + ang_res_y * (np.arange(num_scans) + 0.5))
    A, E = np.meshgrid(az, el, indexing="ij")            # column-major firing order
    d = np.stack([np.cos(E) * np.cos(A), np.cos(E) * np.sin(A), np.sin(E)], axis=-1).reshape(-1, 3)
    t_best = np.full(len(d), np.inf)
    # ground z = -h
    with np.errstate(divide="ignore", invalid="ignore"):
        t = -sensor_height / d[:, 2]
        t_best = np.where((t > 0) & (t < t_best), t, t_best)
        # walls
        for axis, val in ((0, 22.0), (0, -22.0), (1, 13.0), (1, -13.0)):
            t = val / d[:, axis]
            t_best = np.where((t > 0) & (t < t_best), t, t_best)
        # boxes: slab test
        for _ in range(n_boxes):
            c = np.array([rng.uniform(-18, 18), rng.uniform(-10, 10)])
            if np.linalg.norm(c) < 6.0:
                c = c / max(np.linalg.norm(c), 1e-3) * 7.0
            half = np.array([rng.uniform(0.15, 2.2), rng.uniform(0.15, 1.0)])
            height = rng.uniform(1.2, 2.5)
            lo = np.array([c[0] - half[0], c[1] - half[1], -sensor_height])
            hi = np.array([c[0] + half[0], c[1] + half[1], -sensor_height + height])
            t1, t2 = lo / d, hi / d
            tn = np.minimum(t1, t2).max(axis=1); tf = np.maximum(t1, t2).min(axis=1)
            hit = (tn > 0) & (tn <= tf)
            t_best = np.where(hit & (tn < t_best), tn, t_best)
    t_best = t_best + rng.normal(0, sigma, len(d))
    pts = d * t_best[:, None]
    drop = rng.uniform(size=len(d)) < dropout
    pts[drop | ~np.isfinite(t_best)] = np.nan
    out = np.zeros((len(d), 4), dtype=np.float32)
    out[:, :3] = pts
    return out
