/*
 * oracle/aba_oracle.c -- CPU restatement of the articulated-body step.  TEST INFRASTRUCTURE ONLY.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * load this library; the product path (isaacgymenvs_b200/csrc) never does.
 *
 * PARITY UNPINNED against the reference: the function this restates, `gym.simulate(sim)`
 * (call sites isaacgymenvs/ of the reference/tasks/base/vec_task.py:379-382 and
 * tasks/anymal_terrain.py:448), lives in the closed Isaac Gym Preview 4 / PhysX binary, which is
 * absent from the reference checkout and cannot be installed here (SURVEY.md 8c).  The reference holds no
 * golden vectors for it.  What this file pins instead is the algorithm BASELINE.json's north_star
 * prescribes -- Featherstone ABA, PD/effort actuators, semi-implicit Euler, penalty contact -- and
 * it is itself pinned by (tests/test_oracle_physics.py) an independent numpy RNEA inverse-dynamics
 * check, momentum/energy invariants and closed-form cases (free fall, pendulum).
 *
 * Formulation: textbook body-coordinate ABA (Featherstone, "Rigid Body Dynamics Algorithms",
 * Table 7.1, floating base per 9.4).  Spatial vectors are [angular; linear] in LINK coordinates;
 * 6x6 matrices are stored dense.  The CUDA engine deliberately uses a different formulation
 * (world-aligned axes about the root origin, symmetric packed inertias), so agreement between the
 * two is a check of both, not a tautology.
 *
 * Discrete scheme (DESIGN.md "time stepping"), per sub-step h = dt/substeps:
 *   joint force   f_j = clamp(tau_act) - b*qd' - k*(q' - 0) + PD(kp,kd; target) + limit spring,
 *                 all linear terms taken at the END of the sub-step (q' = q + h*qd', qd' = qd + h*qdd)
 *                 => explicit part evaluated at (q + h*qd, qd) and  h*(b+kd+d_lim) + h^2*(k+kp+k_lim)
 *                 added to the joint-space diagonal next to the armature;
 *   contact       sphere vs plane z=0, F = F0(u) - h*G*(J a) with G = diag(gam,gam,cn+h*kn): the
 *                 normal spring/damper and the regularised Coulomb friction are linearised about the
 *                 current contact-point velocity u and folded into the link's articulated inertia;
 *   integration   qd += h*qdd; q += h*qd;  root twist likewise, quaternion by the exponential map.
 *
 * Build: see oracle/Makefile (gcc -O2 -fPIC -shared; -DORACLE_F32 gives the float build, which
 * bench.py times as the "port" CPU baseline and tests use to bound fp32 round-off).
 */
#include <math.h>
#include <string.h>
#include <stdlib.h>
#include <pthread.h>

#ifdef ORACLE_F32
typedef float real;
#define SQRT sqrtf
#define SIN sinf
#define COS cosf
#define FABS fabsf
#else
typedef double real;
#define SQRT sqrt
#define SIN sin
#define COS cos
#define FABS fabs
#endif

#define MAXL 40
#define MAXCP 96

typedef struct {
    int nl, ncp, nb, nsens;
    int root_fixed, gravity_on, substeps, pad0;
    const int *parent;      /* nl */
    const int *jtype;       /* nl: -1 root, 0 hinge, 1 slide */
    const int *limited;     /* nl */
    const int *drive_mode;  /* nl: 1 = position drive */
    const int *cp_link;     /* ncp */
    const int *cp_body;     /* ncp */
    const int *body_link;   /* nb */
    const int *sensor_body; /* nsens */
    const double *axis, *lpos, *lquat;      /* nl x 3,3,4 */
    const double *mass, *com, *inertia;     /* nl x 1,3,6 */
    const double *armature, *damping, *stiffness, *lower, *upper, *effort, *kp, *kd, *limit_k, *limit_d;
    const double *cp_pos, *cp_radius, *cp_mu; /* ncp x 3,1,1 */
    const double *body_pos, *body_quat;     /* nb x 3,4 */
    const double *hfield;                   /* optional height samples (metres), row-major [nx][ny] */
    int hf_nx, hf_ny;
    double hf_scale, hf_ox, hf_oy;          /* horizontal cell size, world position of sample (0,0) */
    double kn, cn, vs;
    double gravity[3];
    double dt;
    /* optional second body per env: a free box (ShadowHand's cube, shadow_hand.py:372) in contact with the
     * articulation's contact spheres, with its box primitives and with the ground */
    int obj_on, obj_gravity_on, nbx;
    int obj_coupling;   /* 0: block-Jacobi (what the CUDA engine does): both bodies implicit in their own acceleration.
                           1: Gauss-Seidel (EXPERIMENT, DESIGN.md 7b): the articulation as in 0, then the object receives exactly
                              the opposite of the forces applied to the links -> linear momentum is conserved
                           k >= 2: EXPERIMENT: (k-1) extra sweeps of the two block solves on the coupled implicit law
                              F = F0 - h G (J a_link - Jo a_obj), both bodies implicit in both accelerations at convergence */
    double obj_mass, obj_inertia[3], obj_half[3], obj_kn, obj_cn, obj_mu;
    const int *box_link, *box_body;         /* nbx: link carrying the box, body it belongs to */
    const double *box_pos, *box_quat, *box_half;   /* nbx x 3,4,3 (link frame) */
    /* fixed tendons (shared.xml:54-69): length = c0 q[d0] + c1 q[d1], penalty outside [lo, hi] */
    int nten, pad2;
    const int *ten_dof;                     /* nten x 2 (dof indices) */
    const double *ten_coef, *ten_range;     /* nten x 2 */
    double ten_k, ten_d;
    /* AssetOptions.angular_damping / linear_damping / max_angular_velocity (humanoid.py:153-154, anymal_terrain.py:225-226):
     * every link's COM twist is damped with acceleration -d v (wrench -d_a Ic w ; -d_l m v_c, explicit), the base's angular
     * speed is clamped after integration; same for the free object (its own AssetOptions, shadow_hand.py:279-282) */
    double angular_damping, linear_damping, max_angular_velocity, obj_angular_damping, obj_linear_damping;
    /* self-collision (create_actor collision filter 0: humanoid.py:194, anymal_terrain.py:282): contact spheres of links that
     * are not joint neighbours against each other.  Same linearised spring / damper / regularised-friction law as the
     * ground contact with its own gains; block-Jacobi like the hand-object contact: each link is implicit in its own
     * acceleration (h J^T G J joins ITS articulated inertia), explicit in the other link's velocity. */
    int self_on, pad3;
    const unsigned char *self_pairs;        /* ncp x ncp, 1 = this ordered pair may collide */
    double self_kn, self_cn, self_mu;       /* self_kn, self_cn: dimensionless (gains per pair from the reduced link mass and h) */
    /* the free object is a ROUNDED box: all points within obj_round of the box obj_half (0: the block; half = (0,0,L) + round r:
     * a capsule along z -- objectType pen, pen.xml:19; the egg's spheroid, egg.xml:10, is carried as the capsule of equal extent) */
    double obj_round;
    double obj_max_angular_velocity;        /* the object's AssetOptions.max_angular_velocity: clamp after every sub-step (0: none) */
} OracleModel;

/* ---------------------------------------------------------------- small linear algebra */
static void quat_to_mat(const real *q, real R[9]) {
    real x = q[0], y = q[1], z = q[2], w = q[3];
    real n = SQRT(x * x + y * y + z * z + w * w);
    x /= n; y /= n; z /= n; w /= n;
    R[0] = 1 - 2 * (y * y + z * z); R[1] = 2 * (x * y - z * w); R[2] = 2 * (x * z + y * w);
    R[3] = 2 * (x * y + z * w); R[4] = 1 - 2 * (x * x + z * z); R[5] = 2 * (y * z - x * w);
    R[6] = 2 * (x * z - y * w); R[7] = 2 * (y * z + x * w); R[8] = 1 - 2 * (x * x + y * y);
}
static void mat_to_quat(const real R[9], real q[4]) {
    real t = R[0] + R[4] + R[8], s;
    if (t > 0) { s = SQRT(t + 1) * 2; q[3] = s / 4; q[0] = (R[7] - R[5]) / s; q[1] = (R[2] - R[6]) / s; q[2] = (R[3] - R[1]) / s; }
    else if (R[0] > R[4] && R[0] > R[8]) { s = SQRT(1 + R[0] - R[4] - R[8]) * 2; q[3] = (R[7] - R[5]) / s; q[0] = s / 4; q[1] = (R[1] + R[3]) / s; q[2] = (R[2] + R[6]) / s; }
    else if (R[4] > R[8]) { s = SQRT(1 + R[4] - R[0] - R[8]) * 2; q[3] = (R[2] - R[6]) / s; q[0] = (R[1] + R[3]) / s; q[1] = s / 4; q[2] = (R[5] + R[7]) / s; }
    else { s = SQRT(1 + R[8] - R[0] - R[4]) * 2; q[3] = (R[3] - R[1]) / s; q[0] = (R[2] + R[6]) / s; q[1] = (R[5] + R[7]) / s; q[2] = s / 4; }
}
static void mat3_mul(const real A[9], const real B[9], real C[9]) {
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {
        real s = 0; for (int k = 0; k < 3; k++) s += A[3 * i + k] * B[3 * k + j]; C[3 * i + j] = s; }
}
static void mat3_vec(const real A[9], const real v[3], real o[3]) {
    for (int i = 0; i < 3; i++) o[i] = A[3 * i] * v[0] + A[3 * i + 1] * v[1] + A[3 * i + 2] * v[2];
}
static void mat3T_vec(const real A[9], const real v[3], real o[3]) {
    for (int i = 0; i < 3; i++) o[i] = A[i] * v[0] + A[3 + i] * v[1] + A[6 + i] * v[2];
}
static void cross3(const real a[3], const real b[3], real o[3]) {
    o[0] = a[1] * b[2] - a[2] * b[1]; o[1] = a[2] * b[0] - a[0] * b[2]; o[2] = a[0] * b[1] - a[1] * b[0];
}
static void axis_angle_mat(const real a[3], real th, real R[9]) {
    real c = COS(th), s = SIN(th), t = 1 - c;
    R[0] = c + a[0] * a[0] * t; R[1] = a[0] * a[1] * t - a[2] * s; R[2] = a[0] * a[2] * t + a[1] * s;
    R[3] = a[1] * a[0] * t + a[2] * s; R[4] = c + a[1] * a[1] * t; R[5] = a[1] * a[2] * t - a[0] * s;
    R[6] = a[2] * a[0] * t - a[1] * s; R[7] = a[2] * a[1] * t + a[0] * s; R[8] = c + a[2] * a[2] * t;
}
static void skew(const real v[3], real K[9]) {
    K[0] = 0; K[1] = -v[2]; K[2] = v[1]; K[3] = v[2]; K[4] = 0; K[5] = -v[0]; K[6] = -v[1]; K[7] = v[0]; K[8] = 0;
}

/* Pluecker motion transform parent->child as a dense 6x6: X = [E 0; -E rx  E],
 * E = R^T (R maps child coords to parent coords), r = child origin in parent coords. */
static void xform_motion(const real R[9], const real r[3], real X[36]) {
    real E[9], rx[9], Erx[9];
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) E[3 * i + j] = R[3 * j + i];
    skew(r, rx); mat3_mul(E, rx, Erx);
    memset(X, 0, 36 * sizeof(real));
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {
        X[6 * i + j] = E[3 * i + j]; X[6 * (i + 3) + (j + 3)] = E[3 * i + j]; X[6 * (i + 3) + j] = -Erx[3 * i + j]; }
}
static void mat6_vec(const real A[36], const real v[6], real o[6]) {
    for (int i = 0; i < 6; i++) { real s = 0; for (int j = 0; j < 6; j++) s += A[6 * i + j] * v[j]; o[i] = s; }
}
static void mat6T_vec(const real A[36], const real v[6], real o[6]) {
    for (int i = 0; i < 6; i++) { real s = 0; for (int j = 0; j < 6; j++) s += A[6 * j + i] * v[j]; o[i] = s; }
}
/* spatial cross products: crm(v) m  and  crf(v) f = -crm(v)^T f */
static void crm(const real v[6], const real m[6], real o[6]) {
    real a[3], b[3], c[3];
    cross3(v, m, a); cross3(v, m + 3, b); cross3(v + 3, m, c);
    o[0] = a[0]; o[1] = a[1]; o[2] = a[2]; o[3] = b[0] + c[0]; o[4] = b[1] + c[1]; o[5] = b[2] + c[2];
}
static void crf(const real v[6], const real f[6], real o[6]) {
    real a[3], b[3], c[3];
    cross3(v, f, a); cross3(v + 3, f + 3, b); cross3(v, f + 3, c);
    o[0] = a[0] + b[0]; o[1] = a[1] + b[1]; o[2] = a[2] + b[2]; o[3] = c[0]; o[4] = c[1]; o[5] = c[2];
}
/* spatial inertia about the link origin, link coordinates */
static void spatial_inertia(real m, const real c[3], const real Ic6[6], real I[36]) {
    real cx[9], cxcxT[9], Ic[9] = {Ic6[0], Ic6[3], Ic6[4], Ic6[3], Ic6[1], Ic6[5], Ic6[4], Ic6[5], Ic6[2]};
    skew(c, cx);
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {
        real s = 0; for (int k = 0; k < 3; k++) s += cx[3 * i + k] * cx[3 * j + k]; cxcxT[3 * i + j] = s; }
    memset(I, 0, 36 * sizeof(real));
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {
        I[6 * i + j] = Ic[3 * i + j] + m * cxcxT[3 * i + j];
        I[6 * i + (j + 3)] = m * cx[3 * i + j];
        I[6 * (i + 3) + j] = m * cx[3 * j + i];
    }
    for (int i = 0; i < 3; i++) I[6 * (i + 3) + (i + 3)] = m;
}
/* solve A x = b for symmetric positive definite 6x6 (Cholesky) */
static void spd6_solve(const real A[36], const real b[6], real x[6]) {
    real L[36]; memset(L, 0, sizeof(L));
    for (int i = 0; i < 6; i++) for (int j = 0; j <= i; j++) {
        real s = A[6 * i + j]; for (int k = 0; k < j; k++) s -= L[6 * i + k] * L[6 * j + k];
        L[6 * i + j] = (i == j) ? SQRT(s) : s / L[6 * j + j]; }
    real y[6];
    for (int i = 0; i < 6; i++) { real s = b[i]; for (int k = 0; k < i; k++) s -= L[6 * i + k] * y[k]; y[i] = s / L[6 * i + i]; }
    for (int i = 5; i >= 0; i--) { real s = y[i]; for (int k = i + 1; k < 6; k++) s -= L[6 * k + i] * x[k]; x[i] = s / L[6 * i + i]; }
}

/* terrain height and unit normal at world (x,y): plane z=0, or bilinear-free "triangle pair"
 * sampling of the height grid (matches the engine: the cell's lower-left triangle fan) */
static void ground(const OracleModel *m, real x, real y, real *h, real n[3]) {
    if (!m->hfield) { *h = 0; n[0] = 0; n[1] = 0; n[2] = 1; return; }
    real fx = (x - (real)m->hf_ox) / (real)m->hf_scale, fy = (y - (real)m->hf_oy) / (real)m->hf_scale;
    int ix = (int)floor((double)fx), iy = (int)floor((double)fy);
    if (ix < 0) ix = 0; if (iy < 0) iy = 0;
    if (ix > m->hf_nx - 2) ix = m->hf_nx - 2; if (iy > m->hf_ny - 2) iy = m->hf_ny - 2;
    real tx = fx - ix, ty = fy - iy;
    if (tx < 0) tx = 0; if (tx > 1) tx = 1; if (ty < 0) ty = 0; if (ty > 1) ty = 1;
    real h00 = (real)m->hfield[ix * m->hf_ny + iy], h10 = (real)m->hfield[(ix + 1) * m->hf_ny + iy];
    real h01 = (real)m->hfield[ix * m->hf_ny + iy + 1], h11 = (real)m->hfield[(ix + 1) * m->hf_ny + iy + 1];
    real dhx, dhy;
    if (tx + ty <= 1) { dhx = h10 - h00; dhy = h01 - h00; *h = h00 + tx * dhx + ty * dhy; }
    else { dhx = h11 - h01; dhy = h11 - h10; *h = h11 - (1 - tx) * dhx - (1 - ty) * dhy; }
    real gx = dhx / (real)m->hf_scale, gy = dhy / (real)m->hf_scale;
    real inv = 1 / SQRT(gx * gx + gy * gy + 1);
    n[0] = -gx * inv; n[1] = -gy * inv; n[2] = inv;
}

/* sphere (centre c, radius r; world) against a box (centre xb, rotation Rb, half sizes hb): penetration and
 * the unit normal pointing from the box towards the sphere.  Returns 0 when apart. */
static int sphere_box(const real c[3], real r, const real xb[3], const real Rb[9], const real hb[3], real *pen, real n[3]) {
    real d[3] = {c[0] - xb[0], c[1] - xb[1], c[2] - xb[2]}, p[3], q[3], e[3];
    mat3T_vec(Rb, d, p);
    int inside = 1;
    for (int k = 0; k < 3; k++) { q[k] = p[k] < -hb[k] ? -hb[k] : (p[k] > hb[k] ? hb[k] : p[k]); if (q[k] != p[k]) inside = 0; e[k] = p[k] - q[k]; }
    real nl[3] = {0, 0, 0};
    if (!inside) {
        real dist = SQRT(e[0] * e[0] + e[1] * e[1] + e[2] * e[2]);
        if (dist >= r) return 0;
        *pen = r - dist; nl[0] = e[0] / dist; nl[1] = e[1] / dist; nl[2] = e[2] / dist;
    } else {
        int ax = 0; real best = hb[0] - FABS(p[0]);
        for (int k = 1; k < 3; k++) { real m_ = hb[k] - FABS(p[k]); if (m_ < best) { best = m_; ax = k; } }
        *pen = r + best; nl[ax] = p[ax] >= 0 ? 1 : -1;
    }
    mat3_vec(Rb, nl, n);
    return 1;
}

/* One sub-step for one environment.  root: pos3 quat4(xyzw) linvel3 angvel3 (world); dof: (q,qd)
 * interleaved.  cf_body (nb x 3, world) and dof_force (nd) receive the forces of THIS sub-step. */
/* external force on the free object's body, in ITS frame, held over the simulate call: gym.apply_rigid_body_force_tensors(sim,
 * forces, None, LOCAL_SPACE) (shadow_hand.py:708, forceScale > 0).  Set per call by oracle_set_obj_force (nenv,3); acts at the COM. */
static const real *g_obj_force = 0;
static __thread const real *t_obj_fl = 0;
static void substep(const OracleModel *m, real h, real *root, real *dof, const real *tau_act,
                    const real *target, real *cf_body, real *cf_torque_body, real *dof_force,
                    real *Rw_out, real *pw_out, real *vlink_out, real *obj) {
    const int nl = m->nl;
    static __thread real Xup[MAXL][36], S[MAXL][6], v[MAXL][6], c[MAXL][6], IA[MAXL][36], pA[MAXL][6];
    static __thread real U[MAXL][6], Dd[MAXL], u[MAXL], a[MAXL][6], Rw[MAXL][9], pw[MAXL][3], tau[MAXL], diag[MAXL];
    static __thread real cF0[MAXCP][3], cG[MAXCP][9], cJ[MAXCP][18]; static __thread int cact[MAXCP];
    real g[3] = {(real)m->gravity[0], (real)m->gravity[1], (real)m->gravity[2]};
    if (!m->gravity_on) { g[0] = g[1] = g[2] = 0; }

    /* ---- joint forces: explicit part + implicit diagonal */
    for (int i = 1; i < nl; i++) {
        real q = dof[2 * (i - 1)], qd = dof[2 * (i - 1) + 1];
        real qp = q + h * qd;                       /* position the linear terms are taken at */
        real t = tau_act ? tau_act[i - 1] : 0;
        real eff = (real)m->effort[i];
        real b = (real)m->damping[i], k = (real)m->stiffness[i];
        real dg = (real)m->armature[i] + h * b + h * h * k;
        real f = -b * qd - k * qp;
        if (m->drive_mode[i] == 1) {
            real kp = (real)m->kp[i], kd = (real)m->kd[i];
            real pd = kp * ((target ? target[i - 1] : 0) - qp) - kd * qd;
            if (pd > eff) pd = eff; if (pd < -eff) pd = -eff;
            f += pd; dg += h * kd + h * h * kp;
        } else {
            if (t > eff) t = eff; if (t < -eff) t = -eff;
            f += t;
        }
        if (m->limited[i]) {
            real lk = (real)m->limit_k[i], ld = (real)m->limit_d[i];
            if (q < (real)m->lower[i]) { f += lk * ((real)m->lower[i] - qp) - ld * qd; dg += h * ld + h * h * lk; }
            else if (q > (real)m->upper[i]) { f += lk * ((real)m->upper[i] - qp) - ld * qd; dg += h * ld + h * h * lk; }
        }
        tau[i] = f; diag[i] = dg;
    }
    /* fixed tendons: explicit spring/damper on the tendon length outside its range */
    for (int t = 0; t < m->nten; t++) {
        int d0 = m->ten_dof[2 * t], d1 = m->ten_dof[2 * t + 1];
        real c0 = (real)m->ten_coef[2 * t], c1 = (real)m->ten_coef[2 * t + 1];
        real len = c0 * dof[2 * d0] + c1 * dof[2 * d1], rate = c0 * dof[2 * d0 + 1] + c1 * dof[2 * d1 + 1];
        real lo = (real)m->ten_range[2 * t], hi = (real)m->ten_range[2 * t + 1], f = 0;
        if (len > hi) f = -(real)m->ten_k * (len - hi) - (real)m->ten_d * rate;
        else if (len < lo) f = -(real)m->ten_k * (len - lo) - (real)m->ten_d * rate;
        tau[d0 + 1] += c0 * f; tau[d1 + 1] += c1 * f;
    }

    /* ---- pass 1: kinematics, velocities, bias forces */
    real R0[9]; quat_to_mat(root + 3, R0);
    memcpy(Rw[0], R0, sizeof(R0)); pw[0][0] = root[0]; pw[0][1] = root[1]; pw[0][2] = root[2];
    if (m->root_fixed) { for (int k = 0; k < 6; k++) v[0][k] = 0; }
    else { mat3T_vec(R0, root + 10, v[0]); mat3T_vec(R0, root + 7, v[0] + 3); }
    for (int i = 0; i < nl; i++) {
        if (i > 0) {
            int p = m->parent[i];
            real q = dof[2 * (i - 1)], qd = dof[2 * (i - 1) + 1];
            real Rl[9], Rj[9], R[9], r[3], ax[3] = {(real)m->axis[3 * i], (real)m->axis[3 * i + 1], (real)m->axis[3 * i + 2]};
            real lq[4] = {(real)m->lquat[4 * i], (real)m->lquat[4 * i + 1], (real)m->lquat[4 * i + 2], (real)m->lquat[4 * i + 3]};
            quat_to_mat(lq, Rl);
            for (int k = 0; k < 3; k++) r[k] = (real)m->lpos[3 * i + k];
            if (m->jtype[i] == 0) { axis_angle_mat(ax, q, Rj); mat3_mul(Rl, Rj, R); S[i][0] = ax[0]; S[i][1] = ax[1]; S[i][2] = ax[2]; S[i][3] = S[i][4] = S[i][5] = 0; }
            else { memcpy(R, Rl, sizeof(R)); real d[3]; mat3_vec(Rl, ax, d); for (int k = 0; k < 3; k++) r[k] += d[k] * q; S[i][0] = S[i][1] = S[i][2] = 0; S[i][3] = ax[0]; S[i][4] = ax[1]; S[i][5] = ax[2]; }
            xform_motion(R, r, Xup[i]);
            mat3_mul(Rw[p], R, Rw[i]);
            real wr[3]; mat3_vec(Rw[p], r, wr); for (int k = 0; k < 3; k++) pw[i][k] = pw[p][k] + wr[k];
            real vj[6]; for (int k = 0; k < 6; k++) vj[k] = S[i][k] * qd;
            mat6_vec(Xup[i], v[p], v[i]); for (int k = 0; k < 6; k++) v[i][k] += vj[k];
            crm(v[i], vj, c[i]);
        } else { for (int k = 0; k < 6; k++) c[0][k] = 0; }
        real cm[3] = {(real)m->com[3 * i], (real)m->com[3 * i + 1], (real)m->com[3 * i + 2]};
        real Ic[6]; for (int k = 0; k < 6; k++) Ic[k] = (real)m->inertia[6 * i + k];
        spatial_inertia((real)m->mass[i], cm, Ic, IA[i]);
        real Iv[6]; mat6_vec(IA[i], v[i], Iv); crf(v[i], Iv, pA[i]);
        /* gravity as an explicit force: f_g = I * [0; R^T g] */
        real ag[6] = {0, 0, 0, 0, 0, 0}, fg[6]; mat3T_vec(Rw[i], g, ag + 3); mat6_vec(IA[i], ag, fg);
        for (int k = 0; k < 6; k++) pA[i][k] -= fg[k];
        if (m->angular_damping != 0 || m->linear_damping != 0) {
            /* link coordinates: torque about the COM -d_a Ic w, force -d_l m v_c; moved to the link origin */
            real da = (real)m->angular_damping, dl = (real)m->linear_damping, ms = (real)m->mass[i];
            real Iw3[3] = {Ic[0] * v[i][0] + Ic[3] * v[i][1] + Ic[4] * v[i][2], Ic[3] * v[i][0] + Ic[1] * v[i][1] + Ic[5] * v[i][2],
                           Ic[4] * v[i][0] + Ic[5] * v[i][1] + Ic[2] * v[i][2]};
            real wxc[3], f[3], cxf[3]; cross3(v[i], cm, wxc);
            for (int k = 0; k < 3; k++) f[k] = -dl * ms * (v[i][3 + k] + wxc[k]);
            cross3(cm, f, cxf);
            for (int k = 0; k < 3; k++) { pA[i][k] -= -da * Iw3[k] + cxf[k]; pA[i][3 + k] -= f[k]; }
        }
    }

    /* ---- contacts: explicit force + implicit augmentation of the link inertia */
    for (int n = 0; n < m->ncp; n++) {
        int i = m->cp_link[n]; cact[n] = 0;
        real lp[3] = {(real)m->cp_pos[3 * n], (real)m->cp_pos[3 * n + 1], (real)m->cp_pos[3 * n + 2]}, wc[3];
        mat3_vec(Rw[i], lp, wc); for (int k = 0; k < 3; k++) wc[k] += pw[i][k];
        real rad = (real)m->cp_radius[n], hgt, nrm[3];
        ground(m, wc[0], wc[1], &hgt, nrm);
        real d = rad - (wc[2] - hgt) * nrm[2];        /* penetration along the local normal */
        if (d <= 0) continue;
        /* contact point (link coords): sphere centre pushed to its surface along -n */
        real nl_[3]; mat3T_vec(Rw[i], nrm, nl_);
        real rc[3] = {lp[0] - rad * nl_[0], lp[1] - rad * nl_[1], lp[2] - rad * nl_[2]};
        real wxr[3], ul[3], uw[3]; cross3(v[i], rc, wxr);
        for (int k = 0; k < 3; k++) ul[k] = v[i][3 + k] + wxr[k];
        mat3_vec(Rw[i], ul, uw);
        real kn = (real)m->kn, cn = (real)m->cn, gn = cn + h * kn;
        real un = uw[0] * nrm[0] + uw[1] * nrm[1] + uw[2] * nrm[2];
        real Fn = kn * d - gn * un;
        if (Fn <= 0) continue;
        real ut[3] = {uw[0] - un * nrm[0], uw[1] - un * nrm[1], uw[2] - un * nrm[2]};
        real gam = (real)m->cp_mu[n] * Fn / SQRT(ut[0] * ut[0] + ut[1] * ut[1] + ut[2] * ut[2] + (real)(m->vs * m->vs));
        cact[n] = 1;
        for (int k = 0; k < 3; k++) cF0[n][k] = Fn * nrm[k] - gam * ut[k];
        /* G (world) = gam*(1 - n n^T) + gn * n n^T ; J = Rw [ -rc^x  1 ] (3x6, link spatial -> world point vel) */
        real Gw[9]; for (int a_ = 0; a_ < 3; a_++) for (int b_ = 0; b_ < 3; b_++) Gw[3 * a_ + b_] = (a_ == b_ ? gam : 0) + (gn - gam) * nrm[a_] * nrm[b_];
        memcpy(cG[n], Gw, sizeof(Gw));
        real B[18], rx[9]; skew(rc, rx);
        for (int a_ = 0; a_ < 3; a_++) for (int b_ = 0; b_ < 3; b_++) { B[6 * a_ + b_] = -rx[3 * a_ + b_]; B[6 * a_ + 3 + b_] = (a_ == b_); }
        real J[18];
        for (int a_ = 0; a_ < 3; a_++) for (int b_ = 0; b_ < 6; b_++) { real s = 0; for (int k = 0; k < 3; k++) s += Rw[i][3 * a_ + k] * B[6 * k + b_]; J[6 * a_ + b_] = s; }
        memcpy(cJ[n], J, sizeof(J));
        real GJ[18];
        for (int a_ = 0; a_ < 3; a_++) for (int b_ = 0; b_ < 6; b_++) { real s = 0; for (int k = 0; k < 3; k++) s += Gw[3 * a_ + k] * J[6 * k + b_]; GJ[6 * a_ + b_] = s; }
        for (int a_ = 0; a_ < 6; a_++) for (int b_ = 0; b_ < 6; b_++) { real s = 0; for (int k = 0; k < 3; k++) s += J[6 * k + a_] * GJ[6 * k + b_]; IA[i][6 * a_ + b_] += h * s; }
        for (int a_ = 0; a_ < 6; a_++) { real s = 0; for (int k = 0; k < 3; k++) s += J[6 * k + a_] * cF0[n][k]; pA[i][a_] -= s; }
    }

    /* ---- self-collision: sphere n of link i against sphere k of link j (ordered pairs: each link takes its own side) */
    static __thread real sF0[4 * MAXCP][3], sG[4 * MAXCP][9], sJ[4 * MAXCP][18], sPc[4 * MAXCP][3]; static __thread int slink[4 * MAXCP], sbody[4 * MAXCP];
    int nsc = 0;
    if (m->self_on && m->self_pairs) {
        static __thread real wcs[MAXCP][3];
        for (int n = 0; n < m->ncp; n++) {
            int i = m->cp_link[n];
            real lp[3] = {(real)m->cp_pos[3 * n], (real)m->cp_pos[3 * n + 1], (real)m->cp_pos[3 * n + 2]};
            mat3_vec(Rw[i], lp, wcs[n]); for (int k = 0; k < 3; k++) wcs[n][k] += pw[i][k];
        }
        /* gains per pair from the reduced mass of the two LINKS and the sub-step: kn = self_kn * m_red / h^2, cn = self_cn * m_red / h
         * (self_kn, self_cn dimensionless).  Each side of a pair is implicit in its own acceleration but explicit in the partner's
         * velocity; that half-explicit coupling is stable only while h^2 kn / m and h cn / m stay below ~1 for the lighter body --
         * gains tied to the actor's mass (as the ground contact's are) blow up light limbs under persistent actuation. */
        for (int n = 0; n < m->ncp; n++) for (int k2 = 0; k2 < m->ncp; k2++) {
            if (!m->self_pairs[n * m->ncp + k2]) continue;
            real dv[3] = {wcs[n][0] - wcs[k2][0], wcs[n][1] - wcs[k2][1], wcs[n][2] - wcs[k2][2]};
            real rs_ = (real)m->cp_radius[n] + (real)m->cp_radius[k2];
            real d2 = dv[0] * dv[0] + dv[1] * dv[1] + dv[2] * dv[2];
            if (d2 >= rs_ * rs_ || d2 < (real)1e-12 || nsc >= 4 * MAXCP) continue;
            real dist = SQRT(d2), pen = rs_ - dist;
            real nrm[3] = {dv[0] / dist, dv[1] / dist, dv[2] / dist};             /* force on link i: away from sphere k2 */
            real off = (real)m->cp_radius[n] - (real)0.5 * pen;                     /* contact point: middle of the overlap */
            real pc[3] = {wcs[n][0] - off * nrm[0], wcs[n][1] - off * nrm[1], wcs[n][2] - off * nrm[2]};
            int i = m->cp_link[n], j = m->cp_link[k2];
            const real mred = (real)(m->mass[i] * m->mass[j] / (m->mass[i] + m->mass[j]));
            const real skn = (real)m->self_kn * mred / (h * h), sgn = (real)m->self_cn * mred / h + h * skn;
            /* point velocities of both links at pc (world axes) */
            real ri[3] = {pc[0] - pw[i][0], pc[1] - pw[i][1], pc[2] - pw[i][2]}, rj[3] = {pc[0] - pw[j][0], pc[1] - pw[j][1], pc[2] - pw[j][2]};
            real ril[3], rjl[3], t_[3], uil[3], ujl[3], uiw[3], ujw[3];
            mat3T_vec(Rw[i], ri, ril); cross3(v[i], ril, t_); for (int k = 0; k < 3; k++) uil[k] = v[i][3 + k] + t_[k]; mat3_vec(Rw[i], uil, uiw);
            mat3T_vec(Rw[j], rj, rjl); cross3(v[j], rjl, t_); for (int k = 0; k < 3; k++) ujl[k] = v[j][3 + k] + t_[k]; mat3_vec(Rw[j], ujl, ujw);
            real rel[3] = {uiw[0] - ujw[0], uiw[1] - ujw[1], uiw[2] - ujw[2]};
            real un = rel[0] * nrm[0] + rel[1] * nrm[1] + rel[2] * nrm[2];
            real Fn = skn * pen - sgn * un;
            if (Fn <= 0) continue;
            real ut[3] = {rel[0] - un * nrm[0], rel[1] - un * nrm[1], rel[2] - un * nrm[2]};
            real gam = (real)m->self_mu * Fn / SQRT(ut[0] * ut[0] + ut[1] * ut[1] + ut[2] * ut[2] + (real)(m->vs * m->vs));
            real F0_[3], Gw_[9], B_[18], rx_[9], J_[18], GJ_[18];
            for (int k = 0; k < 3; k++) F0_[k] = Fn * nrm[k] - gam * ut[k];
            for (int a_ = 0; a_ < 3; a_++) for (int b_ = 0; b_ < 3; b_++) Gw_[3 * a_ + b_] = (a_ == b_ ? gam : 0) + (sgn - gam) * nrm[a_] * nrm[b_];
            skew(ril, rx_);
            for (int a_ = 0; a_ < 3; a_++) for (int b_ = 0; b_ < 3; b_++) { B_[6 * a_ + b_] = -rx_[3 * a_ + b_]; B_[6 * a_ + 3 + b_] = (a_ == b_); }
            for (int a_ = 0; a_ < 3; a_++) for (int b_ = 0; b_ < 6; b_++) { real s_ = 0; for (int k = 0; k < 3; k++) s_ += Rw[i][3 * a_ + k] * B_[6 * k + b_]; J_[6 * a_ + b_] = s_; }
            for (int a_ = 0; a_ < 3; a_++) for (int b_ = 0; b_ < 6; b_++) { real s_ = 0; for (int k = 0; k < 3; k++) s_ += Gw_[3 * a_ + k] * J_[6 * k + b_]; GJ_[6 * a_ + b_] = s_; }
            for (int a_ = 0; a_ < 6; a_++) for (int b_ = 0; b_ < 6; b_++) { real s_ = 0; for (int k = 0; k < 3; k++) s_ += J_[6 * k + a_] * GJ_[6 * k + b_]; IA[i][6 * a_ + b_] += h * s_; }
            for (int a_ = 0; a_ < 6; a_++) { real s_ = 0; for (int k = 0; k < 3; k++) s_ += J_[6 * k + a_] * F0_[k]; pA[i][a_] -= s_; }
            memcpy(sF0[nsc], F0_, sizeof(F0_)); memcpy(sG[nsc], Gw_, sizeof(Gw_)); memcpy(sJ[nsc], J_, sizeof(J_)); memcpy(sPc[nsc], pc, sizeof(pc));
            slink[nsc] = i; sbody[nsc] = m->cp_body[n]; nsc++;
        }
    }

    /* ---- the free object: contacts with the articulation (block-Jacobi implicit: each body sees its own
     * acceleration implicitly, the other's velocity explicitly), with the ground, then its own 6x6 solve */
    static __thread real oF0[MAXCP + 64][3], oG[MAXCP + 64][9], oJ[MAXCP + 64][18]; static __thread int olink[MAXCP + 64], obody[MAXCP + 64]; static __thread real oPc[MAXCP + 64][3];
    static __thread real IA0[MAXL][36], pA0[MAXL][6], qdd_[MAXL];
    int noc = 0;
    real Ao[36], bo[6], Ro[9];
    if (m->obj_on && obj) {
        quat_to_mat(obj + 3, Ro);
        real Iw[9], T[9], Id[9] = {(real)m->obj_inertia[0], 0, 0, 0, (real)m->obj_inertia[1], 0, 0, 0, (real)m->obj_inertia[2]};
        mat3_mul(Ro, Id, T);
        for (int a_ = 0; a_ < 3; a_++) for (int b_ = 0; b_ < 3; b_++) { real s_ = 0; for (int k = 0; k < 3; k++) s_ += T[3 * a_ + k] * Ro[3 * b_ + k]; Iw[3 * a_ + b_] = s_; }
        memset(Ao, 0, sizeof(Ao));
        for (int a_ = 0; a_ < 3; a_++) { for (int b_ = 0; b_ < 3; b_++) Ao[6 * a_ + b_] = Iw[3 * a_ + b_]; Ao[6 * (a_ + 3) + a_ + 3] = (real)m->obj_mass; }
        real Iww[3], gyro[3]; mat3_vec(Iw, obj + 10, Iww); cross3(obj + 10, Iww, gyro);
        /* unknown = SPATIAL acceleration (alpha ; a_c - w x v_c) so that J*a is the rate of change of the velocity field
         * at the contact point, the same quantity the articulation's contacts use */
        real wxv0[3]; cross3(obj + 10, obj + 7, wxv0);
        for (int k = 0; k < 3; k++) { bo[k] = -gyro[k]; bo[3 + k] = (m->obj_gravity_on ? (real)m->obj_mass * (real)m->gravity[k] : 0) - (real)m->obj_mass * wxv0[k]; }
        for (int k = 0; k < 3; k++) { bo[k] -= (real)m->obj_angular_damping * Iww[k]; bo[3 + k] -= (real)m->obj_linear_damping * (real)m->obj_mass * obj[7 + k]; }
        if (t_obj_fl) { real Fw[3]; mat3_vec(Ro, t_obj_fl, Fw); for (int k = 0; k < 3; k++) bo[3 + k] += Fw[k]; }
        real okn = (real)m->obj_kn, ocn = (real)m->obj_cn, ogn = ocn + h * okn, hb[3] = {(real)m->obj_half[0], (real)m->obj_half[1], (real)m->obj_half[2]};
        /* helper macro: one contact at world point pc with normal nrm (direction of the force on the LINK), penetration pen */
#define OBJ_CONTACT(LI, BI, CPI, PC, NRM, PEN, MU) do {                                                                       \
            real rcw_[3] = {(PC)[0] - pw[LI][0], (PC)[1] - pw[LI][1], (PC)[2] - pw[LI][2]}, rc_[3], wxr_[3], ul_[3], uw_[3];       \
            mat3T_vec(Rw[LI], rcw_, rc_); cross3(v[LI], rc_, wxr_);                                                              \
            for (int k = 0; k < 3; k++) ul_[k] = v[LI][3 + k] + wxr_[k];                                                         \
            mat3_vec(Rw[LI], ul_, uw_);                                                                                          \
            real ro_[3] = {(PC)[0] - obj[0], (PC)[1] - obj[1], (PC)[2] - obj[2]}, wo_[3]; cross3(obj + 10, ro_, wo_);            \
            real rel_[3] = {uw_[0] - obj[7] - wo_[0], uw_[1] - obj[8] - wo_[1], uw_[2] - obj[9] - wo_[2]};                        \
            real un_ = rel_[0] * (NRM)[0] + rel_[1] * (NRM)[1] + rel_[2] * (NRM)[2];                                             \
            real Fn_ = okn * (PEN) - ogn * un_;                                                                                  \
            if (Fn_ > 0 && noc < MAXCP + 64) {                                                                                   \
                real ut_[3] = {rel_[0] - un_ * (NRM)[0], rel_[1] - un_ * (NRM)[1], rel_[2] - un_ * (NRM)[2]};                    \
                real gam_ = (MU) * Fn_ / SQRT(ut_[0] * ut_[0] + ut_[1] * ut_[1] + ut_[2] * ut_[2] + (real)(m->vs * m->vs));     \
                real F0_[3], Gw_[9];                                                                                             \
                for (int k = 0; k < 3; k++) F0_[k] = Fn_ * (NRM)[k] - gam_ * ut_[k];                                             \
                for (int a_ = 0; a_ < 3; a_++) for (int b_ = 0; b_ < 3; b_++) Gw_[3 * a_ + b_] = (a_ == b_ ? gam_ : 0) + (ogn - gam_) * (NRM)[a_] * (NRM)[b_]; \
                real B_[18], rx_[9], J_[18], GJ_[18]; skew(rc_, rx_);                                                            \
                for (int a_ = 0; a_ < 3; a_++) for (int b_ = 0; b_ < 3; b_++) { B_[6 * a_ + b_] = -rx_[3 * a_ + b_]; B_[6 * a_ + 3 + b_] = (a_ == b_); } \
                for (int a_ = 0; a_ < 3; a_++) for (int b_ = 0; b_ < 6; b_++) { real s_ = 0; for (int k = 0; k < 3; k++) s_ += Rw[LI][3 * a_ + k] * B_[6 * k + b_]; J_[6 * a_ + b_] = s_; } \
                for (int a_ = 0; a_ < 3; a_++) for (int b_ = 0; b_ < 6; b_++) { real s_ = 0; for (int k = 0; k < 3; k++) s_ += Gw_[3 * a_ + k] * J_[6 * k + b_]; GJ_[6 * a_ + b_] = s_; } \
                for (int a_ = 0; a_ < 6; a_++) for (int b_ = 0; b_ < 6; b_++) { real s_ = 0; for (int k = 0; k < 3; k++) s_ += J_[6 * k + a_] * GJ_[6 * k + b_]; IA[LI][6 * a_ + b_] += h * s_; } \
                for (int a_ = 0; a_ < 6; a_++) { real s_ = 0; for (int k = 0; k < 3; k++) s_ += J_[6 * k + a_] * F0_[k]; pA[LI][a_] -= s_; } \
                /* object side: Jo = [ -ro^x  1 ] about its COM, world axes */                                                    \
                real Jo_[18], rox_[9], GJo_[18]; skew(ro_, rox_);                                                                \
                for (int a_ = 0; a_ < 3; a_++) for (int b_ = 0; b_ < 3; b_++) { Jo_[6 * a_ + b_] = -rox_[3 * a_ + b_]; Jo_[6 * a_ + 3 + b_] = (a_ == b_); } \
                for (int a_ = 0; a_ < 3; a_++) for (int b_ = 0; b_ < 6; b_++) { real s_ = 0; for (int k = 0; k < 3; k++) s_ += Gw_[3 * a_ + k] * Jo_[6 * k + b_]; GJo_[6 * a_ + b_] = s_; } \
                if (m->obj_coupling != 1) {                                                                                      \
                for (int a_ = 0; a_ < 6; a_++) for (int b_ = 0; b_ < 6; b_++) { real s_ = 0; for (int k = 0; k < 3; k++) s_ += Jo_[6 * k + a_] * GJo_[6 * k + b_]; Ao[6 * a_ + b_] += h * s_; } \
                for (int a_ = 0; a_ < 6; a_++) { real s_ = 0; for (int k = 0; k < 3; k++) s_ += Jo_[6 * k + a_] * F0_[k]; bo[a_] -= s_; } \
                }                                                                                                                \
                memcpy(oF0[noc], F0_, sizeof(F0_)); memcpy(oG[noc], Gw_, sizeof(Gw_)); memcpy(oJ[noc], J_, sizeof(J_));          \
                olink[noc] = LI; obody[noc] = BI; memcpy(oPc[noc], (PC), 3 * sizeof(real)); noc++;                                \
            }                                                                                                                    \
        } while (0)
        /* S1: the articulation's contact spheres against the object's box */
        for (int n = 0; n < m->ncp; n++) {
            int i = m->cp_link[n];
            real lp[3] = {(real)m->cp_pos[3 * n], (real)m->cp_pos[3 * n + 1], (real)m->cp_pos[3 * n + 2]}, wc[3], pen, nrm[3];
            mat3_vec(Rw[i], lp, wc); for (int k = 0; k < 3; k++) wc[k] += pw[i][k];
            real rad = (real)m->cp_radius[n];
            if (!sphere_box(wc, rad + (real)m->obj_round, obj, Ro, hb, &pen, nrm)) continue;   /* rounded box = inflate the sphere */
            real pc[3] = {wc[0] - rad * nrm[0], wc[1] - rad * nrm[1], wc[2] - rad * nrm[2]};
            OBJ_CONTACT(i, m->cp_body[n], n, pc, nrm, pen, (real)m->obj_mu);
        }
        /* S2: the object's corners against the articulation's box primitives */
        for (int b = 0; b < m->nbx; b++) {
            int i = m->box_link[b];
            real bq[4] = {(real)m->box_quat[4 * b], (real)m->box_quat[4 * b + 1], (real)m->box_quat[4 * b + 2], (real)m->box_quat[4 * b + 3]}, Rb[9], Rwb[9];
            real bp[3] = {(real)m->box_pos[3 * b], (real)m->box_pos[3 * b + 1], (real)m->box_pos[3 * b + 2]}, xb[3];
            real bh[3] = {(real)m->box_half[3 * b], (real)m->box_half[3 * b + 1], (real)m->box_half[3 * b + 2]};
            quat_to_mat(bq, Rb); mat3_mul(Rw[i], Rb, Rwb); mat3_vec(Rw[i], bp, xb); for (int k = 0; k < 3; k++) xb[k] += pw[i][k];
            for (int c = 0; c < 8; c++) {
                if (((c & 1) && hb[0] == 0) || ((c & 2) && hb[1] == 0) || ((c & 4) && hb[2] == 0)) continue;   /* degenerate box: each distinct corner once */
                real lc[3] = {(c & 1 ? hb[0] : -hb[0]), (c & 2 ? hb[1] : -hb[1]), (c & 4 ? hb[2] : -hb[2])}, pc[3], pen, nout[3], rr = (real)m->obj_round;
                mat3_vec(Ro, lc, pc); for (int k = 0; k < 3; k++) pc[k] += obj[k];
                if (!sphere_box(pc, rr, xb, Rwb, bh, &pen, nout)) continue;      /* corner (sphere of the rounding radius) inside the link's box */
                real nrm[3] = {-nout[0], -nout[1], -nout[2]};                  /* force on the LINK pushes it away from the corner */
                real pcs[3] = {pc[0] + rr * nrm[0], pc[1] + rr * nrm[1], pc[2] + rr * nrm[2]};
                OBJ_CONTACT(i, m->box_body[b], -1, pcs, nrm, pen, (real)m->obj_mu);
            }
        }
#undef OBJ_CONTACT
        /* S3: the object's corners against the ground */
        for (int c = 0; c < 8; c++) {
            if (((c & 1) && hb[0] == 0) || ((c & 2) && hb[1] == 0) || ((c & 4) && hb[2] == 0)) continue;
            real lc[3] = {(c & 1 ? hb[0] : -hb[0]), (c & 2 ? hb[1] : -hb[1]), (c & 4 ? hb[2] : -hb[2])}, ro_[3], pc[3], hgt, nrm[3];
            mat3_vec(Ro, lc, ro_); for (int k = 0; k < 3; k++) pc[k] = ro_[k] + obj[k];
            ground(m, pc[0], pc[1], &hgt, nrm);
            real d = (real)m->obj_round - (pc[2] - hgt) * nrm[2];
            if (d <= 0) continue;
            for (int k = 0; k < 3; k++) ro_[k] -= (real)m->obj_round * nrm[k];      /* contact point on the corner sphere */
            real wo_[3]; cross3(obj + 10, ro_, wo_);
            real u_[3] = {obj[7] + wo_[0], obj[8] + wo_[1], obj[9] + wo_[2]};
            real un_ = u_[0] * nrm[0] + u_[1] * nrm[1] + u_[2] * nrm[2], Fn_ = okn * d - ogn * un_;
            if (Fn_ <= 0) continue;
            real ut_[3] = {u_[0] - un_ * nrm[0], u_[1] - un_ * nrm[1], u_[2] - un_ * nrm[2]};
            real gam_ = (real)m->obj_mu * Fn_ / SQRT(ut_[0] * ut_[0] + ut_[1] * ut_[1] + ut_[2] * ut_[2] + (real)(m->vs * m->vs));
            real F_[3], Gw_[9], Jo_[18], rox_[9], GJo_[18];
            for (int k = 0; k < 3; k++) F_[k] = Fn_ * nrm[k] - gam_ * ut_[k];
            for (int a_ = 0; a_ < 3; a_++) for (int b_ = 0; b_ < 3; b_++) Gw_[3 * a_ + b_] = (a_ == b_ ? gam_ : 0) + (ogn - gam_) * nrm[a_] * nrm[b_];
            skew(ro_, rox_);
            for (int a_ = 0; a_ < 3; a_++) for (int b_ = 0; b_ < 3; b_++) { Jo_[6 * a_ + b_] = -rox_[3 * a_ + b_]; Jo_[6 * a_ + 3 + b_] = (a_ == b_); }
            for (int a_ = 0; a_ < 3; a_++) for (int b_ = 0; b_ < 6; b_++) { real s_ = 0; for (int k = 0; k < 3; k++) s_ += Gw_[3 * a_ + k] * Jo_[6 * k + b_]; GJo_[6 * a_ + b_] = s_; }
            for (int a_ = 0; a_ < 6; a_++) for (int b_ = 0; b_ < 6; b_++) { real s_ = 0; for (int k = 0; k < 3; k++) s_ += Jo_[6 * k + a_] * GJo_[6 * k + b_]; Ao[6 * a_ + b_] += h * s_; }
            for (int a_ = 0; a_ < 6; a_++) { real s_ = 0; for (int k = 0; k < 3; k++) s_ += Jo_[6 * k + a_] * F_[k]; bo[a_] += s_; }
        }
    }

    /* coupled-implicit experiment: repeat the two block solves, each seeing the other's latest acceleration */
    const int sweeps = (m->obj_on && obj && m->obj_coupling >= 2) ? m->obj_coupling : 1;
    real ao_prev[6] = {0, 0, 0, 0, 0, 0}, bo0[6];
    if (m->obj_on && obj) memcpy(bo0, bo, sizeof(bo0));
    if (sweeps > 1) { memcpy(IA0, IA, sizeof(real) * 36 * nl); memcpy(pA0, pA, sizeof(real) * 6 * nl); }
    for (int sweep = 0; sweep < sweeps; sweep++) {
    if (sweep > 0) {
        memcpy(IA, IA0, sizeof(real) * 36 * nl); memcpy(pA, pA0, sizeof(real) * 6 * nl);
        for (int n = 0; n < noc; n++) {        /* the link also feels + h G (Jo a_obj) */
            real ro_[3] = {oPc[n][0] - obj[0], oPc[n][1] - obj[1], oPc[n][2] - obj[2]}, axr[3], Jao[3], cf_[3];
            cross3(ao_prev, ro_, axr);
            for (int k = 0; k < 3; k++) Jao[k] = ao_prev[3 + k] + axr[k];
            for (int a_ = 0; a_ < 3; a_++) { real s_ = 0; for (int k = 0; k < 3; k++) s_ += oG[n][3 * a_ + k] * Jao[k]; cf_[a_] = h * s_; }
            for (int a_ = 0; a_ < 6; a_++) { real s_ = 0; for (int k = 0; k < 3; k++) s_ += oJ[n][6 * k + a_] * cf_[k]; pA[olink[n]][a_] -= s_; }
        }
    }
    /* ---- pass 2: articulated inertias, leaf -> root */
    for (int i = nl - 1; i >= 1; i--) {
        int p = m->parent[i];
        mat6_vec(IA[i], S[i], U[i]);
        real D = diag[i], Sp = 0;
        for (int k = 0; k < 6; k++) { D += S[i][k] * U[i][k]; Sp += S[i][k] * pA[i][k]; }
        Dd[i] = D; u[i] = tau[i] - Sp;
        real Ia[36], pa[6], Iac[6];
        for (int a_ = 0; a_ < 6; a_++) for (int b_ = 0; b_ < 6; b_++) Ia[6 * a_ + b_] = IA[i][6 * a_ + b_] - U[i][a_] * U[i][b_] / D;
        mat6_vec(Ia, c[i], Iac);
        for (int k = 0; k < 6; k++) pa[k] = pA[i][k] + Iac[k] + U[i][k] * u[i] / D;
        /* IA_p += X^T Ia X ; pA_p += X^T pa   (X = motion transform parent->child) */
        real T[36];
        for (int a_ = 0; a_ < 6; a_++) for (int b_ = 0; b_ < 6; b_++) { real s = 0; for (int k = 0; k < 6; k++) s += Ia[6 * a_ + k] * Xup[i][6 * k + b_]; T[6 * a_ + b_] = s; }
        for (int a_ = 0; a_ < 6; a_++) for (int b_ = 0; b_ < 6; b_++) { real s = 0; for (int k = 0; k < 6; k++) s += Xup[i][6 * k + a_] * T[6 * k + b_]; IA[p][6 * a_ + b_] += s; }
        real pp[6]; mat6T_vec(Xup[i], pa, pp); for (int k = 0; k < 6; k++) pA[p][k] += pp[k];
    }

    /* ---- root acceleration, pass 3 */
    if (m->root_fixed) { for (int k = 0; k < 6; k++) a[0][k] = 0; }
    else { real nb_[6]; for (int k = 0; k < 6; k++) nb_[k] = -pA[0][k]; spd6_solve(IA[0], nb_, a[0]); }
    for (int i = 1; i < nl; i++) {
        int p = m->parent[i];
        mat6_vec(Xup[i], a[p], a[i]); for (int k = 0; k < 6; k++) a[i][k] += c[i][k];
        real Ua = 0; for (int k = 0; k < 6; k++) Ua += U[i][k] * a[i][k];
        real qdd = (u[i] - Ua) / Dd[i];
        for (int k = 0; k < 6; k++) a[i][k] += S[i][k] * qdd;
        qdd_[i] = qdd;
    }
    if (sweeps > 1) {      /* the object, seeing the links' accelerations of this sweep: bo = bo0 + sum Jo^T h G (J a_link) */
        real bo_[6], ro_[3], Ja[3], f_[3], tq_[3];
        memcpy(bo_, bo0, sizeof(bo_));
        for (int n = 0; n < noc; n++) {
            for (int a_ = 0; a_ < 3; a_++) { real s_ = 0; for (int k = 0; k < 6; k++) s_ += oJ[n][6 * a_ + k] * a[olink[n]][k]; Ja[a_] = s_; }
            for (int a_ = 0; a_ < 3; a_++) { real s_ = 0; for (int k = 0; k < 3; k++) s_ += oG[n][3 * a_ + k] * Ja[k]; f_[a_] = h * s_; }
            for (int k = 0; k < 3; k++) ro_[k] = oPc[n][k] - obj[k];
            cross3(ro_, f_, tq_);
            for (int k = 0; k < 3; k++) { bo_[k] += tq_[k]; bo_[3 + k] += f_[k]; }
        }
        spd6_solve(Ao, bo_, ao_prev);
        memcpy(bo, bo_, sizeof(bo_));
    }
    }   /* sweeps */
    for (int i = 1; i < nl; i++) {
        real qdd = qdd_[i];
        if (dof_force) dof_force[i - 1] = tau[i] - (diag[i] - (real)m->armature[i]) * qdd;
        dof[2 * (i - 1) + 1] += h * qdd;
        dof[2 * (i - 1)] += h * dof[2 * (i - 1) + 1];
    }

    /* ---- contact forces actually applied over this sub-step: F = F0 - h G J a */
    if (cf_body) { memset(cf_body, 0, sizeof(real) * 3 * m->nb); memset(cf_torque_body, 0, sizeof(real) * 3 * m->nb); }
    for (int n = 0; n < m->ncp && cf_body; n++) {
        if (!cact[n]) continue;
        int i = m->cp_link[n], b = m->cp_body[n];
        real Ja[3], F[3];
        for (int a_ = 0; a_ < 3; a_++) { real s = 0; for (int k = 0; k < 6; k++) s += cJ[n][6 * a_ + k] * a[i][k]; Ja[a_] = s; }
        for (int a_ = 0; a_ < 3; a_++) { real s = 0; for (int k = 0; k < 3; k++) s += cG[n][3 * a_ + k] * Ja[k]; F[a_] = cF0[n][a_] - h * s; }
        /* torque about the BODY frame origin (world axes) */
        real lp[3] = {(real)m->cp_pos[3 * n], (real)m->cp_pos[3 * n + 1], (real)m->cp_pos[3 * n + 2]}, wc[3], hgt, nrm[3];
        mat3_vec(Rw[i], lp, wc); for (int k = 0; k < 3; k++) wc[k] += pw[i][k];
        ground(m, wc[0], wc[1], &hgt, nrm);
        real bp[3] = {(real)m->body_pos[3 * b], (real)m->body_pos[3 * b + 1], (real)m->body_pos[3 * b + 2]}, wb[3], arm[3], tq[3];
        mat3_vec(Rw[i], bp, wb);
        for (int k = 0; k < 3; k++) arm[k] = (wc[k] - (real)m->cp_radius[n] * nrm[k]) - (pw[i][k] + wb[k]);
        cross3(arm, F, tq);
        for (int k = 0; k < 3; k++) { cf_body[3 * b + k] += F[k]; cf_torque_body[3 * b + k] += tq[k]; }
    }

    /* ---- self-contacts: force applied to each side's own body over the sub-step */
    for (int n = 0; n < nsc && cf_body; n++) {
        int i = slink[n], b = sbody[n];
        real Ja[3], F[3];
        for (int a_ = 0; a_ < 3; a_++) { real s_ = 0; for (int k = 0; k < 6; k++) s_ += sJ[n][6 * a_ + k] * a[i][k]; Ja[a_] = s_; }
        for (int a_ = 0; a_ < 3; a_++) { real s_ = 0; for (int k = 0; k < 3; k++) s_ += sG[n][3 * a_ + k] * Ja[k]; F[a_] = sF0[n][a_] - h * s_; }
        if (b < 0) continue;
        real bp[3] = {(real)m->body_pos[3 * b], (real)m->body_pos[3 * b + 1], (real)m->body_pos[3 * b + 2]}, wb[3], arm[3], tq[3];
        mat3_vec(Rw[i], bp, wb);
        for (int k = 0; k < 3; k++) arm[k] = sPc[n][k] - (pw[i][k] + wb[k]);
        cross3(arm, F, tq);
        for (int k = 0; k < 3; k++) { cf_body[3 * b + k] += F[k]; cf_torque_body[3 * b + k] += tq[k]; }
    }

    /* ---- hand-object contacts: forces applied to the articulation's bodies (sensors), then the object itself */
    if (m->obj_on && obj) {
        for (int n = 0; n < noc; n++) {
            int i = olink[n], b = obody[n];
            real Ja[3], F[3];
            for (int a_ = 0; a_ < 3; a_++) { real s_ = 0; for (int k = 0; k < 6; k++) s_ += oJ[n][6 * a_ + k] * a[i][k]; Ja[a_] = s_; }
            for (int a_ = 0; a_ < 3; a_++) { real s_ = 0; for (int k = 0; k < 3; k++) s_ += oG[n][3 * a_ + k] * Ja[k]; F[a_] = oF0[n][a_] - h * s_; }
            if (m->obj_coupling == 1) {        /* the object gets the opposite of what the link got */
                real ro_[3] = {oPc[n][0] - obj[0], oPc[n][1] - obj[1], oPc[n][2] - obj[2]}, mF[3] = {-F[0], -F[1], -F[2]}, tq_[3];
                cross3(ro_, mF, tq_);
                for (int k = 0; k < 3; k++) { bo[k] += tq_[k]; bo[3 + k] += mF[k]; }
            }
            if (b < 0 || !cf_body) continue;
            real bp[3] = {(real)m->body_pos[3 * b], (real)m->body_pos[3 * b + 1], (real)m->body_pos[3 * b + 2]}, wb[3], arm[3], tq[3];
            mat3_vec(Rw[i], bp, wb);
            for (int k = 0; k < 3; k++) arm[k] = oPc[n][k] - (pw[i][k] + wb[k]);
            cross3(arm, F, tq);
            for (int k = 0; k < 3; k++) { cf_body[3 * b + k] += F[k]; cf_torque_body[3 * b + k] += tq[k]; }
        }
        real ao[6];
        spd6_solve(Ao, bo, ao);
        real wxv1[3]; cross3(obj + 10, obj + 7, wxv1);
        for (int k = 0; k < 3; k++) { obj[10 + k] += h * ao[k]; obj[7 + k] += h * (ao[3 + k] + wxv1[k]); }
        if (m->obj_max_angular_velocity > 0) {
            real wn2 = obj[10] * obj[10] + obj[11] * obj[11] + obj[12] * obj[12], mx = (real)m->obj_max_angular_velocity;
            if (wn2 > mx * mx) { real k_ = mx / SQRT(wn2); obj[10] *= k_; obj[11] *= k_; obj[12] *= k_; }
        }
        for (int k = 0; k < 3; k++) obj[k] += h * obj[7 + k];
        real w[3] = {obj[10], obj[11], obj[12]};
        real wn = SQRT(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]), th = wn * h, dq[4];
        if (wn > 1e-12) { real s_ = SIN(th / 2) / wn; dq[0] = w[0] * s_; dq[1] = w[1] * s_; dq[2] = w[2] * s_; dq[3] = COS(th / 2); }
        else { dq[0] = w[0] * h / 2; dq[1] = w[1] * h / 2; dq[2] = w[2] * h / 2; dq[3] = 1; }
        real *q = obj + 3, x = q[0], y = q[1], z = q[2], ww = q[3];
        real nq[4] = { dq[3] * x + dq[0] * ww + dq[1] * z - dq[2] * y, dq[3] * y - dq[0] * z + dq[1] * ww + dq[2] * x,
                       dq[3] * z + dq[0] * y - dq[1] * x + dq[2] * ww, dq[3] * ww - dq[0] * x - dq[1] * y - dq[2] * z };
        real nn = SQRT(nq[0] * nq[0] + nq[1] * nq[1] + nq[2] * nq[2] + nq[3] * nq[3]);
        for (int k = 0; k < 4; k++) q[k] = nq[k] / nn;
    }

    /* ---- root integration (world-frame twist of the root origin) */
    if (!m->root_fixed) {
        real al[3], wxv[3], t1[3], dw[3], dv[3];
        cross3(v[0], v[0] + 3, wxv);
        for (int k = 0; k < 3; k++) t1[k] = a[0][3 + k] + wxv[k];
        mat3_vec(R0, a[0], dw); mat3_vec(R0, t1, dv); (void)al;
        for (int k = 0; k < 3; k++) { root[10 + k] += h * dw[k]; root[7 + k] += h * dv[k]; }
        for (int k = 0; k < 3; k++) root[k] += h * root[7 + k];
        if (m->max_angular_velocity > 0) {
            real wn2 = root[10] * root[10] + root[11] * root[11] + root[12] * root[12], mx = (real)m->max_angular_velocity;
            if (wn2 > mx * mx) { real sc = mx / SQRT(wn2); root[10] *= sc; root[11] *= sc; root[12] *= sc; }
        }
        real w[3] = {root[10], root[11], root[12]};
        real wn = SQRT(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]), th = wn * h, dq[4];
        if (wn > 1e-12) { real s = SIN(th / 2) / wn; dq[0] = w[0] * s; dq[1] = w[1] * s; dq[2] = w[2] * s; dq[3] = COS(th / 2); }
        else { dq[0] = w[0] * h / 2; dq[1] = w[1] * h / 2; dq[2] = w[2] * h / 2; dq[3] = 1; }
        real *q = root + 3, x = q[0], y = q[1], z = q[2], ww = q[3];
        real nq[4] = { dq[3] * x + dq[0] * ww + dq[1] * z - dq[2] * y,
                       dq[3] * y - dq[0] * z + dq[1] * ww + dq[2] * x,
                       dq[3] * z + dq[0] * y - dq[1] * x + dq[2] * ww,
                       dq[3] * ww - dq[0] * x - dq[1] * y - dq[2] * z };
        real nn = SQRT(nq[0] * nq[0] + nq[1] * nq[1] + nq[2] * nq[2] + nq[3] * nq[3]);
        for (int k = 0; k < 4; k++) q[k] = nq[k] / nn;
    }
    if (Rw_out) { memcpy(Rw_out, Rw, sizeof(real) * 9 * nl); memcpy(pw_out, pw, sizeof(real) * 3 * nl); memcpy(vlink_out, v, sizeof(real) * 6 * nl); }
}

/* forward kinematics + link twists for the CURRENT state -> public rigid-body states
 * (pos3 quat4 linvel3 angvel3 per body, world frame, velocity of the body-frame origin) */
static void body_states(const OracleModel *m, const real *root, const real *dof, real *out) {
    const int nl = m->nl;
    real Rw[MAXL][9], pw[MAXL][3], w[MAXL][3], vl[MAXL][3];
    quat_to_mat(root + 3, Rw[0]);
    for (int k = 0; k < 3; k++) { pw[0][k] = root[k]; vl[0][k] = m->root_fixed ? 0 : root[7 + k]; w[0][k] = m->root_fixed ? 0 : root[10 + k]; }
    for (int i = 1; i < nl; i++) {
        int p = m->parent[i];
        real q = dof[2 * (i - 1)], qd = dof[2 * (i - 1) + 1];
        real Rl[9], Rj[9], R[9], r[3], ax[3] = {(real)m->axis[3 * i], (real)m->axis[3 * i + 1], (real)m->axis[3 * i + 2]};
        real lq[4] = {(real)m->lquat[4 * i], (real)m->lquat[4 * i + 1], (real)m->lquat[4 * i + 2], (real)m->lquat[4 * i + 3]};
        quat_to_mat(lq, Rl);
        for (int k = 0; k < 3; k++) r[k] = (real)m->lpos[3 * i + k];
        real wr[3], waxis[3], d[3], wxr[3];
        mat3_vec(Rl, ax, d);
        if (m->jtype[i] == 0) { axis_angle_mat(ax, q, Rj); mat3_mul(Rl, Rj, R); }
        else { memcpy(R, Rl, sizeof(R)); for (int k = 0; k < 3; k++) r[k] += d[k] * q; }
        mat3_mul(Rw[p], R, Rw[i]);
        mat3_vec(Rw[p], r, wr); mat3_vec(Rw[p], d, waxis);
        cross3(w[p], wr, wxr);
        for (int k = 0; k < 3; k++) { pw[i][k] = pw[p][k] + wr[k]; vl[i][k] = vl[p][k] + wxr[k]; w[i][k] = w[p][k]; }
        if (m->jtype[i] == 0) for (int k = 0; k < 3; k++) w[i][k] += waxis[k] * qd;
        else for (int k = 0; k < 3; k++) vl[i][k] += waxis[k] * qd;
    }
    for (int b = 0; b < m->nb; b++) {
        int i = m->body_link[b];
        real bp[3] = {(real)m->body_pos[3 * b], (real)m->body_pos[3 * b + 1], (real)m->body_pos[3 * b + 2]}, wb[3], wxb[3];
        real bq[4] = {(real)m->body_quat[4 * b], (real)m->body_quat[4 * b + 1], (real)m->body_quat[4 * b + 2], (real)m->body_quat[4 * b + 3]}, Rb[9], Rwb[9];
        mat3_vec(Rw[i], bp, wb); cross3(w[i], wb, wxb);
        quat_to_mat(bq, Rb); mat3_mul(Rw[i], Rb, Rwb);
        real *o = out + 13 * b;
        for (int k = 0; k < 3; k++) { o[k] = pw[i][k] + wb[k]; o[7 + k] = vl[i][k] + wxb[k]; o[10 + k] = w[i][k]; }
        mat_to_quat(Rwb, o + 3);
        if (o[6] < 0) for (int k = 3; k < 7; k++) o[k] = -o[k];
    }
}

/* ------------------------------------------------------------------ exported entry points */
int oracle_real_size(void) { return (int)sizeof(real); }

/* gym.simulate(): `substeps` sub-steps of dt/substeps for `nenv` independent environments.
 * root (nenv,13), dof (nenv,nd,2) updated in place; outputs may be NULL.
 * sensor (nenv,nsens,6): net contact force / torque on the sensor's body in the body frame,
 * torque about the body origin, from the LAST sub-step. */
typedef struct {
    const OracleModel *m; int e0, e1; real *root, *dof; const real *tau_act, *target;
    real *body_state, *contact_force, *sensor, *dof_force, *obj;
} SimJob;

static void *simulate_range(void *arg) {
    SimJob *j = (SimJob *)arg; const OracleModel *m = j->m;
    const int nd = m->nl - 1;
    real h = (real)(m->dt / m->substeps);
    for (int e = j->e0; e < j->e1; e++) {
        real cf[3 * MAXL], ct[3 * MAXL], df[MAXL], bs[13 * MAXL];
        real *r = j->root + 13 * e, *d = j->dof + 2 * nd * e;
        real Rw[9 * MAXL], pw[3 * MAXL], vl[6 * MAXL];
        t_obj_fl = (g_obj_force && j->obj) ? g_obj_force + 3 * e : 0;
        for (int s = 0; s < m->substeps; s++)
            substep(m, h, r, d, j->tau_act ? j->tau_act + nd * e : 0, j->target ? j->target + nd * e : 0, cf, ct, df, Rw, pw, vl, j->obj ? j->obj + 13 * e : 0);
        if (j->dof_force) memcpy(j->dof_force + nd * e, df, sizeof(real) * nd);
        if (j->contact_force) memcpy(j->contact_force + 3 * m->nb * e, cf, sizeof(real) * 3 * m->nb);
        if (j->body_state) { body_states(m, r, d, bs); memcpy(j->body_state + 13 * m->nb * e, bs, sizeof(real) * 13 * m->nb); }
        /* sensors: the contact wrench of the last sub-step in the body frame AS IT WAS when the
         * forces were evaluated (start of that sub-step) */
        if (j->sensor) for (int s = 0; s < m->nsens; s++) {
            int b = m->sensor_body[s], li = m->body_link[b]; real Rb[9], Rwb[9];
            real bq[4] = {(real)m->body_quat[4 * b], (real)m->body_quat[4 * b + 1], (real)m->body_quat[4 * b + 2], (real)m->body_quat[4 * b + 3]};
            quat_to_mat(bq, Rb); mat3_mul(Rw + 9 * li, Rb, Rwb);
            mat3T_vec(Rwb, cf + 3 * b, j->sensor + 6 * (m->nsens * e + s));
            mat3T_vec(Rwb, ct + 3 * b, j->sensor + 6 * (m->nsens * e + s) + 3);
        }
    }
    return 0;
}

void oracle_set_obj_force(const real *f) { g_obj_force = f; }      /* NULL: none; the pointer must outlive the simulate call */
static int g_threads = 1;
void oracle_set_threads(int n) { g_threads = n < 1 ? 1 : (n > 256 ? 256 : n); }

void oracle_simulate_obj(const OracleModel *m, int nenv, real *root, real *dof, const real *tau_act,
                          const real *target, real *body_state, real *contact_force, real *sensor,
                          real *dof_force, real *obj);
void oracle_simulate(const OracleModel *m, int nenv, real *root, real *dof, const real *tau_act,
                     const real *target, real *body_state, real *contact_force, real *sensor,
                     real *dof_force) {
    oracle_simulate_obj(m, nenv, root, dof, tau_act, target, body_state, contact_force, sensor, dof_force, 0);
}
/* same, with the optional free object per env: obj (nenv,13) pos quat linvel angvel, updated in place */
void oracle_simulate_obj(const OracleModel *m, int nenv, real *root, real *dof, const real *tau_act,
                          const real *target, real *body_state, real *contact_force, real *sensor,
                          real *dof_force, real *obj) {
    int nt = g_threads; if (nt > nenv) nt = nenv > 0 ? nenv : 1;
    SimJob jobs[256]; pthread_t th[256];
    for (int t = 0; t < nt; t++) {
        SimJob j = {m, (int)((long long)nenv * t / nt), (int)((long long)nenv * (t + 1) / nt), root, dof,
                    tau_act, target, body_state, contact_force, sensor, dof_force, obj};
        jobs[t] = j;
    }
    if (nt == 1) { simulate_range(&jobs[0]); return; }
    for (int t = 0; t < nt; t++) pthread_create(&th[t], 0, simulate_range, &jobs[t]);
    for (int t = 0; t < nt; t++) pthread_join(th[t], 0);
}

/* forward kinematics only (refresh_rigid_body_state_tensor on a freshly set state) */
void oracle_body_states(const OracleModel *m, int nenv, const real *root, const real *dof, real *body_state) {
    const int nd = m->nl - 1;
    for (int e = 0; e < nenv; e++) body_states(m, root + 13 * e, dof + 2 * nd * e, body_state + 13 * m->nb * e);
}

/* joint accelerations + root spatial acceleration for one state, WITHOUT integrating: used by the
 * inverse-dynamics (RNEA) cross-check in tests.  qdd (nd), a0 (6, root link coords). */
void oracle_forward_dynamics(const OracleModel *m, const real *root_in, const real *dof_in,
                             const real *tau_act, real *qdd, real *root_after, real *dof_after) {
    const int nd = m->nl - 1;
    real r[13], d[2 * MAXL], h = (real)(m->dt / m->substeps);
    memcpy(r, root_in, sizeof(r)); memcpy(d, dof_in, sizeof(real) * 2 * nd);
    substep(m, h, r, d, tau_act, 0, 0, 0, 0, 0, 0, 0, 0);
    for (int i = 0; i < nd; i++) qdd[i] = (d[2 * i + 1] - dof_in[2 * i + 1]) / h;
    memcpy(root_after, r, sizeof(r)); memcpy(dof_after, d, sizeof(real) * 2 * nd);
}

/* ------------------------------------------------------------------ kinematic / inertial tensors
 * gym.acquire_jacobian_tensor / acquire_mass_matrix_tensor + refresh_* (tasks/franka_cube_stack.py:388-392,439-440
 * in the reference: the operational-space controller reads the end effector's rows of J and the arm's block of M).
 * The closed binary defines the layouts; what the call sites fix is: J[env, body row, 0:3 linear | 3:6 angular, dof
 * column] in the world frame, a fixed-base articulation has no row for its base link and no base columns
 * (`jacobian[:, hand_joint_index, :, :7]` indexes by JOINT), M[env, dof, dof].  For a floating base we put the six base
 * coordinates FIRST -- world linear velocity of the root origin, then world angular velocity, the way the root-state
 * tensor carries them -- so J is (nb, 6, 6 + nd) and M is (6 + nd, 6 + nd).  [layout for floating bases unverifiable
 * here; written down in DESIGN.md]
 *   J maps generalised velocities to the twist of each BODY-frame origin (what rigid_body_state reports);
 *   M is the joint-space inertia (composite-rigid-body algorithm, body coordinates -- Featherstone 2008 table 6.2
 *   extended with the floating base, section 9.4) plus the joint armature on the diagonal.  The implicit-integration
 *   terms of the sub-step (h b + h^2 k ...) are NOT part of M. */
static void kin_tree(const OracleModel *m, const real *root, const real *dof, real Rw[][9], real pw[][3], real aw[][3],
                     real Xup[][36], real S[][6]) {
    const int nl = m->nl;
    quat_to_mat(root + 3, Rw[0]);
    for (int k = 0; k < 3; k++) { pw[0][k] = root[k]; aw[0][k] = 0; }
    for (int i = 1; i < nl; i++) {
        int p = m->parent[i];
        real q = dof[2 * (i - 1)];
        real Rl[9], Rj[9], R[9], r[3], ax[3] = {(real)m->axis[3 * i], (real)m->axis[3 * i + 1], (real)m->axis[3 * i + 2]};
        real lq[4] = {(real)m->lquat[4 * i], (real)m->lquat[4 * i + 1], (real)m->lquat[4 * i + 2], (real)m->lquat[4 * i + 3]};
        quat_to_mat(lq, Rl);
        for (int k = 0; k < 3; k++) r[k] = (real)m->lpos[3 * i + k];
        for (int k = 0; k < 6; k++) S[i][k] = 0;
        if (m->jtype[i] == 0) { axis_angle_mat(ax, q, Rj); mat3_mul(Rl, Rj, R); for (int k = 0; k < 3; k++) S[i][k] = ax[k]; }
        else { memcpy(R, Rl, sizeof(R)); real d[3]; mat3_vec(Rl, ax, d); for (int k = 0; k < 3; k++) { r[k] += d[k] * q; S[i][3 + k] = ax[k]; } }
        xform_motion(R, r, Xup[i]);
        mat3_mul(Rw[p], R, Rw[i]);
        real wr[3]; mat3_vec(Rw[p], r, wr);
        for (int k = 0; k < 3; k++) pw[i][k] = pw[p][k] + wr[k];
        mat3_vec(Rw[i], ax, aw[i]);             /* joint axis in world axes (the joint rotation leaves it fixed) */
    }
}

/* jac: (nrows, 6, ncols) with nrows = nb (floating) or nb - 1 (fixed: every body but the base body 0), in body order;
 * ncols = nd (+ 6 base columns first when floating).  Returns nrows. */
static int jacobian_env(const OracleModel *m, const real *root, const real *dof, real *jac) {
    const int nl = m->nl, nd = nl - 1, nbase = m->root_fixed ? 0 : 6, nc = nd + nbase;
    static __thread real Rw[MAXL][9], pw[MAXL][3], aw[MAXL][3], Xup[MAXL][36], S[MAXL][6];
    kin_tree(m, root, dof, Rw, pw, aw, Xup, S);
    int row = 0;
    for (int b = 0; b < m->nb; b++) {
        const int l = m->body_link[b];
        if (m->root_fixed && b == 0) continue;         /* a fixed base: no row for the base body (PhysX: num_links - 1 rows) */
        real bp[3] = {(real)m->body_pos[3 * b], (real)m->body_pos[3 * b + 1], (real)m->body_pos[3 * b + 2]}, wb[3], pb[3];
        mat3_vec(Rw[l], bp, wb);
        for (int k = 0; k < 3; k++) pb[k] = pw[l][k] + wb[k];
        real *J = jac + (size_t)row * 6 * nc;
        memset(J, 0, sizeof(real) * 6 * nc);
        if (nbase) {
            real r[3] = {pb[0] - pw[0][0], pb[1] - pw[0][1], pb[2] - pw[0][2]}, K[9];
            skew(r, K);                                   /* v_b = v_0 + w_0 x r = v_0 - [r]x w_0 */
            for (int k = 0; k < 3; k++) {
                J[k * nc + k] = 1; J[(3 + k) * nc + 3 + k] = 1;
                for (int c = 0; c < 3; c++) J[k * nc + 3 + c] = -K[3 * k + c];
            }
        }
        for (int j = l; j > 0; j = m->parent[j]) {         /* the joints between the base and this body's link */
            const int col = nbase + j - 1;
            if (m->jtype[j] == 0) {
                real r[3] = {pb[0] - pw[j][0], pb[1] - pw[j][1], pb[2] - pw[j][2]}, lin[3];
                cross3(aw[j], r, lin);
                for (int k = 0; k < 3; k++) { J[k * nc + col] = lin[k]; J[(3 + k) * nc + col] = aw[j][k]; }
            } else for (int k = 0; k < 3; k++) J[k * nc + col] = aw[j][k];
        }
        row++;
    }
    return row;
}

static void mat6T_mat6_mat6(const real X[36], const real I[36], real out[36]) {   /* X^T I X */
    real t[36];
    for (int i = 0; i < 6; i++) for (int j = 0; j < 6; j++) { real s = 0; for (int k = 0; k < 6; k++) s += I[6 * i + k] * X[6 * k + j]; t[6 * i + j] = s; }
    for (int i = 0; i < 6; i++) for (int j = 0; j < 6; j++) { real s = 0; for (int k = 0; k < 6; k++) s += X[6 * k + i] * t[6 * k + j]; out[6 * i + j] = s; }
}

/* M: (nc, nc), nc = nd (+ 6 when floating: base coordinates first, world linear then world angular) */
static void mass_matrix_env(const OracleModel *m, const real *root, const real *dof, real *M) {
    const int nl = m->nl, nd = nl - 1, nbase = m->root_fixed ? 0 : 6, nc = nd + nbase;
    static __thread real Rw[MAXL][9], pw[MAXL][3], aw[MAXL][3], Xup[MAXL][36], S[MAXL][6], Ic[MAXL][36];
    kin_tree(m, root, dof, Rw, pw, aw, Xup, S);
    for (int i = 0; i < nl; i++) {
        real cm[3] = {(real)m->com[3 * i], (real)m->com[3 * i + 1], (real)m->com[3 * i + 2]}, I6[6];
        for (int k = 0; k < 6; k++) I6[k] = (real)m->inertia[6 * i + k];
        spatial_inertia((real)m->mass[i], cm, I6, Ic[i]);
    }
    for (int i = nl - 1; i > 0; i--) {
        real t[36]; mat6T_mat6_mat6(Xup[i], Ic[i], t);
        for (int k = 0; k < 36; k++) Ic[m->parent[i]][k] += t[k];
    }
    memset(M, 0, sizeof(real) * nc * nc);
    /* base coordinates u = (v world, w world); base-link spatial velocity [w_b; v_b] = T u, T = [0 R^T; R^T 0] */
    real T[36]; memset(T, 0, sizeof(T));
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) { T[6 * i + 3 + j] = Rw[0][3 * j + i]; T[6 * (3 + i) + j] = Rw[0][3 * j + i]; }
    if (nbase) {
        real B[36]; mat6T_mat6_mat6(T, Ic[0], B);
        for (int i = 0; i < 6; i++) for (int j = 0; j < 6; j++) M[i * nc + j] = B[6 * i + j];
    }
    for (int i = 1; i < nl; i++) {
        real F[6]; mat6_vec(Ic[i], S[i], F);
        real d = 0; for (int k = 0; k < 6; k++) d += S[i][k] * F[k];
        M[(nbase + i - 1) * nc + nbase + i - 1] = d + (real)m->armature[i];
        int j = i;
        while (m->parent[j] > 0) {
            real G[6]; mat6T_vec(Xup[j], F, G); memcpy(F, G, sizeof(F));
            j = m->parent[j];
            real s = 0; for (int k = 0; k < 6; k++) s += S[j][k] * F[k];
            M[(nbase + i - 1) * nc + nbase + j - 1] = s; M[(nbase + j - 1) * nc + nbase + i - 1] = s;
        }
        if (nbase) {
            real G[6], Fb[6]; mat6T_vec(Xup[j], F, G);       /* now in base-link coordinates */
            mat6T_vec(T, G, Fb);
            for (int k = 0; k < 6; k++) { M[k * nc + nbase + i - 1] = Fb[k]; M[(nbase + i - 1) * nc + k] = Fb[k]; }
        }
    }
}

int oracle_jacobian_rows(const OracleModel *m) {
    int rows = 0;
    return m->root_fixed ? m->nb - 1 : m->nb;
}
void oracle_jacobian(const OracleModel *m, int nenv, const real *root, const real *dof, real *jac) {
    const int nd = m->nl - 1, nc = nd + (m->root_fixed ? 0 : 6), rows = oracle_jacobian_rows(m);
    for (int e = 0; e < nenv; e++) jacobian_env(m, root + 13 * e, dof + 2 * nd * e, jac + (size_t)e * rows * 6 * nc);
}
void oracle_mass_matrix(const OracleModel *m, int nenv, const real *root, const real *dof, real *M) {
    const int nd = m->nl - 1, nc = nd + (m->root_fixed ? 0 : 6);
    for (int e = 0; e < nenv; e++) mass_matrix_env(m, root + 13 * e, dof + 2 * nd * e, M + (size_t)e * nc * nc);
}
