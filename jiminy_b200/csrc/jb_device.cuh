// Device code of the batched rigid-body step (sm_90a, fp64).
//
// One warp = 32/L environments; the L lanes of an env walk the lane plan of jb_plan.h.  All
// per-env working data lives in shared memory as `field-major x 32 lanes` (conflict-free 8-byte
// accesses), the hot per-joint quantities of a sweep live in registers and are carried from one
// record to the next.  The reference functions each block replaces are cited inline
// (paths relative to the reference's source tree).
#pragma once
#ifdef JB_HOST_EMUL
#include "jb_emul_shim.h"   // tests/emul: CPU thread emulation of a warp (test infrastructure only)
#else
#include <cuda_runtime.h>
#endif
#include <math.h>
#include <stdint.h>

#include "jb_plan.h"

namespace jb {

constexpr int MAX_REC = 48;
constexpr double D_EPS = 2.220446049250313e-16;
#define D_INF (__longlong_as_double(0x7ff0000000000000LL))
constexpr double STEPPER_MIN_TIMESTEP = 1e-10;   // core/include/jiminy/core/constants.h:18-20
constexpr double SIMULATION_MIN_TIMESTEP = 1e-6;

enum : int32_t { MODE_START = 0, MODE_STEP = 1, MODE_DYNAMICS = 2 };
enum : int32_t { SCH_T = 0, SCH_DT = 1, SCH_DTLARGEST = 2, SCH_DTLARGESTPREV = 3, SCH_TERROR = 4, SCH_TPREV = 5, SCH_N = 6 };

// Values that change from one launch to the next travel as the kernel's parameter (constant bank 0); everything in
// KParams below is persistent per batch and is uploaded to constant memory only when it changed.
struct LaunchArgs {
    int32_t mode;                  // MODE_*
    int32_t peer_on;               // MODE_STEP of a connected batch: publish the sensor rows to the peers, signal at the end
    int32_t peer_parity;           // which of the two gathered buffers this step fills
    int32_t validate;              // MODE_START from device inputs: each env checks its own (q0, v0) row first
    long long peer_step;           // step counter the completion flags are set to
    double step_dt;
    const uint8_t* mask;           // MODE_START: envs to (re)start, null = all
    const double* command;         // MODE_DYNAMICS: the command of this evaluation (the held command of the running envs is not touched)
};

// One sensor of the measurement pipeline (AbstractSensorOptions, core/include/jiminy/core/hardware/abstract_sensor.h:66-100)
struct SensorDesc {
    int32_t type, index, nf, ns;   // sensor type (0 Imu, 1 Force, 2 Encoder, 3 Effort, 4 Contact), index within the type, fields, sensors of the type
    int32_t offset;                // column of (field 0, sensor 0) of the type in the observation row
    int32_t order, has_noise, has_bias;
    double delay, jitter;
    double noise_std[6], bias[6];
};

struct KParams {
    int32_t n_env, n_pad;
    int32_t L, nrec, ntrunk, npool, ncslot, nimuslot, nfields;
    int32_t pool_off, cslot_off, imu_off;
    int32_t sph_off;               // where the RS_* block of a spherical record starts (RF_KA + 6 * n_hist)
    int32_t nq, nv, nmotors, njoints, n_hist;
    int32_t nimu, nforce, nenc, neff, ncs;
    int32_t want_extra;
    int32_t rec_off[MAX_REC];
    uint8_t rec_free[MAX_REC];
    uint8_t trunk_reduce[MAX_REC];
    uint8_t kind_u[MAX_REC];       // lane-uniform record kind (0 = lanes differ)
    int32_t sig_id;                // static plan signature matched at batch creation (0 = none)
    int32_t rhs_variant;           // hot-path evaluation of the quadruped signature: 1 = composite-rigid-body form, 0 = ABA sweeps
    int32_t quad_stage;            // 1: an RK4 stage of the quadruped hot path is one call (stage_quadruped_crba), composite form only
    double contact_inv_vt;         // 1 / contacts.transitionVelocity
    double contact_blend_k;        // -2 / contacts.transitionEps, 0 when the blend is off (<= D_EPS)
    int32_t fast_bounds;          // 1: joint position bounds are solved inside the hot-path evaluation (quadruped, composite form)
    int32_t uniform_solver;        // 1: full-mask collectives in the structured solver when the whole warp is in it
    double pgs_relax[100];         // relaxation factor of PGS iteration i (constraint_solvers.cc:236-248), tabulated by the host
    int32_t fast_bounds_io;        // (development) 0: skip the load / store of the bound state around the step
    int32_t all_uniform;           // 1: every record has the same integer descriptor on all lanes
    RecInt rint_u[MAX_REC];        // lane-uniform record descriptors (valid when all_uniform)
    JbSensorLayout lay;
    JbOptions opt;
    double stepper_update_period;
    const RecInt* rint;
    const RecDbl* rdbl;
    const ContactSlot* cslots;
    const double* imu_placement;   // [nimu][12]
    const double* springs;         // [2][nv] stiffness, damping (may be null)
    const double* pd_gains;        // [2][nmotors] kp, kd of the device-side PD controller (may be null)
    double* cmd_torque;            // [n_env][nmotors] torque command held between launches (PD mode)
    double* mahony;                // [n_env][nimu][10] MahonyFilter state (quaternion 4, gyro bias 3, angular velocity 3); null = off
    double mahony_kp, mahony_ki;
    const double* pdf;             // PDController block: kp | kd | lower[3] | upper[3] | (safety: kp kd lo hi vmax), each [nmotors]; null = off
    double* pdf_state;             // [n_env][3][nmotors] target position / velocity / acceleration
    int32_t pdf_safety;
    // persistent state, structure-of-arrays [component][n_pad]
    double* q; double* v; double* a; double* sched; long long* iters; int32_t* status;
    const double* command;         // [n_env][nmotors] (AoS, as uploaded)
    double* sensors;               // [n_env][width]   (AoS, as downloaded)
    double* qv_out;                // [n_env][nq+nv]   (AoS device view) or null
    // MODE_START / MODE_DYNAMICS inputs (AoS) and MODE_DYNAMICS outputs
    const double* q_in; const double* v_in;
    double* a_out; double* fext_out; double* u_out;
    // efforts / extra terms outputs (AoS), refreshed at the end of MODE_START / MODE_STEP
    double* eff_u; double* eff_umotor; double* eff_fext;
    double* extra_energy; double* extra_a; double* extra_f;
    // sensor measurement pipeline (delay ring, white noise, bias; see measure_sensors): off unless a sensor option was set
    int32_t sp_on, sp_cap, sp_nsens;
    const SensorDesc* sp_desc;     // [sp_nsens]
    double sp_delay_max[5];        // per sensor type: max over its sensors of delay + jitter
    unsigned long long* sp_rng;    // [n_env][sp_nsens] PCG32 states
    const unsigned long long* sp_rng_init;   // [n_env][sp_nsens] states a (re)started env begins with (seeding chain done on the host)
    double* sp_times;              // [n_env][sp_cap] sample times, circular
    int32_t* sp_count;             // [n_env][6]: physical index of the newest sample, samples held by each of the 5 types
    double* sp_ring;               // [n_env][sp_cap][width] true values, circular
    const uint32_t* zig_kn; const float* zig_fn; const float* zig_wn;   // ziggurat tables of the normal sampler [128] each
    int32_t* sp_snap_count; unsigned long long* sp_snap_rng;            // copies taken at the top of a hot-path pass (restored on hand-off)
    double* extra_ycrb; double* extra_com; double* extra_vcom; double* extra_hg;   // [n_env][njoints][10 | 3 | 3], [n_env][12]; null = off
    double total_mass;
    // model variants (jb_set_model_variants): `rdbl` holds n_variants tables of rdbl_rows rows; the envs of a block (one
    // warp) share the variant variant_of_block[block]; block_mass[block] = total mass of that variant
    int32_t n_variants, rdbl_rows;
    const int32_t* variant_of_block;
    const double* block_mass;
    // external forces (impulse + profile forces), see jb_plan.h:ExtSlot
    int32_t n_eslot, ext_off, n_imp, n_prof;
    int32_t imp_slot[MAX_IMPULSE];
    int32_t prof_slot[MAX_PROFILE];
    double prof_period[MAX_PROFILE];
    const ExtSlot* eslots;         // [n_eslot][L]
    const double* imp_data;        // [n_imp][IMPULSE_ROWS][n_pad]: t, dt, wrench
    const double* prof_pending;    // [n_prof][6][n_pad]: what the force "function" returns (host buffer)
    double* prof_latched;          // [n_prof][6][n_pad]: value held since the last update (finite period)
    // constraint path (jb_constraints.cuh)
    // observation exchange over peer memory (jb_peer_obs_*): gathered buffers [2][world][n_env][width] of every rank
    int32_t peer_n, peer_rank;     // connected world size (0 = no exchange), this rank
    double* peer_obs[8];
    long long* peer_flags[8];      // [2][world] completion flags inside every rank's buffer
    unsigned int* peer_counter;    // blocks of this launch that have finished
    int32_t* needs_full;           // [n_pad] env must be stepped by the full body (enabled constraints / bounds just left)
    double* pdf_snap;              // [n_env][3][nmotors] PDController state at the top of the launch (restored on hand-off)
    double* mahony_snap;           // [n_env][nimu][10]   MahonyFilter state at the top of the launch (restored on hand-off)
    int32_t cons_on;               // workspace allocated: bounds / contact constraints are solved on the device
    int32_t cons_off;              // per-lane shared-memory field: number of enabled constraints this lane owns
    int32_t cq_on, cq_off;         // structured solver for quadruped-shaped plans (jb_constraints_quadruped.cuh) and its fields
    int32_t n_jc, n_cc, m_max;     // joint constraints, contact constraints, total constraint rows
    const JointMap* jmap;          // [njoints]
    const ContactMap* cmap;        // [ncontacts]
    const int32_t* jc_joint;       // [n_jc] joint of each joint constraint
    const int32_t* jc_of_joint;    // [njoints] joint constraint index or -1
    int32_t cs_total, cw_total;    // doubles per env of the two tables below
    double* cstate;                // [n_pad][cs_total] persistent constraint state, one contiguous row per env
    double* cwork;                 // [resident slots x envs per warp][cw_total] workspace (contiguous per env: rows of the dense matrices share cache lines)
    unsigned int* cw_slots;        // [cw_n_sm] occupancy bitmask of the workspace slots of each SM
    int32_t cw_blocks_per_sm;      // resident blocks per SM the workspace is sized for
    int32_t cw_n_sm;               // rows of cw_slots (SM ids are folded into it: %smid need not be < the SM count)
    // lane-block solver (jb_constraints_blocks.cuh)
    int32_t lb_on;                 // L > 1 and the trunk fits: used for every solve but the start-time equality solve
    int32_t lb_nt, lb_nl, lb_ml;   // trunk dofs, max private dofs per lane, max constraint rows owned by a lane
    int32_t lb_nl_of[8];           // private dofs of each sub-lane
    int32_t lw_total;              // doubles per lane of the workspace below
    const int32_t* lb_dof0;        // [nrec][L] first dof of the record inside its block (trunk block / the lane's private block)
    double* lwork;                 // [resident slots x 32 lanes][lw_total]
    // body-space contact solver (jb_constraints_bodies.cuh)
    int32_t bd_on, bd_n, bd_ncar;  // enabled; contact bodies; max bodies owned by one lane
    int32_t bd_off, bd_lsh;        // shared-memory region of the sweep (2 x 6 bd_n doubles per env, spread over its lanes); log2(L)
    int32_t bd_rec[4], bd_owner[4], bd_slot[4];   // record of each contact body, owning sub-lane, index among the owner's bodies
    const int32_t* bd_of_contact;  // [ncontacts] contact body of each contact frame
    // (appended last: the offsets of every field above, which the step path reads, stay what they were)
    const double* q_bounds;        // [2][nq] position lower / upper bounds, for the input checks of LaunchArgs::validate
};

// Launch parameters live in constant memory (uniform constant-bank operands in every device
// function, no parameter pointer to chase) and the per-warp working set in dynamic shared memory
// addressed through the symbol itself, so that the compiler emits LDS / STS rather than generic
// loads.  The host serialises (copy to symbol, launch) per device.
#ifdef JB_HOST_EMUL
extern KParams g_kp_host;
#define KP (&g_kp_host)
#define jb_smem emul_smem
#else
__constant__ KParams g_kp;
#define KP (&g_kp)
extern __shared__ double jb_smem[];
#endif
// workspace slot of this block (full kernel, constraint path): the workspace is sized for the blocks that can be
// resident at once, not for the batch, so that it stays in L2
__shared__ int jb_cw_slot;
// Development build only (-DJB_PROFILE_CLOCKS, tools/build_prof.sh): cycle accounting of the full body with clock64(),
// summed over the warps of the launch (lane 0 of each warp adds its own intervals).  Never defined in the product build.
#if defined(JB_PROFILE_CLOCKS) && !defined(JB_HOST_EMUL)
__device__ unsigned long long jb_prof[16];
#define JB_PROF_T(var) const long long var = clock64()
#define JB_PROF_ADD(i, t0) do { if ((threadIdx.x & 31) == 0) atomicAdd(&jb_prof[i], static_cast<unsigned long long>(clock64() - (t0))); } while (0)
#define JB_PROF_COUNT(i, n) do { if ((threadIdx.x & 31) == 0) atomicAdd(&jb_prof[i], static_cast<unsigned long long>(n)); } while (0)
#else
#define JB_PROF_T(var)
#define JB_PROF_ADD(i, t0)
#define JB_PROF_COUNT(i, n)
#endif
// model variants: the first row of this block's variant in KP->rdbl rides in the upper bits of Ctx::flags (0 without
// variants) -- a shift and an add where the tables are read, no register and no memory access of its own
constexpr int CTX_ROW_SHIFT = 8;
#define JB_RDBL (KP->rdbl + (c.flags >> CTX_ROW_SHIFT))

// ------------------------------------------------------------------------------------------
// small fixed-size algebra in registers
// ------------------------------------------------------------------------------------------
struct V3 { double x, y, z; };
struct Xf { double R[9]; V3 p; };         // SE3, R row-major: child -> parent
struct Mot { V3 l, a; };                  // spatial motion or force: (linear, angular)
struct SymY { double A[6], B[9], D[6]; }; // 6x6 symmetric [[A, B], [B^T, D]]; A, D in (xx,xy,yy,xz,yz,zz)

#define JB_DI __device__ __forceinline__
#define JB_HD __host__ __device__ __forceinline__

JB_DI V3 mk(double x, double y, double z) { V3 r; r.x = x; r.y = y; r.z = z; return r; }
JB_DI V3 operator+(V3 a, V3 b) { return mk(a.x + b.x, a.y + b.y, a.z + b.z); }
JB_DI V3 operator-(V3 a, V3 b) { return mk(a.x - b.x, a.y - b.y, a.z - b.z); }
JB_DI V3 operator*(double s, V3 a) { return mk(s * a.x, s * a.y, s * a.z); }
JB_DI double dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
JB_DI V3 cross(V3 a, V3 b) { return mk(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
JB_DI V3 rmul(const double* R, V3 v) {   // R v
    return mk(R[0] * v.x + R[1] * v.y + R[2] * v.z, R[3] * v.x + R[4] * v.y + R[5] * v.z, R[6] * v.x + R[7] * v.y + R[8] * v.z);
}
JB_DI V3 rtmul(const double* R, V3 v) {  // R^T v
    return mk(R[0] * v.x + R[3] * v.y + R[6] * v.z, R[1] * v.x + R[4] * v.y + R[7] * v.z, R[2] * v.x + R[5] * v.y + R[8] * v.z);
}
JB_DI void mat3mul(const double* A, const double* B, double* C) {
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}
JB_DI Mot mzero() { Mot m; m.l = mk(0, 0, 0); m.a = mk(0, 0, 0); return m; }
JB_DI Mot operator+(Mot a, Mot b) { Mot m; m.l = a.l + b.l; m.a = a.a + b.a; return m; }
JB_DI Mot operator-(Mot a, Mot b) { Mot m; m.l = a.l - b.l; m.a = a.a - b.a; return m; }
// SE3::actInv / act on motions and forces (pinocchio/spatial/se3-tpl.hpp)
JB_DI Mot motion_act_inv(const Xf& M, Mot m) { Mot r; r.l = rtmul(M.R, m.l - cross(M.p, m.a)); r.a = rtmul(M.R, m.a); return r; }
JB_DI Mot force_act(const Xf& M, Mot f) { Mot r; r.l = rmul(M.R, f.l); r.a = rmul(M.R, f.a) + cross(M.p, r.l); return r; }
JB_DI Mot motion_cross(Mot a, Mot b) { Mot r; r.l = cross(a.l, b.a) + cross(a.a, b.l); r.a = cross(a.a, b.a); return r; }
JB_DI Mot motion_cross_force(Mot v, Mot f) { Mot r; r.l = cross(v.a, f.l); r.a = cross(v.a, f.a) + cross(v.l, f.l); return r; }
JB_DI V3 symmul(const double* S, V3 w) {
    return mk(S[0] * w.x + S[1] * w.y + S[3] * w.z, S[1] * w.x + S[2] * w.y + S[4] * w.z, S[3] * w.x + S[4] * w.y + S[5] * w.z);
}
// InertiaTpl::__mult__: I * v for a rigid body (mass, lever c, I about the CoM)
JB_DI Mot inertia_mul(double mass, V3 c, const double* I, Mot v) {
    Mot f;
    f.l = mass * (v.l - cross(c, v.a));
    f.a = symmul(I, v.a) + cross(c, f.l);
    return f;
}
// InertiaTpl::matrix() as the symmetric block form
JB_DI void inertia_to_sym(double m, V3 c, const double* I, SymY& Y) {
    Y.A[0] = m; Y.A[1] = 0; Y.A[2] = m; Y.A[3] = 0; Y.A[4] = 0; Y.A[5] = m;
    // B = -m [c]x
    Y.B[0] = 0;        Y.B[1] = m * c.z;  Y.B[2] = -m * c.y;
    Y.B[3] = -m * c.z; Y.B[4] = 0;        Y.B[5] = m * c.x;
    Y.B[6] = m * c.y;  Y.B[7] = -m * c.x; Y.B[8] = 0;
    // D = I - m [c]x [c]x ; [c]x[c]x = c c^T - |c|^2 1
    const double cc = dot(c, c);
    Y.D[0] = I[0] - m * (c.x * c.x - cc);
    Y.D[1] = I[1] - m * (c.x * c.y);
    Y.D[2] = I[2] - m * (c.y * c.y - cc);
    Y.D[3] = I[3] - m * (c.x * c.z);
    Y.D[4] = I[4] - m * (c.y * c.z);
    Y.D[5] = I[5] - m * (c.z * c.z - cc);
}
JB_DI Mot sym_mul_motion(const SymY& Y, Mot m) {  // [[A,B],[B^T,D]] (l; a)
    Mot f;
    f.l = symmul(Y.A, m.l) + rmul(Y.B, m.a);
    f.a = rtmul(Y.B, m.l) + symmul(Y.D, m.a);
    return f;
}
JB_DI void sym_add(SymY& Y, const SymY& Z) {
#pragma unroll
    for (int k = 0; k < 6; ++k) { Y.A[k] += Z.A[k]; Y.D[k] += Z.D[k]; }
#pragma unroll
    for (int k = 0; k < 9; ++k) Y.B[k] += Z.B[k];
}
// S3 = R S R^T for symmetric S (6) -> symmetric (6)
JB_DI void rot_sym(const double* R, const double* S, double* O) {
    double T[9];  // T = R S
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        T[3 * i + 0] = R[3 * i] * S[0] + R[3 * i + 1] * S[1] + R[3 * i + 2] * S[3];
        T[3 * i + 1] = R[3 * i] * S[1] + R[3 * i + 1] * S[2] + R[3 * i + 2] * S[4];
        T[3 * i + 2] = R[3 * i] * S[3] + R[3 * i + 1] * S[4] + R[3 * i + 2] * S[5];
    }
    O[0] = T[0] * R[0] + T[1] * R[1] + T[2] * R[2];
    O[1] = T[0] * R[3] + T[1] * R[4] + T[2] * R[5];
    O[2] = T[3] * R[3] + T[4] * R[4] + T[5] * R[5];
    O[3] = T[0] * R[6] + T[1] * R[7] + T[2] * R[8];
    O[4] = T[3] * R[6] + T[4] * R[7] + T[5] * R[8];
    O[5] = T[6] * R[6] + T[7] * R[7] + T[8] * R[8];
}
// pinocchio::internal::SE3actOn: Y' = X* Y X*^T, X* = [[R,0],[[p]x R, R]]  (child -> parent)
//   A' = R A R^T ; B' = R B R^T - A' [p]x ; D' = R D R^T + [p]x B' + ([p]x R B R^T)^T
JB_DI void sym_transform(const Xf& M, const SymY& Y, SymY& O) {
    double Br[9], T[9];
    rot_sym(M.R, Y.A, O.A);
    mat3mul(M.R, Y.B, T);
    // Br = T R^T
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) Br[3 * i + j] = T[3 * i] * M.R[3 * j] + T[3 * i + 1] * M.R[3 * j + 1] + T[3 * i + 2] * M.R[3 * j + 2];
    rot_sym(M.R, Y.D, O.D);
    const double px = M.p.x, py = M.p.y, pz = M.p.z;
    // Ar [p]x : column j of [p]x is (e_j x p)... compute (Ar px)_{ik} = sum_j Ar_ij px_jk, px = [[0,-pz,py],[pz,0,-px],[-py,px,0]]
    const double a00 = O.A[0], a01 = O.A[1], a11 = O.A[2], a02 = O.A[3], a12 = O.A[4], a22 = O.A[5];
    double ApX[9];
    ApX[0] = a01 * pz - a02 * py; ApX[1] = -a00 * pz + a02 * px; ApX[2] = a00 * py - a01 * px;
    ApX[3] = a11 * pz - a12 * py; ApX[4] = -a01 * pz + a12 * px; ApX[5] = a01 * py - a11 * px;
    ApX[6] = a12 * pz - a22 * py; ApX[7] = -a02 * pz + a22 * px; ApX[8] = a02 * py - a12 * px;
#pragma unroll
    for (int k = 0; k < 9; ++k) O.B[k] = Br[k] - ApX[k];
    // px M : row i of (px M) = (p x column...) -> (px M)_{ij} = (p x M_col_j)_i
    // E = px B' ; F = px Br ; D' = Dr + E + F^T  (symmetric part kept)
    double E[9], F[9];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        E[0 + j] = py * O.B[6 + j] - pz * O.B[3 + j];
        E[3 + j] = pz * O.B[0 + j] - px * O.B[6 + j];
        E[6 + j] = px * O.B[3 + j] - py * O.B[0 + j];
        F[0 + j] = py * Br[6 + j] - pz * Br[3 + j];
        F[3 + j] = pz * Br[0 + j] - px * Br[6 + j];
        F[6 + j] = px * Br[3 + j] - py * Br[0 + j];
    }
    O.D[0] += E[0] + F[0];
    O.D[1] += E[1] + F[3];
    O.D[2] += E[4] + F[4];
    O.D[3] += E[2] + F[6];
    O.D[4] += E[5] + F[7];
    O.D[5] += E[8] + F[8];
}
JB_DI void quat_to_R(double x, double y, double z, double w, double* R) {  // Eigen::Quaternion::toRotationMatrix
    const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
    const double twx = tx * w, twy = ty * w, twz = tz * w;
    const double txx = tx * x, txy = ty * x, txz = tz * x;
    const double tyy = ty * y, tyz = tz * y, tzz = tz * z;
    R[0] = 1 - (tyy + tzz); R[1] = txy - twz;       R[2] = txz + twy;
    R[3] = txy + twz;       R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy;       R[7] = tyz + twx;       R[8] = 1 - (txx + tyy);
}
JB_DI void axis_angle_R(V3 ax, double ca, double sa, double* R) {  // Eigen::AngleAxis::toRotationMatrix
    const V3 sin_axis = sa * ax;
    const V3 cos1_axis = (1.0 - ca) * ax;
    double tmp;
    tmp = cos1_axis.x * ax.y; R[1] = tmp - sin_axis.z; R[3] = tmp + sin_axis.z;
    tmp = cos1_axis.x * ax.z; R[2] = tmp + sin_axis.y; R[6] = tmp - sin_axis.y;
    tmp = cos1_axis.y * ax.z; R[5] = tmp - sin_axis.x; R[7] = tmp + sin_axis.x;
    R[0] = cos1_axis.x * ax.x + ca; R[4] = cos1_axis.y * ax.y + ca; R[8] = cos1_axis.z * ax.z + ca;
}

// ---- unit quaternions, (x, y, z, w): the Lie group of JointModelSpherical (the flexibility joints).  Pinocchio 2.7.0
// explog-quaternion.hpp / SpecialOrthogonalOperationTpl<3> restated from the published algorithm, like the oracle's.
constexpr double TAYLOR_PREC3 = 1.220703125e-4;           // eps^(1/4)
constexpr double TAYLOR_PREC2 = 6.0554544523933395e-6;    // eps^(1/3)
constexpr double DBL_EPS2 = 2.220446049250313e-16 * 2.220446049250313e-16;
JB_DI void quat_mul(const double* a, const double* b, double* o) {   // Eigen: a * b
    const double x = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
    const double y = a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2];
    const double z = a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0];
    const double w = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
    o[0] = x; o[1] = y; o[2] = z; o[3] = w;
}
JB_DI void quat_exp3(V3 v, double* o) {   // quaternion::exp3
    const double t2 = dot(v, v);
    const double t = sqrt(t2 + DBL_EPS2);
    if (t2 > TAYLOR_PREC3 * TAYLOR_PREC3) {
        double sh, ch;
        sincos(0.5 * t, &sh, &ch);
        o[0] = sh * (v.x / t); o[1] = sh * (v.y / t); o[2] = sh * (v.z / t); o[3] = ch;
    } else {
        const double t2_2 = t2 / 4.0;
        const double k = 0.5 * (1.0 - t2_2 / 6.0 + t2_2 * t2_2 / 120.0);
        o[0] = k * v.x; o[1] = k * v.y; o[2] = k * v.z;
        o[3] = 1.0 - t2_2 / 2.0 + t2_2 * t2_2 / 24.0;
    }
}
JB_DI V3 quat_log3(const double* q, double& theta) {   // quaternion::log3
    const double norm_squared = q[0] * q[0] + q[1] * q[1] + q[2] * q[2];
    const double norm = sqrt(norm_squared + DBL_EPS2);
    const double pos_neg = q[3] >= 0.0 ? 1.0 : -1.0;
    const double w = pos_neg * q[3];
    const V3 vec = mk(pos_neg * q[0], pos_neg * q[1], pos_neg * q[2]);
    const double theta_2 = atan2(norm, w);
    const double y_x = norm / w;
    const double y_x_sq = norm_squared / (w * w);
    const bool small = norm_squared < TAYLOR_PREC2;
    theta = small ? 2.0 * (1.0 - y_x_sq / 3.0) * y_x : 2.0 * theta_2;
    const double th2_2 = theta * theta / 4.0;
    const double inv_sinc = small ? 2.0 * (1.0 + th2_2 / 6.0 + 7.0 / 360.0 * th2_2 * th2_2) : theta / sin(theta_2);
    return inv_sinc * vec;
}
// Jlog3(theta, log) applied to a vector: (alpha log log^T + diag 1 + [log / 2]x) x
JB_DI V3 jlog3_mul(double theta, V3 lg, V3 x) {
    double st, ct;
    sincos(theta, &st, &ct);
    const double st_1mct = st / (1.0 - ct);
    const bool small = theta < TAYLOR_PREC3;
    const double alpha = small ? 1.0 / 12.0 + theta * theta / 720.0 : 1.0 / (theta * theta) - st_1mct / (2.0 * theta);
    const double diag = small ? 0.5 * (2.0 - theta * theta / 6.0) : 0.5 * (theta * st_1mct);
    const V3 h = 0.5 * lg;
    // rows of Jlog, entry by entry like the reference builds the matrix, then the product
    const V3 r0 = mk(alpha * lg.x * lg.x + diag, alpha * lg.x * lg.y - h.z, alpha * lg.x * lg.z + h.y);
    const V3 r1 = mk(alpha * lg.y * lg.x + h.z, alpha * lg.y * lg.y + diag, alpha * lg.y * lg.z - h.x);
    const V3 r2 = mk(alpha * lg.z * lg.x - h.y, alpha * lg.z * lg.y + h.x, alpha * lg.z * lg.z + diag);
    return mk(dot(r0, x), dot(r1, x), dot(r2, x));
}
// SpecialOrthogonalOperationTpl<3>::difference_impl: log3(q0.conjugate() * q1)
JB_DI V3 difference_sph(const double* q0, const double* q1) {
    const double q0c[4] = {-q0[0], -q0[1], -q0[2], q0[3]};
    double dq[4], theta;
    quat_mul(q0c, q1, dq);
    return quat_log3(dq, theta);
}
// ------------------------------------------------------------------------------------------
// execution context of one lane
// ------------------------------------------------------------------------------------------
struct Ctx {
    int lane, sub, env;
    unsigned gmask;    // lanes of this env
    bool valid;
    int flags;         // CTX_* bits
};
// Engine::start, first INIT iteration (engine.cc:1400-1467): every joint effort is still zero, and the enabled
// constraints are solved as equalities (computeAcceleration(..., ignoreBounds = true))
constexpr int CTX_ZERO_U = 1, CTX_IGNORE_BOUNDS = 2;
// ... and the later INIT iterations see the multipliers of the enabled joint-bound constraints inside u: computeAcceleration
// adds them to uInternal and u (engine.cc:3770-3788) and the loop rebuilds u from that uInternal (engine.cc:1452-1461)
constexpr int CTX_START_FEEDBACK = 4;
// all 32 lanes of the warp entered a constraint solver together (see cons_solve_quadruped)
constexpr int CTX_UNIFORM_WARP = 8;

// ---- collectives among the L lanes of one env ------------------------------------------------------------------
// A warp-level primitive whose mask differs from lane to lane (eight env groups of four lanes, each naming its own
// lanes) is executed by the hardware one distinct mask after the other: ~8 passes for what looks like one instruction.
// When all 32 lanes are converged at the call -- the normal case on the hot path and inside the solvers -- the same
// result comes from ONE full-mask primitive: a full barrier is a group barrier, a shuffle reads the same absolute lane,
// a vote is a ballot restricted to the group's bits.  `__activemask()` is uniform over the lanes that execute it
// together, so all of them take the same branch; any other situation (groups apart, lanes retired) keeps the group mask.
#ifdef JB_HOST_EMUL
JB_DI void jb_syncwarp(const Ctx& c) { __syncwarp(c.gmask); }
JB_DI bool jb_any(const Ctx& c, bool p) { return __any_sync(c.gmask, p); }
JB_DI bool jb_all(const Ctx& c, bool p) { return __all_sync(c.gmask, p); }
JB_DI double jb_shfl(const Ctx& c, double x, int src) { return __shfl_sync(c.gmask, x, src); }
JB_DI double jb_shfl_xor(const Ctx& c, double x, int o) { return __shfl_xor_sync(c.gmask, x, o); }
JB_DI int jb_shfl_xor(const Ctx& c, int x, int o) { return __shfl_xor_sync(c.gmask, x, o); }
#else
JB_DI void jb_syncwarp(const Ctx& c) { if (__activemask() == 0xffffffffu) __syncwarp(); else __syncwarp(c.gmask); }
JB_DI bool jb_any(const Ctx& c, bool p) {
    if (__activemask() == 0xffffffffu) return (__ballot_sync(0xffffffffu, p) & c.gmask) != 0u;
    return __any_sync(c.gmask, p);
}
JB_DI bool jb_all(const Ctx& c, bool p) {
    if (__activemask() == 0xffffffffu) return (__ballot_sync(0xffffffffu, p) & c.gmask) == c.gmask;
    return __all_sync(c.gmask, p);
}
JB_DI double jb_shfl(const Ctx& c, double x, int src) {
    if (__activemask() == 0xffffffffu) return __shfl_sync(0xffffffffu, x, src);
    return __shfl_sync(c.gmask, x, src);
}
JB_DI double jb_shfl_xor(const Ctx& c, double x, int o) {
    if (__activemask() == 0xffffffffu) return __shfl_xor_sync(0xffffffffu, x, o);
    return __shfl_xor_sync(c.gmask, x, o);
}
JB_DI int jb_shfl_xor(const Ctx& c, int x, int o) {
    if (__activemask() == 0xffffffffu) return __shfl_xor_sync(0xffffffffu, x, o);
    return __shfl_xor_sync(c.gmask, x, o);
}
#endif
// sin and cos of a joint angle on the hot path.  Same construction as the library's (three-term Cody-Waite reduction by
// pi/2 carried by fused multiply-adds, the fdlibm kernels on [-pi/4, pi/4], quadrant swap; ~1 ulp) without what a joint
// angle never needs: the Payne-Hanek path for huge arguments, the special-value handling, the coefficient loads.
// Valid for |x| < 1e6 rad (the reduction keeps full accuracy up to ~1e5, like the library's fast path).
JB_DI void jb_sincos(const double x, double* s, double* c) {
    const double t = fma(x, 0.63661977236758138, 6755399441055744.0);   // x * 2/pi rounded to nearest integer, in the low bits
    const double kd = t - 6755399441055744.0;
#ifdef JB_HOST_EMUL
    long long tb; std::memcpy(&tb, &t, sizeof tb);
    const int k = static_cast<int>(tb & 0xffffffffll);
#else
    const int k = __double2loint(t);
#endif
    double r = fma(-kd, 1.5707963267948966e+00, x);
    r = fma(-kd, 6.1232339957367574e-17, r);
    r = fma(-kd, 8.4784276603688985e-32, r);
    const double z = r * r;
    double ps = fma(z, 1.58969099521155010221e-10, -2.50507602534068634195e-08);
    double pc = fma(z, -1.13596475577881948265e-11, 2.08757232129817482790e-09);
    ps = fma(ps, z, 2.75573137070700676789e-06);   pc = fma(pc, z, -2.75573143513906633035e-07);
    ps = fma(ps, z, -1.98412698298579493134e-04);  pc = fma(pc, z, 2.48015872894767294178e-05);
    ps = fma(ps, z, 8.33333333332248946124e-03);   pc = fma(pc, z, -1.38888888888741095749e-03);
    ps = fma(ps, z, -1.66666666666666324348e-01);  pc = fma(pc, z, 4.16666666666666019037e-02);
    const double sr = fma(ps * z, r, r);                       // r + r^3 S(z)
    const double cr = fma(z * z, pc, fma(-0.5, z, 1.0));       // 1 - z/2 + z^2 C(z)
    const double a = (k & 1) ? cr : sr, b = (k & 1) ? sr : cr;
    *s = (k & 2) ? -a : a;
    *c = ((k + 1) & 2) ? -b : b;
}
#define SMF(c, off) (jb_smem[(off) * 32 + (c).lane])   // field `off` of this lane
#define RP(off) (rp[(off) * 32])   // field of the current record  (rp = record base of this lane)
#define PO(off) (pp[(off) * 32])   // field of the current pool entry
#define CO(off) (cp[(off) * 32])   // field of the current contact slot

JB_DI void sm_store_xf(const Ctx& c, int off, const Xf& M) {
    double* const p = jb_smem + off * 32 + c.lane;
#pragma unroll
    for (int k = 0; k < 9; ++k) p[k * 32] = M.R[k];
    p[9 * 32] = M.p.x; p[10 * 32] = M.p.y; p[11 * 32] = M.p.z;
}
JB_DI void sm_load_xf(const Ctx& c, int off, Xf& M) {
    const double* const p = jb_smem + off * 32 + c.lane;
#pragma unroll
    for (int k = 0; k < 9; ++k) M.R[k] = p[k * 32];
    M.p = mk(p[9 * 32], p[10 * 32], p[11 * 32]);
}
JB_DI void sm_store_mot(const Ctx& c, int off, Mot m) {
    double* const p = jb_smem + off * 32 + c.lane;
    p[0] = m.l.x; p[32] = m.l.y; p[64] = m.l.z; p[96] = m.a.x; p[128] = m.a.y; p[160] = m.a.z;
}
JB_DI Mot sm_load_mot(const Ctx& c, int off) {
    const double* const p = jb_smem + off * 32 + c.lane;
    Mot m;
    m.l = mk(p[0], p[32], p[64]);
    m.a = mk(p[96], p[128], p[160]);
    return m;
}
JB_DI V3 ld3(const double* p) { return mk(p[0], p[1], p[2]); }

// record kind of this lane: from constant memory when all lanes agree (0 = mixed -> per-lane table)
JB_DI int lane_kind(int r, const Ctx& c) {
    const int ku = KP->kind_u[r];
    return ku ? ku : (KP->rint + (r * KP->L + c.sub))->kind;
}
JB_DI double group_sum(double x, const Ctx& c, int L) {
    for (int o = 1; o < L; o <<= 1) x += jb_shfl_xor(c, x, o);
    return x;
}

// Engine::computeContactDynamics (core/src/engine/engine.cc:3197-3238), flat ground n = z.
JB_DI V3 contact_dynamics(const JbOptions& o, double depth, V3 vw) {
    const double vDepth = vw.z;
    const double fN = -fmin(o.contact_stiffness * depth + o.contact_damping * vDepth, 0.0);
    const V3 vT = mk(vw.x, vw.y, 0.0);   // v - vDepth * n
    const double vRatio = fmin(sqrt(vT.x * vT.x + vT.y * vT.y) / o.contact_transition_velocity, 1.0);
    const double fT = o.contact_friction * vRatio * fN;
    V3 f = mk(-fT * vT.x, -fT * vT.y, fN);
    if (o.contact_transition_eps > D_EPS) {
        const double blend = tanh(2.0 * (-depth / o.contact_transition_eps));
        f = blend * f;
    }
    return f;
}
// The same law without a branch, for a depth clamped to <= 0 (the caller selects the result by the sign of the unclamped
// depth): the blend is a select on the host-computed -2 / transitionEps, the divisions are products with host-computed
// reciprocals.  Finite for every finite input, depth 0 and zero sliding velocity included.
JB_DI V3 contact_dynamics_nb(const JbOptions& o, double depth, V3 vw) {
    const double vDepth = vw.z;
    const double fN = -fmin(o.contact_stiffness * depth + o.contact_damping * vDepth, 0.0);
    const double vRatio = fmin(sqrt(vw.x * vw.x + vw.y * vw.y) * KP->contact_inv_vt, 1.0);
    const double fT = o.contact_friction * vRatio * fN;
    const double bk = KP->contact_blend_k;
    const double blend = bk != 0.0 ? tanh(depth * bk) : 1.0;
    return mk(blend * (-fT * vw.x), blend * (-fT * vw.y), blend * fN);
}

// Motor constants the forward sweep needs, fetched at the top of a record (four 16-byte loads issued together with
// the joint constants) so that their latency is hidden behind the kinematics instead of stalling computeEffort.
struct MotorConst { double red, effLim, velLim, invSlope, invSpan, thr; };
JB_DI MotorConst load_motor_const(const RecDbl* rd) {
    MotorConst m;
#ifdef JB_HOST_EMUL
    m.red = rd->motor[0]; m.effLim = rd->motor[1]; m.velLim = rd->motor[2]; m.invSlope = rd->motor[3]; m.invSpan = rd->motor[9]; m.thr = rd->pad;
#else
    const double2* p = reinterpret_cast<const double2*>(rd->motor);   // RecDbl: motor[] starts at double 28 -> 16-byte aligned
    const double2 a = __ldg(p), b = __ldg(p + 1), c = __ldg(p + 4), d = __ldg(p + 5);
    m.red = a.x; m.effLim = a.y; m.velLim = b.x; m.invSlope = b.y; m.invSpan = c.y; m.thr = d.y;   // motor[8..9] | enc_reduction, pad
#endif
    return m;
}
JB_DI void motor_effort_pre(const MotorConst& mc, const RecDbl* rd, int flags, double cmd, double vj, double& uMotor, double& uTrans) {
    const double vMotor = mc.red * vj;
    double eMin = -D_INF, eMax = D_INF;
    if (flags & 1) {
        eMin = -mc.effLim; eMax = mc.effLim;
        if (flags & 2) {
            const double velocityDelta = mc.effLim * mc.invSlope;
            if (velocityDelta > 0.0 && fabs(vMotor) > mc.thr) {
                eMin *= fmin(fmax((mc.velLim + vMotor) * mc.invSpan, 0.0), 1.0);
                eMax *= fmin(fmax((mc.velLim - vMotor) * mc.invSpan, 0.0), 1.0);
            }
        }
    }
    uMotor = fmin(fmax(cmd, eMin), eMax);
    uTrans = mc.red * uMotor;
    if (flags & 4) {
        if (vj > 0.0) uTrans += rd->motor[4] * vj + rd->motor[6] * tanh(rd->motor[8] * vj);
        else uTrans += rd->motor[5] * vj + rd->motor[7] * tanh(rd->motor[8] * vj);
    }
}
// motor_effort_pre for flags 3 (effort limit and velocity taper, no friction) with the taper as a select, not a branch
JB_DI void motor_effort_limited_nb(const MotorConst& mc, double cmd, double vj, double& uMotor, double& uTrans) {
    const double vMotor = mc.red * vj;
    const bool taper = mc.effLim * mc.invSlope > 0.0 && fabs(vMotor) > mc.thr;
    const double kMin = fmin(fmax((mc.velLim + vMotor) * mc.invSpan, 0.0), 1.0);
    const double kMax = fmin(fmax((mc.velLim - vMotor) * mc.invSpan, 0.0), 1.0);
    const double eMin = taper ? -mc.effLim * kMin : -mc.effLim, eMax = taper ? mc.effLim * kMax : mc.effLim;
    uMotor = fmin(fmax(cmd, eMin), eMax);
    uTrans = mc.red * uMotor;
}

// SimpleMotor::computeEffort (core/src/hardware/basic_motors.cc:83-143)
JB_DI void motor_effort(const RecDbl* rd, int flags, double cmd, double vj, double& uMotor, double& uTrans) {
    const double red = rd->motor[0], effLim = rd->motor[1], velLim = rd->motor[2], invSlope = rd->motor[3];
    const double vMotor = red * vj;
    double eMin = -D_INF, eMax = D_INF;
    if (flags & 1) {
        eMin = -effLim; eMax = effLim;
        if (flags & 2) {
            const double velocityDelta = effLim * invSlope;
            // below the taper threshold both factors are exactly 1 (rd->pad holds velocityThr)
            if (velocityDelta > 0.0 && fabs(vMotor) > rd->pad) {
                const double invSpan = rd->motor[9];   // 1 / (velLim - velocityThr), precomputed by the planner
                eMin *= fmin(fmax((velLim + vMotor) * invSpan, 0.0), 1.0);
                eMax *= fmin(fmax((velLim - vMotor) * invSpan, 0.0), 1.0);
            }
        }
    }
    uMotor = fmin(fmax(cmd, eMin), eMax);
    uTrans = red * uMotor;
    if (flags & 4) {
        if (vj > 0.0) uTrans += rd->motor[4] * vj + rd->motor[6] * tanh(rd->motor[8] * vj);
        else uTrans += rd->motor[5] * vj + rd->motor[7] * tanh(rd->motor[8] * vj);
    }
}

// 6x6 SPD solve Y x = b for the free-flyer root.  The reference inverts S^T Y S with an LLT
// (PerformStYSInversion, core/include/jiminy/core/robot/pinocchio_overload_algorithms.h:358-378); a
// Cholesky factorisation is a chain of six dependent rsqrt steps, which is the worst shape for a
// lane that has no second warp to hide latency behind.  Same solution through the 3x3 block Schur
// complement of Y = [[A, B], [B^T, D]] (A, D symmetric positive definite): two adjugate inverses,
// two divisions, dependency depth ~15.
JB_DI void sym3_inverse(const double* S, double* I) {   // (xx,xy,yy,xz,yz,zz) -> same order
    const double c00 = S[2] * S[5] - S[4] * S[4];
    const double c01 = S[3] * S[4] - S[1] * S[5];
    const double c02 = S[1] * S[4] - S[3] * S[2];
    const double inv_det = 1.0 / (S[0] * c00 + S[1] * c01 + S[3] * c02);
    I[0] = c00 * inv_det;
    I[1] = c01 * inv_det;
    I[2] = (S[0] * S[5] - S[3] * S[3]) * inv_det;
    I[3] = c02 * inv_det;
    I[4] = (S[1] * S[3] - S[0] * S[4]) * inv_det;
    I[5] = (S[0] * S[2] - S[1] * S[1]) * inv_det;
}
JB_DI void spd_solve6(const SymY& Y, const double* b, double* x) {
    double Ai[6];
    sym3_inverse(Y.A, Ai);
    // T = A^-1 B (3x3), columns of B transformed by the symmetric A^-1
    double T[9];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        const V3 col = symmul(Ai, mk(Y.B[j], Y.B[3 + j], Y.B[6 + j]));
        T[j] = col.x; T[3 + j] = col.y; T[6 + j] = col.z;
    }
    // S = D - B^T T (symmetric)
    double S[6];
    S[0] = Y.D[0] - (Y.B[0] * T[0] + Y.B[3] * T[3] + Y.B[6] * T[6]);
    S[1] = Y.D[1] - (Y.B[0] * T[1] + Y.B[3] * T[4] + Y.B[6] * T[7]);
    S[2] = Y.D[2] - (Y.B[1] * T[1] + Y.B[4] * T[4] + Y.B[7] * T[7]);
    S[3] = Y.D[3] - (Y.B[0] * T[2] + Y.B[3] * T[5] + Y.B[6] * T[8]);
    S[4] = Y.D[4] - (Y.B[1] * T[2] + Y.B[4] * T[5] + Y.B[7] * T[8]);
    S[5] = Y.D[5] - (Y.B[2] * T[2] + Y.B[5] * T[5] + Y.B[8] * T[8]);
    double Si[6];
    sym3_inverse(S, Si);
    const V3 y1 = symmul(Ai, mk(b[0], b[1], b[2]));
    const V3 r2 = mk(b[3], b[4], b[5]) - rtmul(Y.B, y1);
    const V3 x2 = symmul(Si, r2);
    const V3 x1 = y1 - rmul(T, x2);
    x[0] = x1.x; x[1] = x1.y; x[2] = x1.z; x[3] = x2.x; x[4] = x2.y; x[5] = x2.z;
}

#include "jb_constraints.cuh"
#include "jb_constraints_quadruped.cuh"
#include "jb_constraints_blocks.cuh"
#include "jb_constraints_bodies.cuh"

// ------------------------------------------------------------------------------------------
// The ODE right-hand side:  Engine::computeRobotsDynamics (core/src/engine/engine.cc:3585-3708)
//   = forward kinematics (:2957-3014) + contact forces (:3117-3238, :3394-3425,
//     utilities/pinocchio.cc:794-809) + motor efforts (:3683-3702) + ABA with rotor inertia
//     (pinocchio_overload_algorithms.h:446-489).
// Evaluated at the *stage* state (fields QS / VS of every record), writes ddq into the A fields.
// `up_to_date` reuses the cached contact forces (engine.cc:3411-3414).
//
// UNIFORM = true: every record has the same descriptor on all lanes (symmetric robots such as
// ANYmal): the descriptor is read from constant memory, so that all per-record control flow is
// warp-uniform and costs no memory latency.  Otherwise the per-lane row is fetched from global
// memory with five 16-byte loads issued back to back.  Per-lane joint constants (placement, axis,
// inertia, ...) are always fetched up front with 16-byte loads, so that their latency overlaps.
// ------------------------------------------------------------------------------------------
struct RecConst {   // the first 28 doubles of a RecDbl row
    double placement[12]; double axis[3]; double inertia[10]; double armature, q_lo, q_hi;
};
JB_DI void load_doubles(const double* __restrict__ src, double* dst, int n2) {   // n2 16-byte pairs
#ifdef JB_HOST_EMUL
    for (int k = 0; k < 2 * n2; ++k) dst[k] = src[k];
#else
    const double2* s2 = reinterpret_cast<const double2*>(src);
#pragma unroll
    for (int k = 0; k < n2; ++k) { const double2 t = __ldg(s2 + k); dst[2 * k] = t.x; dst[2 * k + 1] = t.y; }
#endif
}
template <bool UNIFORM>
JB_DI RecInt fetch_recint(int r, int L, int sub) {
    if (UNIFORM) return KP->rint_u[r];
    RecInt out;
#ifdef JB_HOST_EMUL
    out = KP->rint[r * L + sub];
#else
    const int4* s4 = reinterpret_cast<const int4*>(KP->rint + (r * L + sub));
    int4* d4 = reinterpret_cast<int4*>(&out);
#pragma unroll
    for (int k = 0; k < static_cast<int>(sizeof(RecInt) / 16); ++k) d4[k] = __ldg(s4 + k);
#endif
    return out;
}

// ---- plan signatures: how rhs_impl learns the shape of the lane plan ----------------------------
// SigDynamic reads everything at run time (any robot).  A static signature describes one lane-uniform
// plan at compile time: the record loop unrolls, every per-record branch folds away, shared-memory
// offsets become immediates, and the scheduler can overlap the independent head of record r + 1
// (constant loads, sincos, placement product) with the dependent tail of record r.
template <int N> struct IntC { JB_HD constexpr operator int() const { return N; } };
template <bool UNIFORM, bool EXT = true>
struct SigDynamic {
    static constexpr bool has_ext = EXT;     // external-force slots are honoured
    static constexpr bool has_cons = EXT;    // constraint contacts and the start-time evaluation flags are honoured
    static constexpr bool pool_single_writer = false;
    JB_DI static int lanes() { return KP->L; }
    JB_DI static int ntrunk() { return KP->ntrunk; }
    JB_DI static int npool() { return KP->npool; }
    JB_DI static int rec_off(int r) { return KP->rec_off[r]; }
    JB_DI static int pool_off() { return KP->pool_off; }
    JB_DI static int cslot_off() { return KP->cslot_off; }
    JB_DI static int imu_off() { return KP->imu_off; }
    JB_DI static bool trunk_reduce(int r) { return KP->trunk_reduce[r]; }
    JB_DI static RecInt rec(int r, int L, int sub) { return fetch_recint<UNIFORM>(r, L, sub); }
    JB_DI static int kind(int r, const Ctx& c) { return lane_kind(r, c); }
    template <class F> JB_DI static void for_each_forward(F&& f) {
#pragma unroll 1
        for (int r = 0; r < KP->nrec; ++r) f(r);
    }
    template <class F> JB_DI static void for_each_backward(F&& f) {
#pragma unroll 1
        for (int r = KP->nrec - 1; r >= 0; --r) f(r);
    }
};
// Quadruped-like plan (ANYmal): L = 4, one trunk free-flyer carrying the IMU, then a chain of three
// motorised, bounded revolute joints about +-x per lane with one contact frame on the last one.
template <bool CONS>
struct SigQuadrupedT {
    static constexpr int ID = 1;
    static constexpr bool has_ext = false;   // the host falls back to SigDynamic when forces are registered
    static constexpr bool has_cons = CONS;   // second instance of the sweeps for `contacts.model = constraint`
    // every lane adds exactly one contribution (its first leg record) to the trunk's pool accumulator: it can be
    // stored instead of zeroed and accumulated
    static constexpr bool pool_single_writer = true;
    JB_HD static constexpr int lanes() { return 4; }
    JB_HD static constexpr int ntrunk() { return 1; }
    JB_HD static constexpr int npool() { return 1; }
    JB_HD static constexpr int rec_off(int r) { return r == 0 ? 0 : (r == 1 ? RF_KA : (r == 2 ? RF_KA + R1_KA : RF_KA + 2 * R1_KA)); }
    JB_HD static constexpr int pool_off() { return RF_KA + 3 * R1_KA; }
    JB_HD static constexpr int cslot_off() { return pool_off() + POOL_SIZE; }
    JB_HD static constexpr int imu_off() { return cslot_off() + CSLOT_SIZE; }
    JB_HD static constexpr bool trunk_reduce(int r) { return r == 0; }
    JB_HD static constexpr RecInt rec(int r, int, int) {
        RecInt d{};
        d.kind = r == 0 ? REC_FREE : REC_REVX;
        d.joint = 0; d.parent_rec = r - 1;
        d.carry_in = r >= 2; d.carry_out = r >= 2;
        d.pool = r == 0 ? 0 : -1; d.parent_pool = r == 1 ? 0 : -1;
        d.take_carry = (r == 1 || r == 2);
        d.idx_q = 0; d.idx_v = 0;
        d.motor = r == 0 ? -1 : 0; d.motor_flags = r == 0 ? 0 : 3;
        d.ncontact = r == 3 ? 1 : 0; d.contact0 = 0;
        d.imu = r == 0 ? 0 : -1; d.owner = 1; d.has_limit = r != 0; d.encoder = -1; d.effort = -1;
        d.imu_slot = r == 0 ? 0 : -1;
        return d;
    }
    JB_HD static constexpr int kind(int r, const Ctx&) { return r == 0 ? REC_FREE : REC_REVX; }
    template <class F> JB_DI static void for_each_forward(F&& f) { f(IntC<0>{}); f(IntC<1>{}); f(IntC<2>{}); f(IntC<3>{}); }
    template <class F> JB_DI static void for_each_backward(F&& f) { f(IntC<3>{}); f(IntC<2>{}); f(IntC<1>{}); f(IntC<0>{}); }
    // does a run-time plan have exactly this shape?  (host side, at batch creation)
    static bool matches(const KParams& kp) {
        if (!kp.all_uniform || kp.L != 4 || kp.nrec != 4 || kp.ntrunk != 1 || kp.npool != 1 || kp.ncslot != 1 ||
            kp.nimuslot != 1 || kp.n_hist != 0 || kp.pool_off != pool_off() || kp.cslot_off != cslot_off() ||
            kp.imu_off != imu_off())
            return false;
        for (int r = 0; r < 4; ++r) {
            const RecInt a = kp.rint_u[r], b = rec(r, 4, 0);
            if (kp.rec_off[r] != rec_off(r) || (kp.trunk_reduce[r] != 0) != trunk_reduce(r)) return false;
            if (a.kind != b.kind || a.parent_rec != b.parent_rec || a.carry_in != b.carry_in || a.pool != b.pool ||
                a.parent_pool != b.parent_pool || a.carry_out != b.carry_out || a.take_carry != b.take_carry ||
                (a.motor >= 0) != (b.motor >= 0) || a.motor_flags != b.motor_flags || a.ncontact != b.ncontact ||
                a.contact0 != b.contact0 || a.imu_slot != b.imu_slot || a.has_limit != b.has_limit)
                return false;
        }
        return true;
    }
};
using SigQuadruped = SigQuadrupedT<false>;
using SigQuadrupedCons = SigQuadrupedT<true>;

template <class SIG>
JB_DI bool rhs_impl(const Ctx c, const bool up_to_date, int* status) {
    const int L = SIG::lanes();
    const JbOptions& opt = KP->opt;
    bool out_of_bounds = false;   // a bounded joint of this lane is outside [lo, hi] (handled by the caller, rhs())
    // ======================= pass 1: kinematics, bias terms, contacts, motors =================
    {
        Xf oMc; Mot vc = mzero();   // (oMi, v) of the previous record
        bool out_any = false;       // a bounded joint of this lane is outside [lo, hi]
#pragma unroll
        for (int k = 0; k < 9; ++k) oMc.R[k] = 0.0;
        oMc.p = mk(0, 0, 0);
        auto body = [&](auto r_) {
            const int r = r_;
            const RecInt ri = SIG::rec(r, L, c.sub);
            const int kind = ri.kind;
            if (kind == REC_PAD) return;
            const RecDbl* rd = JB_RDBL + (r * L + c.sub);
            RecConst K;
            load_doubles(rd->placement, K.placement, 14);
            MotorConst mc{};
            if (ri.motor >= 0) mc = load_motor_const(rd);
            const int base = SIG::rec_off(r);
            double* const rp = jb_smem + base * 32 + c.lane;
            // parent kinematics, in place in the carry variables
            if (ri.parent_rec >= 0 && !ri.carry_in) {
                const int po = SIG::pool_off() + POOL_SIZE * ri.parent_pool;
                sm_load_xf(c, po, oMc);
                vc = sm_load_mot(c, po + 12);
            }
            // joint transform  (JointModel*::calc of Pinocchio 2.7)
            Xf li; Mot vJ = mzero();
            const V3 ax = ld3(K.axis);
            double qd = 0.0;
            if (kind == REC_FREE) {
                double Rq[9];
                quat_to_R(RP(RF_QS + 3), RP(RF_QS + 4), RP(RF_QS + 5), RP(RF_QS + 6), Rq);
                mat3mul(K.placement, Rq, li.R);
                li.p = ld3(K.placement + 9) + rmul(K.placement, mk(RP(RF_QS), RP(RF_QS + 1), RP(RF_QS + 2)));
                vJ = sm_load_mot(c, base + RF_VS);
            } else if (kind == REC_SPH) {
                // JointModelSphericalTpl::calc: M = (quat.matrix(), 0), v = (0, omega)
                double Rq[9];
                quat_to_R(RP(RF_QS + 3), RP(RF_QS + 4), RP(RF_QS + 5), RP(RF_QS + 6), Rq);
                mat3mul(K.placement, Rq, li.R);
                li.p = ld3(K.placement + 9);
                vJ.a = mk(RP(RF_VS + 3), RP(RF_VS + 4), RP(RF_VS + 5));
            } else if (kind == REC_PRISM) {
#pragma unroll
                for (int k = 0; k < 9; ++k) li.R[k] = K.placement[k];
                li.p = ld3(K.placement + 9) + rmul(K.placement, RP(R1_QS) * ax);
                qd = RP(R1_VS);
                vJ.l = qd * ax;
            } else if (kind == REC_REVX) {
                // revolute about +-x of the joint frame (JointModelRX, or RevoluteUnaligned with axis -x):
                // liMi.R = Rp Rx(+-q) touches two columns only
                double ca, sa;
                sincos(RP(R1_QS), &sa, &ca);
                const double s = ax.x * sa;
#pragma unroll
                for (int i = 0; i < 3; ++i) {
                    li.R[3 * i] = K.placement[3 * i];
                    li.R[3 * i + 1] = ca * K.placement[3 * i + 1] + s * K.placement[3 * i + 2];
                    li.R[3 * i + 2] = ca * K.placement[3 * i + 2] - s * K.placement[3 * i + 1];
                }
                li.p = ld3(K.placement + 9);
                qd = RP(R1_VS);
                vJ.a = mk(ax.x * qd, 0.0, 0.0);
            } else {
                double ca, sa;
                if (kind == REC_REVU) { ca = RP(R1_QS); sa = RP(R1_QS + 1); }
                else sincos(RP(R1_QS), &sa, &ca);
                double Rj[9];
                axis_angle_R(ax, ca, sa, Rj);
                mat3mul(K.placement, Rj, li.R);
                li.p = ld3(K.placement + 9);
                qd = RP(R1_VS);
                vJ.a = qd * ax;
            }
            // oMi = oMi[parent] * liMi ; v = vJ + liMi.actInv(v[parent]) ; a_gf bias = v x vJ (c == 0 for
            // every supported joint).  A child of the universe has oMi = liMi, v = vJ, bias = 0.
            Xf oM; Mot v, bias;
            if (ri.parent_rec < 0) {
                oM = li; v = vJ; bias = mzero();
            } else {
                mat3mul(oMc.R, li.R, oM.R);
                oM.p = oMc.p + rmul(oMc.R, li.p);
                v = motion_act_inv(li, vc) + vJ;
                if (kind == REC_PRISM) { bias.l = cross(v.a, vJ.l); bias.a = mk(0, 0, 0); }
                else if (kind == REC_REVX) {
                    const double w = vJ.a.x;
                    bias.l = mk(0.0, v.l.z * w, -v.l.y * w); bias.a = mk(0.0, v.a.z * w, -v.a.y * w);
                }
                else if (rec_is_big(kind)) bias = motion_cross(v, vJ);
                else { bias.l = cross(v.l, vJ.a); bias.a = cross(v.a, vJ.a); }
            }
            // f = v x* (I v)
            Mot f = motion_cross_force(v, inertia_mul(K.inertia[0], ld3(K.inertia + 1), K.inertia + 4, v));
            // contact forces on this joint
            if (ri.ncontact > 0) {
                Mot fext = mzero();
                for (int k = 0; k < ri.ncontact; ++k) {
                    const int cs = ri.contact0 + k;
                    const ContactSlot* ct = KP->cslots + (cs * L + c.sub);
                    const int co = SIG::cslot_off() + CSLOT_SIZE * cs;
                    double* const cp = jb_smem + co * 32 + c.lane;
                    const V3 pc = ld3(ct->placement + 9);
                    V3 Fl;
                    if (SIG::has_cons && opt.contact_model == JB_CONTACT_CONSTRAINT) {
                        // constraint contact model: the wrench comes out of the constraint solver afterwards
                        if (!up_to_date) {
                            if (ct->contact >= 0) cons_update_contact(c, ct->contact, oM, ct->placement, (KP->rint + (r * L + c.sub))->owner != 0);
#pragma unroll
                            for (int e = 0; e < CSLOT_SIZE; ++e) CO(e) = 0.0;
                        }
                        continue;
                    }
                    if (!up_to_date) {
                        // Engine::computeContactDynamicsAtFrame (engine.cc:3117-3195)
                        const V3 pos = oM.p + rmul(oM.R, pc);
                        const double depth = pos.z;   // (z - 0) * n_z, flat ground (engine.h:292-302)
                        Fl = mk(0, 0, 0);
                        if (depth < 0.0) {
                            // world velocity of the contact point: R_f * (P.actInv(v).linear)
                            const V3 vw = rmul(oM.R, v.l + cross(v.a, pc));
                            const V3 fw = contact_dynamics(opt, depth, vw);
                            Fl = rtmul(oM.R, fw);   // convertForceGlobalFrameToJoint (utilities/pinocchio.cc:794-809)
                        }
                        CO(0) = Fl.x; CO(1) = Fl.y; CO(2) = Fl.z;
                    } else {
                        Fl = mk(CO(0), CO(1), CO(2));
                    }
                    fext.l = fext.l + Fl;
                    fext.a = fext.a + cross(pc, Fl);
                }
                f = f - fext;
            }
            // impulse / profile forces on this joint (Engine::computeExternalForces, engine.cc:3455-3495)
            if (SIG::has_ext && KP->n_eslot > 0) {
                for (int e = 0; e < KP->n_eslot; ++e) {
                    const ExtSlot* es = KP->eslots + (e * L + c.sub);
                    if (es->rec != r) continue;
                    double* const xp = jb_smem + (KP->ext_off + ESLOT_SIZE * e) * 32 + c.lane;
                    // convertForceGlobalFrameToJoint (utilities/pinocchio.cc:794-809)
                    const V3 Fl = rtmul(oM.R, mk(xp[0], xp[32], xp[64]));
                    const V3 Fa = rtmul(oM.R, mk(xp[96], xp[128], xp[160])) + cross(ld3(es->p), Fl);
                    xp[6 * 32] = Fl.x; xp[7 * 32] = Fl.y; xp[8 * 32] = Fl.z;
                    xp[9 * 32] = Fa.x; xp[10 * 32] = Fa.y; xp[11 * 32] = Fa.z;
                    f.l = f.l - Fl; f.a = f.a - Fa;
                }
            }
            // joint efforts: u = uInternal + uCustom + uTransmission (engine.cc:3694-3702)
            if (kind == REC_SPH) {
                // flexibility joint (Engine::computeInternalDynamics, engine.cc:3367-3391):
                // uInternal = -Jlog3(angle, angleAxis) (stiffness o angleAxis) - damping o omega
                const double qs[4] = {RP(RF_QS + 3), RP(RF_QS + 4), RP(RF_QS + 5), RP(RF_QS + 6)};
                double angle;
                const V3 aa = quat_log3(qs, angle);
                const V3 t = jlog3_mul(angle, aa, mk(rd->motor[0] * aa.x, rd->motor[1] * aa.y, rd->motor[2] * aa.z));
                const bool zero = SIG::has_cons && (c.flags & CTX_ZERO_U);
                double* const xp = rp + KP->sph_off * 32;
                xp[(RS_TAU + 0) * 32] = zero ? 0.0 : (0.0 - t.x) - rd->motor[3] * vJ.a.x;
                xp[(RS_TAU + 1) * 32] = zero ? 0.0 : (0.0 - t.y) - rd->motor[4] * vJ.a.y;
                xp[(RS_TAU + 2) * 32] = zero ? 0.0 : (0.0 - t.z) - rd->motor[5] * vJ.a.z;
                sm_store_xf(c, base + RF_LIMI, li);
                sm_store_mot(c, base + RF_F, f);
                sm_store_mot(c, base + KP->sph_off + RS_BIAS, bias);
            } else if (kind != REC_FREE) {
                double u = 0.0;
                if (KP->springs != nullptr && kind != REC_REVU)
                {
                    const int iv = (KP->rint + (r * L + c.sub))->idx_v;   // per-lane index even on the uniform path
                    u = -KP->springs[iv] * RP(R1_QS) - KP->springs[KP->nv + iv] * qd;
                }
                if (ri.motor >= 0) {
                    double uM, uT;
                    motor_effort_pre(mc, rd, ri.motor_flags, RP(R1_CMD), qd, uM, uT);
                    RP(R1_UMOTOR) = uM;
                    u += uT;
                }
                if (SIG::has_cons && (c.flags & CTX_START_FEEDBACK)) {
                    const int kc = KP->jc_of_joint[(KP->rint + (r * L + c.sub))->joint];
                    if (kc >= 0 && CST(cs_joint(kc)) != 0.0) u += CST(cs_joint(kc) + 3);
                }
                RP(R1_U) = (SIG::has_cons && (c.flags & CTX_ZERO_U)) ? 0.0 : u;
                // joint position bounds: only detected here, handled after the sweep (off the unrolled hot path)
                if (ri.has_limit && !up_to_date) {
                    const double qj = RP(R1_QS);
                    out_any = out_any || K.q_hi < qj || qj < K.q_lo;
                }
                sm_store_xf(c, base + R1_LIMI, li);
                sm_store_mot(c, base + R1_BIAS, bias);
                sm_store_mot(c, base + R1_FU, f);
            } else {
                sm_store_xf(c, base + RF_LIMI, li);
                sm_store_mot(c, base + RF_F, f);
            }
            if (ri.pool >= 0) {
                const int po = SIG::pool_off() + POOL_SIZE * ri.pool;
                sm_store_xf(c, po, oM);
                sm_store_mot(c, po + 12, v);
            }
            if (ri.imu_slot >= 0) sm_store_mot(c, SIG::imu_off() + IMUSLOT_SIZE * ri.imu_slot, v);
            oMc = oM; vc = v;
        };
        SIG::template for_each_forward(body);
        out_of_bounds = out_any;
    }
    jb_syncwarp(c);
    // ======================= pass 2: backward sweep (AbaBackwardStep) ==========================
    {
        // the pool entries become (Y, f) accumulators
        if (!SIG::pool_single_writer)
            for (int k = 0; k < POOL_SIZE * SIG::npool(); ++k) SMF(c, SIG::pool_off() + k) = 0.0;
        SymY Yc; Mot fc = mzero();   // contribution of record r + 1 to its parent (when that is record r)
#pragma unroll
        for (int k = 0; k < 6; ++k) { Yc.A[k] = 0; Yc.D[k] = 0; }
#pragma unroll
        for (int k = 0; k < 9; ++k) Yc.B[k] = 0;
        auto body = [&](auto r_) {
            const int r = r_;
            const RecInt ri = SIG::rec(r, L, c.sub);
            const int kind = ri.kind;
            const bool reduce = (r < SIG::ntrunk()) && SIG::trunk_reduce(r) && L > 1;
            // every lane of the env holds a partial accumulator for this trunk joint: make them visible
            if (reduce) jb_syncwarp(c);
            if (kind == REC_PAD) return;
            const RecDbl* rd = JB_RDBL + (r * L + c.sub);
            double Kd[14];   // axis (3), inertia (10), armature
            // RecDbl: placement[12] | axis[3] inertia[10] armature : doubles 12..25 -> 7 aligned 16-byte pairs
            load_doubles(rd->placement + 12, Kd, 7);
            const V3 ax = mk(Kd[0], Kd[1], Kd[2]);
            const int base = SIG::rec_off(r);
            double* const rp = jb_smem + base * 32 + c.lane;
            SymY Y;
            inertia_to_sym(Kd[3], mk(Kd[4], Kd[5], Kd[6]), Kd + 7, Y);
            Mot f = sm_load_mot(c, base + (rec_is_big(kind) ? RF_F : R1_FU));
            if (ri.take_carry) { sym_add(Y, Yc); f = f + fc; }
            if (ri.pool >= 0) {
                const int po = SIG::pool_off() + POOL_SIZE * ri.pool;
                if (reduce) {
                    // trunk joint: all-reduce over the L lanes of the env straight out of shared memory,
                    // every lane summing the L partial accumulators in the same (sub-lane) order so that
                    // the trunk stays bit-identical on all lanes
                    const double* const p0 = jb_smem + po * 32 + (c.lane - c.sub);
                    for (int s = 0; s < L; ++s) {
#pragma unroll
                        for (int k = 0; k < 6; ++k) { Y.A[k] += p0[k * 32 + s]; Y.D[k] += p0[(15 + k) * 32 + s]; }
#pragma unroll
                        for (int k = 0; k < 9; ++k) Y.B[k] += p0[(6 + k) * 32 + s];
                        f.l.x += p0[21 * 32 + s]; f.l.y += p0[22 * 32 + s]; f.l.z += p0[23 * 32 + s];
                        f.a.x += p0[24 * 32 + s]; f.a.y += p0[25 * 32 + s]; f.a.z += p0[26 * 32 + s];
                    }
                } else {
                    double* const pp = jb_smem + po * 32 + c.lane;
#pragma unroll
                    for (int k = 0; k < 6; ++k) { Y.A[k] += PO(k); Y.D[k] += PO(15 + k); }
#pragma unroll
                    for (int k = 0; k < 9; ++k) Y.B[k] += PO(6 + k);
                    f = f + sm_load_mot(c, po + 21);
                }
            }
            if (kind == REC_FREE) {
                // root free-flyer (parent = universe): ddq = (Y + Im)^-1 (tau - f) - a_gf, Im == 0, tau == 0
                Xf li; sm_load_xf(c, base + RF_LIMI, li);
                Mot g0; g0.l = mk(-opt.gravity[0], -opt.gravity[1], -opt.gravity[2]); g0.a = mk(-opt.gravity[3], -opt.gravity[4], -opt.gravity[5]);
                const Mot agf = motion_act_inv(li, g0);
                const double b[6] = {-f.l.x, -f.l.y, -f.l.z, -f.a.x, -f.a.y, -f.a.z};
                double x[6];
                spd_solve6(Y, b, x);
                RP(RF_A + 0) = x[0] - agf.l.x; RP(RF_A + 1) = x[1] - agf.l.y; RP(RF_A + 2) = x[2] - agf.l.z;
                RP(RF_A + 3) = x[3] - agf.a.x; RP(RF_A + 4) = x[4] - agf.a.y; RP(RF_A + 5) = x[5] - agf.a.z;
                return;
            }
            if (kind == REC_SPH) {
                // calc_aba of the spherical joint (pinocchio_overload_algorithms.h:305-328): S = [0; 1_3], U = Ia S = [B; D],
                // Dinv = (D + diag(Im))^-1; `ax` holds the three rotor inertias.  u = tau - S^T f.
                double* const xp = rp + KP->sph_off * 32;
                const double Dm[6] = {Y.D[0] + ax.x, Y.D[1], Y.D[2] + ax.y, Y.D[3], Y.D[4], Y.D[5] + ax.z};
                double Di[6];
                sym3_inverse(Dm, Di);
                const V3 u = mk(xp[(RS_TAU + 0) * 32] - f.a.x, xp[(RS_TAU + 1) * 32] - f.a.y, xp[(RS_TAU + 2) * 32] - f.a.z);
                const double Df[9] = {Y.D[0], Y.D[1], Y.D[3], Y.D[1], Y.D[2], Y.D[4], Y.D[3], Y.D[4], Y.D[5]};
#pragma unroll
                for (int j = 0; j < 3; ++j) {   // column j of U: linear part = column j of B, angular part = column j of D
                    xp[(RS_U + 6 * j + 0) * 32] = Y.B[j]; xp[(RS_U + 6 * j + 1) * 32] = Y.B[3 + j]; xp[(RS_U + 6 * j + 2) * 32] = Y.B[6 + j];
                    xp[(RS_U + 6 * j + 3) * 32] = Df[j]; xp[(RS_U + 6 * j + 4) * 32] = Df[3 + j]; xp[(RS_U + 6 * j + 5) * 32] = Df[6 + j];
                }
#pragma unroll
                for (int k = 0; k < 6; ++k) xp[(RS_DINV + k) * 32] = Di[k];
                xp[(RS_TAU + 0) * 32] = u.x; xp[(RS_TAU + 1) * 32] = u.y; xp[(RS_TAU + 2) * 32] = u.z;
                if (ri.parent_rec >= 0) {
                    // UDinv = [B Dinv; D Dinv] ; Ia -= UDinv U^T ; pa = f + Ia a_gf + UDinv u
                    const double Dif[9] = {Di[0], Di[1], Di[3], Di[1], Di[2], Di[4], Di[3], Di[4], Di[5]};
                    double BD[9], DD[9];
                    mat3mul(Y.B, Dif, BD);
                    mat3mul(Df, Dif, DD);
                    double BDB[9], BDD[9], DDD[9];   // BD B^T, BD D, DD D
#pragma unroll
                    for (int i = 0; i < 3; ++i)
#pragma unroll
                        for (int j = 0; j < 3; ++j) {
                            BDB[3 * i + j] = BD[3 * i] * Y.B[3 * j] + BD[3 * i + 1] * Y.B[3 * j + 1] + BD[3 * i + 2] * Y.B[3 * j + 2];
                            BDD[3 * i + j] = BD[3 * i] * Df[j] + BD[3 * i + 1] * Df[3 + j] + BD[3 * i + 2] * Df[6 + j];
                            DDD[3 * i + j] = DD[3 * i] * Df[j] + DD[3 * i + 1] * Df[3 + j] + DD[3 * i + 2] * Df[6 + j];
                        }
                    Y.A[0] -= BDB[0]; Y.A[1] -= BDB[1]; Y.A[2] -= BDB[4]; Y.A[3] -= BDB[2]; Y.A[4] -= BDB[5]; Y.A[5] -= BDB[8];
#pragma unroll
                    for (int k = 0; k < 9; ++k) Y.B[k] -= BDD[k];
                    Y.D[0] -= DDD[0]; Y.D[1] -= DDD[1]; Y.D[2] -= DDD[4]; Y.D[3] -= DDD[2]; Y.D[4] -= DDD[5]; Y.D[5] -= DDD[8];
                    const Mot bias = sm_load_mot(c, base + KP->sph_off + RS_BIAS);
                    Mot pa = f + sym_mul_motion(Y, bias);
                    pa.l = pa.l + rmul(BD, u); pa.a = pa.a + rmul(DD, u);
                    Xf li; sm_load_xf(c, base + RF_LIMI, li);
                    sym_transform(li, Y, Yc);
                    fc = force_act(li, pa);
                    if (!ri.carry_out) {
                        const bool add = (r >= SIG::ntrunk()) || (c.sub == 0);
                        if (add) {
                            const int po = SIG::pool_off() + POOL_SIZE * ri.parent_pool;
                            double* const pp = jb_smem + po * 32 + c.lane;
#pragma unroll
                            for (int k = 0; k < 6; ++k) { PO(k) += Yc.A[k]; PO(15 + k) += Yc.D[k]; }
#pragma unroll
                            for (int k = 0; k < 9; ++k) PO(6 + k) += Yc.B[k];
                            PO(21) += fc.l.x; PO(22) += fc.l.y; PO(23) += fc.l.z;
                            PO(24) += fc.a.x; PO(25) += fc.a.y; PO(26) += fc.a.z;
                        }
                    }
                }
                return;
            }
            // calc_aba (pinocchio_overload_algorithms.h:169-260): U = Ia S, Dinv = 1 / (S^T U + Im)
            Mot U; double u = RP(R1_U);
            double Dj;
            if (kind == REC_PRISM) {
                U.l = symmul(Y.A, ax); U.a = rtmul(Y.B, ax);
                u -= dot(ax, f.l);
                Dj = dot(ax, U.l) + Kd[13];
            } else if (kind == REC_REVX) {
                // S = sx e_4 with sx = +-1: work with the unsigned column and u' = sx u (sx^2 = 1), so that
                // UDinv U^T, UDinv u and (below) S ddq need no further sign handling
                U.l = mk(Y.B[0], Y.B[3], Y.B[6]); U.a = mk(Y.D[0], Y.D[1], Y.D[3]);
                u = ax.x * u - f.a.x;
                Dj = Y.D[0] + Kd[13];
            } else {
                U.l = rmul(Y.B, ax); U.a = symmul(Y.D, ax);
                u -= dot(ax, f.a);
                Dj = dot(ax, U.a) + Kd[13];
            }
            const double Dinv = 1.0 / Dj;
            sm_store_mot(c, base + R1_FU, U);
            RP(R1_DINV) = Dinv;
            RP(R1_U) = u;
            if (ri.parent_rec >= 0) {
                // Ia -= UDinv U^T ; pa = f + Ia a_gf + UDinv u ; parent += liMi.act(...)
                const V3 ul = Dinv * U.l, ua = Dinv * U.a;
                Y.A[0] -= ul.x * U.l.x; Y.A[1] -= ul.x * U.l.y; Y.A[2] -= ul.y * U.l.y;
                Y.A[3] -= ul.x * U.l.z; Y.A[4] -= ul.y * U.l.z; Y.A[5] -= ul.z * U.l.z;
                Y.B[0] -= ul.x * U.a.x; Y.B[1] -= ul.x * U.a.y; Y.B[2] -= ul.x * U.a.z;
                Y.B[3] -= ul.y * U.a.x; Y.B[4] -= ul.y * U.a.y; Y.B[5] -= ul.y * U.a.z;
                Y.B[6] -= ul.z * U.a.x; Y.B[7] -= ul.z * U.a.y; Y.B[8] -= ul.z * U.a.z;
                Y.D[0] -= ua.x * U.a.x; Y.D[1] -= ua.x * U.a.y; Y.D[2] -= ua.y * U.a.y;
                Y.D[3] -= ua.x * U.a.z; Y.D[4] -= ua.y * U.a.z; Y.D[5] -= ua.z * U.a.z;
                const Mot bias = sm_load_mot(c, base + R1_BIAS);
                Mot pa = f + sym_mul_motion(Y, bias);
                pa.l = pa.l + u * ul; pa.a = pa.a + u * ua;
                Xf li; sm_load_xf(c, base + R1_LIMI, li);
                // the parent's share goes straight into the carry; it is spilled to the parent's pool
                // accumulator when the parent is not the next record of the sweep
                sym_transform(li, Y, Yc);
                fc = force_act(li, pa);
                if (!ri.carry_out) {
                    // trunk joints hold identical values on every lane: only sub-lane 0 contributes
                    const bool add = (r >= SIG::ntrunk()) || (c.sub == 0);
                    if (add) {
                        const int po = SIG::pool_off() + POOL_SIZE * ri.parent_pool;
                        double* const pp = jb_smem + po * 32 + c.lane;
                        if (SIG::pool_single_writer) {
#pragma unroll
                            for (int k = 0; k < 6; ++k) { PO(k) = Yc.A[k]; PO(15 + k) = Yc.D[k]; }
#pragma unroll
                            for (int k = 0; k < 9; ++k) PO(6 + k) = Yc.B[k];
                            PO(21) = fc.l.x; PO(22) = fc.l.y; PO(23) = fc.l.z;
                            PO(24) = fc.a.x; PO(25) = fc.a.y; PO(26) = fc.a.z;
                        } else {
#pragma unroll
                            for (int k = 0; k < 6; ++k) { PO(k) += Yc.A[k]; PO(15 + k) += Yc.D[k]; }
#pragma unroll
                            for (int k = 0; k < 9; ++k) PO(6 + k) += Yc.B[k];
                            PO(21) += fc.l.x; PO(22) += fc.l.y; PO(23) += fc.l.z;
                            PO(24) += fc.a.x; PO(25) += fc.a.y; PO(26) += fc.a.z;
                        }
                    }
                }
            }
        };
        SIG::template for_each_backward(body);
    }
    jb_syncwarp(c);
    // ======================= pass 3: forward sweep (AbaForwardStep2) ===========================
    {
        Mot agc = mzero();   // a_gf of the previous record
        auto body = [&](auto r_) {
            const int r = r_;
            const RecInt ri = SIG::rec(r, L, c.sub);
            const int kind = ri.kind;
            if (kind == REC_PAD) return;
            const RecDbl* rd = JB_RDBL + (r * L + c.sub);
            double Ka[4];
            load_doubles(rd->placement + 12, Ka, 2);   // axis (3) + inertia[0]
            const int base = SIG::rec_off(r);
            double* const rp = jb_smem + base * 32 + c.lane;
            if (ri.parent_rec < 0) {
                agc.l = mk(-opt.gravity[0], -opt.gravity[1], -opt.gravity[2]);
                agc.a = mk(-opt.gravity[3], -opt.gravity[4], -opt.gravity[5]);
            } else if (!ri.carry_in) agc = sm_load_mot(c, SIG::pool_off() + POOL_SIZE * ri.parent_pool);
            Mot ag;
            if (kind == REC_FREE) {
                Xf li; sm_load_xf(c, base + RF_LIMI, li);
                ag = motion_act_inv(li, agc) + sm_load_mot(c, base + RF_A);
            } else if (kind == REC_SPH) {
                // ddq = Dinv (u - U^T a_gf) ; a_gf += S ddq
                const double* const xp = rp + KP->sph_off * 32;
                Xf li; sm_load_xf(c, base + RF_LIMI, li);
                ag = sm_load_mot(c, base + KP->sph_off + RS_BIAS) + motion_act_inv(li, agc);
                double t[3];
#pragma unroll
                for (int j = 0; j < 3; ++j) {
                    const double* const uj = xp + (RS_U + 6 * j) * 32;
                    t[j] = xp[(RS_TAU + j) * 32] - ((uj[0] * ag.l.x + uj[32] * ag.l.y + uj[64] * ag.l.z) +
                                                   (uj[96] * ag.a.x + uj[128] * ag.a.y + uj[160] * ag.a.z));
                }
                double Di[6];
#pragma unroll
                for (int k = 0; k < 6; ++k) Di[k] = xp[(RS_DINV + k) * 32];
                const V3 ddq = symmul(Di, mk(t[0], t[1], t[2]));
                RP(RF_A + 0) = 0.0; RP(RF_A + 1) = 0.0; RP(RF_A + 2) = 0.0;
                RP(RF_A + 3) = ddq.x; RP(RF_A + 4) = ddq.y; RP(RF_A + 5) = ddq.z;
                ag.a = ag.a + ddq;
            } else {
                Xf li; sm_load_xf(c, base + R1_LIMI, li);
                ag = sm_load_mot(c, base + R1_BIAS) + motion_act_inv(li, agc);
                const Mot U = sm_load_mot(c, base + R1_FU);
                const double ddq = RP(R1_DINV) * (RP(R1_U) - (dot(U.l, ag.l) + dot(U.a, ag.a)));
                const V3 ax = mk(Ka[0], Ka[1], Ka[2]);
                if (kind == REC_REVX) { RP(R1_A) = ax.x * ddq; ag.a.x += ddq; }   // ddq here is sx * (joint acceleration)
                else {
                    RP(R1_A) = ddq;
                    if (kind == REC_PRISM) ag.l = ag.l + ddq * ax;
                    else ag.a = ag.a + ddq * ax;
                }
            }
            if (ri.pool >= 0) sm_store_mot(c, SIG::pool_off() + POOL_SIZE * ri.pool, ag);
            if (ri.imu_slot >= 0) sm_store_mot(c, SIG::imu_off() + IMUSLOT_SIZE * ri.imu_slot + 6, ag);
            agc = ag;
        };
        SIG::template for_each_forward(body);
    }
    jb_syncwarp(c);
    return out_of_bounds;
}

// Fast-path signatures (env_step_kernel_t<true>): same plans, but the evaluation never enters the constraint
// path -- a joint leaving its position bounds only raises ENV_RETRY_FULL, and the env is re-done by the full
// kernel.  Keeping that code out of the fast kernel keeps its instruction footprint (and its registers) small.
template <class BASE> struct FastOf : BASE { static constexpr bool fast_path = true; };
template <class SIG, class = void> struct sig_is_fast { static constexpr bool value = false; };
template <class BASE> struct sig_is_fast<FastOf<BASE>> { static constexpr bool value = true; };
template <class SIG> struct is_fast_quadruped { static constexpr bool value = false; };
template <> struct is_fast_quadruped<FastOf<SigQuadruped>> { static constexpr bool value = true; };
constexpr int ENV_RETRY_FULL = 1 << 30;   // internal status bit, never stored

// The three ABA sweeps are compiled once per plan signature, as out-of-line functions; the static one is a leaf
// (no calls), which is what keeps its register allocation tight.  They return whether a bounded joint of this
// lane is outside its position bounds.
__device__ __noinline__ bool rhs_static_quadruped(const Ctx c, const bool up_to_date, int* status) {
    return rhs_impl<SigQuadruped>(c, up_to_date, status);
}
// the same sweeps with the `constraint` contact model (contact frames handed to the constraint solver, start-time flags)
__device__ __noinline__ bool rhs_static_quadruped_cons(const Ctx c, const bool up_to_date, int* status) {
    return rhs_impl<SigQuadrupedCons>(c, up_to_date, status);
}
template <bool EXT>
__device__ __noinline__ bool rhs_dynamic(const Ctx c, const bool up_to_date, int* status) {
    if (KP->all_uniform) return rhs_impl<SigDynamic<true, EXT>>(c, up_to_date, status);
    return rhs_impl<SigDynamic<false, EXT>>(c, up_to_date, status);
}
// ------------------------------------------------------------------------------------------
// Hot-path evaluation for the quadruped signature, composite-rigid-body form.
//
// Same equations of motion as the articulated-body sweeps above (pinocchio_overload_algorithms.h:446-489: rotor
// inertia on the diagonal, external forces in the joint frames), solved as
//     [ Yc0      M_bl ] [ddq_b]   [ -f_b      ]
//     [ M_lb     M_ll ] [ddq_l] = [ tau - C_l ]
// with the bias forces (f_b, C_l) from one recursive Newton-Euler pass at zero joint acceleration (gravity enters as
// the base acceleration -g) and the joint-space inertia from the composite-rigid-body recursion.  The legs only
// couple through the base, so M_ll is block diagonal: every lane inverts its own 3x3 block, reduces the base
// equation by its Schur complement (one 27-number all-reduce, the same pool entry the ABA sweep uses) and all the
// lanes solve the same 6x6.  Why: the ABA backward sweep is ONE dependent chain through 21-number articulated
// inertias (division, rank-1 update, congruence, per joint), and with a single resident warp per scheduler nothing
// hides its latency; here the bias recursion, the composite inertias and the three inertia columns are independent
// chains of cheap 6- and 10-number transforms.  Used by the hot-path kernel only (the full body keeps the ABA
// sweeps, whose intermediate quantities the constraint solvers read).
// ------------------------------------------------------------------------------------------
// joint-bound constraint state of a leg joint, parked in the record's BIAS field (unused by this form of the evaluation):
// enabled, reversed (upper bound), reference position, multiplier (JointConstraint, joint_constraint.cc); record 1 also
// carries the env's count of successive solver failures
constexpr int R1_BEN = R1_BIAS, R1_BREV = R1_BIAS + 1, R1_BQREF = R1_BIAS + 2, R1_BLAM = R1_BIAS + 3, R1_BFAIL = R1_BIAS + 4;
struct CompI { V3 mc; double Io[6]; };   // composite inertia of a subtree, additive form: first moment, inertia about the frame origin
JB_DI CompI compi_body(double m, V3 c, const double* I) {
    CompI o;
    o.mc = m * c;
    const double cc = dot(c, c);
    o.Io[0] = I[0] - m * (c.x * c.x - cc); o.Io[1] = I[1] - m * (c.x * c.y); o.Io[2] = I[2] - m * (c.y * c.y - cc);
    o.Io[3] = I[3] - m * (c.x * c.z);      o.Io[4] = I[4] - m * (c.y * c.z); o.Io[5] = I[5] - m * (c.z * c.z - cc);
    return o;
}
JB_DI CompI compi_to_parent(const Xf& li, const CompI& a, double m) {
    CompI o;
    const V3 rmc = rmul(li.R, a.mc);
    o.mc = rmc + m * li.p;
    double Ir[6];
    rot_sym(li.R, a.Io, Ir);
    const V3 p = li.p;
    const double pp = dot(p, p), pr = dot(p, rmc);
    o.Io[0] = Ir[0] + m * (pp - p.x * p.x) + 2.0 * (pr - p.x * rmc.x);
    o.Io[1] = Ir[1] - m * (p.x * p.y) - (p.x * rmc.y + rmc.x * p.y);
    o.Io[2] = Ir[2] + m * (pp - p.y * p.y) + 2.0 * (pr - p.y * rmc.y);
    o.Io[3] = Ir[3] - m * (p.x * p.z) - (p.x * rmc.z + rmc.x * p.z);
    o.Io[4] = Ir[4] - m * (p.y * p.z) - (p.y * rmc.z + rmc.y * p.z);
    o.Io[5] = Ir[5] + m * (pp - p.z * p.z) + 2.0 * (pr - p.z * rmc.z);
    return o;
}
// column of the composite inertia for a revolute joint about +x: Yc e_4
JB_DI Mot compi_col_rx(const CompI& a) { Mot F; F.l = mk(0.0, -a.mc.z, a.mc.y); F.a = mk(a.Io[0], a.Io[1], a.Io[3]); return F; }

// ------------------------------------------------------------------------------------------
// Joint position bounds on the hot path (quadruped signature, composite-rigid-body form of the evaluation).
// computePositionLimitsForcesAlgo (engine.cc:3253-3338) enables the constraint of a joint that left [lo, hi] and disables
// it once the joint is transitionEps inside again; PGSSolver::SolveBoxedForwardDynamics (constraint_solvers.cc:320-447)
// then adds M^-1 J^T lambda to the free accelerations, lambda >= 0, rows J = +-e_j.  With the block form of M^-1 at hand
// -- M_ll^-1 and W of every leg, the base Schur complement Yb -- the Delassus matrix is
//     A_jk = s_j s_k ([same leg] (M_ll^-1)_jk + W_j . Yb^-1 W_k)
// and a change of lambda_k moves the base by -s_k Yb^-1 W_k: the sweep keeps zb = sum_k s_k lambda_k Yb^-1 W_k on every
// lane (the owner of a row broadcasts its change), everything else stays local to the lane.  Same row order (joint
// order), warm start, relaxation schedule and stopping rule as the reference.  Called for the envs with a bound in play only.
// ------------------------------------------------------------------------------------------
__device__ __noinline__ void bounds_solve_quadruped(const Ctx c, const bool up_to_date, int* status) {
    using SIG = SigQuadruped;
    constexpr int L = 4;
    const JbOptions& opt = KP->opt;
    {
        {
            const int o1 = SIG::rec_off(1), o2 = SIG::rec_off(2), o3 = SIG::rec_off(3);
            const int off[3] = {o1, o2, o3};
            // what the evaluation left in shared memory: W rows in the FU fields, M_ll^-1 in (DINV, U), the legs' shares of the
            // base inertia in the pool entries
            double sx[3], Mi[6];
            Mot Wv[3];
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                sx[i] = (JB_RDBL + ((i + 1) * L + c.sub))->axis[0];
                Wv[i] = sm_load_mot(c, off[i] + R1_FU);
                Mi[2 * i] = SMF(c, off[i] + R1_DINV); Mi[2 * i + 1] = SMF(c, off[i] + R1_U);
            }
            const double Mf[3][3] = {{Mi[0], Mi[1], Mi[3]}, {Mi[1], Mi[2], Mi[4]}, {Mi[3], Mi[4], Mi[5]}};
            SymY Yb;
            {
                double Kd[14];
                load_doubles((JB_RDBL + c.sub)->placement + 12, Kd, 7);
                inertia_to_sym(Kd[3], mk(Kd[4], Kd[5], Kd[6]), Kd + 7, Yb);
                const double* const p0 = jb_smem + SIG::pool_off() * 32 + (c.lane - c.sub);
#pragma unroll
                for (int sl = 0; sl < L; ++sl) {
#pragma unroll
                    for (int k = 0; k < 6; ++k) { Yb.A[k] += p0[k * 32 + sl]; Yb.D[k] += p0[(15 + k) * 32 + sl]; }
#pragma unroll
                    for (int k = 0; k < 9; ++k) Yb.B[k] += p0[(6 + k) * 32 + sl];
                }
            }
            const double omega = 2.0 * 3.14159265358979323846 * opt.contact_stabilization_freq;   // setBaumgarteFreq (abstract_constraint.cc:88-99)
            const double kp = omega * omega, kd = 2.0 * omega, eps = opt.contact_transition_eps;
            bool en[3];
            double sg[3], bb[3], lam[3], rg[3], iad[3], Yr[3] = {0, 0, 0}, Yp[3] = {0, 0, 0};
            Mot hv[3];
            Spd6 sf;
            spd6_factor(Yb, sf);
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                double* const rp = jb_smem + off[i] * 32 + c.lane;
                const RecDbl* rd = JB_RDBL + ((i + 1) * L + c.sub);
                const double q = RP(R1_QS), vj = RP(R1_VS), lo = rd->q_lo, hi = rd->q_hi;
                bool e = RP(R1_BEN) != 0.0, rev = RP(R1_BREV) != 0.0;
                double qref = RP(R1_BQREF), l = RP(R1_BLAM);
                if (!up_to_date) {
                    if (hi < q || q < lo) {
                        qref = fmin(fmax(q, lo), hi); rev = hi < q; e = true;
                        *status |= JB_ENV_JOINT_LIMIT;
                    } else if (lo + eps < q && q < hi - eps) { e = false; l = 0.0; }
                    RP(R1_BEN) = e ? 1.0 : 0.0; RP(R1_BREV) = rev ? 1.0 : 0.0; RP(R1_BQREF) = qref;
                }
                const double sgn = rev ? -1.0 : 1.0;
                en[i] = e;
                sg[i] = e ? sgn * sx[i] : 0.0;                              // row in the unsigned-axis coordinates
                lam[i] = e ? l : 0.0;
                bb[i] = -sgn * (kp * (q - qref) + kd * vj) - sgn * RP(R1_A);   // -drift - J ddq_free
                hv[i] = spd6_apply(sf, Wv[i]);
                const double a0 = Mf[i][i] + (dot(Wv[i].l, hv[i].l) + dot(Wv[i].a, hv[i].a));
                rg[i] = fmax(a0 * opt.constraint_regularization, CONS_MIN_REGULARIZER);
                iad[i] = 1.0 / (a0 + rg[i]);
            }
            // zb = sum over the rows of the env of s_k lambda_k Yb^-1 W_k (warm start)
            Mot zp = mzero();
#pragma unroll
            for (int i = 0; i < 3; ++i) { zp.l = zp.l + (sg[i] * lam[i]) * hv[i].l; zp.a = zp.a + (sg[i] * lam[i]) * hv[i].a; }
            double zb[6];
            zb[0] = cq_bcast_sum4(c, zp.l.x); zb[1] = cq_bcast_sum4(c, zp.l.y); zb[2] = cq_bcast_sum4(c, zp.l.z);
            zb[3] = cq_bcast_sum4(c, zp.a.x); zb[4] = cq_bcast_sum4(c, zp.a.y); zb[5] = cq_bcast_sum4(c, zp.a.z);
            bool slot_on[4][3];
#pragma unroll
            for (int l4 = 0; l4 < 4; ++l4)
#pragma unroll
                for (int i = 0; i < 3; ++i) slot_on[l4][i] = __any_sync(c.gmask, c.sub == l4 && en[i]);
            const int lane0 = c.lane - c.sub;
            bool ok = false;
            for (int iter = 0; iter < CONS_PGS_MAX_ITER && !ok; ++iter) {
#pragma unroll
                for (int i = 0; i < 3; ++i) Yp[i] = Yr[i];
                const double ratio = (static_cast<double>(CONS_PGS_MAX_ITER - CONS_RELAX_MIN_ITER) - iter) /
                                     (CONS_PGS_MAX_ITER - CONS_RELAX_MIN_ITER - CONS_RELAX_MAX_ITER);
                double wr = CONS_RELAX_MAX;
                if (ratio < 1.0) {
                    wr = CONS_RELAX_MIN;
                    if (ratio > 0.0) wr += (CONS_RELAX_MAX - CONS_RELAX_MIN) * (ratio * ratio);
                }
#pragma unroll
                for (int l4 = 0; l4 < 4; ++l4)
#pragma unroll
                    for (int i = 0; i < 3; ++i) {
                        if (!slot_on[l4][i]) continue;
                        double dz[6] = {0, 0, 0, 0, 0, 0};
                        if (c.sub == l4 && en[i]) {
                            const double loc = Mf[i][0] * (sg[0] * lam[0]) + Mf[i][1] * (sg[1] * lam[1]) + Mf[i][2] * (sg[2] * lam[2]);
                            const double wz = (Wv[i].l.x * zb[0] + Wv[i].l.y * zb[1] + Wv[i].l.z * zb[2]) +
                                              (Wv[i].a.x * zb[3] + Wv[i].a.y * zb[4] + Wv[i].a.z * zb[5]);
                            const double y = bb[i] - sg[i] * (loc + wz) - rg[i] * lam[i];
                            Yr[i] = y;
                            const double e = fmax(lam[i] + wr * y * iad[i], 0.0);
                            const double d = sg[i] * (e - lam[i]);
                            lam[i] = e;
                            dz[0] = d * hv[i].l.x; dz[1] = d * hv[i].l.y; dz[2] = d * hv[i].l.z;
                            dz[3] = d * hv[i].a.x; dz[4] = d * hv[i].a.y; dz[5] = d * hv[i].a.z;
                        }
#pragma unroll
                        for (int d = 0; d < 6; ++d) zb[d] += __shfl_sync(c.gmask, dz[d], lane0 + l4);
                    }
                // stopping criterion on the stagnation of the residuals (constraint_solvers.cc:256-274)
                double ymax = fmax(fabs(Yr[0]), fmax(fabs(Yr[1]), fabs(Yr[2])));
                for (int o = 1; o < L; o <<= 1) ymax = fmax(ymax, __shfl_xor_sync(c.gmask, ymax, o));
                const double tol = opt.tol_abs + opt.tol_rel * ymax + D_EPS;
                bool conv = true;
#pragma unroll
                for (int i = 0; i < 3; ++i) conv = conv && (fabs(Yr[i] - Yp[i]) < tol);
                ok = __all_sync(c.gmask, conv);
            }
            // ddq += M^-1 J^T lambda: the base moves by -zb, the leg by M_ll^-1 (s lambda) + W zb
            {
                double* const rp = jb_smem + c.lane;
                double* const ip = jb_smem + (SIG::imu_off() + 6) * 32 + c.lane;
#pragma unroll
                for (int d = 0; d < 6; ++d) { RP(RF_A + d) -= zb[d]; ip[d * 32] -= zb[d]; }
            }
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                const double loc = Mf[i][0] * (sg[0] * lam[0]) + Mf[i][1] * (sg[1] * lam[1]) + Mf[i][2] * (sg[2] * lam[2]);
                const double wz = (Wv[i].l.x * zb[0] + Wv[i].l.y * zb[1] + Wv[i].l.z * zb[2]) +
                                  (Wv[i].a.x * zb[3] + Wv[i].a.y * zb[4] + Wv[i].a.z * zb[5]);
                SMF(c, off[i] + R1_A) += sx[i] * (loc + wz);
                SMF(c, off[i] + R1_BLAM) = lam[i];
            }
            // successiveSolveFailed (constraint_solvers.cc:436-446): reset on success
            SMF(c, o1 + R1_BFAIL) = ok ? 0.0 : SMF(c, o1 + R1_BFAIL) + 1.0;
        }
    }
}

// SE(3) integrate of the free-flyer, q1 = integrate(q0, dv), in quaternion form: the same map as integrate_free
// (M1 = M0 exp6(v, w)) with the rotation composed as q0 (x) (sin(t/2) w / t, cos(t/2)), t = |w|, instead of building
// exp6's rotation matrix and converting R0 Re back to a quaternion.  sin t = 2 s c and 1 - cos t = 2 s^2 come from one
// jb_sincos(t / 2) (t / 2 is bounded by dt |w| / 2), 1 / t from one reciprocal square root; the Taylor branch of exp6
// below TAYLOR_PREC3 is a select, so the whole integrate is one basic block.  Same sign continuity and first-order
// normalisation as integrate_free.
JB_DI void integrate_free_quat(const double* q0, const double* dv, double* q1) {
    const V3 v = mk(dv[0], dv[1], dv[2]), w = mk(dv[3], dv[4], dv[5]);
    const double t2 = dot(w, w);
    const bool small = t2 < TAYLOR_PREC3 * TAYLOR_PREC3;     // t < TAYLOR_PREC3 (a power of two: exact)
    const double inv_t = rsqrt(t2);
    double sh, ch;
    jb_sincos(0.5 * (t2 * inv_t), &sh, &ch);
    const double inv_t2 = inv_t * inv_t;
    const double alpha_wxv = small ? 0.5 - t2 * (1.0 / 24.0) : (2.0 * sh * sh) * inv_t2;   // (1 - cos t) / t^2
    const double alpha_v = small ? 1.0 - t2 * (1.0 / 6.0) : (2.0 * sh * ch) * inv_t;       // sin t / t
    const double alpha_w = small ? 1.0 / 6.0 - t2 * (1.0 / 120.0) : (1.0 - alpha_v) * inv_t2;
    const double kq = small ? 0.5 - t2 * (1.0 / 48.0) : sh * inv_t;                         // sin(t / 2) / t
    const double cq = small ? 1.0 - t2 * 0.125 : ch;                                        // cos(t / 2)
    const V3 pe = alpha_v * v + (alpha_w * dot(w, v)) * w + alpha_wxv * cross(w, v);
    double R0[9];
    quat_to_R(q0[3], q0[4], q0[5], q0[6], R0);
    const V3 p1 = mk(q0[0], q0[1], q0[2]) + rmul(R0, pe);
    const double qe[4] = {kq * w.x, kq * w.y, kq * w.z, cq};
    double q[4];
    quat_mul(q0 + 3, qe, q);
    const double dp = q[0] * q0[3] + q[1] * q0[4] + q[2] * q0[5] + q[3] * q0[6];
    const double sg = dp < 0.0 ? -1.0 : 1.0;
    const double N2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
    const double alpha = sg * ((3.0 - N2) / 2.0);
    q1[0] = p1.x; q1[1] = p1.y; q1[2] = p1.z;
    q1[3] = q[0] * alpha; q1[4] = q[1] * alpha; q1[5] = q[2] * alpha; q1[6] = q[3] * alpha;
}

// Evaluation of the quadruped signature in composite-rigid-body form.  STAGE = false: at the stage state already in
// QS / VS.  STAGE = true: one whole Runge-Kutta stage -- forms the stage state QS = integrate(Q, wq kv), VS = V + wq ka
// (kv / ka read at the field offsets kv1 / ka1 of the 1-dof records and kvf / kaf of the free-flyer), evaluates there
// and adds wb (VS, A) to the accumulators (SV, SA) when wb != 0.  The stage state is kept in registers, the contact and
// the springs take no branch: the base's integrate, the legs' position-only terms and the velocity pass form one basic
// block that the scheduler interleaves.
template <bool STAGE>
JB_DI bool quadruped_crba(const Ctx c, const bool up_to_date, int* status, const double wq, const int kv1, const int ka1,
                          const int kvf, const int kaf, const double wb) {
    using SIG = SigQuadruped;
    constexpr int L = 4;
    const JbOptions& opt = KP->opt;
    bool out_any = false;
    double qb[7], vb[6], ql[4], vl[4];      // stage state of the free-flyer and of legs records 1..3
    double spk[4] = {0, 0, 0, 0}, spd[4] = {0, 0, 0, 0};
    if constexpr (STAGE) {
        if (KP->springs != nullptr) {
#pragma unroll
            for (int r = 1; r < 4; ++r) {
                const int iv = (KP->rint + (r * L + c.sub))->idx_v;
                spk[r] = KP->springs[iv]; spd[r] = KP->springs[KP->nv + iv];
            }
        }
        double* const rp = jb_smem + c.lane;
        double q0[7], dv[6];
#pragma unroll
        for (int k = 0; k < 7; ++k) q0[k] = RP(RF_Q + k);
#pragma unroll
        for (int k = 0; k < 6; ++k) { dv[k] = wq * rp[(kvf + k) * 32]; vb[k] = RP(RF_V + k) + wq * rp[(kaf + k) * 32]; }
        integrate_free_quat(q0, dv, qb);
#pragma unroll
        for (int k = 0; k < 7; ++k) RP(RF_QS + k) = qb[k];
#pragma unroll
        for (int k = 0; k < 6; ++k) RP(RF_VS + k) = vb[k];
#pragma unroll
        for (int r = 1; r < 4; ++r) {
            double* const rq = jb_smem + SIG::rec_off(r) * 32 + c.lane;
            ql[r] = rq[R1_Q * 32] + wq * rq[kv1 * 32];
            vl[r] = rq[R1_V * 32] + wq * rq[ka1 * 32];
            rq[R1_QS * 32] = ql[r]; rq[R1_VS * 32] = vl[r];
        }
    } else {
        const double* const rp = jb_smem + c.lane;
#pragma unroll
        for (int k = 0; k < 7; ++k) qb[k] = RP(RF_QS + k);
#pragma unroll
        for (int k = 0; k < 6; ++k) vb[k] = RP(RF_VS + k);
#pragma unroll
        for (int r = 1; r < 4; ++r) { ql[r] = SMF(c, SIG::rec_off(r) + R1_QS); vl[r] = SMF(c, SIG::rec_off(r) + R1_VS); }
    }
    // ======================= forward: kinematics, bias accelerations, bias forces, contact, motors ================
    Xf oMc; Mot vc, ac;
    {
        const RecDbl* rd = JB_RDBL + c.sub;
        RecConst K;
        load_doubles(rd->placement, K.placement, 14);
        double* const rp = jb_smem + c.lane;   // record 0 starts at field 0
        Xf li;
        double Rq[9];
        quat_to_R(qb[3], qb[4], qb[5], qb[6], Rq);
        mat3mul(K.placement, Rq, li.R);
        li.p = ld3(K.placement + 9) + rmul(K.placement, mk(qb[0], qb[1], qb[2]));
        Mot v; v.l = mk(vb[0], vb[1], vb[2]); v.a = mk(vb[3], vb[4], vb[5]);
        Mot g0; g0.l = mk(-opt.gravity[0], -opt.gravity[1], -opt.gravity[2]); g0.a = mk(-opt.gravity[3], -opt.gravity[4], -opt.gravity[5]);
        const Mot a0 = motion_act_inv(li, g0);          // base acceleration at zero joint acceleration (v x vJ = 0 for the root)
        const double m = K.inertia[0];
        const V3 lc = ld3(K.inertia + 1);
        const Mot f = inertia_mul(m, lc, K.inertia + 4, a0) + motion_cross_force(v, inertia_mul(m, lc, K.inertia + 4, v));
        sm_store_xf(c, RF_LIMI, li);
        sm_store_mot(c, RF_F, f);
        sm_store_mot(c, SIG::imu_off(), v);
        sm_store_mot(c, SIG::imu_off() + 6, a0);
        oMc = li; vc = v; ac = a0;
    }
#pragma unroll
    for (int r = 1; r < 4; ++r) {
        const RecDbl* rd = JB_RDBL + (r * L + c.sub);
        RecConst K;
        load_doubles(rd->placement, K.placement, 14);
        const MotorConst mc = load_motor_const(rd);
        const int base = SIG::rec_off(r);
        double* const rp = jb_smem + base * 32 + c.lane;
        const double sx = K.axis[0];
        double ca, sa;
        jb_sincos(ql[r], &sa, &ca);
        const double s = sx * sa;
        Xf li;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            li.R[3 * i] = K.placement[3 * i];
            li.R[3 * i + 1] = ca * K.placement[3 * i + 1] + s * K.placement[3 * i + 2];
            li.R[3 * i + 2] = ca * K.placement[3 * i + 2] - s * K.placement[3 * i + 1];
        }
        li.p = ld3(K.placement + 9);
        const double qd = vl[r], w = sx * qd;
        Xf oM;
        mat3mul(oMc.R, li.R, oM.R);
        oM.p = oMc.p + rmul(oMc.R, li.p);
        Mot v = motion_act_inv(li, vc);
        v.a.x += w;
        Mot a = motion_act_inv(li, ac);                 // + v x vJ, vJ = w e_4
        a.l.y += v.l.z * w; a.l.z -= v.l.y * w; a.a.y += v.a.z * w; a.a.z -= v.a.y * w;
        const double m = K.inertia[0];
        const V3 lc = ld3(K.inertia + 1);
        Mot f = inertia_mul(m, lc, K.inertia + 4, a) + motion_cross_force(v, inertia_mul(m, lc, K.inertia + 4, v));
        if (r == 3) {
            // Engine::computeContactDynamicsAtFrame (engine.cc:3117-3195), one contact frame on the last joint
            const ContactSlot* ct = KP->cslots + c.sub;
            double* const cp = jb_smem + SIG::cslot_off() * 32 + c.lane;
            const V3 pc = ld3(ct->placement + 9);
            V3 Fl;
            if constexpr (STAGE) {
                // evaluated whatever the depth, kept below the ground only
                const V3 pos = oM.p + rmul(oM.R, pc);
                const V3 vw = rmul(oM.R, v.l + cross(v.a, pc));
                const V3 fc = rtmul(oM.R, contact_dynamics_nb(opt, fmin(pos.z, 0.0), vw));
                const bool in = pos.z < 0.0;
                Fl = mk(in ? fc.x : 0.0, in ? fc.y : 0.0, in ? fc.z : 0.0);
                CO(0) = Fl.x; CO(1) = Fl.y; CO(2) = Fl.z;
            } else if (!up_to_date) {
                const V3 pos = oM.p + rmul(oM.R, pc);
                Fl = mk(0, 0, 0);
                if (pos.z < 0.0) {
                    const V3 vw = rmul(oM.R, v.l + cross(v.a, pc));
                    Fl = rtmul(oM.R, contact_dynamics(opt, pos.z, vw));
                }
                CO(0) = Fl.x; CO(1) = Fl.y; CO(2) = Fl.z;
            } else Fl = mk(CO(0), CO(1), CO(2));
            f.l = f.l - Fl;
            f.a = f.a - cross(pc, Fl);
        }
        double u = 0.0;
        if constexpr (STAGE) u = -spk[r] * ql[r] - spd[r] * qd;
        else if (KP->springs != nullptr) {
            const int iv = (KP->rint + (r * L + c.sub))->idx_v;
            u = -KP->springs[iv] * ql[r] - KP->springs[KP->nv + iv] * qd;
        }
        double uM, uT;
        if constexpr (STAGE) motor_effort_limited_nb(mc, RP(R1_CMD), qd, uM, uT);
        else motor_effort_pre(mc, rd, 3, RP(R1_CMD), qd, uM, uT);
        RP(R1_UMOTOR) = uM;
        u += uT;
        RP(R1_U) = sx * u;                               // joint effort along the unsigned axis
        if (!up_to_date) { const double qj = ql[r]; out_any = out_any || K.q_hi < qj || qj < K.q_lo; }
        sm_store_xf(c, base + R1_LIMI, li);
        sm_store_mot(c, base + R1_FU, f);
        oMc = oM; vc = v; ac = a;
    }
    // ======================= backward: composite inertias, bias forces, inertia columns ==========================
    double M11, M12, M13, M22, M23, M33, C1, C2, C3, t1, t2, t3, s1, s2, s3;
    Mot B1, B2, B3, fb;
    CompI Yl;
    double Mi[6];      // M_ll^-1 of this leg (xx, xy, yy, xz, yz, zz)
    {
        // joint 3 (leaf)
        const RecDbl* rd3 = JB_RDBL + (3 * L + c.sub);
        double K3[14]; load_doubles(rd3->placement + 12, K3, 7);
        Xf li3; sm_load_xf(c, SIG::rec_off(3) + R1_LIMI, li3);
        Mot f3 = sm_load_mot(c, SIG::rec_off(3) + R1_FU);
        s3 = K3[0]; t3 = SMF(c, SIG::rec_off(3) + R1_U);
        CompI Y = compi_body(K3[3], mk(K3[4], K3[5], K3[6]), K3 + 7);
        Mot F3 = compi_col_rx(Y);
        M33 = F3.a.x + K3[13];
        C3 = f3.a.x;
        const double m3 = rd3->subtree_mass;
        Y = compi_to_parent(li3, Y, m3);
        F3 = force_act(li3, F3);
        f3 = force_act(li3, f3);
        // joint 2
        const RecDbl* rd2 = JB_RDBL + (2 * L + c.sub);
        double K2[14]; load_doubles(rd2->placement + 12, K2, 7);
        Xf li2; sm_load_xf(c, SIG::rec_off(2) + R1_LIMI, li2);
        Mot f2 = sm_load_mot(c, SIG::rec_off(2) + R1_FU) + f3;
        s2 = K2[0]; t2 = SMF(c, SIG::rec_off(2) + R1_U);
        {
            const CompI b = compi_body(K2[3], mk(K2[4], K2[5], K2[6]), K2 + 7);
            Y.mc = Y.mc + b.mc;
#pragma unroll
            for (int k = 0; k < 6; ++k) Y.Io[k] += b.Io[k];
        }
        Mot F2 = compi_col_rx(Y);
        M22 = F2.a.x + K2[13];
        M23 = F3.a.x;
        C2 = f2.a.x;
        const double m2 = rd2->subtree_mass;
        Y = compi_to_parent(li2, Y, m2);
        F3 = force_act(li2, F3); F2 = force_act(li2, F2);
        f2 = force_act(li2, f2);
        // joint 1
        const RecDbl* rd1 = JB_RDBL + (1 * L + c.sub);
        double K1[14]; load_doubles(rd1->placement + 12, K1, 7);
        Xf li1; sm_load_xf(c, SIG::rec_off(1) + R1_LIMI, li1);
        Mot f1 = sm_load_mot(c, SIG::rec_off(1) + R1_FU) + f2;
        s1 = K1[0]; t1 = SMF(c, SIG::rec_off(1) + R1_U);
        {
            const CompI b = compi_body(K1[3], mk(K1[4], K1[5], K1[6]), K1 + 7);
            Y.mc = Y.mc + b.mc;
#pragma unroll
            for (int k = 0; k < 6; ++k) Y.Io[k] += b.Io[k];
        }
        const Mot F1 = compi_col_rx(Y);
        M11 = F1.a.x + K1[13];
        M12 = F2.a.x; M13 = F3.a.x;
        C1 = f1.a.x;
        const double m1 = rd1->subtree_mass;
        Yl = compi_to_parent(li1, Y, m1);
        B1 = force_act(li1, F1); B2 = force_act(li1, F2); B3 = force_act(li1, F3);
        fb = force_act(li1, f1);
        // ---- the leg's block: Minv = M_ll^-1, W = Minv M_lb, y = Minv (tau - C)
        const double Ml[6] = {M11, M12, M22, M13, M23, M33};
        sym3_inverse(Ml, Mi);
        const double r1 = t1 - C1, r2 = t2 - C2, r3 = t3 - C3;
        const double y1 = Mi[0] * r1 + Mi[1] * r2 + Mi[3] * r3;
        const double y2 = Mi[1] * r1 + Mi[2] * r2 + Mi[4] * r3;
        const double y3 = Mi[3] * r1 + Mi[4] * r2 + Mi[5] * r3;
        Mot W1, W2, W3;
        W1.l = Mi[0] * B1.l + Mi[1] * B2.l + Mi[3] * B3.l; W1.a = Mi[0] * B1.a + Mi[1] * B2.a + Mi[3] * B3.a;
        W2.l = Mi[1] * B1.l + Mi[2] * B2.l + Mi[4] * B3.l; W2.a = Mi[1] * B1.a + Mi[2] * B2.a + Mi[4] * B3.a;
        W3.l = Mi[3] * B1.l + Mi[4] * B2.l + Mi[5] * B3.l; W3.a = Mi[3] * B1.a + Mi[4] * B2.a + Mi[5] * B3.a;
        // ---- contribution to the base equation: K = Yc_leg - M_bl Minv M_lb (symmetric blocks), g = f_leg + M_bl y
        const double ml = m1;
        double* const pp = jb_smem + SIG::pool_off() * 32 + c.lane;
        // A block (xx, xy, yy, xz, yz, zz): m 1 - sum_j B_j.l W_j.l^T
        PO(0) = ml - (B1.l.x * W1.l.x + B2.l.x * W2.l.x + B3.l.x * W3.l.x);
        PO(1) = -(B1.l.x * W1.l.y + B2.l.x * W2.l.y + B3.l.x * W3.l.y);
        PO(2) = ml - (B1.l.y * W1.l.y + B2.l.y * W2.l.y + B3.l.y * W3.l.y);
        PO(3) = -(B1.l.x * W1.l.z + B2.l.x * W2.l.z + B3.l.x * W3.l.z);
        PO(4) = -(B1.l.y * W1.l.z + B2.l.y * W2.l.z + B3.l.y * W3.l.z);
        PO(5) = ml - (B1.l.z * W1.l.z + B2.l.z * W2.l.z + B3.l.z * W3.l.z);
        // B block (row-major 3x3): -[mc]x - sum_j B_j.l W_j.a^T
        const V3 mcv = Yl.mc;
        PO(6)  = -(B1.l.x * W1.a.x + B2.l.x * W2.a.x + B3.l.x * W3.a.x);
        PO(7)  = mcv.z - (B1.l.x * W1.a.y + B2.l.x * W2.a.y + B3.l.x * W3.a.y);
        PO(8)  = -mcv.y - (B1.l.x * W1.a.z + B2.l.x * W2.a.z + B3.l.x * W3.a.z);
        PO(9)  = -mcv.z - (B1.l.y * W1.a.x + B2.l.y * W2.a.x + B3.l.y * W3.a.x);
        PO(10) = -(B1.l.y * W1.a.y + B2.l.y * W2.a.y + B3.l.y * W3.a.y);
        PO(11) = mcv.x - (B1.l.y * W1.a.z + B2.l.y * W2.a.z + B3.l.y * W3.a.z);
        PO(12) = mcv.y - (B1.l.z * W1.a.x + B2.l.z * W2.a.x + B3.l.z * W3.a.x);
        PO(13) = -mcv.x - (B1.l.z * W1.a.y + B2.l.z * W2.a.y + B3.l.z * W3.a.y);
        PO(14) = -(B1.l.z * W1.a.z + B2.l.z * W2.a.z + B3.l.z * W3.a.z);
        // D block: Io - sum_j B_j.a W_j.a^T
        PO(15) = Yl.Io[0] - (B1.a.x * W1.a.x + B2.a.x * W2.a.x + B3.a.x * W3.a.x);
        PO(16) = Yl.Io[1] - (B1.a.x * W1.a.y + B2.a.x * W2.a.y + B3.a.x * W3.a.y);
        PO(17) = Yl.Io[2] - (B1.a.y * W1.a.y + B2.a.y * W2.a.y + B3.a.y * W3.a.y);
        PO(18) = Yl.Io[3] - (B1.a.x * W1.a.z + B2.a.x * W2.a.z + B3.a.x * W3.a.z);
        PO(19) = Yl.Io[4] - (B1.a.y * W1.a.z + B2.a.y * W2.a.z + B3.a.y * W3.a.z);
        PO(20) = Yl.Io[5] - (B1.a.z * W1.a.z + B2.a.z * W2.a.z + B3.a.z * W3.a.z);
        const Mot g = fb + Mot{y1 * B1.l + y2 * B2.l + y3 * B3.l, y1 * B1.a + y2 * B2.a + y3 * B3.a};
        PO(21) = g.l.x; PO(22) = g.l.y; PO(23) = g.l.z; PO(24) = g.a.x; PO(25) = g.a.y; PO(26) = g.a.z;
        // the solution of the base equation comes back below: keep what the back-substitution needs
        B1 = W1; B2 = W2; B3 = W3; C1 = y1; C2 = y2; C3 = y3;
        {
            // for the joint-bound solver, should this env need it (no branch here: it would split the block the scheduler
            // works on): W rows and M_ll^-1 in record fields that are dead by now
            sm_store_mot(c, SIG::rec_off(1) + R1_FU, W1); sm_store_mot(c, SIG::rec_off(2) + R1_FU, W2); sm_store_mot(c, SIG::rec_off(3) + R1_FU, W3);
            SMF(c, SIG::rec_off(1) + R1_DINV) = Mi[0]; SMF(c, SIG::rec_off(1) + R1_U) = Mi[1];
            SMF(c, SIG::rec_off(2) + R1_DINV) = Mi[2]; SMF(c, SIG::rec_off(2) + R1_U) = Mi[3];
            SMF(c, SIG::rec_off(3) + R1_DINV) = Mi[4]; SMF(c, SIG::rec_off(3) + R1_U) = Mi[5];
        }
    }
    jb_syncwarp(c);
    // ======================= base: all-reduce, 6x6 solve, back-substitution ======================================
    SymY Yb;
    {
        const RecDbl* rd = JB_RDBL + c.sub;
        double Kd[14];
        load_doubles(rd->placement + 12, Kd, 7);
        inertia_to_sym(Kd[3], mk(Kd[4], Kd[5], Kd[6]), Kd + 7, Yb);
        Mot f = sm_load_mot(c, RF_F);
        const double* const p0 = jb_smem + SIG::pool_off() * 32 + (c.lane - c.sub);
#pragma unroll
        for (int sl = 0; sl < L; ++sl) {
#pragma unroll
            for (int k = 0; k < 6; ++k) { Yb.A[k] += p0[k * 32 + sl]; Yb.D[k] += p0[(15 + k) * 32 + sl]; }
#pragma unroll
            for (int k = 0; k < 9; ++k) Yb.B[k] += p0[(6 + k) * 32 + sl];
            f.l.x += p0[21 * 32 + sl]; f.l.y += p0[22 * 32 + sl]; f.l.z += p0[23 * 32 + sl];
            f.a.x += p0[24 * 32 + sl]; f.a.y += p0[25 * 32 + sl]; f.a.z += p0[26 * 32 + sl];
        }
        const double b[6] = {-f.l.x, -f.l.y, -f.l.z, -f.a.x, -f.a.y, -f.a.z};
        double x[6];
        spd_solve6(Yb, b, x);
        double* const rp = jb_smem + c.lane;
#pragma unroll
        for (int k = 0; k < 6; ++k) RP(RF_A + k) = x[k];
        // IMU capture: base acceleration in the gravity-free frame
        double* const ip = jb_smem + (SIG::imu_off() + 6) * 32 + c.lane;
#pragma unroll
        for (int k = 0; k < 6; ++k) ip[k * 32] += x[k];
        Mot xb; xb.l = mk(x[0], x[1], x[2]); xb.a = mk(x[3], x[4], x[5]);
        const double d1 = C1 - (dot(B1.l, xb.l) + dot(B1.a, xb.a));
        const double d2 = C2 - (dot(B2.l, xb.l) + dot(B2.a, xb.a));
        const double d3 = C3 - (dot(B3.l, xb.l) + dot(B3.a, xb.a));
        SMF(c, SIG::rec_off(1) + R1_A) = s1 * d1;
        SMF(c, SIG::rec_off(2) + R1_A) = s2 * d2;
        SMF(c, SIG::rec_off(3) + R1_A) = s3 * d3;
    }
    // joint position bounds: only envs with a bound in play go on (out of line, everything it needs is in shared memory)
    if (KP->fast_bounds) {
        const bool mine = out_any || SMF(c, SIG::rec_off(1) + R1_BEN) != 0.0 || SMF(c, SIG::rec_off(2) + R1_BEN) != 0.0 ||
                          SMF(c, SIG::rec_off(3) + R1_BEN) != 0.0;
        if (jb_any(c, mine)) { bounds_solve_quadruped(c, up_to_date, status); out_any = false; }
    }
    jb_syncwarp(c);
    if constexpr (STAGE) {
        // Runge-Kutta accumulators: SV += wb VS, SA += wb A (A as the bound solver may have left it)
        if (wb != 0.0) {
            double* const rp = jb_smem + c.lane;
#pragma unroll
            for (int k = 0; k < 6; ++k) { RP(RF_SV + k) += wb * vb[k]; RP(RF_SA + k) += wb * RP(RF_A + k); }
#pragma unroll
            for (int r = 1; r < 4; ++r) {
                double* const rq = jb_smem + SIG::rec_off(r) * 32 + c.lane;
                rq[R1_SV * 32] += wb * vl[r];
                rq[R1_SA * 32] += wb * rq[R1_A * 32];
            }
        }
    }
    return out_any;
}

__device__ __noinline__ bool rhs_quadruped_crba(const Ctx c, const bool up_to_date, int* status) {
    return quadruped_crba<false>(c, up_to_date, status, 0.0, 0, 0, 0, 0, 0.0);
}
// One Runge-Kutta stage of the quadruped hot path (make_stage + rhs_fast + the accumulator update of step_rk4_t) in one
// call; see quadruped_crba.
__device__ __noinline__ void stage_quadruped_crba(const Ctx c, const double wq, const int kv1, const int ka1, const int kvf,
                                                  const int kaf, const double wb, int* status) {
    if (quadruped_crba<true>(c, false, status, wq, kv1, ka1, kvf, kaf, wb)) *status |= ENV_RETRY_FULL;
}

// Engine::computeRobotsDynamics: the sweeps give the unconstrained accelerations; then the constraint path
// (Engine::computeAcceleration with enabled constraints, engine.cc:3709-3866) corrects them if needed.
// Joint position bounds (computePositionLimitsForcesAlgo, engine.cc:3253-3338): leaving [lo, hi] enables the
// joint's constraint; the update also runs while this lane owns enabled constraints (they may switch off).
JB_DI void rhs(const Ctx c, const bool up_to_date, int* status) {
    JB_PROF_T(t_rhs);
    JB_PROF_COUNT(8, 1);                                   // calls of rhs() per warp (each diverged subset counts)
    JB_PROF_COUNT(9, __popc(__activemask()));              // lanes present at the call
    const bool cons_active = KP->cons_on && SMF(c, KP->cons_off) != 0.0;
    const bool out = (KP->sig_id == SigQuadruped::ID)
                         ? (KP->opt.contact_model == JB_CONTACT_CONSTRAINT ? rhs_static_quadruped_cons(c, up_to_date, status)
                                                                           : rhs_static_quadruped(c, up_to_date, status))
                         : rhs_dynamic<true>(c, up_to_date, status);
    JB_PROF_ADD(0, t_rhs);                                 // the sweeps
    if (!KP->cons_on) { if (out) *status |= JB_ENV_JOINT_LIMIT; return; }
    JB_PROF_T(t_upd);
    if (!up_to_date && (out || cons_active)) cons_update_bounds(c, status);
    JB_PROF_ADD(1, t_upd);
    JB_PROF_T(t_solve);
    if (__any_sync(c.gmask, SMF(c, KP->cons_off) != 0.0)) {
        // quadruped-shaped plans with contact constraints only: structured solve; anything else: generic
        bool structured = KP->cq_on && !(c.flags & CTX_IGNORE_BOUNDS);
        if (structured) {
            const double own_contact = CST(cs_contact((KP->cslots + c.sub)->contact)) != 0.0 ? 1.0 : 0.0;
            structured = __all_sync(c.gmask, SMF(c, KP->cons_off) == own_contact);
        }
#ifdef JB_DEBUG_COUNTS
        if (c.sub == 0) {
            extern long long jb_dbg_counts[8];
            const bool bd = KP->bd_on && !(c.flags & CTX_IGNORE_BOUNDS);
            ++jb_dbg_counts[structured ? 0 : (bd ? 1 : ((KP->lb_on && !(c.flags & CTX_IGNORE_BOUNDS)) ? 2 : 3))];
        }
#endif
        if (structured) {
            Ctx cu = c;
#ifndef JB_HOST_EMUL
            if (KP->uniform_solver && __activemask() == 0xffffffffu) cu.flags |= CTX_UNIFORM_WARP;
#endif
            cons_solve_quadruped(cu, status);
        }
        else if (KP->bd_on && !(c.flags & CTX_IGNORE_BOUNDS) && __all_sync(c.gmask, SMF(c, KP->cons_off) < CONS_BOUND_UNIT))
            cons_solve_bodies(c, status);   // contact frames only
        else if (KP->lb_on && !(c.flags & CTX_IGNORE_BOUNDS)) cons_solve_blocks(c, status);
        else constrained_solve(c, status);
    }
    JB_PROF_ADD(2, t_solve);                               // everything after the bound update: votes + solver
}
// fast path: sweeps only
JB_DI void rhs_fast(const Ctx c, const bool up_to_date, int* status) {
    const bool out = (KP->sig_id == SigQuadruped::ID)
                         ? (KP->rhs_variant == 1 ? rhs_quadruped_crba(c, up_to_date, status) : rhs_static_quadruped(c, up_to_date, status))
                         : rhs_dynamic<false>(c, up_to_date, status);
    if (out) *status |= ENV_RETRY_FULL;
}
template <class SIG>
JB_DI void rhs_sig(const Ctx c, const bool up_to_date, int* status) {
    if constexpr (sig_is_fast<SIG>::value) rhs_fast(c, up_to_date, status);
    else rhs(c, up_to_date, status);
}

// ------------------------------------------------------------------------------------------
// Lie-group integration of one record: out = integrate(q, w * kv)   (pinocchio::integrate as used
// by StateBase::sum, core/include/jiminy/core/stepper/lie_group.h:446-455)
// q read at q_off, velocity increment given in registers, result written at out_off.
// ------------------------------------------------------------------------------------------
JB_DI void integrate_free(const Ctx& c, int q_off, const double* dv, int out_off) {
    // SpecialEuclideanOperationTpl<3>::integrate_impl : M1 = M0 * exp6(v)
    const double qx = SMF(c, q_off + 3), qy = SMF(c, q_off + 4), qz = SMF(c, q_off + 5), qw = SMF(c, q_off + 6);
    double R0[9];
    quat_to_R(qx, qy, qz, qw, R0);
    const V3 v = mk(dv[0], dv[1], dv[2]), w = mk(dv[3], dv[4], dv[5]);
    // pinocchio::exp6 (explog.hpp)
    const double t2 = dot(w, w);
    const double t = sqrt(t2);
    double st, ct;
    sincos(t, &st, &ct);
    const double inv_t2 = 1.0 / t2;
    const bool small = t < TAYLOR_PREC3;
    const double alpha_wxv = small ? 0.5 - t2 / 24.0 : (1.0 - ct) * inv_t2;
    const double alpha_v = small ? 1.0 - t2 / 6.0 : st / t;
    const double alpha_w = small ? 1.0 / 6.0 - t2 / 120.0 : (1.0 - alpha_v) * inv_t2;
    const double diag = small ? 1.0 - t2 / 2.0 : ct;
    const V3 pe = alpha_v * v + (alpha_w * dot(w, v)) * w + alpha_wxv * cross(w, v);
    double Re[9];
    Re[0] = alpha_wxv * w.x * w.x + diag; Re[1] = alpha_wxv * w.x * w.y - alpha_v * w.z; Re[2] = alpha_wxv * w.x * w.z + alpha_v * w.y;
    Re[3] = alpha_wxv * w.y * w.x + alpha_v * w.z; Re[4] = alpha_wxv * w.y * w.y + diag; Re[5] = alpha_wxv * w.y * w.z - alpha_v * w.x;
    Re[6] = alpha_wxv * w.z * w.x - alpha_v * w.y; Re[7] = alpha_wxv * w.z * w.y + alpha_v * w.x; Re[8] = alpha_wxv * w.z * w.z + diag;
    double R1[9];
    mat3mul(R0, Re, R1);
    const V3 p1 = mk(SMF(c, q_off), SMF(c, q_off + 1), SMF(c, q_off + 2)) + rmul(R0, pe);
    // rotation -> quaternion (Eigen), sign continuity, first-order normalisation
    double q[4];
    double tr = R1[0] + R1[4] + R1[8];
    if (tr > 0.0) {
        double s = sqrt(tr + 1.0);
        q[3] = 0.5 * s; s = 0.5 / s;
        q[0] = (R1[7] - R1[5]) * s; q[1] = (R1[2] - R1[6]) * s; q[2] = (R1[3] - R1[1]) * s;
    } else {
        int i = 0;
        if (R1[4] > R1[0]) i = 1;
        if (R1[8] > R1[4 * i]) i = 2;
        const int j = (i + 1) % 3, k = (j + 1) % 3;
        double s = sqrt(R1[4 * i] - R1[4 * j] - R1[4 * k] + 1.0);
        double qq[4];
        qq[i] = 0.5 * s; s = 0.5 / s;
        qq[3] = (R1[3 * k + j] - R1[3 * j + k]) * s;
        qq[j] = (R1[3 * j + i] + R1[3 * i + j]) * s;
        qq[k] = (R1[3 * k + i] + R1[3 * i + k]) * s;
        q[0] = qq[0]; q[1] = qq[1]; q[2] = qq[2]; q[3] = qq[3];
    }
    const double dp = q[0] * qx + q[1] * qy + q[2] * qz + q[3] * qw;
    if (dp < 0.0) { q[0] = -q[0]; q[1] = -q[1]; q[2] = -q[2]; q[3] = -q[3]; }
    const double N2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
    const double alpha = (3.0 - N2) / 2.0;
    SMF(c, out_off) = p1.x; SMF(c, out_off + 1) = p1.y; SMF(c, out_off + 2) = p1.z;
    SMF(c, out_off + 3) = q[0] * alpha; SMF(c, out_off + 4) = q[1] * alpha; SMF(c, out_off + 5) = q[2] * alpha; SMF(c, out_off + 6) = q[3] * alpha;
}

// SpecialOrthogonalOperationTpl<3>::integrate_impl on the quaternion slots of a spherical record: quat * exp3(omega),
// firstOrderNormalize; the linear slots stay zero.
JB_DI void integrate_sph(const Ctx& c, int q_off, const double* dv, int out_off) {
    const double q0[4] = {SMF(c, q_off + 3), SMF(c, q_off + 4), SMF(c, q_off + 5), SMF(c, q_off + 6)};
    double pOmega[4], q[4];
    quat_exp3(mk(dv[3], dv[4], dv[5]), pOmega);
    quat_mul(q0, pOmega, q);
    const double N2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
    const double alpha = (3.0 - N2) / 2.0;
    SMF(c, out_off) = 0.0; SMF(c, out_off + 1) = 0.0; SMF(c, out_off + 2) = 0.0;
    SMF(c, out_off + 3) = q[0] * alpha; SMF(c, out_off + 4) = q[1] * alpha; SMF(c, out_off + 5) = q[2] * alpha; SMF(c, out_off + 6) = q[3] * alpha;
}
JB_DI void integrate_big(const Ctx& c, int kind, int q_off, const double* dv, int out_off) {
    if (kind == REC_SPH) integrate_sph(c, q_off, dv, out_off);
    else integrate_free(c, q_off, dv, out_off);
}

JB_DI void integrate_1dof(const Ctx& c, int kind, int q_off, double dv, int out_off) {
    if (kind == REC_REVU) {
        // SpecialOrthogonalOperationTpl<2>::integrate_impl
        const double ca = SMF(c, q_off), sa = SMF(c, q_off + 1);
        double so, co;
        sincos(dv, &so, &co);
        const double o0 = co * ca - so * sa, o1 = so * ca + co * sa;
        const double k = (3.0 - (o0 * o0 + o1 * o1)) / 2.0;
        SMF(c, out_off) = o0 * k; SMF(c, out_off + 1) = o1 * k;
    } else {
        SMF(c, out_off) = SMF(c, q_off) + dv;
    }
}

// Stage state for a Runge-Kutta stage / Euler update over all records of the lane:
//   QS = integrate(Q, wq * kv) ; VS = V + wv * ka          (StateBase::sum)
// kv is read from field `kv_f1 / kv_ff`, ka from `ka_f1 / ka_ff` (offsets inside 1-dof / free records).
template <class SIG>
JB_DI void make_stage(const Ctx& c, double w, int kv1, int ka1, int kvf, int kaf) {
    SIG::for_each_forward([&](auto r_) {
        const int r = r_;
        const int kind = SIG::kind(r, c);
        if (kind == REC_PAD) return;
        const int base = SIG::rec_off(r);
        double* const rp = jb_smem + base * 32 + c.lane;
        if (rec_is_big(kind)) {
            double dv[6], vs[6];
#pragma unroll
            for (int k = 0; k < 6; ++k) { dv[k] = w * RP(kvf + k); vs[k] = RP(RF_V + k) + w * RP(kaf + k); }
            integrate_big(c, kind, base + RF_Q, dv, base + RF_QS);
#pragma unroll
            for (int k = 0; k < 6; ++k) RP(RF_VS + k) = vs[k];
        } else {
            const double dv = w * RP(kv1);
            const double vs = RP(R1_V) + w * RP(ka1);
            integrate_1dof(c, kind, base + R1_Q, dv, base + R1_QS);
            RP(R1_VS) = vs;
        }
    });
}

// copy accepted state -> stage state
template <class SIG>
JB_DI void stage_from_accepted_t(const Ctx& c) {
    SIG::for_each_forward([&](auto r_) {
        const int r = r_;
        const int kind = SIG::kind(r, c);
        if (kind == REC_PAD) return;
        const int base = SIG::rec_off(r);
        double* const rp = jb_smem + base * 32 + c.lane;
        if (rec_is_big(kind)) {
#pragma unroll
            for (int k = 0; k < 7; ++k) RP(RF_QS + k) = RP(RF_Q + k);
#pragma unroll
            for (int k = 0; k < 6; ++k) RP(RF_VS + k) = RP(RF_V + k);
        } else {
            RP(R1_QS) = RP(R1_Q); RP(R1_QS + 1) = RP(R1_Q + 1);
            RP(R1_VS) = RP(R1_V);
        }
    });
}

// returns true when the accepted acceleration of this lane's records contains a NaN
template <class SIG>
JB_DI bool accel_has_nan_t(const Ctx& c) {
    bool bad = false;
    SIG::for_each_forward([&](auto r_) {
        const int r = r_;
        const int kind = SIG::kind(r, c);
        if (kind == REC_PAD) return;
        const int base = SIG::rec_off(r);
        double* const rp = jb_smem + base * 32 + c.lane;
        if (rec_is_big(kind)) {
#pragma unroll
            for (int k = 0; k < 6; ++k) { const double x = RP(RF_A + k); bad |= (x != x); }
        } else { const double x = RP(R1_A); bad |= (x != x); }
    });
    return bad;
}

// ------------------------------------------------------------------------------------------
// Steppers.  EulerExplicitStepper::tryStepImpl (core/src/stepper/euler_explicit_stepper.cc:6-22)
// and AbstractRungeKuttaStepper::tryStepImpl with the RK4 tableau
// (abstract_runge_kutta_stepper.cc:25-77, runge_kutta4_stepper.h:12-23).  Both never fail; they
// leave the new accepted state in (Q, V, A) and return dt = INF.
// ------------------------------------------------------------------------------------------
template <class SIG>
__device__ __noinline__ void step_euler_t(const Ctx c, double dt, int* status) {
    // x <- x (+) dt * dx ; dx <- f(t + dt, x)
    make_stage<SIG>(c, dt, R1_V, R1_A, RF_V, RF_A);
    rhs_sig<SIG>(c, false, status);
    SIG::for_each_forward([&](auto r_) {
        const int r = r_;
        const int kind = SIG::kind(r, c);
        if (kind == REC_PAD) return;
        const int base = SIG::rec_off(r);
        double* const rp = jb_smem + base * 32 + c.lane;
        if (rec_is_big(kind)) {
#pragma unroll
            for (int k = 0; k < 7; ++k) RP(RF_Q + k) = RP(RF_QS + k);
#pragma unroll
            for (int k = 0; k < 6; ++k) RP(RF_V + k) = RP(RF_VS + k);
        } else {
            RP(R1_Q) = RP(R1_QS); RP(R1_Q + 1) = RP(R1_QS + 1);
            RP(R1_V) = RP(R1_VS);
        }
    });
}

template <class SIG>
__device__ __noinline__ void step_rk4_t(const Ctx c, double dt, int* status) {
    // RK4 tableau: A(i, i-1) = {-, 1/2, 1/2, 1}, b = {1/6, 1/3, 1/3, 1/6} -- selected, not indexed (a run-time index
    // would put the tables in local memory and stall every stage on their loads)
    // accumulators: S = (dt b0) k0
    SIG::for_each_forward([&](auto r_) {
        const int r = r_;
        const int kind = SIG::kind(r, c);
        if (kind == REC_PAD) return;
        const int base = SIG::rec_off(r);
        double* const rp = jb_smem + base * 32 + c.lane;
        const double w = dt * (1.0 / 6.0);
        if (rec_is_big(kind)) {
#pragma unroll
            for (int k = 0; k < 6; ++k) { RP(RF_SV + k) = 0.0 + w * RP(RF_V + k); RP(RF_SA + k) = 0.0 + w * RP(RF_A + k); }
        } else {
            RP(R1_SV) = 0.0 + w * RP(R1_V);
            RP(R1_SA) = 0.0 + w * RP(R1_A);
        }
    });
    constexpr bool quad_fast = is_fast_quadruped<SIG>::value;
    const bool one_call = quad_fast && KP->quad_stage;
#pragma unroll 1
    for (int i = 1; i < 4; ++i) {
        // stage state from k_{i-1}: kv_{i-1} is V (i == 1) or the previous stage velocity VS, ka_{i-1} is in A
        const double w = dt * (i == 3 ? 1.0 : 0.5);
        if constexpr (quad_fast) {
            if (one_call) {
                stage_quadruped_crba(c, w, i == 1 ? R1_V : R1_VS, R1_A, i == 1 ? RF_V : RF_VS, RF_A,
                                     dt * (i == 3 ? 1.0 / 6.0 : 1.0 / 3.0), status);
                continue;
            }
        }
        if (i == 1) make_stage<SIG>(c, w, R1_V, R1_A, RF_V, RF_A);
        else make_stage<SIG>(c, w, R1_VS, R1_A, RF_VS, RF_A);
        rhs_sig<SIG>(c, false, status);
        const double wb = dt * (i == 3 ? 1.0 / 6.0 : 1.0 / 3.0);
        SIG::for_each_forward([&](auto r_) {
            const int r = r_;
            const int kind = SIG::kind(r, c);
            if (kind == REC_PAD) return;
            const int base = SIG::rec_off(r);
            double* const rp = jb_smem + base * 32 + c.lane;
            if (rec_is_big(kind)) {
#pragma unroll
                for (int k = 0; k < 6; ++k) { RP(RF_SV + k) += wb * RP(RF_VS + k); RP(RF_SA + k) += wb * RP(RF_A + k); }
            } else {
                RP(R1_SV) += wb * RP(R1_VS);
                RP(R1_SA) += wb * RP(R1_A);
            }
        });
    }
    // candidate solution = x0 (+) sum ; it is always accepted, then dx = f(t + dt, x)
    if constexpr (quad_fast) {
        if (one_call) stage_quadruped_crba(c, 1.0, R1_SV, R1_SA, RF_SV, RF_SA, 0.0, status);
        else make_stage<SIG>(c, 1.0, R1_SV, R1_SA, RF_SV, RF_SA);
    } else {
        make_stage<SIG>(c, 1.0, R1_SV, R1_SA, RF_SV, RF_SA);
    }
    SIG::for_each_forward([&](auto r_) {
        const int r = r_;
        const int kind = SIG::kind(r, c);
        if (kind == REC_PAD) return;
        const int base = SIG::rec_off(r);
        double* const rp = jb_smem + base * 32 + c.lane;
        if (rec_is_big(kind)) {
#pragma unroll
            for (int k = 0; k < 7; ++k) RP(RF_Q + k) = RP(RF_QS + k);
#pragma unroll
            for (int k = 0; k < 6; ++k) RP(RF_V + k) = RP(RF_VS + k);
        } else {
            RP(R1_Q) = RP(R1_QS); RP(R1_Q + 1) = RP(R1_QS + 1);
            RP(R1_V) = RP(R1_VS);
        }
    });
    if (!one_call) rhs_sig<SIG>(c, false, status);
}

// run-time dispatch on the plan signature
JB_DI void stage_from_accepted(const Ctx& c) {
    if (KP->sig_id == SigQuadruped::ID) stage_from_accepted_t<SigQuadruped>(c);
    else stage_from_accepted_t<SigDynamic<false>>(c);
}
JB_DI bool accel_has_nan(const Ctx& c) {
    if (KP->sig_id == SigQuadruped::ID) return accel_has_nan_t<SigQuadruped>(c);
    return accel_has_nan_t<SigDynamic<false>>(c);
}
template <bool FAST>
JB_DI void step_euler(const Ctx c, double dt, int* status) {
    if constexpr (FAST) {
        if (KP->sig_id == SigQuadruped::ID) step_euler_t<FastOf<SigQuadruped>>(c, dt, status);
        else step_euler_t<FastOf<SigDynamic<false>>>(c, dt, status);
    } else {
        if (KP->sig_id == SigQuadruped::ID) step_euler_t<SigQuadruped>(c, dt, status);
        else step_euler_t<SigDynamic<false>>(c, dt, status);
    }
}
template <bool FAST>
JB_DI void step_rk4(const Ctx c, double dt, int* status) {
    if constexpr (FAST) {
        if (KP->sig_id == SigQuadruped::ID) step_rk4_t<FastOf<SigQuadruped>>(c, dt, status);
        else step_rk4_t<FastOf<SigDynamic<false>>>(c, dt, status);
    } else {
        if (KP->sig_id == SigQuadruped::ID) step_rk4_t<SigQuadruped>(c, dt, status);
        else step_rk4_t<SigDynamic<false>>(c, dt, status);
    }
}

// ------------------------------------------------------------------------------------------
// Dormand-Prince 5(4) with step-size control: AbstractRungeKuttaStepper::tryStepImpl
// (core/src/stepper/abstract_runge_kutta_stepper.cc:25-77) with the DOPRI tableau and
// RungeKuttaDOPRIStepper::adjustStep / computeError (runge_kutta_dopri_stepper.cc:18-82,
// runge_kutta_dopri_stepper.h:12-47).  Only the stage accelerations ka_j are stored (7 history
// slots per dof): the stage velocities are kv_j = V + dt * sum_m A_jm ka_m, so that
//   sum_j (dt A_ij) kv_j = dt c_i V + dt^2 sum_m (A A)_im ka_m.
// ------------------------------------------------------------------------------------------
namespace dopri {
__device__ const double A[7][7] = {
    {0, 0, 0, 0, 0, 0, 0},
    {1.0 / 5.0, 0, 0, 0, 0, 0, 0},
    {3.0 / 40.0, 9.0 / 40.0, 0, 0, 0, 0, 0},
    {44.0 / 45.0, -56.0 / 15.0, 32.0 / 9.0, 0, 0, 0, 0},
    {19372.0 / 6561.0, -25360.0 / 2187.0, 64448.0 / 6561.0, -212.0 / 729.0, 0, 0, 0},
    {9017.0 / 3168.0, -355.0 / 33.0, 46732.0 / 5247.0, 49.0 / 176.0, -5103.0 / 18656.0, 0, 0},
    {35.0 / 384.0, 0.0, 500.0 / 1113.0, 125.0 / 192.0, -2187.0 / 6784.0, 11.0 / 84.0, 0}};
__device__ const double A2[7][7] = {   // A * A
    {0, 0, 0, 0, 0, 0, 0},
    {0, 0, 0, 0, 0, 0, 0},
    {0.045, 0, 0, 0, 0, 0, 0},
    {-0.48, 0.8, 0, 0, 0, 0, 0},
    {-1.8667885992988873, 3.2958390489254685, -1.0339887212315195, 0, 0, 0, 0},
    {-2.018939393939394, 4.136363636363637, -1.696969696969697, 0.07954545454545454, 0, 0, 0},
    {0.09114583333333333, 0.0, 0.31446540880503143, 0.13020833333333334, -0.03581957547169811, 0, 0}};
__device__ const double Cn[7] = {0.0, 0.2, 0.3, 0.8, 8.0 / 9.0, 1.0, 1.0};
__device__ const double E[7] = {5179.0 / 57600.0, 0.0, 7571.0 / 16695.0, 393.0 / 640.0, -92097.0 / 339200.0, 187.0 / 2100.0, 1.0 / 40.0};
__device__ const double EA[7] = {0.08849392361111111, 0.0, 0.3206229410002995, 0.12002604166666667, -0.03241671580188679, 0.003273809523809524, 0.0};
}  // namespace dopri

// pinocchio::log3 / log6 (explog.hpp) on register arrays
JB_DI void log6_regs(const double* R, V3 p, double* out) {
    const double PI = 3.14159265358979323846;
    const double tr = R[0] + R[4] + R[8];
    double theta;
    if (tr >= 3.0) theta = 0.0;
    else if (tr <= -1.0) theta = PI;
    else theta = acos((tr - 1.0) / 2.0);
    V3 w;
    if (theta >= PI - 1e-2) {
        const double cphi = -(tr - 1.0) / 2.0;
        const double beta = theta * theta / (1.0 + cphi);
        const double tx = (R[0] + cphi) * beta, ty = (R[4] + cphi) * beta, tz = (R[8] + cphi) * beta;
        w.x = (R[7] > R[5] ? 1.0 : -1.0) * (tx > 0.0 ? sqrt(tx) : 0.0);
        w.y = (R[2] > R[6] ? 1.0 : -1.0) * (ty > 0.0 ? sqrt(ty) : 0.0);
        w.z = (R[3] > R[1] ? 1.0 : -1.0) * (tz > 0.0 ? sqrt(tz) : 0.0);
    } else {
        const double t = ((theta > TAYLOR_PREC3) ? theta / sin(theta) : 1.0) / 2.0;
        w = mk(t * (R[7] - R[5]), t * (R[2] - R[6]), t * (R[3] - R[1]));
    }
    const double t = theta, t2 = t * t;
    double alpha, beta;
    if (t < TAYLOR_PREC3) { alpha = 1.0 - t2 / 12.0 - t2 * t2 / 720.0; beta = 1.0 / 12.0 + t2 / 720.0; }
    else {
        double st, ct;
        sincos(t, &st, &ct);
        alpha = t * st / (2.0 * (1.0 - ct));
        beta = 1.0 / t2 - st / (2.0 * t * (1.0 - ct));
    }
    const V3 lin = alpha * p - 0.5 * cross(w, p) + (beta * dot(w, p)) * w;
    out[0] = lin.x; out[1] = lin.y; out[2] = lin.z; out[3] = w.x; out[4] = w.y; out[5] = w.z;
}
// pinocchio::difference(q0, q1) for the free-flyer: log6(M0^-1 M1)
JB_DI void difference_free(const double* q0, const double* q1, double* out) {
    double R0[9], R1[9], Rr[9];
    quat_to_R(q0[3], q0[4], q0[5], q0[6], R0);
    quat_to_R(q1[3], q1[4], q1[5], q1[6], R1);
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) Rr[3 * i + j] = R0[i] * R1[j] + R0[3 + i] * R1[3 + j] + R0[6 + i] * R1[6 + j];   // R0^T R1
    const V3 dp = rtmul(R0, mk(q1[0] - q0[0], q1[1] - q0[1], q1[2] - q0[2]));
    log6_regs(Rr, dp, out);
}
// SpecialOrthogonalOperationTpl<2>::difference
JB_DI double difference_so2(double c0, double s0, double c1, double s1) {
    const double PI = 3.14159265358979323846;
    const double R00 = c0 * c1 + s0 * s1, R10 = c0 * s1 - s0 * c1;
    const double tr = 2.0 * R00;
    const bool pos = R10 > 0.0;
    if (tr > 2.0) return 0.0;
    if (tr < -2.0) return pos ? PI : -PI;
    if (tr > 2.0 - 1e-2) return asin((R10 - (-R10)) / 2.0);
    return pos ? acos(tr / 2.0) : -acos(tr / 2.0);
}

// returns 0 = success, 1 = failure (step rejected, dt shrunk), 2 = error (NaN)
__device__ __noinline__ int step_dopri(const Ctx c, double* dt_io, int* status) {
    const int L = KP->L;
    const double h = *dt_io;
    // ka_0 = derivative at the accepted state
    for (int r = 0; r < KP->nrec; ++r) {
        const RecInt* ri = KP->rint + (r * L + c.sub);
        if (ri->kind == REC_PAD) continue;
        double* const rp = jb_smem + KP->rec_off[r] * 32 + c.lane;
        if (rec_is_big(ri->kind)) {
#pragma unroll
            for (int k = 0; k < 6; ++k) RP(RF_KA + k) = RP(RF_A + k);
        } else RP(R1_KA) = RP(R1_A);
    }
#pragma unroll 1
    for (int i = 1; i < 7; ++i) {
        for (int r = 0; r < KP->nrec; ++r) {
            const RecInt* ri = KP->rint + (r * L + c.sub);
            if (ri->kind == REC_PAD) continue;
            const int base = KP->rec_off[r];
            double* const rp = jb_smem + base * 32 + c.lane;
            if (rec_is_big(ri->kind)) {
                double dv[6], vs[6];
#pragma unroll
                for (int k = 0; k < 6; ++k) {
                    double s2 = 0.0, s1 = 0.0;
                    for (int m = 0; m < i; ++m) { s2 += dopri::A2[i][m] * RP(RF_KA + 6 * m + k); s1 += dopri::A[i][m] * RP(RF_KA + 6 * m + k); }
                    dv[k] = h * dopri::Cn[i] * RP(RF_V + k) + h * h * s2;
                    vs[k] = RP(RF_V + k) + h * s1;
                }
                integrate_big(c, ri->kind, base + RF_Q, dv, base + RF_QS);
#pragma unroll
                for (int k = 0; k < 6; ++k) RP(RF_VS + k) = vs[k];
            } else {
                double s2 = 0.0, s1 = 0.0;
                for (int m = 0; m < i; ++m) { s2 += dopri::A2[i][m] * RP(R1_KA + m); s1 += dopri::A[i][m] * RP(R1_KA + m); }
                const double dv = h * dopri::Cn[i] * RP(R1_V) + h * h * s2;
                const double vs = RP(R1_V) + h * s1;
                integrate_1dof(c, ri->kind, base + R1_Q, dv, base + R1_QS);
                RP(R1_VS) = vs;
            }
        }
        rhs(c, false, status);
        for (int r = 0; r < KP->nrec; ++r) {
            const RecInt* ri = KP->rint + (r * L + c.sub);
            if (ri->kind == REC_PAD) continue;
            double* const rp = jb_smem + KP->rec_off[r] * 32 + c.lane;
            if (rec_is_big(ri->kind)) {
#pragma unroll
                for (int k = 0; k < 6; ++k) RP(RF_KA + 6 * i + k) = RP(RF_A + k);
            } else RP(R1_KA + i) = RP(R1_A);
        }
    }
    // (QS, VS) now hold the 5th-order candidate (A[6][:] == b).  Error estimate against the embedded
    // 4th-order solution, scaled by tolAbs + tolRel * |x0 (-) neutral|.  NB: Engine::start hands
    // (stepper.tolAbs, stepper.tolRel) to a constructor declared (tolRel, tolAbs) (engine.cc:1161-1163):
    // the two options act swapped, as in the reference.
    const double tolRel_ = KP->opt.tol_abs, tolAbs_ = KP->opt.tol_rel;
    double err = 0.0;
    bool isnan_ = false;
    for (int r = 0; r < KP->nrec; ++r) {
        const RecInt* ri = KP->rint + (r * L + c.sub);
        if (ri->kind == REC_PAD) continue;
        const int base = KP->rec_off[r];
        double* const rp = jb_smem + base * 32 + c.lane;
        if (rec_is_big(ri->kind)) {
            double dv[6], v4[6], q0[7], qc[7], q4[7], sc[6], eq[6];
#pragma unroll
            for (int k = 0; k < 6; ++k) {
                double s2 = 0.0, s1 = 0.0;
                for (int m = 0; m < 7; ++m) { s2 += dopri::EA[m] * RP(RF_KA + 6 * m + k); s1 += dopri::E[m] * RP(RF_KA + 6 * m + k); }
                dv[k] = h * RP(RF_V + k) + h * h * s2;
                v4[k] = RP(RF_V + k) + h * s1;
            }
            integrate_big(c, ri->kind, base + RF_Q, dv, base + RF_SV);   // scratch: SV|SA (12 doubles)
#pragma unroll
            for (int k = 0; k < 7; ++k) { q0[k] = RP(RF_Q + k); qc[k] = RP(RF_QS + k); q4[k] = RP(RF_SV + k); }
            const double qn[7] = {0, 0, 0, 0, 0, 0, 1};
            if (ri->kind == REC_SPH) {
                const V3 s3 = difference_sph(q0 + 3, qn + 3), e3 = difference_sph(qc + 3, q4 + 3);
                sc[0] = sc[1] = sc[2] = 0.0; eq[0] = eq[1] = eq[2] = 0.0;
                sc[3] = s3.x; sc[4] = s3.y; sc[5] = s3.z; eq[3] = e3.x; eq[4] = e3.y; eq[5] = e3.z;
            } else {
                difference_free(q0, qn, sc);
                difference_free(qc, q4, eq);
            }
#pragma unroll
            for (int k = 0; k < 6; ++k) {
                const double e1 = fabs(eq[k] / (fabs(sc[k]) * tolRel_ + tolAbs_));
                const double e2 = fabs((RP(RF_VS + k) - v4[k]) / (fabs(RP(RF_V + k)) * tolRel_ + tolAbs_));
                isnan_ |= (e1 != e1) || (e2 != e2);
                err = fmax(err, fmax(e1, e2));
            }
        } else {
            double s2 = 0.0, s1 = 0.0;
            for (int m = 0; m < 7; ++m) { s2 += dopri::EA[m] * RP(R1_KA + m); s1 += dopri::E[m] * RP(R1_KA + m); }
            const double dv = h * RP(R1_V) + h * h * s2;
            const double v4 = RP(R1_V) + h * s1;
            double eq, sq;
            if (ri->kind == REC_REVU) {
                integrate_1dof(c, ri->kind, base + R1_Q, dv, base + R1_SV);   // scratch: SV, SA
                eq = difference_so2(RP(R1_QS), RP(R1_QS + 1), RP(R1_SV), RP(R1_SA));
                sq = difference_so2(RP(R1_Q), RP(R1_Q + 1), 1.0, 0.0);
            } else {
                eq = (RP(R1_Q) + dv) - RP(R1_QS);
                sq = 0.0 - RP(R1_Q);
            }
            const double e1 = fabs(eq / (fabs(sq) * tolRel_ + tolAbs_));
            const double e2 = fabs((RP(R1_VS) - v4) / (fabs(RP(R1_V)) * tolRel_ + tolAbs_));
            isnan_ |= (e1 != e1) || (e2 != e2);
            err = fmax(err, fmax(e1, e2));
        }
    }
    for (int o = 1; o < L; o <<= 1) err = fmax(err, jb_shfl_xor(c, err, o));
    isnan_ = jb_any(c, isnan_);
    auto restore = [&]() {
        for (int r = 0; r < KP->nrec; ++r) {
            const RecInt* ri = KP->rint + (r * L + c.sub);
            if (ri->kind == REC_PAD) continue;
            double* const rp = jb_smem + KP->rec_off[r] * 32 + c.lane;
            if (rec_is_big(ri->kind)) {
#pragma unroll
                for (int k = 0; k < 6; ++k) RP(RF_A + k) = RP(RF_KA + k);
            } else RP(R1_A) = RP(R1_KA);
        }
    };
    if (isnan_) { restore(); return 2; }   // "The estimated integration error contains 'nan'." -> IS_ERROR
    const double ORDER = 5.0, SAFETY = 0.8, ERROR_THRESHOLD = 0.5, MIN_FACTOR = 0.2, MAX_FACTOR = 5.0;
    if (err < 1.0) {
        if (err < fmin(ERROR_THRESHOLD, pow(SAFETY, ORDER))) {
            const double clipped = fmax(err, pow(MAX_FACTOR / SAFETY, -ORDER));
            *dt_io = h * (SAFETY * pow(clipped, -1.0 / ORDER));
        }
        // accept: x <- candidate, dx <- k7 (FSAL, already in the A fields)
        for (int r = 0; r < KP->nrec; ++r) {
            const RecInt* ri = KP->rint + (r * L + c.sub);
            if (ri->kind == REC_PAD) continue;
            double* const rp = jb_smem + KP->rec_off[r] * 32 + c.lane;
            if (rec_is_big(ri->kind)) {
#pragma unroll
                for (int k = 0; k < 7; ++k) RP(RF_Q + k) = RP(RF_QS + k);
#pragma unroll
                for (int k = 0; k < 6; ++k) RP(RF_V + k) = RP(RF_VS + k);
            } else {
                RP(R1_Q) = RP(R1_QS); RP(R1_Q + 1) = RP(R1_QS + 1);
                RP(R1_V) = RP(R1_VS);
            }
        }
        bool bad = accel_has_nan(c);
        bad = jb_any(c, bad);
        return bad ? 2 : 0;
    }
    *dt_io = h * fmax(SAFETY * pow(err, -1.0 / (ORDER - 2.0)), MIN_FACTOR);
    restore();
    return 1;
}

JB_DI bool period_hit(double t, double period) {
    // `dtNext < SIMULATION_MIN_TIMESTEP || period - dtNext < STEPPER_MIN_TIMESTEP` (engine.cc:1924-1927, :2388-2395)
    const double dtNext = period - fmod(t, period);
    return dtNext < SIMULATION_MIN_TIMESTEP || period - dtNext < STEPPER_MIN_TIMESTEP;
}

// external wrench (joint frame) applied on record r by this lane in the last dynamics evaluation
JB_DI void add_cached_ext_wrench(const Ctx& c, int r, int L, Mot& fext) {
    for (int e = 0; e < KP->n_eslot; ++e) {
        if ((KP->eslots + (e * L + c.sub))->rec != r) continue;
        const double* const xp = jb_smem + (KP->ext_off + ESLOT_SIZE * e) * 32 + c.lane;
        fext.l = fext.l + mk(xp[6 * 32], xp[7 * 32], xp[8 * 32]);
        fext.a = fext.a + mk(xp[9 * 32], xp[10 * 32], xp[11 * 32]);
    }
}

// Active set of the impulse forces, held values of the profile forces (engine.cc:1843-1917, :1214-1238
// at start) -> the slot wrenches the next dynamics evaluations apply.  The active set is a pure function
// of t: active <=> t > t_k - eps and not t >= t_k + dt_k - eps, re-evaluated at every scheduler
// iteration like the reference does.  Returns the next impulse breakpoint (INF if none).
JB_DI double refresh_external_forces(const Ctx& c, double t, bool at_start, bool finite_period, bool& changed) {
    const size_t N = KP->n_pad, col = c.env;
    for (int k = 0; k < ESLOT_SIZE * KP->n_eslot; ++k) SMF(c, KP->ext_off + k) = 0.0;
    double t_next = D_INF;
    for (int i = 0; i < KP->n_imp; ++i) {
        const double* d = KP->imp_data + static_cast<size_t>(i) * IMPULSE_ROWS * N + col;
        const double ti = d[0], dti = d[N];
        bool active;
        if (at_start) active = ti < STEPPER_MIN_TIMESTEP;
        else {
            active = false;
            if (t > ti - STEPPER_MIN_TIMESTEP) { active = true; changed = true; }
            if (t >= ti + dti - STEPPER_MIN_TIMESTEP) { active = false; changed = true; }
            // impulseForceBreakpoints: next one at least STEPPER_MIN_TIMESTEP ahead (engine.cc:1877-1889)
            if (ti - t >= STEPPER_MIN_TIMESTEP) t_next = fmin(t_next, ti);
            if (ti + dti - t >= STEPPER_MIN_TIMESTEP) t_next = fmin(t_next, ti + dti);
        }
        if (active) {
            double* const xp = jb_smem + (KP->ext_off + ESLOT_SIZE * KP->imp_slot[i]) * 32 + c.lane;
#pragma unroll
            for (int k = 0; k < 6; ++k) xp[k * 32] += d[(2 + k) * N];
        }
    }
    for (int j = 0; j < KP->n_prof; ++j) {
        const double P = KP->prof_period[j];
        const double* pend = KP->prof_pending + static_cast<size_t>(j) * 6 * N + col;
        double* lat = KP->prof_latched + static_cast<size_t>(j) * 6 * N + col;
        double F[6];
        if (P > D_EPS) {
            // finite update period: zero until the first update of the first step, then held between updates
            const bool hit = !at_start && finite_period && period_hit(t, P);
            if (hit) changed = true;
#pragma unroll
            for (int k = 0; k < 6; ++k) {
                F[k] = at_start ? 0.0 : (hit ? pend[k * N] : lat[k * N]);
                if ((hit || at_start) && c.valid && c.sub == 0) lat[k * N] = F[k];
            }
        } else {
#pragma unroll
            for (int k = 0; k < 6; ++k) F[k] = pend[k * N];
        }
        double* const xp = jb_smem + (KP->ext_off + ESLOT_SIZE * KP->prof_slot[j]) * 32 + c.lane;
#pragma unroll
        for (int k = 0; k < 6; ++k) xp[k * 32] += F[k];
    }
    return t_next;
}

// ------------------------------------------------------------------------------------------
// computeExtraTerms (core/src/engine/engine.cc:800-905) on the accepted state, at the end of a
// launch: kinetic (+ rotor) and potential energy, true joint spatial accelerations `data.a`, joint
// internal wrenches `data.f`, subtree inertias `data.Ycrb`, subtree centres of mass `data.com` and
// their velocities `data.vcom`, centroidal momentum `data.hg` and its derivative `data.dhg`.  The
// records still hold liMi / ddq / cached contact forces of the last dynamics evaluation, which was
// made at the accepted state.
//
// Backward accumulation, 27 numbers per subtree (exactly one pool entry): f (6), h (6), fExt (6) as
// spatial forces, and the subtree inertia in ADDITIVE form -- first moment m c (3) and inertia about
// the joint origin (6) -- so that the partial sums of the lanes add up like everything else (the
// reference's compact (m, c, I_com) form with its division per sum does not).  Masses are model
// constants (RecDbl::subtree_mass).
// ------------------------------------------------------------------------------------------
struct SubAcc { Mot f, h, fe; V3 mc; double Io[6]; };
JB_DI void acc_zero(SubAcc& a) {
    a.f = mzero(); a.h = mzero(); a.fe = mzero(); a.mc = mk(0, 0, 0);
#pragma unroll
    for (int k = 0; k < 6; ++k) a.Io[k] = 0.0;
}
JB_DI void acc_add(SubAcc& a, const SubAcc& b) {
    a.f = a.f + b.f; a.h = a.h + b.h; a.fe = a.fe + b.fe; a.mc = a.mc + b.mc;
#pragma unroll
    for (int k = 0; k < 6; ++k) a.Io[k] += b.Io[k];
}
// fields of a pool entry <-> accumulator (`stride` selects the lane: 0 = own, s = sub-lane s of the group)
JB_DI void acc_load_add(SubAcc& a, const double* p) {
    a.f.l.x += p[0 * 32]; a.f.l.y += p[1 * 32]; a.f.l.z += p[2 * 32]; a.f.a.x += p[3 * 32]; a.f.a.y += p[4 * 32]; a.f.a.z += p[5 * 32];
    a.h.l.x += p[6 * 32]; a.h.l.y += p[7 * 32]; a.h.l.z += p[8 * 32]; a.h.a.x += p[9 * 32]; a.h.a.y += p[10 * 32]; a.h.a.z += p[11 * 32];
    a.fe.l.x += p[12 * 32]; a.fe.l.y += p[13 * 32]; a.fe.l.z += p[14 * 32]; a.fe.a.x += p[15 * 32]; a.fe.a.y += p[16 * 32]; a.fe.a.z += p[17 * 32];
    a.mc.x += p[18 * 32]; a.mc.y += p[19 * 32]; a.mc.z += p[20 * 32];
#pragma unroll
    for (int k = 0; k < 6; ++k) a.Io[k] += p[(21 + k) * 32];
}
JB_DI void acc_store_add(const SubAcc& a, double* p) {
    p[0 * 32] += a.f.l.x; p[1 * 32] += a.f.l.y; p[2 * 32] += a.f.l.z; p[3 * 32] += a.f.a.x; p[4 * 32] += a.f.a.y; p[5 * 32] += a.f.a.z;
    p[6 * 32] += a.h.l.x; p[7 * 32] += a.h.l.y; p[8 * 32] += a.h.l.z; p[9 * 32] += a.h.a.x; p[10 * 32] += a.h.a.y; p[11 * 32] += a.h.a.z;
    p[12 * 32] += a.fe.l.x; p[13 * 32] += a.fe.l.y; p[14 * 32] += a.fe.l.z; p[15 * 32] += a.fe.a.x; p[16 * 32] += a.fe.a.y; p[17 * 32] += a.fe.a.z;
    p[18 * 32] += a.mc.x; p[19 * 32] += a.mc.y; p[20 * 32] += a.mc.z;
#pragma unroll
    for (int k = 0; k < 6; ++k) p[(21 + k) * 32] += a.Io[k];
}
// express a subtree accumulator of total mass m in the parent frame (li: child -> parent)
JB_DI SubAcc acc_to_parent(const Xf& li, const SubAcc& a, double m) {
    SubAcc o;
    o.f = force_act(li, a.f); o.h = force_act(li, a.h); o.fe = force_act(li, a.fe);
    const V3 rmc = rmul(li.R, a.mc);
    o.mc = rmc + m * li.p;
    // inertia about the parent origin: R Io R^T + m (|p|^2 1 - p p^T) + 2 (p . R mc) 1 - p (R mc)^T - (R mc) p^T
    double Ir[6];
    rot_sym(li.R, a.Io, Ir);
    const V3 p = li.p;
    const double pp = dot(p, p), pr = dot(p, rmc);
    o.Io[0] = Ir[0] + m * (pp - p.x * p.x) + 2.0 * pr - 2.0 * p.x * rmc.x;
    o.Io[1] = Ir[1] - m * (p.x * p.y) - (p.x * rmc.y + rmc.x * p.y);
    o.Io[2] = Ir[2] + m * (pp - p.y * p.y) + 2.0 * pr - 2.0 * p.y * rmc.y;
    o.Io[3] = Ir[3] - m * (p.x * p.z) - (p.x * rmc.z + rmc.x * p.z);
    o.Io[4] = Ir[4] - m * (p.y * p.z) - (p.y * rmc.z + rmc.y * p.z);
    o.Io[5] = Ir[5] + m * (pp - p.z * p.z) + 2.0 * pr - 2.0 * p.z * rmc.z;
    return o;
}
// where the forward pass parks h and fExt of a record until the backward pass (fields that are dead once the step is over)
__device__ constexpr int X1_H = R1_FU;                                    // 6
__device__ constexpr int X1_FE[6] = {R1_DINV, R1_U, R1_QS, R1_QS + 1, R1_VS, R1_SV};
__device__ constexpr int XF_H = RF_QS, XF_FE = RF_VS;                     // 6 + 6

__device__ __noinline__ void extra_terms(const Ctx c) {
    const int L = KP->L;
    const JbOptions& opt = KP->opt;
    const size_t col = c.env;
    const bool cen = KP->extra_ycrb != nullptr;
    double kin = 0.0, pot = 0.0;
    // ---- forward: v, a (from a[0] = 0), a_gf (from -g), f_i = v x* (I v) + I a_gf - fext, h_i = I v, fExt_i = I a + v x* h
    {
        Xf oMc; Mot vc = mzero(), ac = mzero(), agc = mzero();
#pragma unroll
        for (int k = 0; k < 9; ++k) oMc.R[k] = 0.0;
        oMc.p = mk(0, 0, 0);
#pragma unroll 1
        for (int r = 0; r < KP->nrec; ++r) {
            const RecInt* ri = KP->rint + (r * L + c.sub);
            const int kind = ri->kind;
            if (kind == REC_PAD) continue;
            const RecDbl* rd = JB_RDBL + (r * L + c.sub);
            const int base = KP->rec_off[r];
            double* const rp = jb_smem + base * 32 + c.lane;
            if (ri->parent_rec < 0) {
#pragma unroll
                for (int k = 0; k < 9; ++k) oMc.R[k] = (k % 4 == 0) ? 1.0 : 0.0;
                oMc.p = mk(0, 0, 0); vc = mzero(); ac = mzero();
                agc.l = mk(-opt.gravity[0], -opt.gravity[1], -opt.gravity[2]);
                agc.a = mk(-opt.gravity[3], -opt.gravity[4], -opt.gravity[5]);
            } else if (!ri->carry_in) {
                const int po = KP->pool_off + POOL_SIZE * ri->parent_pool;
                sm_load_xf(c, po, oMc);
                vc = sm_load_mot(c, po + 12);
                ac = sm_load_mot(c, po + 18);
                agc.l = mk(jb_smem[(po + 24) * 32 + c.lane], jb_smem[(po + 25) * 32 + c.lane], jb_smem[(po + 26) * 32 + c.lane]);
                agc.a = ac.a;   // a and a_gf differ by a pure linear acceleration (gravity), angular parts coincide
            }
            Xf li; Mot vJ = mzero(), sdd = mzero();
            const V3 ax = ld3(rd->axis);
            if (rec_is_big(kind)) {
                sm_load_xf(c, base + RF_LIMI, li);
                vJ = sm_load_mot(c, base + RF_V);
                sdd = sm_load_mot(c, base + RF_A);
            } else {
                sm_load_xf(c, base + R1_LIMI, li);
                const double qd = RP(R1_V), ddq = RP(R1_A);
                if (kind == REC_PRISM) { vJ.l = qd * ax; sdd.l = ddq * ax; }
                else { vJ.a = qd * ax; sdd.a = ddq * ax; }
            }
            Xf oM;
            mat3mul(oMc.R, li.R, oM.R);
            oM.p = oMc.p + rmul(oMc.R, li.p);
            const Mot v = motion_act_inv(li, vc) + vJ;
            const Mot bias = motion_cross(v, vJ) + sdd;          // ForwardKinematicsAccelerationStep (engine.cc:776-791)
            const Mot a = bias + motion_act_inv(li, ac);
            const Mot ag = bias + motion_act_inv(li, agc);
            const double mass = rd->inertia[0];
            const V3 lever = ld3(rd->inertia + 1);
            const Mot h = inertia_mul(mass, lever, rd->inertia + 4, v);
            const Mot vxh = motion_cross_force(v, h);
            Mot f = vxh + inertia_mul(mass, lever, rd->inertia + 4, ag);
            Mot fext = mzero();
            for (int k = 0; k < ri->ncontact; ++k) {
                const int cs = ri->contact0 + k;
                const ContactSlot* ct = KP->cslots + (cs * L + c.sub);
                const double* const cp = jb_smem + (KP->cslot_off + CSLOT_SIZE * cs) * 32 + c.lane;
                const V3 Fl = mk(CO(0), CO(1), CO(2));
                fext.l = fext.l + Fl; fext.a = fext.a + cross(ld3(ct->placement + 9), Fl) + mk(CO(3), CO(4), CO(5));
            }
            add_cached_ext_wrench(c, r, L, fext);
            f = f - fext;
            sm_store_mot(c, base + (rec_is_big(kind) ? RF_F : R1_BIAS), f);
            if (cen) {
                const Mot fe = vxh + inertia_mul(mass, lever, rd->inertia + 4, a);
                if (rec_is_big(kind)) { sm_store_mot(c, base + XF_H, h); sm_store_mot(c, base + XF_FE, fe); }
                else {
                    sm_store_mot(c, base + X1_H, h);
                    RP(X1_FE[0]) = fe.l.x; RP(X1_FE[1]) = fe.l.y; RP(X1_FE[2]) = fe.l.z;
                    RP(X1_FE[3]) = fe.a.x; RP(X1_FE[4]) = fe.a.y; RP(X1_FE[5]) = fe.a.z;
                }
            }
            if (ri->owner) {
                kin += 0.5 * (dot(v.l, h.l) + dot(v.a, h.a));
                if (kind == REC_SPH) kin += 0.5 * (ax.x * vJ.a.x * vJ.a.x + ax.y * vJ.a.y * vJ.a.y + ax.z * vJ.a.z * vJ.a.z);   // rotor term, `ax` = the three rotor inertias
                else if (kind != REC_FREE) { const double qd = RP(R1_V); kin += 0.5 * rd->armature * qd * qd; }   // rotor term
                const V3 com = oM.p + rmul(oM.R, lever);
                pot -= mass * (opt.gravity[0] * com.x + opt.gravity[1] * com.y + opt.gravity[2] * com.z);
                if (c.valid && KP->extra_a) {
                    double* o = KP->extra_a + (col * KP->njoints + ri->joint) * 6;
                    o[0] = a.l.x; o[1] = a.l.y; o[2] = a.l.z; o[3] = a.a.x; o[4] = a.a.y; o[5] = a.a.z;
                }
            }
            if (ri->pool >= 0) {
                const int po = KP->pool_off + POOL_SIZE * ri->pool;
                sm_store_xf(c, po, oM);
                sm_store_mot(c, po + 12, v);
                sm_store_mot(c, po + 18, a);
                jb_smem[(po + 24) * 32 + c.lane] = ag.l.x; jb_smem[(po + 25) * 32 + c.lane] = ag.l.y; jb_smem[(po + 26) * 32 + c.lane] = ag.l.z;
            }
            oMc = oM; vc = v; ac = a; agc = ag;
        }
    }
    jb_syncwarp(c);
    // ---- backward: data.f[parent] += liMi.act(data.f[i]) for parent > 0; h, fExt and the subtree inertias up to the universe
    Mot h0 = mzero(), fe0 = mzero();   // this lane's contribution to h[0], fExt[0]
    V3 com0 = mk(0, 0, 0);             // data.com[0] = liMi[1].act(com[1])
    {
        for (int k = 0; k < POOL_SIZE * KP->npool; ++k) SMF(c, KP->pool_off + k) = 0.0;
        SubAcc carry;
        acc_zero(carry);
#pragma unroll 1
        for (int r = KP->nrec - 1; r >= 0; --r) {
            const RecInt* ri = KP->rint + (r * L + c.sub);
            const int kind = ri->kind;
            const bool reduce = (r < KP->ntrunk) && KP->trunk_reduce[r] && L > 1;
            if (reduce) jb_syncwarp(c);
            if (kind == REC_PAD) continue;
            const RecDbl* rd = JB_RDBL + (r * L + c.sub);
            const int base = KP->rec_off[r];
            double* const rp = jb_smem + base * 32 + c.lane;
            SubAcc A;
            acc_zero(A);
            A.f = sm_load_mot(c, base + (rec_is_big(kind) ? RF_F : R1_BIAS));
            if (cen) {
                if (rec_is_big(kind)) { A.h = sm_load_mot(c, base + XF_H); A.fe = sm_load_mot(c, base + XF_FE); }
                else {
                    A.h = sm_load_mot(c, base + X1_H);
                    A.fe.l = mk(RP(X1_FE[0]), RP(X1_FE[1]), RP(X1_FE[2])); A.fe.a = mk(RP(X1_FE[3]), RP(X1_FE[4]), RP(X1_FE[5]));
                }
                // the body itself: m c and its inertia about the joint origin (the D block of InertiaTpl::matrix())
                const double m = rd->inertia[0];
                const V3 lc = ld3(rd->inertia + 1);
                SymY Y;
                inertia_to_sym(m, lc, rd->inertia + 4, Y);
                A.mc = m * lc;
#pragma unroll
                for (int k = 0; k < 6; ++k) A.Io[k] = Y.D[k];
            }
            if (ri->take_carry) acc_add(A, carry);
            if (ri->pool >= 0) {
                const int po = KP->pool_off + POOL_SIZE * ri->pool;
                if (reduce) {
                    const double* const p0 = jb_smem + po * 32 + (c.lane - c.sub);
                    for (int s = 0; s < L; ++s) acc_load_add(A, p0 + s);
                } else acc_load_add(A, jb_smem + po * 32 + c.lane);
            }
            const double msub = rd->subtree_mass;
            if (ri->owner && c.valid) {
                if (KP->extra_f) {
                    double* o = KP->extra_f + (col * KP->njoints + ri->joint) * 6;
                    o[0] = A.f.l.x; o[1] = A.f.l.y; o[2] = A.f.l.z; o[3] = A.f.a.x; o[4] = A.f.a.y; o[5] = A.f.a.z;
                }
                if (cen) {
                    // Ycrb[j] = (m, c, I about the subtree CoM); com[j] = c; vcom[j] = h[j].linear / mass[j]
                    // (a massless subtree: InertiaTpl::__pequ__ divides by max(mass, eps), its centre of mass is the origin, not 0 / 0)
                    const double md = fmax(msub, D_EPS);
                    const V3 cc = mk(A.mc.x / md, A.mc.y / md, A.mc.z / md);
                    const double c2 = dot(cc, cc);
                    double* y = KP->extra_ycrb + (col * KP->njoints + ri->joint) * 10;
                    y[0] = msub; y[1] = cc.x; y[2] = cc.y; y[3] = cc.z;
                    y[4] = A.Io[0] - msub * (c2 - cc.x * cc.x); y[5] = A.Io[1] + msub * (cc.x * cc.y);
                    y[6] = A.Io[2] - msub * (c2 - cc.y * cc.y); y[7] = A.Io[3] + msub * (cc.x * cc.z);
                    y[8] = A.Io[4] + msub * (cc.y * cc.z);      y[9] = A.Io[5] - msub * (c2 - cc.z * cc.z);
                    double* o = KP->extra_com + (col * KP->njoints + ri->joint) * 3;
                    o[0] = cc.x; o[1] = cc.y; o[2] = cc.z;
                    double* w = KP->extra_vcom + (col * KP->njoints + ri->joint) * 3;
                    w[0] = A.h.l.x / msub; w[1] = A.h.l.y / msub; w[2] = A.h.l.z / msub;
                }
            }
            Xf li; sm_load_xf(c, base + R1_LIMI, li);   // (RF_LIMI == R1_LIMI == 0)
            if (ri->parent_rec >= 0) {
                carry = acc_to_parent(li, A, msub);
                if (!ri->carry_out) {
                    const bool add = (r >= KP->ntrunk) || (c.sub == 0);
                    if (add) acc_store_add(carry, jb_smem + (KP->pool_off + POOL_SIZE * ri->parent_pool) * 32 + c.lane);
                }
            } else if (cen && ri->owner) {
                // child of the universe
                h0 = h0 + force_act(li, A.h); fe0 = fe0 + force_act(li, A.fe);
                if (ri->joint == 1) {
                    // (a massless subtree: InertiaTpl::__pequ__ divides by max(mass, eps), its centre of mass is the origin, not 0 / 0)
                    const double md = fmax(msub, D_EPS);
                    const V3 cc = mk(A.mc.x / md, A.mc.y / md, A.mc.z / md);
                    com0 = li.p + rmul(li.R, cc);
                }
            }
        }
    }
    jb_syncwarp(c);
    kin = group_sum(kin, c, L);
    pot = group_sum(pot, c, L);
    if (c.valid && c.sub == 0 && KP->extra_energy) { KP->extra_energy[2 * col] = kin; KP->extra_energy[2 * col + 1] = pot; }
    if (cen) {
        // universe row: h[0], fExt[0] summed over the lanes' root joints; hg / dhg about the centre of mass
        h0.l.x = group_sum(h0.l.x, c, L); h0.l.y = group_sum(h0.l.y, c, L); h0.l.z = group_sum(h0.l.z, c, L);
        h0.a.x = group_sum(h0.a.x, c, L); h0.a.y = group_sum(h0.a.y, c, L); h0.a.z = group_sum(h0.a.z, c, L);
        fe0.l.x = group_sum(fe0.l.x, c, L); fe0.l.y = group_sum(fe0.l.y, c, L); fe0.l.z = group_sum(fe0.l.z, c, L);
        fe0.a.x = group_sum(fe0.a.x, c, L); fe0.a.y = group_sum(fe0.a.y, c, L); fe0.a.z = group_sum(fe0.a.z, c, L);
        com0.x = group_sum(com0.x, c, L); com0.y = group_sum(com0.y, c, L); com0.z = group_sum(com0.z, c, L);
        if (c.valid && c.sub == 0) {
            double* o = KP->extra_com + col * KP->njoints * 3;
            o[0] = com0.x; o[1] = com0.y; o[2] = com0.z;
            double* w = KP->extra_vcom + col * KP->njoints * 3;
            const double mtot = KP->block_mass != nullptr ? KP->block_mass[blockIdx.x] : KP->total_mass;
            w[0] = h0.l.x / mtot; w[1] = h0.l.y / mtot; w[2] = h0.l.z / mtot;
            double* y = KP->extra_ycrb + col * KP->njoints * 10;
#pragma unroll
            for (int k = 0; k < 10; ++k) y[k] = 0.0;
            const V3 hga = h0.a + cross(h0.l, com0), dha = fe0.a + cross(fe0.l, com0);
            double* g = KP->extra_hg + col * 12;
            g[0] = h0.l.x; g[1] = h0.l.y; g[2] = h0.l.z; g[3] = hga.x; g[4] = hga.y; g[5] = hga.z;
            g[6] = fe0.l.x; g[7] = fe0.l.y; g[8] = fe0.l.z; g[9] = dha.x; g[10] = dha.y; g[11] = dha.z;
        }
    }
}

// ------------------------------------------------------------------------------------------
// Sensor measurement pipeline: what every jiminy sensor applies on top of the true value its set() wrote
//   AbstractSensorTpl<T>::setAll ............ core/include/jiminy/core/hardware/abstract_sensor.hxx:445-522 (ring of past true values)
//   AbstractSensorTpl<T>::interpolateData ... :305-430 (delay + uniform jitter, zero-order hold or linear interpolation)
//   AbstractSensorBase::measureData ......... core/src/hardware/abstract_sensor.cc:71-85 (white noise, then bias)
// with the reference's generators: PCG32 (core/src/utilities/random.cc:10-37), std::generate_canonical<float> uniforms and
// the float ziggurat normal sampler (random.cc:100-166), one generator per sensor.  Per env: one circular buffer of true
// observation rows shared by the five sensor types, each type keeping its own sample count (its own delayMax decides when
// the oldest sample is dropped, and the bisection below depends on that count exactly like the reference's does).
// ------------------------------------------------------------------------------------------
JB_DI uint32_t pcg32_next(unsigned long long& state) {
    state *= 6364136223846793005ULL;
    unsigned long long s = state;
    const unsigned rshift = static_cast<unsigned>(s >> 61) & 7u;
    s ^= s >> 22;
    return static_cast<uint32_t>(s >> (22 + rshift));
}
JB_DI float rng_uniform01(unsigned long long& st) {   // std::generate_canonical<float, 24> over a 32-bit generator (libstdc++)
#ifdef JB_HOST_EMUL
    float r = static_cast<float>(pcg32_next(st)) / 4294967296.0f;
#else
    float r = __uint2float_rn(pcg32_next(st)) / 4294967296.0f;
#endif
    return r >= 1.0f ? 0.99999994f : r;
}
JB_DI float rng_logf(float x) { return static_cast<float>(log(static_cast<double>(x))); }
JB_DI float rng_expf(float x) { return static_cast<float>(exp(static_cast<double>(x))); }
JB_DI float rng_normal(unsigned long long& st) {      // internal::normal (random.cc:108-160)
    const float r = 3.442620F;
    int32_t hz = static_cast<int32_t>(pcg32_next(st));
    uint32_t iz = static_cast<uint32_t>(hz) & 127u;
    if (fabs(static_cast<double>(hz)) < static_cast<double>(KP->zig_kn[iz])) return static_cast<float>(hz) * KP->zig_wn[iz];
    while (true) {
        float x, y;
        if (iz == 0) {
            while (true) {
                x = -0.2904764F * rng_logf(rng_uniform01(st));
                y = -rng_logf(rng_uniform01(st));
                if (x * x <= y + y) break;
            }
            return hz <= 0 ? -r - x : r + x;
        }
        x = static_cast<float>(hz) * KP->zig_wn[iz];
        if (KP->zig_fn[iz] + rng_uniform01(st) * (KP->zig_fn[iz - 1] - KP->zig_fn[iz]) < rng_expf(-0.5F * x * x)) return x;
        hz = static_cast<int32_t>(pcg32_next(st));
        iz = static_cast<uint32_t>(hz) & 127u;
        if (fabs(static_cast<double>(hz)) < static_cast<double>(KP->zig_kn[iz])) return static_cast<float>(hz) * KP->zig_wn[iz];
    }
}
// setAll's buffer management for every sensor type of this env at time t (one lane of the env calls it): returns the
// physical slot the true values of this refresh go to
JB_DI int sensor_ring_push(int env, double t) {
    const int cap = KP->sp_cap;
    int32_t* cnt = KP->sp_count + static_cast<size_t>(env) * 6;
    double* tm = KP->sp_times + static_cast<size_t>(env) * cap;
    const int head = (cnt[0] + 1) % cap;
    for (int ty = 0; ty < 5; ++ty) {
        const int n = cnt[1 + ty];
        const double front = tm[((head - 1 - (n - 1)) % cap + cap) % cap];      // oldest sample this type still holds
        const double timeMin = t - KP->sp_delay_max[ty] - 0.02;                 // SIMULATION_MAX_TIMESTEP
        // rotate (drop the oldest) or grow; a full buffer always drops (older than anything a lookup can reach)
        if (!(timeMin > front) && n < cap) cnt[1 + ty] = n + 1;
    }
    cnt[0] = head;
    tm[head] = t;
    return head;
}
// interpolateData + measureData of sensor `s` of this env: reads the ring, writes the sensor's fields of the measurement row
JB_DI void measure_sensor(int env, int s) {
    const SensorDesc* d = KP->sp_desc + s;
    const int cap = KP->sp_cap, width = KP->lay.width;
    const int32_t* cnt = KP->sp_count + static_cast<size_t>(env) * 6;
    const double* tm = KP->sp_times + static_cast<size_t>(env) * cap;
    const double* ring = KP->sp_ring + static_cast<size_t>(env) * cap * width;
    double* out = KP->sensors + static_cast<size_t>(env) * width;
    const int head = cnt[0], n = cnt[1 + d->type];
    unsigned long long st = KP->sp_rng[static_cast<size_t>(env) * KP->sp_nsens + s];
    auto phys = [&](int i) { return ((head - (n - 1) + i) % cap + cap) % cap; };   // logical index (0 = oldest of this type) -> slot
    const float jit = static_cast<float>(d->jitter);
    const double delay = d->delay + static_cast<double>((jit - 0.0f) * rng_uniform01(st) + 0.0f);
    double timeDesired = tm[head] - delay;
    if (d->order == 0) timeDesired += STEPPER_MIN_TIMESTEP;
    int idxLeft;
    if (timeDesired >= tm[head]) idxLeft = n - 1;
    else if (timeDesired < tm[phys(0)]) idxLeft = -1;
    else {
        int left = 0, right = n - 1, mid = 0;
        idxLeft = -2;
        while (left < right) {
            mid = (left + right) / 2;
            const double tmid = tm[phys(mid)];
            if (timeDesired < tmid) right = mid;
            else if (timeDesired > tmid) left = mid + 1;
            else { idxLeft = mid; break; }
        }
        if (idxLeft == -2) idxLeft = timeDesired < tm[phys(mid)] ? mid - 1 : mid;
    }
    int mode = 2, i0 = n - 1, i1 = n - 1;     // 0: hold i0, 1: interpolate i0 -> i1, 2: most recent
    double ratio = 0.0;
    if (timeDesired >= 0.0 && idxLeft + 1 < n) {
        i0 = idxLeft < 0 ? 0 : idxLeft;        // (idxLeft < 0: "No data old enough" in the reference; the buffer is sized so that it cannot happen)
        if (d->order == 0) mode = 0;
        else { mode = 1; i1 = i0 + 1; ratio = (timeDesired - tm[phys(i0)]) / (tm[phys(i1)] - tm[phys(i0)]); }
    } else if (d->delay > D_EPS || d->jitter > D_EPS) {
        // the buffer is not old enough yet: the oldest value that is not the initial zero sample
        i0 = n - 1;
        for (int i = 0; i < n; ++i) if (tm[phys(i)] > 0.0) { i0 = i - 1 < 0 ? 0 : i - 1; break; }
        mode = 0;
    }
    const double* r0 = ring + static_cast<size_t>(phys(i0)) * width + d->offset + d->index;
    const double* r1 = ring + static_cast<size_t>(phys(i1)) * width + d->offset + d->index;
    for (int f = 0; f < d->nf; ++f) {
        const double a = r0[f * d->ns];
        double val = mode == 1 ? a + ratio * (r1[f * d->ns] - a) : a;
        if (d->has_noise) val += static_cast<double>(rng_normal(st) * static_cast<float>(d->noise_std[f]) + 0.0F);
        out[d->offset + f * d->ns + d->index] = val;
    }
    if (d->has_bias)
        for (int f = 0; f < d->nf; ++f) out[d->offset + f * d->ns + d->index] += d->bias[f];
    KP->sp_rng[static_cast<size_t>(env) * KP->sp_nsens + s] = st;
}

// ------------------------------------------------------------------------------------------
// Sensors: <Sensor>::set() of IMU / Force / Encoder / Effort / Contact
// (core/src/hardware/basic_sensors.cc:142-164, :267, :368-386, :509-537, :604).  Every value is
// written by exactly one lane straight into the env's row of the AoS observation matrix.
// ------------------------------------------------------------------------------------------
// mahony_filter (blocks/mahony_filter.py:28-101): one iteration of the observer of one IMU, `ms` = its 10-double state
JB_DI void mahony_update(double* ms, V3 gyro, V3 acc) {
    const double q_x = ms[0], q_y = ms[1], q_z = ms[2], q_w = ms[3];
    const double v_x = 2 * (q_x * q_z - q_y * q_w), v_y = 2 * (q_y * q_z + q_w * q_x), v_z = 1 - 2 * (q_x * q_x + q_y * q_y);
    const V3 om = mk(gyro.x - ms[4], gyro.y - ms[5], gyro.z - ms[6]);
    const double ax = acc.x / 9.81, ay = acc.y / 9.81, az = acc.z / 9.81;
    const V3 omes = mk(ay * v_z - az * v_y, az * v_x - ax * v_z, ax * v_y - ay * v_x);
    const V3 cf = om + KP->mahony_kp * omes;
    ms[7] = om.x; ms[8] = om.y; ms[9] = om.z;
    if (!(fabs(cf.x) < 1e-6 && fabs(cf.y) < 1e-6 && fabs(cf.z) < 1e-6)) {
        const double dt = KP->opt.sensors_update_period;
        double theta = sqrt(cf.x * cf.x + cf.y * cf.y + cf.z * cf.z);
        const double a_x = cf.x / theta, a_y = cf.y / theta, a_z = cf.z / theta;
        theta *= dt / 2;
        double sn, p_w;
        sincos(theta, &sn, &p_w);
        const double p_x = a_x * sn, p_y = a_y * sn, p_z = a_z * sn;
        const double n_x = q_x * p_w + q_w * p_x - q_z * p_y + q_y * p_z;
        const double n_y = q_y * p_w + q_z * p_x + q_w * p_y - q_x * p_z;
        const double n_z = q_z * p_w - q_y * p_x + q_x * p_y + q_w * p_z;
        const double n_w = q_w * p_w - q_x * p_x - q_y * p_y - q_z * p_z;
        const double scale = (3.0 - (n_x * n_x + n_y * n_y + n_z * n_z + n_w * n_w)) / 2;
        ms[0] = n_x * scale; ms[1] = n_y * scale; ms[2] = n_z * scale; ms[3] = n_w * scale;
        ms[4] -= KP->mahony_ki * dt * omes.x; ms[5] -= KP->mahony_ki * dt * omes.y; ms[6] -= KP->mahony_ki * dt * omes.z;
    }
}

__device__ __noinline__ void write_sensors(const Ctx c, const bool at_start, const double t) {
    if (!c.valid) return;
    const int L = KP->L;
    const JbSensorLayout& lay = KP->lay;
    double* row = KP->sensors + static_cast<size_t>(c.env) * lay.width;
    if (KP->sp_on) {
        // measurement pipeline: the true values go to a new slot of the env's ring, the public row receives the measurements
        if (c.sub == 0) {
            if (at_start) {
                // resetAll (abstract_sensor.hxx:199-232): one zero sample at t = 0, fresh generators
                int32_t* cnt = KP->sp_count + static_cast<size_t>(c.env) * 6;
                cnt[0] = 0;
                for (int ty = 0; ty < 5; ++ty) cnt[1 + ty] = 1;
                KP->sp_times[static_cast<size_t>(c.env) * KP->sp_cap] = 0.0;
                double* z = KP->sp_ring + static_cast<size_t>(c.env) * KP->sp_cap * lay.width;
                for (int k = 0; k < lay.width; ++k) z[k] = 0.0;
                for (int k = 0; k < KP->sp_nsens; ++k)
                    KP->sp_rng[static_cast<size_t>(c.env) * KP->sp_nsens + k] = KP->sp_rng_init[static_cast<size_t>(c.env) * KP->sp_nsens + k];
            }
            sensor_ring_push(c.env, t);
        }
        jb_syncwarp(c);
        const int slot = KP->sp_count[static_cast<size_t>(c.env) * 6];
        row = KP->sp_ring + (static_cast<size_t>(c.env) * KP->sp_cap + slot) * lay.width;
    }
    for (int r = 0; r < KP->nrec; ++r) {
        const RecInt* ri = KP->rint + (r * L + c.sub);
        if (ri->kind == REC_PAD || !ri->owner) continue;
        const RecDbl* rd = JB_RDBL + (r * L + c.sub);
        const int base = KP->rec_off[r];
        double* const rp = jb_smem + base * 32 + c.lane;
        if (ri->imu >= 0) {
            // gyro = P.actInv(v).angular ; accel = classical frame acceleration - R^T g.  With a_gf
            // (acceleration in the gravity-free frame) the gravity term cancels analytically.
            const double* Pm = KP->imu_placement + 12 * ri->imu;
            Xf Pf;
#pragma unroll
            for (int k = 0; k < 9; ++k) Pf.R[k] = Pm[k];
            Pf.p = ld3(Pm + 9);
            const int io = KP->imu_off + IMUSLOT_SIZE * ri->imu_slot;
            const Mot vf = motion_act_inv(Pf, sm_load_mot(c, io));
            const Mot af = motion_act_inv(Pf, sm_load_mot(c, io + 6));
            const V3 acc = af.l + cross(vf.a, vf.l);
            const int n = KP->nimu, k = ri->imu;
            row[lay.imu_offset + 0 * n + k] = vf.a.x; row[lay.imu_offset + 1 * n + k] = vf.a.y; row[lay.imu_offset + 2 * n + k] = vf.a.z;
            row[lay.imu_offset + 3 * n + k] = acc.x;  row[lay.imu_offset + 4 * n + k] = acc.y;  row[lay.imu_offset + 5 * n + k] = acc.z;
            if (KP->mahony != nullptr) {
                // MahonyFilter observer: one IMU per env is what the early return of the reference looks at
                double* ms = KP->mahony + (static_cast<size_t>(c.env) * n + k) * 10;
                if (at_start) {
                    // exact_init: true orientation of the IMU frame = product of liMi up the tree, times the frame placement
                    double Rw[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
                    for (int rr = r; rr >= 0; rr = (KP->rint + (rr * L + c.sub))->parent_rec) {
                        Xf lj; sm_load_xf(c, KP->rec_off[rr], lj);
                        double T[9];
                        mat3mul(lj.R, Rw, T);
#pragma unroll
                        for (int e = 0; e < 9; ++e) Rw[e] = T[e];
                    }
                    double R[9];
                    mat3mul(Rw, Pf.R, R);
                    // matrices_to_quat (utils/math.py:307-350)
                    double t, o4[4];
                    if (R[8] < 0) {
                        if (R[0] > R[4]) { t = 1 + R[0] - R[4] - R[8]; o4[0] = t; o4[1] = R[3] + R[1]; o4[2] = R[2] + R[6]; o4[3] = R[7] - R[5]; }
                        else { t = 1 - R[0] + R[4] - R[8]; o4[0] = R[3] + R[1]; o4[1] = t; o4[2] = R[7] + R[5]; o4[3] = R[2] - R[6]; }
                    } else {
                        if (R[0] < -R[4]) { t = 1 - R[0] - R[4] + R[8]; o4[0] = R[2] + R[6]; o4[1] = R[7] + R[5]; o4[2] = t; o4[3] = R[3] - R[1]; }
                        else { t = 1 + R[0] + R[4] + R[8]; o4[0] = R[7] - R[5]; o4[1] = R[2] - R[6]; o4[2] = R[3] - R[1]; o4[3] = t; }
                    }
                    const double d = 2 * sqrt(t);
#pragma unroll
                    for (int e = 0; e < 4; ++e) ms[e] = o4[e] / d;
#pragma unroll
                    for (int e = 4; e < 10; ++e) ms[e] = 0.0;
                } else if (!KP->sp_on) mahony_update(ms, vf.a, acc);   // (with the measurement pipeline: after it, on the measured values)
            }
        }
        if (ri->encoder >= 0) {
            double pos;
            if (ri->kind == REC_REVU) pos = atan2(RP(R1_Q + 1), RP(R1_Q));
            else pos = RP(R1_Q);
            row[lay.encoder_offset + ri->encoder] = pos * rd->enc_reduction;
            row[lay.encoder_offset + KP->nenc + ri->encoder] = RP(R1_V) * rd->enc_reduction;
        }
        if (ri->effort >= 0) row[lay.effort_offset + ri->effort] = RP(R1_UMOTOR);
        if (ri->ncontact > 0) {
            Mot fs = mzero();
            int fsensor = -1;
            for (int k = 0; k < ri->ncontact; ++k) {
                const int cs = ri->contact0 + k;
                const ContactSlot* ct = KP->cslots + (cs * L + c.sub);
                const int co = KP->cslot_off + CSLOT_SIZE * cs;
                double* const cp = jb_smem + co * 32 + c.lane;
                const V3 Fl = mk(CO(0), CO(1), CO(2));
                // robot->contactForces_[i] = placement.actInv(fextLocal): torque vanishes at the contact point
                const V3 fc = rtmul(ct->placement, Fl);
                const V3 tc = rtmul(ct->placement, mk(CO(3), CO(4), CO(5)));   // non-zero with torsional friction only
                if (ct->sensor >= 0) {
                    row[lay.contact_offset + 0 * KP->ncs + ct->sensor] = fc.x;
                    row[lay.contact_offset + 1 * KP->ncs + ct->sensor] = fc.y;
                    row[lay.contact_offset + 2 * KP->ncs + ct->sensor] = fc.z;
                }
                if (ct->force >= 0) {
                    fsensor = ct->force;
                    const V3 fl = rmul(ct->force_R, fc);
                    fs.l = fs.l + fl;
                    fs.a = fs.a + cross(ld3(ct->force_p), fl) + rmul(ct->force_R, tc);
                }
            }
            if (fsensor >= 0) {
                const int n = KP->nforce;
                row[lay.force_offset + 0 * n + fsensor] = fs.l.x; row[lay.force_offset + 1 * n + fsensor] = fs.l.y; row[lay.force_offset + 2 * n + fsensor] = fs.l.z;
                row[lay.force_offset + 3 * n + fsensor] = fs.a.x; row[lay.force_offset + 4 * n + fsensor] = fs.a.y; row[lay.force_offset + 5 * n + fsensor] = fs.a.z;
            }
        }
    }
    if (KP->sp_on) {
        // Engine::start refreshes the sensors once per INIT iteration plus once at the end (engine.cc:1441, :1479): five
        // samples at t = 0 on top of the initial zero one, and five rounds of draws from every generator
        const int reps = at_start ? 5 : 1;
        for (int rep = 0; rep < reps; ++rep) {
            jb_syncwarp(c);              // the true values of this refresh are complete
            if (rep > 0) {
                const double* prev = row;
                if (c.sub == 0) sensor_ring_push(c.env, t);
                jb_syncwarp(c);
                row = KP->sp_ring + (static_cast<size_t>(c.env) * KP->sp_cap + KP->sp_count[static_cast<size_t>(c.env) * 6]) * lay.width;
                for (int k = c.sub; k < lay.width; k += L) row[k] = prev[k];
                jb_syncwarp(c);
            }
            for (int s = c.sub; s < KP->sp_nsens; s += L) measure_sensor(c.env, s);
        }
        jb_syncwarp(c);
        // MahonyFilter observer on the MEASURED gyroscope / accelerometer data
        if (KP->mahony != nullptr && !at_start && c.sub == 0) {
            const double* mrow = KP->sensors + static_cast<size_t>(c.env) * lay.width;
            const int n = KP->nimu;
            for (int k = 0; k < n; ++k)
                mahony_update(KP->mahony + (static_cast<size_t>(c.env) * n + k) * 10,
                              mk(mrow[lay.imu_offset + 0 * n + k], mrow[lay.imu_offset + 1 * n + k], mrow[lay.imu_offset + 2 * n + k]),
                              mk(mrow[lay.imu_offset + 3 * n + k], mrow[lay.imu_offset + 4 * n + k], mrow[lay.imu_offset + 5 * n + k]));
        }
    }
}

}  // namespace jb
