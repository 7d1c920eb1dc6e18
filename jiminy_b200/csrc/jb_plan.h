// Lane plan: how one robot's kinematic tree is laid over the L lanes of a warp that cooperate on
// one environment, and how each lane's working set is laid out in shared memory.
//
// Design (DESIGN.md "Kernel mapping"):
//  * A warp holds 32/L environments; the L lanes of an env split the tree by *branch*: joints
//    whose subtree is spread over several lanes form the TRUNK (processed redundantly by all L
//    lanes, bit-identical on each), every other joint is PRIVATE to exactly one lane.
//  * Each lane walks the same list of `nrec` records (trunk records first, then its private
//    records, padded with inactive records), so control flow is warp-uniform; only the data
//    (which joint, its constants) differs per lane.
//  * Forward sweeps carry (oMi, v, a_gf) of the previous record in registers when it is the
//    parent, otherwise read them from the parent's POOL entry; the backward sweep carries the
//    articulated inertia the same way and uses pool entries as accumulators.  Trunk joints
//    all-reduce their accumulators over the L lanes with shuffles before use.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/jiminy_b200.h"

namespace jb {

// Record kinds (what the lane executes for this record)
enum : int32_t { REC_PAD = 0, REC_REV = 1, REC_REVU = 2, REC_PRISM = 3, REC_FREE = 4,
                 REC_REVX = 5 /* bounded revolute about +-x of the joint frame */,
                 REC_SPH = 6 /* spherical (flexibility) joint: lives in a free-flyer-sized record, see RS_* */ };
// records with the free-flyer layout (RF_*)
#if defined(__CUDACC__)
__host__ __device__
#endif
constexpr bool rec_is_big(int kind) { return kind == REC_FREE || kind == REC_SPH; }

constexpr int MAX_CONTACTS_PER_REC = 8;

// Integer table, one row per (record r, sub-lane s): rows[(r * L + s)]
struct RecInt {
    int32_t kind;        // REC_*
    int32_t joint;       // model joint index, -1 for padding
    int32_t parent_rec;  // record index of the parent joint in this lane's list, -1 = universe
    int32_t carry_in;    // 1: parent is the previous record -> forward carries are valid
    int32_t pool;        // pool entry index of THIS joint (its children read / accumulate there), -1 none
    int32_t parent_pool; // pool entry index of the parent (used when !carry_in / !carry_out), -1 none
    int32_t carry_out;   // 1: backward contribution goes to the carry (parent == previous record), else parent_pool
    int32_t take_carry;  // 1: backward sweep of this record consumes the carry produced by record r+1
    int32_t idx_q, idx_v;
    int32_t motor;       // motor index or -1
    int32_t motor_flags;
    int32_t ncontact;    // number of contact frames attached to this joint
    int32_t contact0;    // first index in the per-lane contact slot list
    int32_t imu;         // imu sensor index or -1 (first one attached to this joint)
    int32_t owner;       // 1: this lane writes this joint's outputs (private: always; trunk: sub-lane 0)
    int32_t has_limit;   // 1: bounded 1-dof joint
    int32_t encoder;     // encoder sensor index or -1
    int32_t effort;      // effort sensor index or -1
    int32_t imu_slot;    // per-lane IMU capture slot or -1
};
constexpr int REC_INT_STRIDE = sizeof(RecInt) / sizeof(int32_t);

// Double table, one row per (record, sub-lane)
struct RecDbl {
    double placement[12];  // R row-major, p
    double axis[3];
    double inertia[10];    // mass, lever, I (xx xy yy xz yz zz)
    double armature;
    double q_lo, q_hi;
    double motor[10];      // SimpleMotor params (see jiminy_b200.h)
    double enc_reduction;
    double pad;            // velocity taper threshold of the motor (velocityLimit - effortLimit * velocityEffortInvSlope, >= 0)
    double subtree_mass;   // mass of the subtree rooted at this joint (pinocchio `data.mass[j]`, model.cc:269)
    double pad2;           // keeps rows 16-byte aligned
};
static_assert(sizeof(RecDbl) % 16 == 0, "RecDbl rows are read with 16-byte loads");
constexpr int REC_DBL_STRIDE = sizeof(RecDbl) / sizeof(double);

struct ContactSlot {  // per lane contact slot (rows[(c * L + s)])
    double placement[12];
    int32_t contact;     // contact frame index (-1 pad)
    int32_t sensor;      // contact sensor index or -1
    int32_t force;       // force sensor index or -1
    int32_t pad;
    double force_R[9];   // relative placement contact -> force sensor frame (ForceSensor::refreshProxies)
    double force_p[3];
};

// External-force slot (Engine::registerImpulseForce / registerProfileForce): one per distinct frame
// (parent joint, translation in the joint frame); rows[(e * L + s)].  `rec` is the record that applies the
// slot's wrench on sub-lane s: the joint's record on its owning lane (on every lane for a trunk joint,
// whose own bias force is replicated, not reduced), -1 elsewhere.
struct ExtSlot {
    double p[3];
    int32_t rec;
    int32_t joint;
};
// Constraint path (joint position bounds, contacts.model == "constraint"): lookup tables for the lane that
// walks the whole tree in joint order, and the layout of the per-env state / workspace in global memory.
struct JointMap {      // [njoints], index 0 (universe) unused
    int32_t rec, sub;  // where the joint's record lives (trunk joints: sub-lane 0, replicated on every lane)
    int32_t parent;    // parent joint index (0 = universe)
    int32_t idx_q, idx_v, nvj, kind;
    int32_t trunk;     // 1: replicated on all L lanes
};
struct ContactMap {    // [ncontacts]
    int32_t joint, sub, cslot, trunk;
    double placement[12];
};
// persistent constraint state, one column per env: [CS_*][n_pad]
constexpr int CS_SOLVE_FAILED = 0;       // successiveSolveFailed
constexpr int CS_JOINT0 = 1;             // per joint constraint: enabled, reversed, qRef, lambda
constexpr int CS_JOINT_SIZE = 4;
constexpr int CS_CONTACT_SIZE = 17;      // per contact constraint: enabled, lambda[4], reference R[9], p[3]

constexpr int MAX_ESLOT = 4, MAX_IMPULSE = 16, MAX_PROFILE = 4;
constexpr int MAX_PROCESS = 2;   // process forces (jb_register_process_force), each on a slot of its own
constexpr int ESLOT_SIZE = 12;   // wrench in world-aligned axes at the frame origin (6) | same wrench in the joint frame (6)
constexpr int IMPULSE_ROWS = 8;  // t, dt, wrench[6]

struct Plan {
    int L = 1;                 // lanes per env (1, 2, 4, 8)
    int nrec = 0;              // records per lane
    int ntrunk = 0;            // leading trunk records
    int npool = 0;             // pool entries per lane
    int ncslot = 0;            // contact slots per lane
    int nimuslot = 0;          // IMU capture slots per lane
    int nfields = 0;           // doubles of shared memory per lane
    std::vector<int32_t> rec_off;       // [nrec] field offset of each record (lane-uniform)
    std::vector<int32_t> rec_free;      // [nrec] 1 if the record slot is sized for a free-flyer / spherical joint
    int sph_off = 0;                    // RF_KA + 6 * n_hist: where the RS_* block of a spherical record starts
    std::vector<int32_t> trunk_reduce;  // [nrec] 1 if a trunk record all-reduces its pool accumulator
    int pool_off = 0, cslot_off = 0, imu_off = 0;
    std::vector<RecInt> rint;           // [nrec * L]
    std::vector<RecDbl> rdbl;           // [nrec * L]
    std::vector<ContactSlot> cslots;    // [ncslot * L]
    std::vector<int32_t> joint_lane;    // [njoints] owning sub-lane (-1 trunk)
    double total_mass = 0.0;            // pinocchio `data.mass[0]`
    std::string describe() const;
};

// Field offsets inside a record (doubles).  1-dof record:
constexpr int R1_LIMI = 0;    // 12: liMi (R row-major, p)
constexpr int R1_BIAS = 12;   // 6 : a_gf bias  c + v x vJ
constexpr int R1_FU = 18;     // 6 : f (pass 1 -> pass 2) then U (pass 2 -> pass 3)
constexpr int R1_DINV = 24;   // 1
constexpr int R1_U = 25;      // 1 : joint-space effort after the backward step
constexpr int R1_UMOTOR = 26; // 1
constexpr int R1_CMD = 27;    // 1
constexpr int R1_Q = 28;      // 2 : accepted q (cos, sin for unbounded)
constexpr int R1_V = 30;      // 1
constexpr int R1_A = 31;      // 1 : accepted / last computed acceleration
constexpr int R1_QS = 32;     // 2 : stage q
constexpr int R1_VS = 34;     // 1
constexpr int R1_SV = 35;     // 1 : Runge-Kutta position-increment accumulator
constexpr int R1_SA = 36;     // 1 : Runge-Kutta velocity-increment accumulator
constexpr int R1_KA = 37;     // 1-dof stage derivative history starts here (DOPRI: 7 slots, else 0)
// free-flyer record:
constexpr int RF_LIMI = 0;    // 12
constexpr int RF_F = 12;      // 6 : f (pass 1 -> pass 2)
constexpr int RF_Q = 18;      // 7
constexpr int RF_V = 25;      // 6
constexpr int RF_A = 31;      // 6
constexpr int RF_QS = 37;     // 7
constexpr int RF_VS = 44;     // 6
constexpr int RF_SV = 50;     // 6
constexpr int RF_SA = 56;     // 6
constexpr int RF_KA = 62;     // DOPRI history (7 x 6) starts here
// spherical record = free-flyer layout with the linear halves of q / v / a / stage / accumulator / history slots held at
// zero (every copy / accumulate loop of the steppers serves both kinds unchanged; only integrate, difference, the joint
// transform and the articulated-body step are its own), followed by RS_EXTRA doubles at RF_KA + 6 * n_hist:
constexpr int RS_BIAS = 0;    // 6 : a_gf bias v x vJ
constexpr int RS_U = 6;       // 18: U = Ia S, three columns (linear, angular)
constexpr int RS_DINV = 24;   // 6 : (S^T U + Im)^-1, symmetric (xx xy yy xz yz zz)
constexpr int RS_TAU = 30;    // 3 : joint efforts (flexibility spring-damper), then u = tau - S^T f after the backward step
constexpr int RS_EXTRA = 33;
// RecDbl of a spherical record: axis[3] = armature-like rotor inertia of its three dofs, motor[0..2] = stiffness,
// motor[3..5] = damping (JbModelDesc::flexibility)
constexpr int POOL_SIZE = 27; // union { oMi 12 + v 6 | Y 21 + f 6 | a_gf 6 }
constexpr int CSLOT_SIZE = 6; // cached contact wrench in the joint frame: force at the contact point (3), pure torque (3)
constexpr int IMUSLOT_SIZE = 12; // v (6) captured in pass 1, a_gf (6) captured in pass 3

// Build the plan.  `lanes` = 0 chooses L automatically.  `n_hist` = number of stage-derivative
// history slots per dof (0 for Euler / RK4, 7 for DOPRI).
Plan build_plan(const JbModelDesc& m, int lanes, int n_hist);

}  // namespace jb
