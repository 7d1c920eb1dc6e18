/* jiminy_b200 -- C ABI of the H100-native batched rigid-body stepping library.
 *
 * This header is the drop-in boundary for ONE path of duburcqa/jiminy: the per-step rigid-body
 * pipeline of `jiminy::Engine::step` (core/src/engine/engine.cc:1724-2417) and the ODE
 * right-hand side it integrates, `Engine::computeRobotsDynamics` (engine.cc:3585-3708).
 * Every entry point cites the reference interface it replaces.  Plain C: pointers, sizes and
 * int status codes only.  No exception ever crosses this boundary: failures return a negative
 * status and `jb_last_error()` gives the message (the reference throws, python/jiminy_pywrap
 * maps C++ exceptions to Python ones, module.cc:98-102; the Python host layer in
 * `jiminy_b200/core.py` re-raises the matching Python exception class).
 *
 * Memory convention: all host arrays are env-major, C-contiguous, fp64 (`[n_env][width]`), which
 * is what the reference exposes per robot through `RobotState.{q,v,a,command,...}` numpy views
 * (python/jiminy_pywrap/src/engine.cc:175-187), stacked along a leading env axis.  On the device
 * the state is structure-of-arrays `[width][n_env_padded]` (env fastest) so that one warp reads
 * 128-byte-aligned coalesced lines.
 */
#ifndef JIMINY_B200_H
#define JIMINY_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---------------------------------------------------------------- status codes -------- */
#define JB_OK 0
#define JB_ERR_INVALID_ARGUMENT (-1) /* reference: std::invalid_argument -> ValueError      */
#define JB_ERR_BAD_CONTROL_FLOW (-2) /* reference: jiminy::bad_control_flow                 */
#define JB_ERR_RUNTIME (-3)          /* reference: std::runtime_error -> RuntimeError       */
#define JB_ERR_NOT_IMPLEMENTED (-4)  /* reference: jiminy::not_implemented_error            */
#define JB_ERR_CUDA (-5)             /* no CUDA device / CUDA runtime failure (never a CPU fallback) */
#define JB_ERR_PEER_TIMEOUT (-6)     /* multi-GPU observation exchange: a rank never signalled its step     */

/* Per-env status bits written by the device scheduler (jb_get_status).  The reference raises
 * from Engine::step for the first three (engine.cc:1742-1747, :2341-2378). */
#define JB_ENV_OK 0
#define JB_ENV_NAN 1              /* NaN in (q, v, a): "Low-level ode solver failed"                */
#define JB_ENV_ITER_FAILED 2      /* too many successive failed inner iterations                    */
#define JB_ENV_DT_UNDERFLOW 4     /* "The internal time step is getting too small"                  */
#define JB_ENV_JOINT_LIMIT 8      /* informational, sticky: a bounded joint left [lo, hi] at some point,
                                     i.e. its JointConstraint was enabled (engine.cc:3285-3293)     */
#define JB_ENV_NOT_STARTED 16     /* env has never been started (jb_start not called on it)         */
#define JB_ENV_CONTACT_FORCE 32   /* jb_start: initial contact force > 1e5 N (engine.cc:1338-1345)  */
#define JB_ENV_SOLVER_FAILED 64   /* "Too many successive constraint solving failures" (engine.cc:2363-2372) */
#define JB_ENV_CONSTRAINT_OVERFLOW 128 /* more constraint rows enabled at once than the batch was sized for */
#define JB_ENV_BAD_START 256      /* jb_start_device: the env's (q0, v0) row failed Engine::start's input checks
                                     (NaN, q out of bounds); set together with JB_ENV_NOT_STARTED          */

/* ---------------------------------------------------------------- joint model types --- */
/* Pinocchio 2.7 joint models produced by its URDF parser (SURVEY.md App. B). */
enum {
    JB_JOINT_UNIVERSE = 0,
    JB_JOINT_RX = 1, JB_JOINT_RY = 2, JB_JOINT_RZ = 3,      /* JointModelRX/RY/RZ                  */
    JB_JOINT_RU = 4,                                        /* JointModelRevoluteUnaligned         */
    JB_JOINT_RUBX = 5, JB_JOINT_RUBY = 6, JB_JOINT_RUBZ = 7,/* JointModelRUBX/Y/Z  (nq=2: cos,sin) */
    JB_JOINT_RUBU = 8,                                      /* RevoluteUnboundedUnaligned          */
    JB_JOINT_PX = 9, JB_JOINT_PY = 10, JB_JOINT_PZ = 11,    /* JointModelPX/PY/PZ                  */
    JB_JOINT_PU = 12,                                       /* JointModelPrismaticUnaligned        */
    JB_JOINT_FREEFLYER = 13,                                /* JointModelFreeFlyer (nq=7, nv=6)    */
    JB_JOINT_SPHERICAL = 14                                 /* JointModelSpherical (nq=4 quaternion x y z w, nv=3): the flexibility
                                                             * joints of Model::addFlexibilityJointsToExtendedModel (model.cc:1087-1165) */
};

enum { JB_SOLVER_EULER_EXPLICIT = 0, JB_SOLVER_RUNGE_KUTTA_4 = 1, JB_SOLVER_RUNGE_KUTTA_DOPRI = 2 };

/* ---------------------------------------------------------------- model description --- */
/* Flat, read-only description of one robot: what `jiminy::Model`/`jiminy::Robot` yield to the
 * engine (core/src/robot/model.cc, robot.cc) -- tree topology, joint placements, body inertias,
 * rotor inertias, limits, motors, contact frames, sensors -- with Pinocchio's joint / q / v
 * indexing.  All pointers are borrowed for the duration of the call that receives the struct.
 *
 * SE3 placements are 12 doubles: rotation row-major (9) then translation (3), mapping child
 * coordinates to parent coordinates (Pinocchio `SE3`).  Inertias are 10 doubles:
 * mass, lever[3], then the symmetric rotational inertia about the centre of mass in Pinocchio
 * `Symmetric3` order (xx, xy, yy, xz, yz, zz). */
typedef struct JbModelDesc {
    int32_t njoints;              /* including the universe, index 0                              */
    int32_t nq, nv;
    const int32_t* joint_type;    /* [njoints] JB_JOINT_*                                         */
    const int32_t* parent;        /* [njoints] parent joint index (parents precede children)      */
    const int32_t* idx_q;         /* [njoints]                                                    */
    const int32_t* idx_v;         /* [njoints]                                                    */
    const double* placement;      /* [njoints][12] model.jointPlacements                          */
    const double* axis;           /* [njoints][3]  unit axis of 1-dof joints (also set for aligned)*/
    const double* inertia;        /* [njoints][10] model.inertias                                 */
    const double* rotor_inertia;  /* [nv] model.rotorInertia (robot.cc:243-246)                   */
    const double* q_lower;        /* [nq] model.lowerPositionLimit (model.cc:1371-1440)           */
    const double* q_upper;        /* [nq]                                                         */

    /* SimpleMotor table, attach order (robot.cc:249; basic_motors.cc:83-143).  Per motor 10
     * doubles: reduction, effort_limit, velocity_limit, velocity_effort_inv_slope,
     * friction_viscous_pos, friction_viscous_neg, friction_dry_pos, friction_dry_neg,
     * friction_dry_slope, reserved.  Per motor flags: bit0 enableEffortLimit,
     * bit1 enableVelocityLimit, bit2 enableFriction. */
    int32_t nmotors;
    const int32_t* motor_joint;   /* [nmotors] joint index                                        */
    const int32_t* motor_flags;   /* [nmotors]                                                    */
    const double* motor_params;   /* [nmotors][10]                                                */

    /* Contact frames (robot->getContactFrameIndices(), sorted by name, robot.py:717). */
    int32_t ncontacts;
    const int32_t* contact_joint;     /* [ncontacts] parent joint                                 */
    const double* contact_placement;  /* [ncontacts][12] frame placement in parent joint           */

    /* Sensors, attach order per type (basic_sensors.cc). */
    int32_t nimu;
    const int32_t* imu_joint;         /* [nimu]                                                   */
    const double* imu_placement;      /* [nimu][12]                                               */
    int32_t nforce;
    const int32_t* force_joint;       /* [nforce]                                                 */
    const double* force_placement;    /* [nforce][12]                                             */
    int32_t nencoder;
    const int32_t* encoder_joint;     /* [nencoder]                                               */
    const double* encoder_reduction;  /* [nencoder] 1.0 when joint side (basic_sensors.cc:529-537) */
    int32_t neffort;
    const int32_t* effort_motor;      /* [neffort] motor index                                    */
    int32_t ncontact_sensor;
    const int32_t* contact_sensor_index; /* [ncontact_sensor] index into the contact frame list   */

    /* Flexibility joints (modelOptions.dynamics.flexibilityConfig, Engine::computeInternalDynamics, engine.cc:3367-3391):
     * per joint stiffness[3] then damping[3]; only the rows of JB_JOINT_SPHERICAL joints are read.  Their armature-like
     * `inertia` goes into rotor_inertia[idx_v .. idx_v + 2] (model.cc:1136-1144).  NULL: every spherical joint is free. */
    const double* flexibility;        /* [njoints][6] or NULL                                     */
} JbModelDesc;

/* ---------------------------------------------------------------- engine options ------ */
/* The subset of `Engine::EngineOptions` (core/include/jiminy/core/engine/engine.h:260-353) the
 * step path reads.  Defaults: jb_default_options(). */
enum { JB_CONTACT_SPRING_DAMPER = 0, JB_CONTACT_CONSTRAINT = 1 };

typedef struct JbOptions {
    int32_t ode_solver;               /* stepper.odeSolver, JB_SOLVER_*                           */
    int32_t successive_iter_failed_max; /* stepper.successiveIterFailedMax (1000)                 */
    int32_t iter_max;                 /* stepper.iterMax (0 = unlimited), reserved                */
    int32_t contact_model;            /* contacts.model: JB_CONTACT_SPRING_DAMPER / JB_CONTACT_CONSTRAINT */
    double tol_abs, tol_rel;          /* stepper.tolAbs / tolRel                                  */
    double dt_max;                    /* stepper.dtMax                                            */
    double dt_restore_threshold_rel;  /* stepper.dtRestoreThresholdRel                            */
    double sensors_update_period;     /* stepper.sensorsUpdatePeriod                              */
    double controller_update_period;  /* stepper.controllerUpdatePeriod                           */
    double contact_stiffness;         /* contacts.stiffness                                       */
    double contact_damping;           /* contacts.damping                                         */
    double contact_friction;          /* contacts.friction                                        */
    double contact_transition_eps;    /* contacts.transitionEps                                   */
    double contact_transition_velocity; /* contacts.transitionVelocity                            */
    double gravity[6];                /* world.gravity (only the linear part acts)                */
    double contact_torsion;           /* contacts.torsion (constraint model)                      */
    double contact_stabilization_freq; /* contacts.stabilizationFreq: Baumgarte frequency [Hz]    */
    double constraint_regularization; /* constraints.regularization (PGS diagonal damping)        */
} JbOptions;

typedef struct JbBatch JbBatch;

/* Layout of one row of the sensor/observation matrix returned by jb_get_sensors: the reference's
 * per-type shared storage matrices `[fields x sensors]` (abstract_sensor.hxx:445-522) flattened
 * field-major per type, concatenated in the order IMU, Force, Encoder, Effort, Contact. */
typedef struct JbSensorLayout {
    int32_t imu_offset, force_offset, encoder_offset, effort_offset, contact_offset;
    int32_t width;
} JbSensorLayout;

/* Message of the last failing call on this thread. */
const char* jb_last_error(void);

/* Library / build identification ("jiminy_b200 <ver> sm_90a"). */
const char* jb_version(void);

/* Engine option defaults, engine.h:260-341 (SURVEY.md App. D). */
void jb_default_options(JbOptions* out);

/* Replaces: Engine::addRobot + the robot lock taken by Engine::start (engine.cc:952-1533).
 * Uploads the model tables and allocates SoA state for `n_env` lockstep environments on CUDA
 * device `device`.  Fails with JB_ERR_CUDA when no device is usable. */
int jb_batch_create(const JbModelDesc* model, const JbOptions* options, int32_t n_env, int32_t device,
                    JbBatch** out);
int jb_batch_destroy(JbBatch* batch);

/* Replaces: Engine::setOptions (engine.cc:2654-2795).  Only allowed while no env is running,
 * except the contact/gravity values which the reference also allows between episodes. */
int jb_set_options(JbBatch* batch, const JbOptions* options);

/* Replaces: the `internalDynamics` functor of FunctionalController (controller_functor.h:27-80,
 * invoked at engine.cc:3690-3691) for the linear case the reference's analytical tests use
 * (`u_custom = -k q - d v` on 1-dof joints).  k, d are [nv]; NULL disables. */
int jb_set_joint_springs(JbBatch* batch, const double* k, const double* d);

/* Replaces: the PD controller block that `gym_jiminy` pipelines run inside the controller callback,
 * `gym_jiminy.common.blocks.pd_controller` (python/gym_jiminy/common/gym_jiminy/common/blocks/
 * proportional_derivative_controller.py:101-165), for zero-order-held position targets with zero
 * target velocity: at every controller breakpoint
 *     command = clip(kp * ((target - q_enc) + kd * (0 - v_enc)), +-motor.effort_limit).
 * While enabled, jb_set_command uploads *targets* (motor-side positions) instead of efforts.
 * kp, kd are [nmotors]; NULL disables.  Requires a discrete controllerUpdatePeriod. */
int jb_set_pd_controller(JbBatch* batch, const double* kp, const double* kd);

/* One-line description of the lane plan / shared-memory footprint chosen for this batch. */
int jb_describe(JbBatch* batch, char* buf, int32_t len);

/* Host-only planner introspection (no device needed): fills `buf` like jb_describe and, when
 * non-NULL, joint_lane[njoints] (-1 = trunk joint shared by all lanes).  lanes = 0: automatic. */
int jb_plan_describe(const JbModelDesc* model, int32_t lanes, char* buf, int32_t len, int32_t* joint_lane);

/* Replaces: the constraint objects of `robot.constraints` read back by user code and tests -- `bounds_joints[...]`
 * and `contact_frames[...]`, their `is_enabled` and `lambda_c` (python/jiminy_pywrap/src/constraints.cc;
 * AbstractConstraintBase::getIsEnabled / lambda_, core/include/jiminy/core/constraints/abstract_constraint.h).
 * joint_enabled [n_env][njoints] and joint_lambda [n_env][njoints] are indexed by joint (0 for joints without a bound
 * constraint), contact_enabled [n_env][ncontacts], contact_lambda [n_env][ncontacts][4] (x, y, z, torsion) by contact
 * frame.  Any pointer may be NULL.  State after the last dynamics evaluation of each env. */
int jb_get_constraints(JbBatch* batch, uint8_t* joint_enabled, double* joint_lambda, uint8_t* contact_enabled,
                       double* contact_lambda);

/* Replaces: Engine::start(q, v) (engine.cc:952-1533) for every env with mask[i] != 0 (NULL mask =
 * all).  q0 is [n_env][nq], v0 is [n_env][nv] (rows of unmasked envs are ignored).  Normalises q,
 * runs forward kinematics, the initial contact-force guard, the INIT_ITERATIONS fixed-point loop
 * and the first sensor refresh; sets t = 0, dt = SIMULATION_MIN_TIMESTEP. */
int jb_start(JbBatch* batch, const uint8_t* mask, const double* q0, const double* v0);
/* jb_start with device inputs of the same layouts (mask_dev may be NULL: all envs), enqueued on the batch stream without
 * any host synchronisation: the caller keeps the buffers alive until the stream has passed the call.  The input checks
 * of Engine::start run inside the kernel, per env: an env whose row holds a NaN, or a q outside [q_lower - eps,
 * q_upper + eps] (eps = 2.22e-16, as jb_start), is not started -- its status word becomes JB_ENV_NOT_STARTED |
 * JB_ENV_BAD_START and nothing else of it is written -- while the other envs start normally.  The generator start
 * states of the sensor pipeline are recomputed on the host only after jb_set_seeds / jb_set_sensor_options. */
int jb_start_device(JbBatch* batch, const uint8_t* mask_dev, const double* q0_dev, const double* v0_dev);
/* jb_start_device that first puts every started env on the ground: before the input checks, the kernel sets
 * q[2] -= min_i z_i, where z_i is the world height of contact frame i by forward kinematics of the env's own row (its
 * block's model variant included).  This is the rule of BaseJiminyEnv._sample_state (generic.py:1300-1335) as the host
 * envs apply it (robots.ground_base_height): a z shift of the free-flyer onto flat ground, orientation untouched.  The
 * caller's buffers are not written.  A row with a NaN still ends JB_ENV_NOT_STARTED | JB_ENV_BAD_START.  On a model
 * without a free-flyer or without a contact frame the call is jb_start_device. */
int jb_start_device_on_ground(JbBatch* batch, const uint8_t* mask_dev, const double* q0_dev, const double* v0_dev);

/* Replaces: the command buffer written by AbstractController::computeCommand through the
 * FunctionalController callback (engine.cc:3240-3251; controller_functor.h:27-80).  The command is
 * zero-order held until the next call.  cmd is [n_env][nmotors]. */
int jb_set_command(JbBatch* batch, const double* cmd);
/* Same, with `cmd_dev` a device pointer (same layout) on the batch's device: no host copy. */
int jb_set_command_device(JbBatch* batch, const double* cmd_dev);

/* gym_jiminy's `PDController` block on the device (blocks/proportional_derivative_controller.py:301-535), with
 * the optional `MotorSafetyLimit` on top (blocks/motor_safety_limit.py:21-86).  jb_set_command then uploads target
 * motor ACCELERATIONS; at every controller update the (position, velocity, acceleration) targets of each motor are
 * integrated by `integrate_zoh` (:24-98) within [state_lower, state_upper] ([3][nmotors]: position, velocity,
 * acceleration bounds) and the torque is clip(kp ((q_des - q) + kd (v_des - v)), +-effort_limit) (:104-165);
 * jb_start restarts the targets from the clipped measurement.  `safety` = NULL, or [5][nmotors]: kp, kd, soft lower
 * and soft upper position and the velocity limit of `apply_safety_limits` -- what `MotorSafetyLimit.__init__` derives
 * from its arguments (:161-175: position limits +- reduction * soft_position_margin,
 * min(motor velocity limit, reduction * soft_velocity_max)).  kp = NULL disables the block. */
int jb_set_pd_controller_full(JbBatch* batch, const double* kp, const double* kd, const double* state_lower,
                              const double* state_upper, const double* safety);
/* The block's `_command_state` (proportional_derivative_controller.py:390-394, exposed to the pipeline as the
 * controller's state, :451-456): target motor position / velocity / acceleration, [n_env][3][nmotors].  The
 * `PDAdapter` block reads it -- and in its instantaneous mode writes it -- once per env-step
 * (:167-262, :620-640), which is what the getter and the setter are for.  Both need the block enabled. */
int jb_get_pd_controller_state(JbBatch* batch, double* state);
int jb_set_pd_controller_state(JbBatch* batch, const double* state);
/* gym_jiminy's `PDAdapter` block (proportional_derivative_controller.py:166-262, :538-660) on the device, in front of
 * the `PDController` block: jb_set_pd_adapter configures it (order 0: the action is the target motor position at the
 * end of the env-step, 1: the target velocity; `velocity_deadband` [nmotors] or NULL); jb_pd_adapter_device then turns
 * the device action `[n_env][nmotors]` into the target accelerations of the coming env-step -- the command buffer
 * jb_set_command would fill -- reading, and in the instantaneous mode writing, the block's command state, with the
 * bounds given to jb_set_pd_controller_full.  |step_dt| < 1e-9 writes zero accelerations and leaves the state alone.
 * One small kernel on the batch stream, no host synchronisation; the step kernel is not involved. */
int jb_set_pd_adapter(JbBatch* batch, int32_t order, int32_t is_instantaneous, const double* velocity_deadband);
int jb_pd_adapter_device(JbBatch* batch, const double* action_dev, double step_dt);

/* gym_jiminy's `MahonyFilter` observer on the device (blocks/mahony_filter.py:28-101, :337-393 with the default
 * exact_init = True, ignore_twist = False): the attitude estimate of every IMU starts from the true orientation of
 * its frame at jb_start (`matrices_to_quat`, utils/math.py:307-350) and receives one `mahony_filter` iteration with
 * dt = sensorsUpdatePeriod at every sensor refresh of jb_step.  kp < 0 disables it.  jb_get_mahony_filter returns
 * [n_env][nimu][10]: quaternion (x, y, z, w), gyro-bias estimate (3), unbiased angular velocity (3). */
int jb_set_mahony_filter(JbBatch* batch, double kp, double ki);
int jb_get_mahony_filter(JbBatch* batch, double* out);

/* The MahonyFilter with the reference's full option set (jb_set_mahony_filter is this call with exact_init = 1,
 * ignore_twist = 0, compute_rpy = 0, and the same state).  exact_init = 0: at a (re)start the estimate is the swing of
 * the measured accelerometer (`swing_from_vector`, utils/math.py:1066-1137), or the true orientation when every
 * component of the measured acceleration is below 0.1 g (free fall); the start applies no iteration and no twist
 * removal.  ignore_twist: `remove_twist_from_quat` (utils/math.py:1203-1246) after every iteration.  compute_rpy:
 * `quat_to_rpy` (utils/math.py:159-197) after the start and after every iteration. */
int jb_set_mahony_filter_full(JbBatch* batch, double kp, double ki, int32_t exact_init, int32_t ignore_twist, int32_t compute_rpy);

/* gym_jiminy's `BodyObserver` (blocks/body_orientation_observer.py:26-266) on the device, refreshed right after the
 * MahonyFilter at the same times (jb_start at t = 0, then every sensor refresh): the parent body's orientation
 * quat_multiply(q_imu, q_rel, is_right_conjugate=True) and angular velocity q_rel.apply(omega_imu), q_rel the IMU frame's
 * placement rotation in its parent body; twist_time_constant NaN (None) keeps the filter's twist, 0 removes it, > 0
 * removes it and re-estimates it with `update_twist`'s leaky integrator (dt = sensorsUpdatePeriod, zero twist at every
 * (re)start, one update at the start refresh as at the reference's reset); compute_rpy adds `quat_to_rpy`.  enable = 0
 * turns it off.  Only between episodes (JB_ERR_BAD_CONTROL_FLOW while the batch runs); JB_ERR_INVALID_ARGUMENT without
 * the MahonyFilter or for a negative or infinite time constant.  Turning the MahonyFilter off turns it off too.
 * jb_get_observers copies [n_env][nimu][14] to the host: the filter's roll-pitch-yaw (3), the body's quaternion (4),
 * roll-pitch-yaw (3), angular velocity (3) and twist angle (1); fields of an option that is off hold no meaning.
 * JB_ERR_BAD_CONTROL_FLOW when the filter runs its default path only (no record). */
int jb_set_body_observer(JbBatch* batch, int32_t enable, double twist_time_constant, int32_t compute_rpy);
int jb_get_observers(JbBatch* batch, double* out);
/* The device buffer behind jb_get_observers (NULL when there is none); contents are those of the last launch that has
 * completed on the batch stream. */
int jb_device_observer_views(JbBatch* batch, double** observers);

/* gym_jiminy's `StackObservation` wrapper (wrappers/observation_stack.py:185-254) on the device: at every observer
 * refresh of every env -- jb_start at t = 0, then every sensor breakpoint of jb_step, which with
 * sensorsUpdatePeriod == controllerUpdatePeriod is the observer's refresh schedule (observe_dt = control_dt) -- the
 * step kernel updates `num_stack` frames of the chosen leaves, oldest first, with the wrapper's rules: the latest frame
 * always holds the current value; with skip_frames_ratio >= 0 the current value is frozen every skip_frames_ratio + 1
 * refreshes, with -1 at every env-step breakpoint of the refresh time (step_dt of jb_step); the refresh after a freeze
 * drops the oldest frame.  A (re)start zeroes the env's frames and applies one refresh at t = 0.  The last refresh of a
 * jb_step sees the env's end time.  `leaves` [n_leaves] (JB_STACK_*, each at most once, in frame order): the time; a
 * whole sensor-type block of the measured row (jb_get_sensors; field-major, jb_sensor_layout); the PDController
 * block's action, i.e. the command buffer (target accelerations) [nmotors]; the first two rows of its state
 * (jb_get_pd_controller_state) [2][nmotors]; the MahonyFilter quaternions, field-major [4][nimu]; its angular velocity
 * [3][nimu], roll-pitch-yaw [3][nimu] (compute_rpy) and gyro bias [3][nimu]; the BodyObserver's quaternion [4][nimu],
 * roll-pitch-yaw [3][nimu] (compute_rpy) and angular velocity [3][nimu].  A frame is the
 * leaves one after the other.  num_stack = 0 turns stacking off.  Only between episodes (JB_ERR_BAD_CONTROL_FLOW while
 * the batch runs); JB_ERR_NOT_IMPLEMENTED unless sensorsUpdatePeriod == controllerUpdatePeriod > 0; JB_ERR_INVALID_ARGUMENT
 * for num_stack < 0, skip_frames_ratio < -1, no leaf, an unknown or repeated leaf, or a leaf whose sensor type or block
 * is absent.  jb_get_obs_stack copies the frames [n_env][num_stack][frame width] to the host.  The frames are part of
 * no checkpoint: jb_get_stepper_state / jb_set_stepper_state leave them alone. */
#define JB_STACK_T 0
#define JB_STACK_IMU 1
#define JB_STACK_FORCE 2
#define JB_STACK_ENCODER 3
#define JB_STACK_EFFORT 4
#define JB_STACK_CONTACT 5
#define JB_STACK_PD_ACTION 6
#define JB_STACK_PD_STATE 7
#define JB_STACK_MAHONY 8
#define JB_STACK_MAHONY_OMEGA 9
#define JB_STACK_MAHONY_RPY 10
#define JB_STACK_MAHONY_BIAS 11
#define JB_STACK_BODY_QUAT 12
#define JB_STACK_BODY_RPY 13
#define JB_STACK_BODY_OMEGA 14
#define JB_STACK_N_LEAF_KINDS 15
int jb_set_obs_stack(JbBatch* batch, int32_t num_stack, int32_t skip_frames_ratio, const int32_t* leaves, int32_t n_leaves);
int jb_get_obs_stack(JbBatch* batch, double* out);
/* The device buffers behind jb_get_obs_stack (`stack`, NULL when stacking is off) and the command buffer jb_set_command
 * and jb_pd_adapter_device write (`command` [n_env][nmotors]).  Any argument may be NULL.  Contents are those of the last
 * launch that has completed on the batch stream. */
int jb_device_obs_views(JbBatch* batch, double** stack, double** command);

/* Replaces: Engine::stop (engine.cc:2419-2448): every env goes back to "not started", which is what
 * registering or removing forces requires (engine.cc:2456-2461). */
int jb_stop(JbBatch* batch);

/* Replaces: Engine::registerImpulseForce(robot, frame, t, dt, F) (engine.cc:2450-2491;
 * python/jiminy_pywrap/src/engine.cc:651-657) and its use by Engine::step: the wrench is active for
 * t_env in [t, t + dt), both ends are integration breakpoints (engine.cc:1843-1890, :2002-2006, :2228),
 * and it enters the dynamics through computeExternalForces (engine.cc:3463-3480).  The frame is given
 * by its parent joint index and its translation in that joint's frame (the wrench is expressed in
 * world-aligned axes at the frame origin, so the frame's rotation is irrelevant;
 * convertForceGlobalFrameToJoint, utilities/pinocchio.cc:794-809).  One frame for all envs, per-env
 * application time, duration and wrench: t [n_env], dt [n_env], wrench [n_env][6] (linear, angular).
 * Times are relative to each env's own start.  index_out receives the impulse index. */
int jb_register_impulse_force(JbBatch* batch, int32_t joint, const double* frame_translation, const double* t,
                              const double* dt, const double* wrench, int32_t* index_out);
/* Rewrites impulse `index` of the envs selected by mask (NULL = all): what removing and re-registering
 * the forces of one env at an episode reset does (locomotion.py:314-323).  Call it right before the
 * masked jb_start of those envs. */
int jb_set_impulse_force(JbBatch* batch, int32_t index, const uint8_t* mask, const double* t, const double* dt,
                         const double* wrench);
/* Replaces: Engine::registerProfileForce(robot, frame, func, updatePeriod) (engine.cc:2518-2567) where
 * `func` returns the per-env wrench last written with jb_set_profile_force.  update_period == 0: the
 * value is read at every dynamics evaluation (engine.cc:3488-3491); update_period > 0: it is sampled at
 * the multiples of the period, which become breakpoints (engine.cc:1892-1917, :2551-2562), and is zero
 * between start and the first step. */
int jb_register_profile_force(JbBatch* batch, int32_t joint, const double* frame_translation, double update_period,
                              int32_t* slot_out);
int jb_set_profile_force(JbBatch* batch, int32_t slot, const double* wrench /* [n_env][6] */);
/* jb_set_impulse_force from device buffers of the same layouts (mask_dev may be NULL: all envs), one small kernel on the
 * batch stream with no host synchronisation.  Engine::registerImpulseForce's checks (engine.cc:2463-2475) run per env, with
 * NaN added: a row with a NaN, t < 0 or dt < STEPPER_MIN_TIMESTEP is not written and its env's status becomes
 * JB_ENV_NOT_STARTED | JB_ENV_BAD_START, as for a row jb_start_device rejects (a later start of that env clears it). */
int jb_set_impulse_force_device(JbBatch* batch, int32_t index, const uint8_t* mask_dev, const double* t_dev,
                                const double* dt_dev, const double* wrench_dev);
/* Replaces: Engine::registerProfileForce(robot, frame, func, 0) where `func` evaluates periodic tabular processes, as the
 * walker env's disturbance profile does (gym_jiminy locomotion.py:326-330, :340-359, with PeriodicTabularProcess::operator(),
 * core/src/utilities/random.cc:336-400).  Component component[k] (0..5: linear then angular, world-aligned axes at the
 * frame origin) of the wrench is the periodic cubic-Hermite table k of each env: n_knots[k] knots evenly spaced over
 * period[k], evaluated at the env's own time.  update_period == 0: at the time of every dynamics evaluation (every stage
 * of every stepper, and the evaluations of jb_start at t = 0); update_period > 0: sampled at the multiples of the period
 * and held, with the breakpoints and the zero-until-the-first-update rule of jb_register_profile_force.  The force has a
 * slot of its own.  Its tables start at zero; slot_out receives the process-force index. */
int jb_register_process_force(JbBatch* batch, int32_t joint, const double* frame_translation, double update_period,
                              int32_t n_comp, const int32_t* component, const int32_t* n_knots, const double* period,
                              int32_t* slot_out);
/* Rewrites the tables of process force `slot` for the envs selected by mask (NULL = all): values and grads are
 * [n_env][sum of n_knots] (knot values and slopes of the tables one after the other; any gain is folded into both by the
 * caller).  Allowed while envs run; the new tables apply from the next evaluation of those envs.  The _device form takes
 * device buffers of the same layouts and is enqueued on the batch stream without host synchronisation. */
int jb_set_process_force(JbBatch* batch, int32_t slot, const uint8_t* mask, const double* values, const double* grads);
int jb_set_process_force_device(JbBatch* batch, int32_t slot, const uint8_t* mask_dev, const double* values_dev,
                                const double* grads_dev);
/* Replaces: Engine::removeAllForces (engine.cc:568-573, :2569-2638). */
int jb_remove_all_forces(JbBatch* batch);

/* Replaces: Engine::step(stepSize) (engine.cc:1724-2417), all envs in lockstep, one launch.
 * step_dt < EPS selects the reference's default step size rule (engine.cc:1758-1777). */
int jb_step(JbBatch* batch, double step_dt);

/* Replaces: one call of Engine::computeRobotsDynamics (engine.cc:3585-3708) as exposed for parity
 * through `jiminy_py.core.aba`-style helpers (python/jiminy_pywrap/src/helpers.cc:423-477):
 * evaluates a = f(q, v, command) for every env without touching the running state.
 * q [n_env][nq], v [n_env][nv], cmd [n_env][nmotors] -> a [n_env][nv],
 * fext [n_env][njoints][6] (may be NULL), u [n_env][nv] (may be NULL). */
int jb_compute_dynamics(JbBatch* batch, const double* q, const double* v, const double* cmd,
                        double* a, double* fext, double* u);

/* Replaces: the numpy views StepperState.{t,q,v,a} (pywrap engine.cc:134-143).  Any pointer may
 * be NULL.  t [n_env], q [n_env][nq], v/a [n_env][nv]. */
int jb_get_state(JbBatch* batch, double* t, double* q, double* v, double* a);

/* Checkpoint / restore of a running batch.  Replaces: the remaining fields of `StepperState` a resumed rollout needs
 * besides (t, q, v, a) -- `dt`, `dtLargest`, the Kahan error `tError`, ... (core/include/jiminy/core/engine/engine.h:216-250;
 * the reference serialises them nowhere: a simulation can only be replayed from t = 0) -- and the command held since
 * the last controller update (RobotState.command).  sched [n_env][6] = (t, dt, dtLargest, dtLargestPrev, tError,
 * tPrev); command_held [n_env][nmotors].  jb_set_stepper_state overwrites whichever arrays are non-NULL (q [n_env][nq],
 * v / a [n_env][nv], iter / iter_failed [n_env]); contact forces, sensors and extra terms are rebuilt from (q, v, a)
 * by the next jb_step.  Constraint multipliers and the states of the device controller blocks are not touched (they
 * have their own getters / setters); neither are the stacked observation frames (jb_set_obs_stack), which have no setter:
 * a restored batch stacks on from the frames of its last launch. */
int jb_get_stepper_state(JbBatch* batch, double* sched, double* command_held);
int jb_set_stepper_state(JbBatch* batch, const double* sched, const double* q, const double* v, const double* a,
                         const int64_t* iter, const int64_t* iter_failed, const double* command_held);

/* Replaces: RobotState.{u, u_motor, command, f_external} views (pywrap engine.cc:175-187).
 * u [n_env][nv], u_motor [n_env][nmotors], command [n_env][nmotors], fext [n_env][njoints][6]. */
int jb_get_efforts(JbBatch* batch, double* u, double* u_motor, double* command, double* fext);

/* Replaces: robot.sensor_measurements (Robot::computeSensorMeasurements, robot.cc:952) as
 * refreshed by the engine at each sensor breakpoint (engine.cc:2386-2410).  out [n_env][width]. */
int jb_get_sensors(JbBatch* batch, double* out);
int jb_sensor_layout(JbBatch* batch, JbSensorLayout* out);

/* Replaces: AbstractSensorBase::setOptions with the options every sensor shares -- `noiseStd`, `bias`, `delay`, `jitter`,
 * `delayInterpolationOrder` (core/include/jiminy/core/hardware/abstract_sensor.h:66-100) -- i.e. the measurement pipeline
 * applied on top of the true value at every sensor refresh: the value `delay` (+ uniform jitter) seconds ago from a
 * ring of past true values, zero-order hold or linear interpolation (abstract_sensor.hxx:305-430, :445-522), plus white
 * noise, plus bias (abstract_sensor.cc:71-85).  `type`: 0 ImuSensor, 1 ForceSensor, 2 EncoderSensor, 3 EffortSensor,
 * 4 ContactSensor; `index`: attach order within the type; noise_std / bias: one value per field of the type (6, 6, 2, 1,
 * 3), NULL = none.  Once any sensor has options, jb_get_sensors returns MEASUREMENTS (what `robot.sensor_measurements`
 * holds) and jb_get_sensor_data the true values (`sensor.data`); without options both are the true values and the step
 * path is bit-unchanged.  Only between episodes (after jb_stop / before the first jb_start), like the reference; needs
 * a discrete sensorsUpdatePeriod. */
int jb_set_sensor_options(JbBatch* batch, int32_t type, int32_t index, const double* noise_std, const double* bias,
                          double delay, double jitter, int32_t delay_interpolation_order);
/* Replaces: `stepper.randomSeedSeq` of each env's engine (engine.h:331, Engine::reset engine.cc:756-763), one 32-bit
 * seed per env: jb_start derives from it the generator of every sensor of the (re)started envs with the reference's
 * chain -- PCG32(seed_seq{seed}) -> one draw per sensor type -> seed_seq expansion -> PCG32(seed) per sensor
 * (abstract_sensor.hxx:213-226, random.cc:10-37).  Default: 0 for every env. */
int jb_set_seeds(JbBatch* batch, const uint32_t* seeds /* [n_env] */);
int jb_get_sensor_data(JbBatch* batch, double* out /* [n_env][width] true values */);
/* Per-env sensor options: what the walker env's setOptions of every sensor at every reset needs (gym_jiminy
 * locomotion.py:264-286), with envs restarting while others run.  jb_enable_per_env_sensor_options puts every sensor in
 * the measurement pipeline with per-env option tables (initially all zero; noise and bias are applied for every sensor,
 * delayInterpolationOrder 1) and sizes the delay ring once for `delay_bound`, the largest delay + jitter any row may hold.
 * Only between episodes, like jb_set_sensor_options, which it replaces: afterwards that one returns JB_ERR_BAD_CONTROL_FLOW.
 * Needs a discrete sensorsUpdatePeriod.
 * jb_set_sensor_options_env writes the rows of the envs selected by mask (NULL = all): noise_std and bias [n_env][width]
 * in the columns of the sensor matrix (jb_sensor_layout), one value per field of every sensor; delay and jitter
 * [n_env][nsensors] in the pipeline's sensor order (Imu, Force, Encoder, Effort, Contact; attach order within a type).
 * The rows are pending: an env runs with them from its next start (jb_start with the env in its mask, or
 * jb_start_device), which also computes that env's per-type delayMax; a running env is not affected, as a locked robot
 * refuses setOptions in the reference.  A row with a NaN, a negative delay or jitter, or delay + jitter > delay_bound is
 * refused: the host form writes nothing and returns JB_ERR_INVALID_ARGUMENT naming the env; the _device form (device
 * buffers, one kernel on the batch stream, no host synchronisation) skips that row and marks the env, whose starts then
 * leave it JB_ENV_NOT_STARTED | JB_ENV_BAD_START until a valid row for it is written. */
int jb_enable_per_env_sensor_options(JbBatch* batch, double delay_bound);
int jb_set_sensor_options_env(JbBatch* batch, const uint8_t* mask, const double* noise_std, const double* bias,
                              const double* delay, const double* jitter);
int jb_set_sensor_options_env_device(JbBatch* batch, const uint8_t* mask_dev, const double* noise_std_dev,
                                     const double* bias_dev, const double* delay_dev, const double* jitter_dev);
/* jb_set_seeds for the envs selected by mask_dev (NULL = all) from a device buffer seeds_dev [n_env], one kernel on the
 * batch stream: the generator start states of those envs, bit-identical to the ones jb_set_seeds + jb_start derive on the
 * host.  The host does not overwrite them from its own copy of the seeds until the next jb_set_seeds.  Needs the
 * measurement pipeline (a sensor option, or per-env options). */
int jb_set_seeds_device(JbBatch* batch, const uint8_t* mask_dev, const uint32_t* seeds_dev);

/* Replaces: the quantities Engine::computeExtraTerms leaves in pinocchio::Data after each
 * successful step (engine.cc:800-905): per env kinetic+potential energy `energy` [n_env][2],
 * joint spatial accelerations `joint_a` [n_env][njoints][6] (data.a) and joint internal wrenches
 * `joint_f` [n_env][njoints][6] (data.f).  Any pointer may be NULL. */
int jb_get_extra_terms(JbBatch* batch, double* energy, double* joint_a, double* joint_f);

/* Replaces: the centroidal quantities of the same function (engine.cc:817-832, :890-904), read by user code through
 * `robot.pinocchio_data.{Ycrb, com, vcom, hg, dhg}`: subtree inertias `ycrb` [n_env][njoints][10] (mass, lever[3],
 * inertia about the subtree centre of mass xx xy yy xz yz zz -- Pinocchio's `Inertia`; row 0 unused), subtree centres
 * of mass `com` [n_env][njoints][3] in the joint frames (row 0: whole robot, world frame) and their velocities `vcom`
 * [n_env][njoints][3] (h[j].linear / mass[j]), centroidal momentum `hg` [n_env][6] and its derivative `dhg` [n_env][6]
 * (linear, angular about the centre of mass).  Any pointer may be NULL. */
int jb_get_centroidal(JbBatch* batch, double* ycrb, double* com, double* vcom, double* hg, double* dhg);

/* Replaces: the exceptions Engine::step raises per robot; here one word per env (JB_ENV_*). */
int jb_get_status(JbBatch* batch, int32_t* status);

/* Replaces: StepperState.{iter, iter_failed} (pywrap engine.cc:134-143). iter/iter_failed [n_env]. */
int jb_get_iters(JbBatch* batch, int64_t* iter, int64_t* iter_failed);

/* Device-resident views for zero-copy consumers (policy networks on the same GPU): the sensor
 * matrix `[n_env][width]` and the stacked (q, v) `[n_env][nq+nv]`, refreshed by jb_step.  This
 * is the buffer a multi-GPU rollout all-gathers (SURVEY.md 8e). */
int jb_device_views(JbBatch* batch, double** sensors_dev, double** qv_dev);
/* The device buffers behind jb_get_status (`status` [n_env]), jb_get_pd_controller_state (`pd_state`
 * [n_env][3][nmotors]) and jb_get_mahony_filter (`mahony` [n_env][nimu][10]), same layouts; a pointer is NULL when its
 * block is off.  Any argument may be NULL.  Contents are those of the last launch that has completed on the batch stream. */
int jb_device_block_views(JbBatch* batch, int32_t** status, double** pd_state, double** mahony);

/* Model randomisation: `Model::addBiasedToExtendedModel` (core/src/robot/model.cc:1166-1236; options
 * `centerOfMassPositionBodiesBiasStd`, `massBodiesBiasStd`, `inertiaBodiesBiasStd`, `relativePositionBodiesBiasStd`)
 * re-draws the body inertias and joint placements of a robot at every `Engine::reset`.  A batch holds `n_variants` such
 * draws of the model it was created with -- same kinematic tree, hardware and frames, other numbers (anything else is
 * rejected) -- and assigns them per GROUP of jb_envs_per_group() consecutive envs (the envs that share a warp):
 * `variant_of_group[g]` in [0, n_variants), g < ceil(n_env / jb_envs_per_group()).  Takes effect at the next launch;
 * call it before jb_start (or restart the envs afterwards, as the reference's reset does). */
int jb_set_model_variants(JbBatch* batch, int32_t n_variants, const JbModelDesc* models, const int32_t* variant_of_group);
int jb_envs_per_group(JbBatch* batch);

/* Per-env flexibility parameters: the walker env's `model` randomisation (gym_jiminy locomotion.py:288-296) re-draws the
 * stiffness and damping of every flexibility joint at every reset, with envs restarting while others run.
 * jb_enable_per_env_flexibility gives every env its own row [n_flex][6] (stiffness xyz, then damping xyz of each
 * flexibility), flexibilities in the order of `flex_joints` [n_flex] -- the joint indices of the model's spherical
 * joints, each once (`robot.flexibility_joint_indices`); NULL: increasing joint index.  Two device tables, pending and
 * active, both start from each env's model values (its variant's with jb_set_model_variants).  Refused
 * (JB_ERR_INVALID_ARGUMENT) on a model without flexibility joints, with a list that is not a permutation of them, and on
 * a second call.
 * jb_set_flexibility_env writes the pending rows [n_env][n_flex][6] of the envs selected by mask (NULL = all).  An env
 * runs with its pending row from its next start (jb_start with the env in its mask, or jb_start_device), which copies it
 * into the active row before the start's own evaluations; a running env is not affected.  The active rows override the
 * stiffness and damping of every variant; the variant's other numbers still apply.  A row with a value that is not
 * finite or is negative (Model::setOptions, model.cc:1620-1626) is refused: the host form writes nothing and returns
 * JB_ERR_INVALID_ARGUMENT naming the env; the _device form (device buffers, one kernel on the batch stream, no host
 * synchronisation) skips that row and marks the env, whose starts then leave it JB_ENV_NOT_STARTED | JB_ENV_BAD_START
 * until a valid row for it is written.  The mark is the flexibility setter's own: sensor rows neither set nor clear it.
 * jb_get_flexibility_env reads the active rows [n_env][n_flex][6]. */
int jb_enable_per_env_flexibility(JbBatch* batch, int32_t n_flex, const int32_t* flex_joints);
int jb_set_flexibility_env(JbBatch* batch, const uint8_t* mask, const double* rows);
int jb_set_flexibility_env_device(JbBatch* batch, const uint8_t* mask_dev, const double* rows_dev);
int jb_get_flexibility_env(JbBatch* batch, double* out);

/* Per-env model rows: the body biases of Model::addBiasedToExtendedModel (model.cc:1166-1236), which the reference
 * re-draws at every reset (Model::reset -> generateModelExtended, model.cc:398-416), per env.
 * jb_enable_per_env_model gives every env its own copy of the batch's double table and a pending row [njoints][13] in
 * model joint order: per joint, mass, lever xyz, rotational inertia about the centre of mass (xx xy yy xz yz zz), joint-
 * placement translation xyz.  Row 0 (the universe) is ignored.  Tables and rows start from each env's model values (its
 * variant's with jb_set_model_variants, which is refused once this has run).  Refused (JB_ERR_INVALID_ARGUMENT) on a
 * second call and when n_env times the rows of one table reaches 2^23.
 * jb_set_model_env writes the pending rows [n_env][njoints][13] of the envs selected by mask (NULL = all).  Every start of
 * an env expands its pending row into its table (every row of the joint, subtree masses and the total mass recomputed)
 * before the start's grounding (jb_start_device_on_ground) and evaluations; a running env is not affected.  A row with a
 * value that is not finite, or with a mass that is not positive (0 is accepted where the model's body is massless), is
 * refused: the host form writes nothing and returns JB_ERR_INVALID_ARGUMENT naming the env; the _device form (device
 * buffers, one kernel on the batch stream, no host synchronisation) skips that row and marks the env, whose starts then
 * leave it JB_ENV_NOT_STARTED | JB_ENV_BAD_START until a valid row for it is written.  The mark is this setter's own.
 * The expansion runs in a launch of its own ahead of the start kernel, for the started envs that no rejected device row
 * (model rows, sensor options, flexibility parameters) refuses; an env whose start is refused by its input checks has
 * still taken its pending row, which its next start takes again.
 * jb_get_model_env reads the rows every env runs with (taken at its last start) [n_env][njoints][13]. */
int jb_enable_per_env_model(JbBatch* batch);
int jb_set_model_env(JbBatch* batch, const uint8_t* mask, const double* rows);
int jb_set_model_env_device(JbBatch* batch, const uint8_t* mask_dev, const double* rows_dev);
int jb_get_model_env(JbBatch* batch, double* out);

/* Reward and termination compositions: gym_jiminy's trajectory-free terms (jiminy_b200/compositions.py), evaluated per env
 * on the device after every env-step, with no host synchronisation.
 * jb_contact_positions_device enqueues the world position of every contact frame of every env from the accepted state,
 * out_dev [n_env][ncontacts][3] (device memory), by the forward sweep of jb_start_device_on_ground on each env's own model
 * (model variants, per-env model rows).  Envs that are not started or carry NaN read NaN.
 * jb_set_compositions uploads the spec once (synchronising): n_node nodes, the reward tree first (n_reward nodes in
 * post-order, root last), then the termination conditions in evaluation order.  Per node node_int [4] = kind
 * (1 SurviveReward, 2 MinimizeMechanicalPowerConsumption, 3 AdditiveMixtureReward, 4 MultiplicativeMixtureReward,
 * 10 BaseRollPitchTermination, 11 FallingTermination, 12 FlyingTermination, 13 MechanicalSafetyTermination,
 * 14 MechanicalPowerConsumptionTermination), number of components (mixtures), EnergyGenerationMode (power terms),
 * training_only; node_dbl [8] = grace_period, then the kind's numbers: power reward cutoff, horizon; additive order (inf
 * allowed); roll-pitch low roll, low pitch, high roll, high pitch; falling low; flying high (at [3]); safety
 * position_margin, velocity_max; power termination -, horizon (NaN: instantaneous), max_power (at [3]).  A NaN bound is
 * not checked.  weights: the additive mixtures' weights in post-order, n_weight of them.  motor_int [nmotors][2] = q and
 * v index of each motor's joint; motor_dbl [nmotors][3] = reduction, q_lower, q_upper of that joint.  env [3] = step_dt,
 * simulation_duration_max, base height threshold (NaN: none).  A malformed or out-of-range spec (unknown kind or
 * generator mode, a mixture without components, non-positive order, cutoff or horizon, negative or missing weights) is
 * refused with JB_ERR_INVALID_ARGUMENT and nothing is uploaded.  Every env's power stacks are emptied.
 * jb_compositions_device enqueues one launch.  restart_mask_dev null: evaluation after an env-step -- every power stack
 * takes the power of the accepted state, then the env's own rule (base height, failure bits of the status word, time
 * limit), the termination conditions (the first that fires wins) and the reward tree; writes reward [n_env],
 * terminated / truncated [n_env] (0 / 1), index [2][n_env] (the condition that terminated / truncated, -1: none) and
 * values [n_node][n_env] (each node's value, 1 / 0 for a condition that fired / did not, NaN: not evaluated).
 * restart_mask_dev given: the masked envs' stacks are emptied and take the power of the state they (re)started from;
 * nothing else is read or written.  The power uses the command held since the last controller update (the PD block's
 * torque in PD mode, the command buffer otherwise). */
int jb_contact_positions_device(JbBatch* batch, double* out_dev);
int jb_set_compositions(JbBatch* batch, int32_t n_node, int32_t n_reward, const int32_t* node_int, const double* node_dbl,
                        int32_t n_weight, const double* weights, const int32_t* motor_int, const double* motor_dbl,
                        const double* env, int32_t training);
int jb_compositions_device(JbBatch* batch, const uint8_t* restart_mask_dev, const int64_t* num_steps_dev,
                           const double* contact_pos_dev, double* reward, uint8_t* terminated, uint8_t* truncated,
                           int32_t* index, double* values);

/* Stable zero-copy views of the state, like the `StepperState` / `RobotState` members the reference exposes to Python as
 * array views of the engine's own memory (python/jiminy_pywrap/include/jiminy/python/functors.h:57-68, generic.py:688-690:
 * a gym env reads `q`, `v`, the sensor matrix every step without a getter call).  The first call with `host` non-null
 * allocates pinned host mirrors; from then on every jb_start / jb_step refreshes them behind the kernel on the batch
 * stream (contents valid after jb_synchronize or any synchronising getter); the addresses never change.  `device`
 * (optional) receives the device buffers of the same layout (`a` only once host mirrors exist).  Rows are env-major:
 * t [n_env], qv [n_env][nq + nv] (q then v), a [n_env][nv], sensors [n_env][width]. */
typedef struct JbStateViews {
    const double* t;
    const double* qv;
    const double* a;
    const double* sensors;
    int32_t n_env, nq, nv, width;
} JbStateViews;
int jb_state_ptrs(JbBatch* batch, JbStateViews* host, JbStateViews* device);

/* Asynchronous device-to-device copy (on the batch stream) of the sensor matrix `[n_env][width]` into a
 * caller-owned device buffer, e.g. the send buffer of the observation all-gather. */
int jb_copy_sensors_device(JbBatch* batch, double* dst_dev);

/* ---- multi-GPU observation exchange over peer memory (NVLink / NVSwitch), one process per GPU ----
 * Replaces the end-of-step observation concat of a sharded rollout (SURVEY.md 8e) -- an ncclAllGather in the
 * plain layout -- by stores issued from inside the step kernel: every env writes its sensor row straight into
 * the gathered buffer `[world][n_env][width]` of every rank, so the exchange overlaps the physics of the other
 * warps and costs no collective.  Protocol: each rank calls jb_peer_obs_create (allocates its buffer, returns
 * the 64-byte CUDA IPC handle), the handles are exchanged out of band (e.g. torch.distributed
 * all_gather_object), each rank calls jb_peer_obs_connect with all of them.  From then on jb_step publishes and
 * signals; jb_peer_obs_wait enqueues (on the batch stream) the wait for every rank's signal of the last step
 * (it gives up after JB_PEER_TIMEOUT_S seconds, default 2: the next synchronising call -- jb_synchronize,
 * jb_get_sensors -- then returns JB_ERR_PEER_TIMEOUT naming the silent rank);
 * jb_peer_obs_view returns the gathered buffer of that step (two buffers alternate, so a fast rank never
 * overwrites what a slower one is still reading). */
int jb_peer_obs_create(JbBatch* batch, int32_t world, int32_t rank, uint8_t handle_out[64]);
int jb_peer_obs_connect(JbBatch* batch, const uint8_t* handles /* [world][64], rank order */);
int jb_peer_obs_wait(JbBatch* batch);
/* on = 0: jb_step stops publishing / signalling (a rank that connected while another could not -- all ranks then
 * use the plain all-gather); on = 1 resumes.  Every rank must hold the same setting. */
int jb_peer_obs_enable(JbBatch* batch, int32_t on);
int jb_peer_obs_view(JbBatch* batch, double** obs_dev /* [world][n_env][width] */);

/* Stream the batch launches on (a `cudaStream_t` cast to void*), for CUDA-event timing. */
int jb_get_stream(JbBatch* batch, void** stream);
/* Number of kernel launches issued by this batch so far (bench.py `gpu_launches`). */
int64_t jb_launch_count(JbBatch* batch);
/* Block until all work queued on the batch stream has completed. */
int jb_synchronize(JbBatch* batch);

#ifdef __cplusplus
}
#endif
#endif /* JIMINY_B200_H */
