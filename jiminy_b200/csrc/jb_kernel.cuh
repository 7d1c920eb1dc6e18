// The env-step kernel: per-env scheduler of Engine::step (core/src/engine/engine.cc:1724-2417)
// around the device steppers, plus Engine::start (engine.cc:952-1533) and a single-RHS mode.
#pragma once
#include "jb_device.cuh"

namespace jb {

// q / v component of a record <-> SoA global state
JB_DI void load_record_state(const Ctx& c, const RecInt* ri, int base, const double* __restrict__ q,
                             const double* __restrict__ v, const double* __restrict__ a, size_t stride, size_t col) {
    double* const rp = jb_smem + base * 32 + c.lane;
    if (ri->kind == REC_SPH) {
        // quaternion / angular velocity in the angular halves of the free-flyer layout, linear halves zero
#pragma unroll
        for (int k = 0; k < 3; ++k) { RP(RF_Q + k) = 0.0; RP(RF_V + k) = 0.0; RP(RF_A + k) = 0.0; }
#pragma unroll
        for (int k = 0; k < 4; ++k) RP(RF_Q + 3 + k) = q[(ri->idx_q + k) * stride + col];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            RP(RF_V + 3 + k) = v[(ri->idx_v + k) * stride + col];
            RP(RF_A + 3 + k) = a ? a[(ri->idx_v + k) * stride + col] : 0.0;
        }
    } else if (ri->kind == REC_FREE) {
#pragma unroll
        for (int k = 0; k < 7; ++k) RP(RF_Q + k) = q[(ri->idx_q + k) * stride + col];
#pragma unroll
        for (int k = 0; k < 6; ++k) {
            RP(RF_V + k) = v[(ri->idx_v + k) * stride + col];
            RP(RF_A + k) = a ? a[(ri->idx_v + k) * stride + col] : 0.0;
        }
    } else {
        RP(R1_Q) = q[ri->idx_q * stride + col];
        RP(R1_Q + 1) = (ri->kind == REC_REVU) ? q[(ri->idx_q + 1) * stride + col] : 0.0;
        RP(R1_V) = v[ri->idx_v * stride + col];
        RP(R1_A) = a ? a[ri->idx_v * stride + col] : 0.0;
    }
}

// Loads from env-major (AoS) arrays: element (env, k) at p[env * width + k]
JB_DI void load_record_state_aos(const Ctx& c, const RecInt* ri, int base, const double* __restrict__ q,
                                 const double* __restrict__ v, int env) {
    double* const rp = jb_smem + base * 32 + c.lane;
    const double* qe = q + static_cast<size_t>(env) * KP->nq;
    const double* ve = v + static_cast<size_t>(env) * KP->nv;
    if (ri->kind == REC_SPH) {
#pragma unroll
        for (int k = 0; k < 3; ++k) { RP(RF_Q + k) = 0.0; RP(RF_V + k) = 0.0; RP(RF_V + 3 + k) = ve[ri->idx_v + k]; }
#pragma unroll
        for (int k = 0; k < 4; ++k) RP(RF_Q + 3 + k) = qe[ri->idx_q + k];
#pragma unroll
        for (int k = 0; k < 6; ++k) RP(RF_A + k) = 0.0;
    } else if (ri->kind == REC_FREE) {
#pragma unroll
        for (int k = 0; k < 7; ++k) RP(RF_Q + k) = qe[ri->idx_q + k];
#pragma unroll
        for (int k = 0; k < 6; ++k) { RP(RF_V + k) = ve[ri->idx_v + k]; RP(RF_A + k) = 0.0; }
    } else {
        RP(R1_Q) = qe[ri->idx_q];
        RP(R1_Q + 1) = (ri->kind == REC_REVU) ? qe[ri->idx_q + 1] : 0.0;
        RP(R1_V) = ve[ri->idx_v];
        RP(R1_A) = 0.0;
    }
}

// pinocchio::normalize on the record (Engine::start, engine.cc:1042-1043)
JB_DI void normalize_record(const Ctx& c, const RecInt* ri, int base) {
    double* const rp = jb_smem + base * 32 + c.lane;
    if (rec_is_big(ri->kind)) {
        double n2 = 0.0;
#pragma unroll
        for (int k = 3; k < 7; ++k) n2 += RP(RF_Q + k) * RP(RF_Q + k);
        const double n = sqrt(n2);
#pragma unroll
        for (int k = 3; k < 7; ++k) RP(RF_Q + k) /= n;
    } else if (ri->kind == REC_REVU) {
        const double n = sqrt(RP(R1_Q) * RP(R1_Q) + RP(R1_Q + 1) * RP(R1_Q + 1));
        RP(R1_Q) /= n; RP(R1_Q + 1) /= n;
    }
}

// Forward sweep of the lane's records from the loaded positions, with the step's joint transforms (joint_calc), pool
// transforms and contact slots: on_contact(slot, world position) for every contact slot of the lane.  Shared by the
// grounding of a start (place_on_ground) and the contact-frame pass (contact_positions_kernel).
template <class F>
JB_DI void contact_frame_sweep(const Ctx& c, F&& on_contact) {
    const int L = KP->L;
    stage_from_accepted(c);
    Xf oMc;
#pragma unroll
    for (int k = 0; k < 9; ++k) oMc.R[k] = 0.0;
    oMc.p = mk(0, 0, 0);
    for (int r = 0; r < KP->nrec; ++r) {
        const RecInt* ri = KP->rint + (r * L + c.sub);
        if (ri->kind == REC_PAD) continue;
        const RecDbl* rd = JB_RDBL + (r * L + c.sub);
        const int base = KP->rec_off[r];
        double* const rp = jb_smem + base * 32 + c.lane;
        if (ri->parent_rec >= 0 && !ri->carry_in) sm_load_xf(c, KP->pool_off + POOL_SIZE * ri->parent_pool, oMc);
        Xf li; Mot vJ = mzero();
        double qd = 0.0;
        joint_calc(c, ri->kind, rd->placement, ld3(rd->axis), rp, base, li, vJ, qd);
        Xf oM;
        if (ri->parent_rec < 0) oM = li;
        else {
            mat3mul(oMc.R, li.R, oM.R);
            oM.p = oMc.p + rmul(oMc.R, li.p);
        }
        for (int k = 0; k < ri->ncontact; ++k) {
            const ContactSlot* ct = KP->cslots + ((ri->contact0 + k) * L + c.sub);
            on_contact(ct, oM.p + rmul(oM.R, ld3(ct->placement + 9)));
        }
        if (ri->pool >= 0) sm_store_xf(c, KP->pool_off + POOL_SIZE * ri->pool, oM);
        oMc = oM;
    }
}

// jb_start_device_on_ground: `robots.ground_base_height` on the device (the rule of BaseJiminyEnv._sample_state,
// generic.py:1300-1335): q[2] of this env's input row is lowered or raised so that its lowest contact frame touches the
// flat ground z = 0.  The forward kinematics runs on the row as given (before the start's quaternion normalisation), with
// the forward sweep's joint transforms (joint_calc) and this block's model variant.  Each lane takes the min over its own
// contact slots, then every lane reads the group's lane minima in the order 0 .. L-1, so that all of them agree bit for
// bit.  Sub-lane 0 writes q[2] into the batch's own copy of the row (KP->q_in), which the input checks and the loads of
// the start then read.  The min keeps a NaN, so a row that yields one still fails the checks.  Without a free-flyer at
// q[0:7] or without a contact frame the row is left as it is.
__device__ __noinline__ void place_on_ground(const Ctx c) {
    const int L = KP->L;
    bool has_free = false;
    for (int r = 0; r < KP->nrec; ++r) {
        const RecInt* ri = KP->rint + (r * L + c.sub);
        if (ri->kind == REC_PAD) continue;
        load_record_state_aos(c, ri, KP->rec_off[r], KP->q_in, KP->v_in, c.env);
        has_free = has_free || (ri->kind == REC_FREE && ri->idx_q == 0);
    }
    double zmin = D_INF;
    bool any_contact = false;
    contact_frame_sweep(c, [&](const ContactSlot*, const V3& p) {
        zmin = (p.z < zmin || p.z != p.z) ? p.z : zmin;
        any_contact = true;
    });
    double zg = D_INF;
    for (int k = 0; k < L; ++k) {
        const double z = jb_shfl(c, zmin, c.lane - c.sub + k);
        zg = (z < zg || z != z) ? z : zg;
    }
    if (jb_any(c, has_free) && jb_any(c, any_contact) && c.valid && c.sub == 0)
        const_cast<double*>(KP->q_in)[static_cast<size_t>(c.env) * KP->nq + 2] -= zg;
    jb_syncwarp(c);
}

// Device-side controller block: gym_jiminy.common.blocks.pd_controller
// (python/gym_jiminy/common/gym_jiminy/common/blocks/proportional_derivative_controller.py:101-165)
// for a zero-order-held position target and zero target velocity,
//     tau = clip(kp * ((q_des - q_enc) + kd * (0 - v_enc)), +-effort_limit),
// evaluated on the motor-side encoder data of the accepted state at every controller breakpoint.
// The action buffer (`command`) holds the targets; the torque goes to the CMD field of the record.
// gym_jiminy `integrate_zoh` (blocks/proportional_derivative_controller.py:24-98) for one motor
JB_DI void integrate_zoh_1(double& position, double& velocity, double& acceleration, double position_min, double position_max,
                           double velocity_min, double velocity_max, double acceleration_min, double acceleration_max, double dt) {
    if (fabs(dt) < 1e-9) return;
    acceleration = fmin(fmax(acceleration, acceleration_min), acceleration_max);
    const double velocity_prev = velocity;
    velocity += acceleration * dt;
    velocity = fmin(fmax(velocity, velocity_min), velocity_max);
    const double horizon = fmax(static_cast<double>(static_cast<long long>(fabs(velocity_prev) / acceleration_max / dt)) * dt, dt);
    double position_min_delta = position_min - position, position_max_delta = position_max - position;
    if (horizon > dt) {
        const double drift = 0.5 * (horizon * (horizon - dt)) * acceleration_max;
        position_min_delta -= drift;
        position_max_delta += drift;
    }
    velocity = fmin(fmax(velocity, position_min_delta / horizon), position_max_delta / horizon);
    if (fabs(velocity) > dt * acceleration_max) {
        const double vmin = -fmax(position_min_delta / velocity, dt) * acceleration_max;
        const double vmax = fmax(position_max_delta / velocity, dt) * acceleration_max;
        velocity = fmin(fmax(velocity, vmin), vmax);
    }
    acceleration = (velocity - velocity_prev) / dt;
    position += dt * velocity;
}

// Controller update.  Two device-side blocks: the plain PD law on a held position target (jb_set_pd_controller), or
// gym_jiminy's PDController block -- integrate_zoh + pd_controller, optionally followed by MotorSafetyLimit's
// apply_safety_limits (jb_set_pd_controller_full).  `running` = false inside Engine::start (control_dt = 0 and the
// targets restart from the clipped measurement, proportional_derivative_controller.py:510-535).
__device__ __noinline__ void update_pd_commands(const Ctx c, bool running) {
    const int L = KP->L, nm = KP->nmotors;
    for (int r = 0; r < KP->nrec; ++r) {
        const RecInt* ri = KP->rint + (r * L + c.sub);
        if (ri->kind == REC_PAD || ri->kind == REC_FREE || ri->motor < 0) continue;
        const RecDbl* rd = JB_RDBL + (r * L + c.sub);
        const int base = KP->rec_off[r];
        double* const rp = jb_smem + base * 32 + c.lane;
        const double red = rd->motor[0], lim = rd->motor[1];
        const double pos = (ri->kind == REC_REVU) ? atan2(RP(R1_Q + 1), RP(R1_Q)) : RP(R1_Q);
        const double q_enc = pos * red, v_enc = RP(R1_V) * red;
        const int m = ri->motor;
        const double action = KP->command[static_cast<size_t>(c.env) * nm + m];
        if (KP->pdf != nullptr) {
            const double* P = KP->pdf;
            double* st = KP->pdf_state + static_cast<size_t>(c.env) * 3 * nm;
            double p = st[m], v = st[nm + m], a = action;
            if (!running) {
                p = fmin(fmax(q_enc, P[2 * nm + m]), P[5 * nm + m]);
                v = fmin(fmax(v_enc, P[3 * nm + m]), P[6 * nm + m]);
            }
            integrate_zoh_1(p, v, a, P[2 * nm + m], P[5 * nm + m], P[3 * nm + m], P[6 * nm + m], P[4 * nm + m], P[7 * nm + m],
                            running ? KP->opt.controller_update_period : 0.0);
            // parked in fields that are free between integrator steps; written back once every lane has read its inputs
            // (trunk motors are evaluated by all the lanes of the env)
            RP(R1_SV) = p; RP(R1_SA) = v; RP(R1_U) = a;
            double tau = P[m] * ((p - q_enc) + P[nm + m] * (v - v_enc));
            tau = fmin(fmax(tau, -lim), lim);
            if (KP->pdf_safety) {
                const double* S = P + 8 * nm;
                const double vlim = S[4 * nm + m];     // min(motor velocity limit, reduction * soft_velocity_max)
                const double sv_lo = vlim * fmin(fmax(-S[m] * (q_enc - S[2 * nm + m]), -1.0), 1.0);
                const double sv_hi = vlim * fmin(fmax(-S[m] * (q_enc - S[3 * nm + m]), -1.0), 1.0);
                const double se_lo = lim * fmin(fmax(-S[nm + m] * (v_enc - sv_lo), -1.0), 1.0);
                const double se_hi = lim * fmin(fmax(-S[nm + m] * (v_enc - sv_hi), -1.0), 1.0);
                tau = fmin(fmax(tau, se_lo), se_hi);
            }
            RP(R1_CMD) = tau;
            continue;
        }
        const double tau = KP->pd_gains[m] * ((action - q_enc) + KP->pd_gains[nm + m] * (0.0 - v_enc));
        RP(R1_CMD) = fmin(fmax(tau, -lim), lim);
    }
    if (KP->pdf != nullptr) {
        jb_syncwarp(c);
        double* st = KP->pdf_state + static_cast<size_t>(c.env) * 3 * nm;
        for (int r = 0; r < KP->nrec; ++r) {
            const RecInt* ri = KP->rint + (r * L + c.sub);
            if (ri->kind == REC_PAD || ri->kind == REC_FREE || ri->motor < 0 || !ri->owner || !c.valid) continue;
            const double* rp = jb_smem + KP->rec_off[r] * 32 + c.lane;
            st[ri->motor] = RP(R1_SV); st[nm + ri->motor] = RP(R1_SA); st[2 * nm + ri->motor] = RP(R1_U);
        }
    }
}

// Copy (restore = false) or put back (restore = true) the per-env state of the device-side PDController / MahonyFilter
// blocks, the sensor pipeline and the stacked observation.  Called by every lane of the env; the L lanes share the copy.
__device__ __noinline__ void snapshot_blocks(const Ctx c, const int L, const bool restore) {
    if (restore) jb_syncwarp(c);   // the owner lanes' writes to the live state come first
    if (KP->pdf != nullptr) {
        const size_t n = 3 * static_cast<size_t>(KP->nmotors);
        double* live = KP->pdf_state + static_cast<size_t>(c.env) * n;
        double* snap = KP->pdf_snap + static_cast<size_t>(c.env) * n;
        for (size_t k = c.sub; k < n; k += L) { if (restore) live[k] = snap[k]; else snap[k] = live[k]; }
    }
    if (KP->mahony != nullptr) {
        const size_t n = 10 * static_cast<size_t>(KP->nimu);
        double* live = KP->mahony + static_cast<size_t>(c.env) * n;
        double* snap = KP->mahony_snap + static_cast<size_t>(c.env) * n;
        for (size_t k = c.sub; k < n; k += L) { if (restore) live[k] = snap[k]; else snap[k] = live[k]; }
        if (KP->obsv != nullptr) {
            // observer outputs and the body observer's twist (refresh_observers)
            const size_t m = OBSV_N * static_cast<size_t>(KP->nimu);
            double* lo = KP->obsv + static_cast<size_t>(c.env) * m;
            double* so = KP->obsv_snap + static_cast<size_t>(c.env) * m;
            for (size_t k = c.sub; k < m; k += L) { if (restore) lo[k] = so[k]; else so[k] = lo[k]; }
        }
    }
    if (KP->sp_on) {
        // sensor measurement pipeline: sample counts and generator states (ring slots written by the aborted pass are rewritten)
        int32_t* lc = KP->sp_count + static_cast<size_t>(c.env) * 6;
        int32_t* sc = KP->sp_snap_count + static_cast<size_t>(c.env) * 6;
        for (int k = c.sub; k < 6; k += L) { if (restore) lc[k] = sc[k]; else sc[k] = lc[k]; }
        unsigned long long* lr = KP->sp_rng + static_cast<size_t>(c.env) * KP->sp_nsens;
        unsigned long long* sr = KP->sp_snap_rng + static_cast<size_t>(c.env) * KP->sp_nsens;
        for (int k = c.sub; k < KP->sp_nsens; k += L) { if (restore) lr[k] = sr[k]; else sr[k] = lr[k]; }
    }
    if (KP->stk != nullptr) {
        // stacked observation: frames and refresh counter
        const size_t n = static_cast<size_t>(KP->stk_num) * KP->stk_w;
        double* live = KP->stk + static_cast<size_t>(c.env) * n;
        double* snap = KP->stk_snap + static_cast<size_t>(c.env) * n;
        for (size_t k = c.sub; k < n; k += L) { if (restore) live[k] = snap[k]; else snap[k] = live[k]; }
        if (c.sub == 0) { if (restore) KP->stk_n[c.env] = KP->stk_n_snap[c.env]; else KP->stk_n_snap[c.env] = KP->stk_n[c.env]; }
    }
    jb_syncwarp(c);
}

// The same for the latched values of the profile / process forces with a finite update period (force-carrying hot path):
// an update hit inside a pass that is handed over overwrites the value the replay starts from.
__device__ __noinline__ void snapshot_latched(const Ctx c, const int L, const bool restore) {
    if (restore) jb_syncwarp(c);   // sub-lane 0 wrote the live values
    const size_t N = KP->n_pad, col = c.env;
    for (int k = c.sub; k < 6 * (KP->n_prof + KP->n_proc); k += L) {
        const int j = k / 6, i = k % 6;
        const bool prof = j < KP->n_prof;
        if (!((prof ? KP->prof_period[j] : KP->proc_period[j - KP->n_prof]) > D_EPS)) continue;
        double* live = (prof ? KP->prof_latched + static_cast<size_t>(j) * 6 * N
                             : KP->proc_latched + static_cast<size_t>(j - KP->n_prof) * 6 * N) + i * N + col;
        double* snap = KP->latch_snap + (static_cast<size_t>(j) * 6 + i) * N + col;
        if (restore) *live = *snap; else *snap = *live;
    }
    jb_syncwarp(c);
}

__device__ __noinline__ void store_outputs(const Ctx c) {
    if (!c.valid) return;
    const int L = KP->L;
    const size_t N = KP->n_pad, col = c.env;
    for (int r = 0; r < KP->nrec; ++r) {
        const RecInt* ri = KP->rint + (r * L + c.sub);
        if (ri->kind == REC_PAD || !ri->owner) continue;
        const RecDbl* rd = JB_RDBL + (r * L + c.sub);
        const int base = KP->rec_off[r];
        double* const rp = jb_smem + base * 32 + c.lane;
        double* qv = KP->qv_out ? KP->qv_out + col * (KP->nq + KP->nv) : nullptr;
        if (ri->kind == REC_SPH) {
#pragma unroll
            for (int k = 0; k < 4; ++k) { const double x = RP(RF_Q + 3 + k); KP->q[(ri->idx_q + k) * N + col] = x; if (qv) qv[ri->idx_q + k] = x; }
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const double x = RP(RF_V + 3 + k);
                KP->v[(ri->idx_v + k) * N + col] = x; if (qv) qv[KP->nq + ri->idx_v + k] = x;
                KP->a[(ri->idx_v + k) * N + col] = RP(RF_A + 3 + k);
            }
            // RobotState.u: uInternal of the flexibility (engine.cc:3367-3391), rebuilt from the accepted state
            if (KP->eff_u) {
                const double qa[4] = {RP(RF_Q + 3), RP(RF_Q + 4), RP(RF_Q + 5), RP(RF_Q + 6)};
                double angle;
                const V3 aa = quat_log3(qa, angle);
                const double* fx = KP->flex_on ? flex_params<SigDynamicFlex<false, true>>(c, r, L, rd) : rd->motor;
                const V3 t = jlog3_mul(angle, aa, mk(fx[0] * aa.x, fx[1] * aa.y, fx[2] * aa.z));
                KP->eff_u[col * KP->nv + ri->idx_v + 0] = (0.0 - t.x) - fx[3] * RP(RF_V + 3);
                KP->eff_u[col * KP->nv + ri->idx_v + 1] = (0.0 - t.y) - fx[4] * RP(RF_V + 4);
                KP->eff_u[col * KP->nv + ri->idx_v + 2] = (0.0 - t.z) - fx[5] * RP(RF_V + 5);
            }
        } else if (ri->kind == REC_FREE) {
#pragma unroll
            for (int k = 0; k < 7; ++k) { const double x = RP(RF_Q + k); KP->q[(ri->idx_q + k) * N + col] = x; if (qv) qv[ri->idx_q + k] = x; }
#pragma unroll
            for (int k = 0; k < 6; ++k) {
                const double x = RP(RF_V + k);
                KP->v[(ri->idx_v + k) * N + col] = x; if (qv) qv[KP->nq + ri->idx_v + k] = x;
                KP->a[(ri->idx_v + k) * N + col] = RP(RF_A + k);
                if (KP->eff_u) KP->eff_u[col * KP->nv + ri->idx_v + k] = 0.0;
            }
        } else {
            const double q0 = RP(R1_Q), q1 = RP(R1_Q + 1), vv = RP(R1_V);
            KP->q[ri->idx_q * N + col] = q0; if (qv) qv[ri->idx_q] = q0;
            if (ri->kind == REC_REVU) { KP->q[(ri->idx_q + 1) * N + col] = q1; if (qv) qv[ri->idx_q + 1] = q1; }
            KP->v[ri->idx_v * N + col] = vv; if (qv) qv[KP->nq + ri->idx_v] = vv;
            KP->a[ri->idx_v * N + col] = RP(R1_A);
            // RobotState.u = uInternal + uCustom + uTransmission (engine.cc:3694-3702), rebuilt from the
            // accepted state because the backward sweep reuses the U field for `data.u`
            if (KP->eff_u) {
                double u = 0.0;
                if (KP->springs != nullptr && ri->kind != REC_REVU) u = -KP->springs[ri->idx_v] * q0 - KP->springs[KP->nv + ri->idx_v] * vv;
                if (ri->motor >= 0) {
                    double uM, uT;
                    motor_effort(rd, ri->motor_flags, RP(R1_CMD), vv, uM, uT);
                    u += uT;
                }
                // an enabled position-bound constraint reports its multiplier in u / uInternal (engine.cc:3770-3788)
                if (KP->cons_on) {
                    const int kc = KP->jc_of_joint[ri->joint];
                    if (kc >= 0 && CST(cs_joint(kc)) != 0.0) u += CST(cs_joint(kc) + 3);
                }
                KP->eff_u[col * KP->nv + ri->idx_v] = u;
            }
            if (KP->eff_umotor && ri->motor >= 0) KP->eff_umotor[col * KP->nmotors + ri->motor] = RP(R1_UMOTOR);
        }
        if (KP->eff_fext) {
            Mot fext = mzero();
            for (int k = 0; k < ri->ncontact; ++k) {
                const int cs = ri->contact0 + k;
                const ContactSlot* ct = KP->cslots + (cs * L + c.sub);
                const int co = KP->cslot_off + CSLOT_SIZE * cs;
                double* const cp = jb_smem + co * 32 + c.lane;
                const V3 Fl = mk(CO(0), CO(1), CO(2));
                fext.l = fext.l + Fl; fext.a = fext.a + cross(ld3(ct->placement + 9), Fl) + mk(CO(3), CO(4), CO(5));
            }
            add_cached_ext_wrench(c, r, L, fext);
            double* o = KP->eff_fext + (col * KP->njoints + ri->joint) * 6;
            o[0] = fext.l.x; o[1] = fext.l.y; o[2] = fext.l.z; o[3] = fext.a.x; o[4] = fext.a.y; o[5] = fext.a.z;
        }
    }
}

// MODE_DYNAMICS outputs: a, fext, u (all AoS)
__device__ __noinline__ void store_dynamics(const Ctx c) {
    if (!c.valid) return;
    const int L = KP->L;
    const size_t col = c.env;
    for (int r = 0; r < KP->nrec; ++r) {
        const RecInt* ri = KP->rint + (r * L + c.sub);
        if (ri->kind == REC_PAD || !ri->owner) continue;
        const RecDbl* rd = JB_RDBL + (r * L + c.sub);
        const int base = KP->rec_off[r];
        double* const rp = jb_smem + base * 32 + c.lane;
        if (ri->kind == REC_SPH) {
#pragma unroll
            for (int k = 0; k < 3; ++k) KP->a_out[col * KP->nv + ri->idx_v + k] = RP(RF_A + 3 + k);
            if (KP->u_out) {
                const double qa[4] = {RP(RF_QS + 3), RP(RF_QS + 4), RP(RF_QS + 5), RP(RF_QS + 6)};
                double angle;
                const V3 aa = quat_log3(qa, angle);
                const double* fx = KP->flex_on ? flex_params<SigDynamicFlex<false, true>>(c, r, L, rd) : rd->motor;
                const V3 t = jlog3_mul(angle, aa, mk(fx[0] * aa.x, fx[1] * aa.y, fx[2] * aa.z));
                KP->u_out[col * KP->nv + ri->idx_v + 0] = (0.0 - t.x) - fx[3] * RP(RF_VS + 3);
                KP->u_out[col * KP->nv + ri->idx_v + 1] = (0.0 - t.y) - fx[4] * RP(RF_VS + 4);
                KP->u_out[col * KP->nv + ri->idx_v + 2] = (0.0 - t.z) - fx[5] * RP(RF_VS + 5);
            }
        } else if (ri->kind == REC_FREE) {
#pragma unroll
            for (int k = 0; k < 6; ++k) {
                KP->a_out[col * KP->nv + ri->idx_v + k] = RP(RF_A + k);
                if (KP->u_out) KP->u_out[col * KP->nv + ri->idx_v + k] = 0.0;
            }
        } else {
            KP->a_out[col * KP->nv + ri->idx_v] = RP(R1_A);
            if (KP->u_out) {
                double u = 0.0;
                const double q0 = RP(R1_QS), vv = RP(R1_VS);
                if (KP->springs != nullptr && ri->kind != REC_REVU) u = -KP->springs[ri->idx_v] * q0 - KP->springs[KP->nv + ri->idx_v] * vv;
                if (ri->motor >= 0) { double uM, uT; motor_effort(rd, ri->motor_flags, RP(R1_CMD), vv, uM, uT); u += uT; }
                KP->u_out[col * KP->nv + ri->idx_v] = u;
            }
        }
        if (KP->fext_out) {
            Mot fext = mzero();
            for (int k = 0; k < ri->ncontact; ++k) {
                const int cs = ri->contact0 + k;
                const ContactSlot* ct = KP->cslots + (cs * L + c.sub);
                const int co = KP->cslot_off + CSLOT_SIZE * cs;
                double* const cp = jb_smem + co * 32 + c.lane;
                const V3 Fl = mk(CO(0), CO(1), CO(2));
                fext.l = fext.l + Fl; fext.a = fext.a + cross(ld3(ct->placement + 9), Fl) + mk(CO(3), CO(4), CO(5));
            }
            add_cached_ext_wrench(c, r, L, fext);
            double* o = KP->fext_out + (col * KP->njoints + ri->joint) * 6;
            o[0] = fext.l.x; o[1] = fext.l.y; o[2] = fext.l.z; o[3] = fext.a.x; o[4] = fext.a.y; o[5] = fext.a.z;
        }
    }
}

// FAST = true: the product hot path only (MODE_STEP, Euler / RK4, spring-damper contacts, no external forces,
// no enabled constraint).  An env that needs anything else leaves untouched (needs_full raised) and is stepped by the
// full body right behind, inside the same launch (`only_flagged`).
// (host emulation of the CPU test suite only, tests/emul/jb_emul_shim.h: "this lane is through / leaves before the loads
// of its env state"; nothing in the device build)
#ifdef JB_HOST_EMUL
#define JB_EMUL_LOADS_DONE(pass) emul::load_fence_wait(pass)
#define JB_EMUL_LEAVES_EARLY(pass) emul::load_fence_drop(pass)
#else
#define JB_EMUL_LOADS_DONE(pass)
#define JB_EMUL_LEAVES_EARLY(pass)
#endif

// EXT = true (with FAST): the force-carrying hot path of the quadruped signature (env_step_kernel_ext).  Everything the
// full body does for impulse / profile / process forces runs here too: slots zeroed at load, refreshed at every
// scheduler iteration (impulse breakpoints, FSAL repair on a change), process forces before every evaluation.
// FLEX (full body only): the batch has per-env flexibility parameters (env_step_kernel_flex): each start latches the
// env's pending row, and the sweeps read the active rows.
// MODEL: the batch has per-env model rows (env_step_kernel_model): every lane reads its env's own table (the row offset in
// Ctx::flags), a start refuses an env whose last device row was rejected, and the centroidal terms divide by the env's
// total mass.
template <bool FAST, bool EXT = false, bool FLEX = false, bool MODEL = false>
__device__ __forceinline__ void env_step_body(const LaunchArgs& la, const bool only_flagged) {
    static_assert(FAST || !EXT, "external forces on the full body need no instance of their own");
    Ctx c;
    c.lane = threadIdx.x & 31;
    const int L = KP->L;
    c.sub = c.lane % L;
    const int epw = 32 / L;
    const int env_raw = blockIdx.x * epw + c.lane / L;
    c.valid = env_raw < KP->n_env;
    c.env = c.valid ? env_raw : (KP->n_env - 1);
    if constexpr (MODEL) c.flags = (c.env * KP->rdbl_rows) << CTX_ROW_SHIFT;
    else c.flags = KP->n_variants > 1 ? (KP->variant_of_block[blockIdx.x] * KP->rdbl_rows) << CTX_ROW_SHIFT : 0;
    c.gmask = (L == 32) ? 0xffffffffu : (((1u << L) - 1u) << (c.lane - c.sub));
    const size_t N = KP->n_pad, col = c.env;
    const int mode = la.mode;
    int status = KP->status[c.env];

    const bool masked_out = (mode == MODE_START) && la.mask != nullptr && la.mask[c.env] == 0;
    if (masked_out) return;   // whole env (all its lanes) leaves: group masks keep the others safe
    if constexpr (!FAST) {
        // per-env model rows: refused if the last device row for this env was.  Otherwise the launch before this one
        // (latch_model_rows_kernel) has made the pending row the model the episode runs with, grounding included.
        if (MODEL && mode == MODE_START && KP->pem_bad[c.env] != 0) {
            if (c.valid && c.sub == 0) KP->status[c.env] = JB_ENV_NOT_STARTED | JB_ENV_BAD_START;
            return;
        }
        if (mode == MODE_START && la.ground) place_on_ground(c);
        // jb_start_device: the input checks jb_start runs on the host (Engine::start, engine.cc:1007-1037), per env.  An env
        // whose row fails them is not started and writes nothing but its status word.
        if (mode == MODE_START && la.validate) {
            const double* qe = KP->q_in + static_cast<size_t>(c.env) * KP->nq;
            const double* ve = KP->v_in + static_cast<size_t>(c.env) * KP->nv;
            const double* lo = KP->q_bounds;
            const double* hi = KP->q_bounds + KP->nq;
            bool bad = false;
            for (int k = c.sub; k < KP->nq; k += L) {
                const double x = qe[k];
                bad = bad || !(x == x) || D_EPS < x - hi[k] || D_EPS < lo[k] - x;
            }
            for (int k = c.sub; k < KP->nv; k += L) bad = bad || !(ve[k] == ve[k]);
            if (jb_any(c, bad)) {
                if (c.valid && c.sub == 0) KP->status[c.env] = JB_ENV_NOT_STARTED | JB_ENV_BAD_START;
                return;
            }
        }
        // per-env sensor options: the last row jb_set_sensor_options_env_device received for this env was rejected
        if (mode == MODE_START && KP->sp_env_on && KP->sp_env_bad[c.env] != 0) {
            if (c.valid && c.sub == 0) KP->status[c.env] = JB_ENV_NOT_STARTED | JB_ENV_BAD_START;
            return;
        }
        // per-env flexibility parameters: refused if the last device row for this env was, else the pending row becomes
        // the one the episode runs with (setOptions before Engine::reset), before the start's own evaluations
        if (FLEX && mode == MODE_START) {
            if (KP->flex_bad[c.env] != 0) {
                if (c.valid && c.sub == 0) KP->status[c.env] = JB_ENV_NOT_STARTED | JB_ENV_BAD_START;
                return;
            }
            if (c.valid) {
                const size_t o = static_cast<size_t>(c.env) * KP->n_flex * 6;
                for (int k = c.sub; k < 6 * KP->n_flex; k += L) KP->flex_active[o + k] = KP->flex_pending[o + k];
            }
            jb_syncwarp(c);
        }
    }
    if (mode == MODE_STEP && (status & (JB_ENV_NOT_STARTED | JB_ENV_NAN | JB_ENV_ITER_FAILED | JB_ENV_DT_UNDERFLOW | JB_ENV_SOLVER_FAILED))) {
        JB_EMUL_LEAVES_EARLY(FAST ? 0 : 1);
        return;
    }
    int32_t* const needs_full = KP->needs_full + (blockIdx.x * epw + c.lane / L);   // own row, also for padding envs
    if constexpr (FAST) { if (*needs_full != 0) { JB_EMUL_LEAVES_EARLY(0); return; } }
    else if (mode == MODE_STEP && only_flagged && *needs_full == 0) { JB_EMUL_LEAVES_EARLY(1); return; }

    // The stateful device blocks (PDController targets, MahonyFilter) advance inside the launch; an env handed over to
    // the full body is replayed from the top of the step, so the fast body keeps a copy to put back.
    if constexpr (FAST) {
        if (c.valid && (KP->pdf != nullptr || KP->mahony != nullptr || KP->sp_on || KP->stk != nullptr)) snapshot_blocks(c, L, false);
    }
    if constexpr (EXT) {
        if (c.valid && KP->n_prof + KP->n_proc > 0) snapshot_latched(c, L, false);
    }
    // ---------------- load state into the lane records
    for (int r = 0; r < KP->nrec; ++r) {
        const RecInt* ri = KP->rint + (r * L + c.sub);
        if (ri->kind == REC_PAD) continue;
        const int base = KP->rec_off[r];
        double* const rp = jb_smem + base * 32 + c.lane;
        if (mode == MODE_STEP) load_record_state(c, ri, base, KP->q, KP->v, KP->a, N, col);
        else {
            load_record_state_aos(c, ri, base, KP->q_in, KP->v_in, c.env);
            if (mode == MODE_START) normalize_record(c, ri, base);
        }
        if (!rec_is_big(ri->kind)) {
            // torque command: the action itself, or (PD mode) the torque held since the last breakpoint
            const double* cmd_src = ((KP->pd_gains != nullptr || KP->pdf != nullptr) && mode == MODE_STEP) ? KP->cmd_torque
                                    : ((mode == MODE_DYNAMICS && la.command != nullptr) ? la.command : KP->command);
            RP(R1_CMD) = (ri->motor >= 0) ? cmd_src[col * KP->nmotors + ri->motor] : 0.0;
            RP(R1_UMOTOR) = 0.0;
        }
    }
    for (int k = 0; k < CSLOT_SIZE * KP->ncslot; ++k) SMF(c, KP->cslot_off + k) = 0.0;
    for (int k = 0; k < IMUSLOT_SIZE * KP->nimuslot; ++k) SMF(c, KP->imu_off + k) = 0.0;
    if constexpr (FAST) {
        if (KP->fast_bounds_io) {
            // joint-bound constraint state of this lane's leg joints (persistent in cstate like the reference's constraint objects)
            for (int r = 1; r < 4; ++r) {
                const int o = cs_joint(KP->jc_of_joint[(KP->rint + (r * L + c.sub))->joint]);
                double* const rp = jb_smem + KP->rec_off[r] * 32 + c.lane;
                RP(R1_BEN) = CST(o); RP(R1_BREV) = CST(o + 1); RP(R1_BQREF) = CST(o + 2); RP(R1_BLAM) = CST(o + 3);
            }
            SMF(c, KP->rec_off[1] + R1_BFAIL) = CST(CS_SOLVE_FAILED);
        }
    }
    if constexpr (!FAST || EXT) {
        for (int k = 0; k < ESLOT_SIZE * KP->n_eslot; ++k) SMF(c, KP->ext_off + k) = 0.0;
    }
    if constexpr (!FAST) {
        if (KP->cons_on) {
            if (mode == MODE_STEP) cons_load_count(c);
            else SMF(c, KP->cons_off) = 0.0;
        }
    }

    if (!FAST && mode == MODE_DYNAMICS) {
        stage_from_accepted(c);
        int st = 0;
        rhs<FLEX>(c, false, &st);
        store_dynamics(c);
        return;
    }

    double t, dt, dtLargest, dtLargestPrev, tError, tPrev;
    long long iter, iterFailed;
    if (!FAST && mode == MODE_START) {
        // Engine::start (engine.cc:952-1533): stepperState_.reset(SIMULATION_MIN_TIMESTEP, ...), forward
        // kinematics, initial contact-force guard, then the INIT_ITERATIONS fixed point, which for a
        // zero-order-held command converges to one evaluation of the dynamics.
        status = JB_ENV_OK;
        t = 0.0; tPrev = 0.0; tError = 0.0;
        dt = SIMULATION_MIN_TIMESTEP; dtLargest = dt; dtLargestPrev = dt;
        iter = 0; iterFailed = 0;
        if (KP->pd_gains != nullptr || KP->pdf != nullptr) update_pd_commands(c, false);
        if (KP->n_eslot > 0) { bool ch = false; refresh_external_forces(c, 0.0, true, false, ch); }
        if (KP->n_proc > 0) eval_process_forces(c, 0.0);
        stage_from_accepted(c);
        if (KP->cons_on) {
            // resetConstraints, then the INIT_ITERATIONS fixed point of engine.cc:1400-1467: the first evaluation sees
            // zero joint efforts and solves the enabled constraints as equalities, the next three run the boxed
            // solver warm-started on an up-to-date state
            cons_reset(c);
            Ctx c0 = c; c0.flags |= CTX_ZERO_U | CTX_IGNORE_BOUNDS;
            rhs<FLEX>(c0, false, &status);
            const bool constrained = jb_any(c, SMF(c, KP->cons_off) != 0.0);
            Ctx c1 = c; c1.flags |= CTX_START_FEEDBACK;
            for (int it = 1; it < (constrained ? 4 : 2); ++it) rhs<FLEX>(c1, true, &status);
        } else rhs<FLEX>(c, false, &status);
        // forceMax > 1e5 guard (engine.cc:1310-1346)
        double fmax2 = 0.0;
        for (int k = 0; k < KP->ncslot; ++k) {
            const int co = KP->cslot_off + CSLOT_SIZE * k;
            double* const cp = jb_smem + co * 32 + c.lane;
            const double fx = CO(0), fy = CO(1), fz = CO(2);
            fmax2 = fmax(fmax2, fx * fx + fy * fy + fz * fz);
        }
        for (int o = 1; o < L; o <<= 1) fmax2 = fmax(fmax2, jb_shfl_xor(c, fmax2, o));
        if (fmax2 > 1e10) status |= JB_ENV_CONTACT_FORCE | JB_ENV_NOT_STARTED;
        bool bad = accel_has_nan(c);
        bad = jb_any(c, bad);
        if (bad) status |= JB_ENV_NAN;
        write_sensors(c, true, 0.0, 0.0, 0.0);
    } else {
        t = KP->sched[SCH_T * N + col]; dt = KP->sched[SCH_DT * N + col];
        dtLargest = KP->sched[SCH_DTLARGEST * N + col]; dtLargestPrev = KP->sched[SCH_DTLARGESTPREV * N + col];
        tError = KP->sched[SCH_TERROR * N + col]; tPrev = KP->sched[SCH_TPREV * N + col];
        iter = KP->iters[col]; iterFailed = KP->iters[N + col];
        JB_EMUL_LOADS_DONE(FAST ? 0 : 1);

        // ------------- Engine::step (engine.cc:1724-2417)
        const JbOptions& opt = KP->opt;
        double stepSize = la.step_dt;
        if (stepSize < D_EPS) {
            if (opt.controller_update_period > D_EPS) stepSize = opt.controller_update_period;
            else if (opt.sensors_update_period > D_EPS) stepSize = opt.sensors_update_period;
            else stepSize = opt.dt_max;
        }
        // Kahan-compensated end time (engine.cc:1793-1795)
        const double stepSizeCorrected = stepSize - tError;
        const double tEnd = t + stepSizeCorrected;
        tError = (tEnd - t) - stepSizeCorrected;
        const double supd = KP->stepper_update_period;
        const bool finitePeriod = supd < 1e300;
        const int failedMax = opt.successive_iter_failed_max;
        int successiveIterTooLarge = 0, successiveIterFailed = 0;
        bool hasDynamicsChanged = false;
        bool failed = false;
        // Shared memory does not persist between launches: the first evaluation of this launch is a
        // full one (it rebuilds the cached contact forces, a pure function of the accepted state).
        bool need_refresh = true;
        // fsal_linear: the last evaluation was the FSAL stage of a one-call RK4 step of the quadruped hot path, at the
        // accepted state, and its block factors of M are still in shared memory -- the FSAL repair of a controller update
        // is then linear (repair_quadruped_crba).  The PDController block parks its state in the U fields that hold
        // M_ll^-1, and the force-carrying kernel can change its slots at the breakpoint: both keep the full evaluation.
        bool fsal_linear = false;
        bool fsal_linear_on = false;
        if constexpr (FAST && !EXT) {
            fsal_linear_on = KP->sig_id == SigQuadruped::ID && KP->quad_stage && KP->pdf == nullptr &&
                             opt.ode_solver != JB_SOLVER_EULER_EXPLICIT;
        }

        // stepper_->tryStep (abstract_stepper.cc:16-62) + the success / failure bookkeeping of
        // engine.cc:2132-2221.  rc: 0 success, 1 failure (adaptive step rejected), 2 error (NaN).
        auto try_step = [&](bool isBreakpointReached) {
            const double t_next = t + dtLargest;
            int rc = 0;
            // successive constraint-solver failures are rolled back with a failed step (engine.cc:2104-2112, :2211-2217)
            double solveFailedBackup = 0.0;
            if constexpr (!FAST) {
                if (KP->cons_on) solveFailedBackup = CST(CS_SOLVE_FAILED);
            }
            if constexpr (!FAST || EXT) {
                if (KP->n_proc > 0) SMF(c, proc_time_field()) = t;   // stage times of the process forces
            }
            JB_PROF_T(t_stepper);
            if (opt.ode_solver == JB_SOLVER_EULER_EXPLICIT) { step_euler<FAST, EXT, FLEX>(c, dtLargest, &status); dtLargest = D_INF; }
            else if (FAST || opt.ode_solver == JB_SOLVER_RUNGE_KUTTA_4) { step_rk4<FAST, EXT, FLEX>(c, dtLargest, &status); dtLargest = D_INF; }
            else { if constexpr (!FAST) rc = step_dopri<FLEX>(c, &dtLargest, &status); }
            if constexpr (FAST) { JB_PROF_ADD(16, t_stepper); JB_PROF_COUNT(21, 1); }   // hot path: stepper calls (RK4: four stage calls)
            need_refresh = false;
            fsal_linear = fsal_linear_on;
            if constexpr (FAST) {
                // one vote for the two rare events of a step: NaN in the new acceleration, or a joint that left its
                // position bounds (this env is then re-done by the full kernel)
                const bool bad = accel_has_nan<EXT>(c), retry = (status & ENV_RETRY_FULL) != 0;
                if (jb_any(c, bad || retry)) {
                    if (jb_any(c, retry)) { status |= ENV_RETRY_FULL; failed = true; }
                    if (jb_any(c, bad)) rc = 2;
                }
            } else if (rc == 0 && opt.ode_solver != JB_SOLVER_RUNGE_KUTTA_DOPRI) {
                bool bad = accel_has_nan(c);
                bad = jb_any(c, bad);
                if (bad) rc = 2;
            }
            if (rc == 0) {
                successiveIterTooLarge = 0; successiveIterFailed = 0;
                t = t_next;
                ++iter;
                if (isBreakpointReached) {
                    const double thr = dtLargestPrev * opt.dt_restore_threshold_rel;
                    if (dt < dtLargest && dtLargest < thr) dtLargest = dtLargestPrev;
                }
                tPrev = t;
                dtLargestPrev = dtLargest;
            } else {
                if (rc == 2) {
                    dtLargest *= 0.1;
                    // a fixed-step stepper that produced NaN has no smaller step to fall back to
                    if (opt.ode_solver != JB_SOLVER_RUNGE_KUTTA_DOPRI) { status |= JB_ENV_NAN; failed = true; }
                }
                if (rc == 1) ++successiveIterTooLarge;
                ++successiveIterFailed;
                ++iterFailed;
                if constexpr (!FAST) { if (KP->cons_on && c.sub == 0) CST(CS_SOLVE_FAILED) = solveFailedBackup; }
            }
            dt = fmin(dtLargest, opt.dt_max);
            return rc;
        };

        while (tEnd - t >= STEPPER_MIN_TIMESTEP && !failed) {
            double tNext = t;
            // impulse forces: active set + next breakpoint; profile forces: held values (engine.cc:1843-1917)
            double tImpulseForceNext = D_INF;
            if constexpr (!FAST || EXT) { if (KP->n_eslot > 0) tImpulseForceNext = refresh_external_forces(c, t, false, finitePeriod, hasDynamicsChanged); }
            if (finitePeriod && opt.controller_update_period > D_EPS) {
                if (period_hit(t, opt.controller_update_period)) {
                    // computeCommand (engine.cc:1920-1940): zero-order hold of the action, or the PD block
                    JB_PROF_T(t_cmd);
                    if (KP->pd_gains != nullptr || KP->pdf != nullptr) update_pd_commands(c, true);
                    if constexpr (FAST) JB_PROF_ADD(17, t_cmd);   // hot path: controller update at a breakpoint
                    hasDynamicsChanged = true;
                }
            }
            if (!finitePeriod && hasDynamicsChanged) {
                stage_from_accepted<EXT>(c);
                if constexpr (!FAST || EXT) { if (KP->n_proc > 0) eval_process_forces(c, t); }
                if constexpr (EXT) rhs_fast_ext(c, !need_refresh, &status);
                else if constexpr (FAST) rhs_fast(c, !need_refresh, &status); else rhs<FLEX>(c, !need_refresh, &status);
                need_refresh = false;
                hasDynamicsChanged = false;
            }
            if (finitePeriod) {
                double dtNextGlobal;
                const double dtNextUpdatePeriod = supd - fmod(t, supd);
                if (dtNextUpdatePeriod < SIMULATION_MIN_TIMESTEP) dtNextGlobal = fmin(dtNextUpdatePeriod + supd, tImpulseForceNext - t);
                else dtNextGlobal = fmin(dtNextUpdatePeriod, tImpulseForceNext - t);
                if (tEnd - t - STEPPER_MIN_TIMESTEP < dtNextGlobal) dtNextGlobal = tEnd - t;
                tNext += dtNextGlobal;
                while (tNext - t > STEPPER_MIN_TIMESTEP && !failed) {
                    if (hasDynamicsChanged) {
                        // FSAL repair: same state, cached contact forces, new command (engine.cc:2032-2037)
                        JB_PROF_T(t_repair);
                        bool repaired = false;
                        if constexpr (FAST && !EXT) repaired = fsal_linear && repair_quadruped_crba(c);
                        if (!repaired) {
                            stage_from_accepted<EXT>(c);
                            if constexpr (!FAST || EXT) { if (KP->n_proc > 0) eval_process_forces(c, t); }
                            if constexpr (EXT) rhs_fast_ext(c, !need_refresh, &status);
                            else if constexpr (FAST) rhs_fast(c, !need_refresh, &status); else rhs<FLEX>(c, !need_refresh, &status);
                        }
                        need_refresh = false;
                        hasDynamicsChanged = false;
                        if constexpr (FAST) { JB_PROF_ADD(18, t_repair); JB_PROF_COUNT(19, 1); }   // hot path: FSAL repairs
                    }
                    if (dt < STEPPER_MIN_TIMESTEP) break;
                    double dtResidualThr = STEPPER_MIN_TIMESTEP;
                    if (successiveIterTooLarge == 0) dtResidualThr = fmin(fmax(0.1 * dt, STEPPER_MIN_TIMESTEP), SIMULATION_MIN_TIMESTEP);
                    if (tNext - t < dt || (successiveIterTooLarge <= 1 && tNext - t < dt + dtResidualThr)) dt = tNext - t;
                    if (dt > SIMULATION_MIN_TIMESTEP) {
                        const double dtResidual = fmod(dt, SIMULATION_MIN_TIMESTEP);
                        if (dtResidual > STEPPER_MIN_TIMESTEP && dtResidual < SIMULATION_MIN_TIMESTEP - STEPPER_MIN_TIMESTEP &&
                            dt - dtResidual > STEPPER_MIN_TIMESTEP)
                            dt -= dtResidual;
                    }
                    if (successiveIterFailed > failedMax) break;
                    const bool isBreakpointReached = (dtLargest > dt);
                    dtLargest = dt;
                    try_step(isBreakpointReached);
                }
            } else {
                dt = fmin(fmin(dt, tEnd - t), tImpulseForceNext - t);
                const bool isBreakpointReached = (dtLargest > dt);
                bool isStepSuccessful = false;
                while (!isStepSuccessful && !failed) {
                    if (successiveIterFailed > failedMax) break;
                    dtLargest = dt;
                    isStepSuccessful = (try_step(isBreakpointReached) == 0);
                }
            }
            if (failed) break;
            if (successiveIterFailed > failedMax) { status |= JB_ENV_ITER_FAILED; failed = true; break; }
            if constexpr (!FAST) {
                if (KP->cons_on && jb_any(c, c.sub == 0 && CST(CS_SOLVE_FAILED) > failedMax)) { status |= JB_ENV_SOLVER_FAILED; failed = true; break; }
            } else if (KP->fast_bounds) {
                if (jb_any(c, SMF(c, KP->rec_off[1] + R1_BFAIL) > failedMax)) { status |= JB_ENV_SOLVER_FAILED; failed = true; break; }
            }
            if (dt < STEPPER_MIN_TIMESTEP) { status |= JB_ENV_DT_UNDERFLOW; failed = true; break; }
            // sensors refresh (engine.cc:2386-2410)
            const double sp = opt.sensors_update_period;
            bool mustUpdateSensors = sp < D_EPS;
            if (!mustUpdateSensors) mustUpdateSensors = period_hit(t, sp);
            JB_PROF_T(t_sensors);
            // (the observer of the env-step's last refresh sees the env's end time, as after the step)
            if (mustUpdateSensors) write_sensors(c, false, t, tEnd - t >= STEPPER_MIN_TIMESTEP ? t : tEnd, stepSize);
            if constexpr (FAST) JB_PROF_ADD(20, t_sensors);   // hot path: sensor refresh
        }
        if (!failed) t = tEnd;
    }

    // ---------------- store
    if constexpr (FAST) {
        if (jb_any(c, (status & ENV_RETRY_FULL) != 0)) {   // nothing of this pass is kept: the full body redoes the env
            if (c.valid && (KP->pdf != nullptr || KP->mahony != nullptr || KP->sp_on || KP->stk != nullptr)) snapshot_blocks(c, L, true);
            if constexpr (EXT) { if (c.valid && KP->n_prof + KP->n_proc > 0) snapshot_latched(c, L, true); }
            if (c.sub == 0) *needs_full = 1;
            return;
        }
    } else if (KP->cons_on) {
        // envs that still own enabled constraints stay with the full body
        const bool any = jb_any(c, SMF(c, KP->cons_off) != 0.0);
        // (the hot-path evaluation of the quadruped signature solves joint bounds itself: nothing to keep the env here for)
        if (c.sub == 0) *needs_full = (any && !(KP->fast_bounds && KP->opt.contact_model == JB_CONTACT_SPRING_DAMPER)) ? 1 : 0;
    } else if (c.sub == 0) *needs_full = 0;   // bounds are only flagged for this robot (JB_ENV_JOINT_LIMIT): back to the hot path
    if constexpr (FAST) {
        if (KP->fast_bounds_io && c.valid) {
            bool any_en = false;
            for (int r = 1; r < 4; ++r) {
                const int o = cs_joint(KP->jc_of_joint[(KP->rint + (r * L + c.sub))->joint]);
                const double* const rp = jb_smem + KP->rec_off[r] * 32 + c.lane;
                CST(o) = RP(R1_BEN); CST(o + 1) = RP(R1_BREV); CST(o + 2) = RP(R1_BQREF); CST(o + 3) = RP(R1_BLAM);
                any_en = any_en || RP(R1_BEN) != 0.0;
            }
            if (c.sub == 0) CST(CS_SOLVE_FAILED) = SMF(c, KP->rec_off[1] + R1_BFAIL);
        }
    }
    if (KP->extra_energy != nullptr && !(status & (JB_ENV_NAN | JB_ENV_NOT_STARTED))) extra_terms<MODEL>(c);
    store_outputs(c);
#ifndef JB_HOST_EMUL
    // multi-GPU: publish the sensor rows into every rank's gathered buffer (stores over NVLink / NVSwitch).  The rows
    // of a warp's envs are contiguous: when the whole warp is here it copies them with coalesced 16-byte stores,
    // otherwise (some env of the warp failed or was handed to the full kernel) every env copies its own row.
    if (la.peer_on) {
        const int width = KP->lay.width;
        const size_t slot = (static_cast<size_t>(la.peer_parity) * KP->peer_n + KP->peer_rank) * KP->n_env;
        const unsigned act = __activemask();
        if (act == 0xffffffffu && (width & 1) == 0) {
            __syncwarp();
            const int env0 = blockIdx.x * epw;
            const int nrow = min(epw, KP->n_env - env0);
            const int n2 = nrow * width / 2;
            const double2* src = reinterpret_cast<const double2*>(KP->sensors + static_cast<size_t>(env0) * width);
            for (int p = 0; p < KP->peer_n; ++p) {
                double2* out = reinterpret_cast<double2*>(KP->peer_obs[p] + (slot + env0) * width);
                for (int i = c.lane; i < n2; i += 32) out[i] = src[i];
            }
        } else if (c.valid) {
            jb_syncwarp(c);   // the row was written by the owner lanes of the env
            const double* row = KP->sensors + col * width;
            for (int p = 0; p < KP->peer_n; ++p) {
                double* out = KP->peer_obs[p] + (slot + col) * width;
                for (int k = c.sub; k < width; k += L) out[k] = row[k];
            }
        }
    }
#endif
    if ((KP->pd_gains != nullptr || KP->pdf != nullptr) && c.valid) {
        for (int r = 0; r < KP->nrec; ++r) {
            const RecInt* ri = KP->rint + (r * L + c.sub);
            if (ri->kind == REC_PAD || ri->kind == REC_FREE || ri->motor < 0 || !ri->owner) continue;
            KP->cmd_torque[col * KP->nmotors + ri->motor] = SMF(c, KP->rec_off[r] + R1_CMD);
        }
    }
    if (c.valid && c.sub == 0) {
        KP->sched[SCH_T * N + col] = t; KP->sched[SCH_DT * N + col] = dt;
        KP->sched[SCH_DTLARGEST * N + col] = dtLargest; KP->sched[SCH_DTLARGESTPREV * N + col] = dtLargestPrev;
        KP->sched[SCH_TERROR * N + col] = tError; KP->sched[SCH_TPREV * N + col] = tPrev;
        KP->iters[col] = iter; KP->iters[N + col] = iterFailed;
    }
    // status bits can be raised by any lane of the env
    for (int o = 1; o < L; o <<= 1) status |= jb_shfl_xor(c, status, o);
    if (c.valid && c.sub == 0) KP->status[c.env] = status;
}

JB_DI unsigned int jb_smid() {
#ifdef JB_HOST_EMUL
    return 0u;
#else
    unsigned int id;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(id));
    return id;
#endif
}

// The full body: every mode, every stepper, the constraint path.  Out of line, so that the hot-path kernel carries one
// call to it instead of a second copy of the code.
template <bool FLEX = false, bool MODEL = false>
__device__ __noinline__ void env_step_full(const LaunchArgs la, const bool only_flagged) {
    // constraint workspace of this block: one row per block of the launch.  (A pool of per-SM slots taken with an atomic
    // spin by lane 0 kept the workspace L2-resident, but left the warp's env groups running one after the other in the
    // constraint solvers -- several times slower on ANYmal with constraint contacts.)
    if (threadIdx.x == 0) jb_cw_slot = static_cast<int>(blockIdx.x);
    __syncwarp();
    env_step_body<false, false, FLEX, MODEL>(la, only_flagged);
}

// One launch = one Engine::step (or start / single evaluation) of every env.  FAST: the hot-path body first; the envs it
// handed over (a joint left its bounds now, or constraints still enabled from an earlier step) go through the full
// body in the same launch, so a step is always exactly one kernel.  EXT: the hot-path body is the force-carrying one.
template <bool FAST, bool EXT, bool FLEX = false, bool MODEL = false>
__device__ __forceinline__ void env_step_launch(const LaunchArgs& la) {
    JB_PROF_T(t_kernel);
    if constexpr (FAST) {
        env_step_body<true, EXT, false, MODEL>(la, false);
        __syncwarp();   // needs_full is written by sub-lane 0 of each env
        const int flag = KP->needs_full[blockIdx.x * (32 / KP->L) + (threadIdx.x & 31) / KP->L];
        if (__any_sync(0xffffffffu, flag != 0)) env_step_full<false, MODEL>(la, true);
    } else env_step_full<FLEX, MODEL>(la, false);
    JB_PROF_ADD(6, t_kernel);                              // the whole kernel
    JB_PROF_COUNT(7, 1);                                   // warps
#ifndef JB_HOST_EMUL
    // observation exchange over peer memory: EVERY block arrives here, whatever its envs did; the last one tells the
    // other ranks that every row of this rank has been published (release: fence, then the flags)
    if (la.peer_on) {
        __syncwarp();
        if (threadIdx.x == 0) {
            __threadfence_system();
            const unsigned int done = atomicAdd(KP->peer_counter, 1u);
            if (done == gridDim.x - 1) {
                *KP->peer_counter = 0u;
                __threadfence_system();
                for (int p = 0; p < KP->peer_n; ++p) KP->peer_flags[p][la.peer_parity * KP->peer_n + KP->peer_rank] = la.peer_step;
            }
        }
    }
#endif
}
template <bool FAST>
__global__ void __launch_bounds__(32) env_step_kernel_t(const LaunchArgs la) { env_step_launch<FAST, false>(la); }
// Batches of the quadruped signature with external forces (composite-rigid-body evaluation, spring-damper contacts,
// Euler / RK4): the forces ride the hot path, the envs it hands over run the full body's force-aware generic sweeps.
__global__ void __launch_bounds__(32) env_step_kernel_ext(const LaunchArgs la) { env_step_launch<true, true>(la); }
// Batches with per-env flexibility parameters (jb_enable_per_env_flexibility): every launch runs the full body with the
// sweep instances that read the env's active rows (SigDynamicFlex), so the kernels above are not touched.
__global__ void __launch_bounds__(32) env_step_kernel_flex(const LaunchArgs la) { env_step_launch<false, false, true>(la); }
// Batches with per-env model rows (jb_enable_per_env_model): the four kernels above, with every env reading its own
// table and its own total mass (MODEL).  The kernels above are not touched.
__global__ void __launch_bounds__(32) env_step_kernel_model_fast(const LaunchArgs la) { env_step_launch<true, false, false, true>(la); }
__global__ void __launch_bounds__(32) env_step_kernel_model_ext(const LaunchArgs la) { env_step_launch<true, true, false, true>(la); }
__global__ void __launch_bounds__(32) env_step_kernel_model(const LaunchArgs la) { env_step_launch<false, false, false, true>(la); }
__global__ void __launch_bounds__(32) env_step_kernel_model_flex(const LaunchArgs la) { env_step_launch<false, false, true, true>(la); }

// jb_contact_positions_device: world position of every contact frame of every env, out[env][contact][3], from the
// accepted state (the SoA q of the last start / step), by the forward sweep of place_on_ground on the env's own model
// (its variant's table, or its own table with per-env model rows).  Same lane layout and shared memory as the step
// kernels; a kernel of its own, so that they are not touched.  Envs that are not started or carry NaN read NaN.
__global__ void __launch_bounds__(32) contact_positions_kernel(double* __restrict__ out, int ncontacts) {
    Ctx c;
    c.lane = threadIdx.x & 31;
    const int L = KP->L;
    c.sub = c.lane % L;
    const int env_raw = blockIdx.x * (32 / L) + c.lane / L;
    c.valid = env_raw < KP->n_env;
    c.env = c.valid ? env_raw : (KP->n_env - 1);
    if (KP->pem_on) c.flags = (c.env * KP->rdbl_rows) << CTX_ROW_SHIFT;
    else c.flags = KP->n_variants > 1 ? (KP->variant_of_block[blockIdx.x] * KP->rdbl_rows) << CTX_ROW_SHIFT : 0;
    c.gmask = (L == 32) ? 0xffffffffu : (((1u << L) - 1u) << (c.lane - c.sub));
    double* const o = out + static_cast<size_t>(c.env) * ncontacts * 3;
    if (KP->status[c.env] & (JB_ENV_NOT_STARTED | JB_ENV_NAN)) {
        if (c.valid) for (int k = c.sub; k < 3 * ncontacts; k += L) o[k] = D_NAN;
        return;
    }
    for (int r = 0; r < KP->nrec; ++r) {
        const RecInt* ri = KP->rint + (r * L + c.sub);
        if (ri->kind != REC_PAD) load_record_state(c, ri, KP->rec_off[r], KP->q, KP->v, nullptr, KP->n_pad, c.env);
    }
    // a trunk contact sits in the slots of every lane of the env, with the same bits in each: every one of them writes it
    contact_frame_sweep(c, [&](const ContactSlot* ct, const V3& p) {
        if (!c.valid || ct->contact < 0) return;
        double* const x = o + 3 * ct->contact;
        x[0] = p.x; x[1] = p.y; x[2] = p.z;
    });
}

// ---- observation exchange over peer memory: the consumer's wait (one thread)
#ifndef JB_HOST_EMUL
// `timed_out` is host-mapped: the host checks it at its next synchronisation point (JB_ERR_PEER_TIMEOUT).
__global__ void peer_wait_kernel(volatile long long* mine, int world, int parity, long long step, long long timeout_cycles,
                                 volatile int* timed_out) {
    const long long t0 = clock64();
    for (int p = 0; p < world; ++p)
        while (mine[parity * world + p] < step)
            if (clock64() - t0 > timeout_cycles) { *timed_out = p + 1; __threadfence_system(); return; }   // rank p never signalled
    __threadfence_system();
}
#endif

}  // namespace jb
