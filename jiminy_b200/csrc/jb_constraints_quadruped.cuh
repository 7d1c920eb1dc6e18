// jiminy_b200 -- structured constraint solve for quadruped-shaped plans (ANYmal): L = 4, one trunk free-flyer,
// a chain of three revolute joints per lane with one contact frame on the last one.
//
// Same mathematics as jb_constraints.cuh (Engine::computeAcceleration with enabled constraints,
// core/src/engine/engine.cc:3709-3866; PGSSolver, core/src/solver/constraint_solvers.cc:107-448), but the
// joint-space inertia is never formed as a dense matrix.  With the dofs ordered (trunk | leg 0 | ... | leg 3)
//       M = [ M_tt   M_t0 ... M_t3 ]        legs couple only through the trunk (branch-induced sparsity), so
//           [ M_0t   M_00          ]          M^-1 = blockdiag(0, M_ll^-1) + [1; -W] S^-1 [1, -W^T],
//           [  ...         ...     ]          W_l = M_ll^-1 M_lt ,  S = M_tt - sum_l M_tl W_l   (6 x 6)
// and for constraint rows r (owned by lane l(r), Jacobian [J_t | J_l]):
//       A_rs = [l(r) = l(s)] J_l,r M_ll^-1 J_l,s^T + g_r . S^-1 g_s ,   g_r = J_t,r - J_l,r W_l(r).
// Every lane builds its own 3 x 3 block, its W, its rows and g, h = S^-1 g in registers / shared memory; the only
// exchanges between the lanes of an env are one 21-number all-reduce (S) and, inside the Gauss-Seidel sweep,
// the 6-vector z = sum_r g_r lambda_r (A.col(k) . lambda = local part + h_k . z).  The sweep order is the
// reference's (contact frames in registry order, normal / torsion / friction blocks breadth-first).
//
// Handles the common case -- contact constraints only, boxed solve.  Envs with an enabled joint-bound constraint,
// and the first start iteration (equality solve), take the generic path of jb_constraints.cuh.
#pragma once

// The solver needs no shared memory of its own (the occupancy of the step kernel is unchanged): the sweep runs on
// registers, the lanes exchange through shuffles, and the few values that must survive the sweep are parked in
// record fields that are dead between the third ABA sweep and the refresh of the accelerations:
//   W (3 x 6) and M_ll^-1 (6) in the U / Dinv / u fields of the three leg records, the world rotation of the foot
//   joint (9) and J_l (4 x 3) in the trunk's pool entry.
constexpr int CQ_SIZE = 0;
JB_DI double cq_bcast_sum4(const Ctx& c, double x, unsigned mask) {   // sum over the 4 lanes of the env, same order on every lane
    const int l0 = c.lane - c.sub;
    double s = __shfl_sync(mask, x, l0);
    s += __shfl_sync(mask, x, l0 + 1);
    s += __shfl_sync(mask, x, l0 + 2);
    s += __shfl_sync(mask, x, l0 + 3);
    return s;
}
JB_DI double cq_bcast_sum4(const Ctx& c, double x) { return cq_bcast_sum4(c, x, c.gmask); }
// votes among the lanes of the env under either kind of mask (a ballot restricted to the group's bits)
JB_DI bool cq_any(unsigned mask, const Ctx& c, bool p) { return (__ballot_sync(mask, p) & c.gmask) != 0u; }
JB_DI bool cq_all(unsigned mask, const Ctx& c, bool p) { return (__ballot_sync(mask, p) & c.gmask) == c.gmask; }

struct Spd6 { double Ai[6], T[9], Si[6]; };
JB_DI void spd6_factor(const SymY& Y, Spd6& f) {
    sym3_inverse(Y.A, f.Ai);
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        const V3 col = symmul(f.Ai, mk(Y.B[j], Y.B[3 + j], Y.B[6 + j]));
        f.T[j] = col.x; f.T[3 + j] = col.y; f.T[6 + j] = col.z;
    }
    double S[6];
    S[0] = Y.D[0] - (Y.B[0] * f.T[0] + Y.B[3] * f.T[3] + Y.B[6] * f.T[6]);
    S[1] = Y.D[1] - (Y.B[0] * f.T[1] + Y.B[3] * f.T[4] + Y.B[6] * f.T[7]);
    S[2] = Y.D[2] - (Y.B[1] * f.T[1] + Y.B[4] * f.T[4] + Y.B[7] * f.T[7]);
    S[3] = Y.D[3] - (Y.B[0] * f.T[2] + Y.B[3] * f.T[5] + Y.B[6] * f.T[8]);
    S[4] = Y.D[4] - (Y.B[1] * f.T[2] + Y.B[4] * f.T[5] + Y.B[7] * f.T[8]);
    S[5] = Y.D[5] - (Y.B[2] * f.T[2] + Y.B[5] * f.T[5] + Y.B[8] * f.T[8]);
    sym3_inverse(S, f.Si);
}
// x = Y^-1 b with Y = [[A, B], [B^T, D]]:  x2 = Si (b2 - T^T b1) ,  x1 = Ai b1 - T x2
JB_DI Mot spd6_apply(const Spd6& f, Mot b) {
    const V3 r2 = b.a - rtmul(f.T, b.l);
    Mot x;
    x.a = symmul(f.Si, r2);
    x.l = symmul(f.Ai, b.l) - rmul(f.T, x.a);
    return x;
}

// does the plan have the shape this solver assumes?  (host side, at batch creation)
static bool cons_quadruped_matches(const KParams& kp, const Plan& P, const JbModelDesc& m) {
    if (kp.L != 4 || kp.nrec != 4 || kp.ntrunk != 1 || kp.ncslot != 1 || m.ncontacts != 4 || kp.n_hist != 0) return false;
    bool seen[4] = {false, false, false, false};
    for (int s = 0; s < 4; ++s) {
        for (int r = 0; r < 4; ++r) {
            const RecInt& ri = P.rint[static_cast<size_t>(r) * 4 + s];
            if (r == 0) { if (ri.kind != REC_FREE || ri.parent_rec >= 0) return false; continue; }
            if ((ri.kind != REC_REV && ri.kind != REC_REVX) || ri.parent_rec != r - 1) return false;
            if (ri.ncontact != (r == 3 ? 1 : 0)) return false;
        }
        const int k = P.cslots[s].contact;
        if (k < 0 || k >= 4 || seen[k]) return false;
        seen[k] = true;
    }
    return true;
}

// Called by the four lanes of the env after the ABA sweeps, when only contact constraints are enabled.
// UNI (CTX_UNIFORM_WARP): all 32 lanes of the warp are in this call together (decided by the caller): every collective
// below then uses the full mask as a compile-time constant -- a primitive whose mask is a run-time value is compiled into
// a converge-and-retry sequence, one whose mask differs from lane to lane is executed one mask after the other -- and the
// sweep loop keeps every env of the warp inside until the last one has converged
template <bool UNI>
__device__ __noinline__ bool cons_solve_quadruped_t(const Ctx c, int* status) {
    constexpr bool uni = UNI;
    const unsigned M = UNI ? 0xffffffffu : c.gmask;
    JB_PROF_T(t_setup);
    JB_PROF_COUNT(uni ? 10 : 11, 1);                       // solves entered with / without the whole warp
    constexpr int L = 4;
    const JbOptions& opt = KP->opt;
    const RecDbl* rd0 = JB_RDBL + (0 * L + c.sub);
    const ContactSlot* ct = KP->cslots + c.sub;       // contact slot 0 of this lane
    const int kc = ct->contact;                        // contact index == constraint index among the contact frames
    const int cso = cs_contact(kc);
    const bool en = CST(cso) != 0.0;
    __syncwarp(M);
    // ---------------- kinematics along the chain, composite inertias, inertia blocks
    Xf oM; Mot v, aD;
    {
        double* const rp = jb_smem + KP->rec_off[0] * 32 + c.lane;
        sm_load_xf(c, KP->rec_off[0] + RF_LIMI, oM);
        v = sm_load_mot(c, KP->rec_off[0] + RF_VS);
        aD = mzero();
        (void)rp;
    }
    const Xf oM0 = oM;
    V3 wax[3], parm[3];        // world axes and world positions of the three leg joints
#pragma unroll
    for (int i = 1; i <= 3; ++i) {
        const RecDbl* rd = JB_RDBL + (i * L + c.sub);
        const int base = KP->rec_off[i];
        Xf li; sm_load_xf(c, base + R1_LIMI, li);
        Xf o2;
        mat3mul(oM.R, li.R, o2.R);
        o2.p = oM.p + rmul(oM.R, li.p);
        oM = o2;
        const V3 ax = ld3(rd->axis);
        Mot vJ = mzero(); vJ.a = SMF(c, base + R1_VS) * ax;
        v = motion_act_inv(li, v) + vJ;
        aD = sm_load_mot(c, base + R1_BIAS) + motion_act_inv(li, aD);
        wax[i - 1] = rmul(oM.R, ax);
        parm[i - 1] = oM.p;
    }
    // composite-rigid-body recursion from the foot to the trunk; F_i = Yc_i S_i carried up to the trunk frame
    double Mll[6];             // (11, 12, 22, 13, 23, 33)
    Mot Ft[3];                 // columns of M_tl (force in the trunk joint frame)
    SymY Yleg;
    {
        SymY Yc;
        Mot F[3];
#pragma unroll
        for (int i = 3; i >= 1; --i) {
            const RecDbl* rd = JB_RDBL + (i * L + c.sub);
            const V3 ax = ld3(rd->axis);
            SymY Yi;
            inertia_to_sym(rd->inertia[0], ld3(rd->inertia + 1), rd->inertia + 4, Yi);
            if (i < 3) {
                Xf lic; sm_load_xf(c, KP->rec_off[i + 1] + R1_LIMI, lic);
                SymY T;
                sym_transform(lic, Yc, T);
                sym_add(Yi, T);
                // forces of the dofs below, one frame up
#pragma unroll
                for (int j = i + 1; j <= 3; ++j) F[j - 1] = force_act(lic, F[j - 1]);
            }
            Yc = Yi;
            Mot S = mzero(); S.a = ax;
            F[i - 1] = sym_mul_motion(Yc, S);
            // row i of M_ll: S_i . F_j (j >= i), all expressed in frame i
            Mll[i == 1 ? 0 : (i == 2 ? 2 : 5)] = dot(ax, F[i - 1].a) + rd->armature;
            if (i == 2) Mll[4] = dot(ax, F[2].a);
            if (i == 1) { Mll[1] = dot(ax, F[1].a); Mll[3] = dot(ax, F[2].a); }
        }
        Xf li1; sm_load_xf(c, KP->rec_off[1] + R1_LIMI, li1);
        sym_transform(li1, Yc, Yleg);
#pragma unroll
        for (int j = 0; j < 3; ++j) Ft[j] = force_act(li1, F[j]);
    }
    double Mi[6];
    sym3_inverse(Mll, Mi);
    // W = M_ll^-1 M_lt (3 x 6), T = Yleg - M_tl W
    double W[3][6];
    SymY Tl;
    {
        const double Mfull[3][3] = {{Mi[0], Mi[1], Mi[3]}, {Mi[1], Mi[2], Mi[4]}, {Mi[3], Mi[4], Mi[5]}};
        double Fv[3][6];
#pragma unroll
        for (int j = 0; j < 3; ++j) { Fv[j][0] = Ft[j].l.x; Fv[j][1] = Ft[j].l.y; Fv[j][2] = Ft[j].l.z; Fv[j][3] = Ft[j].a.x; Fv[j][4] = Ft[j].a.y; Fv[j][5] = Ft[j].a.z; }
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int d = 0; d < 6; ++d) W[i][d] = Mfull[i][0] * Fv[0][d] + Mfull[i][1] * Fv[1][d] + Mfull[i][2] * Fv[2][d];
        auto sp = [&](int a, int b) { return Fv[0][a] * W[0][b] + Fv[1][a] * W[1][b] + Fv[2][a] * W[2][b]; };
        // T = Yleg - M_tl W, symmetric 6 x 6 in SymY layout: A (lin-lin), B[3 a + b] (lin a, ang b), D (ang-ang)
        Tl.A[0] = Yleg.A[0] - sp(0, 0); Tl.A[1] = Yleg.A[1] - sp(0, 1); Tl.A[2] = Yleg.A[2] - sp(1, 1);
        Tl.A[3] = Yleg.A[3] - sp(0, 2); Tl.A[4] = Yleg.A[4] - sp(1, 2); Tl.A[5] = Yleg.A[5] - sp(2, 2);
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
            for (int b = 0; b < 3; ++b) Tl.B[3 * a + b] = Yleg.B[3 * a + b] - sp(a, 3 + b);
        Tl.D[0] = Yleg.D[0] - sp(3, 3); Tl.D[1] = Yleg.D[1] - sp(3, 4); Tl.D[2] = Yleg.D[2] - sp(4, 4);
        Tl.D[3] = Yleg.D[3] - sp(3, 5); Tl.D[4] = Yleg.D[4] - sp(4, 5); Tl.D[5] = Yleg.D[5] - sp(5, 5);
        // park W and M_ll^-1 in the dead U / Dinv / u fields of the leg records, the foot rotation in the pool entry
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            double* const rq = jb_smem + KP->rec_off[i + 1] * 32 + c.lane;
#pragma unroll
            for (int d = 0; d < 6; ++d) rq[(R1_FU + d) * 32] = W[i][d];
            rq[R1_DINV * 32] = Mi[2 * i]; rq[R1_U * 32] = Mi[2 * i + 1];
        }
#pragma unroll
        for (int k = 0; k < 9; ++k) SMF(c, KP->pool_off + k) = oM.R[k];
    }
    // ---------------- S = I_trunk + sum over the lanes (fixed order: identical on every lane), factored once
    Spd6 sf;
    {
        SymY S;
        inertia_to_sym(rd0->inertia[0], ld3(rd0->inertia + 1), rd0->inertia + 4, S);
#pragma unroll
        for (int k = 0; k < 6; ++k) { S.A[k] += cq_bcast_sum4(c, Tl.A[k], M); S.D[k] += cq_bcast_sum4(c, Tl.D[k], M); }
#pragma unroll
        for (int k = 0; k < 9; ++k) S.B[k] += cq_bcast_sum4(c, Tl.B[k], M);
        spd6_factor(S, sf);
    }
    // ---------------- constraint rows of this lane's contact frame (FrameConstraint::computeJacobianAndDrift)
    double G[4][6], H[4][6], AL[4][4], B[4], LA[4], Y[4], YP[4], iAD[4], RG[4], AD01[2];
    Mot zpart = mzero();
    {
        Xf P;
#pragma unroll
        for (int k = 0; k < 9; ++k) P.R[k] = ct->placement[k];
        P.p = ld3(ct->placement + 9);
        double Rf[9];
        mat3mul(oM.R, P.R, Rf);
        const V3 pf = oM.p + rmul(oM.R, P.p);
        // unconstrained accelerations: trunk (6) and this leg (3)
        const Mot at = sm_load_mot(c, KP->rec_off[0] + RF_A);
        const double al[3] = {SMF(c, KP->rec_off[1] + R1_A), SMF(c, KP->rec_off[2] + R1_A), SMF(c, KP->rec_off[3] + R1_A)};
        // drift with Baumgarte stabilisation
        const Mot vLoc = motion_act_inv(P, v), aLoc = motion_act_inv(P, aD);
        const V3 vl = rmul(Rf, vLoc.l), va = rmul(Rf, vLoc.a);
        V3 dl = rmul(Rf, aLoc.l) + cross(va, vl), da = rmul(Rf, aLoc.a);
        const double omega = 2.0 * 3.14159265358979323846 * opt.contact_stabilization_freq;
        const double kp = omega * omega, kd = 2.0 * omega;
        double RrT[9], Rref[9];
#pragma unroll
        for (int e = 0; e < 9; ++e) Rref[e] = CST(cso + 5 + e);
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
            for (int b2 = 0; b2 < 3; ++b2) RrT[3 * a + b2] = Rf[3 * a] * Rref[3 * b2] + Rf[3 * a + 1] * Rref[3 * b2 + 1] + Rf[3 * a + 2] * Rref[3 * b2 + 2];
        dl = dl + kp * (pf - mk(CST(cso + 14), CST(cso + 15), CST(cso + 16))) + kd * vl;
        da = da + kp * cons_log3(RrT) + kd * va;
        const double gamma[4] = {dl.x, dl.y, dl.z, da.z};
        const V3 lever0 = oM0.p - pf;
        const double Mfull[3][3] = {{Mi[0], Mi[1], Mi[3]}, {Mi[1], Mi[2], Mi[4]}, {Mi[3], Mi[4], Mi[5]}};
        double Jl[4][3];
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            const V3 lin = cross(parm[i] - pf, wax[i]);
            Jl[0][i] = lin.x; Jl[1][i] = lin.y; Jl[2][i] = lin.z; Jl[3][i] = wax[i].z;
        }
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            // J_t row: trunk subspace = identity in the trunk joint frame
            double Jt[6];
            if (r < 3) {
#pragma unroll
                for (int d = 0; d < 3; ++d) {
                    const V3 col = mk(oM0.R[d], oM0.R[3 + d], oM0.R[6 + d]);   // R_0 e_d
                    const V3 lin = cross(lever0, col);
                    Jt[d] = (r == 0 ? col.x : (r == 1 ? col.y : col.z));
                    Jt[3 + d] = (r == 0 ? lin.x : (r == 1 ? lin.y : lin.z));
                }
            } else {
                Jt[0] = 0.0; Jt[1] = 0.0; Jt[2] = 0.0; Jt[3] = oM0.R[6]; Jt[4] = oM0.R[7]; Jt[5] = oM0.R[8];
            }
            double g[6];
#pragma unroll
            for (int d = 0; d < 6; ++d) g[d] = Jt[d] - (Jl[r][0] * W[0][d] + Jl[r][1] * W[1][d] + Jl[r][2] * W[2][d]);
            Mot gm; gm.l = mk(g[0], g[1], g[2]); gm.a = mk(g[3], g[4], g[5]);
            const Mot h = spd6_apply(sf, gm);
            const double hv[6] = {h.l.x, h.l.y, h.l.z, h.a.x, h.a.y, h.a.z};
            const double lam = en ? CST(cso + 1 + r) : 0.0;
#pragma unroll
            for (int d = 0; d < 6; ++d) { G[r][d] = en ? g[d] : 0.0; H[r][d] = en ? hv[d] : 0.0; }
#pragma unroll
            for (int i = 0; i < 3; ++i) SMF(c, KP->pool_off + 9 + 3 * r + i) = en ? Jl[r][i] : 0.0;   // parked in the pool entry
            double mj[3];   // M_ll^-1 J_l,r^T
#pragma unroll
            for (int i = 0; i < 3; ++i) mj[i] = Mfull[i][0] * Jl[r][0] + Mfull[i][1] * Jl[r][1] + Mfull[i][2] * Jl[r][2];
#pragma unroll
            for (int q = 0; q < 4; ++q) AL[r][q] = Jl[q][0] * mj[0] + Jl[q][1] * mj[1] + Jl[q][2] * mj[2];
            const double a0 = (Jl[r][0] * mj[0] + Jl[r][1] * mj[1] + Jl[r][2] * mj[2]) + (g[0] * hv[0] + g[1] * hv[1] + g[2] * hv[2] + g[3] * hv[3] + g[4] * hv[4] + g[5] * hv[5]);
            const double reg = fmax(a0 * opt.constraint_regularization, CONS_MIN_REGULARIZER);
            iAD[r] = 1.0 / (a0 + reg); RG[r] = reg;
            if (r < 2) AD01[r] = a0 + reg;
            const double jd = Jt[0] * at.l.x + Jt[1] * at.l.y + Jt[2] * at.l.z + Jt[3] * at.a.x + Jt[4] * at.a.y + Jt[5] * at.a.z +
                              Jl[r][0] * al[0] + Jl[r][1] * al[1] + Jl[r][2] * al[2];
            B[r] = -gamma[r] - jd;
            LA[r] = lam; Y[r] = 0.0; YP[r] = 0.0;
            if (en) { zpart.l = zpart.l + lam * gm.l; zpart.a = zpart.a + lam * gm.a; }
        }
    }
    // z = sum over all rows of g_r lambda_r (all-reduce in fixed order)
    double z[6];
    z[0] = cq_bcast_sum4(c, zpart.l.x, M); z[1] = cq_bcast_sum4(c, zpart.l.y, M); z[2] = cq_bcast_sum4(c, zpart.l.z, M);
    z[3] = cq_bcast_sum4(c, zpart.a.x, M); z[4] = cq_bcast_sum4(c, zpart.a.y, M); z[5] = cq_bcast_sum4(c, zpart.a.z, M);
    // ---------------- projected Gauss-Seidel sweep (constraint_solvers.cc:107-318)
    // Sweep order = contact index order; the lane owning contact k updates its multipliers from the current z and
    // broadcasts the change of z to the other lanes of the env with shuffles.  Everything the sweep touches is in
    // registers (all indices are compile-time after unrolling); divisions by the regularised diagonal are
    // multiplications by its reciprocal.
    JB_PROF_ADD(3, t_setup);                               // solver set-up
    JB_PROF_T(t_loop);
    const double iAmax = 1.0 / fmax(AD01[0], AD01[1]);
    auto residual = [&](int k) {
        const double s = (AL[0][k] * LA[0] + AL[1][k] * LA[1]) + (AL[2][k] * LA[2] + AL[3][k] * LA[3]);
        const double hz = (H[k][0] * z[0] + H[k][1] * z[1]) + (H[k][2] * z[2] + H[k][3] * z[3]) + (H[k][4] * z[4] + H[k][5] * z[5]);
        return B[k] - (s + hz) - RG[k] * LA[k];
    };
    // The sweep is run some forty times per solve and what it costs is instruction fetch: straight-line code beyond the
    // 6 KB L0 instruction cache of the scheduler is delivered at ~45 cycles per 128-byte line, every iteration again
    // (an earlier version unrolled the twelve updates of an iteration, each in its own divergent region, and paid about
    // six cycles per instruction).  So the loops over the contacts are real
    // loops, the owner of a contact is a predicate, not a branch, and the relaxation schedule is a table: a few hundred
    // instructions that stay in the L0 for the whole solve.
    const int lane0 = c.lane - c.sub;
    int src_pack = 0, my_k = -1;
#pragma unroll
    for (int k = 0; k < 4; ++k) { const int o = KP->cmap[k].sub; src_pack |= (lane0 + o) << (8 * k); if (o == c.sub) my_k = k; }
    const bool torsion_on = !(opt.contact_torsion < D_EPS), friction_on = !(opt.contact_friction < D_EPS);
    const double mu = opt.contact_friction, mu_t = opt.contact_torsion;
    bool ok = false;
    for (int iter = 0; uni ? __any_sync(0xffffffffu, iter < CONS_PGS_MAX_ITER && !ok) : (iter < CONS_PGS_MAX_ITER && !ok); ++iter) {
        const bool live = !ok && iter < CONS_PGS_MAX_ITER;   // (uniform warp: an env that is done keeps exchanging zeros)
        const bool upd = en && live;
#pragma unroll
        for (int r = 0; r < 4; ++r) YP[r] = Y[r];
        const double wr = KP->pgs_relax[iter < CONS_PGS_MAX_ITER ? iter : CONS_PGS_MAX_ITER - 1];
        // normal forces, contact by contact
        JB_PROF_T(t_n);
#pragma unroll 1
        for (int k = 0; k < 4; ++k) {
            const bool own = upd && k == my_k;
            const double y = residual(2);
            const double x = LA[2] + wr * y * iAD[2];
            const double e = x > 0.0 ? x : 0.0;
            const double d2 = own ? e - LA[2] : 0.0;
            if (own) { Y[2] = y; LA[2] = e; }
            const int src = (src_pack >> (8 * k)) & 0xff;
#pragma unroll
            for (int d = 0; d < 6; ++d) z[d] += __shfl_sync(M, G[2][d] * d2, src);
        }
        JB_PROF_ADD(13, t_n);                              // normal-force loop
        // torsion
        if (!torsion_on) {
            // disabled: its bounds force the multiplier to zero, after the normal forces of the iteration like in the
            // reference.  Only a warm start can make it non-zero (the equality solve of Engine::start does), so the first
            // iteration is the only one with anything to do
            if (iter == 0) {
                const double d3 = -LA[3];
                LA[3] = 0.0;
                if (uni ? __any_sync(0xffffffffu, d3 != 0.0) : __any_sync(c.gmask, d3 != 0.0)) {
#pragma unroll 1
                    for (int k = 0; k < 4; ++k) {
                        const int src = (src_pack >> (8 * k)) & 0xff;
#pragma unroll
                        for (int d = 0; d < 6; ++d) z[d] += __shfl_sync(M, G[3][d] * d3, src);
                    }
                }
            }
        } else {
#pragma unroll 1
            for (int k = 0; k < 4; ++k) {
                const bool own = upd && k == my_k;
                const double y = residual(3);
                const double thr = mu_t * LA[2];
                const double e = fmin(fmax(LA[3] + wr * y * iAD[3], -thr), thr);
                const double d3 = own ? e - LA[3] : 0.0;
                if (own) { Y[3] = y; LA[3] = e; }
                const int src = (src_pack >> (8 * k)) & 0xff;
#pragma unroll
                for (int d = 0; d < 6; ++d) z[d] += __shfl_sync(M, G[3][d] * d3, src);
            }
        }
        // friction
        JB_PROF_T(t_f);
#pragma unroll 1
        for (int k = 0; k < 4; ++k) {
            const bool own = upd && k == my_k;
            const double y0 = residual(0), y1 = residual(1);
            double e0 = LA[0] + wr * y0 * iAmax, e1 = LA[1] + wr * y1 * iAmax;
            const double thr = mu * LA[2];
            const double sq = e0 * e0 + e1 * e1;
            // projection on the friction cone: thr / sqrt(sq) as thr * rsqrt(sq), branch-free (a double-precision square
            // root plus a division are ~500 cycles of dependent instructions, paid by every lane at every step of the sweep)
            const double scale = sq > thr * thr ? thr * rsqrt(sq) : 1.0;
            e0 *= scale; e1 *= scale;
            if (!friction_on) { e0 = LA[0] * 0.0; e1 = LA[1] * 0.0; }
            const double d0 = own ? e0 - LA[0] : 0.0, d1 = own ? e1 - LA[1] : 0.0;
            if (own) {
                if (friction_on) { Y[0] = y0; Y[1] = y1; }
                LA[0] = e0; LA[1] = e1;
            }
            const int src = (src_pack >> (8 * k)) & 0xff;
#pragma unroll
            for (int d = 0; d < 6; ++d) z[d] += __shfl_sync(M, G[0][d] * d0 + G[1][d] * d1, src);
        }
        JB_PROF_ADD(14, t_f);                              // friction loop
        JB_PROF_T(t_conv);
        // stopping criterion on the stagnation of the residuals (constraint_solvers.cc:256-274)
        double ymax = fmax(fmax(fabs(Y[0]), fabs(Y[1])), fmax(fabs(Y[2]), fabs(Y[3])));
        for (int o = 1; o < L; o <<= 1) ymax = fmax(ymax, __shfl_xor_sync(M, ymax, o));
        const double tol = opt.tol_abs + opt.tol_rel * ymax + D_EPS;
        bool conv = true;
#pragma unroll
        for (int r = 0; r < 4; ++r) conv = conv && (fabs(Y[r] - YP[r]) < tol);
        const bool all_conv = cq_all(M, c, conv || !live);   // (one call site: every lane of the mask takes part)
        if (live) ok = all_conv;
        JB_PROF_ADD(15, t_conv);                           // stopping criterion
        JB_PROF_COUNT(12, 1);                              // sweep iterations
#ifdef JB_DEBUG_COUNTS
        if (c.sub == 0) { extern long long jb_dbg_counts[8]; ++jb_dbg_counts[4]; if (!ok && iter == CONS_PGS_MAX_ITER - 1) ++jb_dbg_counts[5]; }
#endif
    }
    JB_PROF_ADD(4, t_loop);                                // the sweep
    JB_PROF_T(t_post);
    // ---------------- accelerations: ddq_t = ddq_free_t + S^-1 z = ddq_free_t + sum_r h_r lambda_r ;
    //                  ddq_l = ddq_free_l + M_ll^-1 J_l^T lambda - W (ddq_t - ddq_free_t)
    {
        double xp[6] = {0, 0, 0, 0, 0, 0};
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int d = 0; d < 6; ++d) xp[d] += H[r][d] * LA[r];
        double xv[6];
#pragma unroll
        for (int d = 0; d < 6; ++d) xv[d] = cq_bcast_sum4(c, xp[d], M);
        double* const r0 = jb_smem + KP->rec_off[0] * 32 + c.lane;
#pragma unroll
        for (int d = 0; d < 6; ++d) r0[(RF_A + d) * 32] += xv[d];
        double rl[3] = {0, 0, 0};
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int i = 0; i < 3; ++i) rl[i] += SMF(c, KP->pool_off + 9 + 3 * r + i) * LA[r];
        double mi[6];
#pragma unroll
        for (int i = 0; i < 3; ++i) { mi[2 * i] = SMF(c, KP->rec_off[i + 1] + R1_DINV); mi[2 * i + 1] = SMF(c, KP->rec_off[i + 1] + R1_U); }
        const double Mfull[3][3] = {{mi[0], mi[1], mi[3]}, {mi[1], mi[2], mi[4]}, {mi[3], mi[4], mi[5]}};
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            double x = Mfull[i][0] * rl[0] + Mfull[i][1] * rl[1] + Mfull[i][2] * rl[2];
#pragma unroll
            for (int d = 0; d < 6; ++d) x -= SMF(c, KP->rec_off[i + 1] + R1_FU + d) * xv[d];
            SMF(c, KP->rec_off[i + 1] + R1_A) += x;
        }
        // multipliers back into the constraint, contact wrench in the parent joint frame (engine.cc:3790-3822)
        double* const cp = jb_smem + KP->cslot_off * 32 + c.lane;
        if (en) {
#pragma unroll
            for (int r = 0; r < 4; ++r) CST(cso + 1 + r) = LA[r];
            double R3[9];
#pragma unroll
            for (int k = 0; k < 9; ++k) R3[k] = SMF(c, KP->pool_off + k);
            const V3 Fl = rtmul(R3, mk(LA[0], LA[1], LA[2]));
            const V3 Tq = rtmul(R3, mk(0.0, 0.0, LA[3]));
            CO(0) = Fl.x; CO(1) = Fl.y; CO(2) = Fl.z; CO(3) = Tq.x; CO(4) = Tq.y; CO(5) = Tq.z;
        }
        if (c.sub == 0) CST(CS_SOLVE_FAILED) = ok ? 0.0 : CST(CS_SOLVE_FAILED) + 1.0;
    }
    __syncwarp(M);
    cons_refresh_accelerations(c);
    JB_PROF_ADD(5, t_post);                                // multipliers -> accelerations, refresh
    (void)status;
    return ok;
}

JB_DI bool cons_solve_quadruped(const Ctx c, int* status) {
    return (c.flags & CTX_UNIFORM_WARP) ? cons_solve_quadruped_t<true>(c, status) : cons_solve_quadruped_t<false>(c, status);
}
