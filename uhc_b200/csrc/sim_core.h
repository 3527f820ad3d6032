// sim_core.h -- the per-humanoid physics + imitation-task step, one WARP per environment.
//
// Product code (CUDA, sm_90a).  Everything in this header is written in an SPMD "phase" style:
//     LANES_BEGIN ... per-lane code, no cross-lane dependency inside ... LANES_END   (= __syncwarp())
// so that the very same source can also be compiled by g++ as a lane-loop emulation (tests/emu, -DUHC_EMU) and be
// debugged on a CPU-only box.  The emulation is test infrastructure; the C-ABI library only ever launches the CUDA build.
//
// Algorithms (all world-aligned spatial vectors about the reference point O = root position):
//   kinematics            every lane composes its own chain root -> body, lane = body       (a5: mj_kinematics)
//   bias force C(q,v)     spatial recursive Newton-Euler, lane = body / lane = dof         (a5: mj_rne)
//   linear solves         O(n) articulated-body sweeps over a centre-rooted 7-level tree, 6 lanes per body, 3x3 block
//                         elimination, packed fp32 pairs (replaces mj_crb + mj_factorM + cho_solve)
//   stable PD             (M_stale + Kd dt)^-1 rhs by the articulated-body solve             (a3: humanoid_im.py:1014-1076)
//   floor contacts        plane / convex-hull support vertex + hull-graph neighbours, all   (a5: collision)
//                         candidate bodies in one pass (a group of lanes per candidate)
//   constraint solve      primal Newton on the convex soft-constraint cost, Newton direction = articulated-body solve with
//                         contact-augmented body inertias, safeguarded 1-D Newton line search (a5: solver)
//   integration           semi-implicit Euler, quaternion exponential map for the root      (a5: mj_Euler)
//   epilogue              body quats, termination, observation v2, world_rfc_implicit reward (a6, a7, a10)
// Reference behaviour being restated is cited next to each phase (file:line under the reference tree).
#pragma once
#include <math.h>
#include <stdint.h>

#ifndef UHC_EMU
#include <cuda_runtime.h>
#define UHC_DEV __device__ __forceinline__
#define UHC_DEVNI __device__ __noinline__
#define LANES_BEGIN { const int lane = (int)(threadIdx.x & 31);
#define LANES_END } __syncwarp();
#define LANES_END_R }                /* block that exchanged nothing through shared memory: no warp barrier needed */
#define LVAR(T, n) T n
#define LV(n) n
#define LVARA(T, n, K) T n[K]
#define LVA(n) n
#define LV_ARR(n, c) n[c]
#define LV_ALL(n) n
#define UHC_LDG(p) __ldg(p)
// small per-model tables (dof_f, lvl_pack): the kernels stage them in shared memory and point the Model at the copies, so the
// device reads them with shared-space loads (32-bit addressing, no generic-pointer arithmetic)
__device__ __forceinline__ float uhc_lds(const float *p) { float v; asm("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"((unsigned)__cvta_generic_to_shared(p))); return v; }
__device__ __forceinline__ double uhc_lds(const double *p) { double v; asm("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"((unsigned)__cvta_generic_to_shared(p))); return v; }
__device__ __forceinline__ int uhc_lds(const int *p) { int v; asm("ld.shared.s32 %0, [%1];" : "=r"(v) : "r"((unsigned)__cvta_generic_to_shared(p))); return v; }
#define UHC_LDT(p) uhc_lds(p)
#else
#define UHC_DEV static inline
#define UHC_DEVNI static
#define LANES_BEGIN for (int lane = 0; lane < 32; ++lane) {
#define LANES_END }
#define LANES_END_R }
#define LVAR(T, n) T n[32]
#define LV(n) n[lane]
#define LVARA(T, n, K) T n[32][K]
#define LVA(n) n[lane]
#define LV_ARR(n, c) n[lane][c]
#define LV_ALL(n) n
#define UHC_LDG(p) (*(p))
#define UHC_LDT(p) (*(p))
#endif

namespace uhc {

constexpr int NB = 24, NQ = 76, NV = 75, NU = 69, NSUB = 15;
constexpr int OBS_DIM = 657, ACT_DIM = 105;
constexpr int UPPER_BODY0 = 12;               // bodies >= Neck: arms, neck, head
constexpr int MAXCON = 40;
constexpr int MAXLEVEL = 8;
constexpr int LVL_G = 5;                      // max bodies per tree level (lane groups of 6 lanes in the articulated-body solve)
constexpr int BODYF = 20;                     // floats per body in the model table
// per-env state record in HBM (Real units)
// The first ST_BLOCK Reals mirror the head of the shared-memory work set (q v aw C Ib S) byte for byte, so the step kernel moves them with
// ONE bulk-async (TMA) copy in and one out; every field starts on a 16-byte boundary (vector stores for the rest).
constexpr int ST_Q = 0, ST_V = 76, ST_AW = 152, ST_C = 228, ST_IB = 304, ST_S = 544, ST_BLOCK = 996,   // IB: per-body inertia 24x10, S: 75x6 (+2 pad)
              ST_XPOS = 996, ST_XQUAT = 1068, ST_XIPOS = 1164, ST_BQUAT = 1236, ST_PBQUAT = 1332, ST_SIZE = 1428;
// per-env integer record
constexpr int SI_CUR_T = 0, SI_CLIP = 1, SI_START = 2, SI_LEN = 3, SI_EPISODE = 4, SI_FLAGS = 5, SI_NEWTON = 6, SI_NCON = 7, SI_SIZE = 8;
// expert frame record (Real units): qpos 76 | qvel 75 | wbpos 72 | wbquat 96 | bquat 96 | bangvel 72 | ee_wpos 15 | body_com 72 (com = its first 3) | pad
constexpr int EX_QPOS = 0, EX_QVEL = 76, EX_WBPOS = 151, EX_WBQUAT = 223, EX_BQUAT = 319, EX_BANGVEL = 415, EX_EE = 487,
              EX_COM = 502, EX_BCOM = 502, EX_SIZE = 576;
constexpr int OBS_DIM_V1 = 784, MAX_OBS_DIM = 784;   // get_full_obs_v1: v2 without the 17 shape dims plus two 72-wide per-body COM blocks

template <class Real>
struct Model {
    const Real *body_f;   // [NB][BODYF]: offset3 ipos3 mass inertia6(xx,yy,zz,xy,xz,yz) invw bsphere4 diffw pad
    const Real *dof_f;    // [NV][4]: armature, kp, kd, torque_lim
    const Real *dof_lim;  // [NV][4]: joint limit lower, upper (rad), dof_invweight0, pad
    const Real *hull;     // [nvert][3] body-local
    const int *hull_adr, *hull_num, *nbr, *nbradr;
    const int *parent, *depth, *child_adr, *child, *body_sub_end;
    const int *ee;                // [5]
    const int *lvl_tab;           // [MAXLEVEL+1][LVL_G][5]: body, parent's group, groups of <=3 children (-1 = none)
    const int *lvl_pack;          // elimination tree of the solve (hung from the tree's centre), [MAXLEVEL+1][LVL_G]: (body+1) | pgrp<<6 | (cg0+1)<<9 | (cg1+1)<<12 | (cg2+1)<<15
                                  //   | nslot<<18 (max children per body on the level) | (first dof / 3)<<20 | reversed<<25 | nlevels<<26
    Real dt, margin, mu, solref0, solref1, simp0, simp1, simp2, simp3, simp4, gravz;
    int nshape, nvert;            // body_f / hull hold `nshape` consecutive shape variants ([nshape][NB][BODYF], [nshape][nvert][3])
    const void *topo_s;           // device: LaneTopo[32] staged in shared memory by the kernels (per-lane tree links); unused on the host
};

template <class Real>
struct EnvCfg {
    Real base_rot[4], rfc_scale, rfc_lim, rfc_rate, body_diff_thresh;
    int meta_pd, env_episode_len, trail_steps, newton_max_iter;
    Real w[5], k[5], newton_tol;
    int auto_reset, t_min, t_max, num_clips;      // in-kernel re-seeding of finished episodes (dataset_amass_single.py:172-253)
    unsigned long long reset_seed;
    int reactive_v; Real reactive_rate;           // reset_model's reactive_v = 1 branch (humanoid_im.py:1255-1271): start from the standing pose w.p. reactive_rate
    // residual-force mode (cfg.residual_force / residual_force_mode, humanoid_im.py:231-243): 0 = implicit root wrench (6 action dims), 1 = explicit per-body
    // contact point / force / torque (9 dims x 24 bodies), 2 = residual_force: false (no residual-force dims, no applied force, reward term 0).  Action layout: [NU joint targets | vf_dim residual-force dims | 30 meta-PD scales if meta_pd]
    int rfc_mode, vf_dim, act_dim;
    int obs_v, obs_dim;                           // cfg.obs_v: 2 = get_full_obs_v2 (657), 1 = get_full_obs_v1 (784; config/release/uhc_implicit.yml), 5 / 6 = get_full_obs_v5 / v6 (636 / 384 + shape),
    int fut_frames, fut_skip;                     //   3 = get_full_obs_v3 (:505-513): fut_frames v2 blocks against the expert frames cur_t + 1 + i * skip
    int has_shape, obs_block;                     // cfg.has_shape (:499-500): the v2 block ends with the 17 shape dims (657) or not (640); obs_block = its width
    signed char vf_slot[NB];                      // explicit: residual-force slot of body b (vf_bodies = SMPL_BONE_ORDER_NAMES, humanoid_im.py:236-237)
    int term_body, head_body;                     // cfg.env_term_body (humanoid_im.py:1223-1229): 0 body-position error, 1 root height, 2 height of body head_body
    int reward_mul;                               // world_rfc_implicit_v1_mul (reward_function.py:174-250): the product of the terms instead of their weighted mean
};
constexpr int VF_BODY_DIM = 9, MAX_ACT_DIM = NU + VF_BODY_DIM * NB + 30;

// phases of a control step for the cycle accounting of UHC_PHASE_CLOCKS builds (PCLK below, scripts/step_phase_cycles.py)
enum { PC_LOAD, PC_PD, PC_KIN, PC_COLLIDE, PC_SMOOTH, PC_CSETUP, PC_NEWTON_ABA, PC_NEWTON_ROWS, PC_SYNC_SUBSTEP, PC_SYNC_PD, PC_SYNC_SMOOTH,
       PC_INTEGRATE, PC_EPILOGUE, NPHASE };
// sub-phases of PC_KIN (kin_rne_forward's stages, then project_force) and PC_COLLIDE (broad phase, narrow phase, contact ranges); PSUB below
enum { PS_KIN_SINCOS, PS_KIN_LEVELS, PS_KIN_INERTIA, PS_KIN_SUBTREE, PS_KIN_PROJECT, PS_COL_BROAD, PS_COL_NARROW, PS_COL_PREFIX, NSUBPHASE };

// per-environment working set (lives in shared memory on the GPU)
template <class Real>
struct Work {
    // ---- head: the persistent simulator state, laid out exactly like the first ST_BLOCK Reals of the HBM record (bulk-async copy in / out)
    alignas(16) Real q[NQ]; Real v[NV + 1], aw[NV + 1], C[NV + 1];
    Real Ib[NB][10];              // per-body rigid inertia about O, world axes (of the last forward pass)
    alignas(16) Real S[NV + 6][6];   // motion subspaces; rows NV.. are the unit vectors of the solve's virtual dofs
    // ---- derived pose (vector stores to the record), the rest of the working set
    alignas(16) Real xpos[NB][3]; Real xipos[NB][3], xmat[NB][9];
    Real act[ACT_DIM + 3];
    // The articulated-body sweep's scratch is only live inside one aba_solve; it shares its bytes with vectors that are dead across every
    // aba_solve of a substep (1.8 KB less per env, so 16 work sets fit one SM):
    //   Vb  kin_rne_forward -> constraint_setup (the smooth solve only runs when there is no constraint, so none runs in between)
    //   Fb  body-wrench scratch of kin_rne_forward / project_force, rfc_explicit, newton_init, newton_advance (never held across a solve)
    //   fs  smooth phase -> newton_init (same argument as Vb)
    //   xquat  world_quat after the last solve of the step / of the reset -> observation, store_state
    union {
        struct {
            alignas(16) Real aU[NV + 6][6];   // columns of  U D^-1  per 3-dof block (U = IA S, D = S^T U + arm)
            Real au[NV + 6];                // D^-1 u per block
        };
        struct {
            alignas(16) Real xquat[NB][4];
            alignas(16) Real Vb[NB][6], Fb[NB][6];
            Real fs[NV + 1];
        };
    };
    Real as_[NV + 1], a[NV + 1], g[NV + 1], p[NV + 1], Mp[NV + 1], tau[NV + 1];   // Mp: the solve's joint-space diagonal
    alignas(16) Real Ab[NB][6];
    // contacts
    int cbody[MAXCON]; Real cr[MAXCON][3], cdist[MAXCON], cD[MAXCON], caref[MAXCON][4], cres[MAXCON][4], cjp[MAXCON][4];
    int bcon_adr[NB + 1];
    int ncon, upper_contact;
    int nlim;                     // joint-limit rows of this substep (hinges past their range); their data rides in tau (sign * D) and as_ (residual)
    int con_overflow;             // a candidate body's contacts did not fit MAXCON in some substep of this step (the env is failed, never silently truncated)
    alignas(8) unsigned long long mbar;   // mbarrier of this warp's bulk-async state load
    int sync_threads;             // threads taking part in the substep alignment barrier of this warp's group (32 x its warps that own a valid env)
    int sync_id;                  // named barrier of this warp's alignment group (1 + group index; SYNC_GROUP warps per group)
    // this env's model view (shape variant) and config: kept here so that the non-inlined phases read them from shared memory
    // instead of a per-thread local-memory copy
    alignas(8) Model<Real> mdl;
    alignas(8) EnvCfg<Real> cfg;
#if defined(UHC_PHASE_CLOCKS) && !defined(UHC_EMU)
    long long pc_t, pc[NPHASE];   // clock64 of the last phase boundary, cycles per phase of this control step
    long long ps_t, ps[NSUBPHASE];   // clock64 of the last phase or sub-phase boundary, cycles per sub-phase of this control step
#endif
};

// Phase cycle accounting, compiled in only with -DUHC_PHASE_CLOCKS: lane 0 of a warp reads clock64() at every phase boundary of the
// control step and adds the interval since the previous boundary to that phase; env_step_warp adds the totals to EngineView::phase_cyc.
// PCLK(on, w, ph) closes phase ph when `on` (the in-kernel reset runs substep_dynamics without it).  PSUB(on, w, sp) closes sub-phase sp, which
// runs from the last PCLK or PSUB; the sub-phases of a phase end with it, so they split its cycles.  Without the switch all three are empty.
#if defined(UHC_PHASE_CLOCKS) && !defined(UHC_EMU)
#define PCLK_START(w) do { __syncwarp(); if ((threadIdx.x & 31) == 0) { for (int i_ = 0; i_ < NPHASE; i_++) (w).pc[i_] = 0; \
    for (int i_ = 0; i_ < NSUBPHASE; i_++) (w).ps[i_] = 0; (w).pc_t = (w).ps_t = clock64(); } } while (0)
#define PCLK(on, w, ph) do { if (on) { __syncwarp(); if ((threadIdx.x & 31) == 0) { const long long t_ = clock64(); (w).pc[ph] += t_ - (w).pc_t; (w).pc_t = (w).ps_t = t_; } } } while (0)
#define PSUB(on, w, sp) do { if (on) { __syncwarp(); if ((threadIdx.x & 31) == 0) { const long long t_ = clock64(); (w).ps[sp] += t_ - (w).ps_t; (w).ps_t = t_; } } } while (0)
#else
#define PCLK_START(w) do { } while (0)
#define PCLK(on, w, ph) do { (void)sizeof(on); } while (0)
#define PSUB(on, w, sp) do { (void)sizeof(on); } while (0)
#endif

// ------------------------------------------------------------------------------------------------ scalar helpers
// reciprocal: hardware approximation + one Newton step on the GPU (within 1 ulp; no slow-path branch), exact division elsewhere
UHC_DEV float rcp_(float x) {
#if defined(__CUDA_ARCH__)
    float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return fmaf(r, fmaf(-x, r, 1.0f), r);
#else
    return 1.0f / x;
#endif
}
UHC_DEV double rcp_(double x) { return 1.0 / x; }
UHC_DEV float rsqrt_(float x) { return 1.0f / sqrtf(x); }
UHC_DEV double rsqrt_(double x) { return 1.0 / sqrt(x); }
// compact sin/cos (Cody-Waite reduction by pi/2, degree-7/8 minimax polynomials; |err| < 2e-7 for |x| < 1e3) -- joint angles and
// half-angles only; keeps the hot loop free of libdevice's large-argument slow paths
UHC_DEV void sincos_(float x, float *s, float *c) {
    const float k = rintf(x * 0.63661977236758134f);
    float r = fmaf(k, -1.5707962512969971f, x);
    r = fmaf(k, -7.5497894158615964e-8f, r);
    const float r2 = r * r;
    const float sp = r * fmaf(r2, fmaf(r2, fmaf(r2, -1.9515295891e-4f, 8.3321608736e-3f), -1.6666654611e-1f), 1.0f);
    const float cp = fmaf(r2, fmaf(r2, fmaf(r2, fmaf(r2, 2.443315711809948e-5f, -1.388731625493765e-3f), 4.166664568298827e-2f), -0.5f), 1.0f);
    const int q = (int)k & 3;
    const float ss = (q & 1) ? cp : sp, cc = (q & 1) ? sp : cp;
    *s = (q & 2) ? -ss : ss;
    *c = ((q + 1) & 2) ? -cc : cc;
}
UHC_DEV void sincos_(double x, double *s, double *c) { *s = sin(x); *c = cos(x); }
UHC_DEV float acos_(float x) { return acosf(x); }
UHC_DEV double acos_(double x) { return acos(x); }
UHC_DEV float atan2_(float y, float x) { return atan2f(y, x); }
UHC_DEV double atan2_(double y, double x) { return atan2(y, x); }
UHC_DEV float exp_(float x) { return expf(x); }
UHC_DEV double exp_(double x) { return exp(x); }
UHC_DEV float abs_(float x) { return fabsf(x); }
UHC_DEV double abs_(double x) { return fabs(x); }
UHC_DEV float pow_(float x, float y) { return exp2f(y * log2f(x)); }
UHC_DEV double pow_(double x, double y) { return pow(x, y); }
template <class R> UHC_DEV R min_(R a, R b) { return a < b ? a : b; }
template <class R> UHC_DEV R max_(R a, R b) { return a > b ? a : b; }
template <class R> UHC_DEV R clamp_(R x, R lo, R hi) { return x < lo ? lo : (x > hi ? hi : x); }

template <class R> UHC_DEV void cross3(const R *a, const R *b, R *o) {
    R x = a[1] * b[2] - a[2] * b[1], y = a[2] * b[0] - a[0] * b[2], z = a[0] * b[1] - a[1] * b[0];
    o[0] = x; o[1] = y; o[2] = z;
}
template <class R> UHC_DEV R dot3(const R *a, const R *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
template <class R> UHC_DEV R dot6(const R *a, const R *b) {
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2] + a[3] * b[3] + a[4] * b[4] + a[5] * b[5];
}
template <class R> UHC_DEV void qmul(const R *a, const R *b, R *o) {
    R w = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
    R x = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
    R y = a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1];
    R z = a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0];
    o[0] = w; o[1] = x; o[2] = y; o[3] = z;
}
template <class R> UHC_DEV void qinv(const R *q, R *o) {  // conj / |q|^2 (uhc/utils/transformation.py:1509)
    R n = R(1) / (q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    o[0] = q[0] * n; o[1] = -q[1] * n; o[2] = -q[2] * n; o[3] = -q[3] * n;
}
template <class R> UHC_DEV void q2mat(const R *q, R *m) {  // rotation of the normalised quaternion
    R n = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
    R s = R(2) / n;
    R xx = s * q[1] * q[1], yy = s * q[2] * q[2], zz = s * q[3] * q[3];
    R xy = s * q[1] * q[2], xz = s * q[1] * q[3], yz = s * q[2] * q[3];
    R wx = s * q[0] * q[1], wy = s * q[0] * q[2], wz = s * q[0] * q[3];
    m[0] = 1 - yy - zz; m[1] = xy - wz; m[2] = xz + wy;
    m[3] = xy + wz; m[4] = 1 - xx - zz; m[5] = yz - wx;
    m[6] = xz - wy; m[7] = yz + wx; m[8] = 1 - xx - yy;
}
template <class R> UHC_DEV void mtv(const R *m, const R *v, R *o) {  // m^T v
    R a = m[0] * v[0] + m[3] * v[1] + m[6] * v[2], b = m[1] * v[0] + m[4] * v[1] + m[7] * v[2],
      c = m[2] * v[0] + m[5] * v[1] + m[8] * v[2];
    o[0] = a; o[1] = b; o[2] = c;
}
template <class R> UHC_DEV void mv3(const R *m, const R *v, R *o) {
    R a = m[0] * v[0] + m[1] * v[1] + m[2] * v[2], b = m[3] * v[0] + m[4] * v[1] + m[5] * v[2],
      c = m[6] * v[0] + m[7] * v[1] + m[8] * v[2];
    o[0] = a; o[1] = b; o[2] = c;
}
// rigid spatial inertia (10 params: m, h[3]=m*c, I_O{xx,yy,zz,xy,xz,yz}) times motion vector S=(a,b) -> force (n,f)
template <class R> UHC_DEV void rigid_mul(const R *I, const R *S, R *F) {
    const R *h = I + 1, *J = I + 4; const R *a = S, *b = S + 3;
    R hb[3], ha[3];
    cross3(h, b, hb); cross3(h, a, ha);
    F[0] = J[0] * a[0] + J[3] * a[1] + J[4] * a[2] + hb[0];
    F[1] = J[3] * a[0] + J[1] * a[1] + J[5] * a[2] + hb[1];
    F[2] = J[4] * a[0] + J[5] * a[1] + J[2] * a[2] + hb[2];
    F[3] = I[0] * b[0] - ha[0]; F[4] = I[0] * b[1] - ha[1]; F[5] = I[0] * b[2] - ha[2];
}
// packed symmetric 6x6 (21: row-major upper triangle) times vector
UHC_DEV int sym6(int i, int j) { if (i > j) { int t = i; i = j; j = t; } return i * 6 - (i * (i - 1)) / 2 + (j - i); }
template <class R> UHC_DEV void sym6_mul(const R *K, const R *x, R *y) {
#pragma unroll
    for (int i = 0; i < 6; i++) {
        R s = 0;
#pragma unroll
        for (int j = 0; j < 6; j++) s += K[sym6(i, j)] * x[j];
        y[i] = s;
    }
}

// ------------------------------------------------------------------------------------------------ packed pairs
// Two Reals handled together: loaded from shared memory as one 64-bit access, arithmetic component-wise (sm_90 has no packed fp32 instructions).
template <class R> struct alignas(2 * sizeof(R)) Pr { R x, y; };
template <class R> UHC_DEV Pr<R> pbc(R s) { Pr<R> r; r.x = s; r.y = s; return r; }
template <class R> UHC_DEV Pr<R> pfma(Pr<R> a, Pr<R> b, Pr<R> c) { Pr<R> r; r.x = a.x * b.x + c.x; r.y = a.y * b.y + c.y; return r; }
template <class R> UHC_DEV Pr<R> pmul(Pr<R> a, Pr<R> b) { Pr<R> r; r.x = a.x * b.x; r.y = a.y * b.y; return r; }
template <class R> UHC_DEV Pr<R> padd(Pr<R> a, Pr<R> b) { Pr<R> r; r.x = a.x + b.x; r.y = a.y + b.y; return r; }
// 6-vectors as three pairs
template <class R> UHC_DEV R pdot6(const Pr<R> *a, const Pr<R> *b) { Pr<R> t = pmul(a[0], b[0]); t = pfma(a[1], b[1], t); t = pfma(a[2], b[2], t); return t.x + t.y; }
template <class R> UHC_DEV void paxpy6(R s, const Pr<R> *x, Pr<R> *y) { const Pr<R> ss = pbc(s); y[0] = pfma(ss, x[0], y[0]); y[1] = pfma(ss, x[1], y[1]); y[2] = pfma(ss, x[2], y[2]); }
template <class R> UHC_DEV const Pr<R> *as_pairs(const R *p) { return reinterpret_cast<const Pr<R> *>(p); }

// ------------------------------------------------------------------------------------------------ warp primitives
#ifndef UHC_EMU
template <class R> UHC_DEV R warp_sum(R x) {
#pragma unroll 1
    for (int o = 16; o; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    return x;
}
template <class R> UHC_DEV R warp_max(R x) { for (int o = 16; o; o >>= 1) { R y = __shfl_xor_sync(0xffffffffu, x, o); x = x > y ? x : y; } return x; }
template <class R> UHC_DEV void warp_argmin(R &x, int &i) {
    for (int o = 16; o; o >>= 1) { R y = __shfl_xor_sync(0xffffffffu, x, o); int j = __shfl_xor_sync(0xffffffffu, i, o); if (y < x || (y == x && j < i)) { x = y; i = j; } }
}
#define WSUM(n) warp_sum(n)
#define WMAX(n) warp_max(n)
#define WARGMIN(x, i, ox, oi) { ox = x; oi = i; warp_argmin(ox, oi); }
#define WBALLOT(n) __ballot_sync(0xffffffffu, (n) != 0)
UHC_DEV int warp_excl_scan(int x, int lane) { int p = x; for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, p, o); if (lane >= o) p += t; } return p - x; }
#define WEXSCAN(dst, src) { dst = warp_excl_scan(src, (int)(threadIdx.x & 31)); }
// segmented over the aligned groups of G lanes (G a power of two): every lane gets its group's warp_argmin / bitwise OR
template <class R> UHC_DEV void warp_seg_argmin(R &x, int &i, int G) {
#pragma unroll 1
    for (int o = G >> 1; o; o >>= 1) { R y = __shfl_xor_sync(0xffffffffu, x, o); int j = __shfl_xor_sync(0xffffffffu, i, o); if (y < x || (y == x && j < i)) { x = y; i = j; } }
}
UHC_DEV unsigned warp_seg_or(unsigned x, int G) {
#pragma unroll 1
    for (int o = G >> 1; o; o >>= 1) x |= __shfl_xor_sync(0xffffffffu, x, o);
    return x;
}
#define WSEGARGMIN(x, i, G) warp_seg_argmin(x, i, G)
#define WSEGOR(x, G) { x = warp_seg_or(x, G); }
// dst = src of lane SRCL (a per-lane expression of `lane`), any 32-bit type
#define WSHFLV(dst, src, SRCL) { const int lane = (int)(threadIdx.x & 31); (void)lane; dst = __shfl_sync(0xffffffffu, src, (SRCL)); }
// bodies are numbered depth-first, so subtree(b) = lanes [b, sub_end]: subtree sum = difference of an inclusive warp prefix sum
// The scan steps are a rolled loop over the offsets with the K components inside: the same additions per component, a fifth of the code
template <class R, int K> UHC_DEV void subtree_sum(R (&x)[K], int sub_end, int lane) {
#pragma unroll 1
    for (int o = 1; o < 32; o <<= 1) {
#pragma unroll
        for (int i = 0; i < K; i++) { const R t = __shfl_up_sync(0xffffffffu, x[i], o); if (lane >= o) x[i] += t; }
    }
#pragma unroll
    for (int i = 0; i < K; i++) {
        const R hi = __shfl_sync(0xffffffffu, x[i], sub_end), lo = __shfl_up_sync(0xffffffffu, x[i], 1);
        x[i] = hi - (lane > 0 ? lo : R(0));
    }
}
// root -> leaves accumulation along the tree, x_b <- sum over the chain root .. b, by pointer jumping: after round k every lane holds the sum of
// its 2^(k+1) nearest ancestors-or-self (chains are at most MAXLEVEL + 1 = 9 bodies long -> 4 rounds instead of one per level)
template <class R, int K> UHC_DEV void ancestor_sum(R (&x)[K], int a1, int a2, int a4, int a8) {
    static_assert(MAXLEVEL + 1 <= 16, "four pointer-jumping rounds cover chains of 16 bodies");
#pragma unroll 1
    for (int rnd = 0; rnd < 4; ++rnd) {
        const int src = rnd == 0 ? a1 : (rnd == 1 ? a2 : (rnd == 2 ? a4 : a8));
#pragma unroll
        for (int i = 0; i < K; i++) { const R t = __shfl_sync(0xffffffffu, x[i], src < 0 ? 0 : src); if (src >= 0) x[i] += t; }
    }
}
#define WSUBTREE(n, K, tp) subtree_sum<Real, K>(n, tp.sub_end, tp.lane)
template <class R, int K> UHC_DEV void prefix_sum(R (&x)[K], int lane) {   // inclusive, over the 32 lanes (rolled like subtree_sum)
#pragma unroll 1
    for (int o = 1; o < 32; o <<= 1) {
#pragma unroll
        for (int i = 0; i < K; i++) { const R t = __shfl_up_sync(0xffffffffu, x[i], o); if (lane >= o) x[i] += t; }
    }
}
#define WPREFIX(n, K) prefix_sum<Real, K>(n, (int)(threadIdx.x & 31))
#define WANCESTOR(n, K, tp) ancestor_sum<Real, K>(n, tp.parent, tp.anc2, tp.anc4, tp.anc8)
#else
template <class R> static R emu_sum(const R *x) { R s = 0; for (int i = 0; i < 32; i++) s += x[i]; return s; }
template <class R> static R emu_max(const R *x) { R s = x[0]; for (int i = 1; i < 32; i++) s = x[i] > s ? x[i] : s; return s; }
#define WSUM(n) emu_sum(n)
#define WMAX(n) emu_max(n)
#define WARGMIN(x, i, ox, oi) { ox = x[0]; oi = i[0]; for (int l_ = 1; l_ < 32; l_++) if (x[l_] < ox || (x[l_] == ox && i[l_] < oi)) { ox = x[l_]; oi = i[l_]; } }
static unsigned emu_ballot(const int *x) { unsigned m = 0; for (int i = 0; i < 32; i++) if (x[i]) m |= 1u << i; return m; }
#define WBALLOT(n) emu_ballot(n)
#define WEXSCAN(dst, src) { int run_ = 0; for (int l_ = 0; l_ < 32; l_++) { const int t_ = src[l_]; dst[l_] = run_; run_ += t_; } }
#define WSEGARGMIN(x, i, G) { for (int g_ = 0; g_ < 32; g_ += (G)) { __typeof__(x[0]) ox_ = x[g_]; int oi_ = i[g_]; \
    for (int l_ = g_ + 1; l_ < g_ + (G); l_++) if (x[l_] < ox_ || (x[l_] == ox_ && i[l_] < oi_)) { ox_ = x[l_]; oi_ = i[l_]; } \
    for (int l_ = g_; l_ < g_ + (G); l_++) { x[l_] = ox_; i[l_] = oi_; } } }
#define WSEGOR(x, G) { for (int g_ = 0; g_ < 32; g_ += (G)) { unsigned o_ = 0; for (int l_ = g_; l_ < g_ + (G); l_++) o_ |= x[l_]; for (int l_ = g_; l_ < g_ + (G); l_++) x[l_] = o_; } }
#define WSHFLV(dst, src, SRCL) { __typeof__(src[0]) t_[32]; for (int l_ = 0; l_ < 32; l_++) t_[l_] = src[l_]; for (int lane = 0; lane < 32; lane++) dst[lane] = t_[(SRCL)]; }
template <class R, int K, class TP> static void emu_subtree(R (*x)[K], const TP *tp) {
    R out[32][K];
    for (int b = 0; b < 32; b++) for (int i = 0; i < K; i++) { R s = 0; for (int c = b; c <= tp[b].sub_end && c < 32; c++) s += x[c][i]; out[b][i] = s; }
    for (int b = 0; b < 32; b++) for (int i = 0; i < K; i++) x[b][i] = out[b][i];
}
template <class R, int K, class TP> static void emu_ancestor(R (*x)[K], const TP *tp) {
    for (int b = 1; b < NB; b++) for (int i = 0; i < K; i++) x[b][i] += x[tp[b].parent][i];   // depth-first order: parents come first
}
#define WSUBTREE(n, K, tp) emu_subtree<Real, K>(n, tp)
#define WPREFIX(n, K) { for (int l_ = 1; l_ < 32; l_++) for (int i_ = 0; i_ < K; i_++) n[l_][i_] += n[l_ - 1][i_]; }
#define WANCESTOR(n, K, tp) emu_ancestor<Real, K>(n, tp)
#endif
// population count and the position of the k-th set bit (k = 0: the lowest; -1 when m has no more than k set bits)
#ifndef UHC_EMU
UHC_DEV int popc32(unsigned m) { return __popc(m); }
UHC_DEV int nth_bit(unsigned m, int k) { return (int)__fns(m, 0u, k + 1); }
#else
UHC_DEV int popc32(unsigned m) { return __builtin_popcount(m); }
UHC_DEV int nth_bit(unsigned m, int k) { for (int j = 0; j < k && m; ++j) m &= m - 1; return m ? __builtin_ctz(m) : -1; }
#endif

// ================================================================================================ articulated-body solve
// Every linear system of a substep has the form  H x = b,  H = sum_b J_b^T Ihat_b J_b + diag(arm)  with J_b x = sum_{i on chain(b)} S_i x_i:
//   stable PD        Ihat = I_b (previous forward pass),  arm = armature + kd dt        (humanoid_im.py:1014-1031, dense cho_solve there)
//   smooth dynamics  Ihat = I_b,                           arm = armature                (mj_fwdAcceleration)
//   Newton direction Ihat = I_b + K_b (active contacts),   arm = armature                (Hessian of the constraint cost)
// so one O(n) articulated-body sweep solves all three without ever forming the joint-space matrix: lane = body, articulated
// inertia (sym 6x6) / bias wrench in registers, leaves -> root then root -> leaves, children/parent exchange by warp shuffles.
// World-aligned spatial quantities about the common point O need no frame transforms between bodies.
struct LaneTopo { signed char lane, parent, depth, sub_end, ch0, ch1, ch2, anc2, anc4, anc8; short hnum; int hadr; };   // lane = body: tree links (anc_k: ancestor k levels up, -1 = none), hull vertex range
template <class Real>
UHC_DEV LaneTopo lane_topo(const Model<Real> &m, int lane) {
    LaneTopo t; t.lane = lane;
    const int b = lane < NB ? lane : NB - 1;
    t.parent = UHC_LDG(m.parent + b); t.depth = lane < NB ? UHC_LDG(m.depth + b) : 99; t.sub_end = lane < NB ? UHC_LDG(m.body_sub_end + b) : lane;
    const int c0 = UHC_LDG(m.child_adr + b), c1 = UHC_LDG(m.child_adr + b + 1);
    t.ch0 = (lane < NB && c0 < c1) ? UHC_LDG(m.child + c0) : -1;
    t.ch1 = (lane < NB && c0 + 1 < c1) ? UHC_LDG(m.child + c0 + 1) : -1;
    t.ch2 = (lane < NB && c0 + 2 < c1) ? UHC_LDG(m.child + c0 + 2) : -1;
    t.hadr = UHC_LDG(m.hull_adr + b); t.hnum = lane < NB ? UHC_LDG(m.hull_num + b) : 0;
    int a = lane < NB ? b : -1;
    t.anc2 = t.anc4 = t.anc8 = -1;
    for (int k = 1; k <= 8 && a >= 0; ++k) { a = a > 0 ? UHC_LDG(m.parent + a) : -1; if (k == 2) t.anc2 = a; if (k == 4) t.anc4 = a; if (k == 8) t.anc8 = a; }
    if (lane >= NB) t.parent = -1;
    return t;
}
#ifndef UHC_EMU
// the per-lane tree links live in shared memory (staged once per CTA): functions take them by reference without a local-memory copy
#define TOPO_DECL(m) const LaneTopo &tp = reinterpret_cast<const LaneTopo *>((m).topo_s)[threadIdx.x & 31]
#define TP tp
#define TP_OF(m, tp, b) (reinterpret_cast<const LaneTopo *>((m).topo_s)[b])
// parents at depth `lvl` add their children's K floats (children sit at lvl + 1)
template <class R, int K> UHC_DEV void gather_children(R (&x)[K], const LaneTopo &tp, int lvl) {
#pragma unroll 1
    for (int r = 0; r < 3; r++) {
        const int src = r == 0 ? tp.ch0 : (r == 1 ? tp.ch1 : tp.ch2);
        const bool act = tp.depth == lvl && src >= 0;
        if (!__any_sync(0xffffffffu, act)) continue;
#pragma unroll
        for (int i = 0; i < K; i++) { const R t = __shfl_sync(0xffffffffu, x[i], src < 0 ? tp.lane : src); if (act) x[i] += t; }
    }
}
template <class R, int K> UHC_DEV void fetch_parent(const R (&x)[K], R (&o)[K], const LaneTopo &tp) {
#pragma unroll
    for (int i = 0; i < K; i++) o[i] = __shfl_sync(0xffffffffu, x[i], tp.parent < 0 ? 0 : tp.parent);
}
#define WGATHER(n, K, tp, lvl) gather_children<Real, K>(n, tp, lvl)
#define WFETCHP(n, o, K, tp) fetch_parent<Real, K>(n, o, tp)
// dst[i] = src[i] of lane SRCL (a per-lane expression), i < K ; WANY: warp-wide OR of a per-lane flag
#define WSHFL(dst, src, K, SRCL) { const int lane = (int)(threadIdx.x & 31); const int s_ = (SRCL); (void)lane; _Pragma("unroll") for (int i_ = 0; i_ < K; i_++) dst[i_] = __shfl_sync(0xffffffffu, src[i_], s_); }
#define WSHFL1(dst, src, SRCL) { const int lane = (int)(threadIdx.x & 31); (void)lane; dst = __shfl_sync(0xffffffffu, src, (SRCL)); }
#define WANY(flag) __any_sync(0xffffffffu, flag)
#else
#define TOPO_DECL(m) LaneTopo tp[32]; for (int l_ = 0; l_ < 32; l_++) tp[l_] = lane_topo(m, l_)
#define TP tp[lane]
#define TP_OF(m, tp, b) (tp[b])
template <class R, int K> static void emu_gather(R (*x)[K], const LaneTopo *tp, int lvl) {
    for (int b = 0; b < NB; b++) if (tp[b].depth == lvl) {
        const int ch[3] = {tp[b].ch0, tp[b].ch1, tp[b].ch2};
        for (int r = 0; r < 3; r++) if (ch[r] >= 0) for (int i = 0; i < K; i++) x[b][i] += x[ch[r]][i];
    }
}
template <class R, int K> static void emu_fetchp(R (*x)[K], R (*o)[K], const LaneTopo *tp) {
    for (int b = 0; b < 32; b++) for (int i = 0; i < K; i++) o[b][i] = x[tp[b].parent < 0 ? 0 : tp[b].parent][i];
}
#define WGATHER(n, K, tp, lvl) emu_gather<Real, K>(n, tp, lvl)
#define WFETCHP(n, o, K, tp) emu_fetchp<Real, K>(n, o, tp)
#define WSHFL(dst, src, K, SRCL) { Real t_[32][K]; for (int l_ = 0; l_ < 32; l_++) for (int i_ = 0; i_ < K; i_++) t_[l_][i_] = src[l_][i_]; \
    for (int lane = 0; lane < 32; lane++) { const int s_ = (SRCL); for (int i_ = 0; i_ < K; i_++) dst[lane][i_] = t_[s_][i_]; } }
#define WSHFL1(dst, src, SRCL) { Real t_[32]; for (int l_ = 0; l_ < 32; l_++) t_[l_] = src[l_]; for (int lane = 0; lane < 32; lane++) dst = t_[(SRCL)]; }
#define WANY(flag) emu_ballot(flag)
#endif

// pyramid edge directions d_e = n +- mu t  for n = +z, t1 = +y, t2 = -x
template <class Real> UHC_DEV void edge_dir(int e, Real mu, Real *d) {
    d[0] = e == 2 ? -mu : (e == 3 ? mu : Real(0));
    d[1] = e == 0 ? mu : (e == 1 ? -mu : Real(0));
    d[2] = 1;
}

// Row r of a body's 6x6 matrices, (w, v) ordering.  The lane's row is described by the unit vector u = e_(r mod 3) and
// ang = (r < 3), so that every lane runs the same arithmetic (no per-row branches or select chains).
// Contact matrix of body b:  K_b = sum_{own contacts} X^T W X,  X = [-[p]x 1] (point velocity = v + w x p),
// W = D sum_{active edges} d d^T with pyramid edges d = (+-mu or 0, +-mu or 0, 1)  ->  W_xy = 0.
// Row r of X^T W X = [p x (W xr), W xr] with xr = column r of X = (ang ? u x p : u).
template <class Real>
UHC_DEV void contact_matrix_row(const Model<Real> &m, const Work<Real> &w, int b, const Real *u, bool ang, Real *row) {
    const Real mu = m.mu, mu2 = mu * mu;
    for (int c = w.bcon_adr[b]; c < w.bcon_adr[b + 1]; ++c) {
        const Real D = w.cD[c];
        const Real a0 = w.cres[c][0] < 0 ? D : Real(0), a1 = w.cres[c][1] < 0 ? D : Real(0), a2 = w.cres[c][2] < 0 ? D : Real(0), a3 = w.cres[c][3] < 0 ? D : Real(0);
        const Real Wxx = mu2 * (a2 + a3), Wyy = mu2 * (a0 + a1), Wzz = (a0 + a1) + (a2 + a3), Wxz = mu * (a3 - a2), Wyz = mu * (a0 - a1);
        const Real *p = w.cr[c];
        Real t[3], xr[3], v[3], pv[3];
        cross3(u, p, t);
        xr[0] = ang ? t[0] : u[0]; xr[1] = ang ? t[1] : u[1]; xr[2] = ang ? t[2] : u[2];
        v[0] = Wxx * xr[0] + Wxz * xr[2]; v[1] = Wyy * xr[1] + Wyz * xr[2]; v[2] = Wxz * xr[0] + Wyz * xr[1] + Wzz * xr[2];
        cross3(p, v, pv);
        row[0] += pv[0]; row[1] += pv[1]; row[2] += pv[2]; row[3] += v[0]; row[4] += v[1]; row[5] += v[2];
    }
}
// Rigid spatial inertia (m, h = m c, J about O):  [[J, [h]x], [-[h]x, m 1]].  Angular row q: [J u, u x h]; linear row q: [h x u, m u].
template <class Real>
UHC_DEV void rigid_row(const Real *I, const Real *u, bool ang, Real *row) {
    const Real *h = I + 1;
    const Real Ju0 = I[4] * u[0] + I[7] * u[1] + I[8] * u[2], Ju1 = I[7] * u[0] + I[5] * u[1] + I[9] * u[2], Ju2 = I[8] * u[0] + I[9] * u[1] + I[6] * u[2];
    Real t[3]; cross3(u, h, t);
    row[0] = ang ? Ju0 : -t[0]; row[1] = ang ? Ju1 : -t[1]; row[2] = ang ? Ju2 : -t[2];
    row[3] = ang ? t[0] : I[0] * u[0]; row[4] = ang ? t[1] : I[0] * u[1]; row[5] = ang ? t[2] : I[0] * u[2];
}

// x <- H^-1 x  (x: 75-vector in shared memory).  arm_scale: extra joint-space diagonal = arm_scale * kd_i (0 for none).
//
// H = sum_b J_b^T IA_b J_b + diag(arm) is the matrix of a TREE of bodies coupled by joints; the tree can be eliminated towards any
// of its bodies.  The level table (Model::lvl_pack, built by uhc_b200/model.py) hangs it from its centre (Spine for SMPL): 7 levels of
// <= 5 bodies instead of the 9 of the kinematic tree.  A joint on the path centre -> Pelvis is crossed against its kinematic
// direction: with y = -qacc_j it reads a_child = a_parent + S_j y like every other joint, so its right-hand side and solution
// just change sign.  The free joint (no armature) turns into the wrench  S_0^-T b_0  applied to the Pelvis body, and the centre
// body's own spatial acceleration solves the 6 x 6 system  IA a = -pA  directly (Gauss-Jordan across the six lanes holding its rows).
//
// Lane layout: the <= 5 bodies of one level are processed together, 6 lanes per body (lane = 6 g + r owns ROW r of that body's
// articulated inertia; the bias wrench is replicated in the group).  The three dofs of a body's joint are eliminated as ONE block:
//   leaves -> centre:  U = IA S (6x3), D = S^T U + arm (3x3), u = b - S^T pA ;  IA -= U D^-1 U^T ;  pA += U D^-1 u
//   centre -> leaves:  y = D^-1 u - (U D^-1)^T a_parent ;  a = a_parent + S y
// so only  U D^-1  and  D^-1 u  are kept for the back-substitution.
template <class Real>
UHC_DEVNI void aba_solve(const Model<Real> &m, Work<Real> &w, Real arm_scale, bool use_contacts, Real *x) {
    typedef Pr<Real> P;
    LVARA(P, row, 3); LVARA(P, pA, 3); LVARA(P, nrow, 3); LVARA(P, npA, 3); LVARA(Real, trow, 6); LVARA(Real, tpA, 6);
    LVARA(Real, Ur, 3);
    Real *arm = w.Mp;     // joint-space diagonal (armature + arm_scale kd)
    LVAR(int, body); LVAR(int, src); LVAR(int, act); LVAR(int, rr); LVAR(int, ent); LVAR(int, entn);
    const int *lp = m.lvl_pack;   // once: for the compiler the stores of the sweeps may alias the Model, and every level would reload the pointer
    const int nlvl = (UHC_LDT(lp) >> 26) & 15;
    int nslot_n = (UHC_LDT(lp + (nlvl - 1) * LVL_G) >> 18) & 3;   // uniform: most children any body of the level has (fetched one level ahead)
    LANES_BEGIN
    for (int i = 0; i < 3; i++) { LVA(row)[i] = pbc(Real(0)); LVA(pA)[i] = pbc(Real(0)); }
    LV(rr) = lane - 6 * (lane / 6);
    LV(entn) = lane < 6 * LVL_G ? UHC_LDT(lp + (nlvl - 1) * LVL_G + lane / 6) : 0;
    const bool limits = use_contacts && w.nlim > 0;     // an active joint-limit row (J = +-e_i) adds its D to the joint-space diagonal of the Hessian
#pragma unroll 1
    for (int i = lane; i < NV; i += 32) {
        Real d = UHC_LDT(m.dof_f + 4 * i) + arm_scale * UHC_LDT(m.dof_f + 4 * i + 2);   // joint-space diagonal
        if (limits && w.tau[i] != 0 && w.as_[i] < 0) d += abs_(w.tau[i]);
        arm[i] = d;
    }
    LANES_END
#pragma unroll 1
    for (int lvl = nlvl - 1; lvl >= 0; --lvl) {
        const int nslot = nslot_n;
        if (lvl > 0) nslot_n = (UHC_LDT(lp + (lvl - 1) * LVL_G) >> 18) & 3;
        LANES_BEGIN
        const int g = lane / 6, r = LV(rr);
        const int e = LV(entn);            // this level's table entry was fetched one level ahead
        LV(entn) = (g < LVL_G && lvl > 0) ? UHC_LDT(lp + (lvl - 1) * LVL_G + g) : 0;
        const int b = (e & 63) - 1;
        LV(ent) = e; LV(body) = b;
        Real ri[6] = {0, 0, 0, 0, 0, 0}, pi[6] = {0, 0, 0, 0, 0, 0};
        if (b >= 0) {
            const int q = r < 3 ? r : r - 3;
            const Real u[3] = {q == 0 ? Real(1) : Real(0), q == 1 ? Real(1) : Real(0), q == 2 ? Real(1) : Real(0)};
            rigid_row(w.Ib[b], u, r < 3, ri);
            if (use_contacts) contact_matrix_row(m, w, b, u, r < 3, ri);
            if (b == 0) {   // the free joint's right-hand side is a wrench on the Pelvis: bias = -S_0^-T b_0 (S_0 = [0 R; 1 0] is orthogonal)
                const Real b3 = x[3], b4 = x[4], b5 = x[5];
                for (int i = 0; i < 3; i++) { pi[i] = -(w.S[3][i] * b3 + w.S[4][i] * b4 + w.S[5][i] * b5); pi[3 + i] = -x[i]; }
            }
        }
        for (int i = 0; i < 3; i++) { LVA(nrow)[i].x = ri[2 * i]; LVA(nrow)[i].y = ri[2 * i + 1]; LVA(npA)[i].x = pi[2 * i]; LVA(npA)[i].y = pi[2 * i + 1]; }
        LANES_END_R
#pragma unroll 1
        for (int k = 0; k < nslot; ++k) {  // children of this level's bodies: they sit one level deeper, their results are still in row / pA
            LANES_BEGIN
            const int cg = ((LV(ent) >> (9 + 3 * k)) & 7) - 1;
            LV(act) = cg >= 0; LV(src) = cg >= 0 ? cg * 6 + LV(rr) : lane;
            for (int i = 0; i < 3; i++) { LVA(trow)[2 * i] = LVA(row)[i].x; LVA(trow)[2 * i + 1] = LVA(row)[i].y; LVA(tpA)[2 * i] = LVA(pA)[i].x; LVA(tpA)[2 * i + 1] = LVA(pA)[i].y; }
            LANES_END_R
            WSHFL(trow, trow, 6, LV(src));
            WSHFL(tpA, tpA, 6, LV(src));
            LANES_BEGIN
            if (LV(act)) for (int i = 0; i < 3; i++) {
                P a, c; a.x = LVA(trow)[2 * i]; a.y = LVA(trow)[2 * i + 1]; c.x = LVA(tpA)[2 * i]; c.y = LVA(tpA)[2 * i + 1];
                LVA(nrow)[i] = padd(LVA(nrow)[i], a); LVA(npA)[i] = padd(LVA(npA)[i], c);
            }
            LANES_END_R
        }
        LANES_BEGIN
        for (int i = 0; i < 3; i++) { LVA(row)[i] = LVA(nrow)[i]; LVA(pA)[i] = LVA(npA)[i]; }
        LANES_END_R
        if (lvl == 0) break;               // the centre body: solved directly below
        {
            LANES_BEGIN   // this lane's entries of U = IA S
            const int b = LV(body), d0 = 3 * ((LV(ent) >> 20) & 31);
            P Sk[3][3];                    // S of the joint in registers first: a store to aU may alias S for the compiler
#pragma unroll
            for (int k = 0; k < 3; k++) for (int i = 0; i < 3; i++) Sk[k][i] = as_pairs(w.S[d0 + k])[i];
#pragma unroll
            for (int k = 0; k < 3; k++) {
                const Real u = pdot6(LVA(row), Sk[k]);
                LVA(Ur)[k] = u;
                if (b >= 0) w.aU[d0 + k][LV(rr)] = u;
            }
            LANES_END
            LANES_BEGIN
            const int b = LV(body), d0 = 3 * ((LV(ent) >> 20) & 31), r = LV(rr);
            const Real sg = ((LV(ent) >> 25) & 1) ? Real(-1) : Real(1);   // joint crossed against its kinematic direction
            P U0[3], U1[3], U2[3], S0[3], S1[3], S2[3];
#pragma unroll
            for (int i = 0; i < 3; i++) {
                U0[i] = as_pairs(w.aU[d0])[i]; U1[i] = as_pairs(w.aU[d0 + 1])[i]; U2[i] = as_pairs(w.aU[d0 + 2])[i];
                S0[i] = as_pairs(w.S[d0])[i]; S1[i] = as_pairs(w.S[d0 + 1])[i]; S2[i] = as_pairs(w.S[d0 + 2])[i];
            }
            // D = S^T U + arm (symmetric), u = b - S^T pA
            const Real D00 = pdot6(S0, U0) + arm[d0], D11 = pdot6(S1, U1) + arm[d0 + 1], D22 = pdot6(S2, U2) + arm[d0 + 2];
            const Real D01 = pdot6(S0, U1), D02 = pdot6(S0, U2), D12 = pdot6(S1, U2);
            const Real u0 = sg * x[d0] - pdot6(S0, LVA(pA)), u1 = sg * x[d0 + 1] - pdot6(S1, LVA(pA)), u2 = sg * x[d0 + 2] - pdot6(S2, LVA(pA));
            // inverse by the adjugate (D is symmetric positive definite and small)
            const Real c00 = D11 * D22 - D12 * D12, c01 = D02 * D12 - D01 * D22, c02 = D01 * D12 - D02 * D11;
            const Real c11 = D00 * D22 - D02 * D02, c12 = D01 * D02 - D00 * D12, c22 = D00 * D11 - D01 * D01;
            const Real id = rcp_(D00 * c00 + D01 * c01 + D02 * c02);
            const Real i00 = c00 * id, i01 = c01 * id, i02 = c02 * id, i11 = c11 * id, i12 = c12 * id, i22 = c22 * id;
            const Real a0 = LVA(Ur)[0], a1 = LVA(Ur)[1], a2 = LVA(Ur)[2];
            const Real W0 = a0 * i00 + a1 * i01 + a2 * i02, W1 = a0 * i01 + a1 * i11 + a2 * i12, W2 = a0 * i02 + a1 * i12 + a2 * i22;   // row r of U D^-1
            const Real v0 = u0 * i00 + u1 * i01 + u2 * i02, v1 = u0 * i01 + u1 * i11 + u2 * i12, v2 = u0 * i02 + u1 * i12 + u2 * i22;   // D^-1 u
            paxpy6(-W0, U0, LVA(row)); paxpy6(-W1, U1, LVA(row)); paxpy6(-W2, U2, LVA(row));
            paxpy6(v0, U0, LVA(pA)); paxpy6(v1, U1, LVA(pA)); paxpy6(v2, U2, LVA(pA));
            LVA(Ur)[0] = W0; LVA(Ur)[1] = W1; LVA(Ur)[2] = W2;
            if (b >= 0 && r == 0) { w.au[d0] = v0; w.au[d0 + 1] = v1; w.au[d0 + 2] = v2; }
            LANES_END
            LANES_BEGIN   // U D^-1 replaces U (after every lane of the group has read U)
            const int b = LV(body), d0 = 3 * ((LV(ent) >> 20) & 31);
            if (b >= 0) { w.aU[d0][LV(rr)] = LVA(Ur)[0]; w.aU[d0 + 1][LV(rr)] = LVA(Ur)[1]; w.aU[d0 + 2][LV(rr)] = LVA(Ur)[2]; }
            LANES_END
        }
    }
    // ---- the centre body (no joint above it): IA a = -pA, a 6 x 6 symmetric positive definite system whose row r sits in lane r --
    // Gauss-Jordan elimination across the six lanes (one broadcast of the pivot row per step), no pivoting needed
    LVARA(Real, Mx, 7); LVARA(Real, Pk, 7); LVAR(Real, sol); LVARA(Real, acc, 6); LVARA(Real, pacc, 6);
    LANES_BEGIN
    for (int i = 0; i < 3; i++) { LVA(Mx)[2 * i] = LVA(row)[i].x; LVA(Mx)[2 * i + 1] = LVA(row)[i].y; }
    const P t = LV(rr) < 2 ? LVA(pA)[0] : (LV(rr) < 4 ? LVA(pA)[1] : LVA(pA)[2]);
    LVA(Mx)[6] = -((LV(rr) & 1) ? t.y : t.x);
    LANES_END_R
#pragma unroll
    for (int kk = 0; kk < 6; ++kk) {
        const int k = kk < 3 ? kk + 3 : kk - 3;   // linear rows first: their block is m 1 (large, diagonal), and what is left for the angular rows is the
                                                  // inertia about the centre of mass -- eliminating the angular rows first cancels instead
        WSHFL(Pk, Mx, 7, k);
        LANES_BEGIN
        if (lane != k && lane < 6) {
            const Real f = LVA(Mx)[k] * rcp_(LVA(Pk)[k]);
#pragma unroll
            for (int j = 0; j < 7; j++) LVA(Mx)[j] -= f * LVA(Pk)[j];
        }
        LANES_END_R
    }
    LANES_BEGIN
    const int r = LV(rr);
    const Real d = r == 0 ? LVA(Mx)[0] : r == 1 ? LVA(Mx)[1] : r == 2 ? LVA(Mx)[2] : r == 3 ? LVA(Mx)[3] : r == 4 ? LVA(Mx)[4] : LVA(Mx)[5];
    LV(sol) = lane < 6 ? LVA(Mx)[6] * rcp_(d) : Real(0);
    LANES_END_R
    WSHFL1(LVA(pacc)[0], sol, 0); WSHFL1(LVA(pacc)[1], sol, 1); WSHFL1(LVA(pacc)[2], sol, 2);
    WSHFL1(LVA(pacc)[3], sol, 3); WSHFL1(LVA(pacc)[4], sol, 4); WSHFL1(LVA(pacc)[5], sol, 5);
    // centre -> leaves (the spatial acceleration a is replicated in the 6 lanes of a group; every lane starts from the centre body's)
    LANES_BEGIN
    const int bc = (UHC_LDT(lp) & 63) - 1;
    if (use_contacts && lane < 6) w.Ab[bc][lane] = LV(sol);
    LV(entn) = (lane < 6 * LVL_G && nlvl > 1) ? UHC_LDT(lp + LVL_G + lane / 6) : 0;
    LANES_END
#pragma unroll 1
    for (int lvl = 1; lvl < nlvl; ++lvl) {
        LANES_BEGIN
        const int g = lane / 6;
        const int e = LV(entn);
        LV(entn) = (g < LVL_G && lvl + 1 < nlvl) ? UHC_LDT(lp + (lvl + 1) * LVL_G + g) : 0;
        const int b = (e & 63) - 1;
        LV(body) = b; LV(ent) = e;
        LV(src) = b >= 0 ? ((e >> 6) & 7) * 6 : lane;
        LANES_END_R
        WSHFL(acc, pacc, 6, LV(src));
        LANES_BEGIN
        const int b = LV(body), r = LV(rr);
        P a[3];
        for (int i = 0; i < 3; i++) { a[i].x = LVA(acc)[2 * i]; a[i].y = LVA(acc)[2 * i + 1]; }
        if (b >= 0) {
            const Real sg = ((LV(ent) >> 25) & 1) ? Real(-1) : Real(1);
            const int d0 = 3 * ((LV(ent) >> 20) & 31);
            // every operand of the level in registers first: for the compiler the stores to x below may alias S, and each S load would wait for them
            P U0[3], U1[3], U2[3], S0[3], S1[3], S2[3];
#pragma unroll
            for (int i = 0; i < 3; i++) {
                U0[i] = as_pairs(w.aU[d0])[i]; U1[i] = as_pairs(w.aU[d0 + 1])[i]; U2[i] = as_pairs(w.aU[d0 + 2])[i];
                S0[i] = as_pairs(w.S[d0])[i]; S1[i] = as_pairs(w.S[d0 + 1])[i]; S2[i] = as_pairs(w.S[d0 + 2])[i];
            }
            const Real au0 = w.au[d0], au1 = w.au[d0 + 1], au2 = w.au[d0 + 2];
            const Real x0 = au0 - pdot6(U0, a), x1 = au1 - pdot6(U1, a), x2 = au2 - pdot6(U2, a);
            if (r == 0) { x[d0] = sg * x0; x[d0 + 1] = sg * x1; x[d0 + 2] = sg * x2; }
            paxpy6(x0, S0, a); paxpy6(x1, S1, a); paxpy6(x2, S2, a);
            if (b == 0 && r == 0) {   // free-joint accelerations from the Pelvis spatial acceleration: qacc_0 = S_0^-1 a = S_0^T a
                x[0] = a[1].y; x[1] = a[2].x; x[2] = a[2].y;
                for (int k = 0; k < 3; k++) x[3 + k] = w.S[3 + k][0] * a[0].x + w.S[3 + k][1] * a[0].y + w.S[3 + k][2] * a[1].x;
            }
        }
        for (int i = 0; i < 3; i++) { LVA(pacc)[2 * i] = a[i].x; LVA(pacc)[2 * i + 1] = a[i].y; }
        if (use_contacts && b >= 0) {   // the body's spatial acceleration J_b x for the Newton step's contact rows (lane r of the group stores component r)
            const P t = r < 2 ? a[0] : (r < 4 ? a[1] : a[2]);
            w.Ab[b][r] = (r & 1) ? t.y : t.x;
        }
        LANES_END
    }
}

// ================================================================================================ kinematics + RNE
// One body's step of the forward pass, from its parent's pose R / pos, spatial velocity V and velocity-product acceleration A (in place) to
// its own.  The chain of body b applies them root -> b; the motion subspaces are stored only by the lane that owns the body (store_S).
// The root: free joint (translation dofs along world axes, rotation dofs about the body-frame axes through O)
template <class Real>
UHC_DEV void kin_root_step(const Model<Real> &m, Work<Real> &w, Real *R, Real *pos, Real *V, Real *A, bool store_S) {
    Real qn[4] = {w.q[3], w.q[4], w.q[5], w.q[6]};
    Real n = rsqrt_(qn[0] * qn[0] + qn[1] * qn[1] + qn[2] * qn[2] + qn[3] * qn[3]);
    for (int i = 0; i < 4; i++) qn[i] *= n;
    q2mat(qn, R);
    pos[0] = w.q[0]; pos[1] = w.q[1]; pos[2] = w.q[2];
    if (store_S) {
        for (int k = 0; k < 3; k++) {  // translation dofs, world axes
            for (int i = 0; i < 6; i++) w.S[k][i] = 0;
            w.S[k][3 + k] = 1;
        }
        for (int k = 0; k < 3; k++) {  // rotation dofs: body-frame axes through O
            w.S[3 + k][0] = R[k]; w.S[3 + k][1] = R[3 + k]; w.S[3 + k][2] = R[6 + k];
            w.S[3 + k][3] = w.S[3 + k][4] = w.S[3 + k][5] = 0;
        }
    }
    Real wl[3] = {w.v[3], w.v[4], w.v[5]}, ww[3], t[3];
    mv3(R, wl, ww);
    V[0] = ww[0]; V[1] = ww[1]; V[2] = ww[2]; V[3] = w.v[0]; V[4] = w.v[1]; V[5] = w.v[2];
    cross3(ww, V + 3, t);  // spatial acceleration of the free body with qacc = 0 is (0, -w x v); minus gravity
    A[0] = A[1] = A[2] = 0; A[3] = -t[0]; A[4] = -t[1]; A[5] = -t[2] - m.gravz;
}
// Body b >= 1: body-frame offset off[3] in the parent's frame, then three hinges z, y, x, each seen in the frame produced by the previous ones
// (sc: sin, cos of the three joint angles)
template <class Real>
UHC_DEV void kin_hinge_step(Work<Real> &w, int b, const Real *off, const Real *sc, Real *R, Real *pos, Real *V, Real *A, bool store_S) {
    Real p[3];
    mv3(R, off, p);
    for (int i = 0; i < 3; i++) pos[i] += p[i];
    const Real r[3] = {pos[0] - w.q[0], pos[1] - w.q[1], pos[2] - w.q[2]};
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        const int dof = 6 + 3 * (b - 1) + j, col = 2 - j;
        Real ax[3] = {R[col], R[3 + col], R[6 + col]}, t[3]; alignas(16) Real Sj[6], Sd[6];
        cross3(r, ax, t);
        Sj[0] = ax[0]; Sj[1] = ax[1]; Sj[2] = ax[2]; Sj[3] = t[0]; Sj[4] = t[1]; Sj[5] = t[2];
        cross3(V, Sj, Sd);              // Sdot = V x_m S = (w x a, w x b + v x a)
        cross3(V, Sj + 3, Sd + 3);
        cross3(V + 3, Sj, t);
        Sd[3] += t[0]; Sd[4] += t[1]; Sd[5] += t[2];
        const Real qd = w.v[dof];
        if (store_S) for (int i = 0; i < 6; i++) w.S[dof][i] = Sj[i];
        paxpy6(qd, reinterpret_cast<const Pr<Real> *>(Sd), reinterpret_cast<Pr<Real> *>(A));
        paxpy6(qd, reinterpret_cast<const Pr<Real> *>(Sj), reinterpret_cast<Pr<Real> *>(V));
        const Real sn = sc[2 * j], cs = sc[2 * j + 1];
        // R <- R * Rot(axis col, angle): rotate the two other columns
        const int c1 = (col + 1) % 3, c2 = (col + 2) % 3;
        for (int i = 0; i < 3; i++) {
            const Real u = R[3 * i + c1], v2 = R[3 * i + c2];
            R[3 * i + c1] = cs * u + sn * v2;
            R[3 * i + c2] = -sn * u + cs * v2;
        }
    }
}
#ifndef UHC_EMU
#define LGET(n, i, src) __shfl_sync(0xffffffffu, n[i], (src))   // inside a lane block, every lane: element i of lane src's n
#else
#define LGET(n, i, src) n[src][i]
#endif

// Forward pass, lane = body: pose, motion subspaces S (about O = root position), spatial velocity V
// and velocity-product acceleration A (gravity folded in as a base acceleration), then per-body rigid inertia and the
// inertial wrench F = I A + V x* (I V); subtree wrenches by warp prefix sums.
// Every lane composes its own chain root -> body with the same steps (and so the same bits) its ancestors' lanes compute for themselves:
// no level-by-level hand-off through shared memory.
// MuJoCo semantics: SURVEY.md Appendix B (mj_kinematics / mj_comPos / mj_rne / mj_crb).
template <class Real, class TPT>
UHC_DEV void kin_rne_forward(const Model<Real> &m, Work<Real> &w, const TPT &tp, bool clk = false) {
    // joint-angle sines / cosines of every body in one lane = body pass; the chains fetch their ancestors' from the owning lanes
    LVARA(Real, sc, 6);
    LANES_BEGIN
    const int b = lane;
    for (int j = 0; j < 3; ++j) {
        Real sn = 0, cs = 1;
        if (b >= 1 && b < NB) sincos_(w.q[7 + 3 * (b - 1) + j], &sn, &cs);
        LVA(sc)[2 * j] = sn; LVA(sc)[2 * j + 1] = cs;
    }
    LANES_END_R
    PSUB(clk, w, PS_KIN_SINCOS);
    LANES_BEGIN
    const int b = lane, depth = b < NB ? (int)TP.depth : 0;
    Real R[9], pos[3]; alignas(16) Real V[6], A[6];
    kin_root_step(m, w, R, pos, V, A, b == 0);
    int a = 0;       // the chain's body done last (depth d - 1)
#pragma unroll 1
    for (int d = 1; d <= MAXLEVEL; ++d) {
        // next on the chain: the child of a whose subtree (depth-first numbering: [child, ..]) holds b
        const LaneTopo &ta = TP_OF(m, tp, a);
        int c = ta.ch0;
        if (ta.ch1 >= 0 && ta.ch1 <= b) c = ta.ch1;
        if (ta.ch2 >= 0 && ta.ch2 <= b) c = ta.ch2;
        const bool act = d <= depth;
        if (!act) c = 0;
        Real s[6];
        for (int i = 0; i < 6; i++) s[i] = LGET(sc, i, c);      // every lane takes part in the exchange
        if (act) {
            const Real *bf = m.body_f + c * BODYF;
            const Real off[3] = {UHC_LDG(bf), UHC_LDG(bf + 1), UHC_LDG(bf + 2)};
            kin_hinge_step(w, c, off, s, R, pos, V, A, c == b);
            a = c;
        }
    }
    if (b < NB) {
        for (int i = 0; i < 3; i++) w.xpos[b][i] = pos[i];
        for (int i = 0; i < 9; i++) w.xmat[b][i] = R[i];
        for (int i = 0; i < 6; i++) { w.Vb[b][i] = V[i]; w.Ab[b][i] = A[i]; }
    }
    LANES_END
    PSUB(clk, w, PS_KIN_LEVELS);
    // rigid inertia about O in world axes, inertial wrench; then subtree sums (composite inertia, subtree wrench)
    LVARA(Real, IF, 6);
    LANES_BEGIN
    const int b = lane;
    for (int i = 0; i < 6; i++) LVA(IF)[i] = 0;
    if (b < NB) {
        const Real *bf = m.body_f + b * BODYF;
        const Real *R = w.xmat[b], *pos = w.xpos[b], *V = w.Vb[b], *A = w.Ab[b];
        Real cl[3], c[3], I[10], T[9];
        const Real ip[3] = {UHC_LDG(bf + 3), UHC_LDG(bf + 4), UHC_LDG(bf + 5)};
        mv3(R, ip, cl);
        for (int i = 0; i < 3; i++) { w.xipos[b][i] = pos[i] + cl[i]; c[i] = pos[i] + cl[i] - w.q[i]; }
        const Real ms = UHC_LDG(bf + 6);
        const Real i0 = UHC_LDG(bf + 7), i1 = UHC_LDG(bf + 8), i2 = UHC_LDG(bf + 9), i3 = UHC_LDG(bf + 10), i4 = UHC_LDG(bf + 11), i5 = UHC_LDG(bf + 12);
        const Real Il[9] = {i0, i3, i4, i3, i1, i5, i4, i5, i2};
        for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) T[3 * i + j] = R[3 * i] * Il[j] + R[3 * i + 1] * Il[3 + j] + R[3 * i + 2] * Il[6 + j];
        const Real cc = dot3(c, c);
        const int ii[6] = {0, 1, 2, 0, 0, 1}, jj[6] = {0, 1, 2, 1, 2, 2};
        I[0] = ms; I[1] = ms * c[0]; I[2] = ms * c[1]; I[3] = ms * c[2];
        for (int e = 0; e < 6; e++) {
            const int i = ii[e], j = jj[e];
            I[4 + e] = T[3 * i] * R[3 * j] + T[3 * i + 1] * R[3 * j + 1] + T[3 * i + 2] * R[3 * j + 2] + ms * ((i == j ? cc : Real(0)) - c[i] * c[j]);
        }
        Real IA[6], IV[6], t[3], t2[3];
        rigid_mul(I, A, IA); rigid_mul(I, V, IV);
        cross3(V, IV, t); cross3(V + 3, IV + 3, t2);   // V x* F = (w x n + v x f, w x f)
        IA[0] += t[0] + t2[0]; IA[1] += t[1] + t2[1]; IA[2] += t[2] + t2[2];
        cross3(V, IV + 3, t);
        IA[3] += t[0]; IA[4] += t[1]; IA[5] += t[2];
        for (int e = 0; e < 10; e++) w.Ib[b][e] = I[e];
        for (int e = 0; e < 6; e++) LVA(IF)[e] = IA[e];
    }
    LANES_END
    PSUB(clk, w, PS_KIN_INERTIA);
    WSUBTREE(IF, 6, tp);
    LANES_BEGIN
    if (lane < NB) for (int e = 0; e < 6; e++) w.Fb[lane][e] = LVA(IF)[e];
    LANES_END
    PSUB(clk, w, PS_KIN_SUBTREE);
}

// per-body spatial vector  X_b = sum_{i on chain(b)} S_i x_i   (root -> leaves), lane = body
template <class Real, class TPT>
UHC_DEVNI void tree_vel(const Model<Real> &m, Work<Real> &w, const Real *x, Real (*X)[6], const TPT &tp) {
    LVARA(Real, V, 6);
    LANES_BEGIN
    const int b = lane;
    Pr<Real> Vp[3] = {pbc(Real(0)), pbc(Real(0)), pbc(Real(0))};
    if (b < NB) {
        const int d0 = b == 0 ? 0 : 6 + 3 * (b - 1), nd = b == 0 ? 6 : 3;
        for (int j = 0; j < nd; ++j) paxpy6(x[d0 + j], as_pairs(w.S[d0 + j]), Vp);
    }
    for (int i = 0; i < 3; i++) { LVA(V)[2 * i] = Vp[i].x; LVA(V)[2 * i + 1] = Vp[i].y; }
    LANES_END_R
    WANCESTOR(V, 6, tp);
    LANES_BEGIN
    if (lane < NB) for (int i = 0; i < 6; i++) X[lane][i] = LVA(V)[i];
    LANES_END
}
// y_i = S_i . Fsub[body(i)]  for all dofs, lane = dof
template <class Real>
UHC_DEV void project_force(const Model<Real> &m, Work<Real> &w, const Real (*F)[6], Real *y, Real scale, const Real *add) {
    LANES_BEGIN
#pragma unroll 1
    for (int i = lane; i < NV; i += 32) {
        const int b = i < 6 ? 0 : 1 + (i - 6) / 3;
        y[i] = scale * pdot6(as_pairs(w.S[i]), as_pairs(F[b])) + (add ? add[i] : Real(0));
    }
    LANES_END
}

// ================================================================================================ collision
// Floor plane z = 0 against each body hull (oracle/uhc_oracle.c or_collide states the manifold rule).
template <class Real, class TPT>
UHC_DEV void collide(const Model<Real> &m, Work<Real> &w, const TPT &tp, bool clk = false) {
    // broad phase for all bodies at once (lane = body): bounding sphere against the plane
    LVAR(int, near); LVAR(int, cnt); LVAR(int, adr0);
    LANES_BEGIN
    int f = 0;
    if (lane < NB) {
        const Real *bf = m.body_f + lane * BODYF; const Real *R = w.xmat[lane];
        const Real cz = w.xpos[lane][2] + R[6] * UHC_LDG(bf + 14) + R[7] * UHC_LDG(bf + 15) + R[8] * UHC_LDG(bf + 16);
        f = !(cz - UHC_LDG(bf + 17) > m.margin);
    }
    LV(near) = f;
    LANES_END_R
    unsigned cand_b = WBALLOT(near);
    PSUB(clk, w, PS_COL_BROAD);
    // narrow phase for every candidate body at once: candidate k (ascending body order) gets the aligned group of G = 2^lg lanes k G .. k G + G - 1
    const int ncand = popc32(cand_b);
    int lg = 5; while ((ncand << lg) > 32) lg--;
    const int G = 1 << lg;
    LVAR(int, cb); LVAR(Real, bz); LVAR(int, bi); LVAR(unsigned, nmask); LVAR(int, nck); LVAR(int, exk); LVAR(int, acc); LVAR(int, ovf); LVAR(int, up);
    // deepest hull vertex: every lane scans the vertices sub, sub + G, .. of its candidate in ascending order and keeps the first lowest; the
    // group's (height, index) minimum is then today's winner of the whole hull (lowest, then lowest index)
    LANES_BEGIN
    const int k = lane >> lg, sub = lane & (G - 1);
    Real best = Real(1e30); int besti = 1 << 20, b = -1;
    if (k < ncand) {
        b = nth_bit(cand_b, k);
        const Real *R = w.xmat[b];
        const int adr = TP_OF(m, tp, b).hadr, nvt = TP_OF(m, tp, b).hnum;
#pragma unroll 1
        for (int i = sub; i < nvt; i += G) {
            const Real *vv = m.hull + 3 * (adr + i);
            const Real v0 = UHC_LDG(vv), v1 = UHC_LDG(vv + 1), v2 = UHC_LDG(vv + 2);
            const Real z = w.xpos[b][2] + R[6] * v0 + R[7] * v1 + R[8] * v2;
            if (z < best) { best = z; besti = i; }
        }
    }
    LV(cb) = b; LV(bz) = best; LV(bi) = besti;
    LANES_END_R
    WSEGARGMIN(LV_ALL(bz), LV_ALL(bi), G);
    // its hull-graph neighbours within the margin, as a mask in list order (the first three join the manifold)
    LANES_BEGIN
    const int k = lane >> lg, sub = lane & (G - 1), b = LV(cb);
    unsigned f = 0;
    if (k < ncand && !(LV(bz) > m.margin)) {
        const Real *R = w.xmat[b];
        const int adr = TP_OF(m, tp, b).hadr, g = adr + LV(bi), n0 = UHC_LDG(m.nbradr + g), nn = min_(UHC_LDG(m.nbradr + g + 1) - n0, 32);
#pragma unroll 1
        for (int j = sub; j < nn; j += G) {
            const Real *vv = m.hull + 3 * (adr + UHC_LDG(m.nbr + n0 + j));
            const Real v0 = UHC_LDG(vv), v1 = UHC_LDG(vv + 1), v2 = UHC_LDG(vv + 2);
            const Real z = w.xpos[b][2] + R[6] * v0 + R[7] * v1 + R[8] * v2;
            if (z <= m.margin) f |= 1u << j;
        }
    }
    LV(nmask) = f;
    LANES_END_R
    WSEGOR(LV_ALL(nmask), G);
    LANES_BEGIN
    int nc = 0;
    if ((lane >> lg) < ncand && !(LV(bz) > m.margin)) { const int nsel = popc32(LV(nmask)); nc = 1 + (nsel < 3 ? nsel : 3); }
    LV(nck) = nc;
    LANES_END_R
    // lane k <- candidate k's contact count; in body order a candidate is skipped (and the overflow flagged) when the contacts of the ones taken
    // before it leave fewer than 4 of the MAXCON slots.  The first skipped one leaves every later one skipped, so the taken ones are the
    // candidates whose exclusive prefix count is <= MAXCON - 4, and their slots start at that prefix.
    WSHFLV(LV_ALL(exk), LV_ALL(nck), (lane < ncand ? lane << lg : 31));
    LANES_BEGIN
    if (lane >= ncand) LV(exk) = 0;
    LV(acc) = LV(exk);
    LANES_END_R
    WEXSCAN(LV_ALL(exk), LV_ALL(acc));
    LANES_BEGIN
    const bool ok = LV(exk) + 4 <= MAXCON;
    LV(ovf) = lane < ncand && !ok;
    LV(up) = lane < ncand && ok && LV(acc) > 0 && nth_bit(cand_b, lane) >= UPPER_BODY0;
    if (!ok) LV(acc) = 0;
    LANES_END_R
    if (WBALLOT(ovf)) w.con_overflow = 1;   // flagged: env_step_warp turns it into fail (SI_FLAGS bit 0)
    const int upper = WBALLOT(up) != 0;
    // per body (lane = body): its taken count; per group: its candidate's taken count and first slot
    WSHFLV(LV_ALL(cnt), LV_ALL(acc), (((cand_b >> lane) & 1u) ? popc32(cand_b & ((1u << lane) - 1u)) : 31));
    WSHFLV(LV_ALL(nck), LV_ALL(acc), lane >> lg);
    WSHFLV(LV_ALL(exk), LV_ALL(exk), lane >> lg);
    // slot 0: the deepest vertex; slots 1..: the first three neighbours within the margin, in list order (lane sub writes slots sub, sub + G, ..)
    LANES_BEGIN
    const int nc = LV(nck), b = LV(cb);
    if (nc > 0) {
        const Real *R = w.xmat[b];
        const int adr = TP_OF(m, tp, b).hadr, g = adr + LV(bi);
#pragma unroll 1
        for (int c = lane & (G - 1); c < nc; c += G) {
            const int vi = c == 0 ? g : adr + UHC_LDG(m.nbr + UHC_LDG(m.nbradr + g) + nth_bit(LV(nmask), c - 1));
            const Real *vv = m.hull + 3 * vi;
            const Real v0 = UHC_LDG(vv), v1 = UHC_LDG(vv + 1), v2 = UHC_LDG(vv + 2);
            const Real px = w.xpos[b][0] + R[0] * v0 + R[1] * v1 + R[2] * v2;
            const Real py = w.xpos[b][1] + R[3] * v0 + R[4] * v1 + R[5] * v2;
            const Real pz = w.xpos[b][2] + R[6] * v0 + R[7] * v1 + R[8] * v2;
            const int slot = LV(exk) + c;
            w.cbody[slot] = b; w.cdist[slot] = pz;
            w.cr[slot][0] = px - w.q[0]; w.cr[slot][1] = py - w.q[1]; w.cr[slot][2] = Real(0.5) * pz - w.q[2];
        }
    }
    LANES_END
    PSUB(clk, w, PS_COL_NARROW);
    // contact ranges per body: exclusive prefix sum of the per-body counts (lane = body)
    WEXSCAN(LV_ALL(adr0), LV_ALL(cnt));
    LANES_BEGIN
    if (lane <= NB) w.bcon_adr[lane] = LV(adr0);
    if (lane == NB) w.ncon = LV(adr0);
    LANES_END
    w.upper_contact = upper;
#ifndef UHC_EMU
    __syncwarp();
#endif
}


// per-contact soft-constraint parameters (MuJoCo solref/solimp semantics, SURVEY.md Appendix B), lane = contact
template <class Real>
UHC_DEV void constraint_setup(const Model<Real> &m, Work<Real> &w) {
    const Real kk = Real(1) / (m.simp1 * m.simp1 * m.solref0 * m.solref0 * m.solref1 * m.solref1), bb = Real(2) / (m.simp1 * m.solref0);
    LANES_BEGIN
#pragma unroll 1
    for (int c = lane; c < w.ncon; c += 32) {
        const int b = w.cbody[c];
        const Real pos = w.cdist[c] - m.margin;
        Real x = abs_(pos) / m.simp2; if (x > 1) x = 1;
        Real y;
        if (m.simp4 == Real(2)) y = x < m.simp3 ? x * x / m.simp3 : 1 - (1 - x) * (1 - x) / (1 - m.simp3);   // power 2 (the default)
        else if (x < m.simp3) y = pow_(x / m.simp3, m.simp4) * m.simp3;
        else y = 1 - pow_((1 - x) / (1 - m.simp3), m.simp4) * (1 - m.simp3);
        const Real imp = m.simp0 + y * (m.simp1 - m.simp0);
        Real R0 = (1 - imp) * UHC_LDG(m.body_f + b * BODYF + 13) * (1 + m.mu * m.mu) / imp;
        if (R0 < Real(1e-15)) R0 = Real(1e-15);
        w.cD[c] = Real(1) / (2 * m.mu * m.mu * R0);
        Real u[3], t[3];
        cross3(w.Vb[b], w.cr[c], t);
        for (int i = 0; i < 3; i++) u[i] = w.Vb[b][3 + i] + t[i];
        for (int e = 0; e < 4; e++) { Real d[3]; edge_dir(e, m.mu, d); w.caref[c][e] = -bb * dot3(d, u) - kk * imp * pos; }
    }
    LANES_END
}

// joint limits (mj_instantiateLimit with margin 0): a hinge past its range gets ONE unilateral row J = sg e_dof (sg = +1 at the lower, -1 at the upper
// limit), pos = distance to the limit (< 0), default solref / solimp, R = (1 - d)/d * dof_invweight0 (no pyramid factor).  lane = dof.  The row's data
// ride in vectors that are dead during the constraint solve: tau[i] = sg * D (0 = no row), as_[i] = -aref (newton_init turns it into the residual).
template <class Real>
UHC_DEV void limit_setup(const Model<Real> &m, Work<Real> &w) {
    // cheap test first (the ranges sit in shared memory next to the joint gains): in the common case no hinge is past its range and nothing else happens
    LVAR(int, viol);
    LANES_BEGIN
    int f = 0;
#pragma unroll 1
    for (int i = 6 + lane; i < NV; i += 32) { const Real q = w.q[i + 1]; f |= (q < UHC_LDT(m.dof_lim + 4 * i)) | (q > UHC_LDT(m.dof_lim + 4 * i + 1)); }
    LV(viol) = f;
    LANES_END_R
    if (!WBALLOT(viol)) { w.nlim = 0; return; }
    const Real kk = Real(1) / (m.simp1 * m.simp1 * m.solref0 * m.solref0 * m.solref1 * m.solref1), bb = Real(2) / (m.simp1 * m.solref0);
    LANES_BEGIN
#pragma unroll 1
    for (int i = lane; i < NV; i += 32) {
        Real sD = 0;
        if (i >= 6) {
            const Real q = w.q[i + 1], lo = UHC_LDT(m.dof_lim + 4 * i), hi = UHC_LDT(m.dof_lim + 4 * i + 1);
            Real dist = 0, sg = 0;
            if (q - lo < 0) { dist = q - lo; sg = 1; } else if (hi - q < 0) { dist = hi - q; sg = -1; }
            if (sg != 0) {
                Real x = abs_(dist) / m.simp2; if (x > 1) x = 1;
                Real y;
                if (m.simp4 == Real(2)) y = x < m.simp3 ? x * x / m.simp3 : 1 - (1 - x) * (1 - x) / (1 - m.simp3);
                else if (x < m.simp3) y = pow_(x / m.simp3, m.simp4) * m.simp3;
                else y = 1 - pow_((1 - x) / (1 - m.simp3), m.simp4) * (1 - m.simp3);
                const Real imp = m.simp0 + y * (m.simp1 - m.simp0);
                Real R = (1 - imp) * UHC_LDT(m.dof_lim + 4 * i + 2) / imp;
                if (R < Real(1e-15)) R = Real(1e-15);
                sD = sg / R;
                w.as_[i] = bb * sg * w.v[i] + kk * imp * dist;       // -aref
            }
        }
        w.tau[i] = sD;
    }
    LANES_END
    w.nlim = 1;
#ifndef UHC_EMU
    __syncwarp();
#endif
}

// rows: out[c][e] = d_e . (point velocity of body spatial vector X at contact c), lane = contact
template <class Real>
UHC_DEVNI void contact_rows(const Model<Real> &m, Work<Real> &w, const Real (*X)[6], Real (*out)[4], const Real (*sub)[4]) {
    LANES_BEGIN
#pragma unroll 1
    for (int c = lane; c < w.ncon; c += 32) {
        const int b = w.cbody[c]; Real u[3], t[3];
        cross3(X[b], w.cr[c], t);
        for (int i = 0; i < 3; i++) u[i] = X[b][3 + i] + t[i];
        for (int e = 0; e < 4; e++) { Real d[3]; edge_dir(e, m.mu, d); out[c][e] = dot3(d, u) - (sub ? sub[c][e] : Real(0)); }
    }
    LANES_END
}
// body wrenches from per-row multipliers (force on the body along d_e at the contact point), then subtree sums.
// mode 0: lam = D r_-  (gradient term J^T D r_-) ; mode 2: lam = the multipliers the caller left in cjp
// lane = contact: wrench of each contact about O; contacts are ordered by body and bodies depth-first, so the wrench of
// subtree(b) is a contiguous range of contacts = a difference of two inclusive prefix sums (second 32-chunk only when needed).
template <class Real, class TPT>
UHC_DEVNI void contact_force(const Model<Real> &m, Work<Real> &w, int mode, Real (*Fo)[6], const TPT &tp) {
    LVARA(Real, P0, 6); LVARA(Real, P1, 6); LVARA(Real, lo, 6); LVARA(Real, hi, 6); LVAR(int, jlo); LVAR(int, jhi);
    const int nchunk = w.ncon > 32 ? 2 : 1;
    for (int k = 0; k < nchunk; ++k) {
        LVARA(Real, F, 6);
        LANES_BEGIN
        const int c = 32 * k + lane;
        for (int i = 0; i < 6; i++) LVA(F)[i] = 0;
        if (c < w.ncon) {
            // multipliers of the four pyramid edges d = (0, mu, 1), (0, -mu, 1), (-mu, 0, 1), (mu, 0, 1); force = sum_e l_e d_e
            const Real D = w.cD[c];
            Real l[4];
#pragma unroll
            for (int e = 0; e < 4; e++) { const Real r = w.cres[c][e]; l[e] = mode == 2 ? w.cjp[c][e] : (r < 0 ? D * r : Real(0)); }
            const Real f[3] = {m.mu * (l[3] - l[2]), m.mu * (l[0] - l[1]), (l[0] + l[1]) + (l[2] + l[3])};
            Real t[3];
            cross3(w.cr[c], f, t);
            LVA(F)[0] = t[0]; LVA(F)[1] = t[1]; LVA(F)[2] = t[2]; LVA(F)[3] = f[0]; LVA(F)[4] = f[1]; LVA(F)[5] = f[2];
        }
        LANES_END_R
        WPREFIX(F, 6);
        if (k == 0) { LANES_BEGIN for (int i = 0; i < 6; i++) { LVA(P0)[i] = LVA(F)[i]; LVA(P1)[i] = 0; } LANES_END_R }
        else { LANES_BEGIN for (int i = 0; i < 6; i++) LVA(P1)[i] = LVA(F)[i]; LANES_END_R }
    }
    // lane = body: subtree(b) owns contacts [bcon_adr[b], bcon_adr[sub_end(b) + 1])
    LANES_BEGIN
    const int b = lane < NB ? lane : NB - 1;
    LV(jlo) = w.bcon_adr[b] - 1; LV(jhi) = w.bcon_adr[TP.sub_end < NB ? TP.sub_end + 1 : NB] - 1;
    if (lane >= NB) { LV(jlo) = -1; LV(jhi) = -1; }
    LANES_END_R
    WSHFL(lo, P0, 6, (LV(jlo) < 0 ? 0 : LV(jlo)) & 31);
    WSHFL(hi, P0, 6, (LV(jhi) < 0 ? 0 : LV(jhi)) & 31);
    LANES_BEGIN
    for (int i = 0; i < 6; i++) {
        if (LV(jlo) < 0) LVA(lo)[i] = 0;
        if (LV(jhi) < 0) LVA(hi)[i] = 0;
    }
    LANES_END_R
    if (nchunk == 2) {      // indices >= 32 live in the second chunk: P(j) = total of chunk 0 + P1(j - 32)
        LVARA(Real, t0, 6); LVARA(Real, a, 6); LVARA(Real, c2, 6);
        WSHFL(t0, P0, 6, 31);
        WSHFL(a, P1, 6, (LV(jlo) < 0 ? 0 : LV(jlo)) & 31);
        WSHFL(c2, P1, 6, (LV(jhi) < 0 ? 0 : LV(jhi)) & 31);
        LANES_BEGIN
        for (int i = 0; i < 6; i++) {
            if (LV(jlo) >= 32) LVA(lo)[i] = LVA(t0)[i] + LVA(a)[i];
            if (LV(jhi) >= 32) LVA(hi)[i] = LVA(t0)[i] + LVA(c2)[i];
        }
        LANES_END
    }
    LANES_BEGIN
    if (lane < NB) for (int i = 0; i < 6; i++) Fo[lane][i] = LVA(hi)[i] - LVA(lo)[i];
    LANES_END
}

// ================================================================================================ constraint solve
// min_a 1/2 (a-a_s)^T M (a-a_s) + sum_rows 1/2 D min(0, J a - aref)^2 ; primal Newton.  The Hessian H = M + J^T D_act J is never formed:
// the Newton direction is one articulated-body solve with contact-augmented body inertias (aba_solve, use_contacts), and that solve's
// centre -> leaves sweep leaves the body accelerations J_b p of its solution in w.Ab (what the contact rows J p need).
//
// The gradient is carried from iteration to iteration instead of being rebuilt: with r(al) = r + al J p and H p = -g,
//     g(a + al p) = (1 - al) g + J^T D delta,    delta_row = r(al)_- - r_- - al [r < 0] (J p)_row = -|r(al)|  on rows whose active state
// switched between 0 and al, and 0 on every other row -- so an iteration costs one solve, one pass over the contact rows and (only when
// some row switched) one wrench pass; M a, M p and the smooth part of the gradient never appear.  The same identity gives the line search
//     f'(al) = (1 - al) g.p + sum_switched D (J p) delta ,   f''(al) = -g.p + sum_switched (+-) D (J p)^2
// exactly zero at al = 1 when no row switches: the full step is then the minimiser of the (locally quadratic) cost and the solve stops
// without a confirming gradient evaluation.
//
// newton_init: start from the warm start (previous qacc, as MuJoCo's warmstart): residuals r = J a - aref, gradient g = M a - f_s + J^T D r_-
// by O(n) passes, -g in w.p.  The problem is strictly convex, so the minimiser does not depend on the start; starting from the warm start
// makes the unconstrained solve a_s = M^-1 f_s unnecessary whenever contacts are present.  Returns the gradient-norm scale, |g|^2 in *gn2.
template <class Real, class TPT>
UHC_DEV Real newton_init(const Model<Real> &m, Work<Real> &w, const TPT &tp, Real *gn2) {
    tree_vel(m, w, w.aw, w.Ab, tp);
    contact_rows(m, w, w.Ab, w.cres, w.caref);
    contact_force(m, w, 0, w.Fb, tp);
    LVARA(Real, Fm, 6);
    LANES_BEGIN
    for (int i = 0; i < 6; i++) LVA(Fm)[i] = 0;
    if (lane < NB) rigid_mul(w.Ib[lane], w.Ab[lane], LVA(Fm));
    LANES_END_R
    WSUBTREE(Fm, 6, tp);
    LANES_BEGIN
    if (lane < NB) for (int i = 0; i < 6; i++) w.Fb[lane][i] += LVA(Fm)[i];
    LANES_END
    LVAR(Real, part); LVAR(Real, gs);
    LANES_BEGIN
    Real s = 0;
#pragma unroll 1
    for (int i = lane; i < NV; i += 32) {
        const int b = i < 6 ? 0 : 1 + (i - 6) / 3;
        Real gi = pdot6(as_pairs(w.S[i]), as_pairs(w.Fb[b])) + UHC_LDT(m.dof_f + 4 * i) * w.aw[i] - w.fs[i];
        if (w.nlim > 0 && w.tau[i] != 0) {      // joint-limit row: residual r = sg a_i - aref, gradient term J^T D r_- = sg D r_-
            const Real sD = w.tau[i], r = (sD > 0 ? w.aw[i] : -w.aw[i]) + w.as_[i];
            w.as_[i] = r;
            if (r < 0) gi += sD * r;
        }
        w.g[i] = gi; w.p[i] = -gi; w.a[i] = w.aw[i]; s += gi * gi;
    }
    LV(gs) = s;
    LV(part) = lane < NB ? 3 * w.Ib[lane][0] : Real(0);   // gradient tolerance scale ~ trace of the translational block of M
    LANES_END
    *gn2 = WSUM(gs);
    return WSUM(part);
}
// newton_advance: given the Newton direction in w.p (and J_b p in w.Ab, left there by the solve): J p, safeguarded 1-D Newton line search,
// update of a / residuals / gradient (-g again in w.p).  Returns true when the step was an exact Newton step (al = 1, no row switched): the
// new point is the minimiser and the carried gradient is exactly zero.
template <class Real, class TPT>
UHC_DEV bool newton_advance(const Model<Real> &m, Work<Real> &w, const TPT &tp, Real *gn2) {
    contact_rows(m, w, w.Ab, w.cjp, (const Real (*)[4]) nullptr);
    LVAR(Real, pa);
    LANES_BEGIN
    Real sA = 0;
#pragma unroll 1
    for (int i = lane; i < NV; i += 32) sA += w.g[i] * w.p[i];
    LV(pa) = sA;
    LANES_END_R
    const Real gp = WSUM(pa);           // directional derivative at al = 0 (negative: p is a descent direction)
    Real lo = 0, hi = -1, al = 1;
    bool exact = false;
#pragma unroll 1
    for (int ls = 0; ls < 12; ++ls) {
        LVAR(Real, d1); LVAR(Real, d2); LVAR(int, chg);
        LANES_BEGIN
        Real s1 = 0, s2 = 0; int ch = 0;
#pragma unroll 1
        for (int c = lane; c < w.ncon; c += 32) for (int e = 0; e < 4; e++) {
            const Real r0 = w.cres[c][e], jp = w.cjp[c][e], r = r0 + al * jp;
            if ((r0 < 0) != (r < 0)) { const Real dj = w.cD[c] * jp; s1 -= dj * abs_(r); s2 += (r < 0) ? dj * jp : -dj * jp; ch = 1; }
        }
        if (w.nlim > 0) for (int i = lane; i < NV; i += 32) if (w.tau[i] != 0) {     // joint-limit rows: J p = sg p_i
            const Real sD = w.tau[i], r0 = w.as_[i], jp = sD > 0 ? w.p[i] : -w.p[i], r = r0 + al * jp;
            if ((r0 < 0) != (r < 0)) { const Real dj = abs_(sD) * jp; s1 -= dj * abs_(r); s2 += (r < 0) ? dj * jp : -dj * jp; ch = 1; }
        }
        LV(d1) = s1; LV(d2) = s2; LV(chg) = ch;
        LANES_END_R
        const bool any = WBALLOT(chg) != 0;
        const Real f1 = (1 - al) * gp + (any ? WSUM(d1) : Real(0)), f2 = -gp + (any ? WSUM(d2) : Real(0));
        if (f1 > 0) hi = al; else lo = al;
        if (abs_(f1) <= Real(1e-6) * abs_(gp) + Real(1e-30)) { exact = ls == 0 && !any; break; }
        Real nx = f2 > 0 ? al - f1 / f2 : Real(-1);
        if (!(nx > lo) || (hi > 0 && !(nx < hi))) nx = hi > 0 ? Real(0.5) * (lo + hi) : 2 * al;
        if (nx == al) break;
        al = nx;
    }
    // a, residuals; multipliers D delta of the rows that switched between 0 and al (the others carry none) into cjp
    LVAR(int, chg2);
    LANES_BEGIN
#pragma unroll 1
    for (int i = lane; i < NV; i += 32) w.a[i] += al * w.p[i];
    int ch = 0;
#pragma unroll 1
    for (int c = lane; c < w.ncon; c += 32) for (int e = 0; e < 4; e++) {
        const Real r0 = w.cres[c][e], r = r0 + al * w.cjp[c][e];
        const bool sw = (r0 < 0) != (r < 0);
        w.cres[c][e] = r; w.cjp[c][e] = sw ? -w.cD[c] * abs_(r) : Real(0); ch |= sw;
    }
    if (w.nlim > 0) for (int i = lane; i < NV; i += 32) {       // joint-limit rows: new residual, multiplier sg D delta of a switched row into Mp (free between solves)
        Real mult = 0;
        if (w.tau[i] != 0) {
            const Real sD = w.tau[i], r0 = w.as_[i], r = r0 + al * (sD > 0 ? w.p[i] : -w.p[i]);   // p is still the direction here (a is updated above from it)
            w.as_[i] = r;
            if ((r0 < 0) != (r < 0)) { mult = -sD * abs_(r); ch = 1; }
        }
        w.Mp[i] = mult;
    }
    LV(chg2) = ch;
    LANES_END
    const bool any2 = WBALLOT(chg2) != 0;
    if (exact && !any2) {
        LANES_BEGIN
#pragma unroll 1
        for (int i = lane; i < NV; i += 32) { w.g[i] = 0; w.p[i] = 0; }
        LANES_END
        *gn2 = 0;
        return true;
    }
    if (any2) contact_force(m, w, 2, w.Fb, tp);
    LVAR(Real, gs);
    LANES_BEGIN
    Real s = 0;
#pragma unroll 1
    for (int i = lane; i < NV; i += 32) {
        const int b = i < 6 ? 0 : 1 + (i - 6) / 3;
        Real gi = (1 - al) * w.g[i];
        if (any2) gi += pdot6(as_pairs(w.S[i]), as_pairs(w.Fb[b]));
        if (any2 && w.nlim > 0) gi += w.Mp[i];
        w.g[i] = gi; w.p[i] = -gi; s += gi * gi;
    }
    LV(gs) = s;
    LANES_END
    *gn2 = WSUM(gs);
    return false;
}

// ================================================================================================ task layer
template <class Real> UHC_DEV void heading_q(const Real *q, Real *hq) {  // uhc/utils/math_utils.py:134-139
    const Real n = rsqrt_(q[0] * q[0] + q[3] * q[3]);
    hq[0] = q[0] * n; hq[1] = 0; hq[2] = 0; hq[3] = q[3] * n;
}
template <class Real> UHC_DEV Real heading(const Real *q) {  // uhc/utils/math_utils.py:176-183
    Real w = q[0], z = q[3]; if (z < 0) { w = -w; z = -z; }
    return 2 * acos_(clamp_(w * rsqrt_(w * w + z * z), Real(-1), Real(1)));
}
template <class Real> UHC_DEV void remove_base_rot(const EnvCfg<Real> &cfg, const Real *q, Real *o) {  // humanoid_im.py:263
    Real bi[4]; qinv(cfg.base_rot, bi); qmul(q, bi, o);
}
template <class Real> UHC_DEV void euler_zyx_quat(Real e0, Real e1, Real e2, Real *q) {  // quaternion_from_euler(.., "rzyx")
    Real s0, c0, s1, c1, s2, c2;
    sincos_(e0 * Real(0.5), &s0, &c0); sincos_(e1 * Real(0.5), &s1, &c1); sincos_(e2 * Real(0.5), &s2, &c2);
    const Real qz[4] = {c0, 0, 0, s0}, qy[4] = {c1, 0, s1, 0}, qx[4] = {c2, s2, 0, 0}; Real t[4];
    qmul(qz, qy, t); qmul(t, qx, q);
}
constexpr double PI_D = 3.14159265358979323846;

// stable PD torque for substep `it` (humanoid_im.py:1033-1076 + :1014-1031): uses the M, C currently in the work set
// (= previous forward pass: per-body inertias w.Ib, motion subspaces w.S, bias w.C) with the current q, v.  pd_setup leaves the right-hand side in w.p;
// after the shared articulated-body solve pd_finish turns the acceleration into clipped torques in w.tau (:1160).
template <class Real>
UHC_DEV void pd_gains(const EnvCfg<Real> &cfg, const Work<Real> &w, int it, Real *sp, Real *sd) {
    *sp = 1; *sd = 1;
    if (cfg.meta_pd) { *sp = clamp_(w.act[NU + 6 + it] + 1, Real(0), Real(10)); *sd = clamp_(w.act[NU + 6 + it + NSUB] + 1, Real(0), Real(10)); }
}
template <class Real>
UHC_DEV void pd_setup(const Model<Real> &m, const EnvCfg<Real> &cfg, Work<Real> &w, const Real *target, int it) {
    const Real dt = m.dt;
    Real sp, sd; pd_gains(cfg, w, it, &sp, &sd);
    LANES_BEGIN
#pragma unroll 1
    for (int i = lane; i < NV; i += 32) {
        Real rhs = -w.C[i];
        if (i >= 6) {
            const int j = i - 6; const Real qj = w.q[7 + j];
            // humanoid_im.py:1041-1045 (while base - q > pi: base -= 2 pi ; while base - q < -pi: base += 2 pi) in closed form --
            // a loop on a non-finite state would never terminate
            Real base = target[j];
            const Real dlt = base - qj;
            if (dlt > Real(PI_D)) base -= Real(2 * PI_D) * ceil((dlt - Real(PI_D)) / Real(2 * PI_D));
            else if (dlt < -Real(PI_D)) base += Real(2 * PI_D) * ceil((-Real(PI_D) - dlt) / Real(2 * PI_D));
            const Real kp = UHC_LDT(m.dof_f + 4 * i + 1) * sp, kd = UHC_LDT(m.dof_f + 4 * i + 2) * sd;
            const Real err = qj + w.v[i] * dt - (base + w.act[j]);
            rhs += -kp * err - kd * w.v[i];
            w.g[i] = err;  // stash
        }
        w.p[i] = rhs;
    }
    LANES_END
}
template <class Real, class OutT>
UHC_DEV void pd_finish(const Model<Real> &m, const EnvCfg<Real> &cfg, Work<Real> &w, int it, OutT *torque_out) {
    const Real dt = m.dt;
    Real sp, sd; pd_gains(cfg, w, it, &sp, &sd);
    LANES_BEGIN
#pragma unroll 1
    for (int i = 6 + lane; i < NV; i += 32) {
        const Real kp = UHC_LDT(m.dof_f + 4 * i + 1) * sp, kd = UHC_LDT(m.dof_f + 4 * i + 2) * sd, lim = UHC_LDT(m.dof_f + 4 * i + 3);
        const Real t = clamp_(-kp * w.g[i] - kd * (w.v[i] + w.p[i] * dt), -lim, lim);
        w.tau[i - 6] = t;
        if (torque_out) torque_out[it * NU + i - 6] = (OutT)t;
    }
    LANES_END
}
// implicit residual force: humanoid_im.py:1136-1143 (recomputed every substep from the current root quaternion)
template <class Real>
UHC_DEV void rfc_implicit(const EnvCfg<Real> &cfg, const Work<Real> &w, Real *fapp) {
    Real crq[4], hq[4], R[9], vf[6], t[3];
    for (int i = 0; i < 6; i++) vf[i] = w.act[NU + i] * cfg.rfc_scale * cfg.rfc_rate;
    remove_base_rot(cfg, w.q + 3, crq); heading_q(crq, hq); q2mat(hq, R); mv3(R, vf, t);
    vf[0] = t[0]; vf[1] = t[1]; vf[2] = t[2];
    for (int i = 0; i < 6; i++) fapp[i] = clamp_(vf[i], -cfg.rfc_lim, cfg.rfc_lim);
}

// explicit residual force: humanoid_im.py:1080-1132 with the release settings (residual_force_bodies = "all", one point per body, torque on, no
// contact gating / projection).  Per body a contact point, a force and a torque given in the BODY frame of the LAST forward pass
// (mujoco_env.py:171-180 read data.body_xpos / xmat between two sim.step()), scaled by residual_force_scale and applied through mj_applyFT, whose
// Jacobian is also the last forward pass' -- i.e. the stale xpos / xmat / S this work set still holds before kin_rne_forward runs.
// As spatial wrenches about O (the stale root position): F_b = (tau + (p - O) x f, f); qfrc_i = S_i . sum over subtree(body(i)) of F.
template <class Real, class ActT, class TPT>
UHC_DEV void rfc_explicit(const Model<Real> &m, const EnvCfg<Real> &cfg, Work<Real> &w, const TPT &tp, const ActT *act, Real *qfrc) {
    LVARA(Real, F, 6);
    LANES_BEGIN
    for (int i = 0; i < 6; i++) LVA(F)[i] = 0;
    if (lane < NB) {
        const int b = lane;
        const ActT *v = act + NU + VF_BODY_DIM * (int)cfg.vf_slot[b];
        const Real *R = w.xmat[b];
        const Real cp[3] = {(Real)v[0], (Real)v[1], (Real)v[2]}, fl[3] = {(Real)v[3] * cfg.rfc_scale, (Real)v[4] * cfg.rfc_scale, (Real)v[5] * cfg.rfc_scale},
                   tl[3] = {(Real)v[6] * cfg.rfc_scale, (Real)v[7] * cfg.rfc_scale, (Real)v[8] * cfg.rfc_scale};
        Real p[3], f[3], tq[3], n[3];
        mv3(R, cp, p); mv3(R, fl, f); mv3(R, tl, tq);
        for (int k = 0; k < 3; k++) p[k] += w.xpos[b][k] - w.xpos[0][k];
        cross3(p, f, n);
        LVA(F)[0] = tq[0] + n[0]; LVA(F)[1] = tq[1] + n[1]; LVA(F)[2] = tq[2] + n[2]; LVA(F)[3] = f[0]; LVA(F)[4] = f[1]; LVA(F)[5] = f[2];
    }
    LANES_END_R
    WSUBTREE(F, 6, tp);
    LANES_BEGIN
    if (lane < NB) for (int i = 0; i < 6; i++) w.Fb[lane][i] = LVA(F)[i];
    LANES_END
    project_force(m, w, w.Fb, qfrc, Real(1), (const Real *)nullptr);
}
// pose of the last forward pass back into the work set at the start of a control step (only the explicit residual force needs it before the
// first forward pass of the step): xpos from the record, xmat from the stored body quaternions (what data.body_xmat holds: mju_quat2Mat of xquat)
template <class Real>
UHC_DEV void restore_stale_pose(Work<Real> &w, const Real *st_xpos, const Real *st_xquat) {
    LANES_BEGIN
    if (lane < NB) {
        for (int k = 0; k < 3; k++) w.xpos[lane][k] = st_xpos[3 * lane + k];
        const Real q[4] = {st_xquat[4 * lane], st_xquat[4 * lane + 1], st_xquat[4 * lane + 2], st_xquat[4 * lane + 3]};
        q2mat(q, w.xmat[lane]);
    }
    LANES_END
}

template <class Real>
UHC_DEV void integrate(const Model<Real> &m, Work<Real> &w) {
    const Real dt = m.dt;
    LANES_BEGIN
#pragma unroll 1
    for (int i = lane; i < NV; i += 32) { const Real vn = w.v[i] + dt * w.a[i]; w.v[i] = vn; w.aw[i] = w.a[i]; if (i >= 6) w.q[i + 1] += dt * vn; }
    LANES_END
    LANES_BEGIN
    if (lane < 3) w.q[lane] += dt * w.v[lane];
    if (lane == 3) {
        const Real wx = w.v[3], wy = w.v[4], wz = w.v[5], n = sqrt(wx * wx + wy * wy + wz * wz), ang = n * dt;
        Real dq[4] = {1, 0, 0, 0}, qn[4], qo[4] = {w.q[3], w.q[4], w.q[5], w.q[6]};
        if (ang > Real(1e-30)) { Real sn, cs; sincos_(Real(0.5) * ang, &sn, &cs); const Real s = sn / n; dq[0] = cs; dq[1] = wx * s; dq[2] = wy * s; dq[3] = wz * s; }
        qmul(qo, dq, qn);
        const Real nn = rsqrt_(qn[0] * qn[0] + qn[1] * qn[1] + qn[2] * qn[2] + qn[3] * qn[3]);
        for (int i = 0; i < 4; i++) w.q[3 + i] = qn[i] * nn;
    }
    LANES_END
}

// ================================================================================================ one physics substep
// [stable-PD torque] -> mj_forward (position, velocity, actuation, acceleration, constraint) at the current (q, v).
// The three linear solves of a substep (PD: M_stale + Kd dt ; smooth: M ; Newton: M + J^T D J) run through ONE copy of the
// articulated-body solve: a small phase machine sets up the right-hand side, the shared solve runs, the phase post-processes.  Leaves M, C, xpos/xmat/xipos of THIS (pre-integration) configuration in the work set -- the staleness MuJoCo
// exposes to the Python side (SURVEY.md section 7 "stale dynamics").  with_pd = false: reset path (sim.forward with ctrl = 0).
enum { PH_PD = 0, PH_SMOOTH = 1, PH_NEWTON = 2 };
// The warps of a CTA are re-aligned at points every warp passes exactly once per substep: they then run the same code at
// the same time and share instruction-cache lines (the per-substep code is 112 KB of SASS: scripts/step_sass_footprint.py).
// The fp32 kernel runs one 16-warp CTA per SM aligned as two groups of 8 warps (one named barrier each): on an H100 at 4096 envs that
// was ~1 % faster than two 8-warp CTAs per SM aligned as a whole (k_env_step 3.06 vs 3.08 ms).  On the GPU the kernel was first tuned
// on, aligning 7 warps was faster than groups of 2 / 3 / 4 warps and than aligning every 2nd / 3rd substep or each Newton iteration.
// The barrier is a NAMED barrier with an explicit thread count (w.sync_threads = 32 x the warps of the group that own a valid
// environment): warps without work leave the kernel before the substep loop and are simply not counted.
#if !defined(UHC_EMU) && !defined(UHC_NO_CTA_SYNC)
#define UHC_CTA_SYNC(on) do { if (on) asm volatile("bar.sync %0, %1;" :: "r"(w.sync_id), "r"(w.sync_threads) : "memory"); } while (0)
#else
#define UHC_CTA_SYNC(on) do { (void)(on); } while (0)
#endif
template <class Real, class OutT, class TPT>
UHC_DEVNI int substep_dynamics(const Model<Real> &m, const EnvCfg<Real> &cfg, Work<Real> &w, const TPT &tp, const Real *target, int it,
                             bool with_pd, OutT *torque_out, bool cta_sync = false, const OutT *act_global = nullptr) {
    int phase = with_pd ? PH_PD : PH_SMOOTH, iters = 0;
    bool done = false;
    Real scale = 0, gn2 = 0;
    for (;;) {
        // ---- phase set-up: right-hand side into the vector the solve runs on
        Real *rhs = w.p;
        Real arm_scale = 0;
        if (phase == PH_PD) {
            pd_setup(m, cfg, w, target, it);
            Real sp, sd; pd_gains(cfg, w, it, &sp, &sd);
            arm_scale = sd * m.dt;
        } else if (phase == PH_SMOOTH) {
            Real fapp[6] = {0, 0, 0, 0, 0, 0};
            const bool explicit_rf = with_pd && cfg.rfc_mode == 1 && act_global != nullptr;
            if (explicit_rf) rfc_explicit(m, cfg, w, tp, act_global, w.as_);        // generalized force of the per-body residual forces (stale Jacobian) -> as_
            else if (with_pd && cfg.rfc_mode == 0) rfc_implicit(cfg, w, fapp);
            kin_rne_forward(m, w, tp, cta_sync);
            project_force(m, w, w.Fb, w.C, Real(1), (const Real *)nullptr);
            PSUB(cta_sync, w, PS_KIN_PROJECT);
            PCLK(cta_sync, w, PC_KIN);
            collide(m, w, tp, cta_sync);
            PSUB(cta_sync, w, PS_COL_PREFIX);
            PCLK(cta_sync, w, PC_COLLIDE);
            LANES_BEGIN
#pragma unroll 1
            for (int i = lane; i < NV; i += 32) {  // smooth acceleration a_s = M^-1 (tau + f_applied - C)
                Real f = -w.C[i];
                if (explicit_rf) f += w.as_[i];
                else if (i < 6) { const Real fa = i == 0 ? fapp[0] : i == 1 ? fapp[1] : i == 2 ? fapp[2] : i == 3 ? fapp[3] : i == 4 ? fapp[4] : fapp[5]; f += fa; }
                if (i >= 6 && with_pd) f += w.tau[i - 6];
                w.fs[i] = f; w.as_[i] = f;
            }
            LANES_END
            rhs = w.as_;
            limit_setup(m, w);                         // after the loop above consumed tau; touches as_ only on dofs that get a limit row (then no smooth solve runs)
        } else {
            // (aligning the Newton iterations across the CTA as well was measured: the waiting costs more than it saves)
            if (done || iters >= cfg.newton_max_iter || !(gn2 > cfg.newton_tol * cfg.newton_tol * scale * scale)) break;
            ++iters;
        }
        // ---- the one shared O(n) articulated-body solve (not needed for the smooth phase when contacts are present:
        //      Newton starts from the warm start and only needs f_s, not a_s = M^-1 f_s)
        if (!(phase == PH_SMOOTH && (w.ncon > 0 || w.nlim > 0))) aba_solve(m, w, arm_scale, phase == PH_NEWTON, rhs);
        // ---- phase post-processing
        if (phase == PH_PD) {
            pd_finish(m, cfg, w, it, torque_out); phase = PH_SMOOTH;
            PCLK(cta_sync, w, PC_PD);
            UHC_CTA_SYNC(cta_sync);
            PCLK(cta_sync, w, PC_SYNC_PD);
        } else if (phase == PH_SMOOTH) {
            PCLK(cta_sync, w, PC_SMOOTH);
            UHC_CTA_SYNC(cta_sync);
            PCLK(cta_sync, w, PC_SYNC_SMOOTH);
            if (w.ncon == 0 && w.nlim == 0) {
                LANES_BEGIN
#pragma unroll 1
                for (int i = lane; i < NV; i += 32) w.a[i] = w.as_[i];
                LANES_END
                done = true;
            } else {
                constraint_setup(m, w);
                scale = newton_init(m, w, tp, &gn2);
            }
            PCLK(cta_sync, w, PC_CSETUP);
            phase = PH_NEWTON;
        } else {
            PCLK(cta_sync, w, PC_NEWTON_ABA);
            if (newton_advance(m, w, tp, &gn2)) done = true;
            PCLK(cta_sync, w, PC_NEWTON_ROWS);
        }
    }
    return iters;
}

// body quaternions from qpos (humanoid_im.py:925-947), lane = body
template <class Real>
UHC_DEVNI void body_quat(const Work<Real> &w, Real *out) {
    LANES_BEGIN
    const int b = lane;
    if (b == 0) for (int i = 0; i < 4; i++) out[i] = w.q[3 + i];
    else if (b < NB) euler_zyx_quat(w.q[7 + 3 * (b - 1)], w.q[8 + 3 * (b - 1)], w.q[9 + 3 * (b - 1)], out + 4 * b);
    LANES_END
}
// world body quaternions by composing along each body's own chain (no cross-lane dependency), lane = body.
// Matches the pose the last forward pass used (xquat is only consumed by the observation).
template <class Real>
UHC_DEVNI void world_quat(const Model<Real> &m, const Real *qfk, Work<Real> &w) {
    LANES_BEGIN
    const int b = lane;
    if (b < NB) {
        int chain[MAXLEVEL + 1], n = 0;
        for (int a = b; a > 0; a = UHC_LDG(m.parent + a)) chain[n++] = a;
        Real q[4] = {qfk[3], qfk[4], qfk[5], qfk[6]};
        const Real nn = rsqrt_(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
        for (int i = 0; i < 4; i++) q[i] *= nn;
        for (int k = n - 1; k >= 0; --k) {
            const int a = chain[k]; Real ql[4], t[4];
            euler_zyx_quat(qfk[7 + 3 * (a - 1)], qfk[8 + 3 * (a - 1)], qfk[9 + 3 * (a - 1)], ql);
            qmul(q, ql, t);
            const Real n2 = rsqrt_(t[0] * t[0] + t[1] * t[1] + t[2] * t[2] + t[3] * t[3]);
            for (int i = 0; i < 4; i++) q[i] = t[i] * n2;
        }
        for (int i = 0; i < 4; i++) w.xquat[b][i] = q[i];
    }
    LANES_END
}

// observation v2 (humanoid_im.py:419-503, obs_coord "root") and, with cfg.obs_v == 1, v1 (:323-417: the same blocks, then the per-body centres of
// mass relative to the root and their difference to the expert's body_com, the quaternion blocks after those, no shape vector); ex1 = expert frame at cur_t + 1
template <class Real, class OutT>
UHC_DEVNI void obs_v2(const EnvCfg<Real> &cfg, const Work<Real> &w, const Real *ex1, const Real *shape_obs, OutT *obs) {
    Real crq[4], hq[4], hqi[4], trq[4], dh[4], ci[4], dq[4], Rq[9], Rc[9];
    remove_base_rot(cfg, w.q + 3, crq); heading_q(crq, hq); qinv(hq, hqi);
    remove_base_rot(cfg, ex1 + EX_QPOS + 3, trq);
    qmul(hqi, crq, dh); qinv(crq, ci); qmul(trq, ci, dq);
    q2mat(w.q + 3, Rq); q2mat(crq, Rc);
    Real rel_h = heading(trq) - heading(crq);
    if (rel_h > Real(PI_D)) rel_h -= Real(2 * PI_D);
    if (rel_h < -Real(PI_D)) rel_h += Real(2 * PI_D);
    LANES_BEGIN
    if (lane < 4) obs[lane] = (OutT)hq[lane];
    for (int i = lane; i < 74; i += 32) {
        const Real tq = ex1[EX_QPOS + 2 + i];
        Real cur, df;
        if (i == 0) { cur = w.q[2]; df = tq - cur; }
        else if (i < 5) { cur = dh[i - 1]; df = dq[i - 1]; }
        else { cur = w.q[2 + i]; df = tq - cur; }
        obs[4 + i] = (OutT)tq; obs[78 + i] = (OutT)cur; obs[152 + i] = (OutT)df;
    }
    if (lane == 0) {
        Real t[3], t2[3];
        mtv(Rq, w.v, t); mtv(Rc, t, t2);                                   // rotated twice (:425, :451)
        obs[226] = (OutT)t2[0]; obs[227] = (OutT)t2[1]; obs[228] = (OutT)t2[2];
        obs[301] = (OutT)rel_h;
        const Real rp[3] = {trq[0] - w.q[0], trq[1] - w.q[1], trq[2] - w.q[2]};  // the kept bug (:466)
        mtv(Rc, rp, t);
        obs[302] = (OutT)t[0]; obs[303] = (OutT)t[1];
    }
    for (int i = 3 + lane; i < NV; i += 32) obs[226 + i] = (OutT)w.v[i];
    if (lane < NB) {
        const int b = lane; Real r[3], t[3];
        for (int k = 0; k < 3; k++) r[k] = w.xpos[b][k] - w.q[k];
        mtv(Rc, r, t);
        for (int k = 0; k < 3; k++) obs[304 + 24 * k + b] = (OutT)t[k];
        for (int k = 0; k < 3; k++) r[k] = ex1[EX_WBPOS + 3 * b + k] - w.xpos[b][k];
        mtv(Rc, r, t);
        for (int k = 0; k < 3; k++) obs[376 + 24 * k + b] = (OutT)t[k];
        const bool v1 = cfg.obs_v == 1;
        const int oq = v1 ? 592 : 448;
        if (v1) {
            for (int k = 0; k < 3; k++) r[k] = w.xipos[b][k] - w.q[k];
            mtv(Rc, r, t);
            for (int k = 0; k < 3; k++) obs[448 + 24 * k + b] = (OutT)t[k];
            for (int k = 0; k < 3; k++) r[k] = ex1[EX_BCOM + 3 * b + k] - w.xipos[b][k];
            mtv(Rc, r, t);
            for (int k = 0; k < 3; k++) obs[520 + 24 * k + b] = (OutT)t[k];
        }
        const bool use_t = (w.xquat[0][0] == 0);
        const Real *cq = use_t ? ex1 + EX_WBQUAT + 4 * b : w.xquat[b];
        Real o1[4], iq[4], o2[4];
        qmul(hqi, cq, o1);
        if (v1) qinv(cq, iq);                                                                  // v1: quaternion_inverse = conj / |q|^2 (:411)
        else {
            const Real nn = rsqrt_(cq[0] * cq[0] + cq[1] * cq[1] + cq[2] * cq[2] + cq[3] * cq[3]);  // v2: inverse_batch = conj / |q|
            iq[0] = cq[0] * nn; iq[1] = -cq[1] * nn; iq[2] = -cq[2] * nn; iq[3] = -cq[3] * nn;
        }
        qmul(iq, ex1 + EX_WBQUAT + 4 * b, o2);
        for (int k = 0; k < 4; k++) { obs[oq + 4 * b + k] = (OutT)o1[k]; obs[oq + 96 + 4 * b + k] = (OutT)o2[k]; }
    }
    if (cfg.obs_v != 1 && cfg.has_shape && lane < 17) obs[640 + lane] = (OutT)shape_obs[lane];
    LANES_END
}

// the "_new" heading helpers (uhc/utils/math_utils.py:169-207): yaw from the full quaternion, heading quaternion about z
template <class Real> UHC_DEV Real heading_new(const Real *q) { return atan2_(2 * (q[0] * q[3] + q[1] * q[2]), 1 - 2 * (q[2] * q[2] + q[3] * q[3])); }
template <class Real> UHC_DEV void heading_q_new(const Real *q, Real *hq) { Real sn, cs; sincos_(heading_new(q) * Real(0.5), &sn, &cs); hq[0] = cs; hq[1] = 0; hq[2] = 0; hq[3] = sn; }
// observation v5 (humanoid_im.py:505-594: the v2 blocks on the _new heading helpers, no heading quaternion block, the root velocity rotated once, the true root
// offset) and v6 (:596-666: root offset in the heading frame, relative heading, relative root rotation, qvel, joint positions (the y and z ROWS of the
// transformed (3, 24) array: the reference slices `[1:]` after the transform) and joint-position differences of bodies 1..23 in the heading frame, local joint
// quaternions of bodies 1..23 and their differences to the expert's); ex1 = expert frame at cur_t + 1; obs_coord "root", obs_vel "full"
template <class Real, class OutT>
UHC_DEVNI void obs_v56(const EnvCfg<Real> &cfg, const Work<Real> &w, const Real *ex1, const Real *shape_obs, OutT *obs) {
    Real crq[4], trq[4], hq[4], hqi[4], ci[4], relq[4], dh[4], R[9];
    remove_base_rot(cfg, w.q + 3, crq); remove_base_rot(cfg, ex1 + EX_QPOS + 3, trq);
    heading_q_new(crq, hq); qinv(hq, hqi); qinv(crq, ci); qmul(trq, ci, relq); qmul(hqi, crq, dh);
    Real rel_h = heading_new(trq) - heading_new(crq);
    if (rel_h > Real(PI_D)) rel_h -= Real(2 * PI_D);
    if (rel_h < -Real(PI_D)) rel_h += Real(2 * PI_D);
    const bool v5 = cfg.obs_v == 5;
    q2mat(v5 ? crq : hq, R);
    LANES_BEGIN
    if (v5) {
        for (int i = lane; i < 74; i += 32) {
            const Real tq = ex1[EX_QPOS + 2 + i];
            Real cur, df;
            if (i == 0) { cur = w.q[2]; df = tq - cur; }
            else if (i < 5) { cur = dh[i - 1]; df = relq[i - 1]; }
            else { cur = w.q[2 + i]; df = tq - cur; }
            obs[i] = (OutT)tq; obs[74 + i] = (OutT)cur; obs[148 + i] = (OutT)df;
        }
        if (lane == 0) {
            Real t[3];
            mtv(R, w.v, t);                                                       // rotated once (:540)
            obs[222] = (OutT)t[0]; obs[223] = (OutT)t[1]; obs[224] = (OutT)t[2];
            obs[297] = (OutT)rel_h;
            const Real rp[3] = {ex1[EX_QPOS] - w.q[0], ex1[EX_QPOS + 1] - w.q[1], ex1[EX_QPOS + 2] - w.q[2]};
            mtv(R, rp, t);
            obs[298] = (OutT)t[0]; obs[299] = (OutT)t[1];
        }
        for (int i = 3 + lane; i < NV; i += 32) obs[222 + i] = (OutT)w.v[i];
        if (lane < NB) {
            const int b = lane; Real r[3], t[3];
            for (int k = 0; k < 3; k++) r[k] = w.xpos[b][k] - w.q[k];
            mtv(R, r, t);
            for (int k = 0; k < 3; k++) obs[300 + 24 * k + b] = (OutT)t[k];
            for (int k = 0; k < 3; k++) r[k] = ex1[EX_WBPOS + 3 * b + k] - w.xpos[b][k];
            mtv(R, r, t);
            for (int k = 0; k < 3; k++) obs[372 + 24 * k + b] = (OutT)t[k];
            const bool use_t = (w.xquat[0][0] == 0);
            const Real *cq = use_t ? ex1 + EX_WBQUAT + 4 * b : w.xquat[b];
            Real o1[4], iq[4], o2[4];
            qmul(hqi, cq, o1);
            const Real nn = rsqrt_(cq[0] * cq[0] + cq[1] * cq[1] + cq[2] * cq[2] + cq[3] * cq[3]);      // inverse_batch = conj / |q|
            iq[0] = cq[0] * nn; iq[1] = -cq[1] * nn; iq[2] = -cq[2] * nn; iq[3] = -cq[3] * nn;
            qmul(iq, ex1 + EX_WBQUAT + 4 * b, o2);
            for (int k = 0; k < 4; k++) { obs[444 + 4 * b + k] = (OutT)o1[k]; obs[540 + 4 * b + k] = (OutT)o2[k]; }
        }
        if (cfg.has_shape && lane < 17) obs[636 + lane] = (OutT)shape_obs[lane];
    } else {
        if (lane == 0) {
            Real t[3];
            const Real rp[3] = {ex1[EX_QPOS] - w.q[0], ex1[EX_QPOS + 1] - w.q[1], ex1[EX_QPOS + 2] - w.q[2]};
            mtv(R, rp, t);
            obs[0] = (OutT)t[0]; obs[1] = (OutT)t[1]; obs[2] = (OutT)t[2];
            obs[3] = (OutT)rel_h;
            for (int k = 0; k < 4; k++) obs[4 + k] = (OutT)relq[k];
            mtv(R, w.v, t);
            obs[8] = (OutT)t[0]; obs[9] = (OutT)t[1]; obs[10] = (OutT)t[2];
        }
        for (int i = 3 + lane; i < NV; i += 32) obs[8 + i] = (OutT)w.v[i];
        if (lane < NB) {
            const int b = lane; Real r[3], t[3];
            for (int k = 0; k < 3; k++) r[k] = w.xpos[b][k] - w.q[k];
            mtv(R, r, t);
            obs[83 + b] = (OutT)t[1]; obs[107 + b] = (OutT)t[2];                 // rows 1.. of the (3, 24) array (:645)
            if (b >= 1) {
                for (int k = 0; k < 3; k++) r[k] = ex1[EX_WBPOS + 3 * b + k] - w.xpos[b][k];
                mtv(R, r, t);
                for (int k = 0; k < 3; k++) obs[131 + 23 * k + (b - 1)] = (OutT)t[k];
                Real bq[4], iq[4], o2[4];
                euler_zyx_quat(w.q[7 + 3 * (b - 1)], w.q[8 + 3 * (b - 1)], w.q[9 + 3 * (b - 1)], bq);      // get_body_quat() of the current qpos (:925-947)
                const Real nn = rsqrt_(bq[0] * bq[0] + bq[1] * bq[1] + bq[2] * bq[2] + bq[3] * bq[3]);
                iq[0] = bq[0] * nn; iq[1] = -bq[1] * nn; iq[2] = -bq[2] * nn; iq[3] = -bq[3] * nn;
                qmul(iq, ex1 + EX_BQUAT + 4 * b, o2);
                for (int k = 0; k < 4; k++) { obs[200 + 4 * (b - 1) + k] = (OutT)bq[k]; obs[292 + 4 * (b - 1) + k] = (OutT)o2[k]; }
            }
        }
        if (cfg.has_shape && lane < 17) obs[384 + lane] = (OutT)shape_obs[lane];
    }
    LANES_END
}

template <class Real> UHC_DEV void rot_from_quat(const Real *q, Real *rv) {  // transformation.py:362-372
    if (abs_(1 - q[0]) < Real(1e-6) || abs_(1 + q[0]) < Real(1e-6)) { rv[0] = rv[1] = rv[2] = 0; return; }
    const Real ang = 2 * acos_(clamp_(q[0], Real(-1), Real(1)));
    Real sn, cs; sincos_(ang * Real(0.5), &sn, &cs);
    const Real ax[3] = {q[1] / sn, q[2] / sn, q[3] / sn};
    const Real n = rsqrt_(dot3(ax, ax)) * ang;
    rv[0] = ax[0] * n; rv[1] = ax[1] * n; rv[2] = ax[2] * n;
}

// termination metric (humanoid_im.py:1408-1415) and world_rfc_implicit reward (reward_function.py:12-88);
// ext = expert frame at the NEW cur_t; bquat/pbquat = current / previous body quats
// rfc_mode 1: world_rfc_explicit (reward_function.py:253-341) -- angular-velocity error NOT weighted by jpos_diffw, residual-force term = sum over the
// bodies' slots of |force|^2 + |torque|^2 of the raw action (:321-327)
template <class Real, class ActT>
UHC_DEVNI void diff_and_reward(const Model<Real> &m, const EnvCfg<Real> &cfg, const Work<Real> &w, const Real *ext, const Real *bquat,
                             const Real *pbquat, Real *body_diff, Real *reward, Real *cinfo, const ActT *act_global) {
    LVAR(Real, s_bd); LVAR(Real, s_n); LVAR(Real, s_pose); LVAR(Real, s_vel); LVAR(Real, s_ee); LVAR(Real, s_vf);
    const bool explicit_rf = cfg.rfc_mode == 1 && act_global != nullptr;
    const Real dtc = m.dt * NSUB;
    LANES_BEGIN
    Real bd = 0, nn = 0, pose = 0, vel = 0, ee = 0, vfs = 0;
    if (lane < NB) {
        const int b = lane; const Real dw = UHC_LDG(m.body_f + b * BODYF + 18);
        if (dw != 0) { Real dx[3]; for (int k = 0; k < 3; k++) dx[k] = (w.xpos[b][k] - ext[EX_WBPOS + 3 * b + k]) * dw; bd = sqrt(dot3(dx, dx)); nn = 1; }
        Real iq[4], dq[4], rv[3];
        qinv(ext + EX_BQUAT + 4 * b, iq); qmul(bquat + 4 * b, iq, dq);
        const Real a = acos_(clamp_(dq[0], Real(-1), Real(1))) * (b == 0 ? Real(1) : dw);
        pose = a * a;
        qinv(pbquat + 4 * b, iq); qmul(bquat + 4 * b, iq, dq); rot_from_quat(dq, rv);
        const Real vw = explicit_rf ? Real(1) : dw;
        for (int k = 0; k < 3; k++) { const Real dv = (rv[k] / dtc - ext[EX_BANGVEL + 3 * b + k]) * vw; vel += dv * dv; }
        if (explicit_rf) for (int k = 3; k < VF_BODY_DIM; k++) { const Real x = (Real)act_global[NU + VF_BODY_DIM * b + k]; vfs += x * x; }
    }
    if (lane < 5) { const int eb = UHC_LDG(m.ee + lane); for (int k = 0; k < 3; k++) { const Real x = w.xpos[eb][k] - ext[EX_EE + 3 * lane + k]; ee += x * x; } }
    LV(s_bd) = bd; LV(s_n) = nn; LV(s_pose) = pose; LV(s_vel) = vel; LV(s_ee) = ee; LV(s_vf) = vfs;
    LANES_END
    const Real bdsum = WSUM(s_bd), nsum = WSUM(s_n), pose2 = WSUM(s_pose), vel2 = WSUM(s_vel), ee2 = WSUM(s_ee);
    *body_diff = bdsum / nsum;
    Real com2 = 0, vf2 = 0;
    for (int k = 0; k < 3; k++) { const Real x = w.xipos[0][k] - ext[EX_COM + k]; com2 += x * x; }
    if (explicit_rf) vf2 = WSUM(s_vf);
    else for (int i = 0; i < 6; i++) vf2 += w.act[NU + i] * w.act[NU + i];
    cinfo[0] = exp_(-cfg.k[0] * pose2); cinfo[1] = exp_(-cfg.k[1] * vel2); cinfo[2] = exp_(-cfg.k[2] * ee2);
    cinfo[3] = exp_(-cfg.k[3] * com2); cinfo[4] = cfg.rfc_mode == 2 ? Real(0) : exp_(-cfg.k[4] * vf2);     // residual_force off: vf_reward = 0.0 (reward_function.py:68-72)
    if (cfg.reward_mul) { *reward = cinfo[0] * cinfo[1] * cinfo[2] * cinfo[3] * (cfg.w[4] != Real(0) ? cinfo[4] : Real(1)); return; }      // reward_function.py:243-245
    Real r = 0, ws = 0;
    for (int i = 0; i < 5; i++) { r += cfg.w[i] * cinfo[i]; ws += cfg.w[i]; }
    *reward = r / ws;
}

}  // namespace uhc
