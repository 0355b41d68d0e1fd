// lane_kernels.cuh -- the stepper (v5): lane-chain Articulated-Body sweeps, 8 lanes per env, 4 envs per warp.
//
// Replaces, for N envs in lockstep, the body of HumanoidEnv.step (smpl_sim/envs/base_env.py:86-100):
//   physics_step      15 x [ctrler.control + mujoco.mj_step]          smpl_sim/envs/humanoid_env.py:439-453, controllers.py:116-190
//   post_physics_step mj_kinematics, self obs v1/v2, task obs, reward  smpl_sim/envs/humanoid_env.py:388-403,455-469,565-688
//   reset             Default / Fall / MoCap                           smpl_sim/envs/humanoid_env.py:471-512
//
// Mapping (a warp per env kept only ~5 of 32 lanes busy and needed ~16 KB of shared memory per env):
//   * an env is stepped by LM_LPE = 8 lanes; a lane walks a kinematic chain, one body per sweep step (host list schedule in
//     LHdr::sched).  Along a chain the sweep state (articulated inertia 21 + bias force 6 inward; pose / velocity /
//     acceleration outward) is handed from step to step IN REGISTERS; only tree junctions use shared-memory mailboxes;
//   * per-body results a lane produces in one sweep and consumes itself in a later one (joint factors K = U/D, c = u/D, bias
//     force) are lane-private "records", kept per body in the env's shared-memory rows (RECW words a body);
//   * four fused sweeps per substep instead of seven passes:
//       S1 outward: stable-PD acceleration (factors of the previous substep) -> torque, kinematics, velocities, bias forces,
//                   rigid inertias, floor contacts and joint-limit rows
//       S2 inward : articulated inertias + bias forces with the working set folded in -> K, c
//       S3 outward: accelerations, residuals of the constraint rows (working-set test)
//       [S2'/S3' : active-set Newton iterations, S2' only over the chains that carry rows; row-space exact line search]
//       S4 inward : semi-implicit Euler of the body's own dofs, then the stable-PD factors (M + h Kd) for the next substep
//   * everything else per env stays in shared memory too (SMPL: 10.1 KB an env with the records), so that an H100 SM (227 KB
//     per CTA) holds 16 envs (4 warps) of the table-plus-rows layout; 4 096 envs are two waves over 132 SMs.
// The mathematics (ABA in world-aligned spatial coordinates about the root origin, MuJoCo's soft-constraint rows as an
// active-set problem solved by ABA passes) is that of round 1's warp_kernels.cuh; DESIGN.md section 2.
#pragma once
#include "dev_model.cuh"
#include "lane_model.hpp"

#define L_FULL 0xffffffffu
#define L_SOLVER_MAXITER 16
#define L_LS_MAXITER 24
#ifndef L_LS_NOISE
#define L_LS_NOISE 1e-4f
#endif
//   L_LS_NOISE:     // line search: directional derivative below this fraction of its two cancelling parts = converged
#define L_LS_MAXSTEP 16.f    // line search: never extrapolate further than this multiple of the Newton step
#define L_MAXVAL 1e10f       // mjMAXVAL (mj_checkPos / Vel / Acc)
// aux.status bits beyond mj_warning's 1 BADQPOS | 2 BADQVEL | 4 BADQACC
#define L_ST_ROWS_DROPPED 8  // more simultaneous joint-limit rows than the kernel holds: the excess rows were not simulated
#define L_ST_MAXITER 16      // the active-set solve stopped at L_SOLVER_MAXITER without reaching its fixed point
#define L_ST_SELF_CONTACT 32 // SMPLSIM_STATUS_SELF_CONTACT: a geom pair MuJoCo would collide touches (not simulated)

// ------------------------------------------------------------------ compile-time sizes / per-env shared-memory layout (words)
template <int NB_, int NV_, int NG_, int NS_, int NMBI_, int NMBO_, int NCS_, int NLS_, int SELFCOL_ = 0>
struct LCfg {
  static constexpr int NB = NB_, NV = NV_, NQ = NV_ + 1, NU = NV_ - 6, NG = NG_, NS = NS_, NMBI = NMBI_, NMBO = NMBO_, NCS = NCS_, NLS = NLS_;
  static constexpr int SELFCOL = SELFCOL_, LPE = LM_LPE, EPW = 32 / LM_LPE;   // SELFCOL: geom-geom (two-body) rows compiled in
  static constexpr int BODYW = 24, MBIW = 28, MBOW = 32, CONW = 24, LIMW = 8, RECW = 28, ROOTW = 44;
  static constexpr int r4(int n) { return (n + 3) & ~3; }
  static constexpr int qpos = 0, qvel = qpos + r4(NQ), qacc = qvel + r4(NV), act = qacc + r4(NV), tau = act + r4(NU), qstar = tau + r4(NU),
                       body = qstar + r4(NV), mbi = body + BODYW * NB, mbo = mbi + MBIW * NMBI, root = mbo + MBOW * NMBO, con = root + ROOTW,
                       lim = con + CONW * NCS, pfl = lim + LIMW * NLS, PFLW = r4((NS + 3) / 4), misc = pfl + PFLW, tsk = misc + 8,
                       rec = tsk + 12, total_ = rec + RECW * NB;
  static constexpr int total = total_ | 4;   // env stride: a multiple of 4 words (float4 rows) but not of 8 (bank spread)
  // staging of the final kinematics / observation row: aliases the mailboxes, the root's 6 x 6 system and the contact list (dead by then).  When
  // the observation row does not fit beside the xquat rows (SMPL-X) it is written straight to global memory instead.
  static constexpr int OBSW = 4 * ((NB * 18 + 16 + 3) / 4);
  static constexpr bool OBS_STAGED = OBSW + 4 * NB <= lim - mbi;
  static constexpr int obs = mbi, xq = OBS_STAGED ? mbi + OBSW : mbi;
  static_assert(xq + 4 * NB <= lim, "xquat staging does not fit the aliased region");
};
// misc words
#define LMI_NCON 0
#define LMI_NLIM 1
#define LMI_DISP 2   // root displacement x, y accumulated over the substeps of this call (words 2, 3)
#define LMI_NSELF 4  // geom-geom contacts of this substep (two list entries each, starting at LMI_SELF0)
#define LMI_SELF0 5
#define L_MAXSELF 4   // simultaneous geom-geom contacts simulated per env (16 two-body rows, two per lane); more are dropped with L_ST_ROWS_DROPPED
#define L_SELFQ (L_MAXSELF / 2)   // two-body rows per lane: lane li owns rows li, li + 8, ...
#define LCE_SELF 64   // info bit: entry A of a geom-geom contact (entry B follows: [0 | n 3 | b1 | b2 | - - | lam 4 | part1 4 | part2 4 | r0 4])
#define LSB_N 1
#define LSB_B1 4
#define LSB_B2 5
#define LSB_LAM 8
#define LSB_P1 12
#define LSB_P2 16
#define LSB_R0 20
// task words (as in round 1)
#define L_TSK_CHANGE 4
#define L_TSK_CURT 5
#define L_TSK_RECOV 6
#define L_TSK_RNG 7
// body row: [ax 9 | xpos 3 | r10 10 | cinfo 1 | spare 1]
#define LBR_AX 0
#define LBR_X 9
#define LBR_R10 12
#define LBR_CI 22
// contact entry: [info | cpos 3 | t1 3 | D | aref 4 | phi 4 | r 4 | rs 4]; info: bit0 present, bits1-4 working set, bits 8-15 geom, 16-23 slot
#define LCE_INFO 0
#define LCE_CP 1
#define LCE_T1 4
#define LCE_D 7
#define LCE_AREF 8
#define LCE_PHI 12
#define LCE_R 16
#define LCE_RS 20
// root scratch (ROOTW words): [A 21 | p 6 | - ] the 6 x 6 system of the free joint, [36..41] its solution (spatial acceleration)
#define LRT_A 36
// limit entry: [dof | sg | D | aref | phi | flag | r | rs]
#define LLE_DOF 0
#define LLE_SG 1
#define LLE_D 2
#define LLE_AREF 3
#define LLE_PHI 4
#define LLE_FLAG 5
#define LLE_R 6
#define LLE_RS 7

struct LLane {
  int li;          // lane within the env group
  int lane;        // lane within the warp
  int gbase;       // first lane of the group
  unsigned gmask;  // warp mask of this env's lanes
  bool live;
  bool bar;        // CTA barriers are legal here (every warp of the CTA makes this call); false inside warp-divergent redo paths
  int env;
  float* gscr;     // overflow contact entries of this env (global scratch)
  float* gbody;    // body quaternion (4) + spatial velocity about the root origin (6) of the current forward pass [10 nb] (self-collision; NULL: off)
  int* gpfl;       // working set per contact slot carried across launches (handle-internal scratch, r4(NS / 4) words per env)
  float* gsens;    // framelinvel / frameangvel of the last forward pass [6 nb] of this env (global scratch; NULL: not wanted)
};

template <class C> __device__ __forceinline__ const LHdr& l_hdr(const float* ms) { return *(const LHdr*)ms; }
__device__ __forceinline__ const LBody* l_bodies(const float* ms) { return (const LBody*)((const char*)ms + LM_BODY_OFF); }
__device__ __forceinline__ const LGeom* l_geoms(const float* ms) { return (const LGeom*)((const char*)ms + ((const LHdr*)ms)->geom_off); }

__device__ __forceinline__ float l_gsum(float v) {
#pragma unroll
  for (int o = LM_LPE / 2; o > 0; o >>= 1) v += __shfl_xor_sync(L_FULL, v, o);
  return v;
}
__device__ __forceinline__ bool l_gall(bool p, const LLane& w) { return (__ballot_sync(L_FULL, p) & w.gmask) == w.gmask; }
__device__ __forceinline__ bool l_gany(bool p, const LLane& w) { return (__ballot_sync(L_FULL, p) & w.gmask) != 0u; }

// joint-diagonal reciprocal: MUFU.RCP + one multiply (1 ulp) instead of the IEEE division sequence with its slow path
__device__ __forceinline__ float l_rcp(float x) { return __fdividef(1.0f, x); }

__device__ __forceinline__ void l_sincos(float x, float* s, float* c) {
  float k = rintf(x * 0.63661977236758134f);
  float r = fmaf(k, -1.5703125f, x);
  r = fmaf(k, -4.837512969970703125e-4f, r);
  r = fmaf(k, -7.549789954891882e-8f, r);
  float z = r * r;
  float sp = fmaf(fmaf(fmaf(-1.9515295891e-4f, z, 8.3321608736e-3f), z, -1.6666654611e-1f), z * r, r);
  float cp = fmaf(fmaf(fmaf(2.443315711809948e-5f, z, -1.388731625493765e-3f), z, 4.166664568298827e-2f), z * z, fmaf(-0.5f, z, 1.0f));
  int q = ((int)k) & 3;
  float ss = (q & 1) ? cp : sp, cc = (q & 1) ? sp : cp;
  *s = (q & 2) ? -ss : ss;
  *c = ((q + 1) & 2) ? -cc : cc;
}

__device__ __noinline__ float l_impedance(const LHdr& H, float pm) {
  float x = fabsf(pm) / fmaxf(H.solimp[2], 1e-15f);
  if (x >= 1.f) return H.solimp[1];
  if (x <= 0.f) return H.solimp[0];
  float y, pw = H.solimp[4];
  if (pw == 2.0f) y = (x <= H.solimp[3]) ? H.imp_a * x * x : 1.f - H.imp_b * (1.f - x) * (1.f - x);
  else if (pw < 1.0000001f && pw > 0.9999999f) y = x;
  else y = (x <= H.solimp[3]) ? H.imp_a * __powf(x, pw) : 1.f - H.imp_b * __powf(1.f - x, pw);
  return H.solimp[0] + y * (H.solimp[1] - H.solimp[0]);
}

// unit wrench of pyramid row k of a floor contact at cp (relative to the root origin): direction n +- mu t1 | n +- mu t2
__device__ __forceinline__ S6 l_wrench(const LHdr& H, V3 cp, V3 t1, int k) {
  V3 n = ld3(H.plane_n);
  V3 t = (k < 2) ? t1 : cross(n, t1);
  float sg = (k & 1) ? -H.mu : H.mu;
  V3 dir = n + sg * t;
  return s6(cross(cp, dir), dir);
}

// direction of pyramid row k in the contact frame (n, t1, t2 = n x t1): n +- mu t1 | n +- mu t2.  The row's unit wrench about the
// root origin is x_k = [cp x d_k ; d_k], so sums over rows factor through 3-vectors: sum D x x^T = X G X^T with G = D sum d d^T
__device__ __forceinline__ V3 l_pyr_dir(const LHdr& H, V3 n, V3 t1, V3 t2, int k) {
  V3 t = (k < 2) ? t1 : t2;
  float sg = (k & 1) ? -H.mu : H.mu;
  return n + sg * t;
}

// ------------------------------------------------------------------ lane records: [K 18 | c 3 | - | pb 6] per body
#ifdef SMPLSIM_EMU
static inline unsigned __float_as_uint(float f) { return emu_bits(f); }
static inline int __float_as_int(float f) { return (int)emu_bits(f); }
static inline float __int_as_float(int i) { return emu_float((unsigned)i); }
static inline float __uint_as_float(unsigned u) { return emu_float(u); }
#endif

// K (3 x 6) and c (3) of body b (b < 0: a lane without a body this step reads body 0's record and ignores it)
template <class C>
__device__ __forceinline__ void l_rec_ld_Kc(float* sm, int b, float* K, float* c) {
  const float4* p = (const float4*)(sm + C::rec + C::RECW * (b < 0 ? 0 : b));
  float4 v0 = p[0], v1 = p[1], v2 = p[2], v3 = p[3], v4 = p[4], v5 = p[5];
  K[0] = v0.x; K[1] = v0.y; K[2] = v0.z; K[3] = v0.w; K[4] = v1.x; K[5] = v1.y; K[6] = v1.z; K[7] = v1.w;
  K[8] = v2.x; K[9] = v2.y; K[10] = v2.z; K[11] = v2.w; K[12] = v3.x; K[13] = v3.y; K[14] = v3.z; K[15] = v3.w;
  K[16] = v4.x; K[17] = v4.y; c[0] = v4.z; c[1] = v4.w; c[2] = v5.x;
}
template <class C>
__device__ __forceinline__ void l_rec_st_Kc(float* sm, int b, const float* K, const float* c, bool wr) {
  if (wr && b >= 0) {
    float4* p = (float4*)(sm + C::rec + C::RECW * b);
    p[0] = make_float4(K[0], K[1], K[2], K[3]); p[1] = make_float4(K[4], K[5], K[6], K[7]);
    p[2] = make_float4(K[8], K[9], K[10], K[11]); p[3] = make_float4(K[12], K[13], K[14], K[15]);
    p[4] = make_float4(K[16], K[17], c[0], c[1]);
    ((float*)p)[20] = c[2];
  }
}
template <class C>
__device__ __forceinline__ S6 l_rec_ld_pb(float* sm, int b) {
  const float* p = sm + C::rec + C::RECW * (b < 0 ? 0 : b) + 22;
  return s6(v3(p[0], p[1], p[2]), v3(p[3], p[4], p[5]));
}
template <class C>
__device__ __forceinline__ void l_rec_st_pb(float* sm, int b, S6 pb, bool wr) {
  if (wr && b >= 0) {
    float* p = sm + C::rec + C::RECW * b + 22;
    st3(p, pb.a); st3(p + 3, pb.l);
  }
}

// contact entry c: the first NCS live in shared memory, the rest in this env's global scratch
template <class C>
__device__ __forceinline__ float* l_centry(float* sm, const LLane& w, int c) {
  return c < C::NCS ? sm + C::con + C::CONW * c : w.gscr + (size_t)C::CONW * (c - C::NCS);
}

// S of hinge k of body row br (axis in world coordinates, moment about the root origin)
__device__ __forceinline__ S6 l_hingeS(const float* br, int k) {
  V3 a = ld3(br + LBR_AX + 3 * k);
  return s6(a, cross(ld3(br + LBR_X), a));
}
__device__ __forceinline__ void l_s6arr(S6 s, float* o) { o[0] = s.a.x; o[1] = s.a.y; o[2] = s.a.z; o[3] = s.l.x; o[4] = s.l.y; o[5] = s.l.z; }
__device__ __forceinline__ S6 l_arr6(const float* o) { return s6(v3(o[0], o[1], o[2]), v3(o[3], o[4], o[5])); }

// rigid-body inertia about the root origin, world axes: m, m r, I (xx yy zz xy xz yz)
__device__ __forceinline__ void l_rigid10(const LBody& lb, Q4 q, V3 x, float* r10) {
  float R[9];
  q2mat(q, R);
  const float* in = lb.inertia;
  float m = lb.mass;
  V3 r = x + mrot(R, ld3(lb.ipos));
  float Il[9] = {in[0], in[3], in[4], in[3], in[1], in[5], in[4], in[5], in[2]}, T[9];
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) T[3 * i + j] = R[3 * i] * Il[j] + R[3 * i + 1] * Il[3 + j] + R[3 * i + 2] * Il[6 + j];
  float rr = dot(r, r);
  r10[0] = m; r10[1] = m * r.x; r10[2] = m * r.y; r10[3] = m * r.z;
  r10[4] = T[0] * R[0] + T[1] * R[1] + T[2] * R[2] + m * (rr - r.x * r.x);
  r10[5] = T[3] * R[3] + T[4] * R[4] + T[5] * R[5] + m * (rr - r.y * r.y);
  r10[6] = T[6] * R[6] + T[7] * R[7] + T[8] * R[8] + m * (rr - r.z * r.z);
  r10[7] = T[0] * R[3] + T[1] * R[4] + T[2] * R[5] - m * r.x * r.y;
  r10[8] = T[0] * R[6] + T[1] * R[7] + T[2] * R[8] - m * r.x * r.z;
  r10[9] = T[3] * R[6] + T[4] * R[7] + T[5] * R[8] - m * r.y * r.z;
}


// ------------------------------------------------------------------ S1: outward sweep
#define LF_GOUT 1      // stable-PD acceleration from the stored factors (FK rows of the previous forward pass) -> torque
#define LF_FK 2        // kinematics of the state in qpos
#define LF_VEL 4       // + velocities, bias accelerations, rigid inertias, bias forces
#define LF_COLLIDE 8   // + floor contacts and joint-limit rows
#define LF_SENS 16     // park framelinvel / frameangvel (quirk Q2: sensors of the last forward pass)
#define LF_XQUAT 32    // store xquat rows (final kinematics)
// out-mailbox of a junction body: [quat 4 | xpos 3 | - | v 6 | ab 6 | pa 6 | a 6]   (pa: the previous substep's spatial
// acceleration with the new joint axes; a: stable-PD acceleration in S1, trial acceleration in S3)
#define LMO_Q 0
#define LMO_X 4
#define LMO_V 8
#define LMO_AB 14
#define LMO_A 20

struct LFkOut { unsigned long long mask; int nrows; int dropped; };

// exclusive scan of v over the 8 lanes of an env group; *total = group sum
__device__ __forceinline__ int l_gscan(int v, const LLane& w, int* total) {
  int inc = v;
#pragma unroll
  for (int o = 1; o < LM_LPE; o <<= 1) {
    int u = __shfl_up_sync(L_FULL, inc, o);
    if (w.li >= o) inc += u;
  }
  *total = __shfl_sync(L_FULL, inc, w.gbase + LM_LPE - 1);
  return inc - v;
}

// ------------------------------------------------------------------ vectorised shared-memory rows (all rows are 16-byte aligned)
__device__ __forceinline__ void l_ld12(const float* p, float* o) {
  const float4* q = (const float4*)p;
  float4 a = q[0], b = q[1], c = q[2];
  o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w; o[4] = b.x; o[5] = b.y; o[6] = b.z; o[7] = b.w; o[8] = c.x; o[9] = c.y; o[10] = c.z; o[11] = c.w;
}
__device__ __forceinline__ void l_st12(float* p, const float* o) {
  float4* q = (float4*)p;
  q[0] = make_float4(o[0], o[1], o[2], o[3]); q[1] = make_float4(o[4], o[5], o[6], o[7]); q[2] = make_float4(o[8], o[9], o[10], o[11]);
}
// body row words 12..23: rigid inertia (10), contact / limit-row info, spare
__device__ __forceinline__ int l_ld_r10(const float* br, float* r10) {
  float t[12];
  l_ld12(br + LBR_R10, t);
#pragma unroll
  for (int j = 0; j < 10; j++) r10[j] = t[j];
  return __float_as_int(t[10]);
}
// in-mailbox: [IA 21 | pA 6 | dirty]
__device__ __forceinline__ bool l_mbi_add(const float* mi, float* A, S6& p) {
  const float4* q = (const float4*)mi;
  float4 v0 = q[0], v1 = q[1], v2 = q[2], v3_ = q[3], v4 = q[4], v5 = q[5], v6 = q[6];
  A[0] += v0.x; A[1] += v0.y; A[2] += v0.z; A[3] += v0.w; A[4] += v1.x; A[5] += v1.y; A[6] += v1.z; A[7] += v1.w;
  A[8] += v2.x; A[9] += v2.y; A[10] += v2.z; A[11] += v2.w; A[12] += v3_.x; A[13] += v3_.y; A[14] += v3_.z; A[15] += v3_.w;
  A[16] += v4.x; A[17] += v4.y; A[18] += v4.z; A[19] += v4.w; A[20] += v5.x;
  p.a.x += v5.y; p.a.y += v5.z; p.a.z += v5.w; p.l.x += v6.x; p.l.y += v6.y; p.l.z += v6.z;
  return __float_as_int(v6.w) != 0;
}
__device__ __forceinline__ void l_mbi_put(float* mi, const float* A, S6 p, bool dirty) {
  float4* q = (float4*)mi;
  q[0] = make_float4(A[0], A[1], A[2], A[3]); q[1] = make_float4(A[4], A[5], A[6], A[7]); q[2] = make_float4(A[8], A[9], A[10], A[11]);
  q[3] = make_float4(A[12], A[13], A[14], A[15]); q[4] = make_float4(A[16], A[17], A[18], A[19]);
  q[5] = make_float4(A[20], p.a.x, p.a.y, p.a.z); q[6] = make_float4(p.l.x, p.l.y, p.l.z, __int_as_float(dirty ? 1 : 0));
}
// out-mailbox pose part [quat 4 | xpos 3 | - | v 6 | ab 6 | pa 6] (words 0..25) and acceleration part (words 26..31)
struct LPose { Q4 q; V3 x; S6 v, ab, pa; };
__device__ __forceinline__ void l_mbo_put_pose(float* mo, const LPose& P) {
  float4* q = (float4*)mo;
  q[0] = make_float4(P.q.w, P.q.x, P.q.y, P.q.z); q[1] = make_float4(P.x.x, P.x.y, P.x.z, 0.f);
  q[2] = make_float4(P.v.a.x, P.v.a.y, P.v.a.z, P.v.l.x); q[3] = make_float4(P.v.l.y, P.v.l.z, P.ab.a.x, P.ab.a.y);
  q[4] = make_float4(P.ab.a.z, P.ab.l.x, P.ab.l.y, P.ab.l.z); q[5] = make_float4(P.pa.a.x, P.pa.a.y, P.pa.a.z, P.pa.l.x);
  mo[24] = P.pa.l.y; mo[25] = P.pa.l.z;
}
__device__ __forceinline__ void l_mbo_get_pose(const float* mo, LPose& P) {
  const float4* q = (const float4*)mo;
  float4 a = q[0], b = q[1], c = q[2], d = q[3], e = q[4], f = q[5];
  P.q.w = a.x; P.q.x = a.y; P.q.y = a.z; P.q.z = a.w; P.x = v3(b.x, b.y, b.z);
  P.v = s6(v3(c.x, c.y, c.z), v3(c.w, d.x, d.y)); P.ab = s6(v3(d.z, d.w, e.x), v3(e.y, e.z, e.w));
  P.pa = s6(v3(f.x, f.y, f.z), v3(f.w, mo[24], mo[25]));
}
__device__ __forceinline__ void l_mbo_put_acc(float* mo, S6 a) {
  mo[26] = a.a.x; mo[27] = a.a.y;
  ((float4*)mo)[7] = make_float4(a.a.z, a.l.x, a.l.y, a.l.z);
}
__device__ __forceinline__ S6 l_mbo_get_acc(const float* mo) {
  float4 a = ((const float4*)mo)[7];
  return s6(v3(mo[26], mo[27], a.x), v3(a.y, a.z, a.w));
}
// joint axes + body position of a body row (words 0..11)
struct LAxes { V3 a0, a1, a2, x; };
__device__ __forceinline__ LAxes l_ld_axes(const float* br) {
  float t[12];
  l_ld12(br, t);
  LAxes r; r.a0 = v3(t[0], t[1], t[2]); r.a1 = v3(t[3], t[4], t[5]); r.a2 = v3(t[6], t[7], t[8]); r.x = v3(t[9], t[10], t[11]);
  return r;
}
__device__ __forceinline__ V3 l_axis(const LAxes& X, int k) { return k == 0 ? X.a0 : k == 1 ? X.a1 : X.a2; }

// residuals rs = J a - aref of the body's contact rows at acceleration a; returns "sign pattern == working set"
template <class C>
__device__ __forceinline__ bool l_rows_eval(const LHdr& H, float* sm, const LLane& w, int cb, int cn, S6 a) {
  bool same = true;
  for (int c = cb; c < cb + cn; c++) {
    float* ce = (c < C::NCS) ? nullptr : w.gscr + (size_t)C::CONW * (c - C::NCS);
    float e[12];
    if (c < C::NCS) l_ld12(sm + C::con + C::CONW * c, e);
    else for (int j = 0; j < 12; j++) e[j] = ce[j];
    const int info = __float_as_int(e[0]);
    if (!(info & 1)) continue;
    V3 cpt = v3(e[1], e[2], e[3]), t1 = v3(e[4], e[5], e[6]);
    const V3 n = ld3(H.plane_n), t2 = cross(n, t1);
    const V3 ac = a.l + cross(a.a, cpt);    // X^T a: acceleration of the contact point
    int nf = 0;
    float rs[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
      rs[k] = dot(l_pyr_dir(H, n, t1, t2, k), ac) - e[8 + k];
      if (rs[k] < 0.f) nf |= 2 << k;
    }
    if (c < C::NCS) ((float4*)(sm + C::con + C::CONW * c))[LCE_RS / 4] = make_float4(rs[0], rs[1], rs[2], rs[3]);
    else for (int k = 0; k < 4; k++) ce[LCE_RS + k] = rs[k];
    if (nf != (info & 30)) same = false;
  }
  return same;
}

// rigid inertia, bias force, sensors, xquat of the body whose pose is P; returns pb
template <class C>
__device__ __forceinline__ S6 l_body_post(const LBody& lb, float* sm, const LLane& w, int b, int flags, const LPose& P, float* br, int ci) {
  S6 pbv = s6(v3(0.f, 0.f, 0.f), v3(0.f, 0.f, 0.f));
  if (flags & LF_VEL) {
    float t[12];
    l_rigid10(lb, P.q, P.x, t);
    t[10] = __int_as_float(ci); t[11] = 0.f;
    l_st12(br + LBR_R10, t);
    pbv = rb_mul(t, P.ab) + cross_force(P.v, rb_mul(t, P.v));
    if ((flags & LF_SENS) && w.gsens) {
      st3(w.gsens + 6 * b, P.v.l + cross(P.v.a, P.x));
      st3(w.gsens + 6 * b + 3, P.v.a);
    }
  }
  if (flags & LF_XQUAT) ((float4*)(sm + C::xq))[b] = make_float4(P.q.w, P.q.x, P.q.y, P.q.z);
  if (C::SELFCOL && (flags & LF_COLLIDE) && w.gbody) {     // pose / velocity of every body for the geom-geom narrow phase that follows the sweep
    float* gb = w.gbody + 10 * b;
    gb[0] = P.q.w; gb[1] = P.q.x; gb[2] = P.q.y; gb[3] = P.q.z;
    st6(gb + 4, P.v);
  }
  return pbv;
}

// broad phase of the body's geom against the floor: number of contact entries to reserve (exact: > 0 iff at least one contact)
struct LGeomCtx { float R[9]; V3 c, ax; float d0, na; V3 e0, e1, e2; float l0, l1, l2; };   // box: half edges in world axes, their heights along the plane normal
__device__ __forceinline__ int l_broad(const LHdr& H, const LGeom& G, const LPose& P, float h0, LGeomCtx& X) {
  const V3 pn = ld3(H.plane_n);
  q2mat(P.q, X.R);
  X.c = P.x + mrot(X.R, ld3(G.pos));
  X.d0 = h0 + dot(pn, X.c);
  X.ax = v3(0.f, 0.f, 0.f); X.na = 0.f;
  X.e0 = X.e1 = X.e2 = v3(0.f, 0.f, 0.f); X.l0 = X.l1 = X.l2 = 0.f;
  if (G.type == SMPLSIM_GEOM_BOX) {
    X.e0 = G.size[0] * mrot(X.R, v3(G.mat[0], G.mat[3], G.mat[6]));
    X.e1 = G.size[1] * mrot(X.R, v3(G.mat[1], G.mat[4], G.mat[7]));
    X.e2 = G.size[2] * mrot(X.R, v3(G.mat[2], G.mat[5], G.mat[8]));
    X.l0 = dot(pn, X.e0); X.l1 = dot(pn, X.e1); X.l2 = dot(pn, X.e2);
    return (X.d0 - (fabsf(X.l0) + fabsf(X.l1) + fabsf(X.l2)) <= H.margin) ? 4 : 0;
  }
  X.ax = mrot(X.R, v3(G.mat[2], G.mat[5], G.mat[8]));
  X.na = dot(pn, X.ax);
  float hl = (G.type == SMPLSIM_GEOM_CAPSULE) ? G.size[1] : 0.f;
  return (X.d0 - hl * fabsf(X.na) - G.size[0] <= H.margin) ? ((G.type == SMPLSIM_GEOM_CAPSULE) ? 2 : 1) : 0;
}

// narrow phase (plane vs box corners / capsule ends / sphere, SURVEY A.5) into the reserved entries [cb, cb + alloc); returns
// the number of contacts
template <class C>
__device__ __forceinline__ int l_narrow(const LHdr& H, const LGeom& G, int g, const LGeomCtx& X, S6 vb, S6 pa, float tiw0, float* sm, const LLane& w, int cb, int alloc) {
  const V3 pn = ld3(H.plane_n);
  const unsigned char* pf = (const unsigned char*)(sm + C::pfl);
  V3 t1 = ld3(H.t1_default);
  int cnt = 0;
  const int npt = (G.type == SMPLSIM_GEOM_BOX) ? 8 : alloc;
  if (G.type == SMPLSIM_GEOM_CAPSULE) {
    t1 = X.ax - X.na * pn;
    float nn = sqrtf(dot(t1, t1));
    t1 = (nn < 1e-15f) ? v3(1.f, 0.f, 0.f) : (1.0f / nn) * t1;
  }
#pragma unroll 1
  for (int i = 0; i < npt && cnt < alloc; i++) {
    V3 cp; float dist;
    if (G.type == SMPLSIM_GEOM_BOX) {
      const float s0 = (i & 1) ? 1.f : -1.f, s1 = (i & 2) ? 1.f : -1.f, s2 = (i & 4) ? 1.f : -1.f;   // corner = centre +- e0 +- e1 +- e2
      const float l = s0 * X.l0 + s1 * X.l1 + s2 * X.l2;
      if (X.d0 + l > H.margin || l > 0.f) continue;
      dist = X.d0 + l;
      cp = X.c + (s0 * X.e0 + s1 * X.e1 + s2 * X.e2) - (0.5f * dist) * pn;
    } else {
      float hl = (G.type == SMPLSIM_GEOM_CAPSULE) ? G.size[1] : 0.f, sg = i ? -hl : hl;
      dist = X.d0 + sg * X.na - G.size[0];
      if (dist > H.margin) continue;
      cp = X.c + sg * X.ax - (G.size[0] + 0.5f * dist) * pn;
    }
    float pm = dist - H.margin, imp = l_impedance(H, pm);
    float R0 = fmaxf((1.f - imp) / imp * (tiw0 + H.mu * H.mu * tiw0), 1e-15f);
    float R1 = R0 / fmaxf(H.impratio, 1e-15f), mu = H.mu * sqrtf(R1 / R0);
    float kterm = H.K * imp * pm;
    // working set inherited from the slot's previous substep; a new contact starts from the rows that would be violated if the
    // body kept the acceleration it had in the previous substep
    int slot = G.slot0 + cnt, pv = pf[slot], guess = 32;   // bit 5: new this substep
    float e[12];
    e[1] = cp.x; e[2] = cp.y; e[3] = cp.z; e[4] = t1.x; e[5] = t1.y; e[6] = t1.z;
    e[7] = 1.0f / (2.f * mu * mu * R0);
    {
      const V3 t2 = cross(pn, t1);
      const V3 vc = vb.l + cross(vb.a, cp), pc = pa.l + cross(pa.a, cp);   // velocity / previous acceleration of the contact point
#pragma unroll
      for (int k = 0; k < 4; k++) {
        V3 d = l_pyr_dir(H, pn, t1, t2, k);
        e[8 + k] = -H.B * dot(d, vc) - kterm;
        if (dot(d, pc) - e[8 + k] < 0.f) guess |= 2 << k;
      }
    }
    e[0] = __int_as_float(1 | ((pv & 1) ? (pv & 30) : guess) | (g << 8) | (slot << 16));
#ifdef SMPLSIM_STATS
    e[0] = __int_as_float(__float_as_int(e[0]) | ((((pv & 1) ? (pv & 30) : 30) >> 1) << 24) | (((guess & 30) >> 1) << 28));
#endif
    const int c = cb + cnt;
    if (c < C::NCS) l_st12(sm + C::con + C::CONW * c, e);
    else { float* ce = w.gscr + (size_t)C::CONW * (c - C::NCS); for (int j = 0; j < 12; j++) ce[j] = e[j]; }
    cnt++;
  }
  for (int i = cnt; i < alloc; i++) {
    const int c = cb + i;
    if (c < C::NCS) ((int*)(sm + C::con + C::CONW * c))[LCE_INFO] = 0;
    else ((int*)(w.gscr + (size_t)C::CONW * (c - C::NCS)))[LCE_INFO] = 0;
  }
  return cnt;
}

// root body of the outward sweep (free joint; lane 0 of the group, step 0; every lane makes the call): stable-PD
// acceleration of the root (solved at the end of the last inward sweep), pose / velocity / bias acceleration of the state in qpos, qvel,
// rigid inertia, bias force, contacts of the root's geom.  Children read the pose from the root's out-mailbox.
struct LRootOut { int ncon, npresent; unsigned long long gbits; };
template <class C>
__device__ __noinline__ LRootOut l_root_out(const float* ms, float* sm, const LLane& w, int flags, float h0) {
  const LHdr& H = l_hdr<C>(ms);
  const LBody& lb = l_bodies(ms)[0];
  LRootOut R; R.ncon = 0; R.npresent = 0; R.gbits = 0ull;
  const bool actv = w.live && w.li == 0;
  S6 pbv = s6(v3(0.f, 0.f, 0.f), v3(0.f, 0.f, 0.f));
  int alloc = 0;
  if (actv) {
    float* br = sm + C::body;
    float* mo = sm + C::mbo + C::MBOW * lb.out_mbox;
    float* qpos = sm + C::qpos;
    const float* qvel = sm + C::qvel;
    if (flags & LF_GOUT) l_mbo_put_acc(mo, ld6(sm + C::root + LRT_A));   // stable-PD acceleration of the root, solved at the end of the inward sweep
    if (flags & LF_FK) {
      LPose P;
      P.q.w = qpos[3]; P.q.x = qpos[4]; P.q.y = qpos[5]; P.q.z = qpos[6];
      P.q = qnormalize(P.q);
      qpos[3] = P.q.w; qpos[4] = P.q.x; qpos[5] = P.q.y; qpos[6] = P.q.z;
      float Rm[9];
      q2mat(P.q, Rm);
      V3 c0 = v3(Rm[0], Rm[3], Rm[6]), c1 = v3(Rm[1], Rm[4], Rm[7]), c2 = v3(Rm[2], Rm[5], Rm[8]);
      st3(br + LBR_AX, c0); st3(br + LBR_AX + 3, c1); st3(br + LBR_AX + 6, c2);
      P.x = v3(0.f, 0.f, 0.f);
      st3(br + LBR_X, P.x);
      P.v = s6(P.x, P.x); P.ab = P.v; P.pa = P.v;
      if (flags & LF_VEL) {
        V3 vl = ld3(qvel), wv = qvel[3] * c0 + qvel[4] * c1 + qvel[5] * c2;
        P.v = s6(wv, vl);
        P.ab = s6(v3(0.f, 0.f, 0.f), v3(-H.grav[0], -H.grav[1], -H.grav[2]) + cross(vl, wv));
        const float* qa = sm + C::qacc;   // acceleration of the previous substep (qacc_warmstart), new rotation columns
        P.pa = s6(qa[3] * c0 + qa[4] * c1 + qa[5] * c2, ld3(qa));
      }
      l_mbo_put_pose(mo, P);
      LGeomCtx X;
      if ((flags & LF_COLLIDE) && lb.ngeom > 0) alloc = l_broad(H, l_geoms(ms)[lb.geom0], P, h0, X);
      pbv = l_body_post<C>(lb, sm, w, 0, flags, P, br, alloc << 8);
      if (alloc) {
        int cnt = l_narrow<C>(H, l_geoms(ms)[lb.geom0], lb.geom0, X, P.v, P.pa, lb.tiw0, sm, w, 0, alloc);
        if (cnt) R.gbits = 1ull << (lb.geom0 + 1);
        R.npresent = cnt;
      }
    }
  }
  if (flags & LF_VEL) l_rec_st_pb<C>(sm, 0, pbv, actv);
  R.ncon = __shfl_sync(L_FULL, alloc, w.gbase);
  __syncwarp();
  return R;
}

template <class C>
__device__ __noinline__ LFkOut l_sweep_out(const float* ms, float* sm, const LLane& w, int flags, bool ztau) {
  const LHdr& H = l_hdr<C>(ms);
  const LBody* MB = l_bodies(ms);
  const LGeom* MG = l_geoms(ms);
  const int li = w.li, T = H.T;
  const bool live = w.live;
  const float hh = H.h;
  const float h0 = dot(ld3(H.plane_n), ld3(sm + C::qpos) - ld3(H.plane_pos));
  LRootOut R0 = l_root_out<C>(ms, sm, w, flags, h0);
  LPose P;   // pose / velocity / bias acceleration handed down the lane's chain
  P.q.w = 1.f; P.q.x = P.q.y = P.q.z = 0.f; P.x = v3(0.f, 0.f, 0.f); P.v = s6(P.x, P.x); P.ab = P.v; P.pa = P.v;
  S6 casp = P.v;
  int ncon = R0.ncon, nlim = 0, npresent = R0.npresent, dropped = 0;
  unsigned long long gbits = R0.gbits;
  const bool spd_torque = (flags & LF_GOUT) && H.cfg.control_mode == SMPLSIM_CTRL_UHC_PD;
  const bool stepbar = (H.align & 16) && w.bar;
  for (int t = 1; t < T; t++) {
    if (stepbar) __syncthreads();
    const int b = H.sched[t][li];
    const bool actv = live && b >= 0;
    float K[18], kc[3];
    if (flags & LF_GOUT) l_rec_ld_Kc<C>(sm, b, K, kc);
    S6 pbv = s6(v3(0.f, 0.f, 0.f), v3(0.f, 0.f, 0.f));
    float* br = sm + C::body + C::BODYW * (actv ? b : 0);
    int alloc = 0, nlr = 0;   // contact entries / limit rows this lane wants
    LGeomCtx X;
    if (actv) {
      const LBody& lb = MB[b];
      const int d0 = lb.dofadr;
      if (!(lb.flags & LB_CARRY_OUT)) {   // junction: the parent's lane left its state in the mailbox
        const float* mo = sm + C::mbo + C::MBOW * lb.pmbox;
        if (flags & LF_FK) l_mbo_get_pose(mo, P);
        if (flags & LF_GOUT) casp = l_mbo_get_acc(mo);
      }
      const float q0 = sm[C::qpos + d0 + 1], q1 = sm[C::qpos + d0 + 2], q2 = sm[C::qpos + d0 + 3];
      const float qd0 = sm[C::qvel + d0], qd1 = sm[C::qvel + d0 + 1], qd2 = sm[C::qvel + d0 + 2];
      if (flags & LF_GOUT) {
        // stable-PD acceleration of this body's dofs: qdd_k = c_k - K_k . a  (joint axes / position of the last forward pass)
        const LAxes AX = l_ld_axes(br);
        S6 a = casp;
#pragma unroll
        for (int k = 0; k < 3; k++) {
          V3 ax = l_axis(AX, k);
          S6 S = s6(ax, cross(AX.x, ax));
          float qdd = kc[k] - dot6(l_arr6(K + 6 * k), a);
          a = a + qdd * S;
          if (spd_torque) {      // controllers.py:165-190 with the acceleration already solved: tau = -kp (q + qd h - tgt) - kd (qd + qdd h)
            const int i = d0 + k - 6;
            float q = k == 0 ? q0 : k == 1 ? q1 : q2, qd = k == 0 ? qd0 : k == 1 ? qd1 : qd2;
            float tgt = fmaf(sm[C::act + i], lb.ascale[k], lb.aoffset[k]);
            float tq = -lb.kp[k] * (q + qd * hh - tgt) - lb.kd[k] * (qd + qdd * hh);
            tq = fminf(fmaxf(tq, -lb.tlim[k]), lb.tlim[k]);
            sm[C::tau + i] = ztau ? 0.f : tq;
          }
        }
        casp = a;
        if (lb.out_mbox >= 0) l_mbo_put_acc(sm + C::mbo + C::MBOW * lb.out_mbox, casp);
      }
      if (flags & LF_FK) {
        float Rp[9], row[12];
        q2mat(P.q, Rp);
        V3 x = P.x + mrot(Rp, ld3(lb.bpos));
        const bool xyz = H.axes_xyz != 0;     // warp-uniform: identity body quaternion, hinge axes x, y, z (SMPL family)
        Q4 qc = P.q;
        if (!xyz) { Q4 qb; qb.w = lb.bquat[0]; qb.x = lb.bquat[1]; qb.y = lb.bquat[2]; qb.z = lb.bquat[3]; qc = qmul(P.q, qb); }
        S6 v = P.v, ab = P.ab, pa = P.pa;
#pragma unroll
        for (int k = 0; k < 3; k++) {
          V3 al = xyz ? v3(k == 0 ? 1.f : 0.f, k == 1 ? 1.f : 0.f, k == 2 ? 1.f : 0.f) : ld3(lb.axis + 3 * k);
          V3 a;
          if (xyz) {   // column k of the rotation matrix of the running quaternion
            const float qw = qc.w, qx = qc.x, qy = qc.y, qz = qc.z;
            a = (k == 0) ? v3(Rp[0], Rp[3], Rp[6])
              : (k == 1) ? v3(2.f * (qx * qy - qw * qz), 1.f - 2.f * (qx * qx + qz * qz), 2.f * (qy * qz + qw * qx))
                         : v3(2.f * (qx * qz + qw * qy), 2.f * (qy * qz - qw * qx), 1.f - 2.f * (qx * qx + qy * qy));
          } else a = qrot(qc, al);
          row[3 * k] = a.x; row[3 * k + 1] = a.y; row[3 * k + 2] = a.z;
          if (flags & LF_VEL) {
            S6 S = s6(a, cross(x, a));
            float qd = k == 0 ? qd0 : k == 1 ? qd1 : qd2;
            ab = ab + qd * cross_motion(v, S);
            v = v + qd * S;
            if (flags & LF_COLLIDE) pa = pa + sm[C::qacc + d0 + k] * S;   // previous acceleration: working-set guess of new contacts
          }
          float sn, cs;
          l_sincos(0.5f * (k == 0 ? q0 : k == 1 ? q1 : q2), &sn, &cs);
          if (xyz) {   // qc * (cs, sn e_k)
            Q4 r;
            if (k == 0) { r.w = qc.w * cs - qc.x * sn; r.x = qc.w * sn + qc.x * cs; r.y = qc.y * cs + qc.z * sn; r.z = qc.z * cs - qc.y * sn; }
            else if (k == 1) { r.w = qc.w * cs - qc.y * sn; r.x = qc.x * cs - qc.z * sn; r.y = qc.w * sn + qc.y * cs; r.z = qc.z * cs + qc.x * sn; }
            else { r.w = qc.w * cs - qc.z * sn; r.x = qc.x * cs + qc.y * sn; r.y = qc.y * cs - qc.x * sn; r.z = qc.w * sn + qc.z * cs; }
            qc = r;
          } else {
            Q4 qj; qj.w = cs; qj.x = al.x * sn; qj.y = al.y * sn; qj.z = al.z * sn;
            qc = qmul(qc, qj);
          }
        }
        qc = qnormalize(qc);
        row[9] = x.x; row[10] = x.y; row[11] = x.z;
        l_st12(br, row);
        P.q = qc; P.x = x; P.v = v; P.ab = ab; P.pa = pa;
        if (lb.out_mbox >= 0) l_mbo_put_pose(sm + C::mbo + C::MBOW * lb.out_mbox, P);
        if (flags & LF_COLLIDE) {
          if (lb.ngeom > 0) alloc = l_broad(H, MG[lb.geom0], P, h0, X);
#pragma unroll
          for (int k = 0; k < 3; k++) {
            float q = k == 0 ? q0 : k == 1 ? q1 : q2;
            if (((lb.limited >> k) & 1) && (q - lb.rlo[k] < 0.f || lb.rhi[k] - q < 0.f)) nlr++;
          }
        }
      }
    }
    int cb = 0, lbs = 0, lcnt = 0;
    if (flags & LF_COLLIDE) {
      // ---------------- reserve list space: deterministic order (step, lane)
      int tot, ex = l_gscan(alloc | (nlr << 8), w, &tot);
      cb = ncon + (ex & 255); lbs = nlim + (ex >> 8);
      ncon += tot & 255; nlim += tot >> 8;
      lcnt = nlr;
      if (lbs + nlr > C::NLS) { lcnt = max(0, C::NLS - lbs); if (nlr) dropped = 1; }
    }
    if (actv && (flags & LF_FK)) {
      const LBody& lb = MB[b];
      pbv = l_body_post<C>(lb, sm, w, b, flags, P, br, cb | (alloc << 8) | (lbs << 16) | (lcnt << 24));
      if (alloc) {
        int cnt = l_narrow<C>(H, MG[lb.geom0], lb.geom0, X, P.v, P.pa, lb.tiw0, sm, w, cb, alloc);
        if (cnt) gbits |= 1ull << (lb.geom0 + 1);
        npresent += cnt;
      }
      if (lcnt) {
        int e = lbs;
#pragma unroll
        for (int k = 0; k < 3; k++) {
          int d = lb.dofadr + k;
          float q = sm[C::qpos + d + 1], dlo = q - lb.rlo[k], dhi = lb.rhi[k] - q, dist, sg;
          if (!((lb.limited >> k) & 1)) continue;
          if (dlo < 0.f) { dist = dlo; sg = 1.f; }
          else if (dhi < 0.f) { dist = dhi; sg = -1.f; }
          else continue;
          if (e >= lbs + lcnt) continue;
          float* le = sm + C::lim + C::LIMW * e;
          float imp = l_impedance(H, dist);
          float4* l4 = (float4*)le;
          l4[0] = make_float4(__int_as_float(d), sg, 1.0f / fmaxf((1.f - imp) / imp * lb.diw0[k], 1e-15f), -H.B * sg * sm[C::qvel + d] - H.K * imp * dist);
          l4[1] = make_float4(0.f, __int_as_float(1), 0.f, 0.f);
          e++;
        }
        npresent += lcnt;
      }
    }
    if (flags & LF_VEL) l_rec_st_pb<C>(sm, b, pbv, actv);
    __syncwarp();
  }
  LFkOut o;
  if (flags & LF_COLLIDE) {
    if (w.live && w.li == 0) { ((int*)sm)[C::misc + LMI_NCON] = ncon; ((int*)sm)[C::misc + LMI_NLIM] = min(nlim, C::NLS); ((int*)sm)[C::misc + LMI_NSELF] = 0; }
    unsigned lo = (unsigned)(gbits & 0xffffffffull), hi = (unsigned)(gbits >> 32);
#pragma unroll
    for (int of = LM_LPE / 2; of > 0; of >>= 1) {
      lo |= __shfl_xor_sync(L_FULL, lo, of); hi |= __shfl_xor_sync(L_FULL, hi, of);
      npresent += __shfl_xor_sync(L_FULL, npresent, of); dropped |= __shfl_xor_sync(L_FULL, dropped, of);
    }
    o.mask = ((unsigned long long)hi << 32) | lo;
    __syncwarp();
  } else o.mask = 0ull;
  o.nrows = npresent; o.dropped = dropped;
  return o;
}

// ------------------------------------------------------------------ S2 / S4: inward sweep (articulated inertias, bias forces -> K, c)
#define LI_SPD 1        // stable-PD system (controllers.py:165-190): D += h kd, joint force -kp e - kd qd of the state in qpos / qvel, no rows
#define LI_INTEGRATE 2  // semi-implicit Euler of the body's own dofs first (qvel += h qacc ; qpos += h qvel), then LI_SPD on the new state
#define LI_RESWEEP 4    // only bodies whose bit is set in st.rc_bits (chains carrying constraint rows); the other records are kept

struct LSolveLane {       // lane-private sweep bookkeeping of one substep
  unsigned dirty_bits;    // bit t: the body of step t has constraint rows in its subtree
  unsigned rc_bits;       // bit t: the body of step t is recomputed by re-sweeps (dirty, or hands its result over in registers to such a body)
};

// the active rows of the body's contacts folded into its articulated inertia / bias force: A += D x x^T, p -= D aref x
template <class C>
__device__ __forceinline__ void l_fold_contacts(const LHdr& H, float* sm, const LLane& w, int cb, int cn, float* A, S6& p) {
  for (int c = cb; c < cb + cn; c++) {
    float e[12];
    if (c < C::NCS) l_ld12(sm + C::con + C::CONW * c, e);
    else { const float* ce = w.gscr + (size_t)C::CONW * (c - C::NCS); for (int j = 0; j < 12; j++) e[j] = ce[j]; }
    const int info = __float_as_int(e[0]);
    if (!(info & 1) || !(info & 30)) continue;
    V3 cpt = v3(e[1], e[2], e[3]), t1 = v3(e[4], e[5], e[6]);
    const V3 n = ld3(H.plane_n), t2 = cross(n, t1);
    const float D = e[7];
    // G = D sum_active d d^T (xx yy zz xy xz yz), f = D sum_active aref d
    float gxx = 0.f, gyy = 0.f, gzz = 0.f, gxy = 0.f, gxz = 0.f, gyz = 0.f;
    V3 f = v3(0.f, 0.f, 0.f);
#pragma unroll
    for (int k = 0; k < 4; k++) {
      if (!(info & (2 << k))) continue;
      V3 d = l_pyr_dir(H, n, t1, t2, k);
      V3 dd = D * d;
      gxx = fmaf(dd.x, d.x, gxx); gyy = fmaf(dd.y, d.y, gyy); gzz = fmaf(dd.z, d.z, gzz);
      gxy = fmaf(dd.x, d.y, gxy); gxz = fmaf(dd.x, d.z, gxz); gyz = fmaf(dd.y, d.z, gyz);
      f = f + e[8 + k] * dd;
    }
    // A += X G X^T with X = [[cp]x ; I]:  A_ll += G ; A_al += [cp]x G ; A_aa += [cp]x G [cp]x^T
    const V3 g0 = v3(gxx, gxy, gxz), g1 = v3(gxy, gyy, gyz), g2 = v3(gxz, gyz, gzz);   // columns (= rows) of G
    const V3 c0 = cross(cpt, g0), c1 = cross(cpt, g1), c2 = cross(cpt, g2);           // columns of M = [cp]x G  (3 x 3)
    A[sidx(3, 3)] += gxx; A[sidx(4, 4)] += gyy; A[sidx(5, 5)] += gzz; A[sidx(3, 4)] += gxy; A[sidx(3, 5)] += gxz; A[sidx(4, 5)] += gyz;
    A[sidx(0, 3)] += c0.x; A[sidx(1, 3)] += c0.y; A[sidx(2, 3)] += c0.z;
    A[sidx(0, 4)] += c1.x; A[sidx(1, 4)] += c1.y; A[sidx(2, 4)] += c1.z;
    A[sidx(0, 5)] += c2.x; A[sidx(1, 5)] += c2.y; A[sidx(2, 5)] += c2.z;
    // A_aa += M [cp]x^T : row i of M is (c0.i, c1.i, c2.i); (M [cp]x^T)_ij = (cp x row_i)_j ... symmetric, upper triangle
    const V3 r0 = v3(c0.x, c1.x, c2.x), r1 = v3(c0.y, c1.y, c2.y), r2 = v3(c0.z, c1.z, c2.z);
    const V3 m0 = cross(cpt, r0), m1 = cross(cpt, r1), m2 = cross(cpt, r2);
    A[sidx(0, 0)] += m0.x; A[sidx(0, 1)] += m0.y; A[sidx(0, 2)] += m0.z; A[sidx(1, 1)] += m1.y; A[sidx(1, 2)] += m1.z; A[sidx(2, 2)] += m2.z;
    p.l = p.l - f; p.a = p.a - cross(cpt, f);
  }
}

// closest points of the segments c1 + s a1 (|s| <= h1) and c2 + t a2 (|t| <= h2), a1, a2 unit: clamped solution
__device__ __forceinline__ void l_segment_segment(V3 c1, V3 a1, float h1, V3 c2, V3 a2, float h2, float* so, float* to) {
  V3 r = c1 - c2;
  float b = dot(a1, a2), cc = dot(a1, r), f = dot(a2, r), den = 1.0f - b * b;
  float s = (den > 1e-6f) ? (b * f - cc) / den : 0.f;
  s = fminf(fmaxf(s, -h1), h1);
  float t = b * s + f;
  if (t > h2) { t = h2; s = fminf(fmaxf(b * t - cc, -h1), h1); }
  else if (t < -h2) { t = -h2; s = fminf(fmaxf(b * t - cc, -h1), h1); }
  *so = s; *to = t;
}


// ------------------------------------------------------------------ geom-geom contacts (self-collision): two-body rows
// A contact between bodies b1, b2 has J a = x . (a_b2 - a_b1): it cannot be folded into one body's articulated inertia.  Its rows live
// in the same list as the floor rows (entry A: point, tangent, D, aref, phi, r, rs; entry B: normal, bodies, multipliers, partial
// row values) and enter the ABA passes as EXTERNAL wrenches lam_k x_k (+ on b2, - on b1); l_linsolve finds the multipliers of the
// active rows by Woodbury on top of the factors of the current working set.
template <class C>
__device__ __forceinline__ bool l_self_touches(const float* sm, const LLane& w, int b) {
  const int ns = ((const int*)sm)[C::misc + LMI_NSELF];
  bool t = false;
  for (int s = 0; s < ns; s++) {
    const int* eb = (const int*)l_centry<C>((float*)sm, w, ((const int*)sm)[C::misc + LMI_SELF0] + 2 * s + 1);
    t = t || eb[LSB_B1] == b || eb[LSB_B2] == b;
  }
  return t;
}
// bias force of body b -= external wrench of the geom-geom rows: f = sum_k lam_k d_k at cp, + on b2, - on b1
template <class C>
__device__ __forceinline__ void l_self_wrench(const LHdr& H, float* sm, const LLane& w, int b, S6& p) {
  const int ns = ((const int*)sm)[C::misc + LMI_NSELF];
  for (int s = 0; s < ns; s++) {
    const int c0 = ((const int*)sm)[C::misc + LMI_SELF0] + 2 * s;
    const float* ea = l_centry<C>(sm, w, c0); const float* eb = l_centry<C>(sm, w, c0 + 1);
    const int b1 = ((const int*)eb)[LSB_B1], b2 = ((const int*)eb)[LSB_B2];
    if (b != b1 && b != b2) continue;
    const V3 n = ld3(eb + LSB_N), t1 = ld3(ea + LCE_T1), t2 = cross(n, t1), cp = ld3(ea + LCE_CP);
    V3 f = v3(0.f, 0.f, 0.f);
#pragma unroll
    for (int k = 0; k < 4; k++) f = f + eb[LSB_LAM + k] * l_pyr_dir(H, n, t1, t2, k);
    if (b == b1) f = -1.0f * f;
    p.l = p.l - f; p.a = p.a - cross(cp, f);
  }
}
// partial row values x_k . a_b of the geom-geom rows that touch body b (part1 for b1, part2 for b2)
template <class C>
__device__ __forceinline__ void l_self_part(const LHdr& H, float* sm, const LLane& w, int b, S6 a) {
  const int ns = ((const int*)sm)[C::misc + LMI_NSELF];
  for (int s = 0; s < ns; s++) {
    const int c0 = ((const int*)sm)[C::misc + LMI_SELF0] + 2 * s;
    const float* ea = l_centry<C>(sm, w, c0); float* eb = l_centry<C>(sm, w, c0 + 1);
    const int b1 = ((const int*)eb)[LSB_B1], b2 = ((const int*)eb)[LSB_B2];
    if (b != b1 && b != b2) continue;
    const V3 n = ld3(eb + LSB_N), t1 = ld3(ea + LCE_T1), t2 = cross(n, t1), cp = ld3(ea + LCE_CP);
    const V3 ac = a.l + cross(a.a, cp);
#pragma unroll
    for (int k = 0; k < 4; k++) eb[(b == b2 ? LSB_P2 : LSB_P1) + k] = dot(l_pyr_dir(H, n, t1, t2, k), ac);
  }
}
// rows li + 8 q of the env's geom-geom rows (row = 4 * contact + k): rs = part2 - part1 - aref into entry A; rs[q] (0 without a row)
template <class C>
__device__ __forceinline__ void l_self_fix(float* sm, const LLane& w, bool on, float* rs) {
#pragma unroll
  for (int q = 0; q < L_SELFQ; q++) {
    rs[q] = 0.f;
    if (on) {
      const int ns = ((const int*)sm)[C::misc + LMI_NSELF], r = w.li + LM_LPE * q, s = r >> 2, k = r & 3;
      if (s < ns) {
        const int c0 = ((const int*)sm)[C::misc + LMI_SELF0] + 2 * s;
        float* ea = l_centry<C>(sm, w, c0); const float* eb = l_centry<C>(sm, w, c0 + 1);
        rs[q] = eb[LSB_P2 + k] - eb[LSB_P1 + k] - ea[LCE_AREF + k];
        ea[LCE_RS + k] = rs[q];
      }
    }
  }
}

// geom-geom narrow phase on the poses / velocities the outward sweep left in the body scratch: capsule / sphere pairs that pass
// MuJoCo's filters (LPair list), one contact at the closest points, normal from geom1 to geom2, position midway in the overlap,
// default tangent (mju_makeFrame); impedance / R / aref as for the floor rows with tran = invweight0(b1) + invweight0(b2).
// Returns the number of contacts of this lane's env; *dropped: more than L_MAXSELF touched.
template <class C>
__device__ __noinline__ int l_self_collide(const float* ms, float* sm, const LLane& w, int* dropped) {
  const LHdr& H = l_hdr<C>(ms);
  const LBody* MB = l_bodies(ms);
  const LGeom* MG = l_geoms(ms);
  const LPair* PR = (const LPair*)((const char*)ms + H.pair_off);
  const int ncon = ((const int*)sm)[C::misc + LMI_NCON];
  int nself = 0;
  for (int base = 0; base < H.npair; base += LM_LPE) {
    const int i = base + w.li;
    bool hit = false;
    V3 n = v3(1.f, 0.f, 0.f), pos = n; float dist = 0.f; int g1 = 0, g2 = 0;
    if (w.live && i < H.npair) {
      g1 = PR[i].g1; g2 = PR[i].g2;
      const LGeom& G1 = MG[g1]; const LGeom& G2 = MG[g2];
      const V3 x1 = ld3(sm + C::body + C::BODYW * G1.body + LBR_X), x2 = ld3(sm + C::body + C::BODYW * G2.body + LBR_X);
      const float r1 = G1.size[0], r2 = G2.size[0];
      const float h1 = (G1.type == SMPLSIM_GEOM_CAPSULE) ? G1.size[1] : 0.f, h2 = (G2.type == SMPLSIM_GEOM_CAPSULE) ? G2.size[1] : 0.f;
      const V3 dx = x2 - x1;
      const float reach = h1 + h2 + r1 + r2 + H.margin + sqrtf(dot(ld3(G1.pos), ld3(G1.pos))) + sqrtf(dot(ld3(G2.pos), ld3(G2.pos)));
      if (dot(dx, dx) <= reach * reach) {      // body origins close enough: read the orientations
        const float* q1 = w.gbody + 10 * G1.body; const float* q2 = w.gbody + 10 * G2.body;
        Q4 a; a.w = q1[0]; a.x = q1[1]; a.y = q1[2]; a.z = q1[3];
        Q4 b; b.w = q2[0]; b.x = q2[1]; b.y = q2[2]; b.z = q2[3];
        const V3 c1 = x1 + qrot(a, ld3(G1.pos)), c2 = x2 + qrot(b, ld3(G2.pos));
        const V3 dc = c2 - c1;
        const float rc = h1 + h2 + r1 + r2 + H.margin;
        if (dot(dc, dc) <= rc * rc) {
          const V3 a1 = qrot(a, v3(G1.mat[2], G1.mat[5], G1.mat[8])), a2 = qrot(b, v3(G2.mat[2], G2.mat[5], G2.mat[8]));
          float sp, tp;
          l_segment_segment(c1, a1, h1, c2, a2, h2, &sp, &tp);
          const V3 p1 = c1 + sp * a1, p2 = c2 + tp * a2;
          V3 d = p2 - p1;
          const float len = sqrtf(dot(d, d));
          dist = len - r1 - r2;
          if (dist <= H.margin) {
            hit = true;
            n = (len < 1e-15f) ? v3(1.f, 0.f, 0.f) : (1.0f / len) * d;
            pos = p1 + (r1 + 0.5f * dist) * n;
          }
        }
      }
    }
    const unsigned bal = (__ballot_sync(L_FULL, hit) & w.gmask) >> w.gbase;
    const int idx = nself + __popc(bal & ((1u << w.li) - 1u));
    if (hit && idx < L_MAXSELF) {
      const int c0 = ncon + 2 * idx;
      float* ea = l_centry<C>(sm, w, c0); float* eb = l_centry<C>(sm, w, c0 + 1);
      const int b1 = MG[g1].body, b2 = MG[g2].body;
      V3 t1 = (n.y < 0.5f && n.y > -0.5f) ? v3(0.f, 1.f, 0.f) : v3(0.f, 0.f, 1.f);   // mju_makeFrame without a hint
      t1 = t1 - dot(n, t1) * n;
      { float nn = sqrtf(dot(t1, t1)); t1 = (nn < 1e-15f) ? v3(1.f, 0.f, 0.f) : (1.0f / nn) * t1; }
      const V3 t2 = cross(n, t1);
      const float pm = dist - H.margin, imp = l_impedance(H, pm);
      const float tran = MB[b1].tiw0 + MB[b2].tiw0;
      const float R0 = fmaxf((1.f - imp) / imp * (tran + H.mu * H.mu * tran), 1e-15f);
      const float R1 = R0 / fmaxf(H.impratio, 1e-15f), mu = H.mu * sqrtf(R1 / R0);
      const S6 v1 = ld6(w.gbody + 10 * b1 + 4), v2 = ld6(w.gbody + 10 * b2 + 4);
      const V3 vc = (v2.l + cross(v2.a, pos)) - (v1.l + cross(v1.a, pos));
      ((int*)ea)[LCE_INFO] = 1 | 30 | 32 | LCE_SELF | (g2 << 8);
      st3(ea + LCE_CP, pos); st3(ea + LCE_T1, t1);
      ea[LCE_D] = 1.0f / (2.f * mu * mu * R0);
#pragma unroll
      for (int k = 0; k < 4; k++) {
        ea[LCE_AREF + k] = -H.B * dot(l_pyr_dir(H, n, t1, t2, k), vc) - H.K * imp * pm;
        ea[LCE_PHI + k] = 0.f; ea[LCE_R + k] = 0.f; ea[LCE_RS + k] = 0.f;
        eb[LSB_LAM + k] = 0.f; eb[LSB_P1 + k] = 0.f; eb[LSB_P2 + k] = 0.f; eb[LSB_R0 + k] = 0.f;
      }
      ((int*)eb)[LCE_INFO] = 0;
      st3(eb + LSB_N, n);
      ((int*)eb)[LSB_B1] = b1; ((int*)eb)[LSB_B2] = b2;
    }
    nself += __popc(bal);
  }
  *dropped = nself > L_MAXSELF;
  nself = min(nself, L_MAXSELF);
  __syncwarp();
  if (w.live && w.li == 0) {
    ((int*)sm)[C::misc + LMI_NSELF] = nself; ((int*)sm)[C::misc + LMI_SELF0] = ncon;
    ((int*)sm)[C::misc + LMI_NCON] = ncon + 2 * nself;
  }
  __syncwarp();
  return nself;
}

// root body of the inward sweep (every lane makes the call): children arrive through the in-mailboxes; lane 0 of the group assembles the
// root's articulated inertia and bias force (after the semi-implicit Euler of the free joint in S4), the lanes of the group solve the
// 6 x 6 system of its six dofs; the root's spatial acceleration stays in shared memory (LRT_A) for the outward sweeps.  Returns "the root
// has constraint rows in its subtree" (lane 0).
template <class C, bool SPD>
__device__ __noinline__ bool l_root_in(const float* ms, float* sm, const LLane& w, bool need, int flags) {
  const LHdr& H = l_hdr<C>(ms);
  const LBody& lb = l_bodies(ms)[0];
  S6 p = l_rec_ld_pb<C>(sm, 0);
  bool dirty = false;
  float* rt = sm + C::root;
  if (need && w.li == 0) {
    float* br = sm + C::body;
    float A[21], r10[10];
    const int ci = l_ld_r10(br, r10);
    rb_expand(r10, A);
    for (int j = 0; j < lb.nmb; j++) dirty = l_mbi_add(sm + C::mbi + C::MBIW * lb.mb[j], A, p) || dirty;
    if (!SPD) {
      const int cn = (ci >> 8) & 255;
      dirty = dirty || cn > 0;
      l_fold_contacts<C>(H, sm, w, ci & 255, cn, A, p);
      if (C::SELFCOL && ((const int*)sm)[C::misc + LMI_NSELF]) { l_self_wrench<C>(H, sm, w, 0, p); dirty = dirty || l_self_touches<C>(sm, w, 0); }
    }
    if (SPD && (flags & LI_INTEGRATE)) {
      float* qpos = sm + C::qpos; float* qvel = sm + C::qvel; const float* qacc = sm + C::qacc;
      float* misc = sm + C::misc;
      float h = H.h;
#pragma unroll
      for (int d = 0; d < 6; d++) {
        float v = fmaf(h, qacc[d], qvel[d]);
        qvel[d] = v;
        if (d < 3) { float dd = h * v; qpos[d] += dd; if (d < 2) misc[LMI_DISP + d] += dd; }
      }
      V3 wv = ld3(qvel + 3);
      float n = sqrtf(dot(wv, wv)), ang = n * h;
      Q4 q; q.w = qpos[3]; q.x = qpos[4]; q.y = qpos[5]; q.z = qpos[6];
      if (ang > 0.f) {
        float sn, cs;
        l_sincos(0.5f * ang, &sn, &cs);
        float s = sn / n;
        Q4 dq; dq.w = cs; dq.x = wv.x * s; dq.y = wv.y * s; dq.z = wv.z * s;
        q = qmul(q, dq);
      }
      q = qnormalize(q);
      qpos[3] = q.w; qpos[4] = q.x; qpos[5] = q.y; qpos[6] = q.z;
    }
    // free joint: S = [0 R ; I 0] is orthonormal, so eliminating its six dofs = solving (A + S diag(armature) S^T) a = -p for the
    // root's spatial acceleration; the joint accelerations are S^T a (l_root_acc).  System -> shared memory, solved by the lanes below.
    {
      const float ar = H.rarm[3], as = H.rarm[4], at = H.rarm[5];
      A[sidx(3, 3)] += H.rarm[0]; A[sidx(4, 4)] += H.rarm[1]; A[sidx(5, 5)] += H.rarm[2];
      if (ar != 0.f || as != 0.f || at != 0.f) {
        const V3 c0 = ld3(br + LBR_AX), c1 = ld3(br + LBR_AX + 3), c2 = ld3(br + LBR_AX + 6);
        A[sidx(0, 0)] += ar * c0.x * c0.x + as * c1.x * c1.x + at * c2.x * c2.x; A[sidx(0, 1)] += ar * c0.x * c0.y + as * c1.x * c1.y + at * c2.x * c2.y;
        A[sidx(0, 2)] += ar * c0.x * c0.z + as * c1.x * c1.z + at * c2.x * c2.z; A[sidx(1, 1)] += ar * c0.y * c0.y + as * c1.y * c1.y + at * c2.y * c2.y;
        A[sidx(1, 2)] += ar * c0.y * c0.z + as * c1.y * c1.z + at * c2.y * c2.z; A[sidx(2, 2)] += ar * c0.z * c0.z + as * c1.z * c1.z + at * c2.z * c2.z;
      }
      float4* r4 = (float4*)rt;
      r4[0] = make_float4(A[0], A[1], A[2], A[3]); r4[1] = make_float4(A[4], A[5], A[6], A[7]); r4[2] = make_float4(A[8], A[9], A[10], A[11]);
      r4[3] = make_float4(A[12], A[13], A[14], A[15]); r4[4] = make_float4(A[16], A[17], A[18], A[19]);
      r4[5] = make_float4(A[20], p.a.x, p.a.y, p.a.z); r4[6] = make_float4(p.l.x, p.l.y, p.l.z, 0.f);
    }
  }
  __syncwarp();
  {
    // Gauss-Jordan across the lanes of the env (symmetric positive definite: no pivoting): lane j < 6 holds column j, lane 6 the
    // right-hand side -p; after the six pivots lane 6 holds the root's spatial acceleration.  Every lane runs it (warp collectives).
    const bool need_env = __shfl_sync(L_FULL, need ? 1 : 0, w.gbase) != 0;
    const int j = w.li;
    float col[6];
#pragma unroll
    for (int i = 0; i < 6; i++) {
      const int lo = i < j ? i : j, hi = i < j ? j : i;                 // sidx(i, j) with a run-time column
      const int ix = (j < 6) ? (lo * (13 - lo)) / 2 + (hi - lo) : 21 + i;
      const float v = (need_env && j < 7) ? rt[ix] : (i == j ? 1.f : 0.f);
      col[i] = (j == 6) ? -v : v;
    }
#pragma unroll
    for (int k = 0; k < 6; k++) {
      float m[6];
#pragma unroll
      for (int i = 0; i < 6; i++) m[i] = __shfl_sync(L_FULL, col[i], w.gbase + k);   // column k (lives in lane k); m[k] = the pivot
      const float r = col[k] * l_rcp(m[k]);
#pragma unroll
      for (int i = 0; i < 6; i++) if (i != k) col[i] = fmaf(-m[i], r, col[i]);
      col[k] = r;
    }
    if (need_env && j == 6) {
#pragma unroll
      for (int i = 0; i < 6; i++) rt[LRT_A + i] = col[i];
    }
  }
  __syncwarp();
  return dirty;
}

// SPD (compile time): the stable-PD system (LI_SPD, optionally LI_INTEGRATE; never a re-sweep) -- the two uses share no flag-dependent code,
// so each instance carries only its own
template <class C, bool SPD>
__device__ __noinline__ void l_sweep_in(const float* ms, float* sm, const LLane& w, bool run, int flags, LSolveLane& st_) {
  const LHdr& H = l_hdr<C>(ms);
  const LBody* MB = l_bodies(ms);
  LSolveLane st = st_;
  const int li = w.li;
  const float hh = H.h;
  float cA[21];
#pragma unroll
  for (int j = 0; j < 21; j++) cA[j] = 0.f;
  S6 cp = s6(v3(0.f, 0.f, 0.f), v3(0.f, 0.f, 0.f));
  bool cdirty = false;
  constexpr bool spd = SPD;
  const bool resweep = !SPD && (flags & LI_RESWEEP) != 0;
  if (!resweep && !spd) st.dirty_bits = 0u;
  const bool stepbar = (H.align & 16) && w.bar;
  for (int t = H.T - 1; t >= 1; t--) {
    if (stepbar) __syncthreads();
    const int b = H.sched[t][li];
    const bool actv = run && b >= 0;
    const bool need = actv && (!resweep || ((st.rc_bits >> t) & 1u));
    if (resweep && !__any_sync(L_FULL, need)) continue;
    S6 p = l_rec_ld_pb<C>(sm, b);
    float K[18], kc[3];   // written by the lanes that need the body; the others leave the record as it is
    if (need) {
      const LBody& lb = MB[b];
      float* br = sm + C::body + C::BODYW * b;
      float A[21], r10[10];
      const int ci = l_ld_r10(br, r10);
      rb_expand(r10, A);
      bool dirty = false;
      if (lb.flags & LB_CARRY_IN) {
#pragma unroll
        for (int j = 0; j < 21; j++) A[j] += cA[j];
        p = p + cp; dirty = cdirty;
      }
      for (int j = 0; j < lb.nmb; j++) dirty = l_mbi_add(sm + C::mbi + C::MBIW * lb.mb[j], A, p) || dirty;
      float lD[3] = {0.f, 0.f, 0.f}, lT[3] = {0.f, 0.f, 0.f};
      if (!spd) {
        const int cb = ci & 255, cn = (ci >> 8) & 255, lbs = (ci >> 16) & 255, ln = (ci >> 24) & 255;
        dirty = dirty || cn > 0 || ln > 0;
        l_fold_contacts<C>(H, sm, w, cb, cn, A, p);
        if (C::SELFCOL && ((const int*)sm)[C::misc + LMI_NSELF]) { l_self_wrench<C>(H, sm, w, b, p); dirty = dirty || l_self_touches<C>(sm, w, b); }
        for (int e = lbs; e < lbs + ln; e++) {   // joint-limit rows of this body that sit in the working set
          const float4* l4 = (const float4*)(sm + C::lim + C::LIMW * e);
          float4 u = l4[0], v = l4[1];
          if (!(__float_as_int(v.y) & 1)) continue;
          int k = __float_as_int(u.x) - lb.dofadr;
#pragma unroll
          for (int kk = 0; kk < 3; kk++) if (kk == k) { lD[kk] = u.z; lT[kk] = u.y * u.z * u.w; }
        }
      }
      // ---------------- hinge body: three dofs, last joint first
      const int d0 = lb.dofadr;
      const LAxes AX = l_ld_axes(br);
#pragma unroll
      for (int k = 2; k >= 0; k--) {
        const int d = d0 + k, i = d - 6;
        V3 ax = l_axis(AX, k);
        S6 S = s6(ax, cross(AX.x, ax));
        float s[6], Uv[6];
        l_s6arr(S, s);
        sym_mul(A, s, Uv);
        float D = lb.arm[k] + (spd ? hh * lb.kd[k] : lD[k]);
#pragma unroll
        for (int j = 0; j < 6; j++) D = fmaf(s[j], Uv[j], D);
        float di = l_rcp(D), tin;
        if (spd) {
          float q = sm[C::qpos + d + 1], qd = sm[C::qvel + d];
          if (flags & LI_INTEGRATE) {
            qd = fmaf(hh, sm[C::qacc + d], qd); q = fmaf(hh, qd, q);
            sm[C::qvel + d] = qd; sm[C::qpos + d + 1] = q;
          }
          float tgt = fmaf(sm[C::act + i], lb.ascale[k], lb.aoffset[k]);
          tin = -lb.kp[k] * (q + qd * hh - tgt) - lb.kd[k] * qd;
        } else tin = sm[C::tau + i] + lT[k];
        float uu = tin - dot6(S, p);
        sym_rank1(A, Uv, di);
        p = p + (uu * di) * l_arr6(Uv);
#pragma unroll
        for (int j = 0; j < 6; j++) K[6 * k + j] = Uv[j] * di;
        kc[k] = uu * di;
      }
#pragma unroll
      for (int j = 0; j < 21; j++) cA[j] = A[j];
      cp = p; cdirty = dirty;
      if (lb.in_mbox >= 0) l_mbi_put(sm + C::mbi + C::MBIW * lb.in_mbox, A, p, dirty);
      if (!spd && !resweep && dirty) st.dirty_bits |= 1u << t;
    }
    l_rec_st_Kc<C>(sm, b, K, kc, need);
    __syncwarp();
  }
  {   // the root body closes the sweep
    if (stepbar) __syncthreads();
    const bool need0 = run && (!resweep || (st.rc_bits & 1u));
    bool d0 = false;
    if (!resweep || __any_sync(L_FULL, need0)) d0 = l_root_in<C, SPD>(ms, sm, w, need0, flags);
    if (!spd && !resweep && d0 && li == 0) st.dirty_bits |= 1u;
  }
  st_ = st;
}

// root body of the acceleration sweep: the spatial acceleration solved at the end of the inward sweep (l_root_in) -> the six
// free-joint accelerations S^T a, the root's out-mailbox, residuals of the root's contact rows
template <class C>
__device__ __noinline__ void l_root_acc(const float* ms, float* sm, const LLane& w, bool run, float* qout, bool* same) {
  const LHdr& H = l_hdr<C>(ms);
  const LBody& lb = l_bodies(ms)[0];
  if (run && w.li == 0) {
    const float* br = sm + C::body;
    const V3 c0 = ld3(br + LBR_AX), c1 = ld3(br + LBR_AX + 3), c2 = ld3(br + LBR_AX + 6);   // rotation columns = axes of the three rotational dofs
    const S6 a = ld6(sm + C::root + LRT_A);
    st3(qout, a.l);
    qout[3] = dot(c0, a.a); qout[4] = dot(c1, a.a); qout[5] = dot(c2, a.a);
    l_mbo_put_acc(sm + C::mbo + C::MBOW * lb.out_mbox, a);
    const int ci = ((const int*)br)[LBR_CI];
    *same = l_rows_eval<C>(H, sm, w, ci & 255, (ci >> 8) & 255, a) && *same;
    if (C::SELFCOL && ((const int*)sm)[C::misc + LMI_NSELF]) l_self_part<C>(H, sm, w, 0, a);
  }
  __syncwarp();
}

// ------------------------------------------------------------------ S3: outward sweep of the accelerations + residuals of the constraint rows
// qdd -> qacc (no iterate yet) or qstar (trial point of the line search); rs = J a - aref of every row; returns "the sign pattern
// of the rows equals the working set" for this lane's env.
template <class C>
__device__ __noinline__ bool l_sweep_acc(const float* ms, float* sm, const LLane& w, bool run, bool to_qstar) {
  const LHdr& H = l_hdr<C>(ms);
  const LBody* MB = l_bodies(ms);
  S6 ca = s6(v3(0.f, 0.f, 0.f), v3(0.f, 0.f, 0.f));
  bool same = true;
  float* qout = sm + (to_qstar ? C::qstar : C::qacc);
  const bool stepbar = (H.align & 16) && w.bar;
  const int li = w.li, T = H.T;
  if (stepbar) __syncthreads();
  l_root_acc<C>(ms, sm, w, run, qout, &same);
  for (int t = 1; t < T; t++) {
    if (stepbar) __syncthreads();
    const int b = H.sched[t][li];
    const bool actv = run && b >= 0;
    float K[18], kc[3];
    l_rec_ld_Kc<C>(sm, b, K, kc);
    if (actv) {
      const LBody& lb = MB[b];
      const float* br = sm + C::body + C::BODYW * b;
      if (!(lb.flags & LB_CARRY_OUT)) ca = l_mbo_get_acc(sm + C::mbo + C::MBOW * lb.pmbox);
      S6 a = ca;
      float qdd3[3];
      const LAxes AX = l_ld_axes(br);
#pragma unroll
      for (int k = 0; k < 3; k++) {
        V3 ax = l_axis(AX, k);
        S6 S = s6(ax, cross(AX.x, ax));
        float qdd = kc[k] - dot6(l_arr6(K + 6 * k), a);
        qdd3[k] = qdd;
        a = a + qdd * S;
      }
      qout[lb.dofadr] = qdd3[0]; qout[lb.dofadr + 1] = qdd3[1]; qout[lb.dofadr + 2] = qdd3[2];
      ca = a;
      if (lb.out_mbox >= 0) l_mbo_put_acc(sm + C::mbo + C::MBOW * lb.out_mbox, a);
      const int ci = ((const int*)br)[LBR_CI], cb = ci & 255, cn = (ci >> 8) & 255, lbs = (ci >> 16) & 255, ln = (ci >> 24) & 255;
      if (cn) same = l_rows_eval<C>(H, sm, w, cb, cn, a) && same;
      if (C::SELFCOL && ((const int*)sm)[C::misc + LMI_NSELF]) l_self_part<C>(H, sm, w, b, a);
      for (int e = lbs; e < lbs + ln; e++) {
        float* le = sm + C::lim + C::LIMW * e;
        int k = ((const int*)le)[LLE_DOF] - lb.dofadr;
        float qd = (k == 0) ? qdd3[0] : (k == 1) ? qdd3[1] : qdd3[2];
        float rs = le[LLE_SG] * qd - le[LLE_AREF];
        le[LLE_RS] = rs;
        if ((rs < 0.f ? 1 : 0) != (((const int*)le)[LLE_FLAG] & 1)) same = false;
      }
    }
    __syncwarp();
  }
  return l_gall(same || !run, w);
}

// after the first inward sweep of a substep (dirty_bits set): rc_bits = what the re-sweeps recompute: the dirty bodies and the bodies
// that hand their result to one in registers (LHdr::carry_mask)
template <class C>
__device__ __forceinline__ void l_solve_plan(const float* ms, const LLane& w, LSolveLane& st) {
  const LHdr& H = l_hdr<C>(ms);
  const unsigned cm = H.carry_mask[w.li];
  unsigned rc = st.dirty_bits;
  for (int t = 1; t < H.T; t++) if (((cm >> t) & 1u) && ((rc >> (t - 1)) & 1u)) rc |= 1u << t;
  st.rc_bits = rc;
}

// ------------------------------------------------------------------ row-space passes of the exact line search (lane-parallel over the row lists)
// r = J a - aref at the iterate, rs at the trial point, d = rs - r; phi: force of the row at the iterate.
// op 0: adopt  (phi := -D rs on the working set ; set := rs < 0 ; r := rs)
// op 1: sums   (g1 += d phi ; g2 += d (phis - phi) ; s1, s2 at step al)
// op 2: apply  (phi += al (phis - phi) ; r += al d ; set := (r < 0))
// op 3: take   (set unchanged at the trial point: r := rs, phi := -D rs on the set)        [fin with an iterate: bookkeeping only]
// op 4: sums at al = 0 and at al = 1 in one pass: out = g1, g2, s1(0), s1(1), s2(1)   (start of the line search)
template <class C>
__device__ __noinline__ void l_rows(float* sm, const LLane& w, bool run, int op, float al, float* out4) {
  float g1 = 0.f, g2 = 0.f, s1 = 0.f, s2 = 0.f, s10 = 0.f;
  if (op == 4) al = 1.f;
  if (run) {
    const int ncon = ((const int*)sm)[C::misc + LMI_NCON], nlim = ((const int*)sm)[C::misc + LMI_NLIM];
    for (int c = w.li; c < ncon; c += LM_LPE) {
      float* ce = l_centry<C>(sm, w, c);
      int info = ((int*)ce)[LCE_INFO];
      if (!(info & 1)) continue;
      float D = ce[LCE_D];
      int nf = 0;
#pragma unroll
      for (int k = 0; k < 4; k++) {
        float rs = ce[LCE_RS + k], phs = (info & (2 << k)) ? -D * rs : 0.f;
        if (op == 0) { ce[LCE_PHI + k] = phs; ce[LCE_R + k] = rs; if (rs < 0.f) nf |= 2 << k; }
        else {
          float r = ce[LCE_R + k], d = rs - r, ph = ce[LCE_PHI + k], v = fmaf(al, d, r);
          if (op == 1 || op == 4) {
            g1 = fmaf(d, ph, g1); g2 = fmaf(d, phs - ph, g2);
            if (v < 0.f) { s1 = fmaf(D * v, d, s1); s2 = fmaf(D * d, d, s2); }
            if (op == 4 && r < 0.f) s10 = fmaf(D * r, d, s10);
          } else { ce[LCE_PHI + k] = fmaf(al, phs - ph, ph); ce[LCE_R + k] = v; if (v < 0.f) nf |= 2 << k; }
        }
      }
      if (op != 1 && op != 4) ((int*)ce)[LCE_INFO] = (info & ~30) | nf;
    }
    for (int e = w.li; e < nlim; e += LM_LPE) {
      float* le = sm + C::lim + C::LIMW * e;
      int fl = ((int*)le)[LLE_FLAG];
      float D = le[LLE_D], rs = le[LLE_RS], phs = (fl & 1) ? -D * rs : 0.f;
      if (op == 0) { le[LLE_PHI] = phs; le[LLE_R] = rs; ((int*)le)[LLE_FLAG] = rs < 0.f ? 1 : 0; }
      else {
        float r = le[LLE_R], d = rs - r, ph = le[LLE_PHI], v = fmaf(al, d, r);
        if (op == 1 || op == 4) {
          g1 = fmaf(d, ph, g1); g2 = fmaf(d, phs - ph, g2);
          if (v < 0.f) { s1 = fmaf(D * v, d, s1); s2 = fmaf(D * d, d, s2); }
          if (op == 4 && r < 0.f) s10 = fmaf(D * r, d, s10);
        } else { le[LLE_PHI] = fmaf(al, phs - ph, ph); le[LLE_R] = v; ((int*)le)[LLE_FLAG] = v < 0.f ? 1 : 0; }
      }
    }
  }
  out4[0] = g1; out4[1] = g2; out4[2] = s1; out4[3] = s2; out4[4] = s10;
}

#ifdef SMPLSIM_STATS
// debug build (tools/solver_stats.py): why does the first solve of a substep miss?  counters: [0] env-substeps, [1] with rows,
// [2] first pass ok, [3..8] histogram of extra solves 1..6+, [9] rows predicted active but rs >= 0, [10] rows predicted inactive
// but rs < 0, [11] ... of which in a contact new this substep, [12] limit rows flipped, [13] contacts, [14] new contacts
__device__ int g_lstats[32];
#define L_STAT(i, v) atomicAdd(&g_lstats[i], v)
#else
#define L_STAT(i, v) do { } while (0)
#endif

// ------------------------------------------------------------------ one Newton system of the active-set solve
// = ABA factors + accelerations for the current working set.  Envs with geom-geom rows (two-body rows cannot be folded into the
// articulated inertias) get them by Woodbury on top of those factors: with lam the multipliers of the active two-body rows,
// a(lam) = a(0) + M~^-1 Y lam is affine, so one probe solve per active row gives H = Y^T M~^-1 Y column by column (rows of H live in
// the lanes: lane i of the env owns row i), (H + D^-1) lam = -r(0) is solved across the 8 lanes, and a last solve applies lam.
// Returns "sign pattern of all rows == working set" at the resulting point.
template <class C>
__device__ __noinline__ bool l_linsolve(const float* ms, float* sm, const LLane& w, bool run, int inflags, bool to_qstar, bool first, LSolveLane& st) {
  const LHdr& H = l_hdr<C>(ms);
  if (!C::SELFCOL) {   // no geom-geom rows compiled in: the plain ABA pair
    l_sweep_in<C, false>(ms, sm, w, run, inflags, st);
    if (first) l_solve_plan<C>(ms, w, st);
    return l_sweep_acc<C>(ms, sm, w, run, to_qstar);
  }
  const bool hs = run && H.cfg.self_collision && ((const int*)sm)[C::misc + LMI_NSELF] > 0;
  const bool anyhs = __any_sync(L_FULL, hs);
  constexpr int NR = 4 * L_MAXSELF;                 // two-body rows per env; lane li owns rows li + 8 q
  bool valid[L_SELFQ]; float* ea[L_SELFQ]; float* eb[L_SELFQ]; int krow[L_SELFQ];
#pragma unroll
  for (int q = 0; q < L_SELFQ; q++) {
    const int r = w.li + LM_LPE * q;
    krow[q] = r & 3;
    valid[q] = hs && (r >> 2) < ((const int*)sm)[C::misc + LMI_NSELF];
    ea[q] = sm; eb[q] = sm;
    if (valid[q]) {
      const int c0 = ((const int*)sm)[C::misc + LMI_SELF0] + 2 * (r >> 2);
      ea[q] = l_centry<C>(sm, w, c0); eb[q] = l_centry<C>(sm, w, c0 + 1);
      eb[q][LSB_LAM + krow[q]] = 0.f;
    }
  }
  if (anyhs) __syncwarp();
  l_sweep_in<C, false>(ms, sm, w, run, inflags, st);
  if (first) l_solve_plan<C>(ms, w, st);
  bool same = l_sweep_acc<C>(ms, sm, w, run, to_qstar);
  if (!anyhs) return same;
  const int rflags = H.dirtypath ? LI_RESWEEP : 0;
  float r0[L_SELFQ], Dr[L_SELFQ], pscale[L_SELFQ];
  bool act[L_SELFQ];
  l_self_fix<C>(sm, w, hs, r0);
  float Hrow[L_SELFQ][NR];
#pragma unroll
  for (int q = 0; q < L_SELFQ; q++) {
    act[q] = valid[q] && ((((const int*)ea[q])[LCE_INFO] >> (1 + krow[q])) & 1);
    Dr[q] = valid[q] ? ea[q][LCE_D] : 1.f;
    pscale[q] = fmaxf(fabsf(r0[q]) * Dr[q], 1.0f);      // probe magnitude ~ the multiplier the row would carry alone
#pragma unroll
    for (int j = 0; j < NR; j++) Hrow[q][j] = 0.f;
  }
  __syncwarp();
#pragma unroll
  for (int qj = 0; qj < L_SELFQ; qj++) {
#pragma unroll 1
    for (int lj = 0; lj < LM_LPE; lj++) {
      const int j = lj + LM_LPE * qj;                                        // probed row: owned by lane lj, slot qj
      const int actj_ = __shfl_sync(L_FULL, act[qj] ? 1 : 0, w.gbase + lj);  // (collectives never behind a short-circuit)
      const float Pj = __shfl_sync(L_FULL, pscale[qj], w.gbase + lj);
      const bool prb = hs && actj_ != 0;
      if (!__any_sync(L_FULL, prb)) continue;
      if (prb && w.li == lj) eb[qj][LSB_LAM + krow[qj]] = Pj;
      __syncwarp();
      l_sweep_in<C, false>(ms, sm, w, prb, rflags, st);
      l_sweep_acc<C>(ms, sm, w, prb, to_qstar);
      float v[L_SELFQ];
      l_self_fix<C>(sm, w, prb, v);
#pragma unroll
      for (int q = 0; q < L_SELFQ; q++) {
        if (prb && valid[q]) {
          const float hij = (v[q] - r0[q]) / Pj;
#pragma unroll
          for (int jj = 0; jj < NR; jj++) if (jj == j) Hrow[q][jj] = hij;
        }
      }
      if (prb && w.li == lj) eb[qj][LSB_LAM + krow[qj]] = 0.f;
      __syncwarp();
    }
  }
  // (H + D^-1) lam = -r0 on the active rows (identity elsewhere): Gauss-Jordan across the lanes of the env, L_SELFQ rows per lane
  float Mr[L_SELFQ][NR], rhs[L_SELFQ];
#pragma unroll
  for (int qj = 0; qj < L_SELFQ; qj++)
#pragma unroll
    for (int lj = 0; lj < LM_LPE; lj++) {
      const int j = lj + LM_LPE * qj;
      const bool actj = __shfl_sync(L_FULL, act[qj] ? 1 : 0, w.gbase + lj) != 0;
#pragma unroll
      for (int q = 0; q < L_SELFQ; q++) {
        Mr[q][j] = (act[q] && actj) ? Hrow[q][j] : 0.f;
        if (q == qj && lj == w.li) Mr[q][j] = act[q] ? Mr[q][j] + 1.0f / Dr[q] : 1.0f;
      }
    }
#pragma unroll
  for (int q = 0; q < L_SELFQ; q++) rhs[q] = act[q] ? -r0[q] : 0.f;
#pragma unroll
  for (int qp = 0; qp < L_SELFQ; qp++)
#pragma unroll 1
    for (int lp = 0; lp < LM_LPE; lp++) {
      const int pp = lp + LM_LPE * qp;          // pivot row: lane lp, slot qp
      float prow[NR];
#pragma unroll
      for (int c = 0; c < NR; c++) prow[c] = __shfl_sync(L_FULL, Mr[qp][c], w.gbase + lp);
      const float prhs = __shfl_sync(L_FULL, rhs[qp], w.gbase + lp);
      float piv = 1.f;
#pragma unroll
      for (int c = 0; c < NR; c++) if (c == pp) piv = prow[c];
#pragma unroll
      for (int q = 0; q < L_SELFQ; q++) {
        float mp = 0.f;
#pragma unroll
        for (int c = 0; c < NR; c++) if (c == pp) mp = Mr[q][c];
        const float f = (w.li == lp && q == qp) ? 0.f : mp / piv;
#pragma unroll
        for (int c = 0; c < NR; c++) Mr[q][c] = fmaf(-f, prow[c], Mr[q][c]);
        rhs[q] = fmaf(-f, prhs, rhs[q]);
      }
    }
#pragma unroll
  for (int q = 0; q < L_SELFQ; q++) {
    float d = 1.f;
#pragma unroll
    for (int c = 0; c < NR; c++) if (c == w.li + LM_LPE * q) d = Mr[q][c];
    if (valid[q]) eb[q][LSB_LAM + krow[q]] = act[q] ? rhs[q] / d : 0.f;
  }
  __syncwarp();
  l_sweep_in<C, false>(ms, sm, w, hs, rflags, st);
  const bool same2 = l_sweep_acc<C>(ms, sm, w, hs, to_qstar);
  float rsf[L_SELFQ];
  l_self_fix<C>(sm, w, hs, rsf);
  bool okrow = true;
#pragma unroll
  for (int q = 0; q < L_SELFQ; q++) okrow = okrow && (!valid[q] || ((rsf[q] < 0.f) == act[q]));
  const bool sameself = l_gall(okrow, w);
  __syncwarp();
  return hs ? (same2 && sameself) : same;
}

// ------------------------------------------------------------------ constraint solve: active-set Newton, every system one ABA pass (DESIGN.md 2)
// Returns the number of extra solves; *hit_max: stopped at L_SOLVER_MAXITER.
template <class C>
__device__ __noinline__ int l_solve(const float* ms, float* sm, const LLane& w, bool any_rows, LSolveLane& st, bool* hit_max) {
  const LHdr& H = l_hdr<C>(ms);
  // first pass for every live env: the working set inherited from the previous substep is already in the row lists
  bool same0 = l_linsolve<C>(ms, sm, w, w.live, 0, false, true, st);   // qdd -> qacc
  bool run = w.live && any_rows && !same0;
  *hit_max = false;
#ifdef SMPLSIM_STATS
  if (w.live && w.li == 0) {
    L_STAT(0, 1);
    if (any_rows) L_STAT(1, 1);
    if (any_rows && same0) L_STAT(2, 1);
    const int ncon = ((const int*)sm)[C::misc + LMI_NCON], nlim = ((const int*)sm)[C::misc + LMI_NLIM];
    for (int c = 0; c < ncon; c++) {
      const float* ce = l_centry<C>(sm, w, c);
      int info = ((const int*)ce)[LCE_INFO];
      if (!(info & 1)) continue;
      L_STAT(13, 1);
      bool isnew = ((info >> 5) & 1) != 0;
      if (isnew) L_STAT(14, 1);
      for (int k = 0; k < 4; k++) {
        bool act = (info & (2 << k)) != 0, neg = ce[LCE_RS + k] < 0.f;
        if (act && !neg) L_STAT(9, 1);
        if (!act && neg) L_STAT(10, 1);
        if (act != neg && isnew) L_STAT(11, 1);
      }
    }
    for (int e = 0; e < nlim; e++) {
      const float* le = sm + C::lim + C::LIMW * e;
      if ((le[LLE_RS] < 0.f ? 1 : 0) != (((const int*)le)[LLE_FLAG] & 1)) L_STAT(12, 1);
    }
    // [22..25]: first-pass misses whose every flipped row carries a force change |D rs| below 1e-3 / 1e-2 / 1e-1 / 1 N
    if (any_rows && !same0) {
      float worst = 0.f, fsum = 0.f;
      for (int c = 0; c < ncon; c++) {
        const float* ce = l_centry<C>(sm, w, c);
        int info = ((const int*)ce)[LCE_INFO];
        if (!(info & 1)) continue;
        for (int k = 0; k < 4; k++) {
          bool act = (info & (2 << k)) != 0, neg = ce[LCE_RS + k] < 0.f;
          if (act != neg) worst = fmaxf(worst, fabsf(ce[LCE_D] * ce[LCE_RS + k]));
          if (neg) fsum += fabsf(ce[LCE_D] * ce[LCE_RS + k]);
        }
      }
      if (worst < 1e-3f) L_STAT(22, 1);
      if (worst < 1e-2f) L_STAT(23, 1);
      if (worst < 1e-1f) L_STAT(24, 1);
      if (worst < 1.f) L_STAT(25, 1);
      if (worst < 1e-4f * fsum) L_STAT(26, 1);
      if (worst < 1e-3f * fsum) L_STAT(27, 1);
    }
  }
#endif
  // align bit 3: every warp of the CTA makes the same number of iterations (predicated), so all of them stay in the same sweep
  const bool cu = (H.align & 8) && w.bar;
  if (!(cu ? (__syncthreads_or(run) != 0) : __any_sync(L_FULL, run))) return 0;
  // envs whose first trial point changed the sign pattern: adopt it as the iterate, then iterate
  float o4[5];
  l_rows<C>(sm, w, run, 0, 0.f, o4);
  __syncwarp();
  int it = 1, iters = 0;
  for (; it < L_SOLVER_MAXITER; it++) {
    if (!(cu ? (__syncthreads_or(run) != 0) : __any_sync(L_FULL, run))) break;
    bool same = l_linsolve<C>(ms, sm, w, run, H.dirtypath ? LI_RESWEEP : 0, true, false, st);      // qdd -> qstar
    bool fin = run && same, lsrch = run && !same;
    if (__any_sync(L_FULL, lsrch)) {   // exact line search between the iterate (qacc, r, phi) and the trial point (qstar, rs), row space only
      l_rows<C>(sm, w, lsrch, 4, 0.f, o4);      // sums at the iterate (al = 0) and at the trial point (al = 1) in one pass over the rows
      float g1 = l_gsum(o4[0]), g2 = l_gsum(o4[1]), s1 = l_gsum(o4[4]), s11 = l_gsum(o4[2]), s2 = l_gsum(o4[3]);
      float f0 = g1 + s1, al = 0.f, lo = 0.f, hi = -1.f, tol = H.ls_tol * fabsf(f0);
      bool searching = lsrch && (f0 < -L_LS_NOISE * (fabsf(g1) + fabsf(s1)));   // |f0| below the fp32 cancellation floor: converged
      if (searching) al = 1.f;
      s1 = s11;
      for (int ls = 0; ls < L_LS_MAXITER; ls++) {
        if (!__any_sync(L_FULL, searching)) break;
        if (ls > 0) {
          l_rows<C>(sm, w, searching, 1, al, o4);
          s1 = l_gsum(o4[2]); s2 = l_gsum(o4[3]);
        }
        if (searching) {
          float f = g1 + al * g2 + s1, fp = g2 + s2;
          if (fabsf(f) <= tol) searching = false;
          else {
            if (f < 0.f) lo = al; else hi = al;
            float an = (fp > 0.f) ? al - f / fp : -1.f;
            if (!(an > lo) || (hi > 0.f && !(an < hi))) an = (hi > 0.f) ? 0.5f * (lo + hi) : 2.f * al;
            an = fminf(an, L_LS_MAXSTEP);
            if (an == al) searching = false; else al = an;
          }
        }
      }
      bool step = lsrch && (al > 0.f);
      if (lsrch && !step) { run = false; iters = it; }
      l_rows<C>(sm, w, step, 2, al, o4);
      if (step) for (int d = w.li; d < H.nv; d += LM_LPE) sm[C::qacc + d] = fmaf(al, sm[C::qstar + d] - sm[C::qacc + d], sm[C::qacc + d]);
    }
    if (fin) {
      for (int d = w.li; d < H.nv; d += LM_LPE) sm[C::qacc + d] = sm[C::qstar + d];
      run = false; iters = it;
    }
    __syncwarp();
  }
  if (run) { iters = it; *hit_max = true; }
#ifdef SMPLSIM_STATS
  if (w.live && w.li == 0 && iters > 0) L_STAT(2 + (iters > 6 ? 6 : iters), 1);
  if (w.live && w.li == 0 && any_rows) {   // [28] env-substeps with >= 3 extra solves, [29] ... that hold a contact new this substep, [30] env-substeps with a new contact, [31] contacts of [28]
    const int ncon = ((const int*)sm)[C::misc + LMI_NCON];
    int hasnew = 0, np = 0;
    for (int c = 0; c < ncon; c++) {
      int info = ((const int*)l_centry<C>(sm, w, c))[LCE_INFO];
      if (info & 1) { np++; if (info & 32) hasnew = 1; }
    }
    if (hasnew) L_STAT(30, 1);
    if (iters >= 3) { L_STAT(28, 1); if (hasnew) L_STAT(29, 1); L_STAT(31, np); }
  }
  if (w.live && w.li == 0) {   // [16] rows, [17] inherit guess wrong vs the final set, [18] prediction wrong, [19] both wrong, [20] contacts where inherit is right, [21] pred right
    const int ncon = ((const int*)sm)[C::misc + LMI_NCON];
    for (int c = 0; c < ncon; c++) {
      int info = ((const int*)l_centry<C>(sm, w, c))[LCE_INFO];
      if (!(info & 1)) continue;
      int fin = (info >> 1) & 15, inh = (info >> 24) & 15, prd = (info >> 28) & 15;
      L_STAT(16, 4); L_STAT(17, __popc(fin ^ inh)); L_STAT(18, __popc(fin ^ prd)); L_STAT(19, __popc((fin ^ inh) & (fin ^ prd)));
      if (fin == inh) L_STAT(20, 1);
      if (fin == prd) L_STAT(21, 1);
    }
  }
#endif
  return iters;
}

// ------------------------------------------------------------------ elementwise controllers (pd / torque / simple_pid), controllers.py:6-47,186-349
template <class C>
__device__ __noinline__ void l_torque_elem(const float* ms, float* sm, const LLane& w, const SmplsimState& sta) {
  const LHdr& H = l_hdr<C>(ms);
  const LBody* MB = l_bodies(ms);
  const int mode = H.cfg.control_mode;
  if (w.live) {
    for (int i = w.li; i < H.nu; i += LM_LPE) {
      const int b = 1 + i / 3, k = i - 3 * (b - 1);     // SMPL family: three hinges per non-root body, dofs in body order
      const LBody& lb = MB[b];
      float a = sm[C::act + i], tq;
      if (mode == SMPLSIM_CTRL_TORQUE) tq = a * lb.ascale[k];
      else if (mode == SMPLSIM_CTRL_SIMPLE_PID) {   // stateful: integral / last error live in HBM (L2-resident, 2 x nu words per env)
        size_t o = (size_t)w.env * H.nu + i;
        float dt = H.h * (float)H.cfg.nsubsteps, lim = lb.tlim[k];
        float err = fmaf(a, lb.ascale[k], lb.aoffset[k]) - sm[C::qpos + 7 + i], le = sta.pid_last_error[o];
        float derr = (le != le) ? 0.f : err - le;
        float in = fminf(fmaxf(fmaf(err, dt, sta.pid_integral[o]), -lim), lim);
        sta.pid_integral[o] = in; sta.pid_last_error[o] = err;
        tq = lb.kp[k] * err + in + lb.kd[k] * derr / dt;
      } else {
        float tgt = fmaf(a, lb.ascale[k], lb.aoffset[k]), q = sm[C::qpos + 7 + i], qd = sm[C::qvel + 6 + i];
        tq = -lb.kp[k] * (q - tgt) - lb.kd[k] * qd;
      }
      sm[C::tau + i] = fminf(fmaxf(tq, -lb.tlim[k]), lb.tlim[k]);
    }
  }
  __syncwarp();
}

// semi-implicit Euler when no stable-PD sweep follows (elementwise; root quaternion by the first lane)
template <class C>
__device__ __noinline__ void l_integrate(const float* ms, float* sm, const LLane& w, LSolveLane& st) {
  const LHdr& H = l_hdr<C>(ms);
  if (w.live) {
    float h = H.h;
    for (int d = 3 + w.li; d < H.nv; d += LM_LPE) {
      float v = fmaf(h, sm[C::qacc + d], sm[C::qvel + d]);
      sm[C::qvel + d] = v;
      if (d >= 6) sm[C::qpos + d + 1] = fmaf(h, v, sm[C::qpos + d + 1]);
    }
    if (w.li == 0) {   // root translation on the lane that keeps the displacement
#pragma unroll
      for (int d = 0; d < 3; d++) {
        float v = fmaf(h, sm[C::qacc + d], sm[C::qvel + d]), dd = h * v;
        sm[C::qvel + d] = v; sm[C::qpos + d] += dd;
        if (d < 2) sm[C::misc + LMI_DISP + d] += dd;
      }
    }
  }
  __syncwarp();
  if (w.live && w.li == 0) {
    float* qpos = sm + C::qpos;
    V3 wv = ld3(sm + C::qvel + 3);
    float n = sqrtf(dot(wv, wv)), ang = n * H.h;
    Q4 q; q.w = qpos[3]; q.x = qpos[4]; q.y = qpos[5]; q.z = qpos[6];
    if (ang > 0.f) {
      float sn, cs;
      l_sincos(0.5f * ang, &sn, &cs);
      float s = sn / n;
      Q4 dq; dq.w = cs; dq.x = wv.x * s; dq.y = wv.y * s; dq.z = wv.z * s;
      q = qmul(q, dq);
    }
    q = qnormalize(q);
    qpos[3] = q.w; qpos[4] = q.x; qpos[5] = q.y; qpos[6] = q.z;
  }
  __syncwarp();
}

// mj_checkPos / mj_checkVel (what 0, before the forward pass) and mj_checkAcc (what 1, after the solve), SURVEY A.2
// ([MJ-upstream] engine_forward.c): a NaN or |x| > mjMAXVAL raises the warning bit and auto-resets the env's data like
// mj_resetData (qpos = qpos0, qvel = ctrl = qacc_warmstart = 0).  Returns the warning bits of this lane's env.
template <class C>
__device__ __noinline__ int l_check(const float* ms, float* sm, const LLane& w, int what) {
  const LHdr& H = l_hdr<C>(ms);
  bool b0 = false, b1 = false;
  if (w.live) {
    if (what == 0) {
#pragma unroll 1
      for (int i = w.li; i < H.nv + 1; i += LM_LPE) b0 |= !(fabsf(sm[C::qpos + i]) <= L_MAXVAL);
#pragma unroll 1
      for (int i = w.li; i < H.nv; i += LM_LPE) b1 |= !(fabsf(sm[C::qvel + i]) <= L_MAXVAL);
    } else {
#pragma unroll 1
      for (int i = w.li; i < H.nv; i += LM_LPE) b0 |= !(fabsf(sm[C::qacc + i]) <= L_MAXVAL);
    }
  }
  b0 = l_gany(b0, w); b1 = l_gany(b1, w);
  int bits = (what == 0) ? (b0 ? 1 : (b1 ? 2 : 0)) : (b0 ? 4 : 0);
  if (bits && w.live) {
    const LBody* MB = l_bodies(ms);
#pragma unroll 1
    for (int i = w.li; i < H.nv + 1; i += LM_LPE) sm[C::qpos + i] = (i < 3) ? MB[0].bpos[i] : (i < 7) ? MB[0].bquat[i - 3] : 0.f;
#pragma unroll 1
    for (int i = w.li; i < H.nv; i += LM_LPE) { sm[C::qvel + i] = 0.f; sm[C::qacc + i] = 0.f; }
#pragma unroll 1
    for (int i = w.li; i < H.nu; i += LM_LPE) sm[C::tau + i] = 0.f;
  }
  __syncwarp();
  return bits;
}

// the slot -> working-set memory the next substep's contacts inherit from
template <class C>
__device__ __forceinline__ void l_save_working_set(const float* ms, float* sm, const LLane& w) {
  const LHdr& H = l_hdr<C>(ms);
  if (w.live) for (int i = w.li; i < (H.nslot + 3) / 4; i += LM_LPE) ((int*)sm)[C::pfl + i] = 0;
  __syncwarp();
  if (w.live) {
    unsigned char* pf = (unsigned char*)(sm + C::pfl);
    const int ncon = ((const int*)sm)[C::misc + LMI_NCON];
    for (int c = w.li; c < ncon; c += LM_LPE) {
      int info = ((const int*)l_centry<C>(sm, w, c))[LCE_INFO];
      if ((info & 1) && !(info & LCE_SELF)) pf[(info >> 16) & 255] = (unsigned char)(info & 31);
    }
  }
  __syncwarp();
}

struct LFwd { unsigned long long mask; int iters; int status; };



// ------------------------------------------------------------------ nsub x [compute_torque + mj_step]   (humanoid_env.py:439-453)
// Entry condition in stable-PD (stale) mode: records hold the (M + h Kd) factors of the last forward pass for the state in
// qpos / qvel and the action in act (prologue of the kernels: l_spd_prologue).
template <class C>
__device__ __noinline__ void l_substeps(const float* ms, float* sm, const LLane& w, int nsub, int raw, LFwd* fo, const SmplsimState& sta,
                                        bool write_fwd, bool prep_last, LSolveLane& st) {
  const LHdr& H = l_hdr<C>(ms);
  const bool spd = (H.cfg.control_mode == SMPLSIM_CTRL_UHC_PD) && !raw, stale = H.cfg.spd_stale != 0;
  bool restore = false;   // raw mode: the caller's ctrl (kept in act) comes back the substep after an auto-reset zeroed it
  for (int s = 0; s < nsub; s++) {
    if (H.align & 1) __syncthreads();   // keep the warps of a CTA in the same sweep: they then share the instruction-cache lines
    if (!raw) {
      if (!spd) l_torque_elem<C>(ms, sm, w, sta);
    } else if (__any_sync(L_FULL, restore)) {
      if (w.live && restore) for (int i = w.li; i < H.nu; i += LM_LPE) sm[C::tau + i] = sm[C::act + i];
      restore = false;
      __syncwarp();
    }
    int bad = l_check<C>(ms, sm, w, 0);
    if (spd && !stale) {   // spd_inertia = "fresh": factors of the current state, then the torque
      l_sweep_out<C>(ms, sm, w, LF_FK | LF_VEL, false);
      l_sweep_in<C, true>(ms, sm, w, w.live, LI_SPD, st);
      l_sweep_out<C>(ms, sm, w, LF_GOUT, bad != 0);
    }
    const bool last = (s == nsub - 1);
    int f1 = LF_FK | LF_VEL | LF_COLLIDE | ((spd && stale) ? LF_GOUT : 0) | (last ? LF_SENS : 0);
    LFkOut fk = l_sweep_out<C>(ms, sm, w, f1, bad != 0);
    if (C::SELFCOL && H.cfg.self_collision && w.gbody && H.npair > 0) {
      int dr = 0;
      fk.nrows += 4 * l_self_collide<C>(ms, sm, w, &dr);
      fk.dropped |= dr;
    }
    bool hit = false;
    fo->mask = fk.mask;
    if (H.align & 2) __syncthreads();
    fo->iters = l_solve<C>(ms, sm, w, fk.nrows > 0, st, &hit);
    int extra = (fk.dropped ? L_ST_ROWS_DROPPED : 0) | (hit ? L_ST_MAXITER : 0);
    int badacc = l_check<C>(ms, sm, w, 1);
    if (__any_sync(L_FULL, badacc != 0)) {   // mj_checkAcc: forward pass again on the reset data, then integrate
      LLane w2 = w;
      w2.live = w.live && badacc != 0;
      w2.bar = false;
      LFkOut fk2 = l_sweep_out<C>(ms, sm, w2, LF_FK | LF_VEL | LF_COLLIDE | (last ? LF_SENS : 0), false);
      if (C::SELFCOL && H.cfg.self_collision && w.gbody && H.npair > 0) { int dr = 0; fk2.nrows += 4 * l_self_collide<C>(ms, sm, w2, &dr); }
      bool hit2 = false;
      int it2 = l_solve<C>(ms, sm, w2, fk2.nrows > 0, st, &hit2);
      if (badacc) { fo->mask = fk2.mask; fo->iters = it2; }
    }
    l_save_working_set<C>(ms, sm, w);
    bad |= badacc;
    fo->status |= bad | extra;
    if (raw && bad) restore = true;
    if (last && write_fwd && w.live) {
      float* qf = sta.qpos_fwd + (size_t)w.env * (H.nv + 1); float* vf = sta.qvel_fwd + (size_t)w.env * H.nv;
      for (int i = w.li; i < H.nv + 1; i += LM_LPE) qf[i] = sm[C::qpos + i];
      for (int i = w.li; i < H.nv; i += LM_LPE) vf[i] = sm[C::qvel + i];
    }
    if (last && write_fwd) __syncwarp();   // the integration below overwrites what other lanes are still copying
    if (H.align & 4) __syncthreads();
    if (spd && stale && (!last || prep_last)) l_sweep_in<C, true>(ms, sm, w, w.live, LI_SPD | LI_INTEGRATE, st);   // FK rows: s_k ; qpos / qvel: s_{k+1}
    else l_integrate<C>(ms, sm, w, st);
  }
}

// ====================================================================================================================
// env-level kernels
// ====================================================================================================================
// per-env body shapes (smplsim_create_shapes): CTA b stages table blk_img[b]; slot i of the grid works on env slot_env[i] (< 0: none).
// Both NULL: one table, slot == env.
struct LMap { const int* slot_env; const int* blk_img; };
struct LStepArgs {
  SmplsimState st;
  SmplsimAux aux;
  const float* action;
  float* obs;
  float* reward;
  uint8_t* terminated;
  uint8_t* truncated;
  float* gscr;       // [n, (NS - NCS) * CONW] overflow contact entries
  float* gsens;      // [n, 6 nb] or NULL
  float* gbody;      // [n, 10 nb] or NULL (self-collision)
  int* gpfl;         // [n, r4(NS / 4)] working set per contact slot
  LMap map;
  int n, nsub, mode;
};
struct LResetArgs {
  SmplsimState st;
  SmplsimAux aux;
  const uint8_t* mask;
  const float* qpos0;
  const float* qvel0;
  float* obs;
  float* gscr;
  float* gsens;
  float* gbody;
  int* gpfl;
  LMap map;
  int n, init_mode;
};
struct LKinArgs { const float* qpos; float* xpos; float* xquat; LMap map; int n; };

template <class C>
__device__ __forceinline__ void l_copy(float* dst, const float* src, int n, const LLane& w) {
  if (w.live) for (int i = w.li; i < n; i += LM_LPE) dst[i] = src[i];
}
// rows whose length and base are multiples of 4 words move as float4 (state rows are padded to 16 bytes only in shared memory,
// so the global side is checked at run time)
template <class C>
__device__ __forceinline__ void l_copy_in(float* dst, const float* __restrict__ src, int n, const LLane& w) {
  if (!w.live) return;
  if ((((size_t)src) & 15) == 0) {
    int n4 = n >> 2;
    for (int i = w.li; i < n4; i += LM_LPE) ((float4*)dst)[i] = ((const float4*)src)[i];
    for (int i = (n4 << 2) + w.li; i < n; i += LM_LPE) dst[i] = src[i];
  } else for (int i = w.li; i < n; i += LM_LPE) dst[i] = src[i];
}
template <class C>
__device__ __forceinline__ void l_copy_out(float* __restrict__ dst, const float* src, int n, const LLane& w) {
  if (!w.live) return;
  if ((((size_t)dst) & 15) == 0) {
    int n4 = n >> 2;
    for (int i = w.li; i < n4; i += LM_LPE) ((float4*)dst)[i] = ((const float4*)src)[i];
    for (int i = (n4 << 2) + w.li; i < n; i += LM_LPE) dst[i] = src[i];
  } else for (int i = w.li; i < n; i += LM_LPE) dst[i] = src[i];
}

template <class C>
__device__ __noinline__ void l_task_io(float* sm, const LLane& w, const SmplsimState& st, bool store) {
  if (store) __syncwarp();
  if (w.live && w.li == 0) {
    float* t = sm + C::tsk;
    int* ti = (int*)t;
    int env = w.env;
    if (!store) {
      for (int j = 0; j < 4; j++) t[j] = st.task_target[4 * env + j];
      ti[L_TSK_CHANGE] = st.task_change_step[env]; ti[L_TSK_CURT] = st.progress[env]; ti[L_TSK_RECOV] = st.recovery[env];
      ti[L_TSK_RNG] = (int)st.rng_counter[env];
    } else {
      for (int j = 0; j < 4; j++) st.task_target[4 * env + j] = t[j];
      st.task_change_step[env] = ti[L_TSK_CHANGE]; st.progress[env] = ti[L_TSK_CURT]; st.recovery[env] = ti[L_TSK_RECOV];
      st.rng_counter[env] = (uint32_t)ti[L_TSK_RNG];
    }
  }
  if (!store) __syncwarp();
}

// reset_task() of the three tasks (tasks/humanoid_speed.py:97-103, humanoid_reach.py:80-90, humanoid_getup.py:83-89); first lane only
template <class C>
__device__ __noinline__ void l_reset_task(const LHdr& H, float* sm, int env) {
  const SmplsimEnvCfg& c = H.cfg;
  if (c.task == SMPLSIM_TASK_NONE) return;
  float* t = sm + C::tsk;
  int* ti = (int*)t;
  uint32_t r[4];
  philox4x32((uint32_t)ti[L_TSK_RNG], (uint32_t)env, 0u, 0u, (uint32_t)c.seed, (uint32_t)(c.seed >> 32), r);
  ti[L_TSK_RNG] = ti[L_TSK_RNG] + 1;
  if (c.task == SMPLSIM_TASK_SPEED) t[0] = (float)(c.tar_speed_max - c.tar_speed_min) * u01(r[0]) + (float)c.tar_speed_min;
  else if (c.task == SMPLSIM_TASK_REACH) {
    t[0] = (float)c.tar_dist_max * (2.0f * u01(r[0]) - 1.0f);
    t[1] = (float)c.tar_dist_max * (2.0f * u01(r[1]) - 1.0f);
    t[2] = (float)(c.tar_height_max - c.tar_height_min) * u01(r[2]) + (float)c.tar_height_min;
  } else t[0] = (float)(c.tar_height_max - c.tar_height_min) * u01(r[0]) + (float)c.tar_height_min;
  ti[L_TSK_CHANGE] = ti[L_TSK_CURT] + rand_range(r[3], c.change_steps_min, c.change_steps_max);
}

__device__ __forceinline__ Q4 l_heading_inv(const LHdr& H, Q4 root) {
  if (!H.cfg.upright_start) { Q4 bc; bc.w = 0.5f; bc.x = -0.5f; bc.y = -0.5f; bc.z = -0.5f; root = qmul(root, bc); }
  V3 rd = qrot_ref(root, v3(1.f, 0.f, 0.f));
  float hd = atan2f(rd.y, rd.x), sn, cs;
  l_sincos(-0.5f * hd, &sn, &cs);
  Q4 h; h.w = cs; h.x = 0.f; h.y = 0.f; h.z = sn;
  return qnormalize(h);
}

// compute_observations (humanoid_env.py:565-688, tasks/*.py): staged in shared memory, then streamed out coalesced
template <class C>
__device__ __noinline__ void l_write_obs(const float* ms, float* sm, const LLane& w, float* obs_row) {
  const LHdr& H = l_hdr<C>(ms);
  if (w.live && (C::OBS_STAGED || obs_row)) {
    float* ob = C::OBS_STAGED ? sm + C::obs : obs_row;
    const float *qpos = sm + C::qpos, *xq = sm + C::xq, *qvel = sm + C::qvel, *sens = w.gsens;
    int nb = H.nb;
    Q4 r0; r0.w = xq[0]; r0.x = xq[1]; r0.y = xq[2]; r0.z = xq[3];
    Q4 hq = l_heading_inv(H, r0);
    int o = H.cfg.root_height_obs ? 1 : 0, o_rot = o + 3 * (nb - 1), o_vel = o_rot + 6 * nb;
    if (o && w.li == 0) ob[0] = qpos[2];
    for (int b = w.li; b < nb; b += LM_LPE) {
      if (b > 0) st3(ob + o + 3 * (b - 1), qrot_ref(hq, ld3(sm + C::body + C::BODYW * b + LBR_X)));
      Q4 q; q.w = xq[4 * b]; q.x = xq[4 * b + 1]; q.y = xq[4 * b + 2]; q.z = xq[4 * b + 3];
      Q4 lq = qmul(hq, q);
      st3(ob + o_rot + 6 * b, qrot_ref(lq, v3(1.f, 0.f, 0.f)));
      st3(ob + o_rot + 6 * b + 3, qrot_ref(lq, v3(0.f, 0.f, 1.f)));
      if (H.cfg.self_obs_v == 2 && sens) {
        st3(ob + o_vel + 3 * b, qrot_ref(hq, ld3(sens + 6 * b)));
        st3(ob + o_vel + 3 * nb + 3 * b, qrot_ref(hq, ld3(sens + 6 * b + 3)));
      }
    }
    if (H.cfg.self_obs_v == 1) {
      if (w.li == 0) st3(ob + o_vel, qrot_ref(hq, ld3(qvel)));
      if (w.li == 1) st3(ob + o_vel + 3, qrot_ref(hq, ld3(qvel + 3)));
      for (int i = w.li; i < H.nu; i += LM_LPE) ob[o_vel + 6 + i] = qvel[6 + i];
    }
    if (w.li == 2) {
      const float* t = sm + C::tsk;
      int ot = H.self_obs_dim;
      Q4 rq; rq.w = qpos[3]; rq.x = qpos[4]; rq.y = qpos[5]; rq.z = qpos[6];
      if (H.cfg.task == SMPLSIM_TASK_SPEED) {
        V3 d = qrot_ref(l_heading_inv(H, rq), v3(1.f, 0.f, 0.f));
        ob[ot] = d.x; ob[ot + 1] = d.y; ob[ot + 2] = t[0];
      } else if (H.cfg.task == SMPLSIM_TASK_REACH) st3(ob + ot, qrot_ref(l_heading_inv(H, rq), ld3(t) - ld3(qpos)));
      else if (H.cfg.task == SMPLSIM_TASK_GETUP) ob[ot] = t[0];
    }
  }
  __syncwarp();
  if (C::OBS_STAGED && obs_row) l_copy_out<C>(obs_row, sm + C::obs, H.obs_dim, w);
  __syncwarp();
}

template <class C>
__device__ __noinline__ void l_write_aux(const float* ms, float* sm, const LLane& w, const SmplsimAux& aux, const LFwd& fo) {
  const LHdr& H = l_hdr<C>(ms);
  if (!w.live) return;
  V3 root = ld3(sm + C::qpos);
  int nb = H.nb, env = w.env;
  for (int b = w.li; b < nb; b += LM_LPE) {
    size_t bi = (size_t)env * nb + b;
    if (aux.xpos) st3(aux.xpos + bi * 3, ld3(sm + C::body + C::BODYW * b + LBR_X) + root);
    if (w.gsens) {
      if (aux.body_linvel) st3(aux.body_linvel + bi * 3, ld3(w.gsens + 6 * b));
      if (aux.body_angvel) st3(aux.body_angvel + bi * 3, ld3(w.gsens + 6 * b + 3));
    }
  }
  if (aux.xquat) l_copy<C>(aux.xquat + (size_t)env * nb * 4, sm + C::xq, 4 * nb, w);
  if (aux.qacc) l_copy<C>(aux.qacc + (size_t)env * H.nv, sm + C::qacc, H.nv, w);
  if (aux.ctrl) l_copy<C>(aux.ctrl + (size_t)env * H.nu, sm + C::tau, H.nu, w);
  if (w.li == 0) {
    if (aux.contact_mask) aux.contact_mask[env] = fo.mask;
    if (aux.solver_iter) aux.solver_iter[env] = fo.iters;
    if (aux.status) aux.status[env] = (uint8_t)fo.status;
  }
}

// Self-collision is not simulated (SURVEY 8 f4).  Once per env step, on the final kinematics (xquat staging + body rows), test the
// capsule / sphere geom pairs MuJoCo's filters let through (smpl_humanoid.xml:5,24,231-242); a touching pair means the reference
// would have generated a geom-geom contact here.  Returns true for this lane's env.
template <class C>
__device__ __noinline__ bool l_self_contact(const float* ms, float* sm, const LLane& w) {
  const LHdr& H = l_hdr<C>(ms);
  const LGeom* MG = l_geoms(ms);
  const LPair* PR = (const LPair*)((const char*)ms + H.pair_off);
  bool hit = false;
  if (w.live) {
    for (int i = w.li; i < H.npair; i += LM_LPE) {
      const LGeom& G1 = MG[PR[i].g1]; const LGeom& G2 = MG[PR[i].g2];
      const float* q1 = sm + C::xq + 4 * G1.body; const float* q2 = sm + C::xq + 4 * G2.body;
      Q4 a; a.w = q1[0]; a.x = q1[1]; a.y = q1[2]; a.z = q1[3];
      Q4 b; b.w = q2[0]; b.x = q2[1]; b.y = q2[2]; b.z = q2[3];
      V3 c1 = ld3(sm + C::body + C::BODYW * G1.body + LBR_X) + qrot(a, ld3(G1.pos));
      V3 c2 = ld3(sm + C::body + C::BODYW * G2.body + LBR_X) + qrot(b, ld3(G2.pos));
      float r1 = G1.size[0], r2 = G2.size[0];
      float h1 = (G1.type == SMPLSIM_GEOM_CAPSULE) ? G1.size[1] : 0.f, h2 = (G2.type == SMPLSIM_GEOM_CAPSULE) ? G2.size[1] : 0.f;
      V3 dc = c2 - c1;
      float reach = h1 + h2 + r1 + r2 + H.margin;
      if (dot(dc, dc) > reach * reach) continue;                      // bounding spheres
      V3 a1 = qrot(a, v3(G1.mat[2], G1.mat[5], G1.mat[8])), a2 = qrot(b, v3(G2.mat[2], G2.mat[5], G2.mat[8]));
      float s, t;
      l_segment_segment(c1, a1, h1, c2, a2, h2, &s, &t);
      V3 n = (c2 + t * a2) - (c1 + s * a1);
      if (sqrtf(dot(n, n)) - r1 - r2 <= H.margin) hit = true;
    }
  }
  return l_gany(hit, w);
}

#ifdef SMPLSIM_EMU
#define L_SMEM EMU_SMEM_BASE
#else
extern __shared__ float4 l_smem4[];
#define L_SMEM ((float*)l_smem4)
#endif

// CTA prologue: stage the constant table, carve the env rows.  Shared memory: [table | 4 words | env rows]
template <class C>
__device__ __forceinline__ float* l_setup(const float* __restrict__ gimg, int img_bytes, LLane& w, const float*& ms, int n, const LMap& map, float* gscr, float* gsens, int* gpfl, float* gbody = nullptr) {
  float* smem = L_SMEM;
  if (map.blk_img) gimg += (size_t)map.blk_img[blockIdx.x] * (size_t)(img_bytes / 4);   // this CTA's body shape
  unsigned* slot = (unsigned*)(smem + img_bytes / 4);   // [2..3] mbarrier of the table copy
#ifndef SMPLSIM_EMU
  {
    // the constant table arrives as ONE bulk asynchronous copy (TMA engine, cp.async.bulk -> UBLKCP) signalled on an mbarrier: one thread
    // initialises the barrier here and issues the copy behind the CTA barrier below (init -> fence -> CTA sync -> expect_tx + copy)
    const unsigned mb = (unsigned)__cvta_generic_to_shared(slot + 2);
    if (threadIdx.x == 0) {
      asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(mb) : "memory");
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
  }
#else
  {
    const uint4* src = (const uint4*)gimg;
    uint4* dst = (uint4*)smem;
    for (int i = threadIdx.x; i < img_bytes / 16; i += blockDim.x) dst[i] = src[i];
  }
#endif
  ms = smem;
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  __syncthreads();
#ifndef SMPLSIM_EMU
  {   // one thread starts the copy; every thread waits for the table (phase 0 of the mbarrier)
    const unsigned mb = (unsigned)__cvta_generic_to_shared(slot + 2), dst = (unsigned)__cvta_generic_to_shared(smem);
    if (threadIdx.x == 0) {
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mb), "r"((unsigned)img_bytes) : "memory");
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                   ::"r"(dst), "l"(gimg), "r"((unsigned)img_bytes), "r"(mb) : "memory");
    }
    unsigned done = 0;
    while (!done) {
      asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0; selp.u32 %0, 1, 0, p; }" : "=r"(done) : "r"(mb) : "memory");
    }
  }
#endif
  const int sub = lane / LM_LPE;
  w.lane = lane; w.li = lane % LM_LPE; w.gbase = sub * LM_LPE;
  w.gmask = ((1u << LM_LPE) - 1u) << (sub * LM_LPE);
  w.env = (blockIdx.x * wpb + wib) * C::EPW + sub;
  if (map.slot_env) w.env = map.slot_env[w.env];
  w.live = w.env >= 0 && w.env < n;
  w.bar = true;
  w.gscr = gscr + (size_t)(w.live ? w.env : 0) * (size_t)(C::CONW * (C::NS - C::NCS));
  w.gbody = gbody ? gbody + (size_t)(w.live ? w.env : 0) * (size_t)(10 * C::NB) : nullptr;
  w.gpfl = gpfl ? gpfl + (size_t)(w.live ? w.env : 0) * (size_t)C::PFLW : nullptr;
  w.gsens = gsens ? gsens + (size_t)(w.live ? w.env : 0) * (size_t)(6 * C::NB) : nullptr;
  return smem + img_bytes / 4 + 4 + (size_t)(wib * C::EPW + sub) * C::total;
}

// stable PD, stale inertia (quirk Q1): rebuild the (M + h Kd) factors of the state of the last forward pass for the current
// state / action.  On entry qpos / qvel / act hold the current state; qpos_fwd / qvel_fwd come from HBM.
template <class C>
__device__ __noinline__ void l_spd_prologue(const float* ms, float* sm, const LLane& w, const SmplsimState& sta, LSolveLane& st) {
  const LHdr& H = l_hdr<C>(ms);
  size_t eo = w.live ? (size_t)w.env : 0;
  l_copy_in<C>(sm + C::qpos, sta.qpos_fwd + eo * (H.nv + 1), H.nv + 1, w);
  l_copy_in<C>(sm + C::qvel, sta.qvel_fwd + eo * H.nv, H.nv, w);
  __syncwarp();
  l_sweep_out<C>(ms, sm, w, LF_FK | LF_VEL, false);
  l_copy_in<C>(sm + C::qpos, sta.qpos + eo * (H.nv + 1), H.nv + 1, w);
  l_copy_in<C>(sm + C::qvel, sta.qvel + eo * H.nv, H.nv, w);
  __syncwarp();
  l_sweep_in<C, true>(ms, sm, w, w.live, LI_SPD, st);
}

template <class C>
__global__ void __launch_bounds__(256, 1) k_step5(const float* __restrict__ gimg, int img_bytes, LStepArgs a) {
  const float* ms; LLane w;
  float* sm = l_setup<C>(gimg, img_bytes, w, ms, a.n, a.map, a.gscr, a.gsens, a.gpfl, a.gbody);
  const LHdr& H = l_hdr<C>(ms);
  const size_t eo = w.live ? (size_t)w.env : 0;   // lanes without a live env keep running (predicated): warp collectives stay legal
  const bool spd = (H.cfg.control_mode == SMPLSIM_CTRL_UHC_PD);
  LSolveLane st; st.dirty_bits = 0u; st.rc_bits = 0u;
  if (w.live && w.li == 0) { sm[C::misc + LMI_DISP] = 0.f; sm[C::misc + LMI_DISP + 1] = 0.f; ((int*)sm)[C::misc + LMI_NSELF] = 0; ((int*)sm)[C::misc + LMI_NCON] = 0; ((int*)sm)[C::misc + LMI_NLIM] = 0; }
  if (w.live) for (int i = w.li; i < (H.nslot + 3) / 4; i += LM_LPE) ((int*)sm)[C::pfl + i] = w.gpfl ? w.gpfl[i] : 0;   // working set of the previous call
  l_copy_in<C>(sm + C::act, a.action + eo * H.nu, H.nu, w);
  if (spd && H.cfg.spd_stale && a.mode == 0) l_spd_prologue<C>(ms, sm, w, a.st, st);
  else {
    l_copy_in<C>(sm + C::qpos, a.st.qpos + eo * (H.nv + 1), H.nv + 1, w);
    l_copy_in<C>(sm + C::qvel, a.st.qvel + eo * H.nv, H.nv, w);
  }
  l_copy_in<C>(sm + C::qacc, a.st.qacc_warm + eo * H.nv, H.nv, w);
  if (a.mode != 0) l_copy_in<C>(sm + C::tau, a.action + eo * H.nu, H.nu, w);   // raw ctrl (act keeps a copy for the substep after an auto-reset)
  l_task_io<C>(sm, w, a.st, false);
  if (a.mode == 0 && w.live && w.li == 0) {
    int* ti = (int*)(sm + C::tsk);
    if (H.cfg.task != SMPLSIM_TASK_NONE && ti[L_TSK_CURT] >= ti[L_TSK_CHANGE]) l_reset_task<C>(H, sm, w.env);
  }
  __syncwarp();
  LFwd fo; fo.mask = 0ull; fo.iters = 0; fo.status = 0;
  l_substeps<C>(ms, sm, w, a.nsub, a.mode, &fo, a.st, true, false, st);
  l_sweep_out<C>(ms, sm, w, LF_FK | LF_XQUAT, false);
  if (H.npair > 0 && !H.cfg.self_collision && a.aux.status && l_self_contact<C>(ms, sm, w)) fo.status |= L_ST_SELF_CONTACT;   // detected, not simulated
  if (a.mode == 0) {
    int* ti = (int*)(sm + C::tsk);
    if (w.live && w.li == 0) ti[L_TSK_CURT] += 1;
    __syncwarp();
    l_write_obs<C>(ms, sm, w, a.obs ? a.obs + eo * H.obs_dim : nullptr);
    const float dx = sm[C::misc + LMI_DISP], dy = sm[C::misc + LMI_DISP + 1];
    if (w.live && w.li == 0) {
      const SmplsimEnvCfg& c = H.cfg;
      const float* t = sm + C::tsk;
      float rew = 0.f;
      if (c.task == SMPLSIM_TASK_SPEED) {
        float inv_dt = 1.0f / (H.h * (float)a.nsub), vx = dx * inv_dt, vy = dy * inv_dt, e = t[0] - vx;
        rew = expf(-0.25f * (e * e + 0.1f * vy * vy));
      } else if (c.task == SMPLSIM_TASK_REACH) {
        V3 dl = ld3(t) - (ld3(sm + C::body + C::BODYW * c.reach_body + LBR_X) + ld3(sm + C::qpos));
        rew = expf(-4.0f * dot(dl, dl));
      } else if (c.task == SMPLSIM_TASK_GETUP) { float e = t[0] - sm[C::qpos + 2]; rew = expf(-4.0f * e * e); }
      int term = 0, trunc = 0, pass_time = ti[L_TSK_CURT] > c.episode_length;
      if (c.task == SMPLSIM_TASK_NONE) trunc = pass_time;
      else if (c.task == SMPLSIM_TASK_GETUP && ti[L_TSK_RECOV] > 0) ti[L_TSK_RECOV] -= 1;
      else { trunc = pass_time; term = (fo.mask & ~H.legal_mask) != 0ull; }
      if (a.reward) a.reward[w.env] = rew;
      if (a.terminated) a.terminated[w.env] = (uint8_t)term;
      if (a.truncated) a.truncated[w.env] = (uint8_t)trunc;
    }
  }
  l_write_aux<C>(ms, sm, w, a.aux, fo);
  l_copy_out<C>(a.st.qpos + eo * (H.nv + 1), sm + C::qpos, H.nv + 1, w);
  l_copy_out<C>(a.st.qvel + eo * H.nv, sm + C::qvel, H.nv, w);
  l_copy_out<C>(a.st.qacc_warm + eo * H.nv, sm + C::qacc, H.nv, w);
  if (w.live && w.gpfl) for (int i = w.li; i < (H.nslot + 3) / 4; i += LM_LPE) w.gpfl[i] = ((const int*)sm)[C::pfl + i];
  if (a.mode == 0) l_task_io<C>(sm, w, a.st, true);
}

template <class C>
__global__ void __launch_bounds__(256, 1) k_reset5(const float* __restrict__ gimg, int img_bytes, LResetArgs a) {
  const float* ms; LLane w;
  float* sm = l_setup<C>(gimg, img_bytes, w, ms, a.n, a.map, a.gscr, a.gsens, a.gpfl, a.gbody);
  const LHdr& H = l_hdr<C>(ms);
  if (w.live && a.mask && !a.mask[w.env]) w.live = false;
  size_t eo = w.live ? (size_t)w.env : 0;
  const SmplsimEnvCfg& c = H.cfg;
  int init = a.init_mode < 0 ? c.state_init : a.init_mode;
  LSolveLane st; st.dirty_bits = 0u; st.rc_bits = 0u;
  if (w.live && w.li == 0) { sm[C::misc + LMI_DISP] = 0.f; sm[C::misc + LMI_DISP + 1] = 0.f; ((int*)sm)[C::misc + LMI_NSELF] = 0; ((int*)sm)[C::misc + LMI_NCON] = 0; ((int*)sm)[C::misc + LMI_NLIM] = 0; }
  l_task_io<C>(sm, w, a.st, false);
  if (w.live && w.li == 0) {
    int* ti = (int*)(sm + C::tsk);
    if (c.task == SMPLSIM_TASK_GETUP) ti[L_TSK_RECOV] = c.recovery_steps;
    if (!c.legacy_change_step) ti[L_TSK_CURT] = 0;
    l_reset_task<C>(H, sm, w.env);   // sees the old cur_t when legacy_change_step (quirk Q4)
  }
  if (w.live) {
    for (int i = w.li; i < (H.nslot + 3) / 4; i += LM_LPE) ((int*)sm)[C::pfl + i] = 0;
    for (int i = w.li; i < H.nv + 1; i += LM_LPE) sm[C::qpos + i] = 0.f;
    for (int i = w.li; i < H.nv; i += LM_LPE) { sm[C::qvel + i] = 0.f; sm[C::qacc + i] = 0.f; }
    for (int i = w.li; i < H.nu; i += LM_LPE) { sm[C::tau + i] = 0.f; sm[C::act + i] = 0.f; }
  }
  __syncwarp();
  LFwd fo; fo.mask = 0ull; fo.iters = 0; fo.status = 0;
  if (init == SMPLSIM_INIT_MOCAP) {
    l_copy<C>(sm + C::qpos, a.qpos0 + eo * (H.nv + 1), H.nv + 1, w);
    l_copy<C>(sm + C::qvel, a.qvel0 + eo * H.nv, H.nv, w);
  } else if (w.live && w.li == 0) {
    float* q = sm + C::qpos;
    if (init == SMPLSIM_INIT_DEFAULT) { q[2] = 0.94f; q[3] = q[4] = q[5] = q[6] = 0.5f; }
    else { q[2] = 0.3f; q[3] = 1.0f; }
  }
  __syncwarp();
  if (init == SMPLSIM_INIT_FALL) {
    const bool spd_st = (c.control_mode == SMPLSIM_CTRL_UHC_PD && c.spd_stale);
    if (spd_st) l_sweep_out<C>(ms, sm, w, LF_FK | LF_VEL, false);   // mj_forward: inertia / bias of the initial state
    int ngrp = (H.nu + 3) / 4;
    for (int k3 = 0; k3 < 3; k3++) {
      int* ti = (int*)(sm + C::tsk);
      uint32_t base = w.live ? (uint32_t)ti[L_TSK_RNG] : 0u;
      if (w.live) {
        for (int gidx = w.li; gidx < ngrp; gidx += LM_LPE) {
          uint32_t r[4];
          philox4x32(base + (uint32_t)gidx, (uint32_t)w.env, 0u, 0u, (uint32_t)c.seed, (uint32_t)(c.seed >> 32), r);
          for (int j = 0; j < 4 && 4 * gidx + j < H.nu; j++) sm[C::act + 4 * gidx + j] = u01(r[j]) - 0.5f;
        }
      }
      __syncwarp();
      if (w.live && w.li == 0) ti[L_TSK_RNG] = (int)(base + (uint32_t)ngrp);
      __syncwarp();
      if (spd_st) l_sweep_in<C, true>(ms, sm, w, w.live, LI_SPD, st);   // factors of the last forward pass, PD error of the current state and the new action
      l_substeps<C>(ms, sm, w, c.nsubsteps, 0, &fo, a.st, false, false, st);
    }
  }
  // reset_sim(): mj_forward at the reset state
  {
    LFkOut fk = l_sweep_out<C>(ms, sm, w, LF_FK | LF_VEL | LF_COLLIDE | LF_SENS, false);
    fo.mask = fk.mask;
  }
  if (w.live && w.li == 0) ((int*)(sm + C::tsk))[L_TSK_CURT] = 0;
  __syncwarp();
  l_sweep_out<C>(ms, sm, w, LF_FK | LF_XQUAT, false);
  l_write_obs<C>(ms, sm, w, a.obs ? a.obs + eo * H.obs_dim : nullptr);
  l_write_aux<C>(ms, sm, w, a.aux, fo);
  l_copy_out<C>(a.st.qpos + eo * (H.nv + 1), sm + C::qpos, H.nv + 1, w);
  l_copy_out<C>(a.st.qvel + eo * H.nv, sm + C::qvel, H.nv, w);
  l_copy_out<C>(a.st.qpos_fwd + eo * (H.nv + 1), sm + C::qpos, H.nv + 1, w);
  l_copy_out<C>(a.st.qvel_fwd + eo * H.nv, sm + C::qvel, H.nv, w);
  l_copy_out<C>(a.st.qacc_warm + eo * H.nv, sm + C::qacc, H.nv, w);
  if (w.live && w.gpfl) for (int i = w.li; i < (H.nslot + 3) / 4; i += LM_LPE) w.gpfl[i] = ((const int*)sm)[C::pfl + i];
  l_task_io<C>(sm, w, a.st, true);
}

// mujoco.mj_kinematics (humanoid_env.py:389) / poselib global_transformation on caller-supplied qpos rows
template <class C>
__global__ void __launch_bounds__(256, 1) k_kin5(const float* __restrict__ gimg, int img_bytes, LKinArgs a) {
  const float* ms; LLane w;
  float* sm = l_setup<C>(gimg, img_bytes, w, ms, a.n, a.map, nullptr, nullptr, nullptr);
  const LHdr& H = l_hdr<C>(ms);
  size_t eo = w.live ? (size_t)w.env : 0;
  l_copy<C>(sm + C::qpos, a.qpos + eo * (H.nv + 1), H.nv + 1, w);
  __syncwarp();
  l_sweep_out<C>(ms, sm, w, LF_FK | LF_XQUAT, false);
  if (w.live) {
    V3 root = ld3(sm + C::qpos);
    for (int b = w.li; b < H.nb; b += LM_LPE) st3(a.xpos + (eo * H.nb + b) * 3, ld3(sm + C::body + C::BODYW * b + LBR_X) + root);
    l_copy<C>(a.xquat + eo * H.nb * 4, sm + C::xq, 4 * H.nb, w);
  }
}
