// rne_post_kernels.cu -- k_rnep5, the kernel of smplsim_rne_post (semantics in lane_kernels.cuh above LRnepArgs, DESIGN.md 2).
// A translation unit of its own, compiled into libsmplsim_b200.so beside smplsim_capi.cu as centroidal_kernels.cu is: its noinline
// callees (l_sweep_out, l_inv_acc, l_rows) are then instances of this device module, and the kernels of smplsim_capi.cu compile exactly
// as they do without it.  smplsim_capi.cu takes the instances from lane_rnep_kernels (at the end).
// The host emulator compiles everything as one unit (smplsim_capi.cu includes this file under SMPLSIM_EMU).
#include <cuda_runtime.h>

#include <cmath>
#include <cstring>

// lane_kernels.cuh defines two functions that are not templates (l_impedance, k_zero_wrench); smplsim_capi.cu and the other kernel
// modules define them as well, so this unit's copies take names of their own
#define l_impedance l_rnep_impedance
#define k_zero_wrench k_rnep_zero_wrench
#include "lane_kernels.cuh"
#undef l_impedance
#undef k_zero_wrench

// Spatial velocity v and spatial acceleration a = J qacc + Jdot qvel of body b about the root origin (world axes, gravity not
// included), accumulated root first over the dofs of b's path as S1 accumulates v and its bias acceleration: the root's
// [sum_k qacc[3 + k] c_k ; qacc[0:3] + v_l x w], then per hinge a += qacc S + qvel (v x S) with v the velocity before that hinge.
// Bodies are numbered parents first, so the ancestors of b come in path order.
template <class C>
__device__ __forceinline__ void l_rnep_kin(const float* ms, const float* sm, int b, S6& v, S6& a) {
  const LBody* MB = l_bodies(ms);
  const float* qv = sm + C::qvel;
  const float* qa = sm + C::qacc;
  const V3 c0 = ld3(sm + C::body + LBR_AX), c1 = ld3(sm + C::body + LBR_AX + 3), c2 = ld3(sm + C::body + LBR_AX + 6);
  const V3 wv = qv[3] * c0 + qv[4] * c1 + qv[5] * c2, vl = ld3(qv);
  v = s6(wv, vl);
  a = s6(qa[3] * c0 + qa[4] * c1 + qa[5] * c2, ld3(qa) + cross(vl, wv));
  for (int e = 1; e <= b; e++) {
    if (!l_is_anc(MB[b], e)) continue;
    const float* br = sm + C::body + C::BODYW * e;
    const int d0 = MB[e].dofadr;
#pragma unroll
    for (int k = 0; k < 3; k++) {
      const S6 S = l_hingeS(br, k);
      a = a + qa[d0 + k] * S + qv[d0 + k] * cross_motion(v, S);
      v = v + qv[d0 + k] * S;
    }
  }
}

// orientation of body b: the root's quaternion (normalised by S1), then per body of the path its body quaternion and its hinges
template <class C>
__device__ __forceinline__ Q4 l_rnep_quat(const float* ms, const float* sm, int b) {
  const LBody* MB = l_bodies(ms);
  Q4 q; q.w = sm[C::qpos + 3]; q.x = sm[C::qpos + 4]; q.y = sm[C::qpos + 5]; q.z = sm[C::qpos + 6];
  for (int e = 1; e <= b; e++) {
    const LBody& lb = MB[e];
    if (!l_is_anc(MB[b], e)) continue;
    Q4 qb; qb.w = lb.bquat[0]; qb.x = lb.bquat[1]; qb.y = lb.bquat[2]; qb.z = lb.bquat[3];
    q = qmul(q, qb);
    for (int k = 0; k < 3; k++) {
      float sn, cs;
      l_sincos(0.5f * sm[C::qpos + lb.dofadr + 1 + k], &sn, &cs);
      Q4 qj; qj.w = cs; qj.x = lb.axis[3 * k] * sn; qj.y = lb.axis[3 * k + 1] * sn; qj.z = lb.axis[3 * k + 2] * sn;
      q = qmul(q, qj);
    }
  }
  return qnormalize(q);
}

__device__ __forceinline__ V3 l_rnep_rotT(Q4 q, V3 x) { q.x = -q.x; q.y = -q.y; q.z = -q.z; return qrot(q, x); }

// acceleration of the material point at x (relative to the root origin) of a body with spatial velocity v and acceleration a
__device__ __forceinline__ V3 l_rnep_pacc(S6 v, S6 a, V3 x) { return a.l + cross(a.a, x) + cross(v.a, v.l + cross(v.a, x)); }

// Row of the launch: k_inverse5's pass up to the row forces (clear the row counts and working-set memory, S1 with collisions,
// l_inv_acc leaving I_b a_b + pb_b in each record's pb slot, the working set := rs < 0), without its inward sweep.  Then, when a wrench
// output is asked for, each body's own wrench (pb slot - its floor-contact row forces - its xfrc about the root origin) back into its
// pb slot (lanes over bodies), and F_b = the sum of the own wrenches over b's subtree into gf (lanes over bodies; every descendant of b
// has a larger index).  gf is the per-env scratch smplsim_rollout fills and reads within one of its calls, free here: the overflow
// contact entries k_cent5 sums into are in use, because this pass collides.  Body outputs and sites follow (lanes over bodies, sites).
template <class C>
__global__ void __launch_bounds__(256, 1) k_rnep5(const float* __restrict__ gimg, int img_bytes, LRnepArgs a) {
  static_assert(6 * C::NB <= 2 * (2 * C::NV + 1), "the joint-wrench scratch does not fit the rollout's per-env scratch");
  const float* ms; LLane w;
  float* sm = l_setup<C>(gimg, img_bytes, w, ms, a.n, a.map, a.gscr, nullptr, nullptr);
  const LHdr& H = l_hdr<C>(ms);
  const LBody* MB = l_bodies(ms);
  const size_t eo = w.live ? (size_t)w.env : 0;
  const int nb = H.nb, nv = H.nv, li = w.li;
  if constexpr (C::PRM) l_prm_stage<C>(ms, sm, w);
  if (w.live && li == 0) { ((int*)sm)[C::misc + LMI_NSELF] = 0; ((int*)sm)[C::misc + LMI_NCON] = 0; ((int*)sm)[C::misc + LMI_NLIM] = 0; }
  if (w.live) for (int i = li; i < (H.nslot + 3) / 4; i += LM_LPE) ((int*)sm)[C::pfl + i] = 0;
  l_copy_in<C>(sm + C::qpos, a.qpos + eo * (nv + 1), nv + 1, w);
  l_copy_in<C>(sm + C::qvel, a.qvel + eo * nv, nv, w);
  l_copy_in<C>(sm + C::qacc, a.qacc + eo * nv, nv, w);
  __syncwarp();
  l_sweep_out<C>(ms, sm, w, LF_FK | LF_VEL | LF_COLLIDE, false);
  l_inv_acc<C>(ms, sm, w);
  float o4[5];
  l_rows<C>(sm, w, w.live, 0, 0.f, o4);
  __syncwarp();
  float* gf = a.gf + eo * 6 * C::NB;
  const bool frc = a.jw || a.force || a.torque;
  if (frc) {
    if (w.live)
      for (int b = li; b < nb; b += LM_LPE) {
        float r10[10];
        const int ci = l_ld_r10(sm + C::body + C::BODYW * b, r10);
        S6 F = l_rec_ld_pb<C>(w, b) - l_inv_rows<C>(H, sm, w, ci & 255, (ci >> 8) & 255);
        if (a.xfrc) {   // force f at the centre of mass r, torque t: [t + r x f ; f] about the root origin, as l_xfrc_wrench
          const float* x = a.xfrc + (eo * nb + b) * 6;
          const V3 f = ld3(x), t = ld3(x + 3);
          const V3 r = (r10[0] > 0.f ? 1.0f / r10[0] : 0.f) * v3(r10[1], r10[2], r10[3]);
          F.l = F.l - f; F.a = F.a - (t + cross(r, f));
        }
        l_rec_st_pb<C>(w, b, F, true);
      }
    __syncwarp();
    if (w.live)
      for (int b = li; b < nb; b += LM_LPE) {
        S6 F = s6(v3(0.f, 0.f, 0.f), v3(0.f, 0.f, 0.f));
        for (int c = b; c < nb; c++)
          if (l_is_anc(MB[c], b)) F = F + l_rec_ld_pb<C>(w, c);
        st6(gf + 6 * b, F);
      }
    __syncwarp();
  }
  if (!w.live) return;
  if (a.acc || a.jw)
    for (int b = li; b < nb; b += LM_LPE) {
      const V3 x = ld3(sm + C::body + C::BODYW * b + LBR_X);
      float* o;
      if (a.acc) {
        S6 v, ac;
        l_rnep_kin<C>(ms, sm, b, v, ac);
        o = a.acc + (eo * nb + b) * 6;
        st3(o, l_rnep_pacc(v, ac, x)); st3(o + 3, ac.a);
      }
      if (a.jw) {
        const S6 F = ld6(gf + 6 * b);
        o = a.jw + (eo * nb + b) * 6;
        st3(o, F.l); st3(o + 3, F.a - cross(x, F.l));
      }
    }
  const int ns = a.nsite;
  for (int s = li; s < ns; s += LM_LPE) {
    const int b = a.sb[s];
    const Q4 qb = l_rnep_quat<C>(ms, sm, b);
    Q4 qs; qs.w = a.squat[4 * s]; qs.x = a.squat[4 * s + 1]; qs.y = a.squat[4 * s + 2]; qs.z = a.squat[4 * s + 3];
    qs = qnormalize(qmul(qb, qs));
    const V3 x = ld3(sm + C::body + C::BODYW * b + LBR_X) + qrot(qb, v3(a.spos[3 * s], a.spos[3 * s + 1], a.spos[3 * s + 2]));
    const size_t o = (eo * ns + s) * 3;
    if (a.accel || a.gyro) {
      S6 v, ac;
      l_rnep_kin<C>(ms, sm, b, v, ac);
      V3 g;
      if constexpr (C::PRM) g = l_grav<C>(sm);
      else g = v3(H.grav[0], H.grav[1], H.grav[2]);
      if (a.accel) st3(a.accel + o, l_rnep_rotT(qs, l_rnep_pacc(v, ac, x) - g));
      if (a.gyro) st3(a.gyro + o, l_rnep_rotT(qs, v.a));
    }
    if (a.force || a.torque) {
      const S6 F = ld6(gf + 6 * b);
      if (a.force) st3(a.force + o, l_rnep_rotT(qs, F.l));
      if (a.torque) st3(a.torque + o, l_rnep_rotT(qs, F.a - cross(x, F.l)));
    }
  }
}

void lane_rnep_kernels(int cls, void (*k[2])(const float*, int, LRnepArgs)) {
  if (cls == 1) { k[0] = k_rnep5<L_SMPL(0)>; k[1] = k_rnep5<L_SMPL(0)::WithPrm>; }
  else { k[0] = k_rnep5<L_SMPLX(0)>; k[1] = k_rnep5<L_SMPLX(0)::WithPrm>; }
}
