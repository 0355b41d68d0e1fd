// centroidal_kernels.cu -- k_cent5, the kernel of smplsim_centroidal (semantics in lane_kernels.cuh above LCentArgs, DESIGN.md 2).
// A translation unit of its own, compiled into libsmplsim_b200.so beside smplsim_capi.cu as rollout_kernels.cu is: its noinline callees
// (l_sweep_out, l_crb_in) are then instances of this device module, and the kernels of smplsim_capi.cu compile exactly as they do without
// it.  smplsim_capi.cu takes the instances from lane_cent_kernels (at the end).
// The host emulator compiles everything as one unit (smplsim_capi.cu includes this file under SMPLSIM_EMU).
#include <cuda_runtime.h>

#include <cmath>
#include <cstring>

// lane_kernels.cuh defines two functions that are not templates (l_impedance, k_zero_wrench); smplsim_capi.cu and the other kernel
// modules define them as well, so this unit's copies take names of their own
#define l_impedance l_cent_impedance
#define k_zero_wrench k_cent_zero_wrench
#include "lane_kernels.cuh"
#undef l_impedance
#undef k_zero_wrench

// Per-body words in the env's global scratch, in the overflow contact entries (unused: S1 runs without LF_COLLIDE): body b's own
// [m, m r (3), I_b v_b (6)] at LCT_OWN, the same summed over b's subtree at LCT_SUB.  Positions are relative to the root origin, world axes.
#define LCT_W 10
template <class C> __device__ __forceinline__ float* l_cent_own(const LLane& w, int b) { return w.gscr + C::gcon + LCT_W * b; }
template <class C> __device__ __forceinline__ float* l_cent_sub(const LLane& w, int b) { return w.gscr + C::gcon + LCT_W * (C::NB + b); }

// spatial velocity of body b about the root origin: the motion subspaces of the dofs on its path to the root, times qvel
template <class C>
__device__ __forceinline__ S6 l_cent_vel(const float* ms, const float* sm, int b) {
  const LBody* MB = l_bodies(ms);
  const float* qv = sm + C::qvel;
  S6 v = s6(v3(0.f, 0.f, 0.f), v3(0.f, 0.f, 0.f));
  for (int e = b; e > 0; e = MB[e].parent) {
    const float* br = sm + C::body + C::BODYW * e;
    const int d0 = MB[e].dofadr;
#pragma unroll
    for (int k = 0; k < 3; k++) v = v + qv[d0 + k] * l_hingeS(br, k);
  }
  const V3 c0 = ld3(sm + C::body + LBR_AX), c1 = ld3(sm + C::body + LBR_AX + 3), c2 = ld3(sm + C::body + LBR_AX + 6);
  return v + s6(qv[3] * c0 + qv[4] * c1 + qv[5] * c2, ld3(qv));
}

// centre of mass of a subtree's words (relative to the root origin)
__device__ __forceinline__ V3 l_cent_com(const float* s) { return (1.f / s[0]) * v3(s[1], s[2], s[3]); }

// Row of the launch: S1 (kinematics, velocities, rigid inertias, bias forces pb into the lane records) at (qpos, qvel), then
//   own words of every body (lanes over bodies), subtree sums (lanes over bodies; every descendant of b has a larger index),
//   subtree_com / linvel / angmom (lanes over bodies), cmm from l_crb_in's f_d = Ic S_d (lanes over dofs), jac_com (lanes over dofs),
//   cmm_bias on lane 0: the RNE's root wrench at qacc = 0 is the sum of every body's pb = I a_b + v_b x* I v_b (gravity enters as the
//   root's bias acceleration -g, so pb carries it), and I_tot [0 ; g] = [h x g ; m g] takes it back out.
template <class C>
__global__ void __launch_bounds__(256, 1) k_cent5(const float* __restrict__ gimg, int img_bytes, LCentArgs a) {
  static_assert(2 * LCT_W * C::NB <= C::CONW * (C::NS - C::NCS), "the centroidal scratch does not fit the overflow contact entries");
  const float* ms; LLane w;
  float* sm = l_setup<C>(gimg, img_bytes, w, ms, a.n, a.map, a.gscr, nullptr, nullptr);
  const LHdr& H = l_hdr<C>(ms);
  const LBody* MB = l_bodies(ms);
  const size_t eo = w.live ? (size_t)w.env : 0;
  const int nb = H.nb, nv = H.nv, li = w.li;
  if constexpr (C::PRM) l_prm_stage<C>(ms, sm, w);
  l_copy_in<C>(sm + C::qpos, a.qpos + eo * (nv + 1), nv + 1, w);
  if (a.qvel) l_copy_in<C>(sm + C::qvel, a.qvel + eo * nv, nv, w);
  else if (w.live) for (int i = li; i < nv; i += LM_LPE) sm[C::qvel + i] = 0.f;
  if (w.live) for (int i = li; i < nv; i += LM_LPE) sm[C::qacc + i] = 0.f;
  __syncwarp();
  l_sweep_out<C>(ms, sm, w, LF_FK | LF_VEL, false);
  if (a.cmm) l_crb_in<C>(ms, sm, w);
  const bool mom = a.linvel || a.angmom;
  const int nw = mom ? LCT_W : 4;
  if (w.live)
    for (int b = li; b < nb; b += LM_LPE) {
      float r10[10];
      l_ld_r10(sm + C::body + C::BODYW * b, r10);
      float* o = l_cent_own<C>(w, b);
      o[0] = r10[0]; o[1] = r10[1]; o[2] = r10[2]; o[3] = r10[3];
      if (mom) l_s6arr(rb_mul(r10, l_cent_vel<C>(ms, sm, b)), o + 4);
    }
  __syncwarp();
  if (w.live)
    for (int b = li; b < nb; b += LM_LPE) {
      float s[LCT_W];
      for (int j = 0; j < LCT_W; j++) s[j] = 0.f;
      for (int c = b; c < nb; c++) {
        if (!l_is_anc(MB[c], b)) continue;
        const float* o = l_cent_own<C>(w, c);
        for (int j = 0; j < nw; j++) s[j] += o[j];
      }
      float* o = l_cent_sub<C>(w, b);
      for (int j = 0; j < nw; j++) o[j] = s[j];
    }
  __syncwarp();
  if (!w.live) return;
  const float* s0 = l_cent_sub<C>(w, 0);
  const V3 com0 = l_cent_com(s0);
  if (a.com || mom)
    for (int b = li; b < nb; b += LM_LPE) {
      const float* s = l_cent_sub<C>(w, b);
      const V3 cb = l_cent_com(s);
      const size_t o = (eo * nb + b) * 3;
      if (a.com) st3(a.com + o, cb + ld3(sm + C::qpos));
      const S6 p = l_arr6(s + 4);
      if (a.linvel) st3(a.linvel + o, (1.f / s[0]) * p.l);
      if (a.angmom) st3(a.angmom + o, p.a - cross(cb, p.l));
    }
  if (a.cmm) {
    float* o = a.cmm + eo * 6 * nv;
    for (int d = li; d < nv; d += LM_LPE) {
      const S6 f = ld6(l_dof_fp<C>(sm, w, d));
      const V3 t = f.a - cross(com0, f.l);
      o[d] = f.l.x; o[nv + d] = f.l.y; o[2 * nv + d] = f.l.z; o[3 * nv + d] = t.x; o[4 * nv + d] = t.y; o[5 * nv + d] = t.z;
    }
  }
  for (int j = 0; j < a.njac; j++) {
    const int p = a.jb[j];
    const float* sp = l_cent_sub<C>(w, p);
    const V3 cp = l_cent_com(sp);
    float* o = a.jac + (eo * a.njac + j) * 3 * nv;
    for (int d = li; d < nv; d += LM_LPE) {
      const int e = l_dof_body(d);
      V3 jp = v3(0.f, 0.f, 0.f);
      if (l_is_anc(MB[p], e)) {   // the dof moves the whole subtree of p: the velocity of p's centre of mass
        const S6 S = l_dof_S<C>(sm, d);
        jp = S.l + cross(S.a, cp);
      } else if (l_is_anc(MB[e], p)) {   // the dof moves e's subtree only: its centre-of-mass velocity, weighted by its share of p's mass
        const S6 S = l_dof_S<C>(sm, d);
        const float* se = l_cent_sub<C>(w, e);
        jp = (se[0] * (1.f / sp[0])) * (S.l + cross(S.a, l_cent_com(se)));
      }
      o[d] = jp.x; o[nv + d] = jp.y; o[2 * nv + d] = jp.z;
    }
  }
  if (a.cbias && li == 0) {
    S6 F = s6(v3(0.f, 0.f, 0.f), v3(0.f, 0.f, 0.f));
    for (int b = 0; b < nb; b++) F = F + l_rec_ld_pb<C>(w, b);
    V3 g;
    if constexpr (C::PRM) g = l_grav<C>(sm);
    else g = v3(H.grav[0], H.grav[1], H.grav[2]);
    F.a = F.a + cross(v3(s0[1], s0[2], s0[3]), g);
    F.l = F.l + s0[0] * g;
    const V3 t = F.a - cross(com0, F.l);
    float* o = a.cbias + eo * 6;
    o[0] = F.l.x; o[1] = F.l.y; o[2] = F.l.z; o[3] = t.x; o[4] = t.y; o[5] = t.z;
  }
}

void lane_cent_kernels(int cls, int selfcol, void (*k[2])(const float*, int, LCentArgs)) {
  if (cls == 1 && !selfcol) { k[0] = k_cent5<L_SMPL(0)>; k[1] = k_cent5<L_SMPL(0)::WithPrm>; }
  else if (cls == 1) { k[0] = k_cent5<L_SMPL(1)>; k[1] = k_cent5<L_SMPL(1)::WithPrm>; }
  else if (!selfcol) { k[0] = k_cent5<L_SMPLX(0)>; k[1] = k_cent5<L_SMPLX(0)::WithPrm>; }
  else { k[0] = k_cent5<L_SMPLX(1)>; k[1] = k_cent5<L_SMPLX(1)::WithPrm>; }
}
