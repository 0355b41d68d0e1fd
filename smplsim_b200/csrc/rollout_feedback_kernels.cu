// rollout_feedback_kernels.cu -- k_rollfb5, the kernel of smplsim_rollout_feedback (semantics in smplsim.h and in lane_kernels.cuh
// above LRollFbArgs, DESIGN.md 2): k_roll5's steps (rollout_step.cuh) with the control row of each step computed from the row's state.
// A translation unit of its own, as rollout_kernels.cu is: added to that module, its callers of the noinline functions changed the
// SASS of k_roll5's callees.  The host emulator compiles everything as one unit (smplsim_capi.cu includes this file under SMPLSIM_EMU).
#include <cuda_runtime.h>

#include <cmath>
#include <cstring>

// lane_kernels.cuh defines two functions that are not templates (l_impedance, k_zero_wrench); smplsim_capi.cu and the other kernel
// units define them as well, so this unit's copies take names of their own
#define l_impedance l_rollfb_impedance
#define k_zero_wrench k_rollfb_zero_wrench
#include "lane_kernels.cuh"
#undef l_impedance
#undef k_zero_wrench
#include "rollout_step.cuh"

// the start of a row (table, parameter records, empty working-set memory, start state, warm start, the forward-pass state before
// step 0): what k_roll5 does before its first step (written out there, so that k_roll5's SASS stays as it was)
template <class C>
__device__ __forceinline__ float* l_roll_start(const float* gimg, int img_bytes, const LRollArgs& a, LLane& w, const float*& ms) {
  float* sm = l_setup<C>(gimg, img_bytes, w, ms, a.n, a.map, a.gscr, nullptr, nullptr);
  const LHdr& H = l_hdr<C>(ms);
  const size_t eo = w.live ? (size_t)w.env : 0;
  const int nq = H.nv + 1, nv = H.nv;
  if constexpr (C::PRM) l_prm_stage<C>(ms, sm, w);
  if (w.live) for (int i = w.li; i < (H.nslot + 3) / 4; i += LM_LPE) ((int*)sm)[C::pfl + i] = 0;   // empty working-set memory
  l_copy_in<C>(sm + C::qpos, a.qpos0 + eo * nq, nq, w);
  l_copy_in<C>(sm + C::qvel, a.qvel0 + eo * nv, nv, w);
  if (a.qacc_warm0) l_copy_in<C>(sm + C::qacc, a.qacc_warm0 + eo * nv, nv, w);
  else if (w.live) for (int i = w.li; i < nv; i += LM_LPE) sm[C::qacc + i] = 0.f;
  if (a.mode == 0 && H.cfg.control_mode == SMPLSIM_CTRL_UHC_PD && H.cfg.spd_stale && w.live) {
    // the state of the last forward pass before step 0 (the host passes qpos0 / qvel0 for NULL)
    for (int i = w.li; i < nq; i += LM_LPE) a.scr.qpos_fwd[eo * nq + i] = a.qpos_fwd0[eo * nq + i];
    for (int i = w.li; i < nv; i += LM_LPE) a.scr.qvel_fwd[eo * nv + i] = a.qvel_fwd0[eo * nv + i];
  }
  __syncwarp();
  return sm;
}

// u_t of step t into u[0, nu), from the state the row holds before the step (sm qpos / qvel: the start state, or the output row t - 1).
// It runs before l_roll_step, so before l_spd_prologue moves the shared rows to the forward-pass state.  The 8 lanes of the env write
// dx into the env's scratch row, then lane li takes outputs li, li + 8, ... and streams their gain rows through the read-only path.
template <class C>
__device__ __noinline__ void l_roll_feedback(const float* ms, const float* sm, const LLane& w, const LRollFbArgs& a, int t, float* u) {
  const LHdr& H = l_hdr<C>(ms);
  const int nv = H.nv, nq = nv + 1, nu = H.nu, nx = 2 * nv;
  const size_t eo = w.live ? (size_t)w.env : 0, ro = eo * (size_t)a.r.nstep + t;
  const size_t rr = (a.shared_ref ? 0 : eo) * (size_t)a.r.nstep + t;   // row of step t in the [ref_rows, nstep, ...] tensors
  const float* q = sm + C::qpos; const float* v = sm + C::qvel;
  const float* qr = a.qpos_ref + rr * nq; const float* vr = a.qvel_ref + rr * nv;
  float* dx = a.dx + eo * nx;
  if (w.live) {
    for (int i = w.li; i < nx; i += LM_LPE) {
      if (i < 3) dx[i] = q[i] - qr[i];
      else if (i >= 6 && i < nv) dx[i] = q[i + 1] - qr[i + 1];
      else if (i >= nv) dx[i] = v[i - nv] - vr[i - nv];
    }
    if (w.li == 0) {   // dq[3:6] = log(normalise(qbar)^-1 (x) normalise(q)), on the shortest arc
      Q4 b; b.w = qr[3]; b.x = qr[4]; b.y = qr[5]; b.z = qr[6];
      Q4 c; c.w = q[3]; c.x = q[4]; c.y = q[5]; c.z = q[6];
      b = qnormalize(b); c = qnormalize(c);
      // the vector part pairs the products that cancel when c == b; rounded products and sums so that no FMA leaves a residue there
      float rw = b.w * c.w + b.x * c.x + b.y * c.y + b.z * c.z;
      float rx = __fadd_rn(__fsub_rn(__fmul_rn(b.w, c.x), __fmul_rn(b.x, c.w)), __fsub_rn(__fmul_rn(b.z, c.y), __fmul_rn(b.y, c.z)));
      float ry = __fadd_rn(__fsub_rn(__fmul_rn(b.w, c.y), __fmul_rn(b.y, c.w)), __fsub_rn(__fmul_rn(b.x, c.z), __fmul_rn(b.z, c.x)));
      float rz = __fadd_rn(__fsub_rn(__fmul_rn(b.w, c.z), __fmul_rn(b.z, c.w)), __fsub_rn(__fmul_rn(b.y, c.x), __fmul_rn(b.x, c.y)));
      if (rw < 0.f) { rw = -rw; rx = -rx; ry = -ry; rz = -rz; }
      const float s = sqrtf(rx * rx + ry * ry + rz * rz), f = s > 0.f ? 2.f * atan2f(s, rw) / s : 0.f;
      dx[3] = f * rx; dx[4] = f * ry; dx[5] = f * rz;
    }
  }
  __syncwarp();
  if (w.live) {
    const bool clip = a.clip && a.r.mode == 0;
    for (int i = w.li; i < nu; i += LM_LPE) {
      const float* k = a.gain + (rr * nu + i) * nx;
      float s = a.r.control[ro * nu + i];
      for (int j = 0; j < nx; j++) s = fmaf(__ldg(k + j), dx[j], s);
      if (clip && s == s) s = fminf(fmaxf(s, -1.f), 1.f);   // as torch.clamp, a NaN passes
      u[i] = s;
    }
  }
  __syncwarp();
}

template <class C>
__global__ void __launch_bounds__(256, 1) k_rollfb5(const float* __restrict__ gimg, int img_bytes, LRollFbArgs a) {
  const float* ms; LLane w;
  float* sm = l_roll_start<C>(gimg, img_bytes, a.r, w, ms);
  const size_t eo = w.live ? (size_t)w.env : 0;
  const int nu = l_hdr<C>(ms).nu;
  for (int t = 0; t < a.r.nstep; t++) {
    const size_t ro = eo * (size_t)a.r.nstep + t;
    float* u = a.control_applied ? a.control_applied + ro * nu : a.uscr + eo * nu;
    l_roll_feedback<C>(ms, sm, w, a, t, u);
    // l_roll_step loads its control row from r.control + ro * nu: point that row at u (plain loads, after the __syncwarp above)
    LRollArgs r = a.r; r.control = u - ro * nu;
    l_roll_step<C>(ms, sm, w, r, t);
  }
}

void lane_rollfb_kernels(int cls, void (*k[2])(const float*, int, LRollFbArgs)) {
  if (cls == 1) { k[0] = k_rollfb5<L_SMPL(0)>; k[1] = k_rollfb5<L_SMPL(0)::WithPrm>; }
  else { k[0] = k_rollfb5<L_SMPLX(0)>; k[1] = k_rollfb5<L_SMPLX(0)::WithPrm>; }
}
