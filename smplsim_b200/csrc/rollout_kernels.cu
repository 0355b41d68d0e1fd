// rollout_kernels.cu -- k_roll5, the kernel of smplsim_rollout (semantics in lane_kernels.cuh above LRollArgs, DESIGN.md 2).
// A translation unit of its own, compiled into libsmplsim_b200.so beside smplsim_capi.cu: its noinline callees (l_substeps,
// l_spd_prologue, the sweeps, the solve, the sinf slow path) are then instances of this device module, and the kernels of
// smplsim_capi.cu compile exactly as they do without it.  smplsim_capi.cu takes the instances from lane_roll_kernels (at the end).
// The host emulator compiles everything as one unit (smplsim_capi.cu includes this file under SMPLSIM_EMU).
#include <cuda_runtime.h>

#include <cmath>
#include <cstring>

// lane_kernels.cuh defines two functions that are not templates (l_impedance, k_zero_wrench); smplsim_capi.cu defines them as well,
// so this unit's copies take names of their own
#define l_impedance l_roll_impedance
#define k_zero_wrench k_roll_zero_wrench
#include "lane_kernels.cuh"
#undef l_impedance
#undef k_zero_wrench
#include "rollout_step.cuh"   // l_roll_step

template <class C>
__global__ void __launch_bounds__(256, 1) k_roll5(const float* __restrict__ gimg, int img_bytes, LRollArgs a) {
  const float* ms; LLane w;
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
  for (int t = 0; t < a.nstep; t++) l_roll_step<C>(ms, sm, w, a, t);
}

void lane_roll_kernels(int cls, void (*k[2])(const float*, int, LRollArgs)) {
  if (cls == 1) { k[0] = k_roll5<L_SMPL(0)>; k[1] = k_roll5<L_SMPL(0)::WithPrm>; }
  else { k[0] = k_roll5<L_SMPLX(0)>; k[1] = k_roll5<L_SMPLX(0)::WithPrm>; }
}
