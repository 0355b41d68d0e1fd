// rollout_step.cuh -- l_roll_step, one step of a rollout row, shared by the rollout kernels.
// Included by rollout_kernels.cu (k_roll5) and rollout_feedback_kernels.cu (k_rollfb5), each a device module of its own, after
// lane_kernels.cuh.
#pragma once

// step t of the slot's row: control row t through l_substeps (behind l_spd_prologue at a stable-PD call boundary), then the state,
// the status and, when asked, the poses of step t.  A function of its own so that the kernel keeps few registers live across steps.
template <class C>
__device__ __noinline__ void l_roll_step(const float* ms, float* sm, const LLane& w, const LRollArgs& a, int t) {
  const LHdr& H = l_hdr<C>(ms);
  const size_t eo = w.live ? (size_t)w.env : 0, ro = eo * (size_t)a.nstep + t;   // row of step t in the [n, nstep, ...] tensors
  const int nq = H.nv + 1, nv = H.nv, nu = H.nu;
  const bool stale = a.mode == 0 && H.cfg.control_mode == SMPLSIM_CTRL_UHC_PD && H.cfg.spd_stale;
  LSolveLane st; st.dirty_bits = 0u; st.rc_bits = 0u;
  if (w.live && w.li == 0) { sm[C::misc + LMI_DISP] = 0.f; sm[C::misc + LMI_DISP + 1] = 0.f; ((int*)sm)[C::misc + LMI_NSELF] = 0; ((int*)sm)[C::misc + LMI_NCON] = 0; ((int*)sm)[C::misc + LMI_NLIM] = 0; }
  l_copy_in<C>(sm + C::act, a.control + ro * nu, nu, w);
  if (a.mode != 0) l_copy_in<C>(sm + C::tau, a.control + ro * nu, nu, w);   // raw ctrl (act keeps a copy for the substep after an auto-reset)
  if (stale) {   // a call boundary: the prologue reloads the state from the scratch rows after its sweep at the forward-pass state
    l_copy_out<C>(a.scr.qpos + eo * nq, sm + C::qpos, nq, w);
    l_copy_out<C>(a.scr.qvel + eo * nv, sm + C::qvel, nv, w);
    __syncwarp();
    l_spd_prologue<C>(ms, sm, w, a.scr, st);
  }
  __syncwarp();
  LFwd fo; fo.mask = 0ull; fo.iters = 0; fo.status = 0;
  l_substeps<C>(ms, sm, w, a.nsub, a.mode, &fo, a.scr, stale, false, st);
  // k_step5 ends every call with the final kinematics sweep, which normalises the root quaternion in qpos (l_root_out): the same
  // normalisation here with or without the pose output, so that asking for poses changes no bit of the trajectory
  if (a.xpos) l_sweep_out<C>(ms, sm, w, LF_FK | LF_XQUAT, false);
  else {
    if (w.live && w.li == 0) {
      float* qr = sm + C::qpos + 3;
      Q4 q; q.w = qr[0]; q.x = qr[1]; q.y = qr[2]; q.z = qr[3];
      q = qnormalize(q);
      qr[0] = q.w; qr[1] = q.x; qr[2] = q.y; qr[3] = q.z;
    }
    __syncwarp();
  }
  l_copy_out<C>(a.qpos + ro * nq, sm + C::qpos, nq, w);
  l_copy_out<C>(a.qvel + ro * nv, sm + C::qvel, nv, w);
  if (w.live) {
    if (a.xpos) {
      const V3 root = ld3(sm + C::qpos);
      for (int b = w.li; b < H.nb; b += LM_LPE) st3(a.xpos + (ro * H.nb + b) * 3, ld3(sm + C::body + C::BODYW * b + LBR_X) + root);
      l_copy<C>(a.xquat + ro * H.nb * 4, sm + C::xq, 4 * H.nb, w);
    }
    if (a.status && w.li == 0) a.status[ro] = (uint8_t)fo.status;
  }
  __syncwarp();
}
