// inverse_fd_kernels.cu -- k_invfd5, the column kernel of smplsim_inverse_fd (semantics in lane_kernels.cuh above LInvFdArgs, DESIGN.md 2).
// A translation unit of its own, compiled into libsmplsim_b200.so beside smplsim_capi.cu as rollout_kernels.cu is: its noinline callees
// (l_sweep_out, l_inv_acc, l_rows, l_inv_force, l_active_sig) are then instances of this device module, and the kernels of
// smplsim_capi.cu compile exactly as they do without it.  smplsim_capi.cu takes the instances from lane_invfd_kernels (at the end).
// The host emulator compiles everything as one unit (smplsim_capi.cu includes this file under SMPLSIM_EMU).
#include <cuda_runtime.h>

#include <cmath>
#include <cstring>

// lane_kernels.cuh defines two functions that are not templates (l_impedance, k_zero_wrench); smplsim_capi.cu and rollout_kernels.cu
// define them as well, so this unit's copies take names of their own
#define l_impedance l_invfd_impedance
#define k_zero_wrench k_invfd_zero_wrench
#include "lane_kernels.cuh"
#undef l_impedance
#undef k_zero_wrench

// the perturbed input of column col at sign sg (0: the nominal): a qpos entry of the root translation or a hinge, a qvel or a qacc
// entry; for a root-rotation column the angle sg eps of q (x) exp(sg eps e_k)
__device__ __forceinline__ float l_ifd_value(const LInvFdArgs& a, int nv, size_t row, int col, float sg) {
  if (col < nv) return (col >= 3 && col < 6) ? sg * a.eps[0] : a.qpos[row * (nv + 1) + (col < 3 ? col : col + 1)] + sg * a.eps[0];
  if (col < 2 * nv) return a.qvel[row * nv + col - nv] + sg * a.eps[1];
  return a.qacc[row * nv + col - 2 * nv] + sg * a.eps[2];
}

// any entry of the env's n words at p non-finite or beyond mjMAXVAL (mj_checkPos / Vel / Acc's test), on every lane of the env
template <class C>
__device__ __forceinline__ bool l_ifd_bad(const float* p, int n, const LLane& w) {
  bool b = false;
  if (w.live) for (int i = w.li; i < n; i += LM_LPE) b |= !(fabsf(p[i]) <= L_MAXVAL);
  return l_gany(b, w);
}

// one inverse pass of the slot's row with column col's perturbation at sign sg: the row (qpos, qvel, qacc) into shared memory, the
// perturbation (the root rotation as l_fd_load applies it), then k_inverse5's pass -- S1 with collisions, the body accelerations and
// row residuals, the working set := (rs < 0) of every row, the inward force sweep -- leaving qfrc_inverse in the qvel row.  Returns
// L_FD_SOLVER when the pass dropped joint-limit rows or saw a non-finite value in its inputs or its result.
template <class C>
__device__ __noinline__ int l_ifd_pass(const float* ms, float* sm, const LLane& w, const LInvFdArgs& a, size_t row, int col, float sg) {
  const LHdr& H = l_hdr<C>(ms);
  const int nv = H.nv;
  if (w.live && w.li == 0) { ((int*)sm)[C::misc + LMI_NSELF] = 0; ((int*)sm)[C::misc + LMI_NCON] = 0; ((int*)sm)[C::misc + LMI_NLIM] = 0; }
  if (w.live) for (int i = w.li; i < (H.nslot + 3) / 4; i += LM_LPE) ((int*)sm)[C::pfl + i] = 0;
  l_copy_in<C>(sm + C::qpos, a.qpos + row * (nv + 1), nv + 1, w);
  l_copy_in<C>(sm + C::qvel, a.qvel + row * nv, nv, w);
  l_copy_in<C>(sm + C::qacc, a.qacc + row * nv, nv, w);
  __syncwarp();
  if (w.live && w.li == 0) {
    const float x = l_ifd_value(a, nv, row, col, sg);
    if (col >= 3 && col < 6) {   // q (x) exp(x e_k), normalised
      float* qp = sm + C::qpos + 3;
      float sn, cs;
      l_sincos(0.5f * x, &sn, &cs);
      Q4 q; q.w = qp[0]; q.x = qp[1]; q.y = qp[2]; q.z = qp[3];
      Q4 d; d.w = cs; d.x = col == 3 ? sn : 0.f; d.y = col == 4 ? sn : 0.f; d.z = col == 5 ? sn : 0.f;
      q = qnormalize(qmul(q, d));
      qp[0] = q.w; qp[1] = q.x; qp[2] = q.y; qp[3] = q.z;
    } else if (col < nv) sm[C::qpos + (col < 3 ? col : col + 1)] = x;
    else if (col < 2 * nv) sm[C::qvel + col - nv] = x;
    else sm[C::qacc + col - 2 * nv] = x;
  }
  __syncwarp();
  bool bad = l_ifd_bad<C>(sm + C::qpos, nv + 1, w) | l_ifd_bad<C>(sm + C::qvel, nv, w) | l_ifd_bad<C>(sm + C::qacc, nv, w);
  const LFkOut fk = l_sweep_out<C>(ms, sm, w, LF_FK | LF_VEL | LF_COLLIDE, false);
  l_inv_acc<C>(ms, sm, w);
  float o4[5];
  l_rows<C>(sm, w, w.live, 0, 0.f, o4);   // working set := (rs < 0) of every row, as k_inverse5
  __syncwarp();
  l_inv_force<C>(ms, sm, w);
  bad = bad | l_ifd_bad<C>(sm + C::qvel, nv, w);
  return (bad || fk.dropped) ? L_FD_SOLVER : 0;
}

// Slot s of the launch: row s / 3nv, column s % 3nv.  The pass at x + eps (centered: parked in gfd) and the pass at x - eps (or the
// nominal qfrc_inverse), then column col of dfrc, divided by the fp32 difference of the inputs the passes loaded.  The row set's
// signature is l_active_sig's: l_rows (op 0) writes the working-set bits 1-4 of every present contact entry and bit 0 of every
// joint-limit row's flag, which are the bits it reads beside the entries' presence, slot, dof and side.
template <class C>
__global__ void __launch_bounds__(256, 1) k_invfd5(const float* __restrict__ gimg, int img_bytes, LInvFdArgs a) {
  const float* ms; LLane w;
  float* sm = l_setup<C>(gimg, img_bytes, w, ms, a.n, a.map, a.gscr, nullptr, nullptr);
  const LHdr& H = l_hdr<C>(ms);
  const int nv = H.nv, ncol = 3 * nv;
  const size_t eo = w.live ? (size_t)w.env : 0;
  const long long s = a.s0 + (long long)eo;
  const size_t row = (size_t)(s / ncol);
  const int col = (int)(s % ncol);
  unsigned sig0 = 0u;
  int flag = 0;
  for (int p = 0; p <= (a.centered ? 1 : 0); p++) {
    flag |= l_ifd_pass<C>(ms, sm, w, a, row, col, p ? -1.f : 1.f);
    const unsigned sig = l_active_sig<C>(sm, w);
    if (p == 0 && a.centered) {
      sig0 = sig;
      l_copy_out<C>(a.gfd + eo * nv, sm + C::qvel, nv, w);
      __syncwarp();
    } else if (p == 1 && sig != sig0) flag |= L_FD_KINK;
  }
  if (!w.live) return;
  const float den = l_ifd_value(a, nv, row, col, 1.f) - l_ifd_value(a, nv, row, col, a.centered ? -1.f : 0.f);
  const float* fp = a.centered ? a.gfd + eo * nv : sm + C::qvel;
  const float* fm = a.centered ? sm + C::qvel : a.qfrc + row * nv;
  for (int i = w.li; i < nv; i += LM_LPE) {
    const float d = l_div_rn(fp[i] - fm[i], den);
    if (a.dfrc) a.dfrc[(row * nv + i) * ncol + col] = d;
  }
  if (a.flags && w.li == 0) a.flags[row * ncol + col] = (uint8_t)flag;
}

void lane_invfd_kernels(int cls, void (**k)(const float*, int, LInvFdArgs)) {
  *k = cls == 1 ? k_invfd5<L_SMPL(0)> : k_invfd5<L_SMPLX(0)>;
}
