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

// any entry of the env's n words at p non-finite or beyond mjMAXVAL (mj_checkPos / Vel / Acc's test), on every lane of the env
template <class C>
__device__ __forceinline__ bool l_ifd_bad(const float* p, int n, const LLane& w) {
  bool b = false;
  if (w.live) for (int i = w.li; i < n; i += LM_LPE) b |= !(fabsf(p[i]) <= L_MAXVAL);
  return l_gany(b, w);
}

// one inverse pass (l_inv_pass) of the slot's rows with column col's perturbation at sign sg, leaving qfrc_inverse in the qvel row.
// Returns L_FD_SOLVER when the pass dropped joint-limit rows or saw a non-finite value in its inputs or its result.
template <class C>
__device__ __noinline__ int l_ifd_pass(const float* ms, float* sm, const LLane& w, const LFdCols& f, const float* qpos, const float* qvel,
                                       const float* qacc, int col, float sg) {
  const int nv = l_hdr<C>(ms).nv;
  bool bad = false;
  float o4[5];
  const LFkOut fk = l_inv_pass<C>(ms, sm, w, o4, [&] {
    l_copy_in<C>(sm + C::qpos, qpos, nv + 1, w);
    l_copy_in<C>(sm + C::qvel, qvel, nv, w);
    l_copy_in<C>(sm + C::qacc, qacc, nv, w);
    l_fd_perturb<C>(sm, w, f, nv, qpos, qvel, qacc, C::qacc, col, sg);
    bad = l_ifd_bad<C>(sm + C::qpos, nv + 1, w) | l_ifd_bad<C>(sm + C::qvel, nv, w) | l_ifd_bad<C>(sm + C::qacc, nv, w);
  });
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
  const int nv = l_hdr<C>(ms).nv, ncol = a.fd.ncol;
  const size_t eo = w.live ? (size_t)w.env : 0;
  const long long s = a.fd.s0 + (long long)eo;
  const size_t row = (size_t)(s / ncol);
  const int col = (int)(s % ncol);
  const float *qpos = a.qpos + row * (nv + 1), *qvel = a.qvel + row * nv, *qacc = a.qacc + row * nv;
  unsigned sig0 = 0u;
  int flag = 0;
  for (int p = 0; p <= (a.fd.centered ? 1 : 0); p++) {
    flag |= l_ifd_pass<C>(ms, sm, w, a.fd, qpos, qvel, qacc, col, p ? -1.f : 1.f);
    const unsigned sig = l_active_sig<C>(sm, w);
    if (p == 0 && a.fd.centered) {
      sig0 = sig;
      l_copy_out<C>(a.fd.gfd + eo * C::NV, sm + C::qvel, nv, w);
      __syncwarp();
    } else if (p == 1 && sig != sig0) flag |= L_FD_KINK;
  }
  if (!w.live) return;
  const float den = l_fd_den(a.fd, qpos, qvel, qacc, nv, col);
  const float* fp = a.fd.centered ? a.fd.gfd + eo * C::NV : sm + C::qvel;
  const float* fm = a.fd.centered ? sm + C::qvel : a.qfrc + row * nv;
  for (int i = w.li; i < nv; i += LM_LPE) {
    const float d = l_div_rn(fp[i] - fm[i], den);
    if (a.dfrc) a.dfrc[(row * nv + i) * ncol + col] = d;
  }
  if (a.fd.flags && w.li == 0) a.fd.flags[row * ncol + col] = (uint8_t)flag;
}

void lane_invfd_kernels(int cls, void (**k)(const float*, int, LInvFdArgs)) {
  *k = cls == 1 ? k_invfd5<L_SMPL(0)> : k_invfd5<L_SMPLX(0)>;
}
