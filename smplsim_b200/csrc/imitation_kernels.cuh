// imitation_kernels.cuh -- the motion-imitation task (smplsim_imitation): tracking observation, reward, early termination, truncation
// and the mean per-joint position error of every env against its motion-library clip, in one launch after the step (or reset) kernel.
// The definitions are stated in include/smplsim.h; the reference ships no imitation task in its MuJoCo env layer, so they are this
// project's (the published PHC formulation).
//
// A warp per env, lanes over the tracked bodies.  The two reference frames (now: what the reward compares with; next: the target of
// the observation) are read in place from the library's tables, 12 / 16 bytes a lane out of one contiguous row; the simulated body
// state comes from the step kernel's side outputs.  The four means and the maximum are lane partial sums in body-list order followed by
// an xor butterfly: the same order on every run, no atomics.  Options (SmplsimImitationCfg): blended reference states instead of the
// nearest frame, T future targets per observation, and fail-state recovery (instances with REC): far targets pulled in to the root, the
// point-goal reward, the recovery window of the distance termination and the power penalty.
#pragma once
#include "aux_kernels.cuh"

struct ImArgs {
  // motion library (motion_clip, ImRow): per-frame tables [total_frames, nb * {3, 4, 3, 3}] and per-clip rows
  const float *txpos, *txquat, *tvel, *tangvel;
  const float* mlen; const int32_t* nframes; const float* mdt; const int32_t* starts;
  // per env
  const int32_t* ids; const float* t0; const int32_t* progress; const uint8_t* mask;
  const float *xpos, *xquat, *linvel, *angvel;
  const uint8_t* status;
  const float* self_obs;
  float *obs, *reward, *mpjpe;
  uint8_t *terminated, *truncated;
  int32_t* frames;
  float k[4], w[4], term_dist, dt;
  int nmotion, episode_length, n, nb, J, self_dim, self_stride, obs_only;
  unsigned char body[LM_MAXB];
  int T;             // future targets (instances with MULTI only)
  float future_dt;   // seconds between them
};
// fail-state recovery (SmplsimImitationRecovery; read by the instances with REC only).  A kernel parameter of its own, after ImArgs, so
// that ImArgs (which k_track_eval embeds) keeps its layout.
struct ImRec {
  int zof, nu, nv;   // zero_out_far; actuators; dofs (qvel row stride)
  float far, power_k;
  int32_t* recovery; float* goal; const float* qvel; const float* ctrl; float* power;
};

__device__ __forceinline__ Q4 im_conj(Q4 q) { q.x = -q.x; q.y = -q.y; q.z = -q.z; return q; }
__device__ __forceinline__ float im_wsum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(L_FULL, v, o);
  return v;
}

// ImRef reads a body's values from the rows of an ImFrame (aux_kernels.cuh): positions and velocities lerped, rotations slerped (the
// rules of k_motion_blend), or the row as it is.
template <int INTERP>
struct ImRef {
  ImRow r0, r1;
  float b;
  __device__ __forceinline__ ImRef(const ImArgs& a, const ImFrame& f) : r0(a, f.f0), r1(a, INTERP ? f.f1 : f.f0), b(f.b) {}
  __device__ __forceinline__ V3 pos(int j) const { return INTERP ? mb_lerp3(ld3(r0.p + 3 * j), ld3(r1.p + 3 * j), b) : ld3(r0.p + 3 * j); }
  __device__ __forceinline__ V3 vel(int j) const { return INTERP ? mb_lerp3(ld3(r0.v + 3 * j), ld3(r1.v + 3 * j), b) : ld3(r0.v + 3 * j); }
  __device__ __forceinline__ V3 angvel(int j) const { return INTERP ? mb_lerp3(ld3(r0.w + 3 * j), ld3(r1.w + 3 * j), b) : ld3(r0.w + 3 * j); }
  __device__ __forceinline__ Q4 quat(int j) const { return INTERP ? mb_slerp(mb_ldq(r0.q + 4 * j), mb_ldq(r1.q + 4 * j), b) : mb_ldq(r0.q + 4 * j); }
};

// Zero-out-far of one reference pose against the simulated root: P = the reference root, pulled in to far_distance of the simulated
// root when further away; q = the reference root rotation; zero = the pose is more than termination_distance away (every tracked
// body then targets (P, q) with zero velocity differences).  d is the distance before the pull.
struct ImZ { V3 P; Q4 q; bool zero; };
template <int INTERP>
__device__ __forceinline__ ImZ im_zof(const ImRef<INTERP>& r, V3 root, float td, float far) {
  ImZ z;
  const V3 pr = r.pos(0), dd = pr - root;
  const float d = sqrtf(dot(dd, dd));
  z.P = d > far ? root + (far / d) * dd : pr;
  z.q = r.quat(0);
  z.zero = d > td;
  return z;
}

// INTERP: blended reference poses; MULTI: a.T future targets (else one); REC: fail-state recovery (rc.zof, rc.recovery, rc.goal,
// power).  MULTI is a template flag: with the loop count read at run time, the one-target instances become the MULTI ones (<0, 0, 0>:
// 64 registers and 16 B stack instead of 60 and none), 2 - 3 % slower, and the recovery reward changes in the last bits.
template <int INTERP, int MULTI, int REC>
__device__ __forceinline__ void im_task(const float* __restrict__ gimg, const ImArgs& a, const ImRec& rc) {
  const LHdr& H = *(const LHdr*)gimg;   // the heading rule (upright_start) is the same for every body shape of a handle
  const int lane = threadIdx.x & 31;
  const int e = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (e >= a.n || (a.mask && !a.mask[e])) return;   // warp-uniform
  const int nb = a.nb, J = a.J, T = MULTI ? a.T : 1;
  const int id = motion_clip(a, a.ids[e]);
  const float len = a.mlen[id], mdt = a.mdt[id], t0 = a.t0[e];
  const int nf = a.nframes[id], start = a.starts[id], p = a.progress[e];
  // one rounding per time: t0 + k dt as a fused multiply-add
  const float t_now = fmaf((float)p, a.dt, t0), t_next = fmaf((float)(p + 1), a.dt, t0);
  const ImFrame f_now = im_frame<INTERP>(len, mdt, nf, start, t_now), f_next = im_frame<INTERP>(len, mdt, nf, start, t_next);
  if (lane == 0 && a.frames) { a.frames[2 * e] = (int32_t)f_now.f0; a.frames[2 * e + 1] = (int32_t)f_next.f0; }
  const float *xp = a.xpos + (size_t)e * nb * 3, *xq = a.xquat + (size_t)e * nb * 4;
  const float *lv = a.linvel + (size_t)e * nb * 3, *av = a.angvel + (size_t)e * nb * 3;
  float* out = a.obs + (size_t)e * (a.self_dim + 24 * J * T);
  {
    const float* so = a.self_obs + (size_t)e * a.self_stride;
    for (int i = lane; i < a.self_dim; i += 32) out[i] = so[i];
  }
  const bool zof = REC && rc.zof;
  ImZ zn;             // zero-out-far of the reward's now-frame
  float g = 0.f;      // point-goal distance: xy from the simulated root to the unmodified reference root of the now-frame
  {
    const Q4 hq = l_heading_inv(H, mb_ldq(xq)), hc = im_conj(hq);
    const V3 root = ld3(xp);
    if (REC) {
      const ImRef<INTERP> now(a, f_now);
      zn = im_zof(now, root, a.term_dist, rc.far);
      const V3 dg = now.pos(0) - root;
      g = sqrtf(fmaf(dg.x, dg.x, dg.y * dg.y));
    }
    for (int k = 0; k < T; k++) {   // target k at t_next + k future_dt (one fused multiply-add), frame-major blocks of 24 J
      const ImRef<INTERP> r(a, (MULTI && k > 0) ? im_frame<INTERP>(len, mdt, nf, start, fmaf((float)k, a.future_dt, t_next)) : f_next);
      ImZ z;
      if (zof) z = im_zof(r, root, a.term_dist, rc.far);
      float* o = out + a.self_dim + 24 * J * k;
      for (int j = lane; j < J; j += 32) {
        const int b = a.body[j];
        const bool zb = zof && z.zero;
        const V3 pr = (zof && (z.zero || b == 0)) ? z.P : r.pos(b);
        const Q4 qr = zb ? z.q : r.quat(b), hr = qmul(hq, qr);
        st3(o + 3 * j, qrot_ref(hq, pr - ld3(xp + 3 * b)));
        st_tan_norm(o + 3 * J + 6 * j, qmul(qmul(hr, im_conj(mb_ldq(xq + 4 * b))), hc));
        st3(o + 9 * J + 3 * j, zb ? v3(0.f, 0.f, 0.f) : qrot_ref(hq, r.vel(b) - ld3(lv + 3 * b)));
        st3(o + 12 * J + 3 * j, zb ? v3(0.f, 0.f, 0.f) : qrot_ref(hq, r.angvel(b) - ld3(av + 3 * b)));
        st3(o + 15 * J + 3 * j, qrot_ref(hq, pr - root));
        st_tan_norm(o + 18 * J + 6 * j, hr);
      }
    }
  }
  if (a.obs_only) {
    if (REC && rc.goal && lane == 0) rc.goal[e] = g;
    return;
  }
  const ImRef<INTERP> now(a, f_now);
  float sp = 0.f, sr = 0.f, sv = 0.f, sw = 0.f, sd = 0.f, md = 0.f;
  for (int j = lane; j < J; j += 32) {
    const int b = a.body[j];
    V3 dp = now.pos(b) - ld3(xp + 3 * b), dv = now.vel(b) - ld3(lv + 3 * b), dw = now.angvel(b) - ld3(av + 3 * b);
    Q4 dq = qmul(now.quat(b), im_conj(mb_ldq(xq + 4 * b)));
    const float d = sqrtf(dot(dp, dp));              // mpjpe and the termination distance: the unmodified reference
    if (zof) {                                       // the reward: the zeroed-out now-frame
      if (zn.zero || b == 0) dp = zn.P - ld3(xp + 3 * b);
      if (zn.zero) { dv = dw = v3(0.f, 0.f, 0.f); dq = qmul(zn.q, im_conj(mb_ldq(xq + 4 * b))); }
    }
    const float d2 = dot(dp, dp);
    const float th = 2.0f * atan2f(sqrtf(dq.x * dq.x + dq.y * dq.y + dq.z * dq.z), fabsf(dq.w));
    sp += d2; sd += d; md = fmaxf(md, d);
    sr += th * th; sv += dot(dv, dv); sw += dot(dw, dw);
  }
  sp = im_wsum(sp); sr = im_wsum(sr); sv = im_wsum(sv); sw = im_wsum(sw); sd = im_wsum(sd);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) md = fmaxf(md, __shfl_xor_sync(L_FULL, md, o));
  float pw = 0.f;     // power: sum over the actuators of |ctrl qvel|, in actuator order
  if (REC && (rc.power || rc.power_k > 0.f)) {
    const float *c = rc.ctrl + (size_t)e * rc.nu, *v = rc.qvel + (size_t)e * rc.nv + 6;
    for (int j = lane; j < rc.nu; j += 32) pw += fabsf(c[j] * v[j]);
    pw = im_wsum(pw);
  }
  if (lane == 0) {
    const float inv = 1.0f / (float)J;
    float rew = a.w[0] * expf(-a.k[0] * (sp * inv)) + a.w[1] * expf(-a.k[1] * (sr * inv)) + a.w[2] * expf(-a.k[2] * (sv * inv)) +
                a.w[3] * expf(-a.k[3] * (sw * inv));
    if (REC) {
      if (zof && zn.zero) rew = fminf(fmaxf((rc.goal[e] - g) / a.dt, 0.f), 1.f);   // off the clip: walk back to its root
      if (rc.power_k > 0.f && p > 3) rew -= rc.power_k * pw;
      if (rc.power) rc.power[e] = pw;
      if (rc.goal) rc.goal[e] = g;
    }
    a.reward[e] = rew;
    a.mpjpe[e] = sd * inv;
    const bool bad = a.status && (a.status[e] & 7);   // the stepper put this env back to qpos0 (mj_checkPos / Vel / Acc): off its clip
    bool far = p > 1 && md > a.term_dist;
    if (REC && rc.recovery) {                         // the recovery window: no distance termination
      const int32_t left = rc.recovery[e];
      if (left > 0) { far = false; rc.recovery[e] = left - 1; }
    }
    a.terminated[e] = (far || bad) ? 1 : 0;
    a.truncated[e] = (t_next > len || p > a.episode_length) ? 1 : 0;
  }
}

// A wrapper, not the body itself: with im_task's code written in the kernel, nvcc fuses one sum of squares of <0, 0, 1> in the other
// order and its reward changes in the last bits.
template <int INTERP, int MULTI, int REC>
__global__ void __launch_bounds__(256) k_imitation(const float* __restrict__ gimg, ImArgs a, ImRec rc) {
  im_task<INTERP, MULTI, REC>(gimg, a, rc);
}
