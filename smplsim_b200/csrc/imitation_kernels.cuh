// imitation_kernels.cuh -- the motion-imitation task (smplsim_imitation): tracking observation, reward, early termination, truncation
// and the mean per-joint position error of every env against its motion-library clip, in one launch after the step (or reset) kernel.
// The definitions are stated in include/smplsim.h; the reference ships no imitation task in its MuJoCo env layer, so they are this
// project's (the published PHC formulation).
//
// A warp per env, lanes over the tracked bodies.  The two reference frames (now: what the reward compares with; next: the target of
// the observation) are read in place from the library's tables, 12 / 16 bytes a lane out of one contiguous row; the simulated body
// state comes from the step kernel's side outputs.  The four means and the maximum are lane partial sums in body-list order followed by
// an xor butterfly: the same order on every run, no atomics.
#pragma once
#include "aux_kernels.cuh"

struct ImArgs {
  // motion library: per-frame tables [total_frames, nb * {3, 4, 3, 3}] and per-clip rows
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
};

__device__ __forceinline__ Q4 im_ldq(const float* p) { Q4 q; q.w = p[0]; q.x = p[1]; q.y = p[2]; q.z = p[3]; return q; }
__device__ __forceinline__ Q4 im_conj(Q4 q) { q.x = -q.x; q.y = -q.y; q.z = -q.z; return q; }
__device__ __forceinline__ void im_st6(float* p, Q4 q) {   // six(q), as pack_self_obs
  st3(p, qrot_ref(q, v3(1.f, 0.f, 0.f)));
  st3(p + 3, qrot_ref(q, v3(0.f, 0.f, 1.f)));
}
__device__ __forceinline__ float im_wsum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(L_FULL, v, o);
  return v;
}

__global__ void __launch_bounds__(256) k_imitation(const float* __restrict__ gimg, ImArgs a) {
  const LHdr& H = *(const LHdr*)gimg;   // the heading rule (upright_start) is the same for every body shape of a handle
  const int lane = threadIdx.x & 31;
  const int e = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (e >= a.n || (a.mask && !a.mask[e])) return;   // warp-uniform
  const int nb = a.nb, J = a.J;
  const int id = min(max(a.ids[e], 0), a.nmotion - 1);
  const float len = a.mlen[id], mdt = a.mdt[id], t0 = a.t0[e];
  const int nf = a.nframes[id], start = a.starts[id], p = a.progress[e];
  // one rounding per time: t0 + k dt as a fused multiply-add
  const float t_now = fmaf((float)p, a.dt, t0), t_next = fmaf((float)(p + 1), a.dt, t0);
  const size_t r_now = (size_t)(start + motion_frame(len, mdt, nf, t_now)), r_next = (size_t)(start + motion_frame(len, mdt, nf, t_next));
  if (lane == 0 && a.frames) { a.frames[2 * e] = (int32_t)r_now; a.frames[2 * e + 1] = (int32_t)r_next; }
  const float *xp = a.xpos + (size_t)e * nb * 3, *xq = a.xquat + (size_t)e * nb * 4;
  const float *lv = a.linvel + (size_t)e * nb * 3, *av = a.angvel + (size_t)e * nb * 3;
  float* out = a.obs + (size_t)e * (a.self_dim + 24 * J);
  {
    const float* so = a.self_obs + (size_t)e * a.self_stride;
    for (int i = lane; i < a.self_dim; i += 32) out[i] = so[i];
  }
  {
    const Q4 hq = l_heading_inv(H, im_ldq(xq)), hc = im_conj(hq);
    const V3 root = ld3(xp);
    const float *rp = a.txpos + r_next * nb * 3, *rq = a.txquat + r_next * nb * 4, *rv = a.tvel + r_next * nb * 3, *rw = a.tangvel + r_next * nb * 3;
    float* o = out + a.self_dim;
    for (int j = lane; j < J; j += 32) {
      const int b = a.body[j];
      const V3 pr = ld3(rp + 3 * b);
      const Q4 qr = im_ldq(rq + 4 * b), hr = qmul(hq, qr);
      st3(o + 3 * j, qrot_ref(hq, pr - ld3(xp + 3 * b)));
      im_st6(o + 3 * J + 6 * j, qmul(qmul(hr, im_conj(im_ldq(xq + 4 * b))), hc));
      st3(o + 9 * J + 3 * j, qrot_ref(hq, ld3(rv + 3 * b) - ld3(lv + 3 * b)));
      st3(o + 12 * J + 3 * j, qrot_ref(hq, ld3(rw + 3 * b) - ld3(av + 3 * b)));
      st3(o + 15 * J + 3 * j, qrot_ref(hq, pr - root));
      im_st6(o + 18 * J + 6 * j, hr);
    }
  }
  if (a.obs_only) return;
  const float *rp = a.txpos + r_now * nb * 3, *rq = a.txquat + r_now * nb * 4, *rv = a.tvel + r_now * nb * 3, *rw = a.tangvel + r_now * nb * 3;
  float sp = 0.f, sr = 0.f, sv = 0.f, sw = 0.f, sd = 0.f, md = 0.f;
  for (int j = lane; j < J; j += 32) {
    const int b = a.body[j];
    const V3 dp = ld3(rp + 3 * b) - ld3(xp + 3 * b), dv = ld3(rv + 3 * b) - ld3(lv + 3 * b), dw = ld3(rw + 3 * b) - ld3(av + 3 * b);
    const Q4 dq = qmul(im_ldq(rq + 4 * b), im_conj(im_ldq(xq + 4 * b)));
    const float d2 = dot(dp, dp), d = sqrtf(d2);
    const float th = 2.0f * atan2f(sqrtf(dq.x * dq.x + dq.y * dq.y + dq.z * dq.z), fabsf(dq.w));
    sp += d2; sd += d; md = fmaxf(md, d);
    sr += th * th; sv += dot(dv, dv); sw += dot(dw, dw);
  }
  sp = im_wsum(sp); sr = im_wsum(sr); sv = im_wsum(sv); sw = im_wsum(sw); sd = im_wsum(sd);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) md = fmaxf(md, __shfl_xor_sync(L_FULL, md, o));
  if (lane == 0) {
    const float inv = 1.0f / (float)J;
    a.reward[e] = a.w[0] * expf(-a.k[0] * (sp * inv)) + a.w[1] * expf(-a.k[1] * (sr * inv)) + a.w[2] * expf(-a.k[2] * (sv * inv)) +
                  a.w[3] * expf(-a.k[3] * (sw * inv));
    a.mpjpe[e] = sd * inv;
    const bool bad = a.status && (a.status[e] & 7);   // the stepper put this env back to qpos0 (mj_checkPos / Vel / Acc): off its clip
    a.terminated[e] = ((p > 1 && md > a.term_dist) || bad) ? 1 : 0;
    a.truncated[e] = (t_next > len || p > a.episode_length) ? 1 : 0;
  }
}
