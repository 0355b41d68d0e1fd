// aux_kernels.cuh -- small standalone kernels around the stepper: self observations on caller-supplied body states,
// the motion-library gather, GAE.  One row per warp / thread; nothing here is on the hot path.
#pragma once
#include "lane_kernels.cuh"

// compute_humanoid_self_obs_v1 / _v2 (humanoid_env.py:565-688) on caller-supplied body states
__device__ __forceinline__ void pack_self_obs(const LHdr& H, int version, int lane, float root_h, const float* xpos_rel, const float* xquat,
                                              const float* qvel, const float* sens, float* out) {
  int nb = H.nb;
  Q4 r0; r0.w = xquat[0]; r0.x = xquat[1]; r0.y = xquat[2]; r0.z = xquat[3];
  Q4 hq = l_heading_inv(H, r0);
  int o = 0;
  if (H.cfg.root_height_obs) { if (lane == 0) out[0] = root_h; o = 1; }
  int o_rot = o + 3 * (nb - 1), o_vel = o_rot + 6 * nb;
  for (int b = lane; b < nb; b += 32) {
    if (b > 0) st3(out + o + 3 * (b - 1), qrot_ref(hq, ld3(xpos_rel + 3 * b)));
    Q4 q; q.w = xquat[4 * b]; q.x = xquat[4 * b + 1]; q.y = xquat[4 * b + 2]; q.z = xquat[4 * b + 3];
    Q4 lq = qmul(hq, q);
    st3(out + o_rot + 6 * b, qrot_ref(lq, v3(1.f, 0.f, 0.f)));
    st3(out + o_rot + 6 * b + 3, qrot_ref(lq, v3(0.f, 0.f, 1.f)));
    if (version == 2) {
      st3(out + o_vel + 3 * b, qrot_ref(hq, ld3(sens + 6 * b)));
      st3(out + o_vel + 3 * nb + 3 * b, qrot_ref(hq, ld3(sens + 6 * b + 3)));
    }
  }
  if (version == 1) {
    if (lane == 0) st3(out + o_vel, qrot_ref(hq, ld3(qvel)));
    if (lane == 1) st3(out + o_vel + 3, qrot_ref(hq, ld3(qvel + 3)));
    for (int i = lane; i < H.nu; i += 32) out[o_vel + 6 + i] = qvel[6 + i];
  }
}

__global__ void k_self_obs(const float* __restrict__ gimg, int version, const float* qvel, const float* xpos, const float* xquat,
                           const float* linvel, const float* angvel, float* obs, int n, int self_dim) {
  const LHdr& H = *(const LHdr*)gimg;
  int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  int env = blockIdx.x * (blockDim.x >> 5) + wib;
  if (env >= n) return;
  float* sm = L_SMEM + (size_t)wib * (16 * LM_MAXB);
  float *xr = sm, *sens = sm + 3 * LM_MAXB;
  const float* xp = xpos + (size_t)env * H.nb * 3;
  V3 root = ld3(xp);
  for (int b = lane; b < H.nb; b += 32) {
    st3(xr + 3 * b, ld3(xp + 3 * b) - root);
    if (version == 2) {
      st3(sens + 6 * b, ld3(linvel + ((size_t)env * H.nb + b) * 3));
      st3(sens + 6 * b + 3, ld3(angvel + ((size_t)env * H.nb + b) * 3));
    }
  }
  __syncwarp();
  pack_self_obs(H, version, lane, root.z, xr, xquat + (size_t)env * H.nb * 4, qvel ? qvel + (size_t)env * H.nv : nullptr, sens,
                obs + (size_t)env * self_dim);
}

// get_motion_state_intervaled: frame = floor(clip(t,0,len)/dt) clipped to the clip, + length_starts[id]; row gather of every table
#define SM_MAXTABLES 16
struct GatherArgs {
  const int32_t* ids; const float* times; const float* mlen; const int32_t* nframes; const float* mdt; const int32_t* starts;
  const float* tables[SM_MAXTABLES]; float* outs[SM_MAXTABLES]; int widths[SM_MAXTABLES];
  int32_t* frame_idx; int n, ntab;
};
// the frame of a clip (length len, nf frames, frame period dt) at time t: motion_lib_base.py:448-458 + :321-323 (quirk Q12): phase clip,
// float idx0, blend, int() truncation.  The one frame rule of the library: the gather and the imitation task both call it.
__device__ __forceinline__ int motion_frame(float len, float dt, int nf, float t) {
  float phase = fminf(fmaxf(t / len, 0.f), 1.f);
  if (t < 0.f) t = 0.f;
  float idx0 = phase * (float)(nf - 1);
  float idx1 = fminf(idx0 + 1.f, (float)(nf - 1));
  float blend = fminf(fmaxf((t - idx0 * dt) / dt, 0.f), 1.f);
  return (int)((1.0f - blend) * idx0 + blend * idx1);
}
__global__ void k_motion_gather(GatherArgs a) {
  int lane = threadIdx.x & 31;
  int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= a.n) return;
  int id = a.ids[i];
  int fr = motion_frame(a.mlen[id], a.mdt[id], a.nframes[id], a.times[i]);
  size_t row = (size_t)(fr + a.starts[id]);
  if (lane == 0 && a.frame_idx) a.frame_idx[i] = (int)row;
  for (int k = 0; k < a.ntab; k++) {
    const float* src = a.tables[k] + row * a.widths[k];
    float* dst = a.outs[k] + (size_t)i * a.widths[k];
    for (int j = lane; j < a.widths[k]; j += 32) dst[j] = src[j];
  }
}

// GAE (SURVEY.md 8 f2): learning_utils.estimate_advantages:198-218 as a reverse scan per env column of the [T,N] rollout;
// thread per env, coalesced across envs at every t.
__global__ void k_gae(const float* __restrict__ rew, const float* __restrict__ not_done, const float* __restrict__ not_dead,
                      const float* __restrict__ val, const float* __restrict__ next_val, float gamma, float tau, int T, int N,
                      float* __restrict__ adv, float* __restrict__ ret) {
  int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= N) return;
  float prev_v = next_val ? next_val[e] : 0.f, prev_a = 0.f;
  for (int t = T - 1; t >= 0; t--) {
    size_t i = (size_t)t * N + e;
    float v = val[i];
    float delta = rew[i] + gamma * prev_v * not_dead[i] - v;
    float a = delta + gamma * tau * prev_a * not_done[i];
    adv[i] = a;
    ret[i] = v + a;
    prev_v = v; prev_a = a;
  }
}

// ------------------------------------------------------------------ per-env parameter records (smplsim_set_env_params / _get_env_params)
// One record of w words per env: [mu | gravity 3 | kp nu | kd nu | torque limit nu | mass scale nb | pad] (LCfg::PRM_*).  One thread per
// word.  set: rec NULL is not allowed; init = 1 first fills every env's record with its table's values (env_img: env -> table, NULL: one
// table), then the envs whose mask byte is set (mask NULL: all) take each non-NULL field.  get: rec NULL reads the tables' values.
struct PrmArgs {
  float* rec;
  const float* gimg;       // the handle's tables, img_words floats each
  const int* env_img;
  const uint8_t* mask;
  const float* f[6];       // mu [N], gravity [N,3], kp / kd / torque limit [N,nu], mass scale [N,nb]
  float* o[6];             // (get) the same layout
  int img_words, n, nu, nb, w, init;
};
// field of word j and its column (-1: padding)
__device__ __forceinline__ int prm_field(const PrmArgs& a, int j, int* col) {
  const int kp = 4, kd = kp + a.nu, tl = kd + a.nu, ms = tl + a.nu;
  if (j == 0) { *col = 0; return 0; }
  if (j < kp) { *col = j - 1; return 1; }
  if (j < kd) { *col = j - kp; return 2; }
  if (j < tl) { *col = j - kd; return 3; }
  if (j < ms) { *col = j - tl; return 4; }
  if (j < ms + a.nb) { *col = j - ms; return 5; }
  *col = 0;
  return -1;
}
__device__ __forceinline__ float prm_nominal(const PrmArgs& a, int e, int fld, int col) {
  const float* img = a.gimg + (size_t)(a.env_img ? a.env_img[e] : 0) * (size_t)a.img_words;
  const LHdr& H = *(const LHdr*)img;
  const LBody* B = (const LBody*)((const char*)img + LM_BODY_OFF);
  switch (fld) {
    case 0: return H.mu;
    case 1: return H.grav[col];
    case 2: return B[1 + col / 3].kp[col % 3];
    case 3: return B[1 + col / 3].kd[col % 3];
    case 4: return B[1 + col / 3].tlim[col % 3];
    case 5: return 1.0f;
    default: return 0.f;
  }
}
__device__ __forceinline__ int prm_width(const PrmArgs& a, int fld) { return fld == 0 ? 1 : fld == 1 ? 3 : fld == 5 ? a.nb : a.nu; }

__global__ void k_prm_set(PrmArgs a) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)a.n * a.w) return;
  const int e = (int)(i / a.w), j = (int)(i % a.w);
  int col;
  const int fld = prm_field(a, j, &col);
  float v = a.init ? prm_nominal(a, e, fld, col) : a.rec[i];
  if (fld >= 0 && a.f[fld] && (!a.mask || a.mask[e])) v = a.f[fld][(size_t)e * prm_width(a, fld) + col];
  a.rec[i] = v;
}

__global__ void k_prm_get(PrmArgs a) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)a.n * a.w) return;
  const int e = (int)(i / a.w), j = (int)(i % a.w);
  int col;
  const int fld = prm_field(a, j, &col);
  if (fld < 0 || !a.o[fld]) return;
  a.o[fld][(size_t)e * prm_width(a, fld) + col] = a.rec ? a.rec[i] : prm_nominal(a, e, fld, col);
}
