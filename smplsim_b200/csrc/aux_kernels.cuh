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

// get_motion_state (the torch motion library, motion_lib_base_torch.py:434-499): two frames around t and a blend weight instead of
// one frame.  Every operation is one float32 rounding, as torch computes it on the CPU: no contraction, correctly rounded division.
#ifdef SMPLSIM_EMU
// the host build of these sources (the tests' SIMT emulator): one rounding per call, the empty asm keeps the compiler from fusing a
// product into a neighbouring add (nvcc never fuses the device intrinsics)
static inline float mb_host_rn(float r) {
#if defined(__x86_64__)
  __asm__("" : "+x"(r));
#else
  volatile float v = r;
  r = v;
#endif
  return r;
}
static inline float __fadd_rn(float a, float b) { return mb_host_rn(a + b); }
static inline float __fsub_rn(float a, float b) { return mb_host_rn(a - b); }
static inline float __fmul_rn(float a, float b) { return mb_host_rn(a * b); }
static inline float __fdiv_rn(float a, float b) { return mb_host_rn(a / b); }
static inline float __fsqrt_rn(float a) { return mb_host_rn(sqrtf(a)); }
#endif
struct MBlend { int f0, f1; float b; };
__device__ __forceinline__ MBlend motion_blend_frames(float len, float dt, int nf, float t) {   // _calc_frame_blend (:528-538)
  const float phase = fminf(fmaxf(__fdiv_rn(t, len), 0.f), 1.f);
  if (t < 0.f) t = 0.f;
  MBlend m;
  m.f0 = (int)__fmul_rn(phase, (float)(nf - 1));
  m.f1 = min(m.f0 + 1, nf - 1);
  m.b = fminf(fmaxf(__fdiv_rn(__fsub_rn(t, __fmul_rn((float)m.f0, dt)), dt), 0.f), 1.f);
  return m;
}
// (1 - b) v0 + b v1
__device__ __forceinline__ float mb_lerp(float v0, float v1, float b) { return __fadd_rn(__fmul_rn(__fsub_rn(1.f, b), v0), __fmul_rn(b, v1)); }
__device__ __forceinline__ V3 mb_lerp3(V3 p, V3 q, float b) { return v3(mb_lerp(p.x, q.x, b), mb_lerp(p.y, q.y, b), mb_lerp(p.z, q.z, b)); }
// torch_utils.slerp (smpl_sim/utils/torch_utils.py:405-426) with its quirks: q1 flipped when the dot product is negative, the plain
// midpoint when |sin(half angle)| < 0.001 whatever the blend, q0 when cos(half angle) >= 1, no normalisation.  Component order free.
__device__ __forceinline__ Q4 mb_slerp(Q4 q0, Q4 q1, float t) {
  float c = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(q0.w, q1.w), __fmul_rn(q0.x, q1.x)), __fmul_rn(q0.y, q1.y)), __fmul_rn(q0.z, q1.z));
  if (c < 0.f) { q1.w = -q1.w; q1.x = -q1.x; q1.y = -q1.y; q1.z = -q1.z; c = -c; }
  if (c >= 1.f) return q0;
  const float s = __fsqrt_rn(__fsub_rn(1.f, __fmul_rn(c, c)));
  float ra = 0.5f, rb = 0.5f;
  if (!(fabsf(s) < 0.001f)) {
    const float ht = acosf(c);
    ra = __fdiv_rn(sinf(__fmul_rn(__fsub_rn(1.f, t), ht)), s); rb = __fdiv_rn(sinf(__fmul_rn(t, ht)), s);
  }
  Q4 r;
  r.w = __fadd_rn(__fmul_rn(ra, q0.w), __fmul_rn(rb, q1.w)); r.x = __fadd_rn(__fmul_rn(ra, q0.x), __fmul_rn(rb, q1.x));
  r.y = __fadd_rn(__fmul_rn(ra, q0.y), __fmul_rn(rb, q1.y)); r.z = __fadd_rn(__fmul_rn(ra, q0.z), __fmul_rn(rb, q1.z));
  return r;
}
__device__ __forceinline__ Q4 mb_ldq(const float* p) { Q4 q; q.w = p[0]; q.x = p[1]; q.y = p[2]; q.z = p[3]; return q; }
__device__ __forceinline__ void mb_stq(float* p, Q4 q) { p[0] = q.w; p[1] = q.x; p[2] = q.y; p[3] = q.z; }
// quat_to_tan_norm: [q * (1,0,0), q * (0,0,1)], a rotation as the observations hold it (the rule of pack_self_obs)
__device__ __forceinline__ void st_tan_norm(float* p, Q4 q) {
  st3(p, qrot_ref(q, v3(1.f, 0.f, 0.f)));
  st3(p + 3, qrot_ref(q, v3(0.f, 0.f, 1.f)));
}

// The motion library as the per-env task kernels (imitation, tracking evaluation, AMP) read it, from the fields their arguments share:
// per-frame body tables txpos / txquat / tvel / tangvel [total_frames, nb * {3, 4, 3, 3}], per-clip rows mlen / nframes / mdt / starts
// and nmotion clips.  The fields stay flat in each argument struct: nested in a struct of their own they cost k_imitation<0, 1, 0>
// 16 registers (a CTA fewer per SM) and a fifth of its time.
// motion_clip: a caller's clip id, clamped to the library
template <class A>
__device__ __forceinline__ int motion_clip(const A& a, int id) { return min(max(id, 0), a.nmotion - 1); }
// The reference pose of a clip at one time.  ImFrame: its table row f0 and, with INTERP, the next row f1 and the blend weight of
// get_motion_state (motion_blend_frames); without, the one row of motion_frame.
struct ImFrame { size_t f0, f1; float b; };
template <int INTERP>
__device__ __forceinline__ ImFrame im_frame(float len, float mdt, int nf, int start, float t) {
  ImFrame f;
  if (INTERP) {
    const MBlend m = motion_blend_frames(len, mdt, nf, t);
    f.f0 = (size_t)(start + m.f0); f.f1 = (size_t)(start + m.f1); f.b = m.b;
  } else {
    f.f0 = f.f1 = (size_t)(start + motion_frame(len, mdt, nf, t)); f.b = 0.f;
  }
  return f;
}
// the body tables' row r of the library in a (with a.nb bodies)
struct ImRow {
  const float *p, *q, *v, *w;
  template <class A>
  __device__ __forceinline__ ImRow(const A& a, size_t r) : p(a.txpos + r * a.nb * 3), q(a.txquat + r * a.nb * 4), v(a.tvel + r * a.nb * 3), w(a.tangvel + r * a.nb * 3) {}
};

// smplsim_motion_blend: per table a value kind (SMPLSIM_BLEND_*, include/smplsim.h)
#define MB_LERP 0
#define MB_POS 1
#define MB_SLERP 2
#define MB_QPOS 3
#define MB_ROW0 4
struct BlendArgs {
  GatherArgs g;   // frame_idx unused
  int kinds[SM_MAXTABLES];
  const float* offset;   // [n, 3] or NULL
  int32_t *frame0, *frame1; float* blend;
};
// a warp per query row, lanes over a table's columns (SLERP: over its quaternions)
__global__ void k_motion_blend(BlendArgs a) {
  const int lane = threadIdx.x & 31;
  const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= a.g.n) return;
  const int id = a.g.ids[i];
  const MBlend m = motion_blend_frames(a.g.mlen[id], a.g.mdt[id], a.g.nframes[id], a.g.times[i]);
  const size_t r0 = (size_t)(m.f0 + a.g.starts[id]), r1 = (size_t)(m.f1 + a.g.starts[id]);
  if (lane == 0) {
    if (a.frame0) a.frame0[i] = (int32_t)r0;
    if (a.frame1) a.frame1[i] = (int32_t)r1;
    if (a.blend) a.blend[i] = m.b;
  }
  float ox = 0.f, oy = 0.f, oz = 0.f;
  if (a.offset) { ox = a.offset[3 * i]; oy = a.offset[3 * i + 1]; oz = a.offset[3 * i + 2]; }
  for (int k = 0; k < a.g.ntab; k++) {
    const int w = a.g.widths[k], kind = a.kinds[k];
    const float *s0 = a.g.tables[k] + r0 * w, *s1 = a.g.tables[k] + r1 * w;
    float* dst = a.g.outs[k] + (size_t)i * w;
    if (kind == MB_SLERP) {
      for (int q = lane; q < w / 4; q += 32) mb_stq(dst + 4 * q, mb_slerp(mb_ldq(s0 + 4 * q), mb_ldq(s1 + 4 * q), m.b));
      continue;
    }
    for (int j = lane; j < w; j += 32) {
      if (kind == MB_ROW0) { dst[j] = s0[j]; continue; }
      if (kind == MB_QPOS && j >= 3 && j < 7) {   // the root quaternion: one lane slerps all four
        if (j == 3) mb_stq(dst + 3, mb_slerp(mb_ldq(s0 + 3), mb_ldq(s1 + 3), m.b));
        continue;
      }
      float v = mb_lerp(s0[j], s1[j], m.b);
      if (a.offset && (kind == MB_POS || (kind == MB_QPOS && j < 3))) v = __fadd_rn(v, j % 3 == 0 ? ox : j % 3 == 1 ? oy : oz);
      dst[j] = v;
    }
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
