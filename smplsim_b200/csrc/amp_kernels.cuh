// amp_kernels.cuh -- adversarial motion priors (smplsim_amp_obs / smplsim_amp_demo): the per-env history of AMP frames and the
// demonstration frames of a motion library, in one launch.  The per-frame feature is the reference's compute_humanoid_observations_smpl
// (smpl_sim/envs/nv/humanoid.py:2530-2602, has_smpl_params = False) with dof_to_obs (:2276-2309); it is stated in include/smplsim.h.
//
// A warp per env (or demo row), lanes over the non-root bodies for the exp-map columns, over the dofs for the velocities and over the
// key bodies.  The history shift moves column c of every frame on lane c % 32 only, so no lane reads a word another lane wrote; the
// new frame 0 is written after a __syncwarp.  No atomics and no reductions: every output word is a function of its inputs alone.
#pragma once
#include "aux_kernels.cuh"

#define AMP_PUSH 0       // shift the history by one frame, the current simulated frame at 0
#define AMP_FILL 1       // the current simulated frame in every slot
#define AMP_FILL_REF 2   // the current simulated frame at 0, the env's clip at t0 + (p - k) dt in slot k >= 1
#define AMP_DEMO 3       // caller rows (motion id, time): ref(t - k dt) in slot k

struct AmpArgs {
  // motion library: per-frame tables [total_frames, nb * {3, 4, 3, 3} | nv - 6 | nv - 6] and per-clip rows (FILL_REF, DEMO)
  const float *txpos, *txquat, *tvel, *tangvel, *tdof, *tdofv;
  const float* mlen; const int32_t* nframes; const float* mdt; const int32_t* starts;
  // per env (per row in DEMO)
  const int32_t* ids; const float* t0; const int32_t* progress; const uint8_t* mask;
  const float *qpos, *qvel, *xpos, *xquat;
  float* out;                        // [n, K, F]
  float dt;
  int n, K, F, nb, nv, nkey, nmotion, mode, local_root, root_h;
  unsigned char key[LM_MAXB];
};

__device__ __forceinline__ Q4 amp_ldq(const float* p) { Q4 q; q.w = p[0]; q.x = p[1]; q.y = p[2]; q.z = p[3]; return q; }
__device__ __forceinline__ void amp_st6(float* p, Q4 q) {   // quat_to_tan_norm: [q * (1,0,0), q * (0,0,1)]
  st3(p, qrot_ref(q, v3(1.f, 0.f, 0.f)));
  st3(p + 3, qrot_ref(q, v3(0.f, 0.f, 1.f)));
}

// One AMP frame into out[0, F).  root_vel / root_ang_vel are world-frame; dof / dofv hold nv - 6 values; bx is the [nb, 3] body
// position row the key bodies are read from.
__device__ __forceinline__ void amp_frame(const LHdr& H, const AmpArgs& a, int lane, V3 root, Q4 rq, V3 rv, V3 rw, const float* dof,
                                          const float* dofv, const float* bx, float* out) {
  const Q4 hq = l_heading_inv(H, rq);   // remove_base_rot first when !upright_start (inside)
  if (!H.cfg.upright_start) { Q4 bc; bc.w = 0.5f; bc.x = -0.5f; bc.y = -0.5f; bc.z = -0.5f; rq = qmul(rq, bc); }
  const int o = a.root_h, od = o + 12, ov = od + 6 * (a.nb - 1), ok = ov + (a.nv - 6);
  if (lane == 0) {
    if (a.root_h) out[0] = root.z;
    amp_st6(out + o, a.local_root ? qmul(hq, rq) : rq);
    st3(out + o + 6, qrot_ref(hq, rv));
    st3(out + o + 9, qrot_ref(hq, rw));
  }
  for (int j = lane; j < a.nb - 1; j += 32) {   // dof_to_obs: exp_map_to_quat then quat_to_tan_norm, per 3-hinge body
    const V3 e = ld3(dof + 3 * j);
    const float ang = sqrtf(dot(e, e));
    const float w = atan2f(sinf(ang), cosf(ang));   // normalize_angle
    Q4 q; q.w = 1.f; q.x = 0.f; q.y = 0.f; q.z = 0.f;
    if (fabsf(w) > 1e-5f) {
      const float inv = 1.0f / ang;
      V3 ax = v3(e.x * inv, e.y * inv, e.z * inv);
      const float an = sqrtf(dot(ax, ax)), s = sinf(0.5f * w) / an;   // quat_from_angle_axis normalises the axis ...
      q.w = cosf(0.5f * w); q.x = ax.x * s; q.y = ax.y * s; q.z = ax.z * s;
      q = qnormalize(q);                                               // ... and the quaternion
    }
    amp_st6(out + od + 6 * j, q);
  }
  for (int i = lane; i < a.nv - 6; i += 32) out[ov + i] = dofv[i];
  for (int k = lane; k < a.nkey; k += 32) st3(out + ok + 3 * k, qrot_ref(hq, ld3(bx + 3 * a.key[k]) - root));
}

// ref(t) of clip id into out.  INTERP = 0: the row motion_frame picks (the gather's nearest-frame rule, no blending).  INTERP = 1: the
// state get_motion_state blends from the frames f0 / f1 of motion_blend_frames, with k_motion_blend's rules (root rotation slerped;
// root and key-body positions, velocities and the dof_pos exp-map triples lerped).  The blended dof_pos, dof_vel and body positions
// are staged in the warp's shared-memory slot and framed by the same amp_frame.
#define AMP_STAGE (2 * 3 * (LM_MAXB - 1) + 3 * LM_MAXB)   // floats per warp: dof_pos, dof_vel, body positions
template <int INTERP>
__device__ __forceinline__ void amp_ref_frame(const LHdr& H, const AmpArgs& a, int lane, int id, float t, float* out) {
  if (INTERP) {
    __shared__ float stage[8][AMP_STAGE];   // 8 warps per CTA (the launches' size)
    float* sd = stage[threadIdx.x >> 5];
    const int nd = a.nv - 6;
    float *sv = sd + nd, *sx = sd + 2 * nd;
    const MBlend m = motion_blend_frames(a.mlen[id], a.mdt[id], a.nframes[id], t);
    const size_t r0 = (size_t)(a.starts[id] + m.f0), r1 = (size_t)(a.starts[id] + m.f1);
    __syncwarp();   // the previous frame's reads of the slot are done
    for (int i = lane; i < nd; i += 32) {
      sd[i] = mb_lerp(a.tdof[r0 * nd + i], a.tdof[r1 * nd + i], m.b);
      sv[i] = mb_lerp(a.tdofv[r0 * nd + i], a.tdofv[r1 * nd + i], m.b);
    }
    for (int i = lane; i < 3 * a.nb; i += 32) sx[i] = mb_lerp(a.txpos[r0 * a.nb * 3 + i], a.txpos[r1 * a.nb * 3 + i], m.b);
    __syncwarp();
    amp_frame(H, a, lane, ld3(sx), mb_slerp(amp_ldq(a.txquat + r0 * a.nb * 4), amp_ldq(a.txquat + r1 * a.nb * 4), m.b),
              mb_lerp3(ld3(a.tvel + r0 * a.nb * 3), ld3(a.tvel + r1 * a.nb * 3), m.b),
              mb_lerp3(ld3(a.tangvel + r0 * a.nb * 3), ld3(a.tangvel + r1 * a.nb * 3), m.b), sd, sv, sx, out);
    return;
  }
  const size_t r = (size_t)(a.starts[id] + motion_frame(a.mlen[id], a.mdt[id], a.nframes[id], t));
  const float* bx = a.txpos + r * a.nb * 3;
  amp_frame(H, a, lane, ld3(bx), amp_ldq(a.txquat + r * a.nb * 4), ld3(a.tvel + r * a.nb * 3), ld3(a.tangvel + r * a.nb * 3),
            a.tdof + r * (a.nv - 6), a.tdofv + r * (a.nv - 6), bx, out);
}

// INTERP: library frames blended (SmplsimAmpCfg.interpolate); <0> reads the nearest frame
template <int INTERP>
__global__ void __launch_bounds__(256) k_amp_obs(const float* __restrict__ gimg, AmpArgs a) {
  const LHdr& H = *(const LHdr*)gimg;   // the heading rule (upright_start) is the same for every body shape of a handle
  const int lane = threadIdx.x & 31;
  const int e = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (e >= a.n || (a.mask && !a.mask[e])) return;   // warp-uniform
  const int K = a.K, F = a.F;
  float* row = a.out + (size_t)e * K * F;
  if (a.mode == AMP_DEMO) {
    const int id = min(max(a.ids[e], 0), a.nmotion - 1);
    const float t = a.t0[e];
    for (int k = 0; k < K; k++) amp_ref_frame<INTERP>(H, a, lane, id, fmaf(-(float)k, a.dt, t), row + (size_t)k * F);
    return;
  }
  if (a.mode == AMP_PUSH) {
    // slots K-2 .. 0 move up one, highest first; a lane owns its columns in every slot, and a group's loads precede its stores
    for (int c = lane; c < F; c += 32) {
      float* col = row + c;
      for (int k = K - 2; k >= 0; k -= 8) {
        float v[8];
#pragma unroll
        for (int i = 0; i < 8; i++) if (i <= k) v[i] = col[(size_t)(k - i) * F];
#pragma unroll
        for (int i = 0; i < 8; i++) if (i <= k) col[(size_t)(k - i + 1) * F] = v[i];
      }
    }
    __syncwarp();
  }
  {   // the simulated frame at slot 0: post-step state; MuJoCo's root angular velocity is body-frame, rotated to world here
    const float *qp = a.qpos + (size_t)e * a.nv + (size_t)e, *qv = a.qvel + (size_t)e * a.nv;   // qpos rows are nv + 1 wide
    const float* bx = a.xpos + (size_t)e * a.nb * 3;
    const Q4 rq = amp_ldq(a.xquat + (size_t)e * a.nb * 4);
    amp_frame(H, a, lane, ld3(bx), rq, ld3(qv), qrot_ref(rq, ld3(qv + 3)), qp + 7, qv + 6, bx, row);
  }
  if (a.mode == AMP_PUSH) return;
  if (a.mode == AMP_FILL) {
    __syncwarp();
    for (int c = lane; c < F; c += 32) {
      const float v = row[c];
      for (int k = 1; k < K; k++) row[(size_t)k * F + c] = v;
    }
    return;
  }
  // AMP_FILL_REF: the env's clip behind the current time, t0 + (p - k) dt as one fused multiply-add (the time rule of k_imitation)
  const int id = min(max(a.ids[e], 0), a.nmotion - 1);
  const int p = a.progress[e];
  for (int k = 1; k < K; k++) amp_ref_frame<INTERP>(H, a, lane, id, fmaf((float)(p - k), a.dt, a.t0[e]), row + (size_t)k * F);
}
