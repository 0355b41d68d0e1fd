// track_eval_kernels.cuh -- tracking evaluation (smplsim_track_eval): the per-frame error metrics of the reference's smpl_eval
// (compute_metrics_lite / compute_metrics_obj: global, root-relative and Procrustes-aligned mean per-joint position error, velocity and
// acceleration error, rotation error) of every active env against its motion-library clip, accumulated per env over an evaluation.
// The definitions are stated in include/smplsim.h.
//
// A warp per env, lanes over the eval bodies (two per lane above 32).  Each body's reference and simulated positions are read once into
// registers; the three passes (means, cross-covariance, aligned error) reuse them.  Sums are lane partials in body-list order followed
// by an xor butterfly, as in k_imitation: no atomics, the outputs are bit-reproducible.  The reference rows come from k_imitation's own
// frame rule (im_frame / ImRef), so a scored frame is exactly the pair the imitation reward compares.
//
// Procrustes step: Horn's closed form.  With centred root-relative points x0 (reference) and y0 (simulated), S = sum_j y0_j x0_j^T;
// the unit quaternion of the proper rotation Q maximising sum_j x0_j . Q y0_j is the eigenvector of the largest eigenvalue of the
// symmetric 4x4 matrix N(S), and that eigenvalue is the maximum itself (= the reference's sign-corrected sum(s) times |X0| |Y0|).
// The eigenvector comes from a fixed number of cyclic Jacobi sweeps, computed redundantly on every lane: no branch depends on the
// data, and a repeated eigenvalue (collinear points, a rank-1 S) needs no special case.
#pragma once
#include "imitation_kernels.cuh"

#define TE_NMETRIC SMPLSIM_TRACK_NMETRIC   // mpjpe_g, mpjpe_l, mpjpe_pa, vel_dist, accel_dist, rot_error
#define TE_SWEEPS 6    // cyclic Jacobi sweeps of the 4x4 eigenproblem (quadratic convergence: 3-4 reach float32 precision)

struct TeArgs {
  ImArgs im;               // the tables, clip / start time / step counter per env, simulated poses, dt, n, nb, J, body list
  const uint8_t *terminated, *truncated;
  uint8_t* active;
  float* prev_diff;        // [n, 2, J, 3]
  int32_t* frames;         // [n]
  double* sums;            // [n, TE_NMETRIC]
  uint8_t* success;        // [n]
  float* frame_metrics;    // [n, TE_NMETRIC] or NULL
};

// one Jacobi rotation of the symmetric a (both triangles kept) zeroing a[p][q]; v accumulates the rotations (columns: eigenvectors).
// t = tan of the rotation angle, Rutishauser's smaller root; a[p][q] = 0 with a[p][p] = a[q][q] gives t = 0 without a branch.
template <int P, int Q>
__device__ __forceinline__ void te_jacobi_rot(float (&a)[4][4], float (&v)[4][4]) {
  const float apq = a[P][Q], d = a[Q][Q] - a[P][P];
  const float den = fabsf(d) + sqrtf(fmaf(d, d, 4.f * apq * apq));
  const float t = den > 0.f ? (d < 0.f ? -2.f * apq : 2.f * apq) / den : 0.f;   // 2 apq sgn(d) / den, sgn(0) = +1
  const float c = rsqrtf(fmaf(t, t, 1.f)), s = t * c;
  a[P][P] -= t * apq; a[Q][Q] += t * apq; a[P][Q] = a[Q][P] = 0.f;
#pragma unroll
  for (int r = 0; r < 4; r++) {
    if (r == P || r == Q) continue;   // compile-time
    const float arp = a[r][P], arq = a[r][Q];
    a[r][P] = a[P][r] = c * arp - s * arq;
    a[r][Q] = a[Q][r] = s * arp + c * arq;
  }
#pragma unroll
  for (int r = 0; r < 4; r++) {
    const float vp = v[r][P], vq = v[r][Q];
    v[r][P] = c * vp - s * vq;
    v[r][Q] = s * vp + c * vq;
  }
}

// Horn's matrix of S (S[a][b] = sum_j y0_a x0_b): the largest eigenvalue lam and its unit eigenvector q (wxyz), the rotation taking y0 onto x0
__device__ __forceinline__ float te_horn(const float (&S)[3][3], Q4& q) {
  const float sxx = S[0][0], sxy = S[0][1], sxz = S[0][2], syx = S[1][0], syy = S[1][1], syz = S[1][2], szx = S[2][0], szy = S[2][1], szz = S[2][2];
  float a[4][4] = {{sxx + syy + szz, syz - szy, szx - sxz, sxy - syx},
                   {syz - szy, sxx - syy - szz, sxy + syx, szx + sxz},
                   {szx - sxz, sxy + syx, syy - sxx - szz, syz + szy},
                   {sxy - syx, szx + sxz, syz + szy, szz - sxx - syy}};
  float v[4][4] = {{1.f, 0.f, 0.f, 0.f}, {0.f, 1.f, 0.f, 0.f}, {0.f, 0.f, 1.f, 0.f}, {0.f, 0.f, 0.f, 1.f}};
#pragma unroll 1
  for (int sw = 0; sw < TE_SWEEPS; sw++) {
    te_jacobi_rot<0, 1>(a, v); te_jacobi_rot<0, 2>(a, v); te_jacobi_rot<0, 3>(a, v);
    te_jacobi_rot<1, 2>(a, v); te_jacobi_rot<1, 3>(a, v); te_jacobi_rot<2, 3>(a, v);
  }
  float lam = a[0][0];
  q.w = v[0][0]; q.x = v[1][0]; q.y = v[2][0]; q.z = v[3][0];
#pragma unroll
  for (int k = 1; k < 4; k++) {   // selects, not branches: the first largest diagonal entry
    const bool up = a[k][k] > lam;
    lam = up ? a[k][k] : lam;
    q.w = up ? v[0][k] : q.w; q.x = up ? v[1][k] : q.x; q.y = up ? v[2][k] : q.y; q.z = up ? v[3][k] : q.z;
  }
  return lam;
}

// Q y for the unit quaternion q (wxyz), as a rotation matrix applied to y
__device__ __forceinline__ void te_qmat(Q4 q, float (&R)[3][3]) {
  const float w = q.w, x = q.x, y = q.y, z = q.z;
  R[0][0] = 1.f - 2.f * (y * y + z * z); R[0][1] = 2.f * (x * y - w * z); R[0][2] = 2.f * (x * z + w * y);
  R[1][0] = 2.f * (x * y + w * z); R[1][1] = 1.f - 2.f * (x * x + z * z); R[1][2] = 2.f * (y * z - w * x);
  R[2][0] = 2.f * (x * z - w * y); R[2][1] = 2.f * (y * z + w * x); R[2][2] = 1.f - 2.f * (x * x + y * y);
}

// INTERP: blended reference states (SmplsimTrackEvalCfg.interpolate), the rule of k_imitation<1, *>
template <int INTERP>
__global__ void __launch_bounds__(256) k_track_eval(TeArgs t) {
  const ImArgs& a = t.im;
  const int lane = threadIdx.x & 31;
  const int e = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (e >= a.n || !t.active[e]) return;   // warp-uniform
  const int nb = a.nb, J = a.J;
  const int id = min(max(a.ids[e], 0), a.nmotion - 1);
  const float len = a.mlen[id], mdt = a.mdt[id], t0 = a.t0[e];
  const int nf = a.nframes[id], start = a.starts[id], p = a.progress[e];
  const ImRef<INTERP> ref(a, im_frame<INTERP>(len, mdt, nf, start, fmaf((float)p, a.dt, t0)));   // the row k_imitation's reward compares
  const float *xp = a.xpos + (size_t)e * nb * 3, *xq = a.xquat + (size_t)e * nb * 4;
  const int f = t.frames[e];   // frames scored before this one
  float* pd = t.prev_diff + (size_t)e * 2 * J * 3;
  float *d1 = pd + (size_t)((f + 1) & 1) * J * 3, *d2 = pd + (size_t)(f & 1) * J * 3;   // slot f % 2 holds frame f - 2, then frame f
  // pass 1: positions into registers; global error, velocity, acceleration and rotation sums; root-relative sums
  V3 x[2], y[2];
  float sg = 0.f, sv = 0.f, sa = 0.f, sr = 0.f;
  V3 mx = v3(0.f, 0.f, 0.f), my = v3(0.f, 0.f, 0.f);
#pragma unroll
  for (int k = 0; k < 2; k++) {
    const int j = lane + 32 * k;
    x[k] = y[k] = v3(0.f, 0.f, 0.f);
    if (j < J) {
      const int b = a.body[j];
      x[k] = ref.pos(b); y[k] = ld3(xp + 3 * b);
      const V3 d = y[k] - x[k];
      sg += sqrtf(dot(d, d));
      if (f >= 1) { const V3 dv = d - ld3(d1 + 3 * j); sv += sqrtf(dot(dv, dv)); }
      if (f >= 2) { const V3 da = (d - ld3(d1 + 3 * j)) - (ld3(d1 + 3 * j) - ld3(d2 + 3 * j)); sa += sqrtf(dot(da, da)); }
      st3(d2 + 3 * j, d);
      const Q4 dq = qmul(ref.quat(b), im_conj(im_ldq(xq + 4 * b)));
      sr += 2.0f * atan2f(sqrtf(dq.x * dq.x + dq.y * dq.y + dq.z * dq.z), fabsf(dq.w));
    }
  }
  // root = the first eval body, held by lane 0 in its first slot
  const V3 xroot = v3(__shfl_sync(L_FULL, x[0].x, 0), __shfl_sync(L_FULL, x[0].y, 0), __shfl_sync(L_FULL, x[0].z, 0));
  const V3 yroot = v3(__shfl_sync(L_FULL, y[0].x, 0), __shfl_sync(L_FULL, y[0].y, 0), __shfl_sync(L_FULL, y[0].z, 0));
  float sl = 0.f;
#pragma unroll
  for (int k = 0; k < 2; k++) {
    if (lane + 32 * k < J) {
      x[k] = x[k] - xroot; y[k] = y[k] - yroot;
      const V3 d = y[k] - x[k];
      sl += sqrtf(dot(d, d));
      mx = mx + x[k]; my = my + y[k];
    }
  }
  sg = im_wsum(sg); sl = im_wsum(sl); sv = im_wsum(sv); sa = im_wsum(sa); sr = im_wsum(sr);
  const float inv = 1.0f / (float)J;
  mx = inv * v3(im_wsum(mx.x), im_wsum(mx.y), im_wsum(mx.z));
  my = inv * v3(im_wsum(my.x), im_wsum(my.y), im_wsum(my.z));
  // pass 2: centred points, cross-covariance S[a][b] = sum y0_a x0_b and |Y0|^2
  float S[3][3], ny = 0.f;
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int c = 0; c < 3; c++) S[r][c] = 0.f;
#pragma unroll
  for (int k = 0; k < 2; k++) {
    if (lane + 32 * k < J) {
      x[k] = x[k] - mx; y[k] = y[k] - my;
      const float yy[3] = {y[k].x, y[k].y, y[k].z}, xx[3] = {x[k].x, x[k].y, x[k].z};
#pragma unroll
      for (int r = 0; r < 3; r++)
#pragma unroll
        for (int c = 0; c < 3; c++) S[r][c] = fmaf(yy[r], xx[c], S[r][c]);
      ny += dot(y[k], y[k]);
    }
  }
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int c = 0; c < 3; c++) S[r][c] = im_wsum(S[r][c]);
  ny = im_wsum(ny);
  Q4 q;
  const float lam = te_horn(S, q);
  const float qn = rsqrtf(q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z);
  q.w *= qn; q.x *= qn; q.y *= qn; q.z *= qn;
  float R[3][3];
  te_qmat(q, R);
  const float scale = ny > 0.f ? lam / ny : 0.f;   // all simulated points at one place: no scale, the aligned points sit at the mean
  // pass 3: aligned error |scale Q y0 - x0|
  float sp = 0.f;
#pragma unroll
  for (int k = 0; k < 2; k++) {
    if (lane + 32 * k < J) {
      const V3 ry = v3(R[0][0] * y[k].x + R[0][1] * y[k].y + R[0][2] * y[k].z, R[1][0] * y[k].x + R[1][1] * y[k].y + R[1][2] * y[k].z,
                       R[2][0] * y[k].x + R[2][1] * y[k].y + R[2][2] * y[k].z);
      const V3 d = scale * ry - x[k];
      sp += sqrtf(dot(d, d));
    }
  }
  sp = im_wsum(sp);
  if (lane == 0) {
    const float nan = __int_as_float(0x7fc00000);
    const float m[TE_NMETRIC] = {1000.f * (sg * inv), 1000.f * (sl * inv), 1000.f * (sp * inv), f >= 1 ? 1000.f * (sv * inv) : nan,
                                 f >= 2 ? 1000.f * (sa * inv) : nan, sr * inv};
    double* s = t.sums + (size_t)e * TE_NMETRIC;
#pragma unroll
    for (int i = 0; i < TE_NMETRIC; i++)
      if (i < 3 || i == 5 || (i == 3 && f >= 1) || (i == 4 && f >= 2)) s[i] += (double)m[i];
    if (t.frame_metrics) {
#pragma unroll
      for (int i = 0; i < TE_NMETRIC; i++) t.frame_metrics[(size_t)e * TE_NMETRIC + i] = m[i];
    }
    t.frames[e] = f + 1;
    const bool term = t.terminated[e] != 0, trunc = t.truncated[e] != 0;
    if (term || trunc) {
      t.active[e] = 0;
      t.success[e] = (trunc && !term) ? 1 : 0;
    }
  }
}
