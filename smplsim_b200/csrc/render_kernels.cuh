// render_kernels.cuh -- batched ray casting (MuJoCo's mj_ray) and camera images of the robot geoms and the floor plane.
//
// Reads body poses xpos [n, nbody, 3] / xquat [n, nbody, 4] (the rows of SmplsimAux.xpos / xquat) and the handle's constant table;
// writes only the caller's outputs.  Nothing here runs in the stepper.
//
// Geometry (fp32 throughout)
//   * per CTA, every robot geom of the CTA's env is staged in shared memory in world coordinates: centre xpos_b + R_b geom_pos,
//     axes R_b geom_mat (R_b from xquat_b, normalised here: motion tables need not hold unit quaternions), half sizes, type, body
//     and a bounding radius (sphere r, capsule r + h, box |size|).  A per-env-shapes handle takes env i's table;
//   * intersection in the geom's local frame, closed form: sphere; capsule = cylinder |z| <= h plus the two end hemispheres;
//     box = slab method; floor = the table's plane (plane_pos, plane_normal), infinite.  The result is the smallest x >= 0 with
//     pnt + x vec on the surface, so a ray that starts inside a geom hits it on the way out, and the plane is hit from its front
//     side only [MJ-upstream: mj_ray / mju_rayGeom, engine_ray.c].  Geom margins are ignored, as in mj_ray [MJ-upstream].
//     A geom whose bounding sphere the ray misses is rejected before the closed form.  Ties go to the lower MuJoCo geom id.
//
// k_ray: caller rays pnt[n,R,3], vec[n,R,3] -> dist[n,R] (x with the hit at pnt + x vec: vec need not be unit) and geomid[n,R]
//   (0 floor, i + 1 robot geom i); -1 / -1 for no hit.  flg_static = 0 skips the floor; bodyexclude >= 0 skips that body's geoms.
//
// k_render: one camera, one image per env.  Camera frame as in MJCF: it looks along its -z axis, +y is up, +x right; fovy is
//   the vertical field of view in degrees and the horizontal one follows from width / height (square pixels).  Row 0 is the top
//   of the image (mujoco.Renderer's order), pixel (r, c) is shot through its centre:
//     d_cam = ((2 (c + 0.5) / W - 1) tan(fovy / 2) W / H,  (1 - 2 (r + 0.5) / H) tan(fovy / 2),  -1).
//   Camera modes (SmplsimCamera.mode): FIXED world pose; TRACKCOM world axes, position = robot centre of mass + pos (the COM is
//   computed here from the table's body masses and COM offsets); BODY pose in the frame of robot body `body`.  exclude_body
//   (-1 none) drops that body's geoms from the primary rays (a head camera does not see the inside of the head).
//   Outputs, each optional:
//     depth[n,H,W] float32  z-depth along the camera's viewing axis in metres (not the ray length); zfar where nothing is hit
//     seg[n,H,W]   int32    MuJoCo geom id (0 floor, i + 1 robot geom i), -1 none
//     rgb[n,H,W,3] uint8    the shading below
//   Work split: a CTA is a 32 x 8 pixel block of one env (8 warps of 8 x 4 pixel tiles).  Each warp culls the geom list against
//   its tile's frustum (bounding spheres), then each lane casts its pixel's ray over the short list.
//
// Shading (this project's formula; approximates the reference scene, it is not MuJoCo's OpenGL pipeline).  With the unit
// normal n facing the ray, camera forward f (-z axis), light direction l = (0, 0, -1) (the reference's tracking light) and
// albedo a:
//     c = clamp(a (0.1 + 0.4 max(0, -n.f) + 1.0 max(0, -n.l) s), 0, 1),   u8 = floor(255 c + 0.5)
//   0.1 / 0.4 are MuJoCo's default headlight ambient / diffuse [MJ-upstream].  s = 0 when a shadow ray from p + 1e-4 n towards
//   -l hits a robot geom (any body, exclude_body included), else 1; it is only cast when -n.l > 0, and a warp tests it only
//   against the geoms whose bounding sphere reaches over its points.
//   Albedo: robot geoms (0.8, 0.6, 0.4), the <default> rgba of the shipped MJCFs, or the caller's per-geom table; floor: a
//   checker of (0, 0, 0) / (0.8, 0.8, 0.8) in the plane's frame (x axis = world x projected on the plane, y = n x x), cell
//   (i, j) = (floor(u / E), floor(v / E)) black when i + j is even, E = R_CHECK_EDGE.  Background (no hit): t (0.4, 0.5, 0.6)
//   with t = (d_z + 1) / 2 of the unit ray direction, the skybox gradient to black.  Not reproduced: reflectance, specular,
//   the geom texture's marks, anti-aliasing.
#pragma once
#include "dev_model.cuh"
#include "lane_model.hpp"

#define R_THREADS 256
#define R_CTA_W 32   // a render CTA's pixel block: 4 x 2 warp tiles of 8 x 4 pixels
#define R_CTA_H 8
// floor checker edge: the texture holds 2 x 2 checks and repeats 60 times over the 200-m plane (texrepeat="60 60",
// size="100 100") [MJ-upstream: planes repeat the texture texrepeat times over the plane's extent]
#define R_CHECK_EDGE (200.0f / 120.0f)
#define R_SHADOW_EPS 1e-4f

struct RGeom { float c[3], rb; float R[9]; float s[3]; int type, body; };   // world centre, bounding radius, axes (row-major), half sizes

struct RScene {
  const float* gimg;     // the handle's tables, img_words floats each
  const int* env_img;    // [n] table of each env row (NULL: table 0)
  const float* xpos;     // [n, nb, 3]
  const float* xquat;    // [n, nb, 4]
  int img_words, geom_off, nb, ng;
  float p0[3], pn[3], pu[3], pv[3];   // floor: point, unit normal, in-plane axes of its frame
};
struct RRayArgs { RScene s; const float* pnt; const float* vec; float* dist; int* geomid; int nray, flg_static, bodyexclude; };
struct RRenderArgs {
  RScene s;
  SmplsimCamera cam;
  float* depth; int* seg; unsigned char* rgb;
  int W, H, tiles_x, tiles;
  float rgb_tab[3 * LM_MAXG];   // albedo per robot geom
};

__device__ __forceinline__ const float* r_img(const RScene& s, int env) {
  return s.gimg + (s.env_img ? (size_t)s.env_img[env] * (size_t)s.img_words : (size_t)0);
}

// body rotations and positions, then the world pose of every geom (all threads of the CTA; ends with a barrier)
__device__ __forceinline__ void r_stage(const RScene& s, int env, float* sbx, RGeom* sg) {
  const float* img = r_img(s, env);
  const LGeom* G = (const LGeom*)((const char*)img + s.geom_off);
  for (int b = threadIdx.x; b < s.nb; b += blockDim.x) {
    const float* xq = s.xquat + ((size_t)env * s.nb + b) * 4;
    const float* xp = s.xpos + ((size_t)env * s.nb + b) * 3;
    Q4 q; q.w = xq[0]; q.x = xq[1]; q.y = xq[2]; q.z = xq[3];
    q2mat(qnormalize(q), sbx + 12 * b);
    sbx[12 * b + 9] = xp[0]; sbx[12 * b + 10] = xp[1]; sbx[12 * b + 11] = xp[2];
  }
  __syncthreads();
  for (int g = threadIdx.x; g < s.ng; g += blockDim.x) {
    const LGeom& L = G[g];
    const float* Rb = sbx + 12 * L.body;
    RGeom& o = sg[g];
    st3(o.c, v3(Rb[9], Rb[10], Rb[11]) + mrot(Rb, ld3(L.pos)));
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) o.R[3 * i + j] = Rb[3 * i] * L.mat[j] + Rb[3 * i + 1] * L.mat[3 + j] + Rb[3 * i + 2] * L.mat[6 + j];
    o.s[0] = L.size[0]; o.s[1] = L.size[1]; o.s[2] = L.size[2];
    o.type = L.type; o.body = L.body;
    const float r = L.type == SMPLSIM_GEOM_SPHERE ? L.size[0] : L.type == SMPLSIM_GEOM_CAPSULE ? L.size[0] + L.size[1]
                                                                                                : sqrtf(dot(ld3(L.size), ld3(L.size)));
    o.rb = 1.001f * r;   // padded: the bound never clips the geom in fp32
  }
  __syncthreads();
}

// roots of |q + x v|^2 = r^2, a = |v|^2 > 0, taken about the ray's closest approach to the centre: no cancellation for grazing rays
__device__ __forceinline__ bool r_roots(V3 q, V3 v, float a, float r, float& x0, float& x1) {
  const float ia = 1.0f / a, tc = -dot(q, v) * ia;
  const V3 m = q + tc * v;
  const float c = dot(m, m) - r * r;
  if (c > 0.f) return false;
  const float h = sqrtf(-c * ia);
  x0 = tc - h; x1 = tc + h;
  return true;
}
__device__ __forceinline__ void r_take(float x, float& best) { if (x >= 0.f && (best < 0.f || x < best)) best = x; }

// world -> geom frame
__device__ __forceinline__ V3 r_local(const RGeom& g, V3 w) {
  return v3(g.R[0] * w.x + g.R[3] * w.y + g.R[6] * w.z, g.R[1] * w.x + g.R[4] * w.y + g.R[7] * w.z, g.R[2] * w.x + g.R[5] * w.y + g.R[8] * w.z);
}

// smallest x >= 0 with P + x V on the geom's surface, -1 if none
__device__ __forceinline__ float r_geom(const RGeom& g, V3 P, V3 V) {
  const V3 w = ld3(g.c) - P;
  const float ww = dot(w, w), rb2 = g.rb * g.rb;
  if (ww > rb2) {   // origin outside the bounding sphere: the ray must point at it and pass within rb of its centre
    const V3 cx = cross(w, V);
    if (dot(w, V) < 0.f || dot(cx, cx) > rb2 * dot(V, V)) return -1.f;
  }
  const V3 p = r_local(g, P - ld3(g.c)), v = r_local(g, V);
  float best = -1.f, x0, x1;
  if (g.type == SMPLSIM_GEOM_SPHERE) {
    if (r_roots(p, v, dot(v, v), g.s[0], x0, x1)) { r_take(x0, best); r_take(x1, best); }
  } else if (g.type == SMPLSIM_GEOM_CAPSULE) {
    const float r = g.s[0], h = g.s[1];
    const float a = v.x * v.x + v.y * v.y;
    if (a > 0.f && r_roots(v3(p.x, p.y, 0.f), v3(v.x, v.y, 0.f), a, r, x0, x1)) {
      if (fabsf(p.z + x0 * v.z) <= h) r_take(x0, best);
      if (fabsf(p.z + x1 * v.z) <= h) r_take(x1, best);
    }
    for (int k = 0; k < 2; k++) {   // end hemispheres at z = +h, -h
      const float sg = k ? -1.f : 1.f;
      const V3 q = v3(p.x, p.y, p.z - sg * h);
      if (r_roots(q, v, dot(v, v), r, x0, x1)) {
        if (sg * (p.z + x0 * v.z) >= h) r_take(x0, best);
        if (sg * (p.z + x1 * v.z) >= h) r_take(x1, best);
      }
    }
  } else {   // box: slab method
    float t0 = -3.0e38f, t1 = 3.0e38f;
    const float pp[3] = {p.x, p.y, p.z}, vv[3] = {v.x, v.y, v.z};
#pragma unroll
    for (int i = 0; i < 3; i++) {
      if (vv[i] != 0.f) {
        const float iv = 1.0f / vv[i], ta = (-g.s[i] - pp[i]) * iv, tb = (g.s[i] - pp[i]) * iv;
        t0 = fmaxf(t0, fminf(ta, tb)); t1 = fminf(t1, fmaxf(ta, tb));
      } else if (fabsf(pp[i]) > g.s[i]) {
        return -1.f;
      }
    }
    if (t1 >= t0 && t1 >= 0.f) best = t0 >= 0.f ? t0 : t1;
  }
  return best;
}

// outward unit normal of the geom at surface point X
__device__ __forceinline__ V3 r_normal(const RGeom& g, V3 X) {
  const V3 q = r_local(g, X - ld3(g.c));
  V3 n;
  if (g.type == SMPLSIM_GEOM_SPHERE) n = q;
  else if (g.type == SMPLSIM_GEOM_CAPSULE) n = v3(q.x, q.y, q.z - fminf(fmaxf(q.z, -g.s[1]), g.s[1]));
  else {   // the face the point is closest to
    const float dx = fabsf(q.x) - g.s[0], dy = fabsf(q.y) - g.s[1], dz = fabsf(q.z) - g.s[2];
    if (dx >= dy && dx >= dz) n = v3(q.x >= 0.f ? 1.f : -1.f, 0.f, 0.f);
    else if (dy >= dz) n = v3(0.f, q.y >= 0.f ? 1.f : -1.f, 0.f);
    else n = v3(0.f, 0.f, q.z >= 0.f ? 1.f : -1.f);
  }
  n = mrot(g.R, n);
  return (1.0f / sqrtf(dot(n, n))) * n;
}

// floor plane, hit from its front side only
__device__ __forceinline__ float r_plane(const RScene& s, V3 P, V3 V) {
  const V3 n = ld3(s.pn);
  const float dn = dot(n, V), h = dot(n, P - ld3(s.p0));
  if (dn >= 0.f || h < 0.f) return -1.f;
  return -h / dn;
}

__global__ void __launch_bounds__(R_THREADS) k_ray(RRayArgs a) {
  __shared__ float sbx[12 * LM_MAXB];
  __shared__ RGeom sg[LM_MAXG];
  const int per = (a.nray + R_THREADS - 1) / R_THREADS;
  const int env = blockIdx.x / per, i = (blockIdx.x % per) * R_THREADS + threadIdx.x;
  r_stage(a.s, env, sbx, sg);
  if (i >= a.nray) return;
  const size_t r = (size_t)env * a.nray + i;
  const V3 P = ld3(a.pnt + 3 * r), V = ld3(a.vec + 3 * r);
  float best = -1.f;
  int gid = -1;
  if (dot(V, V) > 0.f) {
    if (a.flg_static) { best = r_plane(a.s, P, V); if (best >= 0.f) gid = 0; }
    for (int g = 0; g < a.s.ng; g++) {
      if (sg[g].body == a.bodyexclude) continue;
      const float x = r_geom(sg[g], P, V);
      if (x >= 0.f && (best < 0.f || x < best)) { best = x; gid = g + 1; }
    }
  }
  if (a.dist) a.dist[r] = best;
  if (a.geomid) a.geomid[r] = gid;
}

// camera position and world axes (thread 0; after r_stage).  PRM: the handle has per-env parameter records (LHdr::prm), whose mass
// scales weight the TRACKCOM centre of mass; the instance without them is the one every other call runs.
template <int PRM>
__device__ __forceinline__ void r_camera(const RRenderArgs& a, int env, const float* sbx, float* sc) {
  const SmplsimCamera& c = a.cam;
  V3 e = ld3(c.pos);
  V3 ax[3] = {v3(c.mat[0], c.mat[3], c.mat[6]), v3(c.mat[1], c.mat[4], c.mat[7]), v3(c.mat[2], c.mat[5], c.mat[8])};
  if (c.mode == SMPLSIM_CAM_TRACKCOM) {   // robot centre of mass, in body order
    const LBody* B = (const LBody*)((const char*)r_img(a.s, env) + LM_BODY_OFF);
    const float* msc = nullptr;   // (PRM) this env's mass scales: record words [4 + 3 nu, 4 + 3 nu + nb) (LCfg::PRM_MS)
    if constexpr (PRM != 0) {
      const LHdr& H = *(const LHdr*)r_img(a.s, env);
      msc = H.prm + (size_t)env * (size_t)((4 + 3 * H.nu + H.nb + 3) & ~3) + 4 + 3 * H.nu;
    }
    V3 mc = v3(0.f, 0.f, 0.f);
    float m = 0.f;
    for (int b = 0; b < a.s.nb; b++) {
      const float* Rb = sbx + 12 * b;
      float mb = B[b].mass;
      if constexpr (PRM != 0) mb *= __ldg(msc + b);
      mc = mc + mb * (v3(Rb[9], Rb[10], Rb[11]) + mrot(Rb, ld3(B[b].ipos)));
      m += mb;
    }
    e = e + (1.0f / m) * mc;
  } else if (c.mode == SMPLSIM_CAM_BODY) {
    const float* Rb = sbx + 12 * c.body;
    e = v3(Rb[9], Rb[10], Rb[11]) + mrot(Rb, e);
    for (int k = 0; k < 3; k++) ax[k] = mrot(Rb, ax[k]);
  }
  st3(sc, e); st3(sc + 3, ax[0]); st3(sc + 6, ax[1]); st3(sc + 9, ax[2]);
}

__device__ __forceinline__ bool r_shadowed(const RGeom* sg, const unsigned* smask, V3 P) {
  const V3 up = v3(0.f, 0.f, 1.f);   // -l
#pragma unroll
  for (int k = 0; k < 2; k++) {
    unsigned m = smask[k];
    while (m) {
      const int g = __ffs((int)m) - 1 + 32 * k;
      m &= m - 1u;
      if (r_geom(sg[g], P, up) >= 0.f) return true;
    }
  }
  return false;
}

__device__ __forceinline__ unsigned char r_u8(float c) { return (unsigned char)floorf(255.0f * fminf(fmaxf(c, 0.f), 1.f) + 0.5f); }

template <int PRM>
__global__ void __launch_bounds__(R_THREADS) k_render(RRenderArgs a) {
  __shared__ float sbx[12 * LM_MAXB];
  __shared__ RGeom sg[LM_MAXG];
  __shared__ float sc[12];
  const int env = blockIdx.x / a.tiles, tile = blockIdx.x % a.tiles;
  r_stage(a.s, env, sbx, sg);
  if (threadIdx.x == 0) r_camera<PRM>(a, env, sbx, sc);
  __syncthreads();
  const V3 e = ld3(sc), cx = ld3(sc + 3), cy = ld3(sc + 6), cz = ld3(sc + 9);
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c0 = (tile % a.tiles_x) * R_CTA_W + (wid & 3) * 8, r0 = (tile / a.tiles_x) * R_CTA_H + (wid >> 2) * 4;
  const float ty = tanf(a.cam.fovy * (3.14159265358979f / 360.0f)), tx = ty * (float)a.W / (float)a.H;
  const float iW = 1.0f / (float)a.W, iH = 1.0f / (float)a.H;
  // the warp tile's frustum: four planes through the eye, pass when the bounding sphere reaches the inner side
  unsigned mask[2];
  {
    const float xl = (2.f * c0 * iW - 1.f) * tx, xh = (2.f * (c0 + 8) * iW - 1.f) * tx;
    const float yt = (1.f - 2.f * r0 * iH) * ty, yb = (1.f - 2.f * (r0 + 4) * iH) * ty;
#pragma unroll
    for (int k = 0; k < 2; k++) {
      const int g = lane + 32 * k;
      bool pass = false;
      if (g < a.s.ng && sg[g].body != a.cam.exclude_body) {
        const V3 w = ld3(sg[g].c) - e;
        const float qx = dot(w, cx), qy = dot(w, cy), qz = dot(w, cz), rb = sg[g].rb;
        pass = -qz >= -rb && qx + xl * qz >= -rb * sqrtf(1.f + xl * xl) && -qx - xh * qz >= -rb * sqrtf(1.f + xh * xh) &&
               qy + yb * qz >= -rb * sqrtf(1.f + yb * yb) && -qy - yt * qz >= -rb * sqrtf(1.f + yt * yt);
      }
      mask[k] = __ballot_sync(0xffffffffu, pass);
    }
  }
  const int col = c0 + (lane & 7), row = r0 + (lane >> 3);
  const bool in = col < a.W && row < a.H;   // lanes off the image stay for the warp collectives below and write nothing
  const float u = (2.f * ((float)col + 0.5f) * iW - 1.f) * tx, v = (1.f - 2.f * ((float)row + 0.5f) * iH) * ty;
  const V3 D = u * cx + v * cy - cz;   // camera z component -1: the hit distance is the z-depth
  float best = r_plane(a.s, e, D);
  int gid = best >= 0.f ? 0 : -1;
#pragma unroll
  for (int k = 0; k < 2; k++) {
    unsigned m = mask[k];
    while (m) {
      const int g = __ffs((int)m) - 1 + 32 * k;
      m &= m - 1u;
      const float x = r_geom(sg[g], e, D);
      if (x >= 0.f && (best < 0.f || x < best)) { best = x; gid = g + 1; }
    }
  }
  const size_t px = ((size_t)env * a.H + row) * a.W + col;
  if (in && a.depth) a.depth[px] = gid >= 0 ? best : a.cam.zfar;
  if (in && a.seg) a.seg[px] = gid;
  if (!a.rgb) return;
  const V3 X = e + best * D;
  V3 n = v3(0.f, 0.f, 0.f), alb = v3(0.f, 0.f, 0.f);
  if (gid == 0) {
    n = ld3(a.s.pn);
    const V3 d = X - ld3(a.s.p0);
    const int k = (int)floorf(dot(d, ld3(a.s.pu)) * (1.0f / R_CHECK_EDGE)) + (int)floorf(dot(d, ld3(a.s.pv)) * (1.0f / R_CHECK_EDGE));
    const float gr = (k & 1) ? 0.8f : 0.f;
    alb = v3(gr, gr, gr);
  } else if (gid > 0) {
    n = r_normal(sg[gid - 1], X);
    if (dot(n, D) > 0.f) n = -1.f * n;
    alb = ld3(a.rgb_tab + 3 * (gid - 1));
  }
  // shadow rays go straight up (-l): a geom can only shade the warp's points if its bounding sphere reaches over their xy box and
  // above their lowest point; the warp culls the geom list against that, then each lane walks the short list
  const bool shade = in && gid >= 0 && n.z > 0.f;
  const V3 S = X + R_SHADOW_EPS * n;
  float x0 = shade ? S.x : 3.0e38f, x1 = shade ? S.x : -3.0e38f, y0 = shade ? S.y : 3.0e38f, y1 = shade ? S.y : -3.0e38f;
  float z0 = shade ? S.z : 3.0e38f;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    x0 = fminf(x0, __shfl_xor_sync(0xffffffffu, x0, o)); x1 = fmaxf(x1, __shfl_xor_sync(0xffffffffu, x1, o));
    y0 = fminf(y0, __shfl_xor_sync(0xffffffffu, y0, o)); y1 = fmaxf(y1, __shfl_xor_sync(0xffffffffu, y1, o));
    z0 = fminf(z0, __shfl_xor_sync(0xffffffffu, z0, o));
  }
  unsigned smask[2];
#pragma unroll
  for (int k = 0; k < 2; k++) {
    const int g = lane + 32 * k;
    bool pass = false;
    if (g < a.s.ng) {
      const RGeom& G = sg[g];
      const float dx = fmaxf(fmaxf(x0 - G.c[0], G.c[0] - x1), 0.f), dy = fmaxf(fmaxf(y0 - G.c[1], G.c[1] - y1), 0.f);
      pass = dx * dx + dy * dy <= G.rb * G.rb && G.c[2] + G.rb >= z0;
    }
    smask[k] = __ballot_sync(0xffffffffu, pass);
  }
  if (!in) return;
  V3 c;
  if (gid < 0) {
    const float t = 0.5f * (D.z / sqrtf(dot(D, D)) + 1.f);
    c = v3(0.4f * t, 0.5f * t, 0.6f * t);
  } else {
    float lit = 0.1f + 0.4f * fmaxf(0.f, dot(n, cz));   // -n.f with f = -cz
    if (shade && !r_shadowed(sg, smask, S)) lit += n.z;   // -n.l = n.z
    c = lit * alb;
  }
  unsigned char* o = a.rgb + 3 * px;
  o[0] = r_u8(c.x); o[1] = r_u8(c.y); o[2] = r_u8(c.z);
}
