// smplsim_capi.cu -- extern "C" boundary of libsmplsim_b200.so (see include/smplsim.h).
// Host side: constant table + lane schedule (lane_model.hpp), shared-memory sizing, launches of the lane-chain kernels.
#include <cuda_runtime.h>

#include <cmath>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "aux_kernels.cuh"
#include "imitation_kernels.cuh"
#include "track_eval_kernels.cuh"
#include "amp_kernels.cuh"
#include "render_kernels.cuh"

#ifdef SMPLSIM_EMU
#define L_LAUNCH(kern, grid, block, smem, stream, ...) emu::launch(dim3(grid), dim3(block), smem, [&]() { kern(__VA_ARGS__); })
#else
#define L_LAUNCH(kern, grid, block, smem, stream, ...) kern<<<grid, block, smem, stream>>>(__VA_ARGS__)
#endif


struct SmplsimHandle {
  LaneImage img;
  float* dimg = nullptr;   // device copy of the table
  float* gscr = nullptr;   // per-env global scratch: lane records, qstar, overflow contact entries
  float* gsens = nullptr;  // body velocities of the last forward pass (obs v2 / aux)
  int* gpfl = nullptr;     // working set per contact slot, carried from call to call (solver warm start only)
  float* gbody = nullptr;  // body pose / velocity of the current forward pass (self-collision narrow phase)
  float* gfd = nullptr;    // per-env qacc / qfrc of a column's first pass (smplsim_transition_fd, smplsim_inverse_fd; handles without self-collision)
  float* groll = nullptr;  // per-env qpos, qvel, qpos_fwd, qvel_fwd at a rollout's step boundary (smplsim_rollout; as gfd)
  float* gfb = nullptr;    // per-env dx [2nv] and u [nu] of a closed-loop rollout step (smplsim_rollout_feedback; as gfd)
  int num_envs = 0, device = 0, nsm = 132, max_smem = 0;
  int cls = 0;             // 1 SMPL class, 2 SMPL-X class
  int selfcol = 0;         // cfg.env.self_collision: kernels with the geom-geom rows compiled in
  int wpb = 0;             // warps per CTA
  size_t smem = 0, env_words = 0;
  // per-env body shapes (smplsim_create_shapes): envs grouped by shape into whole CTAs
  std::vector<int> env_model;   // [num_envs] or empty (one shape)
  int nmodels = 1, nblocks = 0;
  int* dslot_env = nullptr;     // [nblocks * warps per CTA * envs per warp] slot -> env (-1: none)
  int* dblk_img = nullptr;      // [nblocks] CTA -> table
  int* denv_model = nullptr;    // [num_envs] env -> table (device copy of env_model; ray casting and rendering)
  LMap map() const { LMap m; m.slot_env = dslot_env; m.blk_img = dblk_img; return m; }
  // per-env physics parameters (smplsim_set_env_params): prmw words per env; NULL: none, and the kernels without them run
  float* prm = nullptr;
  int prmw = 0;
  double ctrl_dt = 0;      // control period: model.timestep * nsubsteps (smplsim_imitation)
};

static thread_local std::string g_err;
static int fail(int code, const std::string& msg) { g_err = msg; return code; }
// every entry of the caller's body list body[0, n) is a robot body index in [0, nb)
static bool bodies_in_range(const int32_t* body, int n, int nb) {
  for (int j = 0; j < n; j++)
    if (body[j] < 0 || body[j] >= nb) return false;
  return true;
}
#define CUDA_TRY(x)                                                                                     \
  do {                                                                                                  \
    cudaError_t e_ = (x);                                                                               \
    if (e_ != cudaSuccess) return fail(SMPLSIM_ECUDA, std::string(#x) + ": " + cudaGetErrorString(e_)); \
  } while (0)

struct DeviceGuard {   // every entry point runs on the handle's device and restores the caller's
  int prev = -1;
  explicit DeviceGuard(int dev) { if (cudaGetDevice(&prev) != cudaSuccess) prev = -1; if (prev != dev) cudaSetDevice(dev); else prev = -1; }
  ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

extern "C" const char* smplsim_last_error(void) { return g_err.c_str(); }
extern "C" int smplsim_version(void) { return 300; }   // 300: smplsim_track_eval; 290: smplsim_motion_blend, blended / future imitation targets, blended AMP frames; 280: smplsim_amp_obs / smplsim_amp_demo; 270: smplsim_imitation; 260: smplsim_set_env_params; 250: smplsim_ray / smplsim_render; 240: smplsim_dynamics; 230: smplsim_inverse; 220: SmplsimAux.contact_wrench; 210: SmplsimState.xfrc_applied; 200: lane-chain kernels (ABI structs of 110)

template <class C>
static size_t cta_smem(const SmplsimHandle* h, int wpb) { return (size_t)h->img.hdr()->bytes + 16 + (size_t)wpb * C::EPW * C::total * 4; }

// CTAs of a launch over all envs: every CTA holds envs of one body shape
static long count_blocks(const SmplsimHandle* h, long per) {
  if (h->env_model.empty()) return (h->num_envs + per - 1) / per;
  std::vector<long> cnt(h->nmodels, 0);
  for (int m : h->env_model) cnt[m]++;
  long b = 0;
  for (long c : cnt) b += (c + per - 1) / per;
  return b;
}

// The lane kernels a handle of class C may launch.  pick_wpb raises the shared-memory cap of every entry and the launches take their
// kernel from here, so that no instance runs under the default cap.
struct LaneKernels {
  void (*step[3])(const float*, int, LStepArgs, const float*, float*);   // [0 plain, 1 external wrench, 2 wrench + parameter records]
  void (*reset[2])(const float*, int, LResetArgs);                      // [parameter records]
  void (*kin)(const float*, int, LKinArgs);
  void (*inverse[2])(const float*, int, LInvArgs);                      // [parameter records]
  void (*dyn[2])(const float*, int, LDynArgs);                          // [parameter records]
  void (*fwd[2])(const float*, int, LFwdArgs);                          // [parameter records]
  void (*roll[2])(const float*, int, LRollArgs);                        // [parameter records]
  void (*rollfb[2])(const float*, int, LRollFbArgs);                    // [parameter records]
  void (*invfd)(const float*, int, LInvFdArgs);                         // single shape, no parameter records
  void (*cent[2])(const float*, int, LCentArgs);                        // [parameter records]
  void (*rnep[2])(const float*, int, LRnepArgs);                        // [parameter records]
};
template <class C>
static LaneKernels lane_kernels() {
  typedef typename C::WithPrm P;
  LaneKernels k = {{k_step5<C>, k_step5<typename C::WithXfrc>, k_step5<typename C::WithXfrcPrm>}, {k_reset5<C>, k_reset5<P>}, k_kin5<C>, {}, {}};
  // a self-collision class has no inverse instances (smplsim_inverse refuses such handles): NULL entries, so that none is compiled
  if constexpr (!C::SELFCOL) { k.inverse[0] = k_inverse5<C>; k.inverse[1] = k_inverse5<P>; }
  k.dyn[0] = k_dyn5<C>; k.dyn[1] = k_dyn5<P>;
  if constexpr (!C::SELFCOL) { k.fwd[0] = k_fwd5<C>; k.fwd[1] = k_fwd5<P>; }   // as inverse: none for a self-collision class
  if constexpr (!C::SELFCOL) lane_roll_kernels(C::NB == L_SMPL(0)::NB ? 1 : 2, k.roll);   // a module of its own (rollout_kernels.cu)
  if constexpr (!C::SELFCOL) lane_rollfb_kernels(C::NB == L_SMPL(0)::NB ? 1 : 2, k.rollfb);   // as roll (rollout_feedback_kernels.cu)
  if constexpr (!C::SELFCOL) lane_invfd_kernels(C::NB == L_SMPL(0)::NB ? 1 : 2, &k.invfd);   // as roll (inverse_fd_kernels.cu)
  lane_cent_kernels(C::NB == L_SMPL(0)::NB ? 1 : 2, C::SELFCOL, k.cent);   // as roll (centroidal_kernels.cu); every class, as dyn
  if constexpr (!C::SELFCOL) lane_rnep_kernels(C::NB == L_SMPL(0)::NB ? 1 : 2, k.rnep);   // as roll (rne_post_kernels.cu); as inverse
  return k;
}

// warps per CTA: fewest waves over the SMs first, then the fewest warps (an SM issues faster for few resident warps)
template <class C>
static int pick_wpb(SmplsimHandle* h) {
  int best = 0;
  long best_waves = 1L << 60;
  int forced = 0;
  if (const char* f = std::getenv("SMPLSIM_WPB")) forced = std::atoi(f);
  for (int wpb = 1; wpb <= 8; wpb++) {
    if (forced && wpb != forced) continue;
    if (cta_smem<C>(h, wpb) > (size_t)h->max_smem) continue;
    long per = (long)wpb * C::EPW, blocks = count_blocks(h, per), waves = (blocks + h->nsm - 1) / h->nsm;
    if (waves < best_waves) { best_waves = waves; best = wpb; }
  }
  if (!best) return -1;
  h->wpb = best;
  h->smem = cta_smem<C>(h, best);
  h->env_words = C::total;
  // The shared-memory cap is an attribute of the kernel for the whole process, not of this handle: raise it to the device's
  // opt-in limit rather than to this handle's need, so that a handle created later with smaller CTAs (fewer envs) does not
  // lower the cap under the launches of a live handle with larger ones.  The lane kernels declare no static __shared__ (their
  // only shared memory is the dynamic l_smem4), so the whole opt-in limit is a legal dynamic cap for each of them.
  auto raise = [cap = h->max_smem](auto... k) {   // in order, stopping at the first failure
    return ((!k || cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, cap) == cudaSuccess) && ...);
  };
  const LaneKernels K = lane_kernels<C>();
  if (!raise(K.step[0], K.step[1], K.step[2], K.reset[0], K.reset[1], K.kin, K.inverse[0], K.inverse[1], K.dyn[0], K.dyn[1], K.fwd[0], K.fwd[1],
             K.roll[0], K.roll[1], K.rollfb[0], K.rollfb[1], K.invfd, K.cent[0], K.cent[1], K.rnep[0], K.rnep[1])) return -1;
  return best;
}

// One launch of a lane kernel over `rows` envs, or over the handle's CTAs when it groups envs by body shape
template <class C, class K, class... A>
static void lane_launch(const SmplsimHandle* h, K kern, int rows, cudaStream_t st, const A&... args) {
  const int per = h->wpb * C::EPW, grid = h->nblocks ? h->nblocks : (rows + per - 1) / per;
  L_LAUNCH(kern, grid, 32 * h->wpb, h->smem, st, h->dimg, h->img.hdr()->bytes, args...);
}
// inverse / dynamics on n caller rows of state.  One shape without parameter records: launches of at most num_envs rows (the
// handle's scratch rows), in order on the caller's stream, `advance` moving every row pointer of a chunk to its first row.  Otherwise
// (env_rows holds n == num_envs) one launch, of the instance that reads the records while the handle has them (row i = env i).
template <class A> static int& row_count(A& a) { return a.n; }
static int& row_count(LRollFbArgs& a) { return a.r.n; }   // the rows of the closed-loop rollout are its rollout's
template <class C, class A, class F>
static void state_rows(const SmplsimHandle* h, void (*const kern[2])(const float*, int, A), const A& a, F advance, cudaStream_t st) {
  const int n = row_count(const_cast<A&>(a));
  if (h->prm || h->nblocks) return lane_launch<C>(h, kern[h->prm ? 1 : 0], n, st, a);
  for (int r0 = 0; r0 < n; r0 += h->num_envs) {
    A c = a;
    row_count(c) = std::min(h->num_envs, n - r0);
    advance(c, (size_t)r0);
    lane_launch<C>(h, kern[0], row_count(c), st, c);
  }
}
// dispatch over (model class, self-collision)
#define L_DISPATCH(h, CALL)                                                   \
  do {                                                                        \
    switch (((h)->cls << 1) | (h)->selfcol) {                                 \
      case (1 << 1) | 0: { typedef L_SMPL(0) C_; CALL; } break;               \
      case (1 << 1) | 1: { typedef L_SMPL(1) C_; CALL; } break;               \
      case (2 << 1) | 0: { typedef L_SMPLX(0) C_; CALL; } break;              \
      default: { typedef L_SMPLX(1) C_; CALL; } break;                        \
    }                                                                         \
  } while (0)

static void free_handle(SmplsimHandle* h) {
  cudaFree(h->prm); cudaFree(h->dimg); cudaFree(h->gscr); cudaFree(h->gsens); cudaFree(h->gpfl); cudaFree(h->gbody); cudaFree(h->gfd); cudaFree(h->groll); cudaFree(h->gfb); cudaFree(h->dslot_env); cudaFree(h->dblk_img); cudaFree(h->denv_model);
  delete h;
}

// tables of two body shapes can share the kernels' schedule iff the tree, the joints and the geom layout agree
static bool same_structure(const LaneImage& a, const LaneImage& b) {
  const LHdr& A = *a.hdr(); const LHdr& B = *b.hdr();
  if (A.bytes != B.bytes || A.nb != B.nb || A.nv != B.nv || A.nu != B.nu || A.ng != B.ng || A.nslot != B.nslot || A.nmbi != B.nmbi || A.nmbo != B.nmbo ||
      A.T != B.T || A.npair != B.npair || A.obs_dim != B.obs_dim || std::memcmp(A.sched, B.sched, sizeof A.sched) != 0) return false;
  for (int i = 0; i < A.nb; i++) {
    const LBody& x = a.bodies()[i]; const LBody& y = b.bodies()[i];
    if (x.parent != y.parent || x.dofadr != y.dofadr || x.flags != y.flags || x.geom0 != y.geom0 || x.ngeom != y.ngeom || x.limited != y.limited ||
        x.in_mbox != y.in_mbox || x.out_mbox != y.out_mbox || x.pmbox != y.pmbox || x.nmb != y.nmb || x.step != y.step || x.lane != y.lane) return false;
  }
  return true;
}

static int create_impl(const SmplsimModelDesc* s, int nmodels, const int32_t* env_model, const SmplsimEnvCfg* cfg, int num_envs, int cuda_device, SmplsimHandle** out) {
  if (!s || !cfg || !out || num_envs <= 0 || nmodels < 1) return fail(SMPLSIM_EINVAL, "smplsim_create: null argument or num_envs <= 0");
  if (nmodels > 1 && !env_model) return fail(SMPLSIM_EINVAL, "smplsim_create_shapes: env_model is NULL");
  if (env_model) for (int i = 0; i < num_envs; i++) if (env_model[i] < 0 || env_model[i] >= nmodels) return fail(SMPLSIM_EINVAL, "smplsim_create_shapes: env_model entry out of range");
  if (cfg->self_obs_v != 1 && cfg->self_obs_v != 2) return fail(SMPLSIM_EINVAL, "self_obs_v must be 1 or 2");
  if (cfg->control_mode < 0 || cfg->control_mode > 3) return fail(SMPLSIM_EINVAL, "control_mode must be uhc_pd|pd|torque|simple_pid");
  if (cfg->task < 0 || cfg->task > 3) return fail(SMPLSIM_EINVAL, "unknown task");
  if (cfg->nsubsteps < 1) return fail(SMPLSIM_EINVAL, "nsubsteps < 1");
  if (cfg->task == SMPLSIM_TASK_REACH && (cfg->reach_body < 0 || cfg->reach_body >= s->nbody)) return fail(SMPLSIM_EINVAL, "reach_body out of range");
  SmplsimHandle* h = new SmplsimHandle();
  std::string why = lane_build(s, cfg, h->img);
  if (!why.empty()) { delete h; return fail(SMPLSIM_EUNSUPPORTED, why); }
  LHdr& H = *h->img.hdr();
  { const char* dp = std::getenv("SMPLSIM_DIRTYPATH"); if (dp) H.dirtypath = std::atoi(dp); }
  { const char* ax = std::getenv("SMPLSIM_AXES"); if (ax && std::string(ax) == "generic") H.axes_xyz = 0; }   // FK through the general hinge-axis path
  { const char* al = std::getenv("SMPLSIM_ALIGN"); if (al) H.align = std::atoi(al); }
  if (H.align & 16) H.align |= 8;   // barriers at every sweep step need CTA-uniform solver iteration counts (else the warps disagree on the number of sweeps: deadlock)   // CTA phase-alignment barriers (bit 0 substep, 1 solve, 2 stable-PD sweep)
  for (int b = 0; b < H.nb; b++) if (h->img.bodies()[b].ngeom > 1) { delete h; return fail(SMPLSIM_EUNSUPPORTED, "more than one geom on a body"); }
  std::vector<LaneImage> more(nmodels > 1 ? nmodels - 1 : 0);   // tables of the other body shapes
  for (int k = 1; k < nmodels; k++) {
    std::string w2 = lane_build(s + k, cfg, more[k - 1]);
    if (!w2.empty()) { delete h; return fail(SMPLSIM_EUNSUPPORTED, "body shape " + std::to_string(k) + ": " + w2); }
    LHdr& Hk = *more[k - 1].hdr();
    Hk.dirtypath = H.dirtypath; Hk.align = H.align;
    if (!same_structure(h->img, more[k - 1])) { delete h; return fail(SMPLSIM_EUNSUPPORTED, "body shape " + std::to_string(k) + " differs from shape 0 in tree / joints / geom layout (only offsets, sizes, masses and gains may differ)"); }
  }
  h->nmodels = nmodels;
  if (env_model && nmodels > 1) h->env_model.assign(env_model, env_model + num_envs);
  typedef L_SMPL(0) CS; typedef L_SMPLX(0) CX;
  if (H.nb == CS::NB && H.nv == CS::NV && H.ng <= CS::NG && H.nslot <= CS::NS && H.nmbi <= CS::NMBI && H.nmbo <= CS::NMBO) h->cls = 1;
  else if (H.nb == CX::NB && H.nv == CX::NV && H.ng <= CX::NG && H.nslot <= CX::NS && H.nmbi <= CX::NMBI && H.nmbo <= CX::NMBO) h->cls = 2;
  else {
    char msg[256];
    snprintf(msg, sizeof msg, "model is not one of the compiled classes (SMPL 24 bodies / SMPL-X 52 bodies): nb %d nv %d ng %d slots %d mailboxes %d/%d",
             H.nb, H.nv, H.ng, H.nslot, H.nmbi, H.nmbo);
    delete h;
    return fail(SMPLSIM_EUNSUPPORTED, msg);
  }
  h->num_envs = num_envs; h->device = cuda_device; h->selfcol = cfg->self_collision ? 1 : 0;
  h->ctrl_dt = s->timestep * cfg->nsubsteps;
  DeviceGuard guard(cuda_device);
  cudaError_t e = cudaDeviceGetAttribute(&h->max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, cuda_device);
#ifndef SMPLSIM_EMU
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&h->nsm, cudaDevAttrMultiProcessorCount, cuda_device);
#endif
  if (e != cudaSuccess) { delete h; return fail(SMPLSIM_ECUDA, std::string("smplsim_create: ") + cudaGetErrorString(e)); }
  int ok = 0, per = 1;   // the class constants: warps per CTA (and its shared memory, in h), envs per CTA, scratch words per env
  size_t gs = 0, pw = 0;
  L_DISPATCH(h, ok = pick_wpb<C_>(h); per = h->wpb * C_::EPW; gs = C_::GSCRW; pw = C_::PFLW);
  if (ok <= 0) { delete h; return fail(SMPLSIM_EUNSUPPORTED, "per-env rows exceed shared memory"); }
  e = cudaMalloc(&h->dimg, (size_t)H.bytes * nmodels);
  if (e == cudaSuccess) e = cudaMemcpy(h->dimg, h->img.bytes.data(), H.bytes, cudaMemcpyHostToDevice);
  for (int k = 1; k < nmodels && e == cudaSuccess; k++) e = cudaMemcpy((char*)h->dimg + (size_t)H.bytes * k, more[k - 1].bytes.data(), H.bytes, cudaMemcpyHostToDevice);
  if (e == cudaSuccess && !h->env_model.empty()) {   // envs grouped by shape into whole CTAs (empty slots: -1)
    std::vector<int> slot_env, blk_img;
    for (int k = 0; k < nmodels; k++) {
      int fill = 0;
      for (int i = 0; i < num_envs; i++) {
        if (h->env_model[i] != k) continue;
        if (fill == 0) blk_img.push_back(k);
        slot_env.push_back(i);
        fill = (fill + 1) % per;
      }
      while (fill != 0) { slot_env.push_back(-1); fill = (fill + 1) % per; }
    }
    h->nblocks = (int)blk_img.size();
    e = cudaMalloc(&h->dslot_env, slot_env.size() * sizeof(int));
    if (e == cudaSuccess) e = cudaMemcpy(h->dslot_env, slot_env.data(), slot_env.size() * sizeof(int), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMalloc(&h->dblk_img, blk_img.size() * sizeof(int));
    if (e == cudaSuccess) e = cudaMemcpy(h->dblk_img, blk_img.data(), blk_img.size() * sizeof(int), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMalloc(&h->denv_model, (size_t)num_envs * sizeof(int));
    if (e == cudaSuccess) e = cudaMemcpy(h->denv_model, h->env_model.data(), (size_t)num_envs * sizeof(int), cudaMemcpyHostToDevice);
  }
  if (e == cudaSuccess) e = cudaMalloc(&h->gscr, gs * (size_t)num_envs * 4 + 16);
  if (e == cudaSuccess) e = cudaMalloc(&h->gsens, (size_t)6 * H.nb * num_envs * 4);
  if (e == cudaSuccess) e = cudaMalloc(&h->gpfl, pw * num_envs * 4);
  if (e == cudaSuccess) e = cudaMemset(h->gpfl, 0, pw * num_envs * 4);
  if (e == cudaSuccess && cfg->self_collision) e = cudaMalloc(&h->gbody, (size_t)10 * H.nb * num_envs * 4);
  if (e == cudaSuccess && !cfg->self_collision) e = cudaMalloc(&h->gfd, (size_t)H.nv * num_envs * 4);
  if (e == cudaSuccess && !cfg->self_collision) e = cudaMalloc(&h->groll, (size_t)2 * (2 * H.nv + 1) * num_envs * 4);
  if (e == cudaSuccess && !cfg->self_collision) e = cudaMalloc(&h->gfb, (size_t)(2 * H.nv + H.nu) * num_envs * 4);
  if (e != cudaSuccess) { free_handle(h); return fail(SMPLSIM_ECUDA, std::string("smplsim_create: ") + cudaGetErrorString(e)); }
  if (std::getenv("SMPLSIM_DEBUG"))
    fprintf(stderr, "smplsim_create: class %d, %d bodies, schedule %d steps, mailboxes %d in / %d out, %d geom pairs, table %d B, %zu B per env, %d warps per CTA, %zu B shared memory per CTA, self-collision %d\n",
            h->cls, H.nb, H.T, H.nmbi, H.nmbo, H.npair, H.bytes, h->env_words * 4, h->wpb, h->smem, h->selfcol);
  *out = h;
  return SMPLSIM_OK;
}

extern "C" int smplsim_create(const SmplsimModelDesc* s, const SmplsimEnvCfg* cfg, int num_envs, int cuda_device, SmplsimHandle** out) {
  return create_impl(s, 1, nullptr, cfg, num_envs, cuda_device, out);
}
extern "C" int smplsim_create_shapes(const SmplsimModelDesc* models, int num_models, const int32_t* env_model, const SmplsimEnvCfg* cfg, int num_envs,
                                     int cuda_device, SmplsimHandle** out) {
  return create_impl(models, num_models, env_model, cfg, num_envs, cuda_device, out);
}
extern "C" int smplsim_num_shapes(const SmplsimHandle* h) { return h ? h->nmodels : SMPLSIM_EINVAL; }

extern "C" int smplsim_destroy(SmplsimHandle* h) {
  if (!h) return SMPLSIM_OK;
  DeviceGuard guard(h->device);
  free_handle(h);
  return SMPLSIM_OK;
}
extern "C" int smplsim_obs_dim(const SmplsimHandle* h) { return h ? h->img.hdr()->obs_dim : SMPLSIM_EINVAL; }
extern "C" int smplsim_num_envs(const SmplsimHandle* h) { return h ? h->num_envs : SMPLSIM_EINVAL; }
extern "C" int smplsim_smem_bytes_per_env(const SmplsimHandle* h) { return h ? (int)h->env_words * 4 : SMPLSIM_EINVAL; }
extern "C" int smplsim_warps_per_block(const SmplsimHandle* h) { return h ? h->wpb : SMPLSIM_EINVAL; }
/* 5: lane-chain kernels (lane_kernels.cuh) */
extern "C" int smplsim_kernel_version(const SmplsimHandle* h) { return h ? 5 : SMPLSIM_EINVAL; }
extern "C" int smplsim_schedule_steps(const SmplsimHandle* h) { return h ? h->img.hdr()->T : SMPLSIM_EINVAL; }

static float* aux_wrench(const SmplsimAux* aux) { return aux ? aux->contact_wrench : nullptr; }
static bool state_ok(const SmplsimState* st) {
  return st && st->qpos && st->qvel && st->qpos_fwd && st->qvel_fwd && st->qacc_warm && st->task_target && st->task_change_step &&
         st->progress && st->recovery && st->rng_counter;
}
// the arguments step, mj_step and reset share (LStepArgs, LResetArgs): state and side-output rows, the handle's scratch, every env
template <class A>
static A lane_args(const SmplsimHandle* h, const SmplsimState* st, const SmplsimAux* aux) {
  static_assert(sizeof(LState) == offsetof(SmplsimState, xfrc_applied), "LState must mirror SmplsimState up to xfrc_applied");
  static_assert(sizeof(LAux) == offsetof(SmplsimAux, contact_wrench), "LAux must mirror SmplsimAux up to contact_wrench");
  A a; std::memset(&a, 0, sizeof a);
  std::memcpy(&a.st, st, sizeof a.st);     // the rows before xfrc_applied, in the same order
  if (aux) std::memcpy(&a.aux, aux, sizeof a.aux);   // the rows before contact_wrench, in the same order (all NULL without aux)
  a.gscr = h->gscr; a.gpfl = h->gpfl; a.gbody = h->gbody; a.n = h->num_envs; a.map = h->map();
  const bool sens = h->img.hdr()->cfg.self_obs_v == 2 || (aux && (aux->body_linvel || aux->body_angvel));
  a.gsens = sens ? h->gsens : nullptr;
  return a;
}
// step and mj_step: the instance with the external-wrench code compiled in only when the caller passes xfrc_applied (same layout,
// shared memory and CTA size; without a wrench the kernel is the one without that code).  The contact wrench output is a run-time
// argument of every instance (NULL: not written).  While the handle has per-env parameter records, the instance with both the
// parameter reads and the wrench code runs (its wrench pointer may be NULL).
static int lane_step(const SmplsimHandle* h, const LStepArgs& a, const SmplsimState* st, const SmplsimAux* aux, void* stream) {
  const float* xfrc = st->xfrc_applied;
  L_DISPATCH(h, lane_launch<C_>(h, lane_kernels<C_>().step[h->prm ? 2 : xfrc ? 1 : 0], a.n, (cudaStream_t)stream, a, xfrc, aux_wrench(aux)));
  CUDA_TRY(cudaGetLastError());
  return SMPLSIM_OK;
}
// calls on n caller rows: with per-env body shapes, and for the kernels that read them (prm) per-env parameter records, row i is env i
static int env_rows(const SmplsimHandle* h, int n, const char* fn, bool prm) {
  if (h->nblocks && n != h->num_envs)
    return fail(SMPLSIM_EINVAL, std::string(fn) + ": with per-env body shapes n must be the handle's num_envs (row i uses env i's shape)");
  if (prm && h->prm && n != h->num_envs)
    return fail(SMPLSIM_EINVAL, std::string(fn) + ": with per-env parameters n must be the handle's num_envs (row i uses env i's parameters)");
  return SMPLSIM_OK;
}

extern "C" int smplsim_step(SmplsimHandle* h, const SmplsimState* st, const float* action_dev, float* obs_dev, float* reward_dev,
                            uint8_t* terminated_dev, uint8_t* truncated_dev, const SmplsimAux* aux, void* stream) {
  if (!h || !state_ok(st) || !action_dev) return fail(SMPLSIM_EINVAL, "smplsim_step: null handle/state/action");
  if (h->img.hdr()->cfg.control_mode == SMPLSIM_CTRL_SIMPLE_PID && (!st->pid_integral || !st->pid_last_error))
    return fail(SMPLSIM_EINVAL, "smplsim_step: control_mode simple_pid needs state.pid_integral / pid_last_error");
  DeviceGuard guard(h->device);
  LStepArgs a = lane_args<LStepArgs>(h, st, aux);
  a.action = action_dev; a.obs = obs_dev; a.reward = reward_dev; a.terminated = terminated_dev; a.truncated = truncated_dev;
  a.nsub = h->img.hdr()->cfg.nsubsteps; a.mode = 0;
  return lane_step(h, a, st, aux, stream);
}

extern "C" int smplsim_mj_step(SmplsimHandle* h, const SmplsimState* st, const float* ctrl_dev, int nsub, const SmplsimAux* aux, void* stream) {
  if (!h || !state_ok(st) || !ctrl_dev || nsub < 1) return fail(SMPLSIM_EINVAL, "smplsim_mj_step: bad argument");
  DeviceGuard guard(h->device);
  LStepArgs a = lane_args<LStepArgs>(h, st, aux);
  a.action = ctrl_dev; a.nsub = nsub; a.mode = 1;
  return lane_step(h, a, st, aux, stream);
}

extern "C" int smplsim_reset(SmplsimHandle* h, const SmplsimState* st, const uint8_t* mask_dev, int init_mode, const float* qpos0_dev,
                             const float* qvel0_dev, float* obs_dev, const SmplsimAux* aux, void* stream) {
  if (!h || !state_ok(st)) return fail(SMPLSIM_EINVAL, "smplsim_reset: null handle/state");
  if (h->img.hdr()->cfg.control_mode == SMPLSIM_CTRL_SIMPLE_PID && (!st->pid_integral || !st->pid_last_error))
    return fail(SMPLSIM_EINVAL, "smplsim_reset: control_mode simple_pid needs state.pid_integral / pid_last_error (Fall init runs the controller)");
  int mode = init_mode < 0 ? h->img.hdr()->cfg.state_init : init_mode;
  if (mode < 0 || mode > 2) return fail(SMPLSIM_EINVAL, "smplsim_reset: init_mode");
  if (mode == SMPLSIM_INIT_MOCAP && (!qpos0_dev || !qvel0_dev)) return fail(SMPLSIM_EINVAL, "smplsim_reset: MoCap init needs qpos0/qvel0");
  DeviceGuard guard(h->device);
  LResetArgs a = lane_args<LResetArgs>(h, st, aux);
  a.mask = mask_dev; a.qpos0 = qpos0_dev; a.qvel0 = qvel0_dev; a.obs = obs_dev; a.init_mode = mode;
  L_DISPATCH(h, lane_launch<C_>(h, lane_kernels<C_>().reset[h->prm ? 1 : 0], a.n, (cudaStream_t)stream, a));
  if (float* cw = aux_wrench(aux)) {   // the reset runs no constraint solve: zero wrench rows for the envs it resets
    const int row = 6 * h->img.hdr()->nb;
    L_LAUNCH(k_zero_wrench, (int)(((long)a.n * row + 255) / 256), 256, 0, (cudaStream_t)stream, cw, a.mask, a.n, row);
  }
  CUDA_TRY(cudaGetLastError());
  return SMPLSIM_OK;
}

extern "C" int smplsim_kinematics(SmplsimHandle* h, const float* qpos_dev, float* xpos_dev, float* xquat_dev, int n, void* stream) {
  if (!h || !qpos_dev || !xpos_dev || !xquat_dev || n < 0) return fail(SMPLSIM_EINVAL, "smplsim_kinematics: bad argument");
  if (n == 0) return SMPLSIM_OK;
  DeviceGuard guard(h->device);
  if (int rc = env_rows(h, n, "smplsim_kinematics", false)) return rc;
  LKinArgs a; a.qpos = qpos_dev; a.xpos = xpos_dev; a.xquat = xquat_dev; a.n = n; a.map = h->map();
  L_DISPATCH(h, lane_launch<C_>(h, lane_kernels<C_>().kin, n, (cudaStream_t)stream, a));
  CUDA_TRY(cudaGetLastError());
  return SMPLSIM_OK;
}

extern "C" int smplsim_inverse(SmplsimHandle* h, const float* qpos_dev, const float* qvel_dev, const float* qacc_dev, float* qfrc_inverse_dev,
                               float* contact_wrench_dev, int n, void* stream) {
  if (!h || n < 0) return fail(SMPLSIM_EINVAL, "smplsim_inverse: null handle or n < 0");
  if (h->selfcol)
    return fail(SMPLSIM_EUNSUPPORTED, "smplsim_inverse: the inverse does not build geom-geom contacts (handle created with self_collision = 1)");
  if (n == 0) return SMPLSIM_OK;   // nothing is read: empty tensors may come as NULL
  if (!qpos_dev || !qvel_dev || !qacc_dev || !qfrc_inverse_dev) return fail(SMPLSIM_EINVAL, "smplsim_inverse: null argument");
  if (int rc = env_rows(h, n, "smplsim_inverse", true)) return rc;
  DeviceGuard guard(h->device);
  LInvArgs a; std::memset(&a, 0, sizeof a);
  a.qpos = qpos_dev; a.qvel = qvel_dev; a.qacc = qacc_dev; a.qfrc = qfrc_inverse_dev; a.cwrench = contact_wrench_dev; a.gscr = h->gscr; a.n = n;
  a.map = h->map();
  const size_t nv = h->img.hdr()->nv, nb = h->img.hdr()->nb;
  auto advance = [nv, nb](LInvArgs& c, size_t r) {
    c.qpos += r * (nv + 1); c.qvel += r * nv; c.qacc += r * nv; c.qfrc += r * nv;
    if (c.cwrench) c.cwrench += r * nb * 6;
  };
  L_DISPATCH(h, state_rows<C_>(h, lane_kernels<C_>().inverse, a, advance, (cudaStream_t)stream));
  CUDA_TRY(cudaGetLastError());
  return SMPLSIM_OK;
}

extern "C" int smplsim_dynamics(SmplsimHandle* h, const float* qpos_dev, const float* qvel_dev, int n, float* qM_dev, float* qfrc_bias_dev,
                                const int32_t* jac_body, int njac, float* jac_dev, void* stream) {
  if (!h || n < 0 || njac < 0) return fail(SMPLSIM_EINVAL, "smplsim_dynamics: null handle, n < 0 or njac < 0");
  const LHdr& H = *h->img.hdr();
  if (njac > H.nb) return fail(SMPLSIM_EINVAL, "smplsim_dynamics: njac > nbody");
  if (njac > 0 && !jac_body) return fail(SMPLSIM_EINVAL, "smplsim_dynamics: njac > 0 needs jac_body");
  if (!bodies_in_range(jac_body, njac, H.nb)) return fail(SMPLSIM_EINVAL, "smplsim_dynamics: jac_body entry out of range [0, nbody)");
  if (qfrc_bias_dev && !qvel_dev) return fail(SMPLSIM_EINVAL, "smplsim_dynamics: qfrc_bias needs qvel");
  if (n == 0) return SMPLSIM_OK;   // nothing is read: empty tensors may come as NULL
  if (njac > 0 && !jac_dev) return fail(SMPLSIM_EINVAL, "smplsim_dynamics: njac > 0 needs jac_dev");
  if (!qM_dev && !qfrc_bias_dev && !njac) return fail(SMPLSIM_EINVAL, "smplsim_dynamics: no output requested");
  if (!qpos_dev) return fail(SMPLSIM_EINVAL, "smplsim_dynamics: null qpos");
  if (int rc = env_rows(h, n, "smplsim_dynamics", true)) return rc;
  DeviceGuard guard(h->device);
  LDynArgs a; std::memset(&a, 0, sizeof a);
  a.qpos = qpos_dev; a.qvel = qvel_dev; a.qM = qM_dev; a.bias = qfrc_bias_dev; a.jac = njac ? jac_dev : nullptr; a.gscr = h->gscr; a.n = n;
  a.njac = njac;
  for (int j = 0; j < njac; j++) a.jb[j] = (unsigned char)jac_body[j];
  a.map = h->map();
  const size_t nv = H.nv;
  auto advance = [nv](LDynArgs& c, size_t r) {
    c.qpos += r * (nv + 1);
    if (c.qvel) c.qvel += r * nv;
    if (c.qM) c.qM += r * nv * nv;
    if (c.bias) c.bias += r * nv;
    if (c.jac) c.jac += r * c.njac * 6 * nv;
  };
  L_DISPATCH(h, state_rows<C_>(h, lane_kernels<C_>().dyn, a, advance, (cudaStream_t)stream));
  CUDA_TRY(cudaGetLastError());
  return SMPLSIM_OK;
}

extern "C" int smplsim_centroidal(SmplsimHandle* h, const float* qpos_dev, const float* qvel_dev, int n, float* subtree_com_dev,
                                  float* subtree_linvel_dev, float* subtree_angmom_dev, float* cmm_dev, float* cmm_bias_dev, const int32_t* jac_body,
                                  int njac, float* jac_com_dev, void* stream) {
  if (!h || n < 0 || njac < 0) return fail(SMPLSIM_EINVAL, "smplsim_centroidal: null handle, n < 0 or njac < 0");
  const LHdr& H = *h->img.hdr();
  if (njac > H.nb) return fail(SMPLSIM_EINVAL, "smplsim_centroidal: njac > nbody");
  if (njac > 0 && !jac_body) return fail(SMPLSIM_EINVAL, "smplsim_centroidal: njac > 0 needs jac_body");
  if (!bodies_in_range(jac_body, njac, H.nb)) return fail(SMPLSIM_EINVAL, "smplsim_centroidal: jac_body entry out of range [0, nbody)");
  if ((subtree_linvel_dev || subtree_angmom_dev || cmm_bias_dev) && !qvel_dev)
    return fail(SMPLSIM_EINVAL, "smplsim_centroidal: subtree_linvel, subtree_angmom and cmm_bias need qvel");
  if (n == 0) return SMPLSIM_OK;   // nothing is read: empty tensors may come as NULL
  if (njac > 0 && !jac_com_dev) return fail(SMPLSIM_EINVAL, "smplsim_centroidal: njac > 0 needs jac_com_dev");
  if (!subtree_com_dev && !subtree_linvel_dev && !subtree_angmom_dev && !cmm_dev && !cmm_bias_dev && !njac)
    return fail(SMPLSIM_EINVAL, "smplsim_centroidal: no output requested");
  if (!qpos_dev) return fail(SMPLSIM_EINVAL, "smplsim_centroidal: null qpos");
  if (int rc = env_rows(h, n, "smplsim_centroidal", true)) return rc;
  DeviceGuard guard(h->device);
  LCentArgs a; std::memset(&a, 0, sizeof a);
  a.qpos = qpos_dev; a.qvel = qvel_dev; a.com = subtree_com_dev; a.linvel = subtree_linvel_dev; a.angmom = subtree_angmom_dev;
  a.cmm = cmm_dev; a.cbias = cmm_bias_dev; a.jac = njac ? jac_com_dev : nullptr; a.gscr = h->gscr; a.n = n; a.njac = njac;
  for (int j = 0; j < njac; j++) a.jb[j] = (unsigned char)jac_body[j];
  a.map = h->map();
  const size_t nv = H.nv, nb = H.nb;
  auto advance = [nv, nb](LCentArgs& c, size_t r) {
    c.qpos += r * (nv + 1);
    if (c.qvel) c.qvel += r * nv;
    if (c.com) c.com += r * nb * 3;
    if (c.linvel) c.linvel += r * nb * 3;
    if (c.angmom) c.angmom += r * nb * 3;
    if (c.cmm) c.cmm += r * 6 * nv;
    if (c.cbias) c.cbias += r * 6;
    if (c.jac) c.jac += r * c.njac * 3 * nv;
  };
  L_DISPATCH(h, state_rows<C_>(h, lane_kernels<C_>().cent, a, advance, (cudaStream_t)stream));
  CUDA_TRY(cudaGetLastError());
  return SMPLSIM_OK;
}

extern "C" int smplsim_rne_post(SmplsimHandle* h, const float* qpos_dev, const float* qvel_dev, const float* qacc_dev, const float* xfrc_applied_dev,
                                int n, float* body_acc_dev, float* joint_wrench_dev, const int32_t* site_body, const float* site_pos,
                                const float* site_quat, int nsite, float* accelerometer_dev, float* gyro_dev, float* force_dev, float* torque_dev,
                                void* stream) {
  if (!h || n < 0 || nsite < 0) return fail(SMPLSIM_EINVAL, "smplsim_rne_post: null handle, n < 0 or nsite < 0");
  if (h->selfcol)
    return fail(SMPLSIM_EUNSUPPORTED, "smplsim_rne_post: the inverse's pass does not build geom-geom contacts (handle created with self_collision = 1)");
  const LHdr& H = *h->img.hdr();
  if (nsite > LRNEP_MAXS) return fail(SMPLSIM_EINVAL, "smplsim_rne_post: nsite > 64");
  if (nsite > 0 && (!site_body || !site_pos || !site_quat))
    return fail(SMPLSIM_EINVAL, "smplsim_rne_post: nsite > 0 needs site_body, site_pos and site_quat");
  // not bodies_in_range: each site's body is checked with its quaternion, so a call with a bad quaternion before a bad body reports
  // the quaternion
  for (int s = 0; s < nsite; s++) {
    if (site_body[s] < 0 || site_body[s] >= H.nb) return fail(SMPLSIM_EINVAL, "smplsim_rne_post: site_body entry out of range [0, nbody)");
    const float* q = site_quat + 4 * s;
    const double nq = std::sqrt((double)q[0] * q[0] + (double)q[1] * q[1] + (double)q[2] * q[2] + (double)q[3] * q[3]);
    if (!(std::fabs(nq - 1.0) <= 1e-3)) return fail(SMPLSIM_EINVAL, "smplsim_rne_post: site_quat entry is not a unit quaternion (|norm - 1| > 1e-3)");
  }
  if (n == 0) return SMPLSIM_OK;   // nothing is read: empty tensors may come as NULL
  const bool site_out = accelerometer_dev || gyro_dev || force_dev || torque_dev;
  if (nsite > 0 && !site_out) return fail(SMPLSIM_EINVAL, "smplsim_rne_post: nsite > 0 needs a site output");
  if (nsite == 0 && site_out) return fail(SMPLSIM_EINVAL, "smplsim_rne_post: a site output needs nsite > 0");
  if (!body_acc_dev && !joint_wrench_dev && !site_out) return fail(SMPLSIM_EINVAL, "smplsim_rne_post: no output requested");
  if (!qpos_dev || !qvel_dev || !qacc_dev) return fail(SMPLSIM_EINVAL, "smplsim_rne_post: null qpos, qvel or qacc");
  if (int rc = env_rows(h, n, "smplsim_rne_post", true)) return rc;
  DeviceGuard guard(h->device);
  LRnepArgs a; std::memset(&a, 0, sizeof a);
  a.qpos = qpos_dev; a.qvel = qvel_dev; a.qacc = qacc_dev; a.xfrc = xfrc_applied_dev; a.acc = body_acc_dev; a.jw = joint_wrench_dev;
  a.accel = accelerometer_dev; a.gyro = gyro_dev; a.force = force_dev; a.torque = torque_dev;
  a.gscr = h->gscr; a.gf = h->groll; a.map = h->map(); a.n = n; a.nsite = nsite;
  for (int s = 0; s < nsite; s++) {
    a.sb[s] = (unsigned char)site_body[s];
    for (int j = 0; j < 3; j++) a.spos[3 * s + j] = site_pos[3 * s + j];
    for (int j = 0; j < 4; j++) a.squat[4 * s + j] = site_quat[4 * s + j];
  }
  const size_t nv = H.nv, nb = H.nb, ns = nsite;
  auto advance = [nv, nb, ns](LRnepArgs& c, size_t r) {
    c.qpos += r * (nv + 1); c.qvel += r * nv; c.qacc += r * nv;
    if (c.xfrc) c.xfrc += r * nb * 6;
    if (c.acc) c.acc += r * nb * 6;
    if (c.jw) c.jw += r * nb * 6;
    for (float** p : {&c.accel, &c.gyro, &c.force, &c.torque})
      if (*p) *p += r * ns * 3;
  };
  L_DISPATCH(h, state_rows<C_>(h, lane_kernels<C_>().rnep, a, advance, (cudaStream_t)stream));
  CUDA_TRY(cudaGetLastError());
  return SMPLSIM_OK;
}

// forward pass on n caller rows into qacc (and the other outputs each when non-NULL); the caller has checked the arguments
static int forward_rows(SmplsimHandle* h, const float* qpos, const float* qvel, const float* ctrl, const float* qacc_warm, int n, float* qacc,
                        uint64_t* contact_mask, int32_t* solver_iter, uint8_t* status, float* cwrench, cudaStream_t st) {
  LFwdArgs a; std::memset(&a, 0, sizeof a);
  a.qpos = qpos; a.qvel = qvel; a.ctrl = ctrl; a.qacc_warm = qacc_warm; a.qacc = qacc; a.contact_mask = contact_mask; a.solver_iter = solver_iter;
  a.status = status; a.cwrench = cwrench; a.gscr = h->gscr; a.n = n; a.map = h->map();
  const size_t nv = h->img.hdr()->nv, nu = h->img.hdr()->nu, nb = h->img.hdr()->nb;
  auto advance = [nv, nu, nb](LFwdArgs& c, size_t r) {
    c.qpos += r * (nv + 1); c.qvel += r * nv; c.ctrl += r * nu; c.qacc += r * nv;
    if (c.qacc_warm) c.qacc_warm += r * nv;
    if (c.contact_mask) c.contact_mask += r;
    if (c.solver_iter) c.solver_iter += r;
    if (c.status) c.status += r;
    if (c.cwrench) c.cwrench += r * nb * 6;
  };
  L_DISPATCH(h, state_rows<C_>(h, lane_kernels<C_>().fwd, a, advance, st));
  CUDA_TRY(cudaGetLastError());
  return SMPLSIM_OK;
}

extern "C" int smplsim_forward(SmplsimHandle* h, const float* qpos_dev, const float* qvel_dev, const float* ctrl_dev, const float* qacc_warmstart_dev,
                               int n, float* qacc_dev, uint64_t* contact_mask_dev, int32_t* solver_iter_dev, uint8_t* status_dev,
                               float* contact_wrench_dev, void* stream) {
  if (!h || n < 0) return fail(SMPLSIM_EINVAL, "smplsim_forward: null handle or n < 0");
  if (h->selfcol)
    return fail(SMPLSIM_EUNSUPPORTED, "smplsim_forward: the forward pass on caller rows does not build geom-geom contacts (handle created with self_collision = 1)");
  if (n == 0) return SMPLSIM_OK;   // nothing is read: empty tensors may come as NULL
  if (!qpos_dev || !qvel_dev || !ctrl_dev || !qacc_dev) return fail(SMPLSIM_EINVAL, "smplsim_forward: null argument");
  if (int rc = env_rows(h, n, "smplsim_forward", true)) return rc;
  DeviceGuard guard(h->device);
  return forward_rows(h, qpos_dev, qvel_dev, ctrl_dev, qacc_warmstart_dev, n, qacc_dev, contact_mask_dev, solver_iter_dev, status_dev,
                      contact_wrench_dev, (cudaStream_t)stream);
}

// the refusals smplsim_transition_fd and smplsim_inverse_fd share, in order; selfcol: why fn refuses self-collision handles
static int fd_refusals(const SmplsimHandle* h, const std::string& fn, const char* selfcol, const char* eps_names, const float eps[3]) {
  if (h->selfcol) return fail(SMPLSIM_EUNSUPPORTED, fn + ": " + selfcol + " (handle created with self_collision = 1)");
  if (h->nblocks) return fail(SMPLSIM_EUNSUPPORTED, fn + ": not available with per-env body shapes (the column slots of a row span CTAs of any shape)");
  if (h->prm) return fail(SMPLSIM_EUNSUPPORTED, fn + ": not available while the handle has per-env parameter records (smplsim_clear_env_params)");
  for (int k = 0; k < 3; k++)
    if (!(std::isfinite(eps[k]) && eps[k] > 0.f)) return fail(SMPLSIM_EINVAL, fn + ": " + eps_names + " must be finite and > 0");
  return SMPLSIM_OK;
}

// the column launches of smplsim_transition_fd and smplsim_inverse_fd: n rows of a.fd.ncol slots, in launches of at most num_envs
// slots (the handle's per-env scratch rows), in order on st; kern picks the kernel from lane_kernels
template <class A, class K>
static int fd_columns(SmplsimHandle* h, A a, int n, K kern, cudaStream_t st) {
  a.gscr = h->gscr; a.map = h->map(); a.fd.gfd = h->gfd;
  const long long slots = (long long)n * a.fd.ncol;
  for (long long s0 = 0; s0 < slots; s0 += h->num_envs) {
    a.fd.s0 = s0; a.n = (int)std::min<long long>(h->num_envs, slots - s0);
    L_DISPATCH(h, lane_launch<C_>(h, kern(lane_kernels<C_>()), a.n, st, a));
  }
  CUDA_TRY(cudaGetLastError());
  return SMPLSIM_OK;
}

extern "C" int smplsim_transition_fd(SmplsimHandle* h, const SmplsimFdCfg* cfg, const float* qpos_dev, const float* qvel_dev, const float* ctrl_dev,
                                     int n, float* qacc_dev, float* dqacc_dev, float* A_dev, float* B_dev, uint8_t* flags_dev, void* stream) {
  if (!h || !cfg || n < 0) return fail(SMPLSIM_EINVAL, "smplsim_transition_fd: null handle / cfg or n < 0");
  LFwdArgs a; std::memset(&a, 0, sizeof a);
  a.fd.eps[0] = cfg->eps_qpos; a.fd.eps[1] = cfg->eps_qvel; a.fd.eps[2] = cfg->eps_ctrl;
  if (int rc = fd_refusals(h, "smplsim_transition_fd", "the forward pass on caller rows does not build geom-geom contacts",
                           "eps_qpos, eps_qvel and eps_ctrl", a.fd.eps)) return rc;
  if (n == 0) return SMPLSIM_OK;   // nothing is read: empty tensors may come as NULL
  if (!qpos_dev || !qvel_dev || !ctrl_dev || !qacc_dev) return fail(SMPLSIM_EINVAL, "smplsim_transition_fd: null argument (qpos, qvel, ctrl and qacc are required)");
  if (!dqacc_dev && !A_dev && !B_dev && !flags_dev) return fail(SMPLSIM_EINVAL, "smplsim_transition_fd: no derivative output requested (dqacc, A, B and flags all NULL)");
  DeviceGuard guard(h->device);
  const cudaStream_t st = (cudaStream_t)stream;
  if (int rc = forward_rows(h, qpos_dev, qvel_dev, ctrl_dev, nullptr, n, qacc_dev, nullptr, nullptr, nullptr, nullptr, st)) return rc;
  const LHdr& H = *h->img.hdr();
  a.qpos = qpos_dev; a.qvel = qvel_dev; a.ctrl = ctrl_dev; a.qacc_warm = qacc_dev; a.dqacc = dqacc_dev; a.A = A_dev; a.B = B_dev;
  a.fd.flags = flags_dev; a.fd.ncol = 2 * H.nv + H.nu; a.fd.centered = cfg->centered ? 1 : 0;
  return fd_columns(h, a, n, [](const LaneKernels& k) { return k.fwd[0]; }, st);
}

extern "C" int smplsim_inverse_fd(SmplsimHandle* h, const SmplsimInverseFdCfg* cfg, const float* qpos_dev, const float* qvel_dev,
                                  const float* qacc_dev, int n, float* qfrc_inverse_dev, float* dfrc_dev, uint8_t* flags_dev, void* stream) {
  if (!h || !cfg || n < 0) return fail(SMPLSIM_EINVAL, "smplsim_inverse_fd: null handle / cfg or n < 0");
  LInvFdArgs a; std::memset(&a, 0, sizeof a);
  a.fd.eps[0] = cfg->eps_qpos; a.fd.eps[1] = cfg->eps_qvel; a.fd.eps[2] = cfg->eps_qacc;
  if (int rc = fd_refusals(h, "smplsim_inverse_fd", "the inverse does not build geom-geom contacts", "eps_qpos, eps_qvel and eps_qacc", a.fd.eps)) return rc;
  if (n == 0) return SMPLSIM_OK;   // nothing is read: empty tensors may come as NULL
  if (!qpos_dev || !qvel_dev || !qacc_dev || !qfrc_inverse_dev)
    return fail(SMPLSIM_EINVAL, "smplsim_inverse_fd: null argument (qpos, qvel, qacc and qfrc_inverse are required)");
  if (!dfrc_dev && !flags_dev) return fail(SMPLSIM_EINVAL, "smplsim_inverse_fd: no derivative output requested (dfrc and flags both NULL)");
  // the nominal pass is smplsim_inverse's row path, so qfrc_inverse is bit for bit what smplsim_inverse gives
  if (int rc = smplsim_inverse(h, qpos_dev, qvel_dev, qacc_dev, qfrc_inverse_dev, nullptr, n, stream)) return rc;
  DeviceGuard guard(h->device);
  a.qpos = qpos_dev; a.qvel = qvel_dev; a.qacc = qacc_dev; a.qfrc = qfrc_inverse_dev; a.dfrc = dfrc_dev;
  a.fd.flags = flags_dev; a.fd.ncol = 3 * h->img.hdr()->nv; a.fd.centered = cfg->centered ? 1 : 0;
  return fd_columns(h, a, n, [](const LaneKernels& k) { return k.invfd; }, (cudaStream_t)stream);
}

// the argument checks and row arguments of smplsim_rollout and smplsim_rollout_feedback (fn: the caller, for the error texts).
// *empty: n == 0, nothing to launch.
static int roll_args(SmplsimHandle* h, const char* fn, int mode, int nsub, const float* qpos0_dev, const float* qvel0_dev,
                     const float* qacc_warmstart_dev, const float* qpos_fwd0_dev, const float* qvel_fwd0_dev, const float* control_dev, int n,
                     int nstep, float* qpos_dev, float* qvel_dev, uint8_t* status_dev, float* xpos_dev, float* xquat_dev, LRollArgs& a, bool* empty) {
  const std::string f(fn);
  *empty = false;
  if (!h || n < 0 || nstep < 1) return fail(SMPLSIM_EINVAL, f + ": null handle, n < 0 or nstep < 1");
  if (mode != SMPLSIM_ROLLOUT_ACTION && mode != SMPLSIM_ROLLOUT_CTRL) return fail(SMPLSIM_EINVAL, f + ": unknown mode");
  if (mode == SMPLSIM_ROLLOUT_CTRL && nsub < 1) return fail(SMPLSIM_EINVAL, f + ": SMPLSIM_ROLLOUT_CTRL needs nsub >= 1");
  if (mode == SMPLSIM_ROLLOUT_ACTION && nsub != 0)
    return fail(SMPLSIM_EINVAL, f + ": SMPLSIM_ROLLOUT_ACTION takes nsub = 0 (an action step runs cfg.env.nsubsteps substeps)");
  if (!xpos_dev != !xquat_dev) return fail(SMPLSIM_EINVAL, f + ": give both xpos and xquat, or neither");
  if (h->selfcol)
    return fail(SMPLSIM_EUNSUPPORTED, f + ": the rollout on caller rows does not build geom-geom contacts (handle created with self_collision = 1)");
  const LHdr& H = *h->img.hdr();
  if (mode == SMPLSIM_ROLLOUT_ACTION && H.cfg.control_mode == SMPLSIM_CTRL_SIMPLE_PID)
    return fail(SMPLSIM_EUNSUPPORTED, f + ": control_mode simple_pid keeps its integral / last error in env state, which rollout rows do not have");
  if (n == 0) { *empty = true; return SMPLSIM_OK; }   // nothing is read: empty tensors may come as NULL
  if (!qpos0_dev || !qvel0_dev || !control_dev || !qpos_dev || !qvel_dev)
    return fail(SMPLSIM_EINVAL, f + ": null argument (qpos0, qvel0, control, qpos and qvel are required)");
  if (int rc = env_rows(h, n, fn, true)) return rc;
  const size_t nq = H.nv + 1, nv = H.nv, N = (size_t)h->num_envs;
  std::memset(&a, 0, sizeof a);
  a.qpos0 = qpos0_dev; a.qvel0 = qvel0_dev; a.qacc_warm0 = qacc_warmstart_dev; a.control = control_dev;
  a.qpos_fwd0 = qpos_fwd0_dev ? qpos_fwd0_dev : qpos0_dev; a.qvel_fwd0 = qvel_fwd0_dev ? qvel_fwd0_dev : qvel0_dev;   // as set_state marks
  a.qpos = qpos_dev; a.qvel = qvel_dev; a.status = status_dev; a.xpos = xpos_dev; a.xquat = xquat_dev;
  a.scr.qpos = h->groll; a.scr.qvel = a.scr.qpos + N * nq; a.scr.qpos_fwd = a.scr.qvel + N * nv; a.scr.qvel_fwd = a.scr.qpos_fwd + N * nq;
  a.gscr = h->gscr; a.map = h->map(); a.n = n; a.nstep = nstep; a.mode = mode;
  a.nsub = mode == SMPLSIM_ROLLOUT_ACTION ? H.cfg.nsubsteps : nsub;
  return SMPLSIM_OK;
}
// moves every row pointer of a rollout launch to row r
static void roll_advance(const LHdr& H, LRollArgs& c, size_t r) {
  const size_t nq = H.nv + 1, nv = H.nv, nu = H.nu, nb = H.nb, T = (size_t)c.nstep;
  c.qpos0 += r * nq; c.qvel0 += r * nv; c.qpos_fwd0 += r * nq; c.qvel_fwd0 += r * nv; c.control += r * T * nu;
  if (c.qacc_warm0) c.qacc_warm0 += r * nv;
  c.qpos += r * T * nq; c.qvel += r * T * nv;
  if (c.status) c.status += r * T;
  if (c.xpos) { c.xpos += r * T * nb * 3; c.xquat += r * T * nb * 4; }
}

extern "C" int smplsim_rollout(SmplsimHandle* h, int mode, int nsub, const float* qpos0_dev, const float* qvel0_dev, const float* qacc_warmstart_dev,
                               const float* qpos_fwd0_dev, const float* qvel_fwd0_dev, const float* control_dev, int n, int nstep,
                               float* qpos_dev, float* qvel_dev, uint8_t* status_dev, float* xpos_dev, float* xquat_dev, void* stream) {
  LRollArgs a; bool empty;
  if (int rc = roll_args(h, "smplsim_rollout", mode, nsub, qpos0_dev, qvel0_dev, qacc_warmstart_dev, qpos_fwd0_dev, qvel_fwd0_dev, control_dev,
                         n, nstep, qpos_dev, qvel_dev, status_dev, xpos_dev, xquat_dev, a, &empty)) return rc;
  if (empty) return SMPLSIM_OK;
  DeviceGuard guard(h->device);
  const LHdr& H = *h->img.hdr();
  auto advance = [&H](LRollArgs& c, size_t r) { roll_advance(H, c, r); };
  L_DISPATCH(h, state_rows<C_>(h, lane_kernels<C_>().roll, a, advance, (cudaStream_t)stream));
  CUDA_TRY(cudaGetLastError());
  return SMPLSIM_OK;
}

extern "C" int smplsim_rollout_feedback(SmplsimHandle* h, int mode, int nsub, const float* qpos0_dev, const float* qvel0_dev,
                                        const float* qacc_warmstart_dev, const float* qpos_fwd0_dev, const float* qvel_fwd0_dev,
                                        const float* control_dev, int n, int nstep, float* qpos_dev, float* qvel_dev, uint8_t* status_dev,
                                        float* xpos_dev, float* xquat_dev, const float* gain_dev, const float* qpos_ref_dev,
                                        const float* qvel_ref_dev, int ref_rows, int clip_actions, float* control_applied_dev, void* stream) {
  LRollFbArgs a; bool empty;
  std::memset(&a, 0, sizeof a);
  if (int rc = roll_args(h, "smplsim_rollout_feedback", mode, nsub, qpos0_dev, qvel0_dev, qacc_warmstart_dev, qpos_fwd0_dev, qvel_fwd0_dev,
                         control_dev, n, nstep, qpos_dev, qvel_dev, status_dev, xpos_dev, xquat_dev, a.r, &empty)) return rc;
  if (ref_rows != 1 && ref_rows != n)
    return fail(SMPLSIM_EINVAL, "smplsim_rollout_feedback: ref_rows must be 1 (one schedule for every row) or n (one per row)");
  if (empty) return SMPLSIM_OK;
  if (!gain_dev || !qpos_ref_dev || !qvel_ref_dev)
    return fail(SMPLSIM_EINVAL, "smplsim_rollout_feedback: null argument (gain, qpos_ref and qvel_ref are required)");
  DeviceGuard guard(h->device);
  const LHdr& H = *h->img.hdr();
  const size_t nq = H.nv + 1, nv = H.nv, nu = H.nu, T = (size_t)nstep;
  a.gain = gain_dev; a.qpos_ref = qpos_ref_dev; a.qvel_ref = qvel_ref_dev; a.control_applied = control_applied_dev;
  a.dx = h->gfb; a.uscr = h->gfb + (size_t)2 * nv * h->num_envs;
  a.shared_ref = ref_rows == 1; a.clip = clip_actions != 0;
  auto advance = [&H, nq, nv, nu, T](LRollFbArgs& c, size_t r) {
    roll_advance(H, c.r, r);
    if (c.control_applied) c.control_applied += r * T * nu;
    if (!c.shared_ref) { c.gain += r * T * nu * 2 * nv; c.qpos_ref += r * T * nq; c.qvel_ref += r * T * nv; }
  };
  L_DISPATCH(h, state_rows<C_>(h, lane_kernels<C_>().rollfb, a, advance, (cudaStream_t)stream));
  CUDA_TRY(cudaGetLastError());
  return SMPLSIM_OK;
}

// ray casting / rendering: the scene of n rows of body poses (render_kernels.cuh)
static RScene render_scene(const SmplsimHandle* h, const float* xpos, const float* xquat) {
  const LHdr& H = *h->img.hdr();
  RScene s; std::memset(&s, 0, sizeof s);
  s.gimg = h->dimg; s.env_img = h->denv_model; s.xpos = xpos; s.xquat = xquat;
  s.img_words = H.bytes / 4; s.geom_off = H.geom_off; s.nb = H.nb; s.ng = H.ng;
  // the plane's frame: x = world x projected on the plane (world y if the normal is along x), y = normal x x
  double n[3] = {H.plane_n[0], H.plane_n[1], H.plane_n[2]}, u[3] = {1, 0, 0};
  if (std::fabs(n[0]) > 0.9) { u[0] = 0; u[1] = 1; }
  double d = u[0] * n[0] + u[1] * n[1] + u[2] * n[2];
  for (int k = 0; k < 3; k++) u[k] -= d * n[k];
  double un = std::sqrt(u[0] * u[0] + u[1] * u[1] + u[2] * u[2]);
  for (int k = 0; k < 3; k++) u[k] /= un;
  double v[3] = {n[1] * u[2] - n[2] * u[1], n[2] * u[0] - n[0] * u[2], n[0] * u[1] - n[1] * u[0]};
  for (int k = 0; k < 3; k++) { s.p0[k] = H.plane_pos[k]; s.pn[k] = H.plane_n[k]; s.pu[k] = (float)u[k]; s.pv[k] = (float)v[k]; }
  return s;
}

extern "C" int smplsim_ray(SmplsimHandle* h, const float* xpos_dev, const float* xquat_dev, int n, int nray, const float* pnt_dev,
                           const float* vec_dev, int flg_static, int bodyexclude, float* dist_dev, int32_t* geomid_dev, void* stream) {
  if (!h || n < 0) return fail(SMPLSIM_EINVAL, "smplsim_ray: null handle or n < 0");
  const LHdr& H = *h->img.hdr();
  if (bodyexclude < -1 || bodyexclude >= H.nb) return fail(SMPLSIM_EINVAL, "smplsim_ray: bodyexclude out of range [-1, nbody)");
  if (n == 0) return SMPLSIM_OK;   // nothing is read: empty tensors may come as NULL
  if (nray <= 0) return fail(SMPLSIM_EINVAL, "smplsim_ray: nray <= 0");
  if (!dist_dev && !geomid_dev) return fail(SMPLSIM_EINVAL, "smplsim_ray: no output requested");
  if (!xpos_dev || !xquat_dev || !pnt_dev || !vec_dev) return fail(SMPLSIM_EINVAL, "smplsim_ray: null argument");
  if (int rc = env_rows(h, n, "smplsim_ray", false)) return rc;
  const long grid = (long)n * ((nray + R_THREADS - 1) / R_THREADS);
  if (grid > 0x7fffffffL) return fail(SMPLSIM_EINVAL, "smplsim_ray: n x nray too large for one launch");
  DeviceGuard guard(h->device);
  RRayArgs a; std::memset(&a, 0, sizeof a);
  a.s = render_scene(h, xpos_dev, xquat_dev);
  a.pnt = pnt_dev; a.vec = vec_dev; a.dist = dist_dev; a.geomid = geomid_dev; a.nray = nray; a.flg_static = flg_static ? 1 : 0;
  a.bodyexclude = bodyexclude;
  L_LAUNCH(k_ray, (int)grid, R_THREADS, 0, (cudaStream_t)stream, a);
  CUDA_TRY(cudaGetLastError());
  return SMPLSIM_OK;
}

extern "C" int smplsim_render(SmplsimHandle* h, const float* xpos_dev, const float* xquat_dev, int n, const SmplsimCamera* cam, int width,
                              int height, const float* geom_rgb, float* depth_dev, int32_t* seg_dev, uint8_t* rgb_dev, void* stream) {
  if (!h || !cam || n < 0) return fail(SMPLSIM_EINVAL, "smplsim_render: null handle / camera or n < 0");
  const LHdr& H = *h->img.hdr();
  if (cam->mode < SMPLSIM_CAM_FIXED || cam->mode > SMPLSIM_CAM_BODY) return fail(SMPLSIM_EINVAL, "smplsim_render: unknown camera mode");
  if (cam->mode == SMPLSIM_CAM_BODY && (cam->body < 0 || cam->body >= H.nb)) return fail(SMPLSIM_EINVAL, "smplsim_render: camera body out of range [0, nbody)");
  if (cam->exclude_body < -1 || cam->exclude_body >= H.nb) return fail(SMPLSIM_EINVAL, "smplsim_render: exclude_body out of range [-1, nbody)");
  if (!(cam->fovy > 0.f && cam->fovy < 180.f)) return fail(SMPLSIM_EINVAL, "smplsim_render: fovy outside (0, 180) degrees");
  if (n == 0) return SMPLSIM_OK;
  if (width <= 0 || height <= 0) return fail(SMPLSIM_EINVAL, "smplsim_render: width / height <= 0");
  if (!depth_dev && !seg_dev && !rgb_dev) return fail(SMPLSIM_EINVAL, "smplsim_render: no output requested");
  if (!xpos_dev || !xquat_dev) return fail(SMPLSIM_EINVAL, "smplsim_render: null xpos / xquat");
  if (int rc = env_rows(h, n, "smplsim_render", false)) return rc;
  const bool prm = h->prm && cam->mode == SMPLSIM_CAM_TRACKCOM;   // the robot COM with the env's mass scales
  if (prm && n != h->num_envs) return fail(SMPLSIM_EINVAL, "smplsim_render: a TRACKCOM camera with per-env parameters needs n == num_envs (row i uses env i's masses)");
  const int tiles_x = (width + R_CTA_W - 1) / R_CTA_W, tiles = tiles_x * ((height + R_CTA_H - 1) / R_CTA_H);
  if ((long)n * tiles > 0x7fffffffL) return fail(SMPLSIM_EINVAL, "smplsim_render: n x image too large for one launch");
  DeviceGuard guard(h->device);
  RRenderArgs a; std::memset(&a, 0, sizeof a);
  a.s = render_scene(h, xpos_dev, xquat_dev);
  a.cam = *cam;
  a.depth = depth_dev; a.seg = seg_dev; a.rgb = rgb_dev; a.W = width; a.H = height; a.tiles_x = tiles_x; a.tiles = tiles;
  for (int g = 0; g < H.ng; g++)
    for (int k = 0; k < 3; k++) a.rgb_tab[3 * g + k] = geom_rgb ? geom_rgb[3 * g + k] : (k == 0 ? 0.8f : k == 1 ? 0.6f : 0.4f);   // <default> rgba of the MJCFs
  if (prm) L_LAUNCH(k_render<1>, n * tiles, R_THREADS, 0, (cudaStream_t)stream, a);
  else L_LAUNCH(k_render<0>, n * tiles, R_THREADS, 0, (cudaStream_t)stream, a);
  CUDA_TRY(cudaGetLastError());
  return SMPLSIM_OK;
}

// ------------------------------------------------------------------ per-env physics parameters
// The records' base address goes into the header of every device table (LHdr::prm), where the PRM kernel instances read it from the
// staged copy; the other instances never read that word.  So the kernels keep their argument lists, and without records the launches
// are exactly the ones before records existed.
// Written in stream order on the caller's stream (set: before the records' fill and every later launch there); clear writes NULL
// after a device synchronization, when no launch is left that could read it.
static cudaError_t put_prm_ptr(SmplsimHandle* h, float* const* src, cudaStream_t st) {   // (the host emulator copies at once)
  const LHdr& H = *h->img.hdr();
  cudaError_t e = cudaSuccess;
  for (int k = 0; k < h->nmodels && e == cudaSuccess; k++)
#ifdef SMPLSIM_EMU
    e = cudaMemcpy((char*)h->dimg + (size_t)H.bytes * k + offsetof(LHdr, prm), src, sizeof(float*), cudaMemcpyHostToDevice);
#else
    e = cudaMemcpyAsync((char*)h->dimg + (size_t)H.bytes * k + offsetof(LHdr, prm), src, sizeof(float*), cudaMemcpyHostToDevice, st);
#endif
  return e;
}
static PrmArgs prm_args(const SmplsimHandle* h) {
  const LHdr& H = *h->img.hdr();
  PrmArgs a; std::memset(&a, 0, sizeof a);
  a.rec = h->prm; a.gimg = h->dimg; a.env_img = h->denv_model; a.img_words = H.bytes / 4; a.n = h->num_envs; a.nu = H.nu; a.nb = H.nb;
  a.w = (4 + 3 * H.nu + H.nb + 3) & ~3;
  return a;
}

extern "C" int smplsim_set_env_params(SmplsimHandle* h, const SmplsimEnvParams* p, const uint8_t* mask_dev, void* stream) {
  if (!h || !p) return fail(SMPLSIM_EINVAL, "smplsim_set_env_params: null handle or params");
  DeviceGuard guard(h->device);
  int init = 0;
  if (!h->prm) {
    int w = 0;
    L_DISPATCH(h, w = C_::PRMW);
    float* rec = nullptr;
    CUDA_TRY(cudaMalloc(&rec, (size_t)w * h->num_envs * 4));
    h->prm = rec; h->prmw = w; init = 1;
    const cudaError_t e = put_prm_ptr(h, &h->prm, (cudaStream_t)stream);   // the source is the handle's own field
    if (e != cudaSuccess) {
      cudaDeviceSynchronize(); cudaFree(rec); h->prm = nullptr; h->prmw = 0;
      return fail(SMPLSIM_ECUDA, std::string("smplsim_set_env_params: ") + cudaGetErrorString(e));
    }
  }
  PrmArgs a = prm_args(h);
  if (a.w != h->prmw) return fail(SMPLSIM_EINVAL, "smplsim_set_env_params: record layout mismatch");
  a.mask = mask_dev; a.init = init;
  a.f[0] = p->friction; a.f[1] = p->gravity; a.f[2] = p->kp; a.f[3] = p->kd; a.f[4] = p->torque_limit; a.f[5] = p->body_mass_scale;
  const long tot = (long)a.n * a.w;
  L_LAUNCH(k_prm_set, (int)((tot + 255) / 256), 256, 0, (cudaStream_t)stream, a);
  CUDA_TRY(cudaGetLastError());
  return SMPLSIM_OK;
}

extern "C" int smplsim_get_env_params(SmplsimHandle* h, float* friction_dev, float* gravity_dev, float* kp_dev, float* kd_dev,
                                      float* torque_limit_dev, float* body_mass_scale_dev, void* stream) {
  if (!h) return fail(SMPLSIM_EINVAL, "smplsim_get_env_params: null handle");
  DeviceGuard guard(h->device);
  PrmArgs a = prm_args(h);
  a.o[0] = friction_dev; a.o[1] = gravity_dev; a.o[2] = kp_dev; a.o[3] = kd_dev; a.o[4] = torque_limit_dev; a.o[5] = body_mass_scale_dev;
  const long tot = (long)a.n * a.w;
  L_LAUNCH(k_prm_get, (int)((tot + 255) / 256), 256, 0, (cudaStream_t)stream, a);
  CUDA_TRY(cudaGetLastError());
  return SMPLSIM_OK;
}

extern "C" int smplsim_clear_env_params(SmplsimHandle* h) {
  if (!h) return fail(SMPLSIM_EINVAL, "smplsim_clear_env_params: null handle");
  if (!h->prm) return SMPLSIM_OK;
  DeviceGuard guard(h->device);
  CUDA_TRY(cudaDeviceSynchronize());   // no launch that reads the records is still queued
  static float* const none = nullptr;
  CUDA_TRY(put_prm_ptr(h, &none, 0));
  CUDA_TRY(cudaDeviceSynchronize());
  CUDA_TRY(cudaFree(h->prm));
  h->prm = nullptr; h->prmw = 0;
  return SMPLSIM_OK;
}

extern "C" int smplsim_self_obs(SmplsimHandle* h, int version, const float* qvel_dev, const float* xpos_dev, const float* xquat_dev,
                                const float* linvel_dev, const float* angvel_dev, float* obs_dev, int n, void* stream) {
  if (!h || !xpos_dev || !xquat_dev || !obs_dev || n < 0) return fail(SMPLSIM_EINVAL, "smplsim_self_obs: bad argument");
  if (version == 1 && !qvel_dev) return fail(SMPLSIM_EINVAL, "smplsim_self_obs: v1 needs qvel");
  if (version == 2 && (!linvel_dev || !angvel_dev)) return fail(SMPLSIM_EINVAL, "smplsim_self_obs: v2 needs body velocities");
  if (version != 1 && version != 2) return fail(SMPLSIM_EINVAL, "smplsim_self_obs: version");
  if (n == 0) return SMPLSIM_OK;
  DeviceGuard guard(h->device);
  const LHdr& H = *h->img.hdr();
  int nb = H.nb;
  int self_dim = (H.cfg.root_height_obs ? 1 : 0) + 3 * (nb - 1) + 6 * nb + (version == 1 ? 6 + H.nu : 6 * nb);
  int wpb = 4;
  L_LAUNCH(k_self_obs, (n + wpb - 1) / wpb, 32 * wpb, wpb * 16 * LM_MAXB * 4, (cudaStream_t)stream, h->dimg, version, qvel_dev, xpos_dev, xquat_dev,
           linvel_dev, angvel_dev, obs_dev, n, self_dim);
  CUDA_TRY(cudaGetLastError());
  return SMPLSIM_OK;
}

extern "C" int smplsim_motion_gather(SmplsimHandle* h, const int32_t* motion_ids_dev, const float* motion_times_dev, int n,
                                     const float* motion_len_dev, const int32_t* num_frames_dev, const float* motion_dt_dev,
                                     const int32_t* length_starts_dev, int num_tables, const float* const* tables_dev,
                                     const int32_t* widths, float* const* outs_dev, int32_t* frame_idx_dev, void* stream) {
  if (!motion_ids_dev || !motion_times_dev || !motion_len_dev || !num_frames_dev || !motion_dt_dev || !length_starts_dev || n < 0)
    return fail(SMPLSIM_EINVAL, "smplsim_motion_gather: null argument");
  if (num_tables < 0 || num_tables > SM_MAXTABLES) return fail(SMPLSIM_EINVAL, "smplsim_motion_gather: at most 16 tables");
  if (n == 0) return SMPLSIM_OK;
  DeviceGuard guard(h ? h->device : 0);
  GatherArgs a; std::memset(&a, 0, sizeof a);
  a.ids = motion_ids_dev; a.times = motion_times_dev; a.mlen = motion_len_dev; a.nframes = num_frames_dev; a.mdt = motion_dt_dev;
  a.starts = length_starts_dev; a.frame_idx = frame_idx_dev; a.n = n; a.ntab = num_tables;
  for (int k = 0; k < num_tables; k++) { a.tables[k] = tables_dev[k]; a.outs[k] = outs_dev[k]; a.widths[k] = widths[k]; }
  int wpb = 8;
  L_LAUNCH(k_motion_gather, (n + wpb - 1) / wpb, 32 * wpb, 0, (cudaStream_t)stream, a);
  CUDA_TRY(cudaGetLastError());
  return SMPLSIM_OK;
}

extern "C" int smplsim_motion_blend(SmplsimHandle* h, const int32_t* motion_ids_dev, const float* motion_times_dev, int n,
                                    const float* motion_len_dev, const int32_t* num_frames_dev, const float* motion_dt_dev,
                                    const int32_t* length_starts_dev, int num_tables, const float* const* tables_dev,
                                    const int32_t* widths, const int32_t* kinds, const float* offset_dev, float* const* outs_dev,
                                    int32_t* frame0_dev, int32_t* frame1_dev, float* blend_dev, void* stream) {
  if (!motion_ids_dev || !motion_times_dev || !motion_len_dev || !num_frames_dev || !motion_dt_dev || !length_starts_dev || n < 0)
    return fail(SMPLSIM_EINVAL, "smplsim_motion_blend: null argument");
  if (num_tables < 0 || num_tables > SM_MAXTABLES) return fail(SMPLSIM_EINVAL, "smplsim_motion_blend: at most 16 tables");
  if (num_tables > 0 && (!tables_dev || !widths || !kinds || !outs_dev)) return fail(SMPLSIM_EINVAL, "smplsim_motion_blend: null table list");
  for (int k = 0; k < num_tables; k++) {
    const int w = widths[k], kd = kinds[k];
    if (w < 0) return fail(SMPLSIM_EINVAL, "smplsim_motion_blend: negative width");
    if (kd < SMPLSIM_BLEND_LERP || kd > SMPLSIM_BLEND_ROW0) return fail(SMPLSIM_EINVAL, "smplsim_motion_blend: unknown kind");
    if (kd == SMPLSIM_BLEND_SLERP && w % 4) return fail(SMPLSIM_EINVAL, "smplsim_motion_blend: SLERP needs a width that is a multiple of 4");
    if (kd == SMPLSIM_BLEND_POS && w % 3) return fail(SMPLSIM_EINVAL, "smplsim_motion_blend: POS needs a width that is a multiple of 3");
    if (kd == SMPLSIM_BLEND_QPOS && w < 7) return fail(SMPLSIM_EINVAL, "smplsim_motion_blend: QPOS needs a width of at least 7");
  }
  if (n == 0) return SMPLSIM_OK;
  DeviceGuard guard(h ? h->device : 0);
  BlendArgs a; std::memset(&a, 0, sizeof a);
  a.g.ids = motion_ids_dev; a.g.times = motion_times_dev; a.g.mlen = motion_len_dev; a.g.nframes = num_frames_dev; a.g.mdt = motion_dt_dev;
  a.g.starts = length_starts_dev; a.g.n = n; a.g.ntab = num_tables;
  for (int k = 0; k < num_tables; k++) { a.g.tables[k] = tables_dev[k]; a.g.outs[k] = outs_dev[k]; a.g.widths[k] = widths[k]; a.kinds[k] = kinds[k]; }
  a.offset = offset_dev; a.frame0 = frame0_dev; a.frame1 = frame1_dev; a.blend = blend_dev;
  const int wpb = 8;
  L_LAUNCH(k_motion_blend, (n + wpb - 1) / wpb, 32 * wpb, 0, (cudaStream_t)stream, a);
  CUDA_TRY(cudaGetLastError());
  return SMPLSIM_OK;
}

extern "C" int smplsim_imitation_obs_dim(const SmplsimHandle* h, int num_tracked) {
  return h && num_tracked >= 0 ? h->img.hdr()->self_obs_dim + 24 * num_tracked : SMPLSIM_EINVAL;
}

// a motion library's tables against the handle, into the kernel arguments a (ImArgs, AmpArgs); "" when they are good, else the reason
// (SMPLSIM_EINVAL)
template <class A>
static std::string motion_tables(const LHdr& H, const SmplsimMotionTables* tab, A& a) {
  if (tab->nbody != H.nb) return "the tables' nbody is not the handle's";
  if (tab->num_motions < 1) return "num_motions < 1";
  if (!tab->xpos || !tab->xquat || !tab->body_vel || !tab->body_ang_vel || !tab->motion_len || !tab->num_frames || !tab->motion_dt || !tab->length_starts)
    return "null motion table";
  a.txpos = tab->xpos; a.txquat = tab->xquat; a.tvel = tab->body_vel; a.tangvel = tab->body_ang_vel;
  a.mlen = tab->motion_len; a.nframes = tab->num_frames; a.mdt = tab->motion_dt; a.starts = tab->length_starts; a.nmotion = tab->num_motions;
  return "";
}

// smplsim_imitation (rec NULL) and smplsim_imitation_recovery
static int imitation(SmplsimHandle* h, const SmplsimImitationCfg* cfg, const SmplsimImitationRecovery* rc, const SmplsimMotionTables* tab,
                     const int32_t* motion_ids_dev, const float* motion_t0_dev, const int32_t* progress_dev, const SmplsimAux* aux,
                     const float* self_obs_dev, const uint8_t* mask_dev, int obs_only, float* obs_dev, float* reward_dev,
                     uint8_t* terminated_dev, uint8_t* truncated_dev, float* mpjpe_dev, int32_t* frames_dev, void* stream) {
  if (!h || !cfg || !tab || !aux) return fail(SMPLSIM_EINVAL, "smplsim_imitation: null handle / cfg / tables / aux");
  const LHdr& H = *h->img.hdr();
  if (cfg->num_tracked < 1 || cfg->num_tracked > H.nb) return fail(SMPLSIM_EINVAL, "smplsim_imitation: num_tracked outside [1, nbody]");
  if (!cfg->tracked_bodies && cfg->num_tracked != H.nb) return fail(SMPLSIM_EINVAL, "smplsim_imitation: tracked_bodies NULL needs num_tracked == nbody");
  if (cfg->tracked_bodies && !bodies_in_range(cfg->tracked_bodies, cfg->num_tracked, H.nb))
    return fail(SMPLSIM_EINVAL, "smplsim_imitation: tracked body out of range [0, nbody)");
  // every table check, NULL tables included, precedes the self_obs_dim check: a call with both wrong reports the tables
  ImArgs a; std::memset(&a, 0, sizeof a);
  const std::string why = motion_tables(H, tab, a);
  if (!why.empty()) return fail(SMPLSIM_EINVAL, "smplsim_imitation: " + why);
  if (cfg->self_obs_dim != H.self_obs_dim) return fail(SMPLSIM_EINVAL, "smplsim_imitation: self_obs_dim is not the handle's self-observation width");
  if (!aux->xpos || !aux->xquat || !aux->body_linvel || !aux->body_angvel) return fail(SMPLSIM_EINVAL, "smplsim_imitation: aux needs xpos, xquat, body_linvel, body_angvel");
  if (!motion_ids_dev || !motion_t0_dev || !progress_dev || !self_obs_dev || !obs_dev) return fail(SMPLSIM_EINVAL, "smplsim_imitation: null argument");
  if (!obs_only && (!reward_dev || !terminated_dev || !truncated_dev || !mpjpe_dev)) return fail(SMPLSIM_EINVAL, "smplsim_imitation: null reward / flag / mpjpe output");
  if (cfg->interpolate != 0 && cfg->interpolate != 1) return fail(SMPLSIM_EINVAL, "smplsim_imitation: interpolate must be 0 or 1");
  if (cfg->num_future < 0) return fail(SMPLSIM_EINVAL, "smplsim_imitation: num_future < 0");
  if (!(cfg->future_dt >= 0.f)) return fail(SMPLSIM_EINVAL, "smplsim_imitation: future_dt < 0 or NaN");
  SmplsimImitationRecovery r; std::memset(&r, 0, sizeof r);
  if (rc) r = *rc;
  if (r.zero_out_far != 0 && r.zero_out_far != 1) return fail(SMPLSIM_EINVAL, "smplsim_imitation: zero_out_far must be 0 or 1");
  if (r.zero_out_far && !(r.far_distance > 0.f)) return fail(SMPLSIM_EINVAL, "smplsim_imitation: far_distance <= 0 or NaN with zero_out_far");
  if (r.zero_out_far && !r.goal_dist) return fail(SMPLSIM_EINVAL, "smplsim_imitation: zero_out_far needs goal_dist");
  if (!(r.power_coefficient >= 0.f)) return fail(SMPLSIM_EINVAL, "smplsim_imitation: power_coefficient < 0 or NaN");
  const bool power = r.power_coefficient > 0.f || r.power;
  if (power && (!r.qvel || !aux->ctrl)) return fail(SMPLSIM_EINVAL, "smplsim_imitation: the power needs qvel and aux.ctrl");
  DeviceGuard guard(h->device);
  a.ids = motion_ids_dev; a.t0 = motion_t0_dev; a.progress = progress_dev; a.mask = mask_dev;
  a.xpos = aux->xpos; a.xquat = aux->xquat; a.linvel = aux->body_linvel; a.angvel = aux->body_angvel; a.status = aux->status;
  a.self_obs = self_obs_dev; a.obs = obs_dev; a.reward = reward_dev; a.mpjpe = mpjpe_dev; a.terminated = terminated_dev; a.truncated = truncated_dev;
  a.frames = frames_dev;
  a.k[0] = cfg->k_pos; a.k[1] = cfg->k_rot; a.k[2] = cfg->k_vel; a.k[3] = cfg->k_angvel;
  a.w[0] = cfg->w_pos; a.w[1] = cfg->w_rot; a.w[2] = cfg->w_vel; a.w[3] = cfg->w_angvel;
  a.term_dist = cfg->termination_distance; a.dt = (float)h->ctrl_dt; a.episode_length = cfg->episode_length;
  a.n = h->num_envs; a.nb = H.nb; a.J = cfg->num_tracked; a.self_dim = H.self_obs_dim; a.self_stride = H.obs_dim; a.obs_only = obs_only ? 1 : 0;
  for (int j = 0; j < a.J; j++) a.body[j] = (unsigned char)(cfg->tracked_bodies ? cfg->tracked_bodies[j] : j);
  a.T = std::max(cfg->num_future, 1); a.future_dt = cfg->future_dt;
  ImRec rk; std::memset(&rk, 0, sizeof rk);
  rk.zof = r.zero_out_far; rk.far = r.far_distance; rk.power_k = r.power_coefficient; rk.nu = H.nu; rk.nv = H.nv;
  rk.recovery = r.recovery; rk.goal = r.goal_dist; rk.qvel = r.qvel; rk.ctrl = aux->ctrl; rk.power = r.power;
  // [interpolate][more than one target][recovery]; fail-state recovery runs in its own instances, so that with every recovery field
  // zero the task is the one before it existed
  static void (*const kernels[2][2][2])(const float*, ImArgs, ImRec) = {
      {{k_imitation<0, 0, 0>, k_imitation<0, 0, 1>}, {k_imitation<0, 1, 0>, k_imitation<0, 1, 1>}},
      {{k_imitation<1, 0, 0>, k_imitation<1, 0, 1>}, {k_imitation<1, 1, 0>, k_imitation<1, 1, 1>}}};
  const bool rec = r.zero_out_far || power || r.recovery || r.goal_dist;
  const int wpb = 8, grid = (a.n + wpb - 1) / wpb;
  L_LAUNCH(kernels[cfg->interpolate][a.T > 1][rec], grid, 32 * wpb, 0, (cudaStream_t)stream, h->dimg, a, rk);
  CUDA_TRY(cudaGetLastError());
  return SMPLSIM_OK;
}

extern "C" int smplsim_imitation(SmplsimHandle* h, const SmplsimImitationCfg* cfg, const SmplsimMotionTables* tab, const int32_t* motion_ids_dev,
                                 const float* motion_t0_dev, const int32_t* progress_dev, const SmplsimAux* aux, const float* self_obs_dev,
                                 const uint8_t* mask_dev, int obs_only, float* obs_dev, float* reward_dev, uint8_t* terminated_dev,
                                 uint8_t* truncated_dev, float* mpjpe_dev, int32_t* frames_dev, void* stream) {
  return imitation(h, cfg, nullptr, tab, motion_ids_dev, motion_t0_dev, progress_dev, aux, self_obs_dev, mask_dev, obs_only, obs_dev, reward_dev,
                   terminated_dev, truncated_dev, mpjpe_dev, frames_dev, stream);
}

extern "C" int smplsim_imitation_recovery(SmplsimHandle* h, const SmplsimImitationCfg* cfg, const SmplsimImitationRecovery* rec,
                                          const SmplsimMotionTables* tab, const int32_t* motion_ids_dev, const float* motion_t0_dev,
                                          const int32_t* progress_dev, const SmplsimAux* aux, const float* self_obs_dev, const uint8_t* mask_dev,
                                          int obs_only, float* obs_dev, float* reward_dev, uint8_t* terminated_dev, uint8_t* truncated_dev,
                                          float* mpjpe_dev, int32_t* frames_dev, void* stream) {
  if (!rec) return fail(SMPLSIM_EINVAL, "smplsim_imitation_recovery: null recovery fields");
  return imitation(h, cfg, rec, tab, motion_ids_dev, motion_t0_dev, progress_dev, aux, self_obs_dev, mask_dev, obs_only, obs_dev, reward_dev,
                   terminated_dev, truncated_dev, mpjpe_dev, frames_dev, stream);
}

// ------------------------------------------------------------------ tracking evaluation (track_eval_kernels.cuh)
extern "C" int smplsim_track_eval(SmplsimHandle* h, const SmplsimTrackEvalCfg* cfg, const SmplsimMotionTables* tab, const int32_t* motion_ids_dev,
                                  const float* motion_t0_dev, const int32_t* progress_dev, const SmplsimAux* aux, const uint8_t* terminated_dev,
                                  const uint8_t* truncated_dev, const SmplsimTrackEvalState* state, void* stream) {
  if (!h || !cfg || !tab || !aux || !state) return fail(SMPLSIM_EINVAL, "smplsim_track_eval: null handle / cfg / tables / aux / state");
  const LHdr& H = *h->img.hdr();
  if (cfg->num_bodies < 3 || cfg->num_bodies > H.nb) return fail(SMPLSIM_EINVAL, "smplsim_track_eval: num_bodies outside [3, nbody]");
  if (!cfg->bodies && cfg->num_bodies != H.nb) return fail(SMPLSIM_EINVAL, "smplsim_track_eval: bodies NULL needs num_bodies == nbody");
  if (cfg->bodies && !bodies_in_range(cfg->bodies, cfg->num_bodies, H.nb))
    return fail(SMPLSIM_EINVAL, "smplsim_track_eval: eval body out of range [0, nbody)");
  TeArgs t; std::memset(&t, 0, sizeof t);
  ImArgs& a = t.im;
  const std::string why = motion_tables(H, tab, a);
  if (!why.empty()) return fail(SMPLSIM_EINVAL, "smplsim_track_eval: " + why);
  if (!aux->xpos || !aux->xquat) return fail(SMPLSIM_EINVAL, "smplsim_track_eval: aux needs xpos, xquat");
  if (!motion_ids_dev || !motion_t0_dev || !progress_dev || !terminated_dev || !truncated_dev) return fail(SMPLSIM_EINVAL, "smplsim_track_eval: null argument");
  if (!state->active || !state->prev_diff || !state->frames || !state->sums || !state->success)
    return fail(SMPLSIM_EINVAL, "smplsim_track_eval: null state array");
  if (cfg->interpolate != 0 && cfg->interpolate != 1) return fail(SMPLSIM_EINVAL, "smplsim_track_eval: interpolate must be 0 or 1");
  if (!(cfg->dt >= 0.f)) return fail(SMPLSIM_EINVAL, "smplsim_track_eval: dt < 0 or NaN");
  DeviceGuard guard(h->device);
  a.ids = motion_ids_dev; a.t0 = motion_t0_dev; a.progress = progress_dev;
  a.xpos = aux->xpos; a.xquat = aux->xquat;
  a.dt = cfg->dt > 0.f ? cfg->dt : (float)h->ctrl_dt;
  a.n = h->num_envs; a.nb = H.nb; a.J = cfg->num_bodies;
  for (int j = 0; j < a.J; j++) a.body[j] = (unsigned char)(cfg->bodies ? cfg->bodies[j] : j);
  t.terminated = terminated_dev; t.truncated = truncated_dev;
  t.active = state->active; t.prev_diff = state->prev_diff; t.frames = state->frames; t.sums = state->sums; t.success = state->success;
  t.frame_metrics = state->frame_metrics;
  static void (*const kernels[2])(TeArgs) = {k_track_eval<0>, k_track_eval<1>};   // [interpolate]
  const int wpb = 8, grid = (a.n + wpb - 1) / wpb;
  L_LAUNCH(kernels[cfg->interpolate], grid, 32 * wpb, 0, (cudaStream_t)stream, t);
  CUDA_TRY(cudaGetLastError());
  return SMPLSIM_OK;
}

// ------------------------------------------------------------------ adversarial motion priors (amp_kernels.cuh)
static int amp_dim(const LHdr& H, const SmplsimAmpCfg* cfg) {
  return (cfg->root_height_obs ? 1 : 0) + 12 + 6 * (H.nb - 1) + (H.nv - 6) + 3 * cfg->num_key_bodies;
}
// the arguments every AMP call shares; "" when they are good, else the reason (SMPLSIM_EINVAL, or EUNSUPPORTED when *code says so)
static std::string amp_check(const SmplsimHandle* h, const SmplsimAmpCfg* cfg, int* code) {
  *code = SMPLSIM_EINVAL;
  if (!h || !cfg) return "null handle / cfg";
  const LHdr& H = *h->img.hdr();
  if (cfg->num_steps < 1) return "num_steps < 1";
  if (cfg->interpolate != 0 && cfg->interpolate != 1) return "interpolate must be 0 or 1";
  if (cfg->num_key_bodies < 0 || cfg->num_key_bodies > H.nb) return "num_key_bodies outside [0, nbody]";
  if (cfg->num_key_bodies > 0 && !cfg->key_bodies) return "key_bodies NULL with num_key_bodies > 0";
  if (!bodies_in_range(cfg->key_bodies, cfg->num_key_bodies, H.nb)) return "key body out of range [0, nbody)";
  // dof_to_obs takes every non-root joint as a 3-dof exp map (the reference asserts on any other joint)
  bool hinge3 = H.nv == 6 + 3 * (H.nb - 1);
  for (int b = 1; b < H.nb && hinge3; b++) hinge3 = h->img.bodies()[b].dofadr == 6 + 3 * (b - 1);
  if (!hinge3) { *code = SMPLSIM_EUNSUPPORTED; return "every non-root body must have exactly 3 hinges"; }
  return "";
}
static std::string amp_tables(const LHdr& H, const SmplsimAmpTables* tab, AmpArgs& a) {
  if (!tab || !tab->motion) return "null motion tables";
  const std::string why = motion_tables(H, tab->motion, a);
  if (!why.empty()) return why;
  if (!tab->dof_pos || !tab->dof_vel) return "null motion table";
  a.tdof = tab->dof_pos; a.tdofv = tab->dof_vel;
  return "";
}
static void (*const amp_kernels[2])(const float*, AmpArgs) = {k_amp_obs<0>, k_amp_obs<1>};   // [interpolate]
static void amp_common(const SmplsimHandle* h, const SmplsimAmpCfg* cfg, AmpArgs& a) {
  const LHdr& H = *h->img.hdr();
  a.K = cfg->num_steps; a.F = amp_dim(H, cfg); a.nb = H.nb; a.nv = H.nv; a.nkey = cfg->num_key_bodies;
  a.local_root = cfg->local_root_obs ? 1 : 0; a.root_h = cfg->root_height_obs ? 1 : 0; a.dt = (float)h->ctrl_dt;
  for (int k = 0; k < a.nkey; k++) a.key[k] = (unsigned char)cfg->key_bodies[k];
}

extern "C" int smplsim_amp_obs_dim(const SmplsimHandle* h, const SmplsimAmpCfg* cfg) {
  int code;
  const std::string why = amp_check(h, cfg, &code);
  if (!why.empty()) return fail(code, "smplsim_amp_obs_dim: " + why);
  return amp_dim(*h->img.hdr(), cfg);
}

extern "C" int smplsim_amp_obs(SmplsimHandle* h, const SmplsimAmpCfg* cfg, const SmplsimState* st, const SmplsimAux* aux,
                               const SmplsimAmpTables* tab, const int32_t* motion_ids_dev, const float* motion_t0_dev, const uint8_t* mask_dev,
                               int mode, float* amp_obs_dev, void* stream) {
  int code;
  std::string why = amp_check(h, cfg, &code);
  if (!why.empty()) return fail(code, "smplsim_amp_obs: " + why);
  if (mode < SMPLSIM_AMP_PUSH || mode > SMPLSIM_AMP_FILL_REF) return fail(SMPLSIM_EINVAL, "smplsim_amp_obs: unknown mode");
  if (!st || !st->qpos || !st->qvel || !aux || !aux->xpos || !aux->xquat || !amp_obs_dev)
    return fail(SMPLSIM_EINVAL, "smplsim_amp_obs: null state (qpos, qvel), aux (xpos, xquat) or output");
  AmpArgs a; std::memset(&a, 0, sizeof a);
  if (mode == SMPLSIM_AMP_FILL_REF) {
    why = amp_tables(*h->img.hdr(), tab, a);
    if (!why.empty()) return fail(SMPLSIM_EINVAL, "smplsim_amp_obs: " + why);
    if (!motion_ids_dev || !motion_t0_dev || !st->progress) return fail(SMPLSIM_EINVAL, "smplsim_amp_obs: FILL_REF needs motion_ids, motion_t0 and state.progress");
  }
  DeviceGuard guard(h->device);
  amp_common(h, cfg, a);
  a.ids = motion_ids_dev; a.t0 = motion_t0_dev; a.progress = st->progress; a.mask = mask_dev;
  a.qpos = st->qpos; a.qvel = st->qvel; a.xpos = aux->xpos; a.xquat = aux->xquat; a.out = amp_obs_dev;
  a.n = h->num_envs; a.mode = mode;
  const int wpb = 8;
  L_LAUNCH(amp_kernels[cfg->interpolate], (a.n + wpb - 1) / wpb, 32 * wpb, 0, (cudaStream_t)stream, h->dimg, a);
  CUDA_TRY(cudaGetLastError());
  return SMPLSIM_OK;
}

extern "C" int smplsim_amp_demo(SmplsimHandle* h, const SmplsimAmpCfg* cfg, const SmplsimAmpTables* tab, const int32_t* motion_ids_dev,
                                const float* motion_times_dev, int n, float* out_dev, void* stream) {
  int code;
  std::string why = amp_check(h, cfg, &code);
  if (!why.empty()) return fail(code, "smplsim_amp_demo: " + why);
  if (n < 0) return fail(SMPLSIM_EINVAL, "smplsim_amp_demo: n < 0");
  AmpArgs a; std::memset(&a, 0, sizeof a);
  why = amp_tables(*h->img.hdr(), tab, a);
  if (!why.empty()) return fail(SMPLSIM_EINVAL, "smplsim_amp_demo: " + why);
  if (n == 0) return SMPLSIM_OK;
  if (!motion_ids_dev || !motion_times_dev || !out_dev) return fail(SMPLSIM_EINVAL, "smplsim_amp_demo: null motion_ids / motion_times / output");
  DeviceGuard guard(h->device);
  amp_common(h, cfg, a);
  a.ids = motion_ids_dev; a.t0 = motion_times_dev; a.out = out_dev; a.n = n; a.mode = AMP_DEMO;
  const int wpb = 8;
  L_LAUNCH(amp_kernels[cfg->interpolate], (n + wpb - 1) / wpb, 32 * wpb, 0, (cudaStream_t)stream, h->dimg, a);
  CUDA_TRY(cudaGetLastError());
  return SMPLSIM_OK;
}

extern "C" int smplsim_gae(const float* rewards_dev, const float* not_done_dev, const float* not_dead_dev, const float* values_dev,
                           const float* next_value_dev, float gamma, float tau, int T, int N, float* adv_dev, float* ret_dev, void* stream) {
  if (!rewards_dev || !not_done_dev || !not_dead_dev || !values_dev || !adv_dev || !ret_dev || T < 0 || N < 0)
    return fail(SMPLSIM_EINVAL, "smplsim_gae: null argument");
  if (T == 0 || N == 0) return SMPLSIM_OK;
  L_LAUNCH(k_gae, (N + 127) / 128, 128, 0, (cudaStream_t)stream, rewards_dev, not_done_dev, not_dead_dev, values_dev, next_value_dev, gamma, tau, T, N, adv_dev, ret_dev);
  CUDA_TRY(cudaGetLastError());
  return SMPLSIM_OK;
}

#ifdef SMPLSIM_STATS
extern "C" int smplsim_debug_stats(int* out, int reset) {   // out: L_NSTATS counters
#ifdef SMPLSIM_EMU
  for (int i = 0; i < L_NSTATS; i++) { out[i] = g_lstats[i]; if (reset) g_lstats[i] = 0; }
#else
  cudaDeviceSynchronize();
  cudaMemcpyFromSymbol(out, g_lstats, sizeof(int) * L_NSTATS);
  if (reset) { int z[L_NSTATS] = {0}; cudaMemcpyToSymbol(g_lstats, z, sizeof z); }
#endif
  return 0;
}
#endif

#ifdef SMPLSIM_EMU
#include "rollout_kernels.cu"   // the device build compiles it as a translation unit of its own (_lib.build)
#include "rollout_feedback_kernels.cu"   // as rollout_kernels.cu
#include "inverse_fd_kernels.cu"   // as rollout_kernels.cu
#include "centroidal_kernels.cu"   // as rollout_kernels.cu
#include "rne_post_kernels.cu"   // as rollout_kernels.cu
#endif
