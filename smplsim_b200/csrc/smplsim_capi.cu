// smplsim_capi.cu -- extern "C" boundary of libsmplsim_b200.so (see include/smplsim.h).
// Host side: constant table + lane schedule (lane_model.hpp), shared-memory sizing, launches of the lane-chain kernels.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "aux_kernels.cuh"

#ifdef SMPLSIM_EMU
#define L_LAUNCH(kern, grid, block, smem, stream, ...) emu::launch(dim3(grid), dim3(block), smem, [&]() { kern(__VA_ARGS__); })
#else
#define L_LAUNCH(kern, grid, block, smem, stream, ...) kern<<<grid, block, smem, stream>>>(__VA_ARGS__)
#endif

// model classes the kernels are instantiated for: <bodies, dofs, geoms, contact slots, in-mailboxes, out-mailboxes, contact
// entries in shared memory, limit rows, geom-geom rows compiled in>
#define L_SMPL(SC) LCfg<24, 75, 24, 64, 5, 2, 20, 16, SC>
#define L_SMPLX(SC) LCfg<52, 159, 52, 128, 13, 4, 14, 16, SC>

struct SmplsimHandle {
  LaneImage img;
  float* dimg = nullptr;   // device copy of the table
  float* gscr = nullptr;   // overflow contact entries
  float* gsens = nullptr;  // body velocities of the last forward pass (obs v2 / aux)
  int* gpfl = nullptr;     // working set per contact slot, carried from call to call (solver warm start only)
  float* gbody = nullptr;  // body pose / velocity of the current forward pass (self-collision narrow phase)
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
  LMap map() const { LMap m; m.slot_env = dslot_env; m.blk_img = dblk_img; return m; }
};

static thread_local std::string g_err;
static int fail(int code, const std::string& msg) { g_err = msg; return code; }
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
extern "C" int smplsim_version(void) { return 200; }   // 200: lane-chain kernels (round 2); ABI structs unchanged since 110

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
  if (cudaFuncSetAttribute(k_step5<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->smem) != cudaSuccess) return -1;
  if (cudaFuncSetAttribute(k_reset5<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->smem) != cudaSuccess) return -1;
  if (cudaFuncSetAttribute(k_kin5<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->smem) != cudaSuccess) return -1;
  return best;
}

template <class C>
static void run_step(SmplsimHandle* h, const LStepArgs& a, cudaStream_t st) {
  int wpb = h->wpb, per = wpb * C::EPW;
  L_LAUNCH(k_step5<C>, h->nblocks ? h->nblocks : (a.n + per - 1) / per, 32 * wpb, h->smem, st, h->dimg, h->img.hdr()->bytes, a);
}
template <class C>
static void run_reset(SmplsimHandle* h, const LResetArgs& a, cudaStream_t st) {
  int wpb = h->wpb, per = wpb * C::EPW;
  L_LAUNCH(k_reset5<C>, h->nblocks ? h->nblocks : (a.n + per - 1) / per, 32 * wpb, h->smem, st, h->dimg, h->img.hdr()->bytes, a);
}
template <class C>
static void run_kin(SmplsimHandle* h, const LKinArgs& a, cudaStream_t st) {
  int wpb = h->wpb, per = wpb * C::EPW;
  L_LAUNCH(k_kin5<C>, h->nblocks ? h->nblocks : (a.n + per - 1) / per, 32 * wpb, h->smem, st, h->dimg, h->img.hdr()->bytes, a);
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
  cudaFree(h->dimg); cudaFree(h->gscr); cudaFree(h->gsens); cudaFree(h->gpfl); cudaFree(h->gbody); cudaFree(h->dslot_env); cudaFree(h->dblk_img);
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
  DeviceGuard guard(cuda_device);
  cudaError_t e = cudaDeviceGetAttribute(&h->max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, cuda_device);
#ifndef SMPLSIM_EMU
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&h->nsm, cudaDevAttrMultiProcessorCount, cuda_device);
#endif
  if (e != cudaSuccess) { delete h; return fail(SMPLSIM_ECUDA, std::string("smplsim_create: ") + cudaGetErrorString(e)); }
  int ok = 0;
  L_DISPATCH(h, ok = pick_wpb<C_>(h));
  if (ok <= 0) { delete h; return fail(SMPLSIM_EUNSUPPORTED, "per-env rows exceed shared memory"); }
  size_t gs = 0;
  L_DISPATCH(h, gs = (size_t)C_::CONW * (C_::NS - C_::NCS));
  e = cudaMalloc(&h->dimg, (size_t)H.bytes * nmodels);
  if (e == cudaSuccess) e = cudaMemcpy(h->dimg, h->img.bytes.data(), H.bytes, cudaMemcpyHostToDevice);
  for (int k = 1; k < nmodels && e == cudaSuccess; k++) e = cudaMemcpy((char*)h->dimg + (size_t)H.bytes * k, more[k - 1].bytes.data(), H.bytes, cudaMemcpyHostToDevice);
  if (e == cudaSuccess && !h->env_model.empty()) {   // envs grouped by shape into whole CTAs (empty slots: -1)
    int per = 1;
    L_DISPATCH(h, per = h->wpb * C_::EPW);
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
  }
  if (e == cudaSuccess) e = cudaMalloc(&h->gscr, gs * (size_t)num_envs * 4 + 16);
  if (e == cudaSuccess) e = cudaMalloc(&h->gsens, (size_t)6 * H.nb * num_envs * 4);
  size_t pw = 0;
  L_DISPATCH(h, pw = (size_t)C_::PFLW);
  if (e == cudaSuccess) e = cudaMalloc(&h->gpfl, pw * num_envs * 4);
  if (e == cudaSuccess) e = cudaMemset(h->gpfl, 0, pw * num_envs * 4);
  if (e == cudaSuccess && cfg->self_collision) e = cudaMalloc(&h->gbody, (size_t)10 * H.nb * num_envs * 4);
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

static bool state_ok(const SmplsimState* st) {
  return st && st->qpos && st->qvel && st->qpos_fwd && st->qvel_fwd && st->qacc_warm && st->task_target && st->task_change_step &&
         st->progress && st->recovery && st->rng_counter;
}
static int want_sens(const SmplsimHandle* h, const SmplsimAux* aux) {
  return (h->img.hdr()->cfg.self_obs_v == 2 || (aux && (aux->body_linvel || aux->body_angvel))) ? 1 : 0;
}

extern "C" int smplsim_step(SmplsimHandle* h, const SmplsimState* st, const float* action_dev, float* obs_dev, float* reward_dev,
                            uint8_t* terminated_dev, uint8_t* truncated_dev, const SmplsimAux* aux, void* stream) {
  if (!h || !state_ok(st) || !action_dev) return fail(SMPLSIM_EINVAL, "smplsim_step: null handle/state/action");
  if (h->img.hdr()->cfg.control_mode == SMPLSIM_CTRL_SIMPLE_PID && (!st->pid_integral || !st->pid_last_error))
    return fail(SMPLSIM_EINVAL, "smplsim_step: control_mode simple_pid needs state.pid_integral / pid_last_error");
  DeviceGuard guard(h->device);
  LStepArgs a; std::memset(&a, 0, sizeof a);
  a.st = *st; if (aux) a.aux = *aux;
  a.action = action_dev; a.obs = obs_dev; a.reward = reward_dev; a.terminated = terminated_dev; a.truncated = truncated_dev;
  a.gscr = h->gscr; a.gpfl = h->gpfl; a.gbody = h->gbody; a.n = h->num_envs; a.nsub = h->img.hdr()->cfg.nsubsteps; a.mode = 0; a.map = h->map();
  a.gsens = want_sens(h, aux) ? h->gsens : nullptr;
  L_DISPATCH(h, run_step<C_>(h, a, (cudaStream_t)stream));
  CUDA_TRY(cudaGetLastError());
  return SMPLSIM_OK;
}

extern "C" int smplsim_mj_step(SmplsimHandle* h, const SmplsimState* st, const float* ctrl_dev, int nsub, const SmplsimAux* aux, void* stream) {
  if (!h || !state_ok(st) || !ctrl_dev || nsub < 1) return fail(SMPLSIM_EINVAL, "smplsim_mj_step: bad argument");
  DeviceGuard guard(h->device);
  LStepArgs a; std::memset(&a, 0, sizeof a);
  a.st = *st; if (aux) a.aux = *aux;
  a.action = ctrl_dev; a.gscr = h->gscr; a.gpfl = h->gpfl; a.gbody = h->gbody; a.n = h->num_envs; a.nsub = nsub; a.mode = 1; a.map = h->map();
  a.gsens = want_sens(h, aux) ? h->gsens : nullptr;
  L_DISPATCH(h, run_step<C_>(h, a, (cudaStream_t)stream));
  CUDA_TRY(cudaGetLastError());
  return SMPLSIM_OK;
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
  LResetArgs a; std::memset(&a, 0, sizeof a);
  a.st = *st; if (aux) a.aux = *aux;
  a.mask = mask_dev; a.qpos0 = qpos0_dev; a.qvel0 = qvel0_dev; a.obs = obs_dev; a.gscr = h->gscr; a.gpfl = h->gpfl; a.gbody = h->gbody; a.n = h->num_envs; a.init_mode = mode; a.map = h->map();
  a.gsens = want_sens(h, aux) ? h->gsens : nullptr;
  L_DISPATCH(h, run_reset<C_>(h, a, (cudaStream_t)stream));
  CUDA_TRY(cudaGetLastError());
  return SMPLSIM_OK;
}

extern "C" int smplsim_kinematics(SmplsimHandle* h, const float* qpos_dev, float* xpos_dev, float* xquat_dev, int n, void* stream) {
  if (!h || !qpos_dev || !xpos_dev || !xquat_dev || n < 0) return fail(SMPLSIM_EINVAL, "smplsim_kinematics: bad argument");
  if (n == 0) return SMPLSIM_OK;
  DeviceGuard guard(h->device);
  if (h->nblocks && n != h->num_envs) return fail(SMPLSIM_EINVAL, "smplsim_kinematics: with per-env body shapes n must be the handle's num_envs (row i uses env i's shape)");
  LKinArgs a; a.qpos = qpos_dev; a.xpos = xpos_dev; a.xquat = xquat_dev; a.n = n; a.map = h->map();
  L_DISPATCH(h, run_kin<C_>(h, a, (cudaStream_t)stream));
  CUDA_TRY(cudaGetLastError());
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
extern "C" int smplsim_debug_stats(int* out32, int reset) {
#ifdef SMPLSIM_EMU
  for (int i = 0; i < 32; i++) { out32[i] = g_lstats[i]; if (reset) g_lstats[i] = 0; }
#else
  cudaDeviceSynchronize();
  cudaMemcpyFromSymbol(out32, g_lstats, sizeof(int) * 32);
  if (reset) { int z[32] = {0}; cudaMemcpyToSymbol(g_lstats, z, sizeof z); }
#endif
  return 0;
}
#endif
