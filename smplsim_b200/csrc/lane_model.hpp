// lane_model.hpp -- constant table of the lane-chain stepper (lane_kernels.cuh) and its host-side builder.
//
// The table is the float32 image of SmplsimModelDesc (include/smplsim.h; replaces mujoco.MjModel for this path,
// smpl_sim/envs/base_env.py:139-142) plus a host-computed *lane schedule*: every env is stepped by LM_LPE = 8 lanes, a
// lane walks a kinematic chain one body per sweep step, parents strictly before children.  When a body runs on the lane
// that ran its parent in the previous step the sweep state is handed over in registers ("carry"); every other tree edge
// goes through a small shared-memory mailbox.  One image per handle lives in global memory; each CTA stages it into
// shared memory once (bulk copy).
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "../../include/smplsim.h"

#define LM_LPE 8        // lanes per env
#define LM_TMAX 20      // sweep steps
#define LM_MAXMB 8      // mailbox children per body
#define LM_MAXB 64
#define LM_MAXG 64

// flags of LBody
#define LB_CARRY_OUT 1   // parent ran on this lane in the previous (outward) step: FK / acceleration state arrives in registers
#define LB_CARRY_IN 2    // one child runs on this lane in the next (outward) step: its articulated inertia arrives in registers

struct LHdr {
  int nb, nv, nu, ng, nslot, T, nmbi, nmbo;
  int obs_dim, self_obs_dim, warmset, dirtypath;
  int bytes, body_off, geom_off, align;         // image size, byte offsets of the LBody (== LM_BODY_OFF) / LGeom arrays, CTA alignment bits
  int pair_off, npair, axes_xyz, pad5;          // capsule / sphere geom pairs MuJoCo would collide (LPair array at pair_off); axes_xyz: every non-root
                                                // body has the identity body quaternion and hinge axes x, y, z (the SMPL family's MJCF)
  float ls_tol, margin, mu, impratio;
  float solimp[5], imp_a, imp_b, K;
  float B, h, grav[3], plane_pos[3];
  float plane_n[3], t1_default[3], pad1[2];
  float rarm[6], pad4[2];                      // armature of the six free-joint dofs
  unsigned long long legal_mask;
  const float* prm;                            // device address of the handle's per-env parameter records (smplsim_set_env_params; NULL: none).
                                               // Written into the device copy of the table only; read by the kernel instances with LCfg::PRM
  SmplsimEnvCfg cfg;
  signed char sched[LM_TMAX][LM_LPE];          // body of (step, lane) or -1
  unsigned char step_ng[LM_TMAX];              // per step: max geoms of a scheduled body (uniform loop bounds)
  unsigned char step_nmb[LM_TMAX];             // per step: max mailbox children
  unsigned char step_root[LM_TMAX];            // 1: this step holds the root body (free joint, 6 dofs)
  unsigned char pad3[LM_TMAX];
  unsigned carry_mask[LM_LPE];                 // per lane: bit t = the body of (step t, lane) takes its parent's state in registers (LB_CARRY_OUT)
};

struct LBody {   // 72 words
  float bpos[3], mass;
  float bquat[4];
  float ipos[3], tiw0;
  float inertia[6], pad0[2];
  float axis[9], arm[3];
  float kp[3], kd[3], tlim[3], ascale[3];
  float aoffset[3], diw0[3], rlo[3], rhi[3];
  int parent, dofadr, flags, geom0;
  int ngeom, limited, in_mbox, out_mbox;       // limited: bit k = dof k has a range ; mailbox ids or -1
  int pmbox, nmb, step, lane;                  // pmbox: parent's outward mailbox (-1: carry)
  signed char mb[LM_MAXMB];                    // inward mailboxes of the children that do not arrive by carry
  unsigned anc[2];                             // bit a (word a / 32): body a is this body or one of its ancestors
};

#define LM_BODY_OFF ((sizeof(LHdr) + 15) & ~(size_t)15)   // byte offset of the LBody array in the image (compile-time: the kernels add no header load)

struct LGeom {   // 20 words
  float pos[3], pad0;
  float size[3], pad1;
  float mat[9];
  int type, body, slot0;
};

struct LPair { short g1, g2; };   // geom indices, g1 < g2
struct LaneImage {
  std::vector<unsigned char> bytes;
  LHdr* hdr() { return (LHdr*)bytes.data(); }
  const LHdr* hdr() const { return (const LHdr*)bytes.data(); }
  LBody* bodies() { return (LBody*)(bytes.data() + hdr()->body_off); }
  const LBody* bodies() const { return (const LBody*)(bytes.data() + hdr()->body_off); }
  LGeom* geoms() { return (LGeom*)(bytes.data() + hdr()->geom_off); }
};

static inline int lane_obs_dims(const SmplsimModelDesc* s, const SmplsimEnvCfg* c, int* self_dim) {
  int nb = s->nbody;
  int n = (c->root_height_obs ? 1 : 0) + 3 * (nb - 1) + 6 * nb;   // humanoid_env.py:293-299
  n += (c->self_obs_v == 1) ? 3 + 3 + s->nu : 6 * nb;
  *self_dim = n;
  if (c->task == SMPLSIM_TASK_SPEED || c->task == SMPLSIM_TASK_REACH) n += 3;
  if (c->task == SMPLSIM_TASK_GETUP) n += 1;
  return n;
}

// Builds the image; returns "" on success or the reason the model is outside the supported class.
static inline std::string lane_build(const SmplsimModelDesc* s, const SmplsimEnvCfg* cfg, LaneImage& out) {
  const int nb = s->nbody, ng = s->ngeom;
  if (nb < 1 || nb > LM_MAXB || ng > LM_MAXG) return "model exceeds compiled limits (bodies <= 64, geoms <= 64)";
  if (s->nq != s->nv + 1 || s->nu != s->nv - 6 || s->body_dofnum[0] != 6 || s->body_parent[0] != -1)
    return "model class: one tree rooted at a free joint, hinge joints elsewhere";
  for (int b = 1; b < nb; b++) {
    if (s->body_parent[b] < 0 || s->body_parent[b] >= b) return "bodies must be listed parent-first";
    if (s->body_dofnum[b] != 3) return "model class: exactly three hinges on every non-root body (SMPL family)";
    if (s->body_dofadr[b] != 6 + 3 * (b - 1)) return "model class: dofs numbered in body order";
  }
  // ---- geom pairs that pass MuJoCo's filters (same body, filterparent, contype / conaffinity, <exclude>); capsule / sphere only
  std::vector<LPair> pairs;
  if (s->geom_contype && s->geom_conaffinity) {
    for (int g1 = 0; g1 < ng; g1++) {
      int t1 = s->geom_type[g1], b1 = s->geom_body[g1];
      if (t1 != SMPLSIM_GEOM_CAPSULE && t1 != SMPLSIM_GEOM_SPHERE) continue;
      for (int g2 = g1 + 1; g2 < ng; g2++) {
        int t2 = s->geom_type[g2], b2 = s->geom_body[g2];
        if (t2 != SMPLSIM_GEOM_CAPSULE && t2 != SMPLSIM_GEOM_SPHERE) continue;
        if (b1 == b2 || s->body_parent[b1] == b2 || s->body_parent[b2] == b1) continue;
        if (!((s->geom_contype[g1] & s->geom_conaffinity[g2]) || (s->geom_contype[g2] & s->geom_conaffinity[g1]))) continue;
        bool skip = false;
        for (int e = 0; e < s->nexclude; e++) {
          int x = s->exclude_pairs[2 * e], y = s->exclude_pairs[2 * e + 1];
          if ((x == b1 && y == b2) || (x == b2 && y == b1)) skip = true;
        }
        if (!skip) { LPair p; p.g1 = (short)g1; p.g2 = (short)g2; pairs.push_back(p); }
      }
    }
  }
  size_t body_off = LM_BODY_OFF, geom_off = body_off + sizeof(LBody) * nb;
  size_t pair_off = (geom_off + sizeof(LGeom) * ng + 15) & ~(size_t)15;
  size_t total = (pair_off + sizeof(LPair) * pairs.size() + 15) & ~(size_t)15;
  out.bytes.assign(total, 0);
  LHdr& H = *out.hdr();
  H.nb = nb; H.nv = s->nv; H.nu = s->nu; H.ng = ng; H.bytes = (int)total; H.body_off = (int)body_off; H.geom_off = (int)geom_off;
  H.pair_off = (int)pair_off; H.npair = (int)pairs.size();
  if (!pairs.empty()) memcpy(out.bytes.data() + pair_off, pairs.data(), sizeof(LPair) * pairs.size());
  LBody* B = out.bodies();
  LGeom* G = out.geoms();
  // ---- tree, heights
  std::vector<int> parent(nb), height(nb, 0), step(nb, -1), lane(nb, -1);
  std::vector<std::vector<int>> child(nb);
  for (int b = 0; b < nb; b++) { parent[b] = s->body_parent[b]; if (b) child[parent[b]].push_back(b); }
  for (int b = nb - 1; b > 0; b--) height[parent[b]] = std::max(height[parent[b]], height[b] + 1);
  // ---- list schedule on LM_LPE lanes, chains kept on their lane
  step[0] = 0; lane[0] = 0;
  memset(H.sched, -1, sizeof H.sched);
  H.sched[0][0] = 0;
  int done = 1, t = 1;
  while (done < nb) {
    if (t >= LM_TMAX) return "lane schedule longer than LM_TMAX steps";
    std::vector<int> ready;
    for (int b = 1; b < nb; b++) if (step[b] < 0 && step[parent[b]] >= 0 && step[parent[b]] < t) ready.push_back(b);
    std::sort(ready.begin(), ready.end(), [&](int a, int c) { return height[a] != height[c] ? height[a] > height[c] : a < c; });
    bool taken[LM_LPE] = {false};
    std::vector<int> rest;
    for (int b : ready) {   // carry: the tallest ready child of a body that ran in step t-1 inherits its lane
      int p = parent[b];
      if (step[p] == t - 1 && !taken[lane[p]]) { taken[lane[p]] = true; step[b] = t; lane[b] = lane[p]; done++; }
      else rest.push_back(b);
    }
    for (int b : rest) {
      int L = -1;
      for (int l = 0; l < LM_LPE; l++) if (!taken[l]) { L = l; break; }
      if (L < 0) break;
      taken[L] = true; step[b] = t; lane[b] = L; done++;
    }
    for (int b = 1; b < nb; b++) if (step[b] == t) H.sched[t][lane[b]] = (signed char)b;
    t++;
  }
  H.T = t;
  // ---- bodies
  int nmbi = 0, nmbo = 0;
  for (int b = 0; b < nb; b++) {
    LBody& L = B[b];
    for (int k = 0; k < 3; k++) { L.bpos[k] = (float)s->body_pos[3 * b + k]; L.ipos[k] = (float)s->body_ipos[3 * b + k]; }
    for (int k = 0; k < 4; k++) L.bquat[k] = (float)s->body_quat[4 * b + k];
    for (int k = 0; k < 6; k++) L.inertia[k] = (float)s->body_inertia[6 * b + k];
    L.mass = (float)s->body_mass[b]; L.tiw0 = (float)s->body_invweight0[2 * b];
    L.parent = parent[b]; L.dofadr = s->body_dofadr[b]; L.step = step[b]; L.lane = lane[b];
    L.anc[0] = L.anc[1] = 0u;
    for (int a = b; a >= 0; a = parent[a]) L.anc[a >> 5] |= 1u << (a & 31);
    L.in_mbox = L.out_mbox = L.pmbox = -1; L.nmb = 0; L.geom0 = 0; L.ngeom = 0; L.limited = 0; L.flags = 0;
    memset(L.mb, -1, sizeof L.mb);
    if (b > 0) {
      int d0 = L.dofadr;
      for (int k = 0; k < 3; k++) {
        int d = d0 + k, a = d - 6;
        for (int j = 0; j < 3; j++) L.axis[3 * k + j] = (float)s->dof_axis[3 * d + j];
        L.arm[k] = (float)s->dof_armature[d]; L.diw0[k] = (float)s->dof_invweight0[d];
        L.rlo[k] = (float)s->dof_range[2 * d]; L.rhi[k] = (float)s->dof_range[2 * d + 1];
        if (s->dof_limited[d]) L.limited |= 1 << k;
        L.kp[k] = (float)s->act_kp[a]; L.kd[k] = (float)s->act_kd[a]; L.tlim[k] = (float)s->act_torque_lim[a];
        L.ascale[k] = (float)s->act_scale[a]; L.aoffset[k] = (float)s->act_offset[a];
      }
      // register hand-over along a chain; never into the root: the root carries constraint rows in its subtree in nearly every
      // substep, and a carry child would drag its whole chain into every re-sweep of the active-set iterations
      if (parent[b] != 0 && step[parent[b]] == step[b] - 1 && lane[parent[b]] == lane[b]) { L.flags |= LB_CARRY_OUT; B[parent[b]].flags |= LB_CARRY_IN; }
    }
  }
  for (int b = 1; b < nb; b++) {
    if (B[b].flags & LB_CARRY_OUT) continue;
    LBody& P = B[parent[b]];
    if (P.out_mbox < 0) P.out_mbox = nmbo++;
    B[b].pmbox = P.out_mbox;
    B[b].in_mbox = nmbi++;
    if (P.nmb >= LM_MAXMB) return "more than 8 mailbox children on one body";
    P.mb[P.nmb++] = (signed char)B[b].in_mbox;
  }
  H.nmbi = nmbi; H.nmbo = nmbo;
  H.axes_xyz = 1;
  for (int b = 1; b < nb; b++) {
    const LBody& L = B[b];
    if (L.bquat[0] != 1.f || L.bquat[1] != 0.f || L.bquat[2] != 0.f || L.bquat[3] != 0.f) H.axes_xyz = 0;
    for (int k = 0; k < 3; k++) for (int j = 0; j < 3; j++) if (L.axis[3 * k + j] != (k == j ? 1.f : 0.f)) H.axes_xyz = 0;
  }
  for (int l = 0; l < LM_LPE; l++) {
    H.carry_mask[l] = 0u;
    for (int tt = 1; tt < H.T; tt++) { int b = H.sched[tt][l]; if (b >= 0 && (B[b].flags & LB_CARRY_OUT)) H.carry_mask[l] |= 1u << tt; }
  }
  // ---- geoms (grouped per body) and their contact slots
  int ns = 0;
  H.legal_mask = 1ull;
  {
    std::vector<int> order;
    for (int b = 0; b < nb; b++) for (int g = 0; g < ng; g++) if (s->geom_body[g] == b) order.push_back(g);
    if ((int)order.size() != ng) return "geom attached to an unknown body";
    // geoms keep their MuJoCo index (contact_mask bit g + 1); a body's geoms must be contiguous so (geom0, ngeom) addresses them
    for (int b = 0; b < nb; b++) {
      int first = -1, cnt = 0;
      for (int g = 0; g < ng; g++) if (s->geom_body[g] == b) { if (first < 0) first = g; cnt++; }
      if (cnt && s->geom_body[first + cnt - 1] != b) return "a body's geoms must be contiguous in the geom list";
      for (int g = first; g >= 0 && g < first + cnt; g++) if (s->geom_body[g] != b) return "a body's geoms must be contiguous in the geom list";
      B[b].geom0 = first < 0 ? 0 : first; B[b].ngeom = cnt;
    }
  }
  for (int g = 0; g < ng; g++) {
    LGeom& Q = G[g];
    Q.type = s->geom_type[g]; Q.body = s->geom_body[g];
    int mc = Q.type == SMPLSIM_GEOM_BOX ? 4 : Q.type == SMPLSIM_GEOM_CAPSULE ? 2 : Q.type == SMPLSIM_GEOM_SPHERE ? 1 : -1;
    if (mc < 0 || Q.body < 0 || Q.body >= nb) return "geom type (box|capsule|sphere) / body";
    Q.slot0 = ns; ns += mc;
    for (int k = 0; k < 3; k++) { Q.pos[k] = (float)s->geom_pos[3 * g + k]; Q.size[k] = (float)s->geom_size[3 * g + k]; }
    for (int k = 0; k < 9; k++) Q.mat[k] = (float)s->geom_mat[9 * g + k];
    if (s->geom_legal[g]) H.legal_mask |= 1ull << (g + 1);
  }
  if (ng > 63) return "at most 63 robot geoms (contact_mask is a 64-bit word, bit 0 is the floor)";
  H.nslot = ns;
  for (int tt = 0; tt < H.T; tt++) {
    int mg = 0, mm = 0, rt = 0;
    for (int l = 0; l < LM_LPE; l++) {
      int b = H.sched[tt][l];
      if (b < 0) continue;
      mg = std::max(mg, B[b].ngeom); mm = std::max(mm, B[b].nmb);
      if (b == 0) rt = 1;
    }
    H.step_ng[tt] = (unsigned char)mg; H.step_nmb[tt] = (unsigned char)mm; H.step_root[tt] = (unsigned char)rt;
  }
  // ---- scalars
  double nn = std::sqrt(s->plane_normal[0] * s->plane_normal[0] + s->plane_normal[1] * s->plane_normal[1] + s->plane_normal[2] * s->plane_normal[2]);
  double n[3] = {s->plane_normal[0] / nn, s->plane_normal[1] / nn, s->plane_normal[2] / nn};
  for (int k = 0; k < 3; k++) { H.plane_pos[k] = (float)s->plane_pos[k]; H.plane_n[k] = (float)n[k]; H.grav[k] = (float)s->gravity[k]; }
  { // mju_makeFrame default tangent for this normal (SURVEY.md A.5)
    double tv[3] = {0, 0, 0};
    if (n[1] < 0.5 && n[1] > -0.5) tv[1] = 1; else tv[2] = 1;
    double d = n[0] * tv[0] + n[1] * tv[1] + n[2] * tv[2];
    for (int k = 0; k < 3; k++) tv[k] -= d * n[k];
    double tn = std::sqrt(tv[0] * tv[0] + tv[1] * tv[1] + tv[2] * tv[2]);
    for (int k = 0; k < 3; k++) H.t1_default[k] = (float)(tv[k] / tn);
  }
  H.margin = (float)s->margin; H.mu = (float)s->friction[0]; H.impratio = (float)s->impratio;
  for (int k = 0; k < 5; k++) H.solimp[k] = (float)s->solimp[k];
  { double mid = s->solimp[3], pw = s->solimp[4];
    H.imp_a = (float)(1.0 / std::pow(mid, pw - 1)); H.imp_b = (float)(1.0 / std::pow(1 - mid, pw - 1)); }
  { double dmax = s->solimp[1], tc = s->solref[0], dr = s->solref[1];
    if (tc <= 0) return "direct solref (negative) is not supported";
    if (tc < 2 * s->timestep) tc = 2 * s->timestep;   // refsafe
    H.K = (float)(1.0 / std::fmax(1e-15, dmax * dmax * tc * tc * dr * dr)); H.B = (float)(2.0 / std::fmax(1e-15, dmax * tc)); }
  H.h = (float)s->timestep;
  for (int k = 0; k < 6; k++) H.rarm[k] = (float)s->dof_armature[k];
  H.cfg = *cfg;
  H.obs_dim = lane_obs_dims(s, cfg, &H.self_obs_dim);
  H.warmset = 1; H.dirtypath = 1; H.ls_tol = 1e-6f; H.align = 7;
  return "";
}
