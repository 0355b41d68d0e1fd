/*
 * smplsim.h -- C ABI of libsmplsim_b200.so, the H100-native (sm_90a) batched SMPL-humanoid stepper.
 *
 * The reference (ZhengyiLuo/SMPLSim) has no FFI: its "operator API" for this path is the
 * Python protocol of smpl_sim/envs (SURVEY.md section 8b).  Each entry point below names
 * the reference call it replaces; INTEGRATION.md shows the ctypes binding a maintainer adds.
 *
 * Conventions
 *  - every *_dev pointer is caller-owned, contiguous device memory on the handle's GPU
 *    (PyTorch allocates it); nothing is retained past the call;
 *  - all calls are asynchronous on the caller's stream and never synchronise the host;
 *  - return 0 on success, negative SMPLSIM_E* on error, message via smplsim_last_error();
 *  - quaternions are wxyz (MuJoCo), qvel[3:6] is the root angular velocity in the body frame.
 */
#ifndef SMPLSIM_H_
#define SMPLSIM_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SMPLSIM_OK 0
#define SMPLSIM_EINVAL (-1)
#define SMPLSIM_ECUDA (-2)
#define SMPLSIM_EUNSUPPORTED (-3)

#define SMPLSIM_GEOM_PLANE 0
#define SMPLSIM_GEOM_SPHERE 2
#define SMPLSIM_GEOM_CAPSULE 3
#define SMPLSIM_GEOM_BOX 6

#define SMPLSIM_TASK_NONE 0  /* HumanoidEnv            smpl_sim/envs/humanoid_env.py:139 */
#define SMPLSIM_TASK_SPEED 1 /* HumanoidSpeed          smpl_sim/envs/tasks/humanoid_speed.py:49 */
#define SMPLSIM_TASK_REACH 2 /* HumanoidReach          smpl_sim/envs/tasks/humanoid_reach.py:33 */
#define SMPLSIM_TASK_GETUP 3 /* HumanoidGetup          smpl_sim/envs/tasks/humanoid_getup.py:27 */

#define SMPLSIM_CTRL_UHC_PD 0 /* StablePDController    smpl_sim/envs/controllers.py:50-190 */
#define SMPLSIM_CTRL_PD 1     /* PIDController (ki=0)  smpl_sim/envs/controllers.py:265-349 */
#define SMPLSIM_CTRL_TORQUE 2 /* SimpleTorqueController smpl_sim/envs/controllers.py:6-47 */
#define SMPLSIM_CTRL_SIMPLE_PID 3 /* SimplePID (stateful) smpl_sim/envs/controllers.py:186-262, built at humanoid_env.py:318-319:
                                   * act_kp = jkp/10, act_kd = jkd/10, Ki = 1, dt = timestep * control_freq_inv */

#define SMPLSIM_INIT_DEFAULT 0 /* humanoid_env.py:472-477 */
#define SMPLSIM_INIT_FALL 1    /* humanoid_env.py:478-491 */
#define SMPLSIM_INIT_MOCAP 2   /* state supplied by the caller (motion_lib feed) */

#define SMPLSIM_STATUS_SELF_CONTACT 32

/* The constant tree / inertia / geom / gain table (replaces mujoco.MjModel for this path,
 * smpl_sim/envs/base_env.py:139-142 + smpl_sim/envs/humanoid_env.py:262-370).  Host memory,
 * float64; copied during smplsim_create.  Robot bodies only (the world body is implicit);
 * geoms are the robot geoms, MuJoCo geom id = index + 1, the floor plane is geom 0. */
typedef struct SmplsimModelDesc {
  int32_t nbody, nq, nv, nu, ngeom;
  const int32_t* body_parent;    /* [nbody]  -1 for the root */
  const int32_t* body_dofadr;    /* [nbody]  first dof */
  const int32_t* body_dofnum;    /* [nbody]  6 for the free-joint root, <= 3 hinges otherwise */
  const double* body_pos;        /* [nbody*3] offset in the parent frame */
  const double* body_quat;       /* [nbody*4] */
  const double* body_mass;       /* [nbody] */
  const double* body_ipos;       /* [nbody*3] centre of mass, body frame */
  const double* body_inertia;    /* [nbody*6] xx yy zz xy xz yz about the COM, body frame */
  const double* body_invweight0; /* [nbody*2] */
  const double* dof_axis;        /* [nv*3]   hinge axis, body frame (rows 0..5 unused) */
  const double* dof_armature;    /* [nv] */
  const double* dof_invweight0;  /* [nv] */
  const double* dof_range;       /* [nv*2]   radians */
  const int32_t* dof_limited;    /* [nv] */
  const int32_t* geom_type;      /* [ngeom] */
  const int32_t* geom_body;      /* [ngeom] */
  const double* geom_pos;        /* [ngeom*3] */
  const double* geom_mat;        /* [ngeom*9] row-major 3x3, body frame */
  const double* geom_size;       /* [ngeom*3] box half extents | capsule (r, half_len) | sphere (r) */
  const int32_t* geom_legal;     /* [ngeom]  1: touching the floor does not terminate (contact_bodies) */
  double plane_pos[3];
  double plane_normal[3];
  double margin;
  double friction[3];
  double solref[2];
  double solimp[5];
  double impratio;
  double timestep;
  double gravity[3];
  const double* act_kp;         /* [nu] */
  const double* act_kd;         /* [nu] */
  const double* act_torque_lim; /* [nu] */
  const double* act_scale;      /* [nu] _pd_action_scale (or power_scale*lim in torque mode) */
  const double* act_offset;     /* [nu] */
  /* geom-geom collision filters of the MJCF (smpl_humanoid.xml:5,24,231-242): used to list the capsule / sphere pairs MuJoCo
   * would test.  Self-collision is NOT simulated yet; the pairs are tested once per env step and a touching pair raises
   * SMPLSIM_STATUS_SELF_CONTACT in aux.status.  geom_contype == NULL disables the check. */
  const int32_t* geom_contype;     /* [ngeom] or NULL */
  const int32_t* geom_conaffinity; /* [ngeom] or NULL */
  int32_t nexclude;
  const int32_t* exclude_pairs;    /* [nexclude*2] body indices of <contact><exclude> */
} SmplsimModelDesc;

/* cfg.env.* keys consumed on the path (smpl_sim/data/cfg/env/{speed,reach,getup}.yaml). */
typedef struct SmplsimEnvCfg {
  int32_t task;
  int32_t control_mode;
  int32_t self_obs_v;      /* 1 -> 289-dim, 2 -> 358-dim (SMPL) */
  int32_t root_height_obs; /* 0/1 */
  int32_t upright_start;   /* robot.has_upright_start */
  int32_t nsubsteps;       /* control_frequency_inv */
  int32_t episode_length;
  int32_t state_init;           /* SMPLSIM_INIT_* used by smplsim_reset when init_mode < 0 */
  int32_t spd_stale;            /* 1: SPD reads M,C of the previous forward pass (reference quirk Q1) */
  int32_t legacy_change_step;   /* 1: reset_task() sees the old cur_t (reference quirk Q4) */
  int32_t reach_body;           /* body index of env.reach_body_name */
  int32_t recovery_steps;       /* getup */
  int32_t change_steps_min, change_steps_max; /* speed/tar/height _change_steps_{min,max} */
  double tar_speed_min, tar_speed_max;        /* speed */
  double tar_dist_max;                        /* reach */
  double tar_height_min, tar_height_max;      /* reach / getup */
  uint64_t seed;                              /* Philox key for task sampling and Fall init */
  int32_t self_collision;  /* 1: geom-geom contacts between the capsule / sphere pairs MuJoCo's filters let through are simulated
                            *    (two-body rows; the reference MJCF enables them).  0: detected only (aux.status bit 32). */
  int32_t pad_;
} SmplsimEnvCfg;

/* Per-env simulation state, SoA tensors [N, ...] owned by the caller. */
typedef struct SmplsimState {
  float* qpos;              /* [N,nq] */
  float* qvel;              /* [N,nv] */
  float* qpos_fwd;          /* [N,nq] state of the last forward pass (mj_data.qM / qfrc_bias staleness) */
  float* qvel_fwd;          /* [N,nv] */
  float* qacc_warm;         /* [N,nv] mj_data.qacc_warmstart */
  float* task_target;       /* [N,4]  speed: tar_speed | reach: tar_pos xyz | getup: tar_height */
  int32_t* task_change_step; /* [N] */
  int32_t* progress;        /* [N]  cur_t */
  int32_t* recovery;        /* [N]  getup recovery counter */
  uint32_t* rng_counter;    /* [N]  Philox counter */
  float* pid_integral;      /* [N,nu] SimplePID._integral   (control_mode simple_pid only, else may be NULL); like the reference's
                             *        controller object it is NOT cleared by reset */
  float* pid_last_error;    /* [N,nu] SimplePID._last_error ; NaN = None (first call: d_error = 0) */
  const float* xfrc_applied; /* [N,nbody,6] or NULL: mj_data.xfrc_applied of the robot bodies (row 0 = root), read only.  Per body a
                              * world-frame force (fx fy fz) acting at the body's centre of mass and a world-frame torque (tx ty tz),
                              * as mj_xfrcAccumulate: qfrc_applied = Jp(xipos)^T f + Jr^T t.  It enters qfrc_smooth (hence qacc_smooth,
                              * the constraint solve and qacc), NOT qfrc_bias: the stable-PD controller never sees it directly.
                              * smplsim_step / smplsim_mj_step hold it constant over every substep of the call; smplsim_reset ignores
                              * it.  An env that auto-resets (mj_checkPos/Vel/Acc -> mj_resetData, which zeroes xfrc_applied) runs the
                              * rest of the call without it; the caller's array is never written. */
} SmplsimState;

/* Side outputs of the last forward pass / kinematics (any pointer may be NULL). */
typedef struct SmplsimAux {
  float* xpos;          /* [N,nbody,3]  mj_data.xpos[1:]  (post-integration, mj_kinematics) */
  float* xquat;         /* [N,nbody,4]  mj_data.xquat[1:] */
  float* body_linvel;   /* [N,nbody,3]  sensordata[:3nb]   (pre-integration, quirk Q2) */
  float* body_angvel;   /* [N,nbody,3]  sensordata[3nb:6nb] */
  uint64_t* contact_mask; /* [N] bit g: floor contact with MuJoCo geom id g in the last forward pass */
  float* qacc;          /* [N,nv] */
  float* ctrl;          /* [N,nu] torque applied in the last substep */
  int32_t* solver_iter; /* [N]   constraint-solver iterations of the last substep */
  uint8_t* status;      /* [N]   bits raised during this call (OR over substeps): mj_warning 1 BADQPOS, 2 BADQVEL, 4 BADQACC;
                         *       8 constraint rows dropped (too many simultaneous joint-limit rows), 16 solver stopped at its iteration cap,
                         *       32 SMPLSIM_STATUS_SELF_CONTACT: two robot geoms that MuJoCo would collide touch at the end of the step
                         *       (the contact is not simulated, the state differs from the reference from here on).
                         *       As in mj_step (mj_checkPos/Vel/Acc + mj_resetData) a NaN or |x| > 1e10 auto-resets that env's
                         *       data to qpos0 / zero velocity and the call carries on -- a device fault never traps. */
  float* contact_wrench; /* [N,nbody,6] or NULL: per robot body (rows as xpos / xfrc_applied, row 0 = root) the wrench the contacts of
                          * the last forward pass (the pass contact_mask, qacc and solver_iter describe: last substep, before integration)
                          * apply to it: [0:3] world-frame force, [3:6] world-frame torque of those forces about the body's centre of mass
                          * (xipos) -- the convention of xfrc_applied.  So sum_b Jp_b(xipos_b)^T F_b + Jr_b^T t_b is the contact part of
                          * qfrc_constraint (all of it but the joint-limit rows).  A floor contact on a geom of body b adds
                          * F = sum_k f_k (n +- mu t_k) of its four pyramid rows at the contact point; a geom-geom contact adds +F to the
                          * body of geom2 and -F to the body of geom1.  A body without contact force reads exact zeros.  smplsim_reset
                          * zeroes the rows of the envs it resets (its mj_forward runs no constraint solve) and leaves the others.
                          * [MJ-upstream] mj_contactForce summed per body; MuJoCo's cfrc_ext holds the same wrench (without
                          * xfrc_applied) in com-based form about the root subtree COM, rotation first -- not checked against a wheel. */
} SmplsimAux;

/* A camera of smplsim_render.  Camera frame as in MJCF: the camera looks along its -z axis, +y is up, +x is right. */
#define SMPLSIM_CAM_FIXED 0    /* world pose */
#define SMPLSIM_CAM_TRACKCOM 1 /* world axes; position = the env's robot centre of mass + pos (MJCF mode="trackcom") */
#define SMPLSIM_CAM_BODY 2     /* rides on robot body `body` */
typedef struct SmplsimCamera {
  int32_t mode, body, exclude_body, pad_;  /* body: BODY mode; exclude_body: -1 = none, else that body's geoms are not drawn */
  float pos[3];   /* FIXED: world position | TRACKCOM: offset from the robot COM | BODY: position in the body frame */
  float mat[9];   /* row-major; columns = camera x, y, z axes in the world (FIXED, TRACKCOM) or body (BODY) frame */
  float fovy;     /* vertical field of view, degrees, in (0, 180) */
  float zfar;     /* depth of pixels that hit nothing */
} SmplsimCamera;

typedef struct SmplsimHandle SmplsimHandle;

const char* smplsim_last_error(void);
int smplsim_version(void);   /* 300 = this header (290: before smplsim_track_eval; 280: before smplsim_motion_blend and the interpolation / future-target fields; 270: before smplsim_amp_obs / smplsim_amp_demo; 260: before smplsim_imitation; 250: before smplsim_set_env_params; 240: before smplsim_ray / smplsim_render; 230: before smplsim_dynamics; 220: before smplsim_inverse;
                              * 210: before SmplsimAux.contact_wrench; 200: before SmplsimState.xfrc_applied; 100: before pid_* state and aux.status) */

/* MjModel.from_xml_string + MjData + setup_humanoid_properties/setup_controller
 * (base_env.py:139-142, humanoid_env.py:262-323). */
int smplsim_create(const SmplsimModelDesc* model, const SmplsimEnvCfg* cfg, int num_envs, int cuda_device,
                   SmplsimHandle** out);
/* Per-env body shapes: what one SMPL_Robot per env process gives the reference (humanoid_env.py:219-250: each HumanoidEnv builds
 * its own MJCF from its betas / gender, smpllib/smpl_local_robot.py:1280-1505) in ONE batch.  Env e is simulated with
 * models[env_model[e]].  All models must share tree, joints and geom layout (offsets, geom sizes, masses, inertias, gains and
 * joint ranges may differ); envs of one shape are grouped into whole thread blocks internally, env indexing of every array is
 * unchanged.  num_models == 1 (env_model may be NULL) is smplsim_create. */
int smplsim_create_shapes(const SmplsimModelDesc* models, int num_models, const int32_t* env_model, const SmplsimEnvCfg* cfg,
                          int num_envs, int cuda_device, SmplsimHandle** out);
int smplsim_num_shapes(const SmplsimHandle* h);
int smplsim_destroy(SmplsimHandle* h);
int smplsim_obs_dim(const SmplsimHandle* h);
int smplsim_num_envs(const SmplsimHandle* h);

/* HumanoidTask.reset -> HumanoidEnv.reset -> BaseEnv.reset (humanoid_task.py:6-9,
 * humanoid_env.py:471-512, base_env.py:64-84) for the envs whose mask byte is non-zero
 * (mask_dev == NULL: all).  init_mode < 0 uses cfg.state_init.  qpos0/qvel0 are read for
 * SMPLSIM_INIT_MOCAP.  obs_dev (may be NULL) receives the reset observation of the reset envs. */
int smplsim_reset(SmplsimHandle* h, const SmplsimState* st, const uint8_t* mask_dev, int init_mode,
                  const float* qpos0_dev, const float* qvel0_dev, float* obs_dev, const SmplsimAux* aux,
                  void* cuda_stream);

/* BaseEnv.step = pre_physics_step + physics_step (nsubsteps x [compute_torque + mj_step]) +
 * post_physics_step (base_env.py:86-100, humanoid_env.py:439-469, tasks/ *.py). */
int smplsim_step(SmplsimHandle* h, const SmplsimState* st, const float* action_dev, float* obs_dev,
                 float* reward_dev, uint8_t* terminated_dev, uint8_t* truncated_dev, const SmplsimAux* aux,
                 void* cuda_stream);

/* mj_data.ctrl[:] = ctrl; mujoco.mj_step(model, data)  x nsub  (humanoid_env.py:448-450). */
int smplsim_mj_step(SmplsimHandle* h, const SmplsimState* st, const float* ctrl_dev, int nsub,
                    const SmplsimAux* aux, void* cuda_stream);

/* mujoco.mj_kinematics (humanoid_env.py:389) / poselib SkeletonState.global_transformation
 * (poselib/skeleton/skeleton3d.py:389-408): qpos[N,nq] -> xpos[N,nbody,3], xquat[N,nbody,4]. */
int smplsim_kinematics(SmplsimHandle* h, const float* qpos_dev, float* xpos_dev, float* xquat_dev, int n,
                       void* cuda_stream);

/* mujoco.mj_inverse on n caller rows: qpos[n,nq], qvel[n,nv], qacc[n,nv] -> qfrc_inverse[n,nv];
 * contact_wrench[n,nbody,6] or NULL (same layout / convention as SmplsimAux.contact_wrench).
 * qfrc_inverse = M(qpos) qacc + qfrc_bias(qpos, qvel) - J^T f, f_r = -D_r min(0, J_r qacc - aref_r) over the floor-contact pyramid rows
 * and joint-limit rows that mj_forward at (qpos, qvel) builds; M includes the armature.  Conventions of qfrc_bias / qvel: root dofs
 * [0:3] world-frame force, [3:6] torque about the root body's axes.  If qacc is what the forward pass produced from ctrl (and
 * xfrc_applied), qfrc_inverse = [0_6 ; ctrl] + J_b^T xfrc.  The inverse takes no xfrc_applied, never auto-resets and writes no
 * per-env state (a later smplsim_step is unaffected); a row with non-finite inputs gets unspecified values in that row only.
 * Joint-limit rows past the kernels' cap are dropped, as in smplsim_step.  Single-shape handle: any n >= 0 (launched in pieces of at
 * most num_envs rows on the stream).  Per-env shapes: n == num_envs, row i uses env i's shape.  A handle with self_collision = 1:
 * SMPLSIM_EUNSUPPORTED (no geom-geom rows in the inverse).
 * [MJ-upstream] mj_inverse with mjENBL_INVDISCRETE off (engine_inverse.c); not checked against a MuJoCo wheel. */
int smplsim_inverse(SmplsimHandle* h, const float* qpos_dev, const float* qvel_dev, const float* qacc_dev,
                    float* qfrc_inverse_dev, float* contact_wrench_dev, int n, void* cuda_stream);

/* Mass matrix, bias forces and body Jacobians on n caller rows qpos[n,nq], qvel[n,nv] (each output NULL: skipped):
 *   qM[n,nv,nv]          mujoco.mj_fullM(qM): the dense joint-space inertia, armature on the diagonal; exactly symmetric, exact zeros
 *                        where neither dof is an ancestor of the other;
 *   qfrc_bias[n,nv]      mj_rne at qacc = 0: Coriolis, centrifugal and gravity (no constraint rows, no armature term); qvel_dev may be
 *                        NULL only when qfrc_bias_dev is NULL (qvel is then zero);
 *   jac[n,njac,6,nv]     mujoco.mj_jacBody at each listed body's frame origin (xpos): rows 0-2 jacp (world-frame linear velocity of the
 *                        point), rows 3-5 jacr (world-frame angular velocity); columns of dofs off the body's root path are 0.
 * jac_body: host array of njac robot body indices (0 = root, repeats allowed, njac <= nbody).  Conventions of qvel / qfrc_bias: root
 * dofs [0:3] world-frame translation / force, [3:6] rotation about / torque along the root body's axes c_k; a root rotation's jacp
 * column is c_k x (p - root), a hinge's axis x (p - anchor).  Nothing here depends on contacts, so every handle kind is supported; no
 * per-env state is read or written (a later smplsim_step is unaffected).  Single-shape handle: any n >= 0 (launched in pieces of at
 * most num_envs rows on the stream).  Per-env shapes: n == num_envs, row i uses env i's shape.  SMPLSIM_EINVAL: a bad body index,
 * njac > 0 with jac_dev NULL, qfrc_bias without qvel, or every output NULL with n > 0.
 * [MJ-upstream] mj_fullM / mj_rne / mj_jacBody (engine_support.c, engine_core_smooth.c); not checked against a MuJoCo wheel. */
int smplsim_dynamics(SmplsimHandle* h, const float* qpos_dev, const float* qvel_dev, int n, float* qM_dev, float* qfrc_bias_dev,
                     const int32_t* jac_body, int njac, float* jac_dev, void* cuda_stream);

/* Ray casting and camera images of the robot geoms and the floor, on caller body poses xpos[n,nbody,3] / xquat[n,nbody,4] (the
 * layout of SmplsimAux.xpos / xquat: the post-step poses a batch holds, smplsim_kinematics of any qpos, or motion-table rows).
 * Quaternions are normalised in the kernel.  Geometry: spheres, capsules, boxes and the infinite floor plane in closed form, fp32;
 * the smallest x >= 0 wins, so a ray that starts inside a geom hits it on the way out, and the floor is hit from its front side only;
 * geom margins are ignored [MJ-upstream: mj_ray, engine_ray.c].  Neither call writes env state or handle scratch a later step reads.
 * Single-shape handle: any n >= 0.  Per-env shapes: n == num_envs, row i uses env i's shape.  Every handle kind is supported.
 *
 * smplsim_ray (mujoco.mj_ray for every ray): pnt[n,nray,3], vec[n,nray,3] -> dist[n,nray] = x with the hit at pnt + x vec (vec need
 * not be unit), geomid[n,nray] = MuJoCo geom id (0 floor, i + 1 robot geom i); -1 / -1: no hit (also for vec = 0).  flg_static = 0
 * skips the floor; bodyexclude (-1 = none) skips every geom of that robot body.  Each output may be NULL.
 *
 * smplsim_render: one image per env from *cam (host struct).  Row 0 is the top of the image, pixel (r, c) is shot through its centre;
 * fovy is vertical, the horizontal field follows from width / height.  Outputs, each NULL = skipped:
 *   depth[n,height,width] float32  z-depth along the camera's viewing axis (metres, not ray length); cam->zfar where nothing is hit
 *   seg[n,height,width]   int32    MuJoCo geom id (0 floor, i + 1 robot geom i), -1 none
 *   rgb[n,height,width,3] uint8    c = clamp(a (0.1 + 0.4 max(0, -n.f) + max(0, -n.l) s), 0, 1), u8 = floor(255 c + 0.5): n the unit
 *                                  normal facing the ray, f the camera's forward axis, l = (0, 0, -1), s = 0 when the ray from
 *                                  p + 1e-4 n towards -l hits a robot geom; albedo a = geom_rgb (host [ngeom*3], NULL: 0.8 0.6 0.4)
 *                                  for robot geoms, a 0 / 0.8 grey checker of edge 5/3 m on the floor; no hit: t (0.4, 0.5, 0.6),
 *                                  t = (d_z + 1) / 2 of the unit ray direction.  Details: csrc/render_kernels.cuh.
 * SMPLSIM_EINVAL: a bad body index (cam->body, cam->exclude_body, bodyexclude), an unknown cam->mode, fovy outside (0, 180),
 * width / height / nray <= 0 with n > 0, or every output NULL with n > 0. */
int smplsim_ray(SmplsimHandle* h, const float* xpos_dev, const float* xquat_dev, int n, int nray, const float* pnt_dev,
                const float* vec_dev, int flg_static, int bodyexclude, float* dist_dev, int32_t* geomid_dev, void* cuda_stream);
int smplsim_render(SmplsimHandle* h, const float* xpos_dev, const float* xquat_dev, int n, const SmplsimCamera* cam,
                   int width, int height, const float* geom_rgb, float* depth_dev, int32_t* seg_dev, uint8_t* rgb_dev,
                   void* cuda_stream);

/* Per-env physics parameters (domain randomization).  Env e is simulated exactly as the handle's model (env e's shape on a per-env-shapes
 * handle) with these fields replaced -- MuJoCo's behaviour when MjModel fields are edited in place without mj_setConst:
 *   friction[N]            sliding friction mu (friction[0]) of every floor and geom-geom contact: pyramid directions n +- mu t and the
 *                          rows' R / D (the impratio scaling);
 *   gravity[N,3]           opt.gravity;
 *   kp, kd, torque_limit [N,nu]   act_kp / act_kd / act_torque_lim, the values the configured controller reads (stable PD: torque and
 *                          the (M + h kd) system, quirk Q1 with the env's own kd and masses on both sides; pd; simple_pid: gains and the
 *                          clamp of the torque and of the integral; torque: the clamp only, act_scale stays the model's);
 *   body_mass_scale[N,nbody]      body b's mass AND rotational inertia times s_b; its centre of mass does not move.
 * body_invweight0 / dof_invweight0, and with them the constraint regularisation, keep the nominal model's values (mj_setConst is
 * not rerun).  Every field is a device pointer to a full [N, ...] float32 array, or NULL. */
typedef struct SmplsimEnvParams {
  const float* friction;
  const float* gravity;
  const float* kp;
  const float* kd;
  const float* torque_limit;
  const float* body_mass_scale;
} SmplsimEnvParams;
/* smplsim_set_env_params: for the envs whose mask byte is non-zero (mask_dev NULL: all), each non-NULL field of *p overwrites that
 * parameter in the handle's per-env records; a NULL field keeps the current value.  The first call allocates the records (one per env,
 * [mu | g 3 | kp nu | kd nu | torque_limit nu | mass_scale nbody] padded to 16 bytes: 944 B for SMPL) and fills them with the model's
 * values, in stream order on cuda_stream; launches on other streams must be ordered after it by the caller.  Every call runs
 * asynchronously on the stream.  Nothing the caller passes is kept
 * after the call returns; the values are not checked (finite, mu >= 1e-5, gains >= 0, limits and scales > 0 is the caller's part).
 * While records exist, smplsim_step, smplsim_mj_step, smplsim_reset (its Fall init runs substeps), smplsim_inverse, smplsim_dynamics
 * and smplsim_render (TRACKCOM) use them; inverse and dynamics then need n == num_envs (row i uses env i's parameters), else
 * SMPLSIM_EINVAL.  kinematics, ray, self_obs, motion_gather and gae do not depend on them.  Without records every call runs exactly
 * as before (the same kernels).
 * smplsim_get_env_params: copies the current values into the non-NULL fields of *out ([N, ...] device arrays), the model's values
 * when no records exist.  smplsim_clear_env_params: synchronizes with the device and frees the records; the handle is again exactly
 * what it was before the first set. */
int smplsim_set_env_params(SmplsimHandle* h, const SmplsimEnvParams* p, const uint8_t* mask_dev, void* cuda_stream);
int smplsim_get_env_params(SmplsimHandle* h, float* friction_dev, float* gravity_dev, float* kp_dev, float* kd_dev,
                           float* torque_limit_dev, float* body_mass_scale_dev, void* cuda_stream);
int smplsim_clear_env_params(SmplsimHandle* h);

/* compute_humanoid_self_obs_v1 / _v2 (humanoid_env.py:565-688) on caller-supplied body states:
 * qvel[N,nv] (v1), xpos, xquat, linvel, angvel [N,nbody,*] -> obs[N,self_obs_dim]. */
int smplsim_self_obs(SmplsimHandle* h, int version, const float* qvel_dev, const float* xpos_dev,
                     const float* xquat_dev, const float* linvel_dev, const float* angvel_dev, float* obs_dev,
                     int n, void* cuda_stream);

/* MotionLibBase.get_motion_state_intervaled (smpllib/motion_lib_base.py:313-354,448-458):
 * frame = floor(clip(t,0,len)/dt) + length_starts[id]; gathers row `frame` of each table.
 * tables[k] is [total_frames, widths[k]] float32, outs[k] is [n, widths[k]]. */
int smplsim_motion_gather(SmplsimHandle* h, const int32_t* motion_ids_dev, const float* motion_times_dev, int n,
                          const float* motion_len_dev, const int32_t* num_frames_dev, const float* motion_dt_dev,
                          const int32_t* length_starts_dev, int num_tables, const float* const* tables_dev,
                          const int32_t* widths, float* const* outs_dev, int32_t* frame_idx_dev, void* cuda_stream);

/* MotionLibBaseTorch.get_motion_state (smpl_sim/smpllib/motion_lib_base_torch.py:434-499): the state of clip id at time t blended
 * from the two frames around t, for n query rows.  Arguments as smplsim_motion_gather, plus kinds[k] (host, one SMPLSIM_BLEND_* per
 * table), offset_dev[n,3] (or NULL) and the optional outputs frame0_dev / frame1_dev[n] (table rows, length_starts included) and
 * blend_dev[n].  Frame rule (_calc_frame_blend, :528-538), every operation one float32 rounding as torch on the CPU:
 *     phase = clip(t / len, 0, 1);  t = max(t, 0)
 *     f0 = (int)(phase * (nf - 1));  f1 = min(f0 + 1, nf - 1);  b = clip((t - f0 dt) / dt, 0, 1)
 * Value kinds, v0 / v1 = the rows f0 / f1 of a table:
 *     LERP   (1 - b) v0 + b v1                                        (dof_pos, dof_vel, body_vel, body_ang_vel)
 *     POS    LERP, then + offset[i] on every 3-group                    (rg_pos)
 *     SLERP  every 4-group slerped (width a multiple of 4)              (rb_rot)
 *     QPOS   LERP, columns 3-6 slerped, + offset[i] on columns 0-2      (qpos: this project's extension, the reference returns none)
 *     ROW0   row f0 as it is                                            (motion_aa)
 * slerp is torch_utils.slerp (smpl_sim/utils/torch_utils.py:405-426) with its quirks: q1 negated when q0.q1 < 0; the midpoint
 * 0.5 q0 + 0.5 q1 when |sin(half angle)| < 0.001, whatever b; q0 when cos(half angle) >= 1; the result is not normalised.  Blended qvel
 * rows (LERP of the qvel table) are, like QPOS, this project's extension.  Quaternions are wxyz; the formula does not depend on the order.
 * SMPLSIM_EINVAL: a null argument, more than 16 tables, an unknown kind, SLERP on a width that is not a multiple of 4, POS on one that is
 * not a multiple of 3, QPOS on one below 7. */
#define SMPLSIM_BLEND_LERP 0
#define SMPLSIM_BLEND_POS 1
#define SMPLSIM_BLEND_SLERP 2
#define SMPLSIM_BLEND_QPOS 3
#define SMPLSIM_BLEND_ROW0 4
int smplsim_motion_blend(SmplsimHandle* h, const int32_t* motion_ids_dev, const float* motion_times_dev, int n,
                         const float* motion_len_dev, const int32_t* num_frames_dev, const float* motion_dt_dev,
                         const int32_t* length_starts_dev, int num_tables, const float* const* tables_dev,
                         const int32_t* widths, const int32_t* kinds, const float* offset_dev, float* const* outs_dev,
                         int32_t* frame0_dev, int32_t* frame1_dev, float* blend_dev, void* cuda_stream);

/* Motion-imitation task: every env tracks one clip of a motion library.  One launch, run after smplsim_step / smplsim_reset on the same
 * stream, writes the env's observation row, reward, flags and position error; the stepper itself runs as SMPLSIM_TASK_NONE.  The
 * reference ships no imitation task in its MuJoCo env layer (SURVEY.md 3.4), so the definitions are this project's, after the published
 * PHC formulation.
 *
 * Per env e: clip id m = motion_ids[e] (clamped to [0, num_motions)), clip start time t0 = motion_t0[e], step counter p = progress[e]
 * (SmplsimState.progress, already incremented by the step), control period dt = (float)(model.timestep * nsubsteps), the product taken
 * in double precision.  ref(t) is the row of the tables picked by the frame rule of smplsim_motion_gather (phase clip, float idx0,
 * blend, int() truncation, quirk Q12) for clip m at time t; times are t0 + k dt evaluated in float32 as ONE fused multiply-add.
 * Simulated body state: p_b, q_b = aux.xpos / xquat (post-integration), v_b, w_b = aux.body_linvel / body_angvel (the values obs v2
 * uses, quirk Q2); ^ marks the reference.  h = the heading-inverse quaternion of the simulated root (the one the self observation
 * uses: with has_upright_start = 0 the root is first multiplied by (0.5, -0.5, -0.5, -0.5); heading = atan2 of the rotated x axis;
 * h = rotation by -heading about z).  h * v rotates the vector v; (x) is the quaternion product; q^-1 is the conjugate (the tables and
 * the stepper hold unit quaternions); six(q) = [q * (1,0,0), q * (0,0,1)].  B = cfg.tracked_bodies (J = num_tracked entries; NULL:
 * all nbody bodies in order, num_tracked must then be nbody).
 *
 * Observation, target = ref(t0 + (p + 1) dt), the pose to reach by the next step.  obs row = [self obs, self_obs_dim words copied from
 * self_obs_dev | 24 J words], the 24 J words grouped by kind, bodies in the order of B:
 *     3J  h * (p^_b - p_b)
 *     6J  six(h (x) q^_b (x) q_b^-1 (x) h^-1)
 *     3J  h * (v^_b - v_b)
 *     3J  h * (w^_b - w_b)
 *     3J  h * (p^_b - p_root)            p_root = the simulated root position
 *     6J  six(h (x) q^_b)
 * Reward, compared with ref(t0 + p dt), the pose that should have been reached now:
 *     r = w_pos exp(-k_pos mean_B |p^_b - p_b|^2) + w_rot exp(-k_rot mean_B th_b^2) + w_vel exp(-k_vel mean_B |v^_b - v_b|^2)
 *       + w_angvel exp(-k_angvel mean_B |w^_b - w_b|^2),   th_b = 2 atan2(|xyz|, |w|) of q^_b (x) q_b^-1, in [0, pi].
 * Flags, same reference row:
 *     terminated = (p > 1 and max_B |p^_b - p_b| > termination_distance) or aux.status has bit 1, 2 or 4 (the stepper put the env back
 *                  to qpos0, so it is no longer on its clip; aux.status NULL: not consulted);
 *     truncated  = t0 + (p + 1) dt > motion_len[m] (no next target) or p > episode_length (strict, quirk Q7).
 * mpjpe = mean_B |p^_b - p_b| in metres.  frames (may be NULL) receives the two table rows used, [N,2] = (now, next).
 * The means and the maximum are reduced in a fixed order: the outputs are bit-reproducible.
 *
 * Options (appended fields; their zero values give the task above):
 *   interpolate = 1: ref(t) is the state smplsim_motion_blend gives for (m, t) instead of one row: positions and velocities lerped,
 *     rotations slerped between the frames f0 and f1 of its frame rule.  The slerped q^_b are not renormalised (the reference's
 *     slerp); q * v is evaluated as v (2 w^2 - 1) + 2 w (u x v) + 2 u (u . v) with u = xyz(q), which is the rotation for unit q.  The observation's targets, the reward, mpjpe and the
 *     termination distance all use it; frames then reports the rows f0 of now and next.  Truncation is unchanged.
 *   num_future = T >= 2: T targets, target k = 0..T-1 at fmaf(k, future_dt, t0 + (p + 1) dt); the row is [self obs | T x 24 J], frame
 *     major, each block the 24 J words above against the current simulated state.  T = 0 or 1: one target.  The row is then
 *     self_obs_dim + 24 J T wide (smplsim_imitation_obs_dim gives the one-target width). */
typedef struct SmplsimImitationCfg {
  float k_pos, k_rot, k_vel, k_angvel;   /* defaults of the `im` cfg group: 100, 10, 0.1, 0.1 */
  float w_pos, w_rot, w_vel, w_angvel;   /*                                 0.5, 0.3, 0.1, 0.1 */
  float termination_distance;            /* metres (0.25) */
  int32_t episode_length;
  int32_t self_obs_dim;                  /* must be the handle's self-observation width (the head of a smplsim_step observation row) */
  int32_t num_tracked;                   /* J, in [1, nbody] */
  const int32_t* tracked_bodies;         /* host array [num_tracked] of robot body indices (0 = root), or NULL */
  int32_t interpolate;                   /* 0: the nearest-frame rows; 1: blended reference states (see above) */
  int32_t num_future;                    /* T >= 0 targets per observation (0 and 1: one) */
  float future_dt;                       /* >= 0 seconds between targets (PHC: 1 / trajSampleTimestepInv) */
} SmplsimImitationCfg;
/* Device tables of a motion library (the layout smplsim_motion_gather takes), read in place. */
typedef struct SmplsimMotionTables {
  const float* xpos;          /* [total_frames, nbody*3] */
  const float* xquat;         /* [total_frames, nbody*4] */
  const float* body_vel;      /* [total_frames, nbody*3] */
  const float* body_ang_vel;  /* [total_frames, nbody*3] */
  const float* motion_len;    /* [num_motions] seconds */
  const int32_t* num_frames;  /* [num_motions] */
  const float* motion_dt;     /* [num_motions] frame period */
  const int32_t* length_starts; /* [num_motions] first row of the clip */
  int32_t num_motions;
  int32_t nbody;              /* bodies per table row; must be the handle's */
} SmplsimMotionTables;
/* Width of the observation row smplsim_imitation writes for num_tracked bodies and one target: self-observation width + 24 num_tracked
 * (T targets: self-observation width + 24 num_tracked T). */
int smplsim_imitation_obs_dim(const SmplsimHandle* h, int num_tracked);
/* For the envs whose mask byte is non-zero (mask_dev NULL: all): obs_dev[N, smplsim_imitation_obs_dim] and frames_dev; unless obs_only
 * (the call after a reset) also reward_dev[N], terminated_dev[N], truncated_dev[N], mpjpe_dev[N].  obs_only != 0 leaves those four
 * untouched (they may be NULL).  self_obs_dev: the observation rows smplsim_step / smplsim_reset wrote, row stride = smplsim_obs_dim(h).
 * aux: xpos, xquat, body_linvel, body_angvel are read (required), status if non-NULL.  Works on every handle kind (SMPL, SMPL-X,
 * per-env shapes, self-collision); reads no handle scratch and writes no env state, so the stepper's results do not depend on it.
 * SMPLSIM_EINVAL: a null argument, num_tracked outside [1, nbody], a tracked body outside [0, nbody), tracked_bodies NULL with
 * num_tracked != nbody, tab->nbody != the handle's, num_motions < 1, self_obs_dim != the handle's, interpolate not 0 / 1, num_future < 0,
 * future_dt < 0 or NaN. */
int smplsim_imitation(SmplsimHandle* h, const SmplsimImitationCfg* cfg, const SmplsimMotionTables* tab, const int32_t* motion_ids_dev,
                      const float* motion_t0_dev, const int32_t* progress_dev, const SmplsimAux* aux, const float* self_obs_dev,
                      const uint8_t* mask_dev, int obs_only, float* obs_dev, float* reward_dev, uint8_t* terminated_dev,
                      uint8_t* truncated_dev, float* mpjpe_dev, int32_t* frames_dev, void* cuda_stream);

/* Tracking evaluation: the per-frame metrics of the reference's smpl_eval (smpl_sim/smpllib/smpl_eval.py: compute_metrics_lite,
 * compute_metrics_obj, p_mpjpe, compute_error_vel, compute_error_accel) for every env that tracks a clip, accumulated per env in one
 * launch after each step's smplsim_imitation.  The reference scores recorded trajectories after the fact; here nothing but a [2, J, 3]
 * difference history per env is kept.
 *
 * Eval bodies B = cfg->bodies (J = num_bodies >= 3 entries, NULL: all nbody bodies in order).  The root is the first eval body, B[0]
 * (the reference's root_idx = 0); with a list that does not start at body 0, "root-relative" means relative to body B[0].
 * Scored frame: the pair (the post-step state after step p, ref(t0 + p dt)) for p = progress[e], where ref is the reference pose
 * smplsim_imitation's reward compares -- the same frame rule, nearest row or (interpolate = 1) the blended state -- and dt =
 * cfg->dt, or the handle's control period (smplsim_imitation's) when cfg->dt = 0.  A caller runs it after every step from p = 1 on:
 * the reset state (p = 0) is not scored.  Simulated poses: y_b = aux.xpos, q_b = aux.xquat; reference: x_b, q^_b.  Per scored frame,
 * the f-th since the env's state was cleared (f = 0, 1, ...), with d_j = y_j - x_j and means over j in B:
 *     mpjpe_g     mean |d_j|                                                           mm (x 1000, as the reference)
 *     mpjpe_l     mean |(y_j - y_root) - (x_j - x_root)|                               mm
 *     mpjpe_pa    p_mpjpe of the root-relative points: with x0 / y0 the points centred on their means, the proper rotation Q and scale
 *                 s = lam / sum |y0|^2 maximising lam = sum x0 . Q y0 (the reference's sign_detR correction: never a reflection),
 *                 mean |s Q y0_j - x0_j|; s = 0 when every y0 is zero (the reference divides by zero)   mm
 *     vel_dist    mean |d_j^f - d_j^(f-1)|, f >= 1 only (compute_error_vel)            mm per frame
 *     accel_dist  mean |d_j^f - 2 d_j^(f-1) + d_j^(f-2)|, f >= 2 only (compute_error_accel; not divided by dt)   mm per frame^2
 *     rot_error   mean of th_j = 2 atan2(|xyz|, |w|) of q^_j (x) q_j^-1 (the rotvec norm of compute_metrics_obj; that function takes
 *                 xyzw quaternions, these are wxyz)                                     rad
 * Per env e with active[e] != 0 (the others are not read or written, frame_metrics rows included):
 *     frame_metrics[e] (if non-NULL) = this frame's six values in the order above, NaN where undefined (vel f = 0, accel f <= 1);
 *     sums[e, i] += value i (fp64) when defined; frames[e] = f + 1; prev_diff[e, f % 2] = d^f (slot f % 2 held d^(f-2));
 *     if terminated[e] or truncated[e] (this step's flags, e.g. smplsim_imitation's): scoring ends with this frame, which is scored:
 *     active[e] = 0, success[e] = truncated[e] && !terminated[e] (both set: failed).
 * A clip's value of metric i is sums[e, i] / count_i with counts frames, frames, frames, frames - 1, frames - 2, frames; over a set of
 * clips the frame-weighted mean (sum of sums / sum of counts) is compute_metrics_lite(..., concatenate=True)[k].mean().
 * To start an env, the caller sets active = 1 and zeroes frames, sums and success (prev_diff needs no clearing).  Sums are lane partials in
 * body-list order and an xor butterfly: the outputs are bit-reproducible.  Works on every handle kind; reads and writes no stepper state.
 * SMPLSIM_EINVAL: a null argument or state array (frame_metrics may be NULL), num_bodies outside [3, nbody], an eval body outside
 * [0, nbody), bodies NULL with num_bodies != nbody, tab->nbody != the handle's, num_motions < 1, interpolate not 0 / 1, dt < 0 or NaN. */
#define SMPLSIM_TRACK_NMETRIC 6
#define SMPLSIM_TRACK_MPJPE_G 0
#define SMPLSIM_TRACK_MPJPE_L 1
#define SMPLSIM_TRACK_MPJPE_PA 2
#define SMPLSIM_TRACK_VEL_DIST 3
#define SMPLSIM_TRACK_ACCEL_DIST 4
#define SMPLSIM_TRACK_ROT_ERROR 5
typedef struct SmplsimTrackEvalCfg {
  int32_t num_bodies;            /* J in [3, nbody] (the Procrustes fit needs three points) */
  const int32_t* bodies;         /* host array [num_bodies] of robot body indices (0 = root), or NULL */
  int32_t interpolate;           /* 0: nearest-frame rows; 1: blended reference states (SmplsimImitationCfg.interpolate) */
  float dt;                      /* seconds per step of the frame rule; 0: the handle's control period */
} SmplsimTrackEvalCfg;
typedef struct SmplsimTrackEvalState {
  uint8_t* active;               /* [N]  1: scored this call */
  float* prev_diff;              /* [N, 2, J, 3]  d of the last two scored frames */
  int32_t* frames;               /* [N]  frames scored */
  double* sums;                  /* [N, 6]  per-metric sums over the frames that define them */
  uint8_t* success;              /* [N]  set when scoring ends by truncation alone */
  float* frame_metrics;          /* [N, 6] or NULL: this call's values */
} SmplsimTrackEvalState;
int smplsim_track_eval(SmplsimHandle* h, const SmplsimTrackEvalCfg* cfg, const SmplsimMotionTables* tab, const int32_t* motion_ids_dev,
                       const float* motion_t0_dev, const int32_t* progress_dev, const SmplsimAux* aux, const uint8_t* terminated_dev,
                       const uint8_t* truncated_dev, const SmplsimTrackEvalState* state, void* cuda_stream);

/* Adversarial motion priors (AMP): the discriminator's observation of an env's last K control steps and of a motion library's clips.
 * The per-frame feature is the reference's compute_humanoid_observations_smpl with has_smpl_params = False (smpl_sim/envs/nv/humanoid.py:
 * 2530-2602, dof_to_obs :2276-2309, remove_base_rot :2523-2527); quaternions here are wxyz, the reference's xyzw.  One frame, F floats:
 *     root_h                              root_pos.z, only if root_height_obs (the column is dropped, not zeroed, as in the _smpl variant)
 *     r = root_rot, and r = r (x) conj(0.5, 0.5, 0.5, 0.5) unless upright_start (remove_base_rot; the rule of the heading below)
 *     h = the heading-inverse of r (rotation by -atan2 of r's rotated x axis about z; the h of smplsim_imitation)
 *     tan_norm(local_root_obs ? h (x) r : r)     6   tan_norm(q) = [q * (1,0,0), q * (0,0,1)]
 *     h * root_vel, h * root_ang_vel             3 + 3 (world-frame velocities)
 *     dof_obs                             6 (nbody - 1): per non-root body b, its 3 hinge angles e = dof_pos[3(b-1) : 3b] as an exp map:
 *                                         a = |e| wrapped by atan2(sin a, cos a); |a| <= 1e-5 -> the identity, else the rotation by a about
 *                                         e / |e|; then tan_norm
 *     dof_vel                             nv - 6
 *     h * (key_pos_k - root_pos)          3 per key body, in the order of cfg.key_bodies
 * F = 232 for SMPL (24 bodies, 4 key bodies, root height), 484 for SMPL-X.  A model whose non-root bodies do not all have exactly 3
 * hinges: SMPLSIM_EUNSUPPORTED (the reference asserts on them).
 * Sources:
 *   simulated env e, the post-step state: root_pos, key_pos = aux.xpos, root_rot = aux.xquat[e, 0], root_vel = qvel[0:3], root_ang_vel =
 *     root_rot * qvel[3:6] (MuJoCo's body-frame angular velocity rotated to world), dof_pos = qpos[7:], dof_vel = qvel[6:] -- all from the
 *     same post-integration state, which is what Isaac's rigid-body / dof tensors hold after simulate.  (smplsim_imitation and obs v2
 *     read the pre-integration body velocities instead, quirk Q2.)
 *   motion library, clip m at time t: ref(t) = the row of the xpos, xquat, body_vel[0], body_ang_vel[0], dof_pos, dof_vel tables that the
 *     frame rule of smplsim_motion_gather picks (nearest frame, no slerp, quirk Q12); the clip id is clamped to [0, num_motions).
 * AMP observation: K = num_steps frames newest first, amp_obs[N, K, F], frame k = control step p - k.  dt = (float)(model.timestep *
 * nsubsteps).  Times t - k dt and t0 + (p - k) dt are one float32 fused multiply-add, as in smplsim_imitation.
 * Nothing is reduced and nothing is atomic: the outputs are bit-reproducible.  Neither call writes env state or handle scratch; every
 * handle kind (SMPL, SMPL-X, per-env shapes, self-collision) is supported. */
#define SMPLSIM_AMP_PUSH 0     /* frames 0..K-2 move to 1..K-1 in place, the current simulated frame goes to 0 (after every env step) */
#define SMPLSIM_AMP_FILL 1     /* the current simulated frame in all K slots (Default / Fall resets) */
#define SMPLSIM_AMP_FILL_REF 2 /* the current simulated frame at 0, ref(t0 + (p - k) dt) of the env's clip in slot k >= 1 (MoCap resets) */
typedef struct SmplsimAmpCfg {
  int32_t num_steps;             /* K >= 1 (numAMPObsSteps: 10) */
  int32_t num_key_bodies;        /* in [0, nbody] */
  const int32_t* key_bodies;     /* host array [num_key_bodies] of robot body indices (0 = root); may be NULL when num_key_bodies = 0 */
  int32_t local_root_obs;        /* 0/1 */
  int32_t root_height_obs;       /* 0/1 */
  int32_t interpolate;           /* 0: ref(t) as above; 1: the blended state of smplsim_motion_blend (frames f0 / f1 of its rule: root_rot
                                  * slerped, root_pos, key_pos, velocities and the dof_pos exp-map triples lerped), in FILL_REF and demo rows */
} SmplsimAmpCfg;
/* The tables of ref(t): a motion library (SmplsimMotionTables, read in place) plus its joint tables. */
typedef struct SmplsimAmpTables {
  const SmplsimMotionTables* motion;
  const float* dof_pos;          /* [total_frames, nv - 6] */
  const float* dof_vel;          /* [total_frames, nv - 6] */
} SmplsimAmpTables;
/* F of cfg on this handle (negative SMPLSIM_E* for a bad cfg). */
int smplsim_amp_obs_dim(const SmplsimHandle* h, const SmplsimAmpCfg* cfg);
/* The envs whose mask byte is non-zero (mask_dev NULL: all) get their amp_obs_dev[N, K, F] row updated by mode; the others are not
 * written.  st: qpos, qvel (and progress for FILL_REF) are read; aux: xpos, xquat.  FILL_REF also reads tab, motion_ids_dev[N] and
 * motion_t0_dev[N] (the clip and the clip time of step 0, as smplsim_imitation); the other modes ignore them (they may be NULL).
 * SMPLSIM_EINVAL: a null required pointer, num_steps < 1, a bad key body, tab->motion->nbody != the handle's, num_motions < 1, an
 * unknown mode, interpolate not 0 / 1. */
int smplsim_amp_obs(SmplsimHandle* h, const SmplsimAmpCfg* cfg, const SmplsimState* st, const SmplsimAux* aux, const SmplsimAmpTables* tab,
                    const int32_t* motion_ids_dev, const float* motion_t0_dev, const uint8_t* mask_dev, int mode, float* amp_obs_dev,
                    void* cuda_stream);
/* Demonstration rows: out[i, k] = ref(motion_times[i] - k dt) of clip motion_ids[i], for n >= 0 caller rows (any n on every handle kind:
 * nothing depends on the env's body shape).  SMPLSIM_EINVAL as smplsim_amp_obs. */
int smplsim_amp_demo(SmplsimHandle* h, const SmplsimAmpCfg* cfg, const SmplsimAmpTables* tab, const int32_t* motion_ids_dev,
                     const float* motion_times_dev, int n, float* out_dev, void* cuda_stream);

/* estimate_advantages (smpl_sim/learning/learning_utils.py:198-218) on a [T,N] device rollout: reverse scan per env,
 * delta = r + gamma*V' *not_dead - V ; A = delta + gamma*tau*A' *not_done ; returns = V + A.  next_value (may be NULL = 0)
 * bootstraps the step after the last one.  Normalisation (mean / unbiased std over the whole, possibly multi-rank, batch) is
 * left to the caller (smplsim_b200.learning.estimate_advantages). */
int smplsim_gae(const float* rewards_dev, const float* not_done_dev, const float* not_dead_dev, const float* values_dev,
                const float* next_value_dev, float gamma, float tau, int T, int N, float* adv_dev, float* ret_dev, void* cuda_stream);

#ifdef __cplusplus
}
#endif
#endif /* SMPLSIM_H_ */
