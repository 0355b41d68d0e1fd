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
} SmplsimAux;

typedef struct SmplsimHandle SmplsimHandle;

const char* smplsim_last_error(void);
int smplsim_version(void);   /* 110 = this header (100: before pid_* state and aux.status) */

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
