"""Every refusal of the C entry points that create a handle and launch the lane, AMP and tracking-evaluation kernels: the return code
and the exact smplsim_last_error() text, which _lib.SmplsimError carries to Python callers.  One row per bad argument, in the order
the entry point checks them; each call is refused before it launches anything."""
import ctypes as C

import numpy as np
import torch

from smplsim_b200.abi import (SmplsimAmpCfgC, SmplsimAmpTablesC, SmplsimAuxC, SmplsimCameraC, SmplsimEnvParamsC, SmplsimMotionTablesC,
                              SmplsimStateC, SmplsimTrackEvalCfgC, SmplsimTrackEvalStateC)
from util_states import make_models

EINVAL, EUNSUPPORTED = -1, -3
CAM_FIXED, CAM_TRACKCOM, CAM_BODY = 0, 1, 2
AMP_FILL_REF = 2


def variant(struct, **kw):
    c = type(struct).from_buffer_copy(struct)
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def i32(*v):
    return np.array(v, dtype=np.int32)


def refusals(backend):
    """(name, call, code, message) rows, and the objects the calls point at (kept alive by the caller)."""
    cfg, _ = make_models(control_mode="torque")
    env = backend.batch(cfg, 4)
    pid = backend.batch(make_models(control_mode="simple_pid")[0], 4)
    scol = backend.batch(make_models(env="getup", control_mode="torque", self_collision=True)[0], 4)
    shp = backend.batch(cfg, 4, models=[env.model, env.model], env_model=[0, 1, 0, 1])
    prm = backend.batch(cfg, 4)
    prm.set_env_params(friction=backend.t(np.full(4, 0.5)))
    L, h, nb = env._L(), env._h, env.model.nbody
    buf = torch.zeros(1 << 20, dtype=torch.float32, device=backend.device)   # every pointer that must be valid points here
    P, s = buf.data_ptr(), env._stream()
    keep = [env, pid, scol, shp, prm, buf]   # handles, device memory and the host arrays / structs the calls point at

    def ref(x):   # NULL for None
        if x is None:
            return None
        keep.append(x)
        return C.c_void_p(x.ctypes.data) if isinstance(x, np.ndarray) else C.byref(x)

    st = SmplsimStateC(*([P] * 12))
    aux = SmplsimAuxC(*([P] * 9))
    ecfg, model = env.envcfg, env._cmodel
    models = (type(model) * 2)(model, model)
    out = C.c_void_p()
    cam = SmplsimCameraC(mode=CAM_FIXED, exclude_body=-1, fovy=45.0, zfar=10.0)
    mt = SmplsimMotionTablesC(*([P] * 8), num_motions=1, nbody=nb)
    te = SmplsimTrackEvalCfgC(num_bodies=nb, interpolate=0, dt=0.0)
    ts = SmplsimTrackEvalStateC(*([P] * 6))
    amp = SmplsimAmpCfgC(num_steps=2, num_key_bodies=2, key_bodies=ref(i32(0, 1)).value, interpolate=0)
    atab = SmplsimAmpTablesC(motion=C.addressof(mt), dof_pos=P, dof_vel=P)

    def create(cfg=ecfg, n=4):
        return L.smplsim_create(C.byref(model), ref(cfg), n, 0, C.byref(out))

    def shapes(em):
        return L.smplsim_create_shapes(C.byref(models), 2, ref(em), C.byref(ecfg), 4, 0, C.byref(out))

    def step(h=h, st=st, a=P):
        return L.smplsim_step(h, ref(st), a, P, P, P, P, C.byref(aux), s)

    def mj_step(h=h, c=P, nsub=1):
        return L.smplsim_mj_step(h, C.byref(st), c, nsub, C.byref(aux), s)

    def reset(h=h, st=st, mode=-1, q0=P):
        return L.smplsim_reset(h, ref(st), None, mode, q0, P, P, C.byref(aux), s)

    def kin(h=h, q=P, n=4):
        return L.smplsim_kinematics(h, q, P, P, n, s)

    def inverse(h=h, qacc=P, n=4):
        return L.smplsim_inverse(h, P, P, qacc, P, None, n, s)

    def dyn(h=h, q=P, v=P, n=4, qM=P, bias=P, jb=None, njac=0, jac=P):
        return L.smplsim_dynamics(h, q, v, n, qM, bias, ref(jb), njac, jac, s)

    def ray(h=h, n=4, nray=8, pnt=P, dist=P, geomid=P, excl=-1):
        return L.smplsim_ray(h, P, P, n, nray, pnt, P, 0, excl, dist, geomid, s)

    def render(h=h, cam=cam, n=4, w=8, ht=8, xpos=P, depth=P):
        return L.smplsim_render(h, xpos, P, n, ref(cam), w, ht, None, depth, None, None, s)

    def track(h=h, cfg=te, tab=mt, aux=aux, state=ts, ids=P):
        return L.smplsim_track_eval(h, ref(cfg), ref(tab), ids, P, P, ref(aux), P, P, ref(state), s)

    def amp_obs(h=h, cfg=amp, tab=atab, mode=0, ids=P, out=P):
        return L.smplsim_amp_obs(h, ref(cfg), C.byref(st), C.byref(aux), ref(tab), ids, P, None, mode, out, s)

    def amp_demo(h=h, cfg=amp, tab=atab, n=4, out=P):
        return L.smplsim_amp_demo(h, ref(cfg), ref(tab), P, P, n, out, s)

    mt52, mt0 = variant(mt, nbody=52), variant(mt, num_motions=0)
    keep += [mt52, mt0]
    too_many = " with per-env body shapes n must be the handle's num_envs (row i uses env i's shape)"
    prm_rows = " with per-env parameters n must be the handle's num_envs (row i uses env i's parameters)"
    return L, keep, [
        ("create: null cfg", lambda: L.smplsim_create(C.byref(model), None, 4, 0, C.byref(out)), EINVAL,
         "smplsim_create: null argument or num_envs <= 0"),
        ("create: num_envs 0", lambda: create(n=0), EINVAL, "smplsim_create: null argument or num_envs <= 0"),
        ("create_shapes: env_model NULL", lambda: shapes(None), EINVAL, "smplsim_create_shapes: env_model is NULL"),
        ("create_shapes: env_model entry", lambda: shapes(i32(0, 1, 2, 0)), EINVAL, "smplsim_create_shapes: env_model entry out of range"),
        ("create: self_obs_v", lambda: create(variant(ecfg, self_obs_v=3)), EINVAL, "self_obs_v must be 1 or 2"),
        ("create: control_mode", lambda: create(variant(ecfg, control_mode=4)), EINVAL, "control_mode must be uhc_pd|pd|torque|simple_pid"),
        ("create: task", lambda: create(variant(ecfg, task=4)), EINVAL, "unknown task"),
        ("create: nsubsteps", lambda: create(variant(ecfg, nsubsteps=0)), EINVAL, "nsubsteps < 1"),
        ("create: reach_body", lambda: create(variant(ecfg, task=2, reach_body=nb)), EINVAL, "reach_body out of range"),

        ("step: null handle", lambda: step(h=None), EINVAL, "smplsim_step: null handle/state/action"),
        ("step: null state", lambda: step(st=None), EINVAL, "smplsim_step: null handle/state/action"),
        ("step: null qpos", lambda: step(st=variant(st, qpos=None)), EINVAL, "smplsim_step: null handle/state/action"),
        ("step: null action", lambda: step(a=None), EINVAL, "smplsim_step: null handle/state/action"),
        ("step: simple_pid state", lambda: step(h=pid._h, st=variant(st, pid_integral=None)), EINVAL,
         "smplsim_step: control_mode simple_pid needs state.pid_integral / pid_last_error"),
        ("mj_step: null handle", lambda: mj_step(h=None), EINVAL, "smplsim_mj_step: bad argument"),
        ("mj_step: null ctrl", lambda: mj_step(c=None), EINVAL, "smplsim_mj_step: bad argument"),
        ("mj_step: nsub 0", lambda: mj_step(nsub=0), EINVAL, "smplsim_mj_step: bad argument"),
        ("reset: null handle", lambda: reset(h=None), EINVAL, "smplsim_reset: null handle/state"),
        ("reset: null rng_counter", lambda: reset(st=variant(st, rng_counter=None)), EINVAL, "smplsim_reset: null handle/state"),
        ("reset: simple_pid state", lambda: reset(h=pid._h, st=variant(st, pid_last_error=None)), EINVAL,
         "smplsim_reset: control_mode simple_pid needs state.pid_integral / pid_last_error (Fall init runs the controller)"),
        ("reset: init_mode", lambda: reset(mode=3), EINVAL, "smplsim_reset: init_mode"),
        ("reset: MoCap without qpos0", lambda: reset(mode=2, q0=None), EINVAL, "smplsim_reset: MoCap init needs qpos0/qvel0"),

        ("kinematics: null handle", lambda: kin(h=None), EINVAL, "smplsim_kinematics: bad argument"),
        ("kinematics: null qpos", lambda: kin(q=None), EINVAL, "smplsim_kinematics: bad argument"),
        ("kinematics: n < 0", lambda: kin(n=-1), EINVAL, "smplsim_kinematics: bad argument"),
        ("kinematics: shapes", lambda: kin(h=shp._h, n=2), EINVAL, "smplsim_kinematics:" + too_many),
        ("inverse: null handle", lambda: inverse(h=None), EINVAL, "smplsim_inverse: null handle or n < 0"),
        ("inverse: n < 0", lambda: inverse(n=-1), EINVAL, "smplsim_inverse: null handle or n < 0"),
        ("inverse: self-collision", lambda: inverse(h=scol._h, n=0), EUNSUPPORTED,
         "smplsim_inverse: the inverse does not build geom-geom contacts (handle created with self_collision = 1)"),
        ("inverse: null qacc", lambda: inverse(qacc=None), EINVAL, "smplsim_inverse: null argument"),
        ("inverse: shapes", lambda: inverse(h=shp._h, n=2), EINVAL, "smplsim_inverse:" + too_many),
        ("inverse: parameters", lambda: inverse(h=prm._h, n=2), EINVAL, "smplsim_inverse:" + prm_rows),
        ("dynamics: null handle", lambda: dyn(h=None), EINVAL, "smplsim_dynamics: null handle, n < 0 or njac < 0"),
        ("dynamics: njac < 0", lambda: dyn(njac=-1), EINVAL, "smplsim_dynamics: null handle, n < 0 or njac < 0"),
        ("dynamics: njac > nbody", lambda: dyn(njac=nb + 1), EINVAL, "smplsim_dynamics: njac > nbody"),
        ("dynamics: null jac_body", lambda: dyn(njac=1), EINVAL, "smplsim_dynamics: njac > 0 needs jac_body"),
        ("dynamics: jac_body entry", lambda: dyn(jb=i32(0, nb), njac=2), EINVAL, "smplsim_dynamics: jac_body entry out of range [0, nbody)"),
        ("dynamics: bias without qvel", lambda: dyn(v=None, n=0), EINVAL, "smplsim_dynamics: qfrc_bias needs qvel"),
        ("dynamics: null jac", lambda: dyn(jb=i32(0), njac=1, jac=None), EINVAL, "smplsim_dynamics: njac > 0 needs jac_dev"),
        ("dynamics: no output", lambda: dyn(qM=None, bias=None), EINVAL, "smplsim_dynamics: no output requested"),
        ("dynamics: null qpos", lambda: dyn(q=None), EINVAL, "smplsim_dynamics: null qpos"),
        ("dynamics: shapes", lambda: dyn(h=shp._h, n=2), EINVAL, "smplsim_dynamics:" + too_many),
        ("dynamics: parameters", lambda: dyn(h=prm._h, n=2), EINVAL, "smplsim_dynamics:" + prm_rows),

        ("ray: null handle", lambda: ray(h=None), EINVAL, "smplsim_ray: null handle or n < 0"),
        ("ray: bodyexclude", lambda: ray(excl=nb, n=0), EINVAL, "smplsim_ray: bodyexclude out of range [-1, nbody)"),
        ("ray: nray 0", lambda: ray(nray=0), EINVAL, "smplsim_ray: nray <= 0"),
        ("ray: no output", lambda: ray(dist=None, geomid=None), EINVAL, "smplsim_ray: no output requested"),
        ("ray: null pnt", lambda: ray(pnt=None), EINVAL, "smplsim_ray: null argument"),
        ("ray: shapes", lambda: ray(h=shp._h, n=2), EINVAL, "smplsim_ray:" + too_many),
        ("ray: grid", lambda: ray(n=4096, nray=1 << 30), EINVAL, "smplsim_ray: n x nray too large for one launch"),
        ("render: null handle", lambda: render(h=None), EINVAL, "smplsim_render: null handle / camera or n < 0"),
        ("render: null camera", lambda: render(cam=None), EINVAL, "smplsim_render: null handle / camera or n < 0"),
        ("render: camera mode", lambda: render(cam=variant(cam, mode=3)), EINVAL, "smplsim_render: unknown camera mode"),
        ("render: camera body", lambda: render(cam=variant(cam, mode=CAM_BODY, body=nb)), EINVAL,
         "smplsim_render: camera body out of range [0, nbody)"),
        ("render: exclude_body", lambda: render(cam=variant(cam, exclude_body=nb), n=0), EINVAL,
         "smplsim_render: exclude_body out of range [-1, nbody)"),
        ("render: fovy", lambda: render(cam=variant(cam, fovy=180.0)), EINVAL, "smplsim_render: fovy outside (0, 180) degrees"),
        ("render: width", lambda: render(w=0), EINVAL, "smplsim_render: width / height <= 0"),
        ("render: no output", lambda: render(depth=None), EINVAL, "smplsim_render: no output requested"),
        ("render: null xpos", lambda: render(xpos=None), EINVAL, "smplsim_render: null xpos / xquat"),
        ("render: shapes", lambda: render(h=shp._h, n=2), EINVAL, "smplsim_render:" + too_many),
        ("render: TRACKCOM with parameters", lambda: render(h=prm._h, cam=variant(cam, mode=CAM_TRACKCOM), n=2), EINVAL,
         "smplsim_render: a TRACKCOM camera with per-env parameters needs n == num_envs (row i uses env i's masses)"),
        ("render: grid", lambda: render(n=1 << 20, w=4096, ht=4096), EINVAL, "smplsim_render: n x image too large for one launch"),

        ("set_env_params: null params", lambda: L.smplsim_set_env_params(h, None, None, s), EINVAL,
         "smplsim_set_env_params: null handle or params"),
        ("set_env_params: null handle", lambda: L.smplsim_set_env_params(None, ref(SmplsimEnvParamsC()), None, s), EINVAL,
         "smplsim_set_env_params: null handle or params"),
        ("get_env_params: null handle", lambda: L.smplsim_get_env_params(None, P, P, P, P, P, P, s), EINVAL,
         "smplsim_get_env_params: null handle"),
        ("clear_env_params: null handle", lambda: L.smplsim_clear_env_params(None), EINVAL, "smplsim_clear_env_params: null handle"),

        ("track_eval: null handle", lambda: track(h=None), EINVAL, "smplsim_track_eval: null handle / cfg / tables / aux / state"),
        ("track_eval: null state", lambda: track(state=None), EINVAL, "smplsim_track_eval: null handle / cfg / tables / aux / state"),
        ("track_eval: num_bodies", lambda: track(cfg=variant(te, num_bodies=2)), EINVAL, "smplsim_track_eval: num_bodies outside [3, nbody]"),
        ("track_eval: bodies NULL", lambda: track(cfg=variant(te, num_bodies=5)), EINVAL,
         "smplsim_track_eval: bodies NULL needs num_bodies == nbody"),
        ("track_eval: eval body", lambda: track(cfg=variant(te, num_bodies=3, bodies=ref(i32(0, 1, nb)).value)), EINVAL,
         "smplsim_track_eval: eval body out of range [0, nbody)"),
        ("track_eval: table nbody", lambda: track(tab=mt52), EINVAL, "smplsim_track_eval: the tables' nbody is not the handle's"),
        ("track_eval: num_motions", lambda: track(tab=mt0), EINVAL, "smplsim_track_eval: num_motions < 1"),
        ("track_eval: null table", lambda: track(tab=variant(mt, xpos=None)), EINVAL, "smplsim_track_eval: null motion table"),
        ("track_eval: aux", lambda: track(aux=variant(aux, xquat=None)), EINVAL, "smplsim_track_eval: aux needs xpos, xquat"),
        ("track_eval: null ids", lambda: track(ids=None), EINVAL, "smplsim_track_eval: null argument"),
        ("track_eval: null sums", lambda: track(state=variant(ts, sums=None)), EINVAL, "smplsim_track_eval: null state array"),
        ("track_eval: interpolate", lambda: track(cfg=variant(te, interpolate=2)), EINVAL, "smplsim_track_eval: interpolate must be 0 or 1"),
        ("track_eval: dt", lambda: track(cfg=variant(te, dt=-1.0)), EINVAL, "smplsim_track_eval: dt < 0 or NaN"),

        ("amp_obs: null handle", lambda: amp_obs(h=None), EINVAL, "smplsim_amp_obs: null handle / cfg"),
        ("amp_obs: num_steps", lambda: amp_obs(cfg=variant(amp, num_steps=0)), EINVAL, "smplsim_amp_obs: num_steps < 1"),
        ("amp_obs: interpolate", lambda: amp_obs(cfg=variant(amp, interpolate=2)), EINVAL, "smplsim_amp_obs: interpolate must be 0 or 1"),
        ("amp_obs: num_key_bodies", lambda: amp_obs(cfg=variant(amp, num_key_bodies=nb + 1)), EINVAL,
         "smplsim_amp_obs: num_key_bodies outside [0, nbody]"),
        ("amp_obs: key_bodies NULL", lambda: amp_obs(cfg=variant(amp, key_bodies=None)), EINVAL,
         "smplsim_amp_obs: key_bodies NULL with num_key_bodies > 0"),
        ("amp_obs: key body", lambda: amp_obs(cfg=variant(amp, key_bodies=ref(i32(0, nb)).value)), EINVAL,
         "smplsim_amp_obs: key body out of range [0, nbody)"),
        ("amp_obs: mode", lambda: amp_obs(mode=3), EINVAL, "smplsim_amp_obs: unknown mode"),
        ("amp_obs: null output", lambda: amp_obs(out=None), EINVAL,
         "smplsim_amp_obs: null state (qpos, qvel), aux (xpos, xquat) or output"),
        ("amp_obs: FILL_REF tables", lambda: amp_obs(mode=AMP_FILL_REF, tab=None), EINVAL, "smplsim_amp_obs: null motion tables"),
        ("amp_obs: FILL_REF nbody", lambda: amp_obs(mode=AMP_FILL_REF, tab=variant(atab, motion=C.addressof(mt52))), EINVAL,
         "smplsim_amp_obs: the tables' nbody is not the handle's"),
        ("amp_obs: FILL_REF dof_vel", lambda: amp_obs(mode=AMP_FILL_REF, tab=variant(atab, dof_vel=None)), EINVAL,
         "smplsim_amp_obs: null motion table"),
        ("amp_obs: FILL_REF ids", lambda: amp_obs(mode=AMP_FILL_REF, ids=None), EINVAL,
         "smplsim_amp_obs: FILL_REF needs motion_ids, motion_t0 and state.progress"),
        ("amp_demo: null cfg", lambda: amp_demo(cfg=None), EINVAL, "smplsim_amp_demo: null handle / cfg"),
        ("amp_demo: n < 0", lambda: amp_demo(n=-1), EINVAL, "smplsim_amp_demo: n < 0"),
        ("amp_demo: null tables", lambda: amp_demo(tab=None), EINVAL, "smplsim_amp_demo: null motion tables"),
        ("amp_demo: num_motions", lambda: amp_demo(tab=variant(atab, motion=C.addressof(mt0))), EINVAL, "smplsim_amp_demo: num_motions < 1"),
        ("amp_demo: null output", lambda: amp_demo(out=None), EINVAL, "smplsim_amp_demo: null motion_ids / motion_times / output"),
    ]


def test_every_refusal_has_its_code_and_message(backend):
    L, keep, table = refusals(backend)
    wrong = []
    for name, call, code, msg in table:
        rc = call()
        got = L.smplsim_last_error().decode()
        if rc != code or got != msg:
            wrong.append(f"{name}: {rc} {got!r}, expected {code} {msg!r}")
    assert len(table) > 90 and not wrong, "\n".join(wrong)
