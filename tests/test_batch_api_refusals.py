"""The argument rules of the Python batch API, one table row per rule and call site: caller tensors (type, shape, dtype, device,
contiguity), body names and indices, and env selections.  Each row names the call, the bad argument, the exception type (which
layer refuses it: ``ValueError`` from Python, ``SmplsimError`` from the C ABI) and a message that names the argument.  Runs on the
H100 (-m gpu) and on the host emulator build of the same kernels."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")

from smplsim_b200 import _lib, camera  # noqa: E402
from smplsim_b200.abi import model_from_cfg  # noqa: E402
from smplsim_b200.amp import HumanoidAmpB200  # noqa: E402
from smplsim_b200.cfg import make_cfg  # noqa: E402
from smplsim_b200.imitation import HumanoidImB200  # noqa: E402
from smplsim_b200.motion_lib import synthetic_tables  # noqa: E402
from util_states import make_models  # noqa: E402

N = 2
SITE = ((0.0, 0.0, 0.0), (1.0, 0.0, 0.0, 0.0))


@pytest.fixture
def setup(backend):
    cfg, _ = make_models(control_mode="torque")
    env = backend.batch(cfg, N)
    env.reset()
    m = env.model
    t = backend.t
    z = dict(q=env.qpos.clone(), v=env.qvel.clone(), a=t(np.zeros((N, m.nv))), u=t(np.zeros((N, 2, m.nu))),
             xf=t(np.zeros((N, m.nbody, 6))), p=t(np.zeros((N, 3, 3))), d=t(np.ones((N, 3, 3))))
    return backend, env, m, z


def _noncontig(x):
    """The values of ``x`` as a non-contiguous view (the last two dimensions swapped back from a transposed copy)."""
    y = x.transpose(-1, -2).contiguous().transpose(-1, -2)
    assert not y.is_contiguous() and torch.equal(y, x)
    return y


def _set_xfrc(env, x):
    env.xfrc_applied = x


# (id, call(env, m, z), exception type, match)
TENSOR_ROWS = [
    # caller rows (inverse, forward, dynamics and the other row entry points)
    ("inverse qpos not a tensor", lambda e, m, z: e.inverse(z["q"].cpu().numpy(), z["v"], z["a"]), ValueError, "qpos must be a torch.Tensor"),
    ("inverse qvel width", lambda e, m, z: e.inverse(z["q"], z["v"][:, :5], z["a"]), ValueError, "qvel must have shape"),
    ("inverse qacc n", lambda e, m, z: e.inverse(z["q"], z["v"], z["a"][:1]), ValueError,
     r"qacc must have shape \[n, {nv}\] with the same n as qpos"),
    ("inverse qpos dtype", lambda e, m, z: e.inverse(z["q"].double(), z["v"], z["a"]), ValueError, "qpos must be float32"),
    ("inverse qvel device", lambda e, m, z: e.inverse(z["q"], z["v"].to("meta"), z["a"]), ValueError, "qvel must live on"),
    ("forward qacc_warmstart n", lambda e, m, z: e.forward(z["q"], z["v"], z["a"][:, :m.nu], qacc_warmstart=z["a"][:1]), ValueError,
     r"qacc_warmstart must have shape \[n, {nv}\] with the same n as qpos"),
    ("dynamics qvel width", lambda e, m, z: e.dynamics(z["q"], z["v"][:, :5]), ValueError,
     r"qvel must have shape \[n, {nv}\] with the same n as qpos"),
    ("dynamics qvel dtype", lambda e, m, z: e.dynamics(z["q"], z["v"].double()), ValueError, "qvel must be float32"),
    ("centroidal qvel device", lambda e, m, z: e.centroidal(z["q"], z["v"].to("meta")), ValueError, "qvel must live on"),
    ("rollout qpos_fwd n", lambda e, m, z: e.rollout(z["q"], z["v"], z["u"], qpos_fwd=z["q"][:1]), ValueError,
     r"qpos_fwd must have shape \[n, {nq}\] with the same n as qpos"),
    # other caller tensors (rollout's control, ray, rne_post)
    ("rollout control not a tensor", lambda e, m, z: e.rollout(z["q"], z["v"], z["u"].tolist()), ValueError, "control must be a torch.Tensor"),
    ("rollout control shape", lambda e, m, z: e.rollout(z["q"], z["v"], z["u"][0]), ValueError, "control must have shape"),
    ("rollout control dtype", lambda e, m, z: e.rollout(z["q"], z["v"], z["u"].double()), ValueError, "control must be float32"),
    ("rollout control device", lambda e, m, z: e.rollout(z["q"], z["v"], z["u"].to("meta")), ValueError, "control must live on"),
    ("ray pnt not a tensor", lambda e, m, z: e.ray(z["p"].tolist(), z["d"]), ValueError, "pnt must be a torch.Tensor"),
    ("ray vec shape", lambda e, m, z: e.ray(z["p"], z["d"][:, :2]), ValueError, "vec must have shape"),
    ("ray pnt dtype", lambda e, m, z: e.ray(z["p"].double(), z["d"]), ValueError, "pnt must be float32"),
    ("ray vec device", lambda e, m, z: e.ray(z["p"], z["d"].to("meta")), ValueError, "vec must live on"),
    ("rne_post xfrc_applied shape", lambda e, m, z: e.rne_post(z["q"], z["v"], z["a"], xfrc_applied=z["xf"][:1]), ValueError,
     "xfrc_applied must have shape"),
    ("rne_post xfrc_applied dtype", lambda e, m, z: e.rne_post(z["q"], z["v"], z["a"], xfrc_applied=z["xf"].double()), ValueError,
     "xfrc_applied must be float32"),
    # the xfrc_applied setter
    ("xfrc_applied not a tensor", lambda e, m, z: _set_xfrc(e, z["xf"].cpu().numpy()), ValueError, "xfrc_applied must be a torch.Tensor"),
    ("xfrc_applied shape", lambda e, m, z: _set_xfrc(e, z["xf"][:, :, :3]), ValueError,
     r"xfrc_applied must have shape \({N}, {nbody}, 6\) \(envs, robot bodies, force \+ torque\)"),
    ("xfrc_applied dtype", lambda e, m, z: _set_xfrc(e, z["xf"].double()), ValueError, "xfrc_applied must be float32"),
    ("xfrc_applied device", lambda e, m, z: _set_xfrc(e, z["xf"].to("meta")), ValueError, "xfrc_applied must live on"),
    # set_env_params values
    ("set_env_params friction not a tensor", lambda e, m, z: e.set_env_params(friction=[1.0] * N), ValueError, "friction must be a torch.Tensor"),
    ("set_env_params gravity shape", lambda e, m, z: e.set_env_params(gravity=z["p"][:, 0, :2]), ValueError, r"gravity must have shape \({N}, 3\)"),
    ("set_env_params kp dtype", lambda e, m, z: e.set_env_params(kp=z["a"][:, :m.nu].double()), ValueError, "kp must be float32"),
    ("set_env_params kd device", lambda e, m, z: e.set_env_params(kd=z["a"][:, :m.nu].to("meta")), ValueError, "kd must live on"),
    # refused when not contiguous: tensors the call hands to the kernels as they are
    ("xfrc_applied not contiguous", lambda e, m, z: _set_xfrc(e, _noncontig(z["xf"])), ValueError, "xfrc_applied must be contiguous"),
    ("rne_post xfrc_applied not contiguous", lambda e, m, z: e.rne_post(z["q"], z["v"], z["a"], xfrc_applied=_noncontig(z["xf"])), ValueError,
     "xfrc_applied must be contiguous"),
    ("ray pnt not contiguous", lambda e, m, z: e.ray(_noncontig(z["p"]), z["d"]), ValueError, "pnt must be contiguous"),
    ("ray vec not contiguous", lambda e, m, z: e.ray(z["p"], _noncontig(z["d"])), ValueError, "vec must be contiguous"),
    ("ray xpos not contiguous", lambda e, m, z: e.ray(z["p"], z["d"], xpos=_noncontig(e.xpos), xquat=e.xquat), ValueError,
     "xpos must be contiguous"),
    ("render xquat not contiguous", lambda e, m, z: e.render(xpos=e.xpos, xquat=_noncontig(e.xquat)), ValueError, "xquat must be contiguous"),
]


@pytest.mark.parametrize("row", TENSOR_ROWS, ids=[r[0] for r in TENSOR_ROWS])
def test_caller_tensor_refused(setup, row):
    _, env, m, z = setup
    _, call, exc, match = row
    launches = env.gpu_launches
    with pytest.raises(exc, match=match.format(N=N, nq=m.nq, nv=m.nv, nbody=m.nbody)) as ei:
        call(env, m, z)
    assert ei.type is exc
    assert env.gpu_launches == launches and env.xfrc_applied is None


def test_noncontiguous_inputs_accepted(setup):
    """Inputs a call only reads are copied to contiguous tensors: the results are those of the contiguous inputs."""
    backend, env, m, z = setup
    q, v = z["q"], z["v"]
    a = backend.t(np.random.default_rng(0).normal(size=(N, m.nv)))
    ref = env.inverse(q, v, a)
    assert torch.equal(env.inverse(q, v, _noncontig(a)), ref)
    u = backend.t(np.random.default_rng(1).uniform(-0.5, 0.5, size=(N, 2, m.nu)))
    ref = env.rollout(q, v, u)
    got = env.rollout(q, v, _noncontig(u))
    assert all(torch.equal(got[k], ref[k]) for k in ref)
    g = backend.t(np.tile([0.0, -1.0, -9.0], (N, 1)))
    env.set_env_params(gravity=_noncontig(g))
    assert torch.equal(env.env_params["gravity"], g)


BODY_CALLS = {
    "dynamics jac_bodies": lambda e, b: e.dynamics(e.qpos.clone(), e.qvel.clone(), jac_bodies=[0, b]),
    "centroidal jac_com_bodies": lambda e, b: e.centroidal(e.qpos.clone(), e.qvel.clone(), jac_com_bodies=[0, b]),
    "rne_post imu_sites": lambda e, b: e.rne_post(e.qpos.clone(), e.qvel.clone(), torch.zeros_like(e.qvel), imu_sites=[(0,) + SITE, (b,) + SITE]),
    "camera body": lambda e, b: camera.body(e.model, b),
}
# (call, bad body, exception type, match); "nbody" stands for the first index out of range
BODY_ROWS = [
    ("dynamics jac_bodies", "Tail", ValueError, "unknown body name 'Tail'"),
    ("dynamics jac_bodies", True, ValueError, r"jac_bodies entries must be body names or indices in \[0, {nbody}\), got True"),
    ("dynamics jac_bodies", "nbody", ValueError, r"jac_bodies entries must be body names or indices in \[0, {nbody}\), got {nbody}"),
    ("centroidal jac_com_bodies", "Tail", ValueError, "unknown body name 'Tail'"),
    ("centroidal jac_com_bodies", True, ValueError, r"jac_com_bodies entries must be body names or indices in \[0, {nbody}\), got True"),
    ("centroidal jac_com_bodies", "nbody", ValueError, r"jac_com_bodies entries must be body names or indices in \[0, {nbody}\), got {nbody}"),
    ("rne_post imu_sites", "Tail", ValueError, "unknown body name 'Tail'"),
    ("rne_post imu_sites", True, ValueError, r"imu_sites bodies must be body names or indices in \[0, {nbody}\), got True"),
    ("rne_post imu_sites", "nbody", ValueError, r"imu_sites bodies must be body names or indices in \[0, {nbody}\), got {nbody}"),
    ("camera body", "Tail", ValueError, "unknown body name 'Tail'"),
    ("camera body", True, ValueError, r"body must be a name or an index in \[0, {nbody}\), got True"),
    ("camera body", "nbody", ValueError, r"body must be a name or an index in \[0, {nbody}\), got {nbody}"),
]


@pytest.mark.parametrize("row", BODY_ROWS, ids=[f"{r[0]}-{r[1]}" for r in BODY_ROWS])
def test_body_refused(setup, row):
    _, env, m, _ = setup
    name, b, exc, match = row
    launches = env.gpu_launches
    with pytest.raises(exc, match=match.format(nbody=m.nbody)) as ei:
        BODY_CALLS[name](env, m.nbody if b == "nbody" else b)
    assert ei.type is exc and env.gpu_launches == launches


def test_body_names_resolve(setup):
    _, env, m, _ = setup
    name = m.body_names[4]
    q, v = env.qpos.clone(), env.qvel.clone()
    assert torch.equal(env.dynamics(q, v, jac_bodies=[name])["jacp"], env.dynamics(q, v, jac_bodies=[np.int64(4)])["jacp"])
    assert camera.body(m, name).body == 4 and camera.body(m, 4).body == 4


# imitation tracked_bodies and AMP key_bodies: names are resolved in Python, indices are range-checked by the C ABI
TASK_ROWS = [
    ("imitation tracked_bodies", "Tail", ValueError, "unknown body name 'Tail'"),
    ("imitation tracked_bodies", True, ValueError, "tracked_bodies entries must be body names or indices, got True"),
    ("imitation tracked_bodies", "nbody", _lib.SmplsimError, r"smplsim_imitation: tracked body out of range \[0, nbody\)"),
    ("AMP key_bodies", "Tail", ValueError, "unknown key body name 'Tail'"),
    ("AMP key_bodies", True, ValueError, "key_bodies entries must be body names or indices, got True"),
    ("AMP key_bodies", "nbody", _lib.SmplsimError, r"key body out of range \[0, nbody\)"),
]


@pytest.mark.parametrize("row", TASK_ROWS, ids=[f"{r[0]}-{r[1]}" for r in TASK_ROWS])
def test_task_body_refused(backend, row):
    name, b, exc, match = row
    if b == "nbody":
        b = model_from_cfg(make_cfg(env="im")).nbody
    with pytest.raises(exc, match=match) as ei:
        if name.startswith("imitation"):
            HumanoidImB200(make_cfg(env="im"), lambda bb: synthetic_tables(bb, num_clips=2, frames=8, seed=3), num_envs=N,
                           tracked_bodies=[0, b], batch_factory=backend.batch)
        else:
            cfg = make_cfg(env="speed", overrides={"env.self_obs_v": 2, "robot.create_vel_sensors": True})
            HumanoidAmpB200(backend.batch(cfg, N), amp_cfg=dict(key_bodies=[0, b]))
    assert ei.type is exc


def test_eval_bodies_refused(backend):
    env = HumanoidImB200(make_cfg(env="im"), lambda bb: synthetic_tables(bb, num_clips=2, frames=8, seed=3), num_envs=N,
                         batch_factory=backend.batch)
    launches = env.gpu_launches
    with pytest.raises(ValueError, match="unknown body name 'Tail'"):
        env.evaluate(lambda obs: torch.zeros(N, env.num_actions, device=env.device), eval_bodies=[0, 1, "Tail"])
    with pytest.raises(ValueError, match="eval_bodies entries must be body names or indices, got True"):
        env.evaluate(lambda obs: torch.zeros(N, env.num_actions, device=env.device), eval_bodies=[0, 1, True])
    assert env.gpu_launches == launches


def test_empty_env_selection(setup):
    """An empty index tensor selects no env: ``reset`` and ``set_env_params`` return without a launch (``set_env_params`` checks the
    values' type, shape, dtype and device first, but not their range)."""
    backend, env, m, z = setup
    none = torch.zeros(0, dtype=torch.int64, device=env.device)
    obs = env.obs_buf.clone()
    launches = env.gpu_launches
    assert env.reset(none) is env.obs_buf
    assert env.set_env_params(none, friction=backend.t(np.full(N, np.nan))) is None
    assert env.gpu_launches == launches and torch.equal(env.obs_buf, obs)
    with pytest.raises(ValueError, match="friction must have shape"):
        env.set_env_params(none, friction=backend.t(np.ones(N + 1)))
    assert env.env_params["friction"].shape == (N,)


def test_env_selection_masks(setup):
    """A uint8 mask of num_envs entries goes to the kernel as it is (``reset(reset_buf)`` every step copies nothing); a bool mask and an
    index tensor select the same envs."""
    backend, env, m, z = setup
    env.reset_buf.fill_(1)
    env.reset(env.reset_buf)
    assert env._keep[0] is env.reset_buf
    sel = {}
    for key, ids in (("index", torch.tensor([1], device=env.device)), ("bool", torch.tensor([False, True], device=env.device)),
                     ("uint8", torch.tensor([0, 1], dtype=torch.uint8, device=env.device))):
        env.set_env_params(friction=backend.t(np.full(N, 0.5)))
        env.set_env_params(ids, friction=backend.t(np.full(N, 0.25)))
        sel[key] = env.env_params["friction"].cpu().numpy()
    for v in sel.values():
        assert np.array_equal(v, [0.5, 0.25])
