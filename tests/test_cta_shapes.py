"""The per-env kernels at the CTA shapes production launches, against the fp64 oracle and against 1-warp CTAs.

smplsim_create picks the warps per CTA for the fewest waves over the SMs first, then the fewest warps: 4 001 / 4 096 SMPL envs
step in 8-warp CTAs, 2 049 SMPL-X envs in 4-warp CTAs, while the few dozen envs of the other parity tests step in 1-warp CTAs.
Code that only runs with several warps per CTA -- the CTA phase barriers, the per-warp shared-memory rows and env index, the empty
warps and dead lanes of a ragged last CTA (which run predicated on env 0's global rows), the per-env shape slot map -- is held
here to two things at once:

- the fp64 oracle, with the tolerances the feature tests state (test_gpu_parity, test_xfrc, test_env_params, test_contact_wrench,
  test_inverse, test_dynamics);
- bit identity with the same envs in 1-warp CTAs: the size of an env's CTA must change none of its arithmetic.

On the GPU the production shapes come from the env count alone.  The emulator reports an H100's 132 SMs and shared memory, so
there SMPLSIM_WPB forces the same CTA sizes at a few dozen envs.  Every test asserts the CTA shape it ran.  The 1-warp reference
of state-only calls (mj_step, kinematics, inverse, dynamics, also with per-env shapes and parameter records) replays the same rows
in batches of at most 132 x 4 envs, where one warp per CTA already gives one wave, so the GPU tests need no SMPLSIM_* variable.
Reset and env steps draw from Philox streams keyed by the env index, which a replay in smaller batches would change: their
1-warp reference is the same batch with SMPLSIM_WPB=1, and where that variable no longer forces the CTA size they are held to
the oracle alone.

States are a small pool of mixed kinds tiled over the envs, so that every CTA holds airborne envs (no rows), contact-rich ones
(several active-set iterations), envs past their joint limits and one whose qacc overflows (mj_checkAcc resets it inside the
substep), and the oracle runs once per pool state: every env must also equal every other env of the same pool state bit for bit."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
from oracle import oracle as orc  # noqa: E402
from smplsim_b200.abi import model_from_cfg  # noqa: E402
from test_contact_wrench import oracle_wrench, ref_wrench  # noqa: E402
from test_dynamics import ref_jac  # noqa: E402
from test_env_params import draw, oracle_for, variant  # noqa: E402
from test_inverse import ref_inverse  # noqa: E402
from util_states import airborne_states, elem_relerr, make_models, relerr, rollout_states  # noqa: E402
from xfrc_oracle import XfrcOracleEnv  # noqa: E402

TOL = 1e-4
EPW = 4                  # envs per warp (8 lanes each)
SMS = 132                # H100 SMs (the emulator reports the same)
CHUNK = SMS * EPW        # rows up to which 1-warp CTAs already give one wave: the CTA size rule picks 1 warp
NCS = {"smpl_humanoid": 15, "smplx_humanoid": 14}   # contact entries held in shared memory; the rest live in global scratch
WPB = {"smpl_humanoid": 8, "smplx_humanoid": 4}     # production CTA sizes

# envs per test and backend: the GPU sizes reach the production CTA size by count alone; the emulator sizes are small enough for
# the host (each test well under a minute) and still leave a ragged last CTA
N_SMPL = {"gpu": 4001, "emu": 61}          # 8 warps: 125 full CTAs + 1 env (7 empty warps, 3 dead lanes) / 1 full + 29 envs
N_SMPLX = {"gpu": 2049, "emu": 33}         # 4 warps: 128 full CTAs + 1 env / 2 full + 1 env
N_STEPS = {"smpl_humanoid": {"gpu": 4001, "emu": 33}, "smplx_humanoid": {"gpu": 2049, "emu": 17}}
N_DEAD = {"gpu": (4000, 4001), "emu": (32, 33)}   # (no dead lane, dead lanes in the last CTA)
N_SELF = {"gpu": 4001, "emu": 33}
N_SHAPES = {"gpu": 3990, "emu": 45}          # three shapes, each with a ragged last CTA
N_DYN = {"gpu": (4096, 37), "emu": (32, 5)}   # (num_envs, extra rows: the second launch is a ragged 8-warp grid)


# ------------------------------------------------------------------ shapes
def _wpb(env):
    return env._L().smplsim_warps_per_block(env._h)


def _grid(env):
    """CTAs of a launch over all envs (envs of one body shape per CTA)."""
    per = _wpb(env) * EPW
    if env.env_model is None:
        return -(-env.num_envs // per)
    return int(sum(-(-c // per) for c in np.bincount(env.env_model)))


def _production(backend, monkeypatch, cfg, n, wpb, ragged=True, **kw):
    """A batch at the production CTA size: by env count alone on the GPU, forced with SMPLSIM_WPB on the emulator.  Asserts the
    warps per CTA, one wave, and whether the last CTA is ragged."""
    if backend.name == "emu":
        monkeypatch.setenv("SMPLSIM_WPB", str(wpb))
    else:
        monkeypatch.delenv("SMPLSIM_WPB", raising=False)
    try:
        env = backend.batch(cfg, n, **kw)
    finally:
        monkeypatch.delenv("SMPLSIM_WPB", raising=False)
    assert _wpb(env) == wpb, (n, _wpb(env), wpb)
    grid = _grid(env)
    assert grid <= SMS
    if env.env_model is None:
        assert (n % (wpb * EPW) != 0) == ragged, (n, wpb)
        assert backend.name == "emu" or grid > SMS // 2, grid
    return env


def _one_warp_same_envs(backend, monkeypatch, cfg, n, **kw):
    """The same batch with 1-warp CTAs (same env indices, hence the same Philox streams of reset and env steps, which a replay in
    smaller batches would change), or None where SMPLSIM_WPB no longer forces the CTA size: reset and env steps are then held
    to the oracle alone.  State-only calls use _one_warp_chunks, which needs no knob."""
    monkeypatch.setenv("SMPLSIM_WPB", "1")
    try:
        env = backend.batch(cfg, n, **kw)
    finally:
        monkeypatch.delenv("SMPLSIM_WPB", raising=False)
    return env if _wpb(env) == 1 else None


def _one_warp_chunks(backend, n, make, run, chunk=CHUNK):
    """run(make(rows), rows) over chunks of at most `chunk` rows, where the CTA size rule itself picks 1 warp; outputs concatenated."""
    outs = []
    for r0 in range(0, n, chunk):
        s = slice(r0, min(n, r0 + chunk))
        env = make(s)
        assert _wpb(env) == 1, (s, _wpb(env))
        outs.append(run(env, s))
    return {k: np.concatenate([o[k] for o in outs]) for k in outs[0]}


def _bit_equal(got, ref, what):
    for k in ref:
        a, b = got[k], ref[k]
        assert a.shape == b.shape, (what, k, a.shape, b.shape)
        same = np.all((a == b).reshape(len(a), -1), axis=1)
        assert same.all(), (what, k, "first differing rows", np.flatnonzero(~same)[:8])


def _dups_equal(got, idx, what):
    """Envs stepped from the same pool state give the same bits wherever their CTA, warp and lane."""
    first = np.zeros(idx.max() + 1, dtype=np.int64)
    for k in range(len(first)):
        first[k] = np.flatnonzero(idx == k)[0]
    for k, a in got.items():
        b = a[first[idx]]
        same = np.all((a == b).reshape(len(a), -1), axis=1)
        assert same.all(), (what, k, "rows differing from the first env of their pool state", np.flatnonzero(~same)[:8])


def _outs(env, keys=("qpos", "qvel", "qacc", "qacc_warm", "contact_mask", "solver_iter", "status")):
    out = {k: getattr(env, k).cpu().numpy().copy() for k in keys}
    if env.contact_wrench is not None:
        out["contact_wrench"] = env.contact_wrench.cpu().numpy().copy()
    return out


# ------------------------------------------------------------------ states
def _lying(m, rng):
    """Lying flat on the back, a few cm into the floor: more floor contacts than the shared-memory entries (the rest overflow to
    global scratch)."""
    q = np.zeros(m.nq)
    q[2] = 0.12; q[3] = np.cos(np.pi / 4); q[5] = np.sin(np.pi / 4)
    q[7:] = rng.normal(size=m.nu) * 0.03
    return q


def _pool(robot, self_collision=False, seed_states=11, every=3):
    """(q, v, w, kind) of 30 mixed states: index 0 lying flat (most contacts); then contact-rich rollout states, with every third
    state one of: a rollout state whose qacc overflows ("bad"), airborne states, airborne states with five hinges past their range.
    Any 16 consecutive envs of the tiling hold every kind."""
    if self_collision:
        om_pd = make_models(env="getup", robot=robot, control_mode="uhc_pd", self_collision=True)[1]
        q, v, w = rollout_states(om_pd, 20, seed=7, init_mode=1, control_sigma=0.6)
    else:
        om_pd = make_models(robot=robot, control_mode="uhc_pd")[1]
        q, v, w = rollout_states(om_pd, 20, seed=seed_states, every=every)
    m = om_pd.model
    rng = np.random.default_rng(17)
    qa, va = airborne_states(m, 4, seed=3)
    ql, vl = airborne_states(m, 4, seed=4)
    ql[:, 7:] *= 0.2
    lo, hi = np.asarray(m.dof_range)[6:, 0], np.asarray(m.dof_range)[6:, 1]
    for j in range(4):
        d = rng.choice(m.nu, 5, replace=False)
        up = rng.random(5) < 0.5
        ql[j, 7 + d] = np.where(up, hi[d] + 0.02, lo[d] - 0.02)
        vl[j, 6 + d] = np.where(up, 1.0, -1.0)
    qb, vb = q[5:6].copy(), v[5:6].copy()
    vb[:, 6:] = 8e9                                  # finite state, velocity-product forces overflow: mj_checkAcc
    qs = np.concatenate([_lying(m, rng)[None], q, qb, qa[:2], ql[:2], qa[2:], ql[2:]])
    vs = np.concatenate([np.zeros((1, m.nv)), v, vb, va[:2], vl[:2], va[2:], vl[2:]])
    ws = np.concatenate([np.zeros((1, m.nv)), w, w[5:6], np.zeros((8, m.nv))])
    kinds = ["lying"] + ["rollout"] * 20 + ["bad"] + ["airborne"] * 2 + ["limit"] * 2 + ["airborne"] * 2 + ["limit"] * 2
    order = [0]
    for j in range(9):
        order += [1 + 2 * j, 2 + 2 * j, 21 + j]
    order += [19, 20]
    assert sorted(order) == list(range(30))
    return qs[order], vs[order], ws[order], [kinds[i] for i in order]


def _oracle_step(om, q, v, w, ctrl, xf=None):
    e = XfrcOracleEnv(om) if xf is not None else orc.OracleEnv(om)
    e.qpos[:] = q; e.qvel[:] = v; e.qacc_warm[:] = w; e.ctrl[:] = ctrl
    if xf is not None:
        e.xfrc_applied[:] = xf
    e.warn = 0
    e.mj_step()
    return e


def _check_row(e, r, i, tol, m, kind):
    """One env's mj_step outputs r (dict of rows) against the oracle env e after the same step, with the tolerances of
    test_mj_step_contact_states / test_bad_state_autoreset_matches_mj_step_semantics.  Returns False for a state with a contact
    inside the |dist - margin| < 1e-5 guard band (not compared)."""
    if kind == "bad":
        assert e.warn & 4 and r["status"][i] & 4, (i, e.warn, r["status"][i])
        assert relerr(r["qpos"][i], e.qpos) < 1e-3 and relerr(r["qvel"][i], e.qvel) < 5e-3, i
        return True
    con = e.contacts()
    if e.ncon and (np.abs(con["dist"] - m.margin) < 1e-5).any():
        return False
    assert not r["status"][i] & (1 | 2 | 4 | 8 | 16), (i, kind, r["status"][i])
    assert int(r["contact_mask"][i]) == e.contact_mask, (i, kind, bin(int(r["contact_mask"][i])), bin(e.contact_mask))
    gv, gq = r["qvel"][i], r["qpos"][i]
    assert relerr(gv, e.qvel) < tol, ("qvel", i, kind, relerr(gv, e.qvel), e.ncon)
    assert relerr(gq, e.qpos) < tol, ("qpos", i, kind, relerr(gq, e.qpos))
    assert elem_relerr(gv, e.qvel, 1.0) < 20 * tol, ("qvel per element", i, kind, elem_relerr(gv, e.qvel, 1.0))
    assert elem_relerr(gq, e.qpos, 1.0) < 1e-5, ("qpos per element", i, kind)
    assert relerr(r["qacc"][i], e.qacc) < 5e-4, ("qacc", i, kind, relerr(r["qacc"][i], e.qacc))
    return True


def _tiled(robot, n, seed=2, self_collision=False, **pool):
    q, v, w, kinds = _pool(robot, self_collision, **pool)
    P = len(q)
    assert n >= P
    idx = np.arange(n) % P
    nu = q.shape[1] - 7
    ctrl = np.random.default_rng(seed).uniform(-80, 80, (P, nu))
    return q, v, w, kinds, ctrl, idx


# ------------------------------------------------------------------ 1. mj_step, one substep
@pytest.mark.parametrize("robot,mode", [("smpl_humanoid", "torque"), ("smpl_humanoid", "uhc_pd"), ("smplx_humanoid", "torque")])
def test_mj_step_at_production_shape(backend, monkeypatch, robot, mode):
    """One substep of every env at the production CTA size: against the oracle per pool state, bit-identical between envs of the
    same state and with 1-warp CTAs.  SMPL-X is held to 2e-4 as in test_mj_step_contact_states."""
    tol = TOL if robot == "smpl_humanoid" else 2e-4
    cfg, om = make_models(robot=robot, control_mode=mode)
    m = om.model
    n = (N_SMPL if robot == "smpl_humanoid" else N_SMPLX)[backend.name]
    q, v, w, kinds, ctrl, idx = _tiled(robot, n)
    t = backend.t

    def run(env, s):
        env.set_state(t(q[idx[s]]), t(v[idx[s]]))
        env.qacc_warm.copy_(t(w[idx[s]]))
        env.mj_step(t(ctrl[idx[s]]), 1)
        return _outs(env)

    got = run(_production(backend, monkeypatch, cfg, n, WPB[robot]), slice(0, n))
    _bit_equal(got, _one_warp_chunks(backend, n, lambda s: backend.batch(cfg, s.stop - s.start), run), "8/4-warp vs 1-warp CTAs")
    _dups_equal(got, idx, "same pool state")
    ncmp = nrows = 0
    for k in range(len(q)):
        e = _oracle_step(om, q[k], v[k], w[k], ctrl[k])
        if _check_row(e, got, k, tol, m, kinds[k]):
            ncmp += 1
            nrows += e.nefc > 0
    assert got["solver_iter"][idx == 0].min() >= 2 and got["solver_iter"].max() >= 4   # CTAs mix long and short solves
    assert ncmp >= len(q) - 3 and nrows > len(q) // 2, (ncmp, nrows)


# ------------------------------------------------------------------ 4. dead lanes leave env 0 alone
def test_dead_lanes_leave_env0_alone(backend, monkeypatch):
    """Dead lanes of a ragged last CTA run predicated on env 0's global rows (scratch with the overflow contact entries, working
    set, sensors).  Env 0 lies flat with more contacts than the shared-memory entries; every env, env 0 first, must come out of
    three mj_steps bit for bit the same with and without dead lanes in the last CTA: state, qacc_warm, contact wrench and the
    solver iterations, which show the working set each step hands to the next."""
    robot = "smpl_humanoid"
    cfg, om = make_models(robot=robot, control_mode="torque")
    m = om.model
    n_full, n_dead = N_DEAD[backend.name]
    q, v, w, kinds, ctrl, idx = _tiled(robot, n_dead, seed=4)
    e0 = _oracle_step(om, q[0], v[0], w[0], ctrl[0])
    assert e0.ncon > NCS[robot], e0.ncon
    t = backend.t
    runs = {}
    for n, ragged in ((n_full, False), (n_dead, True)):
        env = _production(backend, monkeypatch, cfg, n, 8, ragged=ragged, contact_wrench=True)
        if ragged:
            assert n % (8 * EPW) == 1        # the last CTA: one live env, 3 dead lanes in its warp, 7 empty warps
        env.set_state(t(q[idx[:n]]), t(v[idx[:n]]))
        env.qacc_warm.copy_(t(w[idx[:n]]))
        runs[n] = []
        for _ in range(3):
            env.mj_step(t(ctrl[idx[:n]]), 1)
            runs[n].append(_outs(env))
    for step, (a, b) in enumerate(zip(runs[n_full], runs[n_dead])):
        _bit_equal({k: x[:n_full] for k, x in b.items()}, a, f"step {step}: with vs without dead lanes")
    r0 = runs[n_full][0]
    assert _check_row(e0, r0, 0, TOL, m, "lying")
    assert all(r[k]["solver_iter"][0] >= 1 for r in (runs[n_full], runs[n_dead]) for k in range(3))


# ------------------------------------------------------------------ 2 + 3. env steps and masked reset
@pytest.mark.parametrize("robot", ["smpl_humanoid", "smplx_humanoid"])
def test_env_steps_and_masked_reset_at_production_shape(backend, monkeypatch, robot):
    """getup: reset (Fall init), three env steps with the stable-PD controller (15 substeps each), some envs of every CTA put in a
    state whose qacc overflows (auto-reset inside the step), then a masked reset of every other env of CTA 0
    and the whole of its last warp.  Against per-env oracles for CTA 0, the last CTA and a stride of the rest (tolerances of
    test_env_step_matches_oracle / test_bad_state_autoreset_matches_mj_step_semantics), and bit-identical with 1-warp CTAs."""
    cfg, om = make_models(env="getup", robot=robot, seed=123)
    m = om.model
    n = N_STEPS[robot][backend.name]
    wpb = WPB[robot]
    per = wpb * EPW
    bad = np.arange(n) % 37 == 5
    rng = np.random.default_rng(9)
    acts = [np.clip(rng.normal(size=(n, m.nu)) * 0.1, -1, 1) for _ in range(3)]   # the action scale of test_env_step_matches_oracle
    mask = np.zeros(n, dtype=np.uint8)
    mask[0:per:2] = 1
    mask[per - EPW:per] = 1
    t = backend.t
    keys = ("qpos", "qvel", "qpos_fwd", "qvel_fwd", "qacc_warm", "progress_buf", "recovery", "rng_counter", "task_target",
            "obs_buf", "status", "solver_iter")

    def run(env):
        out = [{"obs": env.reset().cpu().numpy().copy()}]
        qv = env.qvel.clone()
        qv[torch.as_tensor(bad, device=qv.device), 6:] = 8e9
        env.set_state(env.qpos.clone(), qv)
        for a in acts:
            obs, rew, term, trunc = env.step(t(a))
            out.append({"obs": obs.cpu().numpy().copy(), "rew": rew.cpu().numpy().copy(), "term": term.cpu().numpy().copy(),
                        "trunc": trunc.cpu().numpy().copy(), **_outs(env, keys)})
        env.reset(t(mask, dtype=torch.uint8))
        out.append(_outs(env, keys))
        return out

    got = run(_production(backend, monkeypatch, cfg, n, wpb, seed=123))
    one = _one_warp_same_envs(backend, monkeypatch, cfg, n, seed=123)
    for step, (a, b) in enumerate(zip(got, run(one) if one is not None else [])):
        _bit_equal(a, b, f"call {step}: {wpb}-warp vs 1-warp CTAs")
    assert (got[1]["status"][bad] & 4).all() and not (got[1]["status"][~bad] & 7).any()
    # masked reset: unmasked rows untouched
    keep = mask == 0
    for k in keys:
        if k not in ("status", "solver_iter"):
            assert np.array_equal(got[4][k][keep], got[3][k][keep]), k
    # oracle: CTA 0, the last CTA, a stride of the rest
    last = (n - 1) // per * per
    sample = sorted(set(range(per)) | set(range(last, n)) | set(range(per, last, 97)))
    ncmp = 0
    for i in sample:
        e = orc.OracleEnv(om, env_id=i)
        assert np.abs(got[0]["obs"][i] - e.reset()).max() < 2e-3, ("reset obs", i)
        if bad[i]:
            e.qvel[6:] = 8e9
            e.forward()
        for s in range(3):
            e.warn = 0
            o, r, te, tr = e.step(acts[s][i])
            g = got[s + 1]
            if bad[i]:
                if s == 0:
                    assert e.warn & 4
                    assert relerr(g["qpos"][i], e.qpos) < 1e-3 and relerr(g["qvel"][i], e.qvel) < 5e-3, i
                continue
            tol = 5e-4 * (s + 1) * 10
            assert np.abs(g["obs"][i] - o).max() < tol, (s, i, np.abs(g["obs"][i] - o).max())
            assert abs(g["rew"][i] - r) < tol and bool(g["term"][i]) == te and bool(g["trunc"][i]) == tr, (s, i)
        if mask[i] and not bad[i]:
            assert np.abs(got[4]["obs_buf"][i] - e.reset()).max() < 2e-3, ("masked reset obs", i)
            ncmp += 1
    assert ncmp >= per // 2


# ------------------------------------------------------------------ 5. options: per-env parameters, external wrenches, contact wrench, self-collision
def _paired_params(m, robot, q, kinds, ctrl):
    """Per-env parameter draws for a pool of _pool(seed_states=40, every=9): each rollout state with the draws and ctrl
    test_mj_step_matches_variant_oracle pairs it with; the other states take the remaining draws."""
    P = len(q)
    qr = rollout_states(make_models(robot=robot, control_mode="uhc_pd")[1], 32, seed=40, every=9)[0]
    D, C0 = draw(m, 32, 42), np.random.default_rng(41).uniform(-80, 80, (32, m.nu))
    src, spare = np.zeros(P, dtype=np.int64), iter(range(20, 32))
    for k in range(P):
        hit = np.flatnonzero((qr == q[k]).all(axis=1)) if kinds[k] == "rollout" else []
        src[k] = hit[0] if len(hit) else next(spare)
    assert sum(kd == "rollout" for kd in kinds) == 20 and (src[[kd == "rollout" for kd in kinds]] < 20).all()
    prm = {key: x[src] for key, x in D.items()}
    return prm, np.where(np.array([kd == "rollout" for kd in kinds])[:, None], C0[src], ctrl)


def test_env_params_and_contact_wrench_at_production_shape(backend, monkeypatch):
    """One substep with per-env parameter records (friction, gravity, gains, torque limits, masses: the k_step5 instance that reads
    them; no external wrench here, see test_external_wrench_at_production_shape) and the contact-wrench output, from the states
    test_env_params holds to its tolerances, against the wrench oracle of each env's variant model (tolerances of test_env_params /
    test_contact_wrench) and bit-identical with 1-warp CTAs."""
    robot = "smpl_humanoid"
    cfg, _ = make_models(robot=robot, control_mode="torque")
    m = model_from_cfg(cfg)
    n = N_SMPL[backend.name]
    q, v, w, kinds, ctrl, idx = _tiled(robot, n, seed=6, seed_states=40, every=9)   # the rollout states of test_env_params
    P = len(q)
    prm, ctrl = _paired_params(m, robot, q, kinds, ctrl)
    t = backend.t

    def run(env, s):
        env.set_env_params(**{k: t(x[idx[s]]) for k, x in prm.items()})
        env.set_state(t(q[idx[s]]), t(v[idx[s]]))
        env.qacc_warm.copy_(t(w[idx[s]]))
        env.mj_step(t(ctrl[idx[s]]), 1)
        return _outs(env)

    got = run(_production(backend, monkeypatch, cfg, n, 8, contact_wrench=True), slice(0, n))
    ref = _one_warp_chunks(backend, n, lambda s: backend.batch(cfg, s.stop - s.start, contact_wrench=True), run)
    _bit_equal(got, ref, "8-warp vs 1-warp CTAs")
    _dups_equal(got, idx, "same pool state")
    ncmp = 0
    for k in range(P):
        om_k = oracle_for(cfg, m, prm, k)
        e = _oracle_step(om_k, q[k], v[k], w[k], ctrl[k])
        if kinds[k] == "bad":
            assert got["status"][k] & 4
            continue
        con = e.contacts()
        if e.ncon and (np.abs(con["dist"] - m.margin) < 1e-5).any():
            continue
        assert int(got["contact_mask"][k]) == e.contact_mask, k
        assert relerr(got["qvel"][k], e.qvel) < 2e-4 and relerr(got["qpos"][k], e.qpos) < TOL, (k, relerr(got["qvel"][k], e.qvel))
        f = XfrcOracleEnv(om_k)
        f.qpos[:] = q[k]; f.qvel[:] = v[k]; f.qacc_warm[:] = w[k]; f.ctrl[:] = ctrl[k]
        f.forward()
        W = oracle_wrench(f)
        wt = float(np.sum(variant(m, prm, k).body_mass)) * 9.81
        err = np.abs(got["contact_wrench"][k] - W).max() / max(wt, float(np.abs(W).max()))
        assert err < 2e-3, (k, err, e.ncon)
        if e.ncon == 0:
            assert np.all(got["contact_wrench"][k] == 0.0), k
        ncmp += 1
    assert ncmp >= P - 4


@pytest.mark.parametrize("records", [False, True])
def test_external_wrench_at_production_shape(backend, monkeypatch, records):
    """One substep with xfrc_applied live on two envs in three (forces up to 2 m_b g, torques up to 20 N m on every body) and zero on
    the rest, so that every warp mixes both, through the k_step5 instance with the wrench code (records=False) and the one with the
    wrench code and per-env parameter records (records=True).  Against the wrench oracle (tests/xfrc_oracle.py) -- of each env's
    variant model with records -- with the tolerances of test_mj_step_with_wrench_matches_oracle (qpos / qvel 1e-4, qacc 5e-4) and,
    with records, of test_mj_step_matches_variant_oracle (qvel 2e-4, qpos 1e-4); contact flags bit-exact outside the guard band;
    bit-identical with 1-warp CTAs."""
    robot = "smpl_humanoid"
    cfg, om = make_models(robot=robot, control_mode="torque")
    m = model_from_cfg(cfg)
    n = N_SMPL[backend.name]
    pool = dict(seed_states=40, every=9) if records else {}
    q, v, w, kinds, ctrl, idx = _tiled(robot, n, seed=7, **pool)
    P = len(q)
    prm = None
    if records:
        prm, ctrl = _paired_params(m, robot, q, kinds, ctrl)
    rng = np.random.default_rng(7)
    mass = np.asarray(m.body_mass)[None, :, None]
    xf = np.concatenate([rng.uniform(-1, 1, (P, m.nbody, 3)) * 2.0 * 9.81 * mass, rng.uniform(-1, 1, (P, m.nbody, 3)) * 20.0], axis=2)
    xf[np.arange(P) % 3 == 1] = 0.0
    assert len({int(k % 3 == 1) for k in idx[:EPW]}) == 2          # a warp holds envs with and without a wrench
    t = backend.t

    def run(env, s):
        if records:
            env.set_env_params(**{k: t(x[idx[s]]) for k, x in prm.items()})
        env.xfrc_applied = t(xf[idx[s]])
        env.set_state(t(q[idx[s]]), t(v[idx[s]]))
        env.qacc_warm.copy_(t(w[idx[s]]))
        env.mj_step(t(ctrl[idx[s]]), 1)
        return _outs(env)

    got = run(_production(backend, monkeypatch, cfg, n, 8), slice(0, n))
    _bit_equal(got, _one_warp_chunks(backend, n, lambda s: backend.batch(cfg, s.stop - s.start), run), "8-warp vs 1-warp CTAs")
    _dups_equal(got, idx, "same pool state")
    ncmp = moved = 0
    for k in range(P):
        om_k = oracle_for(cfg, m, prm, k) if records else om
        e = _oracle_step(om_k, q[k], v[k], w[k], ctrl[k], xf[k])
        if kinds[k] == "bad":
            assert e.warn & 4 and got["status"][k] & 4, k
            continue
        con = e.contacts()
        if e.ncon and (np.abs(con["dist"] - m.margin) < 1e-5).any():
            continue
        assert not got["status"][k] & (8 | 16), (k, got["status"][k])
        assert int(got["contact_mask"][k]) == e.contact_mask, ("contact flags", k)
        gv, gq = got["qvel"][k], got["qpos"][k]
        assert relerr(gv, e.qvel) < (2e-4 if records else TOL), ("qvel", k, kinds[k], relerr(gv, e.qvel), e.ncon)
        assert relerr(gq, e.qpos) < TOL, ("qpos", k, kinds[k], relerr(gq, e.qpos))
        if not records:
            assert relerr(got["qacc"][k], e.qacc) < 5e-4, ("qacc", k, relerr(got["qacc"][k], e.qacc))
        if k % 3 != 1 and k < 12:      # the wrench matters: without it the same step lands elsewhere
            e0 = _oracle_step(om_k, q[k], v[k], w[k], ctrl[k])
            moved += relerr(gv, e0.qvel) > 100 * TOL
        ncmp += 1
    assert ncmp >= P - 4 and moved >= 4, (ncmp, moved)


def test_self_collision_at_production_shape(backend, monkeypatch):
    """A self-collision handle (its own kernel class, hence its own CTA size): one substep from tangled getup states, against the
    self-colliding oracle (tolerances of test_mj_step_self_contact_states) and bit-identical with 1-warp CTAs."""
    robot = "smpl_humanoid"
    cfg, om = make_models(env="getup", robot=robot, control_mode="torque", self_collision=True)
    m = om.model
    n = N_SELF[backend.name]
    q, v, w, kinds, ctrl, idx = _tiled(robot, n, seed=3, self_collision=True)
    ctrl *= 0.75                                      # U(-60, 60) as test_mj_step_self_contact_states
    t = backend.t

    def run(env, s):
        env.set_state(t(q[idx[s]]), t(v[idx[s]]))
        env.qacc_warm.copy_(t(w[idx[s]]))
        env.mj_step(t(ctrl[idx[s]]), 1)
        return _outs(env)

    got = run(_production(backend, monkeypatch, cfg, n, 8), slice(0, n))
    _bit_equal(got, _one_warp_chunks(backend, n, lambda s: backend.batch(cfg, s.stop - s.start), run), "8-warp vs 1-warp CTAs")
    _dups_equal(got, idx, "same pool state")
    nself = ncmp = 0
    for k in range(len(q)):
        e = _oracle_step(om, q[k], v[k], w[k], ctrl[k])
        st = got["status"][k]
        if kinds[k] == "bad":
            assert e.warn & 4 and st & 4
            continue
        con = e.contacts()
        ns = int((con["geom1"] > 0).sum())
        if e.ncon and (np.abs(con["dist"] - m.margin) < 1e-5).any():
            continue
        if ns > 4:
            assert st & 8, (k, ns, st)
            continue
        assert not st & (8 | 16 | 32), (k, ns, st)
        assert relerr(got["qvel"][k], e.qvel) < TOL and relerr(got["qpos"][k], e.qpos) < TOL, (k, ns, relerr(got["qvel"][k], e.qvel))
        assert relerr(got["qacc"][k], e.qacc) < 5e-4, (k, ns)
        nself += ns > 0
        ncmp += 1
    assert nself >= 4 and ncmp >= len(q) // 2, (nself, ncmp)


# ------------------------------------------------------------------ 6. per-env body shapes at 8-warp CTAs
def _shape_variant(tmp_path, leg=1.18, arm=0.88, trunk=1.07, girth=1.15, density=1.2):
    """A differently proportioned SMPL body (other bone offsets, geom sizes and hence masses / inertias; same tree, joints and geom
    types), as a `*.model.json` for cfg.robot.xml_path -- as test_per_env_body_shapes_match_oracle builds it."""
    import json
    from smplsim_b200 import model as M
    p = M.load_parsed("smpl")
    d = M._to_jsonable(p)

    def fac(name):
        if any(k in name for k in ("Hip", "Knee", "Ankle", "Toe")):
            return leg
        if any(k in name for k in ("Shoulder", "Elbow", "Wrist", "Hand", "Thorax")):
            return arm
        return trunk
    for b in d["bodies"]:
        f = fac(b["name"])
        b["pos"] = [x * (leg if b["free"] else f) for x in b["pos"]]
    names = [b["name"] for b in d["bodies"]]
    for g in d["geoms"]:
        f = fac(names[g["body"]] if isinstance(g["body"], int) else g["body"])
        g["pos"] = [x * f for x in g["pos"]]
        s = list(g["size"])
        if g["type"] == 3:
            s[0] *= girth; s[1] *= f
        else:
            s = [x * girth for x in s]
        g["size"] = s
        g["density"] = g["density"] * density
    path = tmp_path / "variant.model.json"
    path.write_text(json.dumps(d))
    return str(path)


def test_per_env_body_shapes_at_production_shape(backend, monkeypatch, tmp_path):
    """Three body shapes interleaved over the envs in ragged groups, so that every shape's last CTA has empty slots (slot_env -1):
    kinematics, one mj_step and reset + two stable-PD env steps, each against the oracle of the env's own shape (tolerances of
    test_per_env_body_shapes_match_oracle) and bit-identical with 1-warp CTAs."""
    from smplsim_b200.model import fk_numpy
    (tmp_path / "a").mkdir(); (tmp_path / "b").mkdir()
    paths = [None, _shape_variant(tmp_path / "a"), _shape_variant(tmp_path / "b", leg=0.85, arm=1.1, trunk=0.93, girth=0.9, density=0.9)]

    def mk(mode, k, seed=0):
        return make_models(control_mode=mode, seed=seed, **({"robot.xml_path": paths[k]} if paths[k] else {}))
    n = N_SHAPES[backend.name]
    env_model = np.array([(i * 7 + i // 5) % 3 for i in range(n)], dtype=np.int32)
    cnt = np.bincount(env_model)
    assert (cnt % 32 != 0).all(), cnt                 # every shape's last CTA is ragged
    cfg_t = [mk("torque", k)[0] for k in range(3)]
    om_t = [mk("torque", k)[1] for k in range(3)]
    models = [model_from_cfg(c) for c in cfg_t]
    pools = [rollout_states(mk("uhc_pd", k)[1], 12, seed=20 + k, every=9) for k in range(3)]
    pidx = np.zeros(n, dtype=np.int64)
    seen = [0, 0, 0]
    for i, k in enumerate(env_model):
        pidx[i] = seen[k] % 12
        seen[k] += 1
    q = np.array([pools[k][0][pidx[i]] for i, k in enumerate(env_model)])
    v = np.array([pools[k][1][pidx[i]] for i, k in enumerate(env_model)])
    w = np.array([pools[k][2][pidx[i]] for i, k in enumerate(env_model)])
    ctrl = np.random.default_rng(6).uniform(-80, 80, (12, models[0].nu))[pidx]
    t = backend.t

    def run(env, s):
        xp, xq = env.kinematics(t(q[s]))
        env.set_state(t(q[s]), t(v[s]))
        env.qacc_warm.copy_(t(w[s]))
        env.mj_step(t(ctrl[s]), 1)
        return {"xpos": xp.cpu().numpy(), "xquat": xq.cpu().numpy(), **_outs(env)}

    got = run(_production(backend, monkeypatch, cfg_t[0], n, 8, models=models, env_model=env_model), slice(0, n))
    # 1-warp reference in chunks of 516 envs: at most 129 + 3 one-warp CTAs over the three shapes' groups, one wave
    ref = _one_warp_chunks(backend, n, lambda s: backend.batch(cfg_t[0], s.stop - s.start, models=models, env_model=env_model[s]), run,
                           chunk=CHUNK - 12)
    _bit_equal(got, ref, "8-warp vs 1-warp CTAs")
    key = env_model * 12 + pidx
    _dups_equal(got, np.unique(key, return_inverse=True)[1], "same shape and state")
    ncon = ncmp = 0
    for kk in np.unique(key):
        i = int(np.flatnonzero(key == kk)[0])
        k = env_model[i]
        ep, eq_, _ = fk_numpy(models[k], q[i])
        assert np.abs(got["xpos"][i] - ep).max() < 2e-5, ("kinematics with env i's shape", i)
        gx = got["xquat"][i]
        assert np.minimum(np.abs(gx - eq_).max(axis=1), np.abs(gx + eq_).max(axis=1)).max() < 1e-5, ("xquat with env i's shape", i)
        e = _oracle_step(om_t[k], q[i], v[i], w[i], ctrl[i])
        con = e.contacts()
        if e.ncon and (np.abs(con["dist"] - models[k].margin) < 1e-5).any():
            continue
        assert int(got["contact_mask"][i]) == e.contact_mask, (i, k)
        assert relerr(got["qvel"][i], e.qvel) < (TOL if k == 0 else 2e-4) and relerr(got["qpos"][i], e.qpos) < TOL, (i, k)
        ncon += e.ncon > 0
        ncmp += 1
    assert ncmp >= 30 and ncon > ncmp // 3, (ncmp, ncon)
    # env steps: stable PD with the gains and inertias of the env's own shape
    cfgs = [mk("uhc_pd", k, seed=9) for k in range(3)]
    kw2 = dict(seed=9, models=[model_from_cfg(c) for c, _ in cfgs], env_model=env_model)
    rng = np.random.default_rng(2)
    acts = [np.clip(rng.normal(size=(n, models[0].nu)) * 0.1, -1, 1) for _ in range(2)]

    def steps(env):
        out = [env.reset().cpu().numpy().copy()]
        for a in acts:
            out.append(torch.cat([x.float().reshape(n, -1) for x in env.step(t(a))], 1).cpu().numpy().copy())
        return out
    got2 = steps(_production(backend, monkeypatch, cfgs[0][0], n, 8, **kw2))
    one = _one_warp_same_envs(backend, monkeypatch, cfgs[0][0], n, **kw2)
    for s, (a, b) in enumerate(zip(got2, steps(one) if one is not None else [])):
        assert np.array_equal(a, b), (s, "8-warp vs 1-warp CTAs", np.flatnonzero((a != b).any(1))[:8])
    per = 8 * EPW
    sample = sorted(set(range(per)) | set(range(n - per, n)) | set(range(per, n - per, 61)))
    no = got2[0].shape[1]
    for i in sample:
        e = orc.OracleEnv(cfgs[env_model[i]][1], env_id=i)
        assert np.abs(got2[0][i] - e.reset()).max() < 1e-5, i
        for s in range(2):
            o, r, te, tr = e.step(acts[s][i])
            g = got2[s + 1][i]
            assert np.abs(g[:no] - o).max() < 5e-4 * (s + 1), (s, i, env_model[i], np.abs(g[:no] - o).max())
            assert abs(g[no] - r) < 5e-4 * (s + 1) and bool(g[no + 1]) == te and bool(g[no + 2]) == tr, (s, i)


# ------------------------------------------------------------------ 7. inverse dynamics, mass matrix / bias / Jacobians, kinematics
def test_inverse_dynamics_kinematics_at_production_shape(backend, monkeypatch):
    """Through an 8-warp handle: kinematics, mj_fullM / qfrc_bias / mj_jacBody and the inverse on num_envs + a few rows (the second
    launch is a ragged 8-warp grid), then the instances that read per-env parameter records.  Against the oracle (tolerances of
    test_dynamics / test_inverse; records: against one-env batches of each env's variant model, as test_env_params) and
    bit-identical with 1-warp CTAs."""
    from smplsim_b200.model import fk_numpy
    robot = "smpl_humanoid"
    cfg, om = make_models(robot=robot, control_mode="torque")
    m = om.model
    nenv, extra = N_DYN[backend.name]
    n = nenv + extra
    q, v, w, kinds, _, idx = _tiled(robot, n)
    keep = np.array([k != "bad" for k in kinds])
    v = np.where(keep[:, None], v, 0.0)
    P = len(q)
    qacc = np.random.default_rng(1).normal(size=(P, m.nv)) * 3.0
    jb = list(range(m.nbody))
    t = backend.t

    def run(env, s):
        tq, tv = t(q[idx[s]]), t(v[idx[s]])
        xp, xq = env.kinematics(tq)
        d = env.dynamics(tq, tv, jac_bodies=jb)
        inv, cw = env.inverse(tq, tv, t(qacc[idx[s]]), contact_wrench=True)
        return {"xpos": xp.cpu().numpy(), "xquat": xq.cpu().numpy(), "qM": d["qM"].cpu().numpy(),
                "bias": d["qfrc_bias"].cpu().numpy(), "jac": torch.cat([d["jacp"], d["jacr"]], 2).cpu().numpy(),
                "inv": inv.cpu().numpy(), "cw": cw.cpu().numpy()}

    env = _production(backend, monkeypatch, cfg, nenv, 8, ragged=False)
    assert extra % (8 * EPW) != 0
    got = run(env, slice(0, n))
    _bit_equal(got, _one_warp_chunks(backend, n, lambda s: backend.batch(cfg, 8), run), "8-warp vs 1-warp CTAs")
    _dups_equal(got, idx, "same pool state")
    wt = float(np.sum(m.body_mass)) * 9.81
    nwrench = 0
    for k in range(P):
        qk = np.float32(q[k]).astype(np.float64)
        e = orc.OracleEnv(om)
        e.qpos[:] = qk; e.qvel[:] = np.float32(v[k]); e.forward()
        ep, _, _ = fk_numpy(m, q[k])
        assert np.abs(got["xpos"][k] - ep).max() < 2e-5, k
        assert np.abs(got["qM"][k] - e.M).max() / np.abs(e.M).max() <= 2e-5, k
        assert np.abs(got["bias"][k] - e.qfrc_bias).max() / max(wt, float(np.abs(e.qfrc_bias).max())) <= 2e-5, k
        Jr = ref_jac(m, qk, e.xpos.copy(), e.xquat.copy())
        sc = np.abs(Jr).max(axis=1)
        assert float((np.abs(got["jac"][k] - Jr).max(axis=1)[sc > 0] / sc[sc > 0]).max()) <= 2e-5, k
        if e.nefc - 4 * e.ncon > 16:
            continue
        a = np.float32(qacc[k]).astype(np.float64)
        ref, f, r = ref_inverse(e, a)
        con = e.contacts()
        if (e.ncon and (np.abs(con["dist"] - m.margin) < 1e-5).any()) or (np.abs(r) < 1e-4 * np.abs(e.efc()["aref"])).any():
            continue
        assert np.abs(got["inv"][k] - ref).max() / max(wt, float(np.abs(ref).max())) <= 2e-3, k
        nc = e.ncon
        W = ref_wrench(m, con, f[e.nefc - 4 * nc:].reshape(nc, 4), e.xpos.copy(), e.xquat.copy())
        assert np.abs(got["cw"][k] - W).max() / max(wt, float(np.abs(W).max())) <= 2e-3, ("inverse contact wrench", k)
        if nc == 0:
            assert np.all(got["cw"][k] == 0.0), k
        nwrench += nc > 0
    assert nwrench >= P // 3, nwrench
    # the instances that read per-env parameter records (n == num_envs)
    prm = draw(m, P, 81)
    s = slice(0, nenv)

    def run_prm(env, s):
        env.set_env_params(**{k: t(x[idx[s]]) for k, x in prm.items()})
        out = run(env, s)
        return {k: out[k] for k in ("qM", "bias", "jac", "inv")}
    got = run_prm(env, s)
    _bit_equal(got, _one_warp_chunks(backend, nenv, lambda c: backend.batch(cfg, c.stop - c.start), run_prm), "records: 8-warp vs 1-warp CTAs")
    _dups_equal(got, idx[s], "records: same pool state")
    for k in range(min(P, 12)):
        one = backend.batch(cfg, 1, model=variant(m, prm, k))
        d = one.dynamics(t(q[k:k + 1]), t(v[k:k + 1]), jac_bodies=jb)
        Mr = d["qM"][0].cpu().numpy()
        assert np.abs(got["qM"][k] - Mr).max() / np.abs(Mr).max() < 2e-5, k
        wk = float(np.sum(m.body_mass * prm["body_mass_scale"][k]) * 9.81)
        assert np.abs(got["bias"][k] - d["qfrc_bias"][0].cpu().numpy()).max() / wk < 2e-5, k
        assert np.abs(got["jac"][k, :, :3] - d["jacp"][0].cpu().numpy()).max() < 2e-5, k
        assert np.abs(got["jac"][k, :, 3:] - d["jacr"][0].cpu().numpy()).max() < 2e-5, k
        ir = one.inverse(t(q[k:k + 1]), t(v[k:k + 1]), t(qacc[k:k + 1])).cpu().numpy()[0]
        assert np.abs(got["inv"][k] - ir).max() / max(1.0, np.abs(ir).max()) < 2e-5, k


# ------------------------------------------------------------------ a smaller handle next to a live 8-warp one
@pytest.mark.gpu_only
def test_smaller_handle_leaves_live_8_warp_handle_alone(backend, monkeypatch):
    """The kernels' dynamic shared-memory cap (cudaFuncSetAttribute) holds for the whole process.  Creating a 1-warp handle (8 envs)
    after an 8-warp one (4 001 envs) must leave every launch of the 8-warp handle working and its results unchanged: mj_step (with and
    without a wrench, with parameter records), reset, kinematics, dynamics and inverse, before and after the small handle runs."""
    robot = "smpl_humanoid"
    cfg, _ = make_models(robot=robot, control_mode="uhc_pd")
    m = model_from_cfg(cfg)
    n = N_SMPL[backend.name]
    q, v, w, kinds, ctrl, idx = _tiled(robot, n)
    q, v, w, ctrl = q[idx], v[idx], w[idx], ctrl[idx]
    xf = np.zeros((n, m.nbody, 6)); xf[::2, :, 2] = 5.0
    prm = draw(m, n, 5)
    t = backend.t
    big = _production(backend, monkeypatch, cfg, n, 8, contact_wrench=True)

    def run():
        out = {}
        big.clear_env_params()
        for x in (big.rng_counter, big.progress_buf, big.task_change_step, big.task_target):   # the reset's task draw starts over
            x.zero_()
        big.reset()
        out["reset"] = big.obs_buf.cpu().numpy().copy()
        for tag, wrench, records in (("plain", None, False), ("xfrc", xf, False), ("records", xf, True)):
            if records:
                big.set_env_params(**{k: t(x) for k, x in prm.items()})
            big.xfrc_applied = None if wrench is None else t(wrench)
            big.set_state(t(q), t(v))
            big.qacc_warm.copy_(t(w))
            big.mj_step(t(ctrl), 1)
            out.update({f"{tag}_{k}": x for k, x in _outs(big).items()})
        big.xfrc_applied = None
        xp, _ = big.kinematics(t(q))
        d = big.dynamics(t(q), t(v), jac_bodies=[0, 5])
        out["xpos"] = xp.cpu().numpy()
        out["qM"] = d["qM"].cpu().numpy()
        out["inv"] = big.inverse(t(q), t(v), t(w)).cpu().numpy()
        return out

    before = run()
    small = backend.batch(cfg, 8)
    assert _wpb(small) == 1
    small.reset()
    small.step(t(np.zeros((8, m.nu))))
    _bit_equal(run(), before, "8-warp handle after a 1-warp handle was created")
