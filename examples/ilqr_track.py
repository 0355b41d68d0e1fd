"""iLQR tracking on SMPL with closed-loop rollouts: track the trajectory of one open-loop control sequence by optimising another.

Ctrl mode with nsub = 1, so that every rollout step is the one mj_step that transition_fd linearises and its A and B describe
exactly the step being rolled out.  Each iteration is

  1. one transition_fd call on the nominal's T pre-step states;
  2. a Riccati backward pass in torch fp64 (the gains K_t and the feedforward steps k_t);
  3. one rollout(gains=K) launch whose rows are the line-search step sizes alpha in {0, 1/4, 1/2, 1}: row j applies
     u_t = ubar_t + alpha_j k_t + K_t (x_t (-) xbar_t), every row sharing K and the nominal xbar;
  4. the row of least cost, with its states and its applied "control", becomes the next nominal.

The alpha = 0 row reproduces the nominal bit for bit, so the cost never rises.  No data files: the target comes from the model.

    python examples/ilqr_track.py --iters 5 --T 30
"""
from __future__ import annotations

import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from smplsim_b200.batched import HumanoidBatchB200  # noqa: E402
from smplsim_b200.cfg import make_cfg  # noqa: E402

ALPHAS = (0.0, 0.25, 0.5, 1.0)
W_POS, W_VEL, R_CTRL, MU = 1e2, 1.0, 1e-4, 1e-1   # state and control weights, Quu regularisation


def make_problem(env: HumanoidBatchB200, T: int = 30, seed: int = 0):
    """Start state (an env after reset), the target trajectory (an open-loop run of random torques) and the first nominal's
    controls (the target's, scaled down)."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    m = env.model
    env.reset()
    q0, v0 = env.qpos[:1].clone(), env.qvel[:1].clone()
    u_tgt = (torch.randn(1, T, m.nu, generator=g) * 20.0).to(env.device)
    tgt = env.rollout(q0, v0, u_tgt, mode="ctrl", nsub=1)
    return {"q0": q0, "v0": v0, "T": T, "qpos_tgt": tgt["qpos"][0].double(), "qvel_tgt": tgt["qvel"][0].double(), "u0": 0.3 * u_tgt[0]}


def _dev(env, prob, qpos, qvel):
    """Tangent deviation [T, 2nv] of post-step states from the target (fp64)."""
    return torch.cat([env.differentiate_pos(prob["qpos_tgt"], qpos.double()), qvel.double() - prob["qvel_tgt"]], -1)


def _cost(env, prob, qpos, qvel, u):
    nv = env.model.nv
    e = _dev(env, prob, qpos, qvel)
    return float(0.5 * (W_POS * (e[:, :nv] ** 2).sum() + W_VEL * (e[:, nv:] ** 2).sum() + R_CTRL * (u.double() ** 2).sum()))


def nominal(env: HumanoidBatchB200, prob):
    """The first nominal: an open-loop rollout of the problem's initial controls."""
    out = env.rollout(prob["q0"], prob["v0"], prob["u0"][None].contiguous(), mode="ctrl", nsub=1)
    nom = {k: out[k] for k in ("qpos", "qvel", "status")}
    nom["control"] = prob["u0"][None].contiguous()
    nom["cost"] = _cost(env, prob, out["qpos"][0], out["qvel"][0], prob["u0"])
    return nom


def backward(env: HumanoidBatchB200, prob, nom):
    """transition_fd on the nominal's pre-step states and the Riccati pass: (K [T, nu, 2nv], k [T, nu]) in fp64, and the pre-step
    states (qpos [T, nq], qvel [T, nv]) they are written around."""
    m, T = env.model, prob["T"]
    nv, nu = m.nv, m.nu
    qs = torch.cat([prob["q0"], nom["qpos"][0, :-1]])          # pre-step states x_t, t = 0 .. T-1
    vs = torch.cat([prob["v0"], nom["qvel"][0, :-1]])
    ub = nom["control"][0]
    fd = env.transition_fd(qs, vs, ub)
    A, B = fd["A"].double(), fd["B"].double()
    # backward pass: stage cost 1/2 r |u_t|^2, state cost 1/2 e^T W e on the post-step states x_1 .. x_T
    w = torch.cat([torch.full((nv,), W_POS), torch.full((nv,), W_VEL)]).double().to(A.device)
    e = _dev(env, prob, nom["qpos"][0], nom["qvel"][0])
    Vx, Vxx = w * e[T - 1], torch.diag(w)
    K = torch.zeros(T, nu, 2 * nv, dtype=torch.float64, device=A.device)
    k = torch.zeros(T, nu, dtype=torch.float64, device=A.device)
    I = torch.eye(nu, dtype=torch.float64, device=A.device)
    for t in range(T - 1, -1, -1):
        At, Bt = A[t], B[t]
        Qx, Qu = At.T @ Vx, R_CTRL * ub[t].double() + Bt.T @ Vx
        Qxx, Quu, Qux = At.T @ Vxx @ At, R_CTRL * I + Bt.T @ Vxx @ Bt + MU * I, Bt.T @ Vxx @ At
        L = torch.linalg.cholesky(0.5 * (Quu + Quu.T))
        k[t] = -torch.cholesky_solve(Qu[:, None], L)[:, 0]
        K[t] = -torch.cholesky_solve(Qux, L)
        Vx = Qx + K[t].T @ Quu @ k[t] + K[t].T @ Qu + Qux.T @ k[t]
        Vxx = Qxx + K[t].T @ Quu @ K[t] + K[t].T @ Qux + Qux.T @ K[t]
        Vxx = 0.5 * (Vxx + Vxx.T)
        if t > 0:
            Vx, Vxx = Vx + w * e[t - 1], Vxx + torch.diag(w)
    return K, k, qs, vs


def iteration(env: HumanoidBatchB200, prob, nom):
    """One iLQR iteration from nominal `nom`; returns every line-search row, the best cost and the next nominal."""
    K, k, qs, vs = backward(env, prob, nom)
    ub = nom["control"][0]
    # forward pass: the line-search rows in one closed-loop launch
    n = len(ALPHAS)
    al = torch.tensor(ALPHAS, dtype=torch.float32, device=ub.device)[:, None, None]
    ubar = (ub[None] + al * k.float()[None]).contiguous()
    out = env.rollout(prob["q0"].expand(n, -1).contiguous(), prob["v0"].expand(n, -1).contiguous(), ubar, mode="ctrl", nsub=1,
                      gains=K.float()[None].contiguous(), qpos_ref=qs[None].contiguous(), qvel_ref=vs[None].contiguous())
    rows = [{key: out[key][j:j + 1] for key in ("qpos", "qvel", "status", "control")} for j in range(n)]
    costs = [_cost(env, prob, r["qpos"][0], r["qvel"][0], r["control"][0]) for r in rows]
    j = min(range(n), key=lambda i: costs[i])
    best = dict(rows[j], cost=costs[j])
    return {"rows": rows, "costs": costs, "best_cost": costs[j], "alpha": ALPHAS[j], "next": best}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--T", type=int, default=30)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    cfg = make_cfg(env="speed", robot="smpl_humanoid", overrides={"env.control_mode": "torque"})
    env = HumanoidBatchB200(cfg, num_envs=len(ALPHAS), seed=args.seed)
    prob = make_problem(env, T=args.T, seed=args.seed)
    nom = nominal(env, prob)
    print(f"iter 0  cost {nom['cost']:.6e}")
    for i in range(1, args.iters + 1):
        it = iteration(env, prob, nom)
        nom = it["next"]
        print(f"iter {i}  cost {it['best_cost']:.6e}  alpha {it['alpha']}  line search " + " ".join(f"{c:.3e}" for c in it["costs"]))


if __name__ == "__main__":
    main()
