#!/usr/bin/env python
"""PPO on the GPU stepper -- the loop of smpl_sim/run.py (AgentHumanoid.optimize_policy: sample -> update_params -> log) with
the batched pieces of this repo: HumanoidBatchB200 (env shard on this GPU), BatchedSampler (device-resident rollout),
smplsim_gae (advantages), PPOLearner (AgentPPO.update_params semantics, gradients / moments all-reduced over ranks).

    python examples/train_ppo.py --env speed --num-envs 4096 --horizon 16 --epochs 5
    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 examples/train_ppo.py --env getup
    python examples/train_ppo.py --env im --num-envs 4096      # motion imitation (HumanoidImB200) on synthetic clips
    python examples/train_ppo.py --env im --amp                # ... plus the AMP style reward (HumanoidAmpB200, AMPLearner)
    python examples/train_ppo.py --env im --eval-every 5 --auto-pmcp hard   # score every clip every 5 epochs, train on the failed ones

``--horizon x --num-envs`` plays the role of ``learning.min_batch_size`` (51 200 in the reference yaml = 4096 envs x 12.5 steps)."""
import argparse
import os
import sys
import time

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from smplsim_b200.batched import HumanoidBatchB200  # noqa: E402
from smplsim_b200.cfg import make_cfg  # noqa: E402
from smplsim_b200.dist import max_over_ranks, rank_seed  # noqa: E402
from smplsim_b200.learning import BatchedSampler  # noqa: E402
from smplsim_b200.ppo import PolicyGaussian, PPOLearner, Value  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--env", default="speed", choices=["speed", "reach", "getup", "im"])
    ap.add_argument("--num-envs", type=int, default=4096, help="envs on THIS GPU")
    ap.add_argument("--horizon", type=int, default=16)
    ap.add_argument("--epochs", type=int, default=5)
    ap.add_argument("--units", type=int, nargs="+", default=[2048, 1536, 1024, 1024, 512, 512])   # data/cfg/learning/simple_mlp.yaml
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--amp", action="store_true", help="adversarial motion priors: discriminator reward mixed into the task reward")
    ap.add_argument("--eval-every", type=int, default=0, help="--env im: evaluate the mean policy on every clip every E epochs (0: never)")
    ap.add_argument("--auto-pmcp", default="off", choices=["off", "hard", "soft"],
                    help="after each evaluation, sample training clips from the failed ones (the reference's auto_pmcp / auto_pmcp_soft)")
    a = ap.parse_args()
    if (a.eval_every or a.auto_pmcp != "off") and (a.env != "im" or a.amp):
        ap.error("--eval-every / --auto-pmcp need --env im without --amp")
    rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dev = f"cuda:{local}"
    if world > 1:
        torch.distributed.init_process_group("nccl", device_id=torch.device(dev))
    torch.manual_seed(a.seed)                         # identical initial weights on every rank
    if a.env == "im":     # every env tracks a clip of the library; the synthetic clips stand in for an AMASS table (motion_loader.py)
        from smplsim_b200.imitation import HumanoidImB200
        from smplsim_b200.motion_lib import synthetic_tables
        env = HumanoidImB200(make_cfg(env="im"), lambda b: synthetic_tables(b, num_clips=64, frames=300), num_envs=a.num_envs, device=dev,
                             seed=a.seed, rank=rank)
    else:
        env = HumanoidBatchB200(make_cfg(env=a.env), num_envs=a.num_envs, device=dev, seed=a.seed, rank=rank, with_aux=a.amp)
    amp_learner = None
    if a.amp:             # the demonstrations: the imitation env's library, or synthetic clips for the other tasks
        from smplsim_b200.amp import HumanoidAmpB200
        from smplsim_b200.motion_lib import MotionLibB200, synthetic_tables
        lib = None if a.env == "im" else MotionLibB200(env, synthetic_tables(env, num_clips=64, frames=300))
        env = HumanoidAmpB200(env, lib)
        amp_learner = env.make_learner()
    policy = PolicyGaussian(env.num_obs, env.num_actions, a.units, "silu", -2.5, True).to(dev)
    value = Value(env.num_obs, a.units, "silu").to(dev)
    learner = PPOLearner(policy, value)               # gamma .99, tau .95, clip .2, 10 epochs, lr 5e-5 / 3e-4, grad clip 25
    gen = torch.Generator(device=dev); gen.manual_seed(rank_seed(a.seed, rank))

    def act(obs):
        policy.eval()                                 # to_test during sampling: RunningNorm frozen (agents/agent.py:123)
        return policy.select_action(obs, generator=gen)

    sampler = BatchedSampler(env, act)
    for ep in range(a.epochs):
        t0 = time.time()
        batch = sampler.sample(a.horizon)
        torch.cuda.synchronize(); t1 = time.time()
        info = learner.update(batch)
        if amp_learner is not None:
            info.update(amp_learner.update(env.drain_amp_obs()))
        torch.cuda.synchronize(); t2 = time.time()
        ts, tu = max_over_ranks(t1 - t0, dev), max_over_ranks(t2 - t1, dev)
        if rank == 0:
            n = a.horizon * a.num_envs * world
            print(f"epoch {ep}: {n} samples  sample {ts:.2f}s ({n / ts / 1e3:.0f}k env-steps/s)  update {tu:.2f}s  "
                  f"reward {info['mean_reward']:.4f}  policy_loss {info['policy_loss']:.4f}  value_loss {info['value_loss']:.4f}", flush=True)
            if amp_learner is not None:
                print(f"  amp: task reward {float(env.extras['task_rew_buf'].mean()):.4f}  disc reward {float(env.disc_rew_buf.mean()):.4f}  "
                      f"disc_loss {info['disc_loss']:.4f}  acc agent {info['disc_agent_acc']:.3f} demo {info['disc_demo_acc']:.3f}", flush=True)
        if a.eval_every and (ep + 1) % a.eval_every == 0:
            with torch.no_grad():
                policy.eval()
                res = env.evaluate(lambda obs: policy.select_action(torch.clamp(obs, -5.0, 5.0), mean_action=True))
            sampler.restart()                         # evaluate left every env flagged for reset
            if a.auto_pmcp == "hard":
                env.lib.update_hard_sampling_weight(res.failed_keys)
            elif a.auto_pmcp == "soft":
                env.lib.update_soft_sampling_weight(res.failed_keys)
            if rank == 0:
                s = res.summary()
                print(f"  eval: {s['num_clips']} clips, {s['frames']} frames, success {s['success_rate']:.3f}, failed clips "
                      f"{len(res.failed_keys)}  mpjpe_g {s['mpjpe_g']:.1f} mm  mpjpe_l {s['mpjpe_l']:.1f} mm  mpjpe_pa {s['mpjpe_pa']:.1f} mm  "
                      f"vel {s['vel_dist']:.2f}  accel {s['accel_dist']:.2f}  rot {s['rot_error']:.3f} rad  (pmcp: {a.auto_pmcp})", flush=True)
    if world > 1:
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
