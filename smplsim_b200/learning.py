"""GPU-side pieces of the PPO update that sit right after the hot path (SURVEY.md 8 f1/f2): a batched on-device sampler
replacing ``Agent.sample / sample_worker`` (smpl_sim/agents/agent.py:64-145: N OS processes, batch-1 policy forward on the
CPU, Python ``Memory.push``) and ``estimate_advantages`` (smpl_sim/learning/learning_utils.py:198-218: a Python loop over
51 200 samples on the CPU) as a CUDA reverse scan.  The learner itself (``AgentPPO.update_policy``) stays PyTorch."""
from __future__ import annotations

import ctypes as C
from typing import Callable, Dict, Optional

import torch

from . import _lib
from .dist import global_moments


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def estimate_advantages(rewards, not_done, not_dead, values, gamma: float, tau: float, next_value: Optional[torch.Tensor] = None,
                        normalize: bool = True):
    """[T,N] float32 CUDA tensors -> (advantages, returns), same recursion as the reference; normalisation uses the mean and the
    *unbiased* std (torch's default, as in learning_utils.py:215) over the whole batch of all ranks."""
    T, N = rewards.shape
    f = lambda t: t.to(torch.float32).contiguous()  # noqa: E731
    rewards, not_done, not_dead, values = f(rewards), f(not_done), f(not_dead), f(values)
    adv = torch.empty_like(rewards)
    ret = torch.empty_like(rewards)
    nv = None if next_value is None else f(next_value)
    _lib.check(_lib.lib().smplsim_gae(_p(rewards), _p(not_done), _p(not_dead), _p(values), _p(nv), float(gamma), float(tau), T, N,
                                      _p(adv), _p(ret), C.c_void_p(torch.cuda.current_stream(rewards.device).cuda_stream)))
    if normalize:
        mean, std_pop, n = global_moments(adv, with_count=True)       # n: elements over ALL ranks (shards may be uneven)
        std = std_pop * (n / max(n - 1.0, 1.0)) ** 0.5
        adv = (adv - mean) / std
    return adv, ret


class BatchedSampler:
    """Collect ``horizon`` steps from all N envs on the device.

    ``policy(obs[N,D]) -> action[N,A]`` is any callable on CUDA tensors (e.g. ``lambda o: policy_net.select_action(o, mean_action)``).
    Pre/post-processing follows Agent.preprocess_obs / preprocess_actions (agents/agent.py:147-161): observations clipped to
    +-obs_clip (5); the env receives the action clipped to [-1, 1] while the RAW sampled action is what the batch records
    (agent.py:81-93, "action processing should not affect the recorded action": the PPO ratio needs the density the action was
    drawn from).  Envs that terminate or time out are reset in-stream (masked reset kernel).  Pinned against a trajectory
    recorded by the reference's own Agent.sample_worker + Memory / TrajBatch (tests/golden/sampler.npz, tests/test_sampler_cpu.py)."""

    def __init__(self, env, policy: Callable[[torch.Tensor], torch.Tensor], obs_clip: float = 5.0):
        self.env = env
        self.policy = policy
        self.obs_clip = obs_clip
        self._obs = None

    def restart(self):
        """Forget the cached observation: the next ``sample`` starts with ``env.reset()`` (after the env was used elsewhere, e.g. by
        ``HumanoidImB200.evaluate``)."""
        self._obs = None

    def _pre(self, obs):
        return torch.clamp(obs, -self.obs_clip, self.obs_clip) if self.obs_clip else obs

    @torch.no_grad()
    def sample(self, horizon: int) -> Dict[str, torch.Tensor]:
        env = self.env
        N, D, A, dv = env.num_envs, env.num_obs, env.num_actions, env.device
        if self._obs is None:
            self._obs = self._pre(env.reset()).clone()
        out = dict(states=torch.empty(horizon, N, D, device=dv), actions=torch.empty(horizon, N, A, device=dv),
                   rewards=torch.empty(horizon, N, device=dv), not_done=torch.empty(horizon, N, device=dv),
                   not_dead=torch.empty(horizon, N, device=dv), next_states=torch.empty(horizon, N, D, device=dv))
        for t in range(horizon):
            a_raw = self.policy(self._obs)
            out["states"][t] = self._obs
            out["actions"][t] = a_raw
            obs, rew, term, trunc = env.step(torch.clamp(a_raw, -1.0, 1.0))
            out["rewards"][t] = rew
            out["not_dead"][t] = 1.0 - term.float()
            out["not_done"][t] = 1.0 - env.reset_buf.float()
            out["next_states"][t] = self._pre(obs)
            env.reset_done()                       # obs_buf rows of reset envs now hold the post-reset observation
            self._obs = self._pre(env.obs_buf).clone()
        out["last_obs"] = self._obs
        return out
