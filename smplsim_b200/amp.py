"""Adversarial motion priors (AMP, Peng et al. 2021) on the batched tensor protocol.

The reference trains imitation with ``algo: im_amp`` / ``model: amp``: a discriminator tells the agent's last K control steps from
motion-library clips, and its output is a style reward mixed into the task reward.  Here the observation side is one CUDA kernel
(``smplsim_amp_obs`` / ``smplsim_amp_demo``, csrc/amp_kernels.cuh): the per-env history is pushed in place after every step and filled at
resets, and demonstration rows are read from the library's tables on demand, so no demo buffer is kept.  The per-frame feature is the
reference's ``compute_humanoid_observations_smpl`` (stated in include/smplsim.h).  The discriminator and its update are PyTorch.

- ``HumanoidAmpB200`` wraps a ``HumanoidBatchB200`` (speed / reach / getup / none, ``with_aux=True``) or a ``HumanoidImB200`` and keeps
  their tensor protocol, so ``BatchedSampler`` and ``GymVectEnvB200`` take it unchanged.
- ``AMPDiscriminator`` / ``AMPLearner``: the discriminator loss, its regularisers, the replay buffer of agent rows and the input
  normalisation, with gradients and moments reduced over ranks as ``PPOLearner`` does.
- ``AMP_DEFAULTS``: the reference's values."""
from __future__ import annotations

import ctypes as C
from typing import Any, Callable, Dict, Optional

import numpy as np
import torch
import torch.nn as nn

from .abi import AMP_FILL, AMP_FILL_REF, AMP_PUSH, SmplsimAmpCfgC
from .batched import _ptr
from .dist import allreduce_mean_grads
from .ppo import MLP, RunningNorm, _dist_on

# smpl_sim/envs/nv/data/cfg/phc_prim_iccv.yaml (every PHC env config sets the same four) and train/rlg/im.yaml
AMP_DEFAULTS: Dict[str, Any] = dict(
    num_amp_obs_steps=10,                                   # phc_prim_iccv.yaml:49  numAMPObsSteps
    local_root_obs=True,                                    # phc_prim_iccv.yaml:51  localRootObs
    root_height_obs=True,                                   # phc_prim_iccv.yaml:52  rootHeightObs
    key_bodies=["R_Ankle", "L_Ankle", "R_Wrist", "L_Wrist"],  # phc_prim_iccv.yaml:53  keyBodies
    interpolate=False,                                      # this project's: demo / MoCap-reset frames blended as get_motion_state
    disc_units=[1024, 512],                                 # im.yaml:38  network.disc.units
    disc_activation="relu",                                 # im.yaml:39  network.disc.activation
    lr=2e-5,                                                # im.yaml:59  learning_rate
    amp_replay_buffer_size=200000,                          # im.yaml:80
    amp_replay_keep_prob=0.01,                              # im.yaml:81
    amp_minibatch_size=4096,                                # im.yaml:83
    disc_coef=5.0,                                          # im.yaml:84
    disc_logit_reg=0.01,                                    # im.yaml:85
    disc_grad_penalty=5.0,                                  # im.yaml:86
    disc_reward_scale=2.0,                                  # im.yaml:87
    disc_weight_decay=1e-4,                                 # im.yaml:88
    normalize_amp_input=True,                               # im.yaml:89
    task_reward_w=0.5,                                      # im.yaml:91
    disc_reward_w=0.5,                                      # im.yaml:92
)


def amp_config(amp_cfg: Optional[Dict[str, Any]] = None) -> Dict[str, Any]:
    """``AMP_DEFAULTS`` updated with the caller's keys (unknown keys are refused)."""
    c = dict(AMP_DEFAULTS)
    for k, v in (amp_cfg or {}).items():
        if k not in AMP_DEFAULTS:
            raise ValueError(f"unknown AMP key {k!r} (have {sorted(AMP_DEFAULTS)})")
        c[k] = v
    return c


def amp_c_cfg(model, amp_cfg: Dict[str, Any]):
    """The ``SmplsimAmpCfg`` of a config, and the key-body array it points at (keep both alive while the struct is used)."""
    keys = [model.body_index(x, "key_bodies entries must be body names or indices", kind="key body") for x in amp_cfg["key_bodies"]]
    arr = np.ascontiguousarray(np.asarray(keys, dtype=np.int32))
    c = SmplsimAmpCfgC(num_steps=int(amp_cfg["num_amp_obs_steps"]), num_key_bodies=len(keys), key_bodies=arr.ctypes.data if keys else None,
                       local_root_obs=int(bool(amp_cfg["local_root_obs"])), root_height_obs=int(bool(amp_cfg["root_height_obs"])),
                       interpolate=int(bool(amp_cfg["interpolate"])))
    return c, arr


# ------------------------------------------------------------------ discriminator
class AMPDiscriminator(nn.Module):
    """``D(x)``: input normalisation (``normalize_amp_input``: running mean / std of agent and demo rows, clipped to +-5) -> ``activation``
    MLP -> one logit.  The normalisation moments change only in ``AMPLearner.update``; the forward never updates them and never
    synchronises with the host."""

    def __init__(self, input_dim: int, units=(1024, 512), activation: str = "relu", normalize: bool = True):
        super().__init__()
        self.input_dim = int(input_dim)
        self.norm = RunningNorm(self.input_dim, clip=5.0) if normalize else None
        self.register_buffer("norm_ready", torch.zeros((), dtype=torch.bool))   # set by the first moment update
        self.mlp = MLP(self.input_dim, list(units), activation)
        self.logits = nn.Linear(self.mlp.out_dim, 1)
        with torch.no_grad():                    # the AMP discriminator's logit initialisation: U(-1, 1) weights, zero bias
            self.logits.weight.uniform_(-1.0, 1.0)
            self.logits.bias.zero_()

    def normalize(self, x: torch.Tensor) -> torch.Tensor:
        if self.norm is None:
            return x
        y = ((x - self.norm.mean) / (self.norm.std + 1e-8)).clamp(-5.0, 5.0)
        return torch.where(self.norm_ready, y, x)

    @torch.no_grad()
    def update_norm(self, x: torch.Tensor):
        if self.norm is not None:
            self.norm.update(x)
            self.norm_ready.fill_(True)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self.logits(self.mlp(self.normalize(x)))

    def weights(self):
        """The linear weights the weight decay acts on (every layer, logits included)."""
        return [m.weight for m in self.mlp.affine_layers] + [self.logits.weight]

    @torch.no_grad()
    def reward(self, x: torch.Tensor, scale: float = 2.0) -> torch.Tensor:
        """``-log(max(1 - sigmoid(D(x)), 1e-4)) * scale`` per row of ``x [M, input_dim]``: ``[M]``."""
        prob = torch.sigmoid(self.forward(x)).squeeze(-1)
        return -torch.log(torch.clamp(1.0 - prob, min=1e-4)) * scale


def disc_loss_terms(disc: AMPDiscriminator, agent: torch.Tensor, demo: torch.Tensor) -> Dict[str, torch.Tensor]:
    """The AMP discriminator objective on one minibatch (inputs before normalisation): binary cross-entropy with agent rows -> 0 and demo
    rows -> 1 (the mean of the two), the squared logit weights, the gradient penalty ``mean |dD/dx|^2`` on the demo rows (taken with
    respect to the normalised input, as the reference's discriminator sees it) and the squared weights of every layer.  Also the
    logits and the accuracies."""
    agent_in = disc.normalize(agent)
    demo_in = disc.normalize(demo).detach().requires_grad_(True)
    la = disc.logits(disc.mlp(agent_in))
    ld = disc.logits(disc.mlp(demo_in))
    bce = nn.functional.binary_cross_entropy_with_logits
    loss = 0.5 * (bce(la, torch.zeros_like(la)) + bce(ld, torch.ones_like(ld)))
    logit_reg = torch.sum(disc.logits.weight ** 2)
    g = torch.autograd.grad(ld, demo_in, grad_outputs=torch.ones_like(ld), create_graph=True, retain_graph=True, only_inputs=True)[0]
    grad_penalty = torch.mean(torch.sum(g * g, dim=-1))
    weight_decay = sum(torch.sum(w ** 2) for w in disc.weights())
    return dict(loss=loss, logit_reg=logit_reg, grad_penalty=grad_penalty, weight_decay=weight_decay, agent_logit=la.detach(),
                demo_logit=ld.detach(), agent_acc=(la.detach() < 0).float().mean(), demo_acc=(ld.detach() > 0).float().mean())


def disc_total_loss(terms: Dict[str, torch.Tensor], c: Dict[str, Any]) -> torch.Tensor:
    return c["disc_coef"] * (terms["loss"] + c["disc_logit_reg"] * terms["logit_reg"] + c["disc_grad_penalty"] * terms["grad_penalty"]
                             + c["disc_weight_decay"] * terms["weight_decay"])


class AMPReplayBuffer:
    """Agent AMP rows of earlier updates (a ring of ``size`` rows on the device).  While fewer than ``size`` rows were ever stored every row
    goes in; after that each row is kept with probability ``keep_prob``.  When more rows come than fit, a random ``size`` of them."""

    def __init__(self, size: int, dim: int, keep_prob: float, device, generator: Optional[torch.Generator] = None,
                 dtype: torch.dtype = torch.float32):
        self.size, self.keep_prob = int(size), float(keep_prob)
        self.buf = torch.zeros(self.size, dim, device=device, dtype=dtype)
        self.head = 0            # next row written
        self.count = 0           # rows holding data (<= size)
        self.total = 0           # rows ever stored
        self.gen = generator

    def store(self, x: torch.Tensor):
        if self.total > self.size:
            keep = torch.rand(x.shape[0], device=x.device, generator=self.gen) < self.keep_prob
            x = x[keep]
        if x.shape[0] > self.size:
            x = x[torch.randperm(x.shape[0], device=x.device, generator=self.gen)[: self.size]]
        n = x.shape[0]
        if n == 0:
            return
        idx = (self.head + torch.arange(n, device=x.device)) % self.size
        self.buf[idx] = x
        self.head = (self.head + n) % self.size
        self.count = min(self.count + n, self.size)
        self.total += n

    def sample(self, n: int) -> torch.Tensor:
        idx = torch.randint(0, self.count, (int(n),), device=self.buf.device, generator=self.gen)
        return self.buf[idx]


class AMPLearner:
    """Discriminator updates.  ``update(agent_amp_obs)`` takes the agent rows of a rollout (``[..., K * F]``, e.g. what
    ``HumanoidAmpB200.drain_amp_obs`` returns), shuffles them into minibatches of ``amp_minibatch_size`` rows, each half fresh rows and
    half replay rows (fresh rows only while the replay buffer is empty), draws as many demonstration rows from ``demo(n)`` (default the
    library's ``amp_obs_demo``), merges both into the input moments, and takes one Adam step on ``disc_total_loss`` per minibatch.  Then
    the fresh rows go into the replay buffer.  Under ``torch.distributed`` the gradients are averaged and the input moments are those of
    all ranks' rows."""

    def __init__(self, disc: AMPDiscriminator, demo: Callable[[int], torch.Tensor], amp_cfg: Optional[Dict[str, Any]] = None,
                 generator: Optional[torch.Generator] = None):
        self.disc, self.demo, self.cfg = disc, demo, amp_config(amp_cfg)
        p0 = next(disc.parameters())
        self.gen = generator
        self.optimizer = torch.optim.Adam(disc.parameters(), lr=float(self.cfg["lr"]), eps=1e-8)
        self.replay = AMPReplayBuffer(self.cfg["amp_replay_buffer_size"], disc.input_dim, self.cfg["amp_replay_keep_prob"], p0.device,
                                     generator, p0.dtype)

    def update(self, agent_amp_obs: torch.Tensor) -> Dict[str, float]:
        c, disc = self.cfg, self.disc
        x = agent_amp_obs.reshape(-1, disc.input_dim)
        n = x.shape[0]
        mb = max(1, int(c["amp_minibatch_size"]))
        perm = torch.randperm(n, device=x.device, generator=self.gen)
        acc = {k: 0.0 for k in ("disc_loss", "disc_agent_acc", "disc_demo_acc", "disc_grad_penalty", "disc_logit_reg")}
        steps = 0
        disc.train()
        for i in range(0, n, mb):
            fresh = x[perm[i:i + mb]]
            if self.replay.count > 0:
                h = max(1, fresh.shape[0] // 2)
                agent = torch.cat([fresh[:h], self.replay.sample(fresh.shape[0] - h)])
            else:
                agent = fresh
            demo = self.demo(agent.shape[0])
            disc.update_norm(torch.cat([agent, demo]))
            terms = disc_loss_terms(disc, agent, demo)
            loss = disc_total_loss(terms, c)
            self.optimizer.zero_grad()
            loss.backward()
            if _dist_on():
                allreduce_mean_grads(disc.parameters())
            self.optimizer.step()
            steps += 1
            acc["disc_loss"] += float(loss.detach())
            acc["disc_agent_acc"] += float(terms["agent_acc"])
            acc["disc_demo_acc"] += float(terms["demo_acc"])
            acc["disc_grad_penalty"] += float(terms["grad_penalty"].detach())
            acc["disc_logit_reg"] += float(terms["logit_reg"].detach())
        disc.eval()
        self.replay.store(x.detach())
        return {k: v / max(steps, 1) for k, v in acc.items()}


# ------------------------------------------------------------------ env wrapper
class HumanoidAmpB200:
    """An env with its AMP observation history.  ``env``: a ``HumanoidBatchB200`` (speed / reach / getup / none, built with
    ``with_aux=True``) or a ``HumanoidImB200``.  ``motion_lib``: the ``MotionLibB200`` demonstrations come from (default: the imitation
    env's own library).  ``amp_cfg``: keys of ``AMP_DEFAULTS`` to override.  ``discriminator``: an ``AMPDiscriminator`` (or None: no style
    reward; it can be attached later by setting ``.discriminator``).

    The tensor protocol of the wrapped env (``num_envs, num_obs, num_actions, device, obs_buf, rew_buf, terminate_buf, truncate_buf,
    reset_buf, progress_buf, extras, step, reset, reset_done``), plus ``amp_obs_buf [N, K, F]`` (newest frame first) and
    ``amp_obs [N, K * F]`` (a view of it, the discriminator's input).

    - ``step(actions)``: the env's step, then the history push.  With a discriminator ``rew_buf = task_reward_w * task +
      disc_reward_w * r_d``; ``extras["task_rew_buf"]`` / ``extras["disc_rew_buf"]`` hold the two parts.  The step's AMP rows (before any
      reset) are kept for ``drain_amp_obs``.  In stream order, no host sync.
    - ``reset(env_ids, ...)`` / ``reset_done()``: the env's reset, then the history of the same envs filled: the current frame in every
      slot, or for an imitation env the current frame and the clip's frames behind the reset time (MoCap init).  With an imitation env's
      fail-state recovery on, by ``reset_kind``: MoCap envs from the clip, fall envs from their state, recovery envs untouched (their state
      and history continue)."""

    def __init__(self, env, motion_lib=None, amp_cfg: Optional[Dict[str, Any]] = None, discriminator: Optional[AMPDiscriminator] = None):
        from .imitation import HumanoidImB200
        self.env = env
        self.imitation = isinstance(env, HumanoidImB200)
        self.batch = env.batch if self.imitation else env
        self.lib = motion_lib if motion_lib is not None else (env.lib if self.imitation else None)
        b = self.batch
        if b._aux.xpos is None or b._aux.xquat is None:
            raise ValueError("HumanoidAmpB200 needs the batch's body poses (HumanoidBatchB200(..., with_aux=True))")
        # an imitation env's frame rule carries over to its AMP frames unless the caller sets the key
        self.cfg = amp_config(dict({"interpolate": env.interpolate} if self.imitation else {}, **(amp_cfg or {})))
        self.num_envs, self.num_actions, self.device = env.num_envs, env.num_actions, env.device
        self.dt, self.max_episode_length = env.dt, env.max_episode_length
        self._ccfg, self._keys = amp_c_cfg(b.model, self.cfg)
        F = b._L().smplsim_amp_obs_dim(b._h, C.byref(self._ccfg))
        if F < 0:
            b._check(F)
        self.num_amp_obs_steps, self.amp_frame_dim = int(self.cfg["num_amp_obs_steps"]), F
        self.num_amp_obs = self.num_amp_obs_steps * F
        self.amp_obs_buf = torch.zeros(self.num_envs, self.num_amp_obs_steps, F, dtype=torch.float32, device=self.device)
        self.amp_obs = self.amp_obs_buf.view(self.num_envs, self.num_amp_obs)
        if self.lib is not None:
            self.lib.set_amp_cfg(self.cfg)
        self._tab = self.lib._amp_tables() if self.lib is not None else None
        self.discriminator = discriminator
        self._rew = torch.zeros(self.num_envs, dtype=torch.float32, device=self.device)
        self.disc_rew_buf = torch.zeros(self.num_envs, dtype=torch.float32, device=self.device)
        self.extras = dict(env.extras)
        self.extras["task_rew_buf"] = env.rew_buf
        self.extras["disc_rew_buf"] = self.disc_rew_buf
        self._rows = []

    # protocol: the wrapped env's buffers
    num_obs = property(lambda self: self.env.num_obs)
    obs_buf = property(lambda self: self.env.obs_buf)
    terminate_buf = property(lambda self: self.env.terminate_buf)
    truncate_buf = property(lambda self: self.env.truncate_buf)
    reset_buf = property(lambda self: self.env.reset_buf)
    progress_buf = property(lambda self: self.env.progress_buf)
    gpu_launches = property(lambda self: self.batch.gpu_launches)

    @property
    def rew_buf(self):
        return self._rew if self.discriminator is not None else self.env.rew_buf

    def _amp(self, mask: Optional[torch.Tensor], mode: int):
        b = self.batch
        ids = t0 = None
        if mode == AMP_FILL_REF:
            ids, t0 = self.env.motion_ids, self.env.motion_start_times
        b._check(b._L().smplsim_amp_obs(b._h, C.byref(self._ccfg), C.byref(b._state), C.byref(b._aux),
                                        C.byref(self._tab) if self._tab is not None else None, _ptr(ids), _ptr(t0), _ptr(mask), int(mode),
                                        _ptr(self.amp_obs_buf), b._stream()))
        b.gpu_launches += 1

    def step(self, actions: torch.Tensor):
        env = self.env
        env.step(actions)
        self._amp(None, AMP_PUSH)
        self._rows.append(self.amp_obs.clone())
        if self.discriminator is not None:
            self.disc_rew_buf.copy_(self.discriminator.reward(self.amp_obs, float(self.cfg["disc_reward_scale"])))
            torch.add(env.rew_buf * float(self.cfg["task_reward_w"]), self.disc_rew_buf * float(self.cfg["disc_reward_w"]), out=self._rew)
        return self.obs_buf, self.rew_buf, self.terminate_buf, self.truncate_buf

    def _mask(self, env_ids):
        if env_ids is None:
            return None
        if env_ids.dtype in (torch.bool, torch.uint8) and env_ids.numel() == self.num_envs:
            return env_ids.to(self.device, torch.uint8).contiguous()
        mask = torch.zeros(self.num_envs, dtype=torch.uint8, device=self.device)
        mask[env_ids.to(self.device).long()] = 1
        return mask

    def reset(self, env_ids: Optional[torch.Tensor] = None, *args, **kw):
        """The wrapped env's ``reset(env_ids, ...)`` (further arguments go to it), then the AMP history of the same envs."""
        if env_ids is not None and env_ids.numel() == 0:
            return self.obs_buf
        mask = self._mask(env_ids)
        out = self.env.reset(mask, *args, **kw)
        if self.imitation and self.env.fail_states:    # by kind: MoCap from the clip, fall from the state; recovery envs continue
            from .imitation import RESET_FALL, RESET_MOCAP
            kind = self.env.reset_kind
            mocap, fall = (kind == RESET_MOCAP).to(torch.uint8), (kind == RESET_FALL).to(torch.uint8)
            self._amp(mocap, AMP_FILL_REF)
            self._amp(fall, AMP_FILL)
            mask = (mocap, fall)
        else:
            self._amp(mask, AMP_FILL_REF if self.imitation else AMP_FILL)
        self._keep_mask = mask
        return out

    def reset_done(self):
        return self.reset(self.env.reset_buf)

    def drain_amp_obs(self) -> torch.Tensor:
        """The AMP rows of every step since the last drain, ``[steps, N, K * F]`` (empty when there was no step)."""
        rows = torch.stack(self._rows) if self._rows else self.amp_obs.new_zeros(0, self.num_envs, self.num_amp_obs)
        self._rows = []
        return rows

    def make_discriminator(self) -> AMPDiscriminator:
        """A fresh discriminator for this env's AMP rows, from ``disc_units`` / ``disc_activation`` / ``normalize_amp_input``."""
        c = self.cfg
        return AMPDiscriminator(self.num_amp_obs, c["disc_units"], c["disc_activation"], bool(c["normalize_amp_input"])).to(self.device)

    def make_learner(self, discriminator: Optional[AMPDiscriminator] = None, generator: Optional[torch.Generator] = None) -> AMPLearner:
        """Attach ``discriminator`` (default: ``make_discriminator()``) and return its ``AMPLearner`` on the library's demo rows."""
        if self.lib is None:
            raise ValueError("an AMP learner needs a motion library for the demonstration rows (motion_lib=)")
        self.discriminator = discriminator if discriminator is not None else self.make_discriminator()
        return AMPLearner(self.discriminator, lambda n: self.lib.amp_obs_demo(n).view(n, -1), self.cfg, generator)
