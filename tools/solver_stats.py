#!/usr/bin/env python
"""Why does the first active-set solve of a substep miss?  Runs the bench workload (cfg2: speed task, random actions) on the
host emulator build with -DSMPLSIM_STATS and prints the counters of lane_kernels.cuh (g_lstats).  The per-CTA figures mean what
they mean on the GPU only at the CTA size a full launch picks there (8 warps = 32 SMPL envs): set SMPLSIM_WPB=8.
usage: SMPLSIM_WPB=8 SMPLSIM_EMU_SO=/tmp/emu_stats.so python tools/solver_stats.py [envs] [steps]"""
import ctypes as C
import os
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
import emu_env  # noqa: E402
from smplsim_b200.cfg import make_cfg  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 64
steps = int(sys.argv[2]) if len(sys.argv) > 2 else 30
env = emu_env.EmuBatch(make_cfg(env="speed"), n, seed=0, with_aux=False)
env.reset()
g = torch.Generator(); g.manual_seed(0)
L = emu_env.lib()
out = (C.c_int * 64)()
L.smplsim_debug_stats(out, 1)
for i in range(steps):
    a = torch.clamp(torch.randn(n, env.num_actions, generator=g) * 0.0821, -1, 1)
    env.step(a); env.reset_done()
L.smplsim_debug_stats(out, 1)
s = list(out)
print(f"env-substeps {s[0]}  with rows {s[1]} ({s[1] / max(1, s[0]):.2f})  first pass ok {s[2]} ({s[2] / max(1, s[1]):.2f} of those with rows)")
print("extra solves histogram 1..6+:", s[3:9], " mean over envs with rows:", sum((i + 1) * v for i, v in enumerate(s[3:9])) / max(1, s[1]))
for name, h in (("env", [s[0] - sum(s[3:9])] + s[3:9]), ("warp maximum", s[32:39]), ("CTA maximum", s[39:46])):
    tot = max(1, sum(h))
    print(f"per-{name} extra solves 0..6+ per substep: {h}  = {[round(100 * v / tot, 1) for v in h]} %  mean {sum(i * v for i, v in enumerate(h)) / tot:.3f}")
print(f"contacts {s[13]} (new {s[14]});  rows predicted active but free {s[9]}, predicted free but active {s[10]}, of both in new contacts {s[11]}; limit rows flipped {s[12]}")
print(f"rows {s[16]}: inherit wrong {s[17]} ({s[17] / max(1, s[16]):.3f}), prediction wrong {s[18]} ({s[18] / max(1, s[16]):.3f}), both wrong {s[19]}; contacts with exact inherit {s[20]}, exact prediction {s[21]} of {s[13]}")
miss = s[1] - s[2]
print(f"first-pass misses {miss}: every flipped row below 1e-3 N: {s[22]}, 1e-2 N: {s[23]}, 0.1 N: {s[24]}, 1 N: {s[25]}; below 1e-4 / 1e-3 of the total contact force: {s[26]} / {s[27]}")
print(f"env-substeps with >= 3 extra solves: {s[28]} (of which with a contact new this substep: {s[29]}; mean contacts {s[31] / max(1, s[28]):.1f} vs {s[13] / max(1, s[1]):.1f} overall); env-substeps with a new contact: {s[30]}")
