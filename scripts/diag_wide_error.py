"""Where does the value error of the wide presets come from?  c4 (or c3) at E=3, env 1: errors of encode, policy-prior
actions and first-iteration values against the fp32 CPU oracle, per engine (simt = fp32 FFMA on the same split operands)."""
import os, sys, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import torch
torch.set_num_threads(min(16, os.cpu_count() or 1))
from tdmpc2_b200.config import workload
from tdmpc2_b200.synth import synth_state_dict
from tdmpc2_b200.planner import Planner
from oracle.plan_oracle import plan_oracle
from helpers import mixed_noise
wl = sys.argv[1] if len(sys.argv) > 1 else "c4"
engines = sys.argv[2:] or ["tcgen05", "simt"]
E = 3
cfg = workload(wl, num_envs=E, iterations=2)
sd = synth_state_dict(cfg, seed=9)
g = torch.Generator().manual_seed(33)
obs = torch.randn(E, cfg.obs_shape["state"][0], generator=g)
prev = 0.3 * torch.randn(E, cfg.horizon, cfg.action_dim, generator=g)
t0 = torch.zeros(E, dtype=torch.uint8)
task = (torch.arange(E) * 7 + 3) % len(cfg.tasks) if cfg.multitask else None
envs = [0, 1, 2]
nz, on = mixed_noise(cfg, E, envs, 400)
want = plan_oracle(cfg, sd, obs[envs], task=None if task is None else [int(task[e]) for e in envs], t0=[False] * 3, prev_mean=prev[envs], noise=on)
taskv = None if task is None else task.to(torch.int32).cuda()
symlog = lambda x: torch.sign(x) * torch.log1p(x.abs())
for eng in engines:
    pl = Planner(cfg, E, "cuda:0", engine=eng)
    pl.pack(sd)
    a, m, tr = pl.plan(obs.cuda(), taskv, t0.cuda(), prev.cuda(), nz, trace=True)
    torch.cuda.synchronize()
    out = {"engine": eng, "workload": wl}
    out["z_err"] = float((tr["z"].cpu() - want.z).abs().max())
    out["pi_actions_err"] = float((tr["pi_actions"].cpu() - want.pi_actions).abs().max())
    v, w = tr["values"][:, 0].cpu(), want.values[:, 0]
    out["values_range"] = [float(w.min()), float(w.max())]
    out["value_abs_err_per_env"] = [f"{float((v[e] - w[e]).abs().max()):.2e}" for e in range(E)]
    out["value_rel_err_per_env"] = [f"{float(((v[e] - w[e]).abs() / w[e].abs().clamp_min(1.0)).max()):.2e}" for e in range(E)]
    out["symlog_err_per_env"] = [f"{float((symlog(v[e]) - symlog(w[e])).abs().max()):.2e}" for e in range(E)]
    out["value_err_median"] = f"{float((v - w).abs().median()):.2e}"
    out["signed_mean_err"] = f"{float((v - w).mean()):.2e}"
    print(json.dumps(out), flush=True)
    del pl
