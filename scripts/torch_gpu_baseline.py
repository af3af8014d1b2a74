"""Strong baseline for SURVEY.md section 8(d)(iii): the planner restated as BATCHED eager PyTorch (rows = E x N
through the same torch ops the reference uses: F.linear / layer_norm / mish / softmax / topk), runnable on the
same H100 as the fused kernels.  Measurement aid, not product code and not the parity oracle (that is
oracle/plan_oracle.py; tests/test_torch_batched_baseline.py holds this file to it on CPU).

    python scripts/torch_gpu_baseline.py [--workload c2] [--envs 256] [--steps 5] [--device cuda:0]

Prints one JSON line: planning steps/s of `plan()` with inputs resident on the device, noise drawn per call like
bench.py does.  Follows the reference line by line (tdmpc2.py:122-206, world_model.py:88-216), with a leading
environment axis; like the reference it evaluates ALL num_q heads and then picks two (world_model.py:207-216).
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tdmpc2_b200.config import workload, get_discount      # noqa: E402
from tdmpc2_b200.synth import synth_state_dict             # noqa: E402


class BatchedTorchPlanner:
    def __init__(self, cfg, sd, device):
        self.cfg, self.dev = cfg, torch.device(device)
        self.sd = {k: v.to(self.dev, torch.float32) for k, v in sd.items() if torch.is_tensor(v) and v.is_floating_point()}
        self.bins = torch.linspace(cfg.vmin, cfg.vmax, cfg.num_bins, device=self.dev)
        if cfg.multitask:
            self.gamma = torch.tensor([get_discount(cfg, ep) for ep in cfg.episode_lengths], device=self.dev)
            w = self.sd["_task_emb.weight"]
            n = torch.linalg.vector_norm(w, dim=1, keepdim=True)                       # nn.Embedding(max_norm=1)
            self.emb = torch.where(n > 1.0, w * (1.0 / (n + 1e-7)), w)
        else:
            self.gamma = get_discount(cfg, cfg.episode_length)

    # ---- layers.py:94-133 on rows [..., in]
    def _mlp(self, prefix, x, last="none", head=None):
        i = 0
        while f"{prefix}.{i}.weight" in self.sd:
            w, b = self.sd[f"{prefix}.{i}.weight"], self.sd[f"{prefix}.{i}.bias"]
            g, beta = self.sd.get(f"{prefix}.{i}.ln.weight"), self.sd.get(f"{prefix}.{i}.ln.bias")
            if head is not None:        # all heads at once: x [E, R, in] -> [Q, E, R, out]
                x = torch.einsum("eri,qoi->qero" if i == 0 else "qeri,qoi->qero", x, w) + b[:, None, None, :]
                if g is not None:
                    mu = x.mean(-1, keepdim=True)
                    var = x.var(-1, unbiased=False, keepdim=True)
                    x = (x - mu) * torch.rsqrt(var + 1e-5) * g[:, None, None, :] + beta[:, None, None, :]
                    x = F.mish(x)
            else:
                x = F.linear(x, w, b)
                if g is not None:
                    x = F.layer_norm(x, (x.shape[-1],), g, beta, 1e-5)
                    is_last = f"{prefix}.{i + 1}.weight" not in self.sd
                    if is_last and last == "simnorm":
                        shp = x.shape
                        x = F.softmax(x.view(*shp[:-1], -1, self.cfg.simnorm_dim), dim=-1).view(*shp)
                    else:
                        x = F.mish(x)
            i += 1
        return x

    def _emb(self, x, task):            # x [E, R, ·], task [E]
        if not self.cfg.multitask:
            return x
        return torch.cat([x, self.emb[task][:, None, :].expand(-1, x.shape[1], -1)], dim=-1)

    def two_hot_inv(self, x):
        x = torch.sum(F.softmax(x, dim=-1) * self.bins, dim=-1, keepdim=True)
        return torch.sign(x) * (torch.exp(torch.abs(x)) - 1)

    def next(self, z, a, task):
        return self._mlp("_dynamics", torch.cat([self._emb(z, task), a], -1), "simnorm")

    def reward(self, z, a, task):
        return self.two_hot_inv(self._mlp("_reward", torch.cat([self._emb(z, task), a], -1)))

    def pi(self, z, task, eps):
        mean, log_std = self._mlp("_pi", self._emb(z, task)).chunk(2, dim=-1)
        log_std = self.sd["log_std_min"] + 0.5 * self.sd["log_std_dif"] * (torch.tanh(log_std) + 1)
        if self.cfg.multitask:
            m = self.sd["_action_masks"][task][:, None, :]
            mean, log_std, eps = mean * m, log_std * m, eps * m
        return torch.tanh(mean + eps * log_std.exp())

    def q_avg(self, z, a, task, qidx):  # qidx [E, 2]
        out = self._mlp("_Qs.params", torch.cat([self._emb(z, task), a], -1), head=True)   # [Q, E, N, B]
        E = z.shape[0]
        sel = out[qidx.t(), torch.arange(E, device=self.dev)[None, :]]                      # [2, E, N, B]
        return self.two_hot_inv(sel).sum(0) / 2

    def estimate_value(self, z, actions, task, eps_pi, qidx):
        """z [E,N,L], actions [E,H,N,A] -> [E,N,1]   (tdmpc2.py:122-136)"""
        cfg = self.cfg
        G, discount = 0, 1
        termination = torch.zeros(z.shape[0], z.shape[1], 1, device=self.dev)
        gamma = self.gamma[task][:, None, None] if cfg.multitask else self.gamma
        for t in range(cfg.horizon):
            reward = self.reward(z, actions[:, t], task)
            z = self.next(z, actions[:, t], task)
            G = G + discount * (1 - termination) * reward
            discount = discount * gamma
            if cfg.episodic:
                termination = torch.clip(termination + (torch.sigmoid(self._mlp("_termination", z)) > 0.5).float(), max=1.)
        action = self.pi(z, task, eps_pi)
        return G + discount * (1 - termination) * self.q_avg(z, action, task, qidx)

    @torch.no_grad()
    def plan(self, obs, task, t0, prev_mean, noise, eval_mode=False, iter_major=False):
        """obs [E,obs], task [E] | None, t0 [E] bool, prev_mean [E,H,A]; noise: prior [E,H,P,A], r [E,I,H,N-P,A],
        pi [E,I,N,A], qidx [E,I,2], expo [E,K], final [E,A] | None.  Returns (action [E,A], mean [E,H,A], values [E,I,N])."""
        cfg = self.cfg
        E, H, N, P, A, K = obs.shape[0], cfg.horizon, cfg.num_samples, cfg.num_pi_trajs, cfg.action_dim, cfg.num_elites
        at = (lambda t, it: t[it]) if iter_major else (lambda t, it: t[:, it])   # planner.Noise is [I,E,...], the oracle's [E,I,...]
        x = obs[:, None, :]
        z0 = self._mlp("_encoder.state", self._emb(x, task), "simnorm")                     # [E,1,L]
        pi_actions = torch.zeros(E, H, P, A, device=self.dev)
        if P > 0:
            _z = z0.expand(-1, P, -1)
            for t in range(H - 1):
                pi_actions[:, t] = self.pi(_z, task, noise.prior[:, t])
                _z = self.next(_z, pi_actions[:, t], task)
            pi_actions[:, -1] = self.pi(_z, task, noise.prior[:, H - 1])
        z = z0.expand(-1, N, -1)
        mean = torch.zeros(E, H, A, device=self.dev)
        std = torch.full((E, H, A), float(cfg.max_std), device=self.dev)
        warm = (~t0.bool())[:, None, None]
        mean[:, :-1] = torch.where(warm, prev_mean[:, 1:], mean[:, :-1])
        actions = torch.empty(E, H, N, A, device=self.dev)
        actions[:, :, :P] = pi_actions
        mask = self.sd["_action_masks"][task][:, None, None, :] if cfg.multitask else None
        values = []
        for it in range(cfg.iterations):
            actions[:, :, P:] = (mean.unsqueeze(2) + std.unsqueeze(2) * at(noise.r, it)).clamp(-1, 1)
            if mask is not None:
                actions = actions * mask
            value = self.estimate_value(z, actions, task, at(noise.pi, it), at(noise.qidx, it).long()).nan_to_num(0)
            elite_idxs = torch.topk(value.squeeze(-1), K, dim=1).indices                    # [E,K]
            elite_value = torch.gather(value, 1, elite_idxs[:, :, None])                    # [E,K,1]
            elite_actions = torch.gather(actions, 2, elite_idxs[:, None, :, None].expand(-1, H, -1, A))   # [E,H,K,A]
            score = torch.exp(cfg.temperature * (elite_value - elite_value.max(1, keepdim=True).values))
            score = score / score.sum(1, keepdim=True)
            sw = score[:, None, :, :]                                                        # [E,1,K,1]
            mean = (sw * elite_actions).sum(2) / (score.sum(1)[:, None, :] + 1e-9)
            std = ((sw * (elite_actions - mean.unsqueeze(2)) ** 2).sum(2) / (score.sum(1)[:, None, :] + 1e-9)).sqrt()
            std = std.clamp(cfg.min_std, cfg.max_std)
            if mask is not None:
                mean, std = mean * mask[:, :, 0], std * mask[:, :, 0]
            values.append(value.squeeze(-1))
        logits = score.squeeze(-1).log() - noise.expo.log()                                 # math.py:86-94
        pick = logits.softmax(-1).argmax(-1)
        a = elite_actions[torch.arange(E, device=self.dev), 0, pick]
        if not eval_mode:
            a = a + std[:, 0] * noise.final
        return a.clamp(-1, 1), mean, torch.stack(values, 1)


def run(workload_name="c2", envs=None, steps=5, device="cuda:0", tf32=False, budget_s=60.0):
    """Time `plan()` of the batched eager-PyTorch restatement (CUDA events on a GPU, wall clock on CPU);
    returns the JSON-able record.  `envs` environments are planned per call (a bounded sample of the workload);
    tf32=True lets cuBLAS use TF32 tensor cores (torch.backends.cuda.matmul.allow_tf32), fp32 otherwise."""
    from tdmpc2_b200.planner import draw_noise
    over = {} if envs is None else {"num_envs": envs}
    cfg = workload(workload_name, iterations_effective=True, **over)
    dev = torch.device(device)
    E = cfg.num_envs
    prev_tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = bool(tf32)
    try:
        pl = BatchedTorchPlanner(cfg, synth_state_dict(cfg, seed=1), dev)
        obs = torch.randn(E, cfg.obs_shape["state"][0], device=dev)
        task = (torch.arange(E, device=dev) % len(cfg.tasks)) if cfg.multitask else None
        state = {"prev": torch.zeros(E, cfg.horizon, cfg.action_dim, device=dev)}
        on_gpu = dev.type == "cuda"
        sync = (lambda: torch.cuda.synchronize(dev)) if on_gpu else (lambda: None)

        def step(t0):
            n = draw_noise(cfg, E, dev, reference_order=False)
            a, state["prev"], _ = pl.plan(obs, task, torch.full((E,), t0, device=dev), state["prev"], n, iter_major=True)
            return a

        step(True); step(False); sync()
        t_begin, times = time.perf_counter(), []
        for _ in range(steps):
            if times and time.perf_counter() - t_begin > budget_s:
                break
            if on_gpu:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(); step(False); e1.record(); sync()
                times.append(e0.elapsed_time(e1))
            else:
                t = time.perf_counter(); step(False); times.append((time.perf_counter() - t) * 1e3)
        ms = sum(times) / len(times)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev_tf32
    return {"impl": "batched eager PyTorch / cuBLAS (reference algorithm, all num_q heads)", "device": str(dev),
            "matmul": "tf32" if tf32 else "fp32", "workload": workload_name, "envs": E, "ms_per_step": ms,
            "value": E * cfg.num_samples * cfg.horizon / (ms * 1e-3), "unit": "steps/s", "steps": len(times)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c2")
    ap.add_argument("--envs", type=int, default=None)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--device", default="cuda:0")
    ap.add_argument("--tf32", action="store_true")
    args = ap.parse_args()
    print(json.dumps(run(args.workload, args.envs, args.steps, args.device, args.tf32)))


if __name__ == "__main__":
    main()
