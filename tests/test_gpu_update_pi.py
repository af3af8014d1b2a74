"""agent.update_pi on the H100 kernels (ROP_PI_LOSS forward + grad_kernels.cuh backward) against fixtures minted from the
reference's own update_pi and against the float64 oracle (oracle/pi_oracle.py) by the ratio rule."""
import pytest
import torch

from helpers import level_model, ratio_rule
from oracle.pi_oracle import CASES, PI_KEYS, load_case, update_pi_oracle

pytestmark = pytest.mark.gpu
ENGINES = ["simt", "tcgen05"]
DEV = "cuda"
REAL_CLIP = torch.nn.utils.clip_grad_norm_


def make_agent(cfg, sd, engine):
    from tdmpc2_b200.tdmpc2 import TDMPC2
    agent = TDMPC2(cfg, device=DEV, engine=engine)
    agent.model.load_state_dict(sd)
    return agent


def run(agent, zs, task, eps, qidx, drop=None, capture=None, monkeypatch=None):
    """agent.update_pi with explicit draws; `capture` receives the .grad tensors before clipping (by key)."""
    if capture is not None:
        real = REAL_CLIP

        def clip(params, max_norm, *a, **k):
            params = list(params)
            keys = agent._pi_keys
            for key, p in zip(keys, params):
                capture[key] = p.grad.detach().clone()
            if agent.cfg.multitask:
                capture["_task_emb.weight"] = agent.model.tensor("_task_emb.weight").grad.detach().clone()
            return real(params, max_norm, *a, **k)
        monkeypatch.setattr(torch.nn.utils, "clip_grad_norm_", clip)
    dv = lambda t: None if t is None else t.to(DEV)
    return agent.update_pi(dv(zs), dv(task), eps=dv(eps), qidx=dv(qidx), dropout_mask=dv(drop))


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", list(CASES))
def test_fixture_through_update_pi(engine, name, monkeypatch):
    cfg, sd, x, want = load_case(name)
    agent = make_agent(cfg, sd, engine)
    agent.scale.value.copy_(x["scale0"])
    grads = {}
    info = run(agent, x["zs"], x["task"], x["eps"], x["qidx"], x["drop"], grads, monkeypatch)
    assert abs(float(info["pi_loss"]) - float(want["loss"])) <= 1e-4 * abs(float(want["loss"])) + 1e-6
    assert torch.allclose(info["pi_scale"].cpu(), want["scale_after"].float(), rtol=1e-5)
    assert abs(float(info["pi_grad_norm"]) - float(want["grad_norm"])) <= 1e-3 * float(want["grad_norm"])
    for k in PI_KEYS + (["_task_emb.weight"] if cfg.multitask else []):
        w = want["grad/" + k].double()
        g = grads[k][:w.shape[0]].double().cpu()
        assert float((g - w).abs().max()) <= 1e-3 * float(w.abs().max()) + 1e-9, k
    for k in PI_KEYS:
        w = want["param/" + k].double()
        got = agent.model.tensor(k).detach()[:w.shape[0]].double().cpu()
        # one Adam step moves a parameter by about lr: a near-tied sign of a tiny gradient can flip its direction
        assert float((got - w).abs().max()) <= 2.5 * agent.cfg.lr, k


def qualifying_batch(cfg, sd, T, B, seed):
    """zs [T, B, L], task [B] | None, eps [T, B, A], qidx: rows where the float64 |log_pi| > 1e-2 and min(1 - a^2) > 1e-3
    (the squash term and the entropy scale are ill-conditioned elsewhere; the same exclusion as row_mode_ratio_rule)."""
    import torch.nn.functional as F
    from oracle.wm_oracle import WMOracle
    g = torch.Generator().manual_seed(seed)
    N = 256 * T * B                                               # candidate rows; column b takes task b % num_tasks
    ntask = len(cfg.tasks) if cfg.multitask else 1
    zs = F.softmax(torch.randn(N, cfg.latent_dim // 8, 8, generator=g) * 3, dim=-1).reshape(N, -1)
    eps = torch.randn(N, cfg.action_dim, generator=g)
    cand_task = torch.arange(N) % ntask
    o64 = WMOracle(cfg, sd, torch.float64)
    a, info = o64.pi(zs, cand_task if cfg.multitask else None, eps)
    ok = ((1 - a ** 2).min(-1).values > 1e-3) & (info["entropy"].squeeze(-1).abs() > 1e-2)
    task = torch.arange(B) % ntask
    cols = []
    for b in range(B):
        idx = torch.nonzero(ok & (cand_task == task[b])).reshape(-1)[T * (b // ntask):T * (b // ntask + 1)]
        assert idx.numel() == T, f"column {b}: too few qualifying rows"
        cols.append(idx)
    sel = torch.stack(cols, dim=1)                                # [T, B]
    return zs[sel], task if cfg.multitask else None, eps[sel], torch.randperm(cfg.num_q, generator=g)[:2]


def split_weights(sd):
    """`sd` with every pi and Q weight matrix rounded as the kernels' forward stores it: two fp16 planes (hi, lo) of
    W * 2^k, max|W| 2^k in [128, 256), per matrix and head (api.cu, split_weight_kernel)."""
    out = dict(sd)
    for k, w in sd.items():
        if k.endswith(".weight") and ".ln." not in k and k.startswith(("_pi.", "_Qs.params.")):
            w = w.float()
            amax = w.abs().amax(dim=(-2, -1), keepdim=True)
            s = torch.ldexp(torch.ones_like(amax), 8 - torch.frexp(amax).exponent)
            hi = (w * s).half().float()
            out[k] = (hi + (w * s - hi).half().float()) / s
    return out


def yardstick(q, o32, o32s, o64):
    """the fp32 result (exact or on the kernels' rounded weights) farther from float64: the error fp32 arithmetic makes
    on the operands the forward multiplies"""
    e = lambda t: float((t.double() - o64.double()).abs().max())
    return o32 if e(o32) >= e(o32s) else o32s


def oracle_pair(cfg, sd, zs, task, eps, qidx, drop=None, steps=1):
    out = []
    for dt in (torch.float32, torch.float64):
        sdd, state, r = dict(sd), None, None
        scale = torch.ones(1)
        for _ in range(steps):
            r = update_pi_oracle(cfg, sdd, zs, task, eps, qidx, drop, scale, dt, state)
            state, scale = r["adam"], r["scale"]
            sdd.update(r["params"])
        out.append(r)
    return out


RATIO_CASES = [("c1", {}, 4, 64), ("tiny-mt", {"task_dim": 5, "action_dims": [5, 1, 4, 2]}, 3, 32),
               ("tiny", {"action_dim": 128, "num_bins": 256, "latent_dim": 8}, 2, 16)]


# (case, level): at "mid" every one of the wide-head corner's 128 action dims would have to stay unsaturated for a row to
# qualify, and none does
RATIO_PARAMS = [(c, lv) for c in RATIO_CASES for lv in ("init", "mid") if not (lv == "mid" and c[1].get("action_dim") == 128)]


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("case,level", RATIO_PARAMS, ids=lambda c: c if isinstance(c, str) else c[0] + ("-corner" if c[1] else ""))
def test_ratio_rule_against_float64(engine, case, level, monkeypatch):
    wl, over, T, B = case
    cfg, sd = level_model(wl, level, **over)
    zs, task, eps, qidx = qualifying_batch(cfg, sd, T, B, 5)
    o32, o64 = oracle_pair(cfg, sd, zs, task, eps, qidx)
    o32s = update_pi_oracle(cfg, split_weights(sd), zs, task, eps, qidx)
    agent = make_agent(cfg, sd, engine)
    grads = {}
    info = run(agent, zs, task, eps, qidx, None, grads, monkeypatch)
    tag = f"update_pi/{wl}{'-corner' if over else ''}/{level}/{engine}"
    for q, k in (("pi_loss", info["pi_loss"]), ("pi_grad_norm", info["pi_grad_norm"])):
        key = "loss" if q == "pi_loss" else "grad_norm"
        ratio_rule(q, tag, k.reshape(1), yardstick(q, o32[key], o32s[key], o64[key]).reshape(1), o64[key].reshape(1))
    # a Linear's bias is the weight of a constant input: its gradient is compared with the weight's as one [W | b]
    # tensor (the bias gradient alone is a cancelling sum over rows, far smaller than its terms)
    aug = lambda g, i: torch.cat([g[f"_pi.{i}.weight"].double().cpu(), g[f"_pi.{i}.bias"].double().cpu().unsqueeze(1)], 1)
    for i in range(3):
        ratio_rule(f"grad _pi.{i}.[weight|bias]", tag, aug(grads, i),
                   yardstick(i, aug(o32["grads"], i), aug(o32s["grads"], i), aug(o64["grads"], i)), aug(o64["grads"], i))
    for k in [k for k in PI_KEYS if ".ln." in k] + (["_task_emb.weight"] if cfg.multitask else []):
        ratio_rule("grad " + k, tag, grads[k], yardstick(k, o32["grads"][k], o32s["grads"][k], o64["grads"][k]), o64["grads"][k])
    for k in PI_KEYS:
        # parameters after the step: the step is taken from each arm's own gradient, on the unrounded weights
        step = lambda r: r["params"][k] - sd[k].to(r["params"][k].dtype)
        ratio_rule("step " + k, tag, agent.model.tensor(k).detach().cpu() - sd[k], yardstick(k, step(o32), step(o32s), step(o64)),
                   step(o64))


@pytest.mark.parametrize("engine", ENGINES)
def test_three_steps_and_dropout(engine):
    cfg, sd = level_model("tiny", "init")
    zs, task, eps, qidx = qualifying_batch(cfg, sd, 3, 32, 9)
    g = torch.Generator().manual_seed(4)
    drop = (torch.rand(cfg.num_q, 3, 32, cfg.mlp_dim, generator=g) < 0.99).float() / 0.99
    o32, o64 = oracle_pair(cfg, sd, zs, task, eps, qidx, drop, steps=3)
    agent = make_agent(cfg, sd, engine)
    agent.model.train()
    for _ in range(3):
        run(agent, zs, task, eps, qidx, drop)
    for k in PI_KEYS:
        ratio_rule("3 steps " + k, f"update_pi/tiny/{engine}", agent.model.tensor(k).detach(), o32["params"][k], o64["params"][k])
    ratio_rule("3 steps scale", f"update_pi/tiny/{engine}", agent.scale.value, o32["scale"], o64["scale"])


@pytest.mark.parametrize("engine", ENGINES)
def test_gradients_deterministic_and_accumulating(engine, monkeypatch):
    cfg, sd = level_model("tiny-mt", "init")
    zs, task, eps, qidx = qualifying_batch(cfg, sd, 3, 48, 3)
    first, second, acc = {}, {}, {}
    run(make_agent(cfg, sd, engine), zs, task, eps, qidx, None, first, monkeypatch)
    run(make_agent(cfg, sd, engine), zs, task, eps, qidx, None, second, monkeypatch)
    for k in first:
        assert torch.equal(first[k], second[k]), k
    agent = make_agent(cfg, sd, engine)
    keys = PI_KEYS + ["_task_emb.weight"]
    g0 = {k: torch.randn_like(agent.model.tensor(k)) for k in keys}
    for k in keys:
        agent.model.tensor(k).grad = g0[k].clone()
    run(agent, zs, task, eps, qidx, None, acc, monkeypatch)
    for k in keys:
        torch.testing.assert_close(acc[k], g0[k] + first[k], rtol=0, atol=0)
    # pi_optim zeroes the pi gradients; the embedding keeps its accumulated gradient; nothing else gets one
    assert all(agent.model.tensor(k).grad is None for k in PI_KEYS)
    assert torch.equal(agent.model.tensor("_task_emb.weight").grad, acc["_task_emb.weight"])
    for name, p in agent.model.named_parameters():
        if "_pi__" not in name and "_task_emb" not in name:
            assert p.grad is None, name


@pytest.mark.parametrize("engine", ENGINES)
def test_no_host_sync_and_act_after_step(engine):
    from tdmpc2_b200.tdmpc2 import TDMPC2
    cfg, sd = level_model("tiny", "init")
    agent = make_agent(cfg, sd, engine)
    zs = torch.softmax(torch.randn(3, 64, cfg.latent_dim // 8, 8, device=DEV), -1).reshape(3, 64, -1)
    agent.update_pi(zs, None)                                   # first call: planner set-up
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        agent.update_pi(zs, None)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    fresh = TDMPC2(cfg, device=DEV, engine=engine)
    fresh.load(agent.model.state_dict())
    obs = torch.randn(cfg.num_envs, cfg.obs_shape["state"][0])
    outs = []
    for a in (agent, fresh):
        a.generator = torch.Generator(device=DEV).manual_seed(11)
        outs.append(a.act(obs, t0=True))
    assert torch.equal(outs[0], outs[1])


def test_input_errors():
    cfg, sd = level_model("tiny-mt", "init")
    agent = make_agent(cfg, sd, "tcgen05")
    zs = torch.rand(2, 4, cfg.latent_dim, device=DEV)
    task = torch.zeros(4, dtype=torch.long, device=DEV)
    with pytest.raises(ValueError):
        agent.update_pi(zs[0], task)                             # not [T, B, L]
    with pytest.raises(ValueError):
        agent.update_pi(zs, None)                                # multi-task without a task
    with pytest.raises(ValueError):
        agent.update_pi(zs, task, eps=torch.zeros(2, 4, 1, device=DEV))
    with pytest.raises(ValueError):
        agent.update_pi(zs, task, qidx=torch.tensor([0], device=DEV))
    with pytest.raises(ValueError):
        agent.update_pi(zs, task, dropout_mask=torch.ones(1, device=DEV))
