"""The fused kernels, driven through the reference-shaped agent API (TDMPC2._plan), against the
golden vectors minted from the REFERENCE's own unmodified `_plan` (oracle/make_golden.py).
E == 1, every model preset of BASELINE.json.  Run on an H100: pytest -m gpu."""
import pytest
import torch

from helpers import load_golden, stable_positions, boundary_separated

pytestmark = pytest.mark.gpu

CASES = ["tiny", "tiny_mt", "c1_dog5m", "c3_humanoid48m_e1", "c4_mt80_317m_e1", "tiny_episodic", "c1_dog5m_episodic", "tiny_rgb",
         "tiny_nopi", "tiny_h1", "tiny_knobs", "tiny_mt_t5", "tiny_wide_heads", "tiny_odd_widths"]
# A termination decision flips a trajectory value by O(1): samples whose termination logit lies within this margin
# of the 0.5 boundary (by the oracle, which is bit-identical to the reference) are not compared.
TERM_MARGIN = 2e-5
# Trajectory values: |got - golden| <= 5e-5 + 1e-5 |golden| for EVERY preset (the 317M preset's values reach ~17).  The
# 3-pass fp16-split GEMM carries ~22 bits per product; the tensor core's toward-zero accumulate drift over long
# reductions (K = 4096) is bounded by handing partial sums off every 512 / 1024 elements of K (see test_gpu_multitrip).
VALUE_ATOL, VALUE_RTOL = 5e-5, 1e-5


@pytest.mark.parametrize("name", CASES)
def test_agent_matches_reference_golden(name):
    from oracle.plan_oracle import draw_noise as oracle_noise
    from tdmpc2_b200.planner import Noise
    from tdmpc2_b200.tdmpc2 import TDMPC2
    cfg, sd, calls = load_golden(name)
    cfg.iterations_effective = True          # fixtures carry the effective loop count
    cfg.num_envs = 1
    agent = TDMPC2(cfg, device="cuda:0")
    agent.load(sd)
    K = cfg.num_elites
    checked_actions = 0
    for c in calls:
        n = oracle_noise(cfg, c["seed"], 1, eval_mode=c["eval_mode"])
        noise = Noise.from_env_major(n.prior, n.r, n.pi, n.qidx, n.expo, None if c["eval_mode"] else n.final, device="cuda",
                                     shift=n.shift)
        agent._prev_mean.copy_(c["prev_mean"].cuda())
        action, tr = agent._plan(c["obs"].cuda().unsqueeze(0), t0=c["t0"], eval_mode=c["eval_mode"],
                                 task=None if c["task"] is None else torch.tensor([c["task"]]).cuda(),
                                 noise=noise, return_trace=True)
        torch.cuda.synchronize()
        assert action.shape == (cfg.action_dim,)                    # reference return shape
        values = tr["values"][0].cpu()
        decided = torch.ones(cfg.iterations, cfg.num_samples, dtype=torch.bool)
        if cfg.episodic:
            from oracle.plan_oracle import plan_oracle
            want = plan_oracle(cfg, sd, c["obs"][None], t0=[c["t0"]], prev_mean=c["prev_mean"][None], noise=n,
                               eval_mode=c["eval_mode"])
            # the oracle is the reference restated (bit-identical on the machine that minted the fixture, a few ulp elsewhere)
            assert torch.allclose(want.values[0][want.term_margin[0] > TERM_MARGIN],
                                  c["values"][want.term_margin[0] > TERM_MARGIN], atol=2e-5, rtol=0)
            decided = want.term_margin[0] > TERM_MARGIN
        clean = True
        for it in range(cfg.iterations):
            if not clean:
                break
            tol = VALUE_ATOL + VALUE_RTOL * float(c["values"][it].abs().max())
            err = (values[it] - c["values"][it]).abs()[decided[it]].max().item()
            assert torch.allclose(values[it][decided[it]], c["values"][it][decided[it]], atol=VALUE_ATOL, rtol=VALUE_RTOL), \
                f"{name}: values it={it} err={err:.3e}"
            if not bool(decided[it].all()):
                clean = False                    # a knife-edge termination may have moved one sample across the elite set
                continue
            stable = stable_positions(c["values"][it], K, 2 * tol)
            assert torch.equal(tr["elite_idx"][0, it].cpu()[stable], c["elite_idx"][it][stable]), f"top-k it={it}"
            clean = bool(boundary_separated(c["values"][it], K, 2 * tol))
        if clean:
            assert torch.allclose(agent._prev_mean.cpu(), c["mean"], atol=1e-4, rtol=0)
            # the gumbel pick is position-wise: compare the action when the sorted order was unambiguous
            if all(bool(stable_positions(c["values"][it], K, 2 * tol).all()) for it in range(cfg.iterations)):
                assert torch.allclose(action.cpu(), c["action"], atol=1e-4, rtol=0)
                checked_actions += 1
    print(f"[{name}] calls={len(calls)} actions compared={checked_actions}")
