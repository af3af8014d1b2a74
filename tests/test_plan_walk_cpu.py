"""The plan-versus-oracle walk of tests/helpers.py (_walk_plan, through compare_with_oracle and compare_plans) on the host:
the fp32 oracle's plan, laid out as the kernel's trace, passes both value criteria against the float64 oracle, and each
kind of fault a kernel could make fails the walk with a message naming the quantity."""
import functools

import pytest
import torch

from helpers import TERM_MARGIN, boundary_separated, compare_plans, compare_with_oracle, stable_positions
from oracle.plan_oracle import balance_termination, draw_noise, plan_oracle
from tdmpc2_b200.config import workload
from tdmpc2_b200.synth import synth_state_dict

E = 4
CASES = {"tiny": ("tiny", {}), "tiny-mt": ("tiny-mt", {}), "episodic": ("tiny", {"episodic": True})}
CRITERIA = ["absolute", "ratio"]
SEPARATED = 1e-3          # wider than either criterion's top-k gap on these models


@functools.lru_cache(maxsize=None)
def planned(case):
    """(cfg, fp32 PlanTrace, float64 PlanTrace, noise) of one plan of E environments, odd ones warm-started."""
    wl, over = CASES[case]
    cfg = workload(wl, num_envs=E, **over)
    sd = synth_state_dict(cfg, seed=7, perturb=True, emb_scale=60.0 if cfg.multitask else 1.0)
    if cfg.episodic:
        balance_termination(cfg, sd)
    g = torch.Generator().manual_seed(3)
    obs = torch.randn(E, cfg.obs_shape["state"][0], generator=g)
    prev = 0.3 * torch.randn(E, cfg.horizon, cfg.action_dim, generator=g)
    args = dict(task=[(2 * i + 1) % len(cfg.tasks) for i in range(E)] if cfg.multitask else None,
                t0=[i % 2 == 0 for i in range(E)], prev_mean=prev, noise=draw_noise(cfg, 40, E))
    return cfg, plan_oracle(cfg, sd, obs, **args), plan_oracle(cfg, sd, obs, dtype=torch.float64, **args), args["noise"]


def kernel_view(w32):
    """The fp32 plan as plan(trace=True) returns it: (trace dict, action, new mean), copies that a test may corrupt."""
    tr = {q: getattr(w32, q).clone() for q in ("values", "elite_idx", "iter_mean", "iter_std", "pick")}
    return tr, w32.action.clone(), w32.mean.clone()


def walk(criterion, case, tr, action, new_mean):
    cfg, w32, w64, noise = planned(case)
    if criterion == "absolute":
        keep = w64.term_margin > TERM_MARGIN if cfg.episodic else None
        return compare_with_oracle(cfg, tr, action, new_mean, w64, noise, range(E), keep=keep)
    return compare_plans(cfg, f"cpu walk/{case}", tr, action, new_mean, w32, w64, noise)


@pytest.mark.parametrize("criterion", CRITERIA)
@pytest.mark.parametrize("case", list(CASES))
def test_fp32_oracle_passes_the_walk(case, criterion):
    n = walk(criterion, case, *kernel_view(planned(case)[1]))
    assert n["values"] > 0 and n["topk"] > 0 and n["refit"] > 0 and n["means"] > 0 and n["actions"] > 0, n


def first_refit_env(case):
    """An environment whose first iteration is compared through its refit under either criterion."""
    cfg, _, w64, _ = planned(case)
    keep = w64.term_margin > TERM_MARGIN if cfg.episodic else torch.ones_like(w64.values, dtype=torch.bool)
    return next(e for e in range(E) if bool(keep[e, 0].all())
                and bool(boundary_separated(w64.values[e, 0], cfg.num_elites, SEPARATED)))


@pytest.mark.parametrize("fault", ["values", "top-k", "iter_mean", "pick", "action"])
@pytest.mark.parametrize("criterion", CRITERIA)
@pytest.mark.parametrize("case", list(CASES))
def test_the_walk_names_what_is_wrong(case, criterion, fault):
    cfg, w32, w64, _ = planned(case)
    tr, action, new_mean = kernel_view(w32)
    e = first_refit_env(case)
    if fault == "values":                            # one compared value, far past either criterion's allowance
        n = int(torch.nonzero(w64.term_margin[e, 0] > TERM_MARGIN)[0]) if cfg.episodic else 0
        tr["values"][e, 0, n] += 1e-2
    elif fault == "top-k":                           # two separated sorted positions swapped
        p, q = torch.nonzero(stable_positions(w64.values[e, 0], cfg.num_elites, SEPARATED)).view(-1)[:2].tolist()
        tr["elite_idx"][e, 0, [p, q]] = tr["elite_idx"][e, 0, [q, p]]
    elif fault == "iter_mean":                       # the first refit's mean off by 2e-4
        tr["iter_mean"][e, 0] += 2e-4
    elif fault == "pick":                            # every pick moved: the walk compares at least one
        tr["pick"] = (tr["pick"] + 1) % cfg.num_elites
    else:
        action += 1e-3
    with pytest.raises(AssertionError, match=fault):
        walk(criterion, case, tr, action, new_mean)
