"""The training step's backward kernels (grad_kernels.cuh through tdmpc2_wm_loss_backward / tdmpc2_pi_loss_backward)
against a float64 reference anchored on the kernels' own forward.

The oracles (oracle/update_oracle.py, oracle/pi_oracle.py) run with a Tape: every value the forward kernels taped -- the
pre-LayerNorm rows of each LayerNorm layer, the latents, the head logits, pi's action -- replaces the oracle's own while
its derivative still comes from the graph.  Both oracle arms, fp32 and float64, then differentiate the same forward, so
the fp32 arm's distance from float64 is the error of backward arithmetic alone, and the ratio rule
(|kernels - float64| <= RATIO x |fp32 - float64| + FLOOR) holds the backward kernels to it on both engines, at
initialisation and at trained scale.  The same run checks the taped forward: each taped value against what the oracle
computes for that layer from the kernels' own input (the fp32 yardstick the farther of exact and kernel-rounded
operands, as in tests/test_gpu_update.py).

The cases reach the backward's shape arithmetic: the split-K row partition of the parameter gradients (`nsplit` and
the split length `kc` of api.cu, mirrored below), the warp-per-row tails, the model widths of the shape envelope
(tests/test_gpu_shape_envelope.py) and the large presets.  Each asserts the arithmetic that gets it there (`reaches`).
The observed ratios are printed as a table at the end of the module (pytest -s)."""
import functools

import pytest
import torch
import torch.nn.functional as F

from helpers import DEV, level_model, ratio_rule, trained_obs
from helpers import ratio_table  # noqa: F401 (autouse: this module's ratio table)
from oracle.pi_oracle import PI_KEYS, update_pi_oracle
from oracle.update_oracle import Tape, update_oracle
from test_gpu_shape_envelope import CASES as ENVELOPE, shape
from test_gpu_update import split_all
from test_gpu_update_pi import qualifying_batch

pytestmark = pytest.mark.gpu
ENGINES = ["simt", "tcgen05"]
LEVELS = ["init", "mid"]
GBK = 16                 # kGBK: gemm_f32's K tile


# ------------------------------------------------------------------------------------ shape arithmetic (api.cu)
def pad64(n):
    return (n + 63) // 64 * 64


def nsplit(rows):
    """wm_ws / pi_ws: the split count of every parameter-gradient reduction, from the loss's row count."""
    return max(1, min(8, rows // 256))


def splits(k, ns):
    """gemm_f32's K partition: split s sums rows [s kc, min(k, (s + 1) kc)) -> (kc, the length of each split)."""
    kc = (k + ns - 1) // ns
    return kc, [max(0, min(k, (s + 1) * kc) - s * kc) for s in range(ns)]


def row_shape(H, B):
    """The row partition of the world-model backward at H x B (the dynamics' and heads' reductions run over R = H B
    rows, the encoder's over B rows with R's split count) and of update_pi at T = H, B."""
    R = H * B
    ns = nsplit(R)
    kc, _ = splits(R, ns)
    kc_enc, enc = splits(B, ns)
    return dict(R=R, nsplit=ns, kc=kc, kc_enc=kc_enc, enc_min=min(enc), tail=R % 8)


def n_enc(sd):
    n = 0
    while f"_encoder.state.{n}.weight" in sd:
        n += 1
    return n


# ------------------------------------------------------------------------------------ tape layouts
def decode_wm_tape(cfg, sd, tape, zs, ql, rl, tl, H, B):
    """wm_tape of api.cu -> Tape values: segments enc [B, (n_enc - 1) enc_dim + L], dyn [H B, 2 M + L], rew [H B, 2 M],
    q [H B, 2 M num_q] (head h's layer l at (2 h + l) M), term [H B, 2 M] (episodic), each on a 64-float boundary; the
    latents and the head logits.  The decoded size must be the tdmpc2_wm_loss_tape_bytes query's."""
    L, M, E, nq, R = cfg.latent_dim, cfg.mlp_dim, cfg.enc_dim, cfg.num_q, H * B
    ne = n_enc(sd)
    segs = [("enc", B, (ne - 1) * E + L if ne else 0), ("dyn", R, 2 * M + L), ("rew", R, 2 * M), ("q", R, 2 * M * nq)]
    if cfg.episodic:
        segs.append(("term", R, 2 * M))
    seg, off = {}, 0
    for name, rows, pitch in segs:
        seg[name] = tape[off:off + rows * pitch].view(rows, pitch)
        off += pad64(rows * pitch)
    assert off == tape.numel(), f"wm tape layout: decoded {off} floats, the tape holds {tape.numel()}"
    v = {}
    for i in range(ne):
        c0 = i * E
        v[f"_encoder.state.{i}"] = seg["enc"][:, c0:c0 + (E if i < ne - 1 else L)]
    dyn = seg["dyn"].view(H, B, -1)
    for t in range(H):
        for i, (c0, c1) in enumerate(((0, M), (M, 2 * M), (2 * M, 2 * M + L))):
            v[f"_dynamics@{t}.{i}"] = dyn[t, :, c0:c1]
    for i in range(2):
        v[f"_reward.{i}"] = seg["rew"][:, i * M:(i + 1) * M]
        for h in range(nq):
            v[f"_Qs.{h}.{i}"] = seg["q"][:, (2 * h + i) * M:(2 * h + i + 1) * M]
        if cfg.episodic:
            v[f"_termination.{i}"] = seg["term"][:, i * M:(i + 1) * M]
    v["_reward.2"] = rl
    for h in range(nq):
        v[f"_Qs.{h}.2"] = ql[h]
    if cfg.episodic:
        v["_termination.2"] = tl
    for t in range(H + 1):
        v[f"zs.{t}"] = zs[t]
    return {k: t.detach().cpu() for k, t in v.items()}


def decode_pi_tape(cfg, tape, R):
    """pi_tape of plan_kernels.cuh -> Tape values: per row pi.0 and pi.1 [M], the head's logits [Apad + A] (log_std's
    at column Apad), for each head slot u its layers 0, 1 [M] and logits [num_bins], the action [A] and q, the pitch a
    multiple of 4.  The decoded size must be the tdmpc2_pi_loss_tape_bytes query's."""
    M, A, nb = cfg.mlp_dim, cfg.action_dim, cfg.num_bins
    Apad = (A + 31) // 32 * 32
    pih = 2 * M
    q0 = pih + Apad + A
    q1 = q0 + 2 * M + nb
    act = q1 + 2 * M + nb
    pitch = (act + A + 1 + 3) // 4 * 4
    assert R * pitch == tape.numel(), f"pi tape layout: decoded {R * pitch} floats, the tape holds {tape.numel()}"
    t = tape.view(R, pitch)
    v = {"_pi.0": t[:, :M], "_pi.1": t[:, M:2 * M], "_pi.2": torch.cat([t[:, pih:pih + A], t[:, pih + Apad:pih + Apad + A]], 1),
         "act": t[:, act:act + A]}
    for u, q in enumerate((q0, q1)):
        for i, (c0, c1) in enumerate(((0, M), (M, 2 * M), (2 * M, 2 * M + nb))):
            v[f"_Qs.{u}.{i}"] = t[:, q + c0:q + c1]
    return {k: x.detach().cpu() for k, x in v.items()}


# ------------------------------------------------------------------------------------ cases
# id -> (workload, overrides, H, B, what it reaches, the shape arithmetic that proves it (on row_shape(H, B) and the
# envelope's shape(cfg))).  update_pi runs the same rows as T = H, B.
ROW = "tiny"
CASES = {
    "r255": (ROW, {}, 3, 85, "nsplit 1 one row short of 256, a partial last warp-row block",
             lambda r, s: r["R"] == 255 and r["nsplit"] == 1 and r["tail"] != 0),
    "r256": (ROW, {}, 2, 128, "nsplit 1 at 256 rows", lambda r, s: r["R"] == 256 and r["nsplit"] == 1),
    "r511": (ROW, {}, 7, 73, "nsplit 1 at 511 rows", lambda r, s: r["R"] == 511 and r["nsplit"] == 1 and r["tail"] != 0),
    "r512": (ROW, {}, 4, 128, "the first two-split reduction", lambda r, s: r["R"] == 512 and r["nsplit"] == 2),
    "r767": (ROW, {}, 13, 59, "two splits of 384 rows, a partial warp-row block",
             lambda r, s: r["R"] == 767 and r["nsplit"] == 2 and r["tail"] != 0),
    "r768": (ROW, {}, 3, 256, "three splits of 256 rows (the presets' default H = 3, B = 256)",
             lambda r, s: r["R"] == 768 and r["nsplit"] == 3 and r["kc"] == 256),
    "r2120": (ROW, {}, 5, 424, "eight splits of 265 rows: kc is not a multiple of the 16-row K tile",
              lambda r, s: r["R"] >= 2048 and r["nsplit"] == 8 and r["kc"] % GBK != 0),
    "h256b8": (ROW, {}, 256, 8, "eight splits: the encoder's dW over B = 8 rows in one-row splits",
               lambda r, s: r["nsplit"] == 8 and r["kc_enc"] == 1 and r["enc_min"] <= 1),
}
ROW_CASES = list(CASES)
# the model-shape cases of the shape envelope (not the planner's), at H = 3, B = 16
PLANNER_ONLY = ("pi128", "pi_all", "elite1", "samples1", "pi1_e130")
WIDTH_CASES = [c for c in ENVELOPE if c not in PLANNER_ONLY]
for c in WIDTH_CASES:
    wl, over, what, check, _ = ENVELOPE[c]
    CASES[c] = (wl, over, 3, 16, what, lambda r, s, check=check: check(s))
CASES.update({
    "c1": ("c1", {}, 3, 256, "c1 at its default batch: three splits of 256 rows",
           lambda r, s: (s["M"], s["L"]) == (512, 512) and r["nsplit"] == 3),
    "c3": ("c3", {}, 2, 256, "the 1792-wide preset over 512 rows (two splits)",
           lambda r, s: s["M"] == 1792 and r["R"] >= 512 and r["nsplit"] == 2),
    "c4": ("c4", {}, 2, 256, "the 4096-wide preset: latent 1376, 8 Q heads, 80 tasks, 512 rows",
           lambda r, s: (s["M"], s["L"], s["Q"]) == (4096, 1376, 8) and r["R"] >= 512),
    "episodic": ("tiny", {"episodic": True}, 3, 32, "the termination head (tests/test_gpu_update.py's episodic case)",
                 lambda r, s: True),
    "corner": ("tiny", {"action_dim": 128, "num_bins": 256, "latent_dim": 8}, 2, 16,
               "256 bins, 128 actions, latent 8 (tests/test_gpu_update.py's corner case)",
               lambda r, s: (s["B"], s["A"], s["L"]) == (256, 128, 8)),
    "mt_t5_b64": ("tiny-mt", {"task_dim": 5, "action_dims": [5, 1, 4, 2]}, 3, 64, "multi-task: T = 5, masked actions",
                  lambda r, s: s["T"] == 5 and 1 in s["action_dims"]),
    "rgb": ("tiny-rgb", {}, 3, 32, "a pixel model: the latent variant, dL/dz_0 out", lambda r, s: s is None),
})
PRESETS = ["c1", "c3", "c4", "episodic", "corner", "mt_t5_b64", "rgb"]
# qualifying_batch's candidate pool per row: the float64 pi of the widest presets is costly on the host
PI_POOL = {"c3": 8, "c4": 4}
# at "mid" a row with any saturated action dim does not qualify for the policy loss: with 97-256 action dims none does
SATURATED_POLICY = ("a97", "a128", "corner")
# Measured, not yet explained; strict: a fix makes the check fail until the entry is removed.
#   wm forward: the SIMT engine's Q logits of the 4096-wide preset at trained scale (a 4096-term head layer; the wgmma
#   engine's ratio is 1.5) miss the rule at 8.95; at init they reach 8.28, inside the rule by its floor.  The backward
#   of the same case passes.
#   pi grad: pi layer 2's [W | b] of the 256-bin model at trained scale on the SIMT engine's tape misses at 11.6 (the
#   same backward kernels pass on the wgmma engine's tape, and every other tensor of the case passes).  The squash
#   term's derivative 2 a / (1 - a^2) is ill-conditioned for rows near the qualification limit 1 - a^2 > 1e-3.
KNOWN = {("wm forward", "c4", "mid", "simt"): "_Qs.5.2", ("pi grad", "bins256", "mid", "simt"): "_pi.2.[weight|bias]"}


def assert_passed(fail, kind, case, level, engine):
    known = KNOWN.get((kind, case, level, engine))
    if known:
        assert [f.split(":")[0] for f in fail] == [known], f"the known miss changed: {list(fail)}"
        pytest.xfail(f"{kind}: {fail[0]}")
    assert not fail, "\n".join(fail)


def case_params(cases):
    return [pytest.param(c, lv, id=f"{c}-{lv}") for c in cases for lv in LEVELS]


@functools.lru_cache(maxsize=2)
def model(case, level):
    wl, over = CASES[case][:2]
    return level_model(wl, level, **over)


def reaches(case, cfg):
    H, B, what, check = CASES[case][2:]
    r, s = row_shape(H, B), shape(cfg) if "state" in cfg.obs_shape else None
    assert check(r, s), f"{case} does not reach {what!r}: {r} {s}"


class Failures(list):
    def rule(self, kind, key, case, k, o32, o64):
        """The ratio rule on one quantity; the table records it under `kind`, a failure names `key`."""
        try:
            ratio_rule(kind, case, k, o32, o64)
        except AssertionError as e:
            self.append(f"{key}: {str(e).splitlines()[0]}")


def augmented(g, k):
    """A Linear's gradient as one [W | b] tensor (the bias is the weight of a constant input)."""
    return torch.cat([g[k].double().cpu(), g[k[:-len("weight")] + "bias"].double().cpu().unsqueeze(-1)], -1)


def compare_grads(fail, kind, case, got, o32, o64):
    for k in o64:
        if k.endswith(".weight") and ".ln." not in k and k != "_task_emb.weight":
            fail.rule(kind, k[:-len("weight")] + "[weight|bias]", case, augmented(got, k), augmented(o32, k), augmented(o64, k))
        elif ".ln." in k or k == "_task_emb.weight":
            fail.rule(kind, k, case, got[k], o32[k], o64[k])


def compare_tape(fail, kind, case, values, t32, t32s, t64):
    """Each taped value against the oracles' value of that layer on the kernels' input; the yardstick is the fp32 arm
    (exact or kernel-rounded operands) farther from float64."""
    for key, v in values.items():
        if key not in t64.got:
            continue
        e = lambda t: float((t.double() - t64.got[key]).abs().max())
        y = t32.got[key] if e(t32.got[key]) >= e(t32s.got[key]) else t32s.got[key]
        fail.rule(kind, key, case, v, y, t64.got[key])


# ------------------------------------------------------------------------------------ the world-model loss
def wm_batch(cfg, H, B, seed):
    g = torch.Generator().manual_seed(seed)
    A, M, L, nq = cfg.action_dim, cfg.mlp_dim, cfg.latent_dim, cfg.num_q
    keep = 1.0 - cfg.dropout
    simnorm = lambda *s: F.softmax(torch.randn(*s, L // cfg.simnorm_dim, cfg.simnorm_dim, generator=g) * 3, -1).reshape(*s, L)
    latent = cfg.get("obs", "state") == "rgb"
    return dict(obs0=None if latent else trained_obs(cfg, B, seed), z0=simnorm(B) if latent else None,
                action=torch.rand(H, B, A, generator=g) * 2 - 1, reward=torch.randn(H, B, 1, generator=g) * 3,
                terminated=(torch.rand(H, B, 1, generator=g) < 0.3).float() if cfg.episodic else torch.zeros(H, B, 1),
                task=torch.randint(0, len(cfg.tasks), (B,), generator=g) if cfg.multitask else None,
                drop=(torch.rand(nq, H, B, M, generator=g) < keep).float() / keep,
                next_z=simnorm(H, B), td=torch.randn(H, B, 1, generator=g) * 3)


def wm_kernels(cfg, sd, engine, x, H, B):
    """The taped forward and the backward into zeroed .grad tensors, as agent._update runs them -> (Tape values,
    grads by key, dz0 | None)."""
    from tdmpc2_b200.tdmpc2 import TDMPC2
    agent = TDMPC2(cfg, device=DEV, engine=engine)
    agent.model.load_state_dict(sd)
    pl, A, nq, R = agent.planner, cfg.action_dim, cfg.num_q, H * B
    dv = lambda t: None if t is None else t.to(DEV).contiguous()
    taskv = agent.model._task_rows(pl, dv(x["task"]), (H, B))
    act, drop = dv(x["action"]).reshape(R, A), dv(x["drop"]).reshape(nq, R, -1)
    obs0, zs = dv(x["obs0"]), None
    if obs0 is None:
        zs = torch.empty(H + 1, B, cfg.latent_dim, device=DEV)
        zs[0] = dv(x["z0"])
    tape, zs, ql, rl, tl = pl.wm_loss_forward(obs0, act, taskv, drop, H, B, zs=zs)
    grads = {k: torch.zeros_like(agent.model.tensor(k)) for k in agent._wm_keys}
    dz0 = pl.wm_loss_backward(agent.model.tensor, tape, obs0, act, taskv, drop, H, B, zs, ql, rl, tl, dv(x["next_z"]),
                              dv(x["reward"]), dv(x["td"]), dv(x["terminated"]), grads)
    torch.cuda.synchronize()
    values = decode_wm_tape(cfg, sd, tape, zs, ql, rl, tl, H, B)
    return values, {k: v.cpu() for k, v in grads.items()}, None if dz0 is None else dz0.cpu()


def wm_oracle(cfg, sd, x, values, dtype, split=False):
    tape = Tape(dict(values, next_z=x["next_z"], td=x["td"]))
    obs = torch.zeros(1, *x["z0"].shape) if x["obs0"] is None else x["obs0"].unsqueeze(0)
    r = update_oracle(cfg, split_all(sd) if split else sd, obs, x["action"], x["reward"], x["terminated"], x["task"],
                      None, None, x["drop"], None, None, None, dtype=dtype, split=split, tape=tape)
    return r, tape


def check_wm(case, level, engine):
    cfg, sd = model(case, level)
    H, B = CASES[case][2:4]
    cfg = cfg.replace(horizon=H, batch_size=B)
    reaches(case, cfg)
    x = wm_batch(cfg, H, B, 11)
    values, grads, dz0 = wm_kernels(cfg, sd, engine, x, H, B)
    (o32, t32), (o64, t64) = wm_oracle(cfg, sd, x, values, torch.float32), wm_oracle(cfg, sd, x, values, torch.float64)
    _, t32s = wm_oracle(cfg, sd, x, values, torch.float32, split=True)
    tag, fail, fwd = f"{case}/{level}/{engine}", Failures(), Failures()
    assert set(o64["grads"]) <= set(grads)
    compare_grads(fail, "wm grad", tag, grads, o32["grads"], o64["grads"])
    if dz0 is not None:
        fail.rule("wm dz0", "dz0", tag, dz0, o32["dz0"], o64["dz0"])
    assert len(t64.got) == len(values) - (1 if dz0 is not None else 0), sorted(set(values) - set(t64.got))
    compare_tape(fwd, "wm forward", tag, values, t32, t32s, t64)
    assert_passed(fail, "wm grad", case, level, engine)
    assert_passed(fwd, "wm forward", case, level, engine)


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("case,level", case_params(ROW_CASES))
def test_wm_backward_rows(case, level, engine):
    """The world-model loss's parameter gradients and taped forward at the row counts that walk the split-K partition."""
    check_wm(case, level, engine)


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("case,level", case_params(WIDTH_CASES))
def test_wm_backward_widths(case, level, engine):
    """The world-model loss at the model widths of the shape envelope: LayerNorm / SimNorm lane tails, head widths,
    encoder depth and pitches, ensemble sizes."""
    check_wm(case, level, engine)


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("case,level", case_params(PRESETS))
def test_wm_backward_presets(case, level, engine):
    """The world-model loss on the presets, the episodic and corner models of tests/test_gpu_update.py, a multi-task
    model with masked actions and a pixel model (dL/dz_0 of the latent variant)."""
    check_wm(case, level, engine)


# ------------------------------------------------------------------------------------ the policy loss
def pi_kernels(cfg, sd, engine, zs, task, eps, qidx, drop, scale0):
    """update_pi's taped forward, the running scale's update and the backward into zeroed .grad tensors -> (Tape
    values with the scale, grads by key)."""
    from tdmpc2_b200.tdmpc2 import TDMPC2
    agent = TDMPC2(cfg, device=DEV, engine=engine)
    agent.model.load_state_dict(sd)
    pl = agent.planner
    T, B = zs.shape[:2]
    R = T * B
    z = zs.reshape(R, -1).to(DEV).contiguous()
    e = eps.reshape(R, -1).to(DEV).contiguous()
    q32 = qidx.to(DEV, torch.int32).contiguous()
    d = drop.reshape(cfg.num_q, R, -1).to(DEV).contiguous()
    taskv = agent.model._task_rows(pl, None if task is None else task.to(DEV), (T, B))
    tape, _, q, _ = pl.pi_loss_forward(z, taskv, e, q32, d)
    agent.scale.value.copy_(scale0)
    agent.scale.update(q.view(T, B, 1)[0])
    grads = {k: torch.zeros_like(agent.model.tensor(k)) for k in PI_KEYS}
    emb = torch.zeros_like(agent.model.tensor("_task_emb.weight")) if cfg.multitask else None
    pl.pi_loss_backward(agent.model.tensor, tape, z, taskv, e, q32, d, T, B, agent.scale.value, cfg.entropy_coef, cfg.rho,
                        grads, emb)
    torch.cuda.synchronize()
    values = decode_pi_tape(cfg, tape, R)
    values["scale"] = agent.scale.value.detach().cpu().clone()
    out = {k: v.cpu() for k, v in grads.items()}
    if emb is not None:
        out["_task_emb.weight"] = emb.cpu()
    return values, out


def check_pi(case, level, engine):
    cfg, sd = model(case, level)
    T, B = CASES[case][2:4]
    reaches(case, cfg)
    zs, task, eps, qidx = qualifying_batch(cfg, sd, T, B, 5, pool=PI_POOL.get(case, 256))
    g = torch.Generator().manual_seed(6)
    keep = 1.0 - cfg.dropout
    drop = (torch.rand(cfg.num_q, T, B, cfg.mlp_dim, generator=g) < keep).float() / keep
    scale0 = torch.tensor([1.7])
    values, grads = pi_kernels(cfg, sd, engine, zs, task, eps, qidx, drop, scale0)

    def oracle(dtype, split=False):
        tape = Tape(values)
        r = update_pi_oracle(cfg, split_all(sd) if split else sd, zs, task, eps, qidx, drop, scale0, dtype, tape=tape,
                             split=split)
        return r, tape
    (o32, t32), (o64, t64), (_, t32s) = oracle(torch.float32), oracle(torch.float64), oracle(torch.float32, True)
    tag, fail, fwd = f"pi/{case}/{level}/{engine}", Failures(), Failures()
    compare_grads(fail, "pi grad", tag, grads, o32["grads"], o64["grads"])
    assert len(t64.got) == len(values) - 1, sorted(set(values) - set(t64.got))
    compare_tape(fwd, "pi forward", tag, values, t32, t32s, t64)
    assert_passed(fwd, "pi forward", case, level, engine)
    assert_passed(fail, "pi grad", case, level, engine)


PI_CASES = [c for c in CASES if c != "rgb"]


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("case,level", [p for p in case_params(PI_CASES)
                                        if not (p.values[0] in SATURATED_POLICY and p.values[1] == "mid")])
def test_pi_backward(case, level, engine):
    """The policy loss's parameter and embedding gradients and its taped forward (rows qualified as in
    tests/test_gpu_update_pi.py), at the row counts, widths and presets above (T = H)."""
    check_pi(case, level, engine)
