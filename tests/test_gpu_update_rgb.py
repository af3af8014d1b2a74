"""agent._update of pixel models on the H100 kernels (the taped conv forward of pixel_encoder.cuh, the latent world-model
loss and the conv backward of pixel_grad_kernels.cuh), on both engines: against fixtures minted from the reference's own
_update, against the float64 oracle by the ratio rule, and the conv backward alone against float64 autograd."""
import pytest
import torch

from helpers import FLOOR, RATIO, level_model, ratio_rule
from oracle.update_rgb_oracle import RGB_CASES, RGB_MULTI_STEP, case_inputs, load_case, run_case, update_rgb_oracle
from rgb_update_checks import check_state_rgb
from test_gpu_update import REAL_CLIP, make_agent, split_all, yardstick
from update_checks import check_info

pytestmark = pytest.mark.gpu
ENGINES = ["simt", "tcgen05"]
DEV = "cuda"
CONV = [f"_encoder.rgb.{i}" for i in (2, 4, 6, 8)]
SCALAR_ULPS = 4


def step(agent, x, capture=None, monkeypatch=None, draws=True):
    """agent._update on pixel frames with the case's explicit draws (shift included); `capture` receives the world
    model's .grad tensors before clipping."""
    if capture is not None:
        names = {id(agent.model.tensor(k)): k for k in agent.model.keys() if not k.startswith("_detach_Qs_params.")}
        calls = []

        def clip(params, max_norm, *a, **k):
            params = list(params)
            if not calls:                                   # the first call clips the world model; update_pi's comes next
                for p in params:
                    capture[names[id(p)]] = p.grad.detach().clone()
            calls.append(1)
            return REAL_CLIP(params, max_norm, *a, **k)
        monkeypatch.setattr(torch.nn.utils, "clip_grad_norm_", clip)
    dv = lambda t: None if t is None else t.to(DEV)
    kw = {}
    if draws:
        kw = dict(shift=dv(x["shift"]), td_eps=dv(x["td_eps"]), td_qidx=dv(x["td_qidx"]), dropout_mask=dv(x["drop"]),
                  pi_eps=dv(x["pi_eps"]), pi_qidx=dv(x["pi_qidx"]), pi_dropout_mask=dv(x["pi_drop"]))
    return agent._update(dv(x["obs"]), dv(x["action"]), dv(x["reward"]), dv(x["terminated"]), **kw)


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", list(RGB_CASES) + list(RGB_MULTI_STEP))
def test_update_matches_reference_fixture(engine, name, monkeypatch):
    """Every step's info dict, the last step's gradients before clipping (the conv layers' included), the parameters and
    target Q after it, against the reference's own _update."""
    base, steps = RGB_MULTI_STEP.get(name, (name, 1))
    cfg, sd, _, want = load_case(name)
    agent = make_agent(cfg, sd, engine)
    xs = [case_inputs(cfg, base, s) for s in range(steps)]
    agent.scale.value.copy_(xs[0]["scale0"])
    before = {k: agent.model.tensor(k).detach().clone() for k in agent.model.keys() if k.startswith("_encoder.rgb.")}
    for s, x in enumerate(xs):
        grads = {}
        info = step(agent, x, grads, monkeypatch)
        check_info(info, want, "info/" if s == 0 else f"info{s}/", rel=1e-4, gn_rel=1e-3)
    assert sum(k.startswith("_encoder.rgb.") for k in grads) == 8
    # one Adam step moves a parameter by about lr: a near-tied sign of a tiny gradient can flip its direction
    check_state_rgb(grads, agent.model.tensor, None, want, grad_rel=1e-3, param_abs=2.5 * cfg.lr * steps)
    for k, v in before.items():                            # the conv encoder trains
        if not k.endswith("8.bias"):                       # dL/db4 = 0 (rgb_update_checks)
            assert not torch.equal(agent.model.tensor(k).detach(), v), k


# ------------------------------------------------------------------------------------ ratio rule against float64
def rgb_ratio_inputs(cfg, H, B, seed):
    g = torch.Generator().manual_seed(seed)
    A, M, nq = cfg.action_dim, cfg.mlp_dim, cfg.num_q
    return dict(obs=torch.randint(0, 256, (H + 1, B) + tuple(cfg.obs_shape["rgb"]), generator=g).float(),
                action=torch.rand(H, B, A, generator=g) * 2 - 1, reward=torch.randn(H, B, 1, generator=g) * 3,
                terminated=torch.zeros(H, B, 1), task=None,
                td_eps=torch.randn(H, B, A, generator=g), td_qidx=torch.randperm(nq, generator=g)[:2],
                drop=torch.ones(nq, H, B, M), pi_eps=torch.randn(H + 1, B, A, generator=g),
                pi_qidx=torch.randperm(nq, generator=g)[:2], pi_drop=torch.ones(nq, H + 1, B, M), scale0=torch.ones(1),
                shift=torch.randint(0, 7, (H + 1, B, 2), generator=g).float())


def _oracle(cfg, sd, x, dtype, split=False):
    return update_rgb_oracle(cfg, sd, x["obs"], x["shift"], x["action"], x["reward"], x["terminated"], x["td_eps"],
                             x["td_qidx"], x["drop"], x["pi_eps"], x["pi_qidx"], x["pi_drop"], x["scale0"], dtype=dtype,
                             split=split)


def split_linears(sd):
    """split_all (the Linear weights as the kernels store them) with the conv weights untouched: plain fp32."""
    out = split_all(sd)
    out.update({k: v for k, v in sd.items() if k.startswith("_encoder.rgb.")})
    return out


RGB_RATIO_CASES = [("tiny-rgb", {}, 3, 8), ("c1", {"obs": "rgb", "obs_channels": 9}, 3, 4)]
RGB_RATIO_IDS = ["tiny-rgb", "c1-rgb"]


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("level", ["init", "mid"])
@pytest.mark.parametrize("case", RGB_RATIO_CASES, ids=RGB_RATIO_IDS)
def test_ratio_rule_against_float64(engine, case, level, monkeypatch):
    """The losses, grad_norm, every gradient ([W | b] per Linear and per Conv2d, LayerNorm gamma / beta) and every step:
    |kernels - float64| <= RATIO x |fp32 - float64| (+ FLOOR), the fp32 yardstick on exact or kernel-rounded operands
    (the Linear layers' weights and inputs split into two fp16 planes; the conv layers are plain fp32 either way) or with
    ATen's other CPU convolution (mkldnn off), whichever is farthest from float64: the conv kernels sum in their own
    order, and z_0 carries that rounding into every later layer."""
    wl, over, H, B = case
    cfg, sd = level_model(wl, level, **over)
    cfg.horizon, cfg.batch_size = H, B
    x = rgb_ratio_inputs(cfg, H, B, 13)
    o32, o64 = _oracle(cfg, sd, x, torch.float32), _oracle(cfg, sd, x, torch.float64)
    o32s = _oracle(cfg, split_linears(sd), x, torch.float32, split=True)
    with torch.backends.mkldnn.flags(enabled=False):      # ATen's other CPU convolution: another fp32 summation order
        o32c = _oracle(cfg, sd, x, torch.float32)
    ys = lambda f: yardstick(yardstick(f(o32), f(o32s), f(o64)), f(o32c), f(o64))
    agent = make_agent(cfg, sd, engine)
    grads = {}
    info = step(agent, x, grads, monkeypatch)
    tag = f"update-rgb/{RGB_RATIO_IDS[RGB_RATIO_CASES.index(case)]}/{level}/{engine}"
    failed = []

    def rr(*a):
        try:
            ratio_rule(*a)
        except AssertionError as e:
            failed.append(str(e).splitlines()[0])
    for q in ("consistency_loss", "reward_loss", "value_loss", "total_loss", "grad_norm"):
        # a scalar is one sample of fp32 rounding, and z_0 comes from the conv forward, which sums in another order than
        # ATen (pixel_encoder.cuh): the ratio rule with a floor of SCALAR_ULPS ulp of the float64 value (DESIGN.md 4.5)
        k_, y_, w_ = float(info[q]), float(ys(lambda r: r[q])), float(o64[q])
        if abs(k_ - w_) > RATIO * abs(y_ - w_) + SCALAR_ULPS * FLOOR * abs(w_):
            failed.append(f"{q} [{tag}]: |k - o64| {abs(k_ - w_):.3e} > {RATIO} x {abs(y_ - w_):.3e} + {SCALAR_ULPS} ulp")
    # a bias is the weight of a constant input: compared with its weight as one [W | b] tensor (conv: per output channel)
    aug = lambda g, k: torch.cat([g[k].double().cpu().flatten(1) if g[k].ndim == 4 else g[k].double().cpu(),
                                  g[k[:-len("weight")] + "bias"].double().cpu().unsqueeze(-1)], -1)
    for k in o64["grads"]:
        if k.endswith(".weight") and ".ln." not in k:
            rr(f"grad {k[:-len('weight')]}[weight|bias]", tag, aug(grads, k),
               ys(lambda r: aug(r["grads"], k)), aug(o64["grads"], k))
        elif ".ln." in k:
            rr("grad " + k, tag, grads[k], ys(lambda r: r["grads"][k]), o64["grads"][k])
    for k in o64["grads"]:
        stp = lambda r: r["sd"][k] - sd[k].to(r["sd"][k].dtype)
        rr("step " + k, tag, agent.model.tensor(k).detach().cpu() - sd[k], ys(stp), stp(o64))
    assert any(k.startswith("_encoder.rgb.") for k in o64["grads"])
    assert not failed, "\n".join(failed)


# ------------------------------------------------------------------------------------ the conv backward alone
def _pixel_agent(C, nc, seed, w4_scale=1.0):
    from tdmpc2_b200.config import workload
    from tdmpc2_b200.synth import synth_state_dict
    cfg = workload("tiny-rgb", obs_channels=C, num_channels=nc, latent_dim=16 * nc)
    sd = synth_state_dict(cfg, seed=seed, perturb=True)
    sd["_encoder.rgb.8.weight"] = sd["_encoder.rgb.8.weight"] * w4_scale
    from tdmpc2_b200.tdmpc2 import TDMPC2
    agent = TDMPC2(cfg, device=DEV, engine="simt")
    agent.model.load_state_dict(sd)
    return cfg, sd, agent


def _conv_backward(agent, frames, shift, dz):
    """-> z, the conv gradients, and the ReLU masks a_l > 0 of the taped forward ([rows, nc, n, n], l = 1, 2, 3)."""
    pl, nc = agent.planner, agent.cfg.num_channels
    z, tape = pl.encode_pixel_rows_taped(frames.to(DEV), shift.to(DEV))
    keys = [k + s for k in CONV for s in (".weight", ".bias")]
    grads = {k: torch.zeros_like(agent.model.tensor(k)) for k in keys}
    pl.pixel_encode_backward(agent.model.tensor, tape, frames.to(DEV), shift.to(DEV), z, dz.to(DEV), grads)
    torch.cuda.synchronize()
    al = lambda n: (n + 63) // 64 * 64                     # the tape's 64-float segments (pixel_encoder.cuh)
    off, masks = 0, []
    t = tape.view(frames.shape[0], -1).cpu()
    for n in (29, 13, 6):
        masks.append((t[:, off:off + nc * n * n] > 0).view(-1, nc, n, n))
        off += al(nc * n * n)
    return z, {k: v.cpu() for k, v in grads.items()}, masks


def _autograd(cfg, sd, frames, shift, dz, dtype, masks):
    """float64 / fp32 autograd of the conv stack, with the ReLUs' decisions taken from the kernels' forward (`masks`): a
    pre-activation within rounding of 0 may fall on either side, and the weight gradient of the layer below sees the
    flip as a whole term."""
    import torch.nn.functional as F
    from oracle.plan_oracle import OracleModel
    from types import SimpleNamespace
    P = {k: sd[k].detach().to(dtype).clone().requires_grad_(True) for k in sd if k.startswith("_encoder.rgb.")}
    real_relu, it = F.relu, iter(masks)
    F.relu = lambda x: x * next(it).to(x.dtype)
    try:
        z = OracleModel.encode_rgb(SimpleNamespace(cfg=cfg, sd=P, dtype=dtype), frames, shift)
    finally:
        F.relu = real_relu
    (z * dz.to(dtype)).sum().backward()
    return {k: v.grad for k, v in P.items()}


@pytest.mark.parametrize("peaked", [False, True], ids=["plain", "peaked"])
@pytest.mark.parametrize("rows", [1, 133])
@pytest.mark.parametrize("C,nc", [(6, 8), (9, 32), (14, 64)])
def test_conv_backward_against_float64(C, nc, rows, peaked):
    """dL/dW, dL/db of the four Conv2d layers for a random dz, against float64 autograd of the conv stack by the ratio
    rule, the references taking the ReLU decisions of the kernels' forward.  (14, 64) is the widest encoder: conv1's weights are staged in input-channel chunks and conv2's (400 KB) are
    read from global memory.  133 frames exceed the SM count.  `peaked`: conv4's weights scaled up 20x, so that SimNorm
    is peaked and many ReLUs are off."""
    if peaked and (C, nc) != (9, 32):
        pytest.skip("the peaked SimNorm case runs at c1-rgb's shape")
    cfg, sd, agent = _pixel_agent(C, nc, 3 + nc, 20.0 if peaked else 1.0)
    g = torch.Generator().manual_seed(rows + nc)
    frames = torch.randint(0, 256, (rows, C, 64, 64), generator=g).float()
    shift = torch.randint(0, 7, (rows, 2), generator=g).float()
    dz = torch.randn(rows, 16 * nc, generator=g)
    _, k, masks = _conv_backward(agent, frames, shift, dz)
    o32 = _autograd(cfg, sd, frames, shift, dz, torch.float32, masks)
    o64 = _autograd(cfg, sd, frames, shift, dz, torch.float64, masks)
    aug = lambda g_, c: torch.cat([g_[c + ".weight"].double().flatten(1), g_[c + ".bias"].double().unsqueeze(-1)], -1)
    tag = f"conv-backward/C{C}-nc{nc}/rows{rows}" + ("/peaked" if peaked else "")
    for c in CONV:
        ratio_rule(f"grad {c}.[weight|bias]", tag, aug(k, c), aug(o32, c), aug(o64, c))


def test_taped_z_bit_identical_and_zs0():
    """The taped forward's z equals encode_pixel_rows's bit for bit; zs[0] of the latent forward equals
    model.encode(obs[0], shift=shift[0])."""
    cfg, sd, out = run_case("tiny_rgb_update")
    agent = make_agent(cfg, sd, "simt")
    x = {k: (None if v is None else v.to(DEV)) for k, v in out[0][0].items()}
    pl = agent.planner
    C = cfg.obs_shape["rgb"][0]
    f, s = x["obs"].reshape(-1, C, 64, 64), x["shift"].reshape(-1, 2)
    z_t, _ = pl.encode_pixel_rows_taped(f, s)
    assert torch.equal(z_t, pl.encode_pixel_rows(f, s))
    H, B = x["action"].shape[:2]
    zs = torch.empty(H + 1, B, cfg.latent_dim, device=DEV)
    pl.encode_pixel_rows_taped(x["obs"][0], x["shift"][0], out=zs[0])
    pl.wm_loss_forward_latent(zs, x["action"].reshape(H * B, -1).contiguous(), None, None, H, B)
    assert torch.equal(zs[0], agent.model.encode(x["obs"][0], None, shift=x["shift"][0]))
    assert torch.equal(zs[1], agent.model.next(zs[0], x["action"][0], None))


@pytest.mark.parametrize("engine", ENGINES)
def test_deterministic_and_accumulates(engine):
    """The whole backward (latent world-model loss, then the conv chain) twice: identical bits; onto pre-set .grad
    values of 0.25: the same gradients plus 0.25."""
    cfg, sd, out = run_case("c1_rgb_update")
    x = {k: (None if v is None else v.to(DEV)) for k, v in out[0][0].items()}
    H, B = x["action"].shape[:2]

    def once(pre=None):
        agent = make_agent(cfg, sd, engine)
        pl = agent.planner
        next_z = agent.model.encode(x["obs"][1:], None, shift=x["shift"][1:])
        td = agent.model.td_target(next_z, x["reward"], x["terminated"], None, eps=x["td_eps"], qidx=x["td_qidx"])
        zs = torch.empty(H + 1, B, cfg.latent_dim, device=DEV)
        _, ptape = pl.encode_pixel_rows_taped(x["obs"][0], x["shift"][0], out=zs[0])
        act = x["action"].reshape(H * B, -1).contiguous()
        drop = x["drop"].reshape(cfg.num_q, H * B, -1).contiguous()
        tape, zs, ql, rl, tl = pl.wm_loss_forward_latent(zs, act, None, drop, H, B)
        grads = {k: (torch.zeros_like(agent.model.tensor(k)) if pre is None else pre[k].clone().to(DEV)) for k in agent._wm_keys}
        dz0 = pl.wm_loss_backward_latent(agent.model.tensor, tape, act, None, drop, H, B, zs, ql, rl, tl, next_z.contiguous(),
                                         x["reward"].contiguous(), td.contiguous(), x["terminated"].contiguous(), grads)
        pl.pixel_encode_backward(agent.model.tensor, ptape, x["obs"][0], x["shift"][0], zs[0], dz0, grads)
        torch.cuda.synchronize()
        return {k: v.cpu() for k, v in grads.items()}
    a, b = once(), once()
    for k in a:
        assert torch.equal(a[k], b[k]), k
    assert any(float(a[k].abs().max()) > 0 for k in a if k.startswith("_encoder.rgb."))
    c = once({k: torch.full_like(v, 0.25) for k, v in a.items()})
    for k in a:
        assert torch.allclose(c[k], a[k] + 0.25, rtol=0, atol=1e-6), k


@pytest.mark.parametrize("engine", ENGINES)
def test_no_host_sync_and_grads_cleared(engine):
    cfg, sd, out = run_case("tiny_rgb_update", steps=2)
    agent = make_agent(cfg, sd, engine)
    dv = lambda t: None if t is None else t.to(DEV)
    x = out[0][0]
    agent._update(dv(x["obs"]), dv(x["action"]), dv(x["reward"]), dv(x["terminated"]))
    x = {k: dv(v) for k, v in out[1][0].items()}
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        agent._update(x["obs"], x["action"], x["reward"], x["terminated"])
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for k in agent.model.keys():
        assert agent.model.tensor(k).grad is None, k


def test_seeded_generator_draws_in_documented_order():
    """A seeded agent.generator without explicit draws gives the same step as explicit draws taken from an identically
    seeded generator in the documented order: obs[1:]'s shifts, td_eps, td_qidx, obs[0]'s shift, the dropout masks,
    then update_pi's eps, dropout masks and qidx."""
    from tdmpc2_b200.planner import draw_shifts
    cfg, sd, out = run_case("tiny_rgb_update")
    x = {k: (None if v is None else v.to(DEV)) for k, v in out[0][0].items()}
    H, B = x["action"].shape[:2]
    A, M, nq, keep = cfg.action_dim, cfg.mlp_dim, cfg.num_q, 1.0 - cfg.dropout
    a, b = make_agent(cfg, sd, "simt"), make_agent(cfg, sd, "simt")
    a.generator = torch.Generator(device=DEV).manual_seed(1234)
    info_a = a._update(x["obs"], x["action"], x["reward"], x["terminated"])
    g = torch.Generator(device=DEV).manual_seed(1234)
    rest = draw_shifts((H, B), DEV, g)
    td_eps = torch.randn(H, B, A, device=DEV, generator=g)
    td_qidx = torch.randperm(nq, device=DEV, generator=g)[:2]
    s0 = draw_shifts((B,), DEV, g)
    drop = torch.empty(nq, H * B, M, device=DEV).bernoulli_(keep, generator=g).div_(keep)
    pi_eps = torch.randn(H + 1, B, A, device=DEV, generator=g)
    pi_drop = torch.empty(nq, (H + 1) * B, M, device=DEV).bernoulli_(keep, generator=g).div_(keep)
    pi_qidx = torch.randperm(nq, device=DEV, generator=g)[:2]
    info_b = b._update(x["obs"], x["action"], x["reward"], x["terminated"], shift=torch.cat([s0[None], rest]),
                       td_eps=td_eps, td_qidx=td_qidx, dropout_mask=drop.view(nq, H, B, M), pi_eps=pi_eps,
                       pi_qidx=pi_qidx, pi_dropout_mask=pi_drop.view(nq, H + 1, B, M))
    for k in info_a:
        assert torch.equal(info_a[k], info_b[k]), k
    for k in a.model.keys():
        assert torch.equal(a.model.tensor(k), b.model.tensor(k)), k


@pytest.mark.parametrize("engine", ENGINES)
def test_act_after_step_matches_fresh_agent(engine):
    cfg, sd, out = run_case("tiny_rgb_update")
    agent = make_agent(cfg, sd, engine)
    step(agent, out[0][0])
    fresh = make_agent(cfg, {k: (v.detach().clone() if torch.is_tensor(v) else v) for k, v in agent.model.state_dict().items()},
                       engine)
    E = agent.num_envs
    obs = torch.randint(0, 256, (E,) + tuple(cfg.obs_shape["rgb"])).float()
    eps = torch.randn(E, cfg.action_dim, device=DEV)
    agent.generator = torch.Generator(device=DEV).manual_seed(5)      # ShiftAug's draw inside _policy_action
    fresh.generator = torch.Generator(device=DEV).manual_seed(5)
    assert torch.equal(agent._policy_action(obs, eps=eps), fresh._policy_action(obs, eps=eps))


def test_uint8_frames_give_the_same_step():
    cfg, sd, out = run_case("tiny_rgb_update")
    x = out[0][0]
    a, b = make_agent(cfg, sd, "simt"), make_agent(cfg, sd, "simt")
    info_a = step(a, x)
    info_b = step(b, dict(x, obs=x["obs"].to(torch.uint8)))
    for k in info_a:
        assert torch.equal(info_a[k], info_b[k]), k
    for k in a.model.keys():
        assert torch.equal(a.model.tensor(k), b.model.tensor(k)), k


def test_input_errors():
    cfg, sd, out = run_case("tiny_rgb_update")
    agent = make_agent(cfg, sd, "simt")
    x = {k: (None if v is None else v.to(DEV)) for k, v in out[0][0].items()}
    with pytest.raises(ValueError):
        agent._update(x["obs"][..., :-1], x["action"], x["reward"], x["terminated"])
    with pytest.raises(ValueError):
        agent._update(x["obs"][:, :, :-1], x["action"], x["reward"], x["terminated"])
    with pytest.raises(ValueError):
        agent._update(x["obs"][0], x["action"], x["reward"], x["terminated"])
    with pytest.raises(ValueError):
        agent._update(x["obs"], x["action"], x["reward"], x["terminated"], shift=x["shift"][1:])
    with pytest.raises(ValueError):
        agent._update(x["obs"], x["action"], x["reward"], x["terminated"], shift=x["shift"][..., :1])
