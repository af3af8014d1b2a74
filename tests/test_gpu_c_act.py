"""Planning from a plain C host (include/tdmpc2_b200.h: the model file, tdmpc2_plan_draws, tdmpc2_act): the upload is the
state dict bit for bit, the device draws follow their laws, one tdmpc2_act is the Python planner's rng = 'philox' plan
bit for bit when that plan's small draws come from tdmpc2_plan_draws, a captured call replays like eager calls, and
examples/c_act.c computes what the ctypes calls compute.  Run on an H100: pytest -m gpu."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch
from scipy import stats

from helpers import cuda_stream, draw_planner, plan_draws, planner_for
from tdmpc2_b200 import _cabi
from tdmpc2_b200.config import workload
from tdmpc2_b200.export import export_model
from tdmpc2_b200.planner import alloc_noise, discount_table
from tdmpc2_b200.synth import synth_state_dict

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = {"c1": ("c1", {}), "tiny-mt": ("tiny-mt", {}), "episodic": ("tiny", {"episodic": True}), "tiny-rgb": ("tiny-rgb", {})}


def _model(case, E, tmp_path, **over):
    wl, kw = CASES[case]
    cfg = workload(wl, num_envs=E, iterations_effective=True, **kw, **over)     # the file's iterations are cfg.iterations
    sd = synth_state_dict(cfg, seed=5, perturb=True)
    path = str(tmp_path / f"{case}.tdmpc2")
    export_model(sd, cfg, path)
    return cfg, sd, path


class CModel:
    """The C host's sequence through ctypes: open, create, bind, upload, pack, then tdmpc2_act on torch tensors."""

    def __init__(self, path, num_envs=None, horizon=None, seed=1234):
        self.lib = lib = _cabi.load()
        self.f = C.c_void_p()
        _cabi.check(lib.tdmpc2_model_file_open(path.encode(), C.byref(self.f)))
        self.d, self.pd, isp = _cabi.Dims(), _cabi.PixelDims(), C.c_int32()
        _cabi.check(lib.tdmpc2_model_file_dims(self.f, C.byref(self.d), C.byref(self.pd), C.byref(isp)))
        self.pixel = bool(isp.value)
        if num_envs is not None:
            self.d.num_envs = num_envs
        if horizon is not None:
            self.d.horizon = horizon
        self.E = self.d.num_envs
        self.p = C.c_void_p()
        _cabi.check(lib.tdmpc2_planner_create(C.byref(self.d), C.byref(self.p)))
        nb = C.c_size_t()
        u8 = lambda n: torch.empty(n, dtype=torch.uint8, device="cuda")
        _cabi.check(lib.tdmpc2_planner_packed_bytes(self.p, C.byref(nb))); self.packed = u8(nb.value)
        _cabi.check(lib.tdmpc2_planner_workspace_bytes(self.p, C.byref(nb))); self.ws = u8(nb.value)
        _cabi.check(lib.tdmpc2_planner_bind(self.p, self.packed.data_ptr(), self.ws.data_ptr()))
        _cabi.check(lib.tdmpc2_model_file_device_bytes(self.f, C.byref(self.d), C.byref(nb))); self.buf = u8(nb.value)
        self.W, self.conv, self.grid = _cabi.Weights(), _cabi.ConvWeights(), C.c_void_p()
        _cabi.check(lib.tdmpc2_model_file_upload(self.f, C.byref(self.d), self.buf.data_ptr(), C.byref(self.W), C.byref(self.conv),
                                                 C.byref(self.grid), cuda_stream()))
        _cabi.check(lib.tdmpc2_pack_weights(self.p, C.byref(self.W), cuda_stream()))
        self.enc, self.enc_ws = None, None
        if self.pixel:
            self.enc = C.c_void_p()
            _cabi.check(lib.tdmpc2_pixel_encoder_create(C.byref(self.pd), C.byref(self.enc)))
            _cabi.check(lib.tdmpc2_pixel_encoder_workspace_bytes(self.enc, C.byref(nb))); self.enc_ws = u8(nb.value)
        _cabi.check(lib.tdmpc2_act_scratch_bytes(self.p, self.enc, C.byref(nb))); self.scratch = u8(nb.value)
        self.rng_state = torch.tensor([seed, 0], dtype=torch.int64, device="cuda")
        self.prev_mean = torch.zeros(self.E, self.d.horizon, self.d.action_dim, device="cuda")
        self.action = torch.empty(self.E, self.d.action_dim, device="cuda")

    def __del__(self):
        try:
            if self.enc:
                self.lib.tdmpc2_pixel_encoder_destroy(self.enc)
            self.lib.tdmpc2_planner_destroy(self.p)
            self.lib.tdmpc2_model_file_close(self.f)
        except Exception:
            pass

    def tensor_at(self, ptr, shape):
        """The uploaded tensor at device address ptr, copied to the host."""
        off = ptr - self.buf.data_ptr()
        n = int(np.prod(shape)) * 4
        return self.buf[off:off + n].view(torch.float32).view(*shape).cpu()

    def act_rc(self, obs, t0, task=None, eval_mode=False):
        self._args = a = _cabi.ActArgs()
        self._keep = (obs, t0, task)
        a.obs, a.frames = (None, obs.data_ptr()) if self.pixel else (obs.data_ptr(), None)
        a.task = None if task is None else task.data_ptr()
        a.t0, a.eval_mode, a.rng_state = t0.data_ptr(), int(bool(eval_mode)), self.rng_state.data_ptr()
        a.prev_mean, a.action_out, a.grid_base = self.prev_mean.data_ptr(), self.action.data_ptr(), self.grid.value
        return self.lib.tdmpc2_act(self.p, self.enc, None if self.enc_ws is None else self.enc_ws.data_ptr(),
                                   C.byref(self.conv) if self.pixel else None, C.byref(a), self.scratch.data_ptr(), cuda_stream())

    def act(self, *args, **kw):
        _cabi.check(self.act_rc(*args, **kw))
        return self.action.clone(), self.prev_mean.clone()


def _inputs(cfg, E, steps, seed=3):
    g = torch.Generator().manual_seed(seed)
    if cfg.get("obs", "state") == "rgb":
        obs = [torch.randint(0, 256, (E, *cfg.obs_shape["rgb"]), generator=g).float().cuda() for _ in range(steps)]
    else:
        obs = [torch.randn(E, cfg.obs_shape["state"][0], generator=g).cuda() for _ in range(steps)]
    task = torch.tensor([e % len(cfg.tasks) for e in range(E)], dtype=torch.int32, device="cuda") if cfg.multitask else None
    return obs, task


# ------------------------------------------------------------------------------------------------------------ upload
@pytest.mark.parametrize("case", list(CASES))
def test_upload_is_the_state_dict_bit_for_bit(case, tmp_path):
    cfg, sd, path = _model(case, 2, tmp_path)
    m = CModel(path)
    torch.cuda.synchronize()
    W = m.W

    def same(ptr, key):
        want = sd[key].float().contiguous()
        got = m.tensor_at(ptr, tuple(want.shape))
        assert torch.equal(got.view(torch.int32), want.view(torch.int32)), key

    def lin(struct, pfx):
        same(struct.weight, pfx + ".weight"); same(struct.bias, pfx + ".bias")
        if pfx + ".ln.weight" in sd:
            same(struct.ln_weight, pfx + ".ln.weight"); same(struct.ln_bias, pfx + ".ln.bias")
        else:
            assert not struct.ln_weight and not struct.ln_bias

    if m.pixel:
        assert W.num_enc == 0
        for i, idx in enumerate((2, 4, 6, 8)):
            same(m.conv.weight[i], f"_encoder.rgb.{idx}.weight"); same(m.conv.bias[i], f"_encoder.rgb.{idx}.bias")
        eps = 1.0 / 70
        want = torch.linspace(-1.0 + eps, 1.0 - eps, 70, device="cuda", dtype=torch.float32)[:64].cpu()   # Planner.pix_grid
        assert torch.equal(m.tensor_at(m.grid.value, (64,)), want)
    else:
        for i in range(W.num_enc):
            lin(W.enc[i], f"_encoder.state.{i}")
        assert f"_encoder.state.{W.num_enc}.weight" not in sd
    for i in range(3):
        lin(W.dynamics[i], f"_dynamics.{i}"); lin(W.reward[i], f"_reward.{i}"); lin(W.pi[i], f"_pi.{i}")
        lin(W.qs[i], f"_Qs.params.{i}")
        if cfg.episodic:
            lin(W.termination[i], f"_termination.{i}")
    if cfg.multitask:
        same(W.task_emb, "_task_emb.weight"); same(W.action_masks, "_action_masks")
    else:
        assert not W.task_emb and not W.action_masks
    bins = torch.linspace(cfg.vmin, cfg.vmax, cfg.num_bins, device="cuda", dtype=torch.float32).cpu()   # what Planner.pack packs
    assert torch.equal(m.tensor_at(W.bins, (cfg.num_bins,)), bins)
    disc = discount_table(cfg, "cpu")
    assert torch.equal(m.tensor_at(W.discount_pow, tuple(disc.shape)), disc)


@pytest.mark.parametrize("case", ["c1", "tiny-mt"])
def test_discount_powers_follow_an_overridden_horizon(case, tmp_path):
    cfg, sd, path = _model(case, 1, tmp_path)
    for H in (1, 7):
        m = CModel(path, horizon=H)
        torch.cuda.synchronize()
        disc = discount_table(cfg.replace(horizon=H), "cpu")
        assert disc.shape[1] == H + 1
        assert torch.equal(m.tensor_at(m.W.discount_pow, tuple(disc.shape)), disc)


# ------------------------------------------------------------------------------------------------------------ draw laws
# a planner whose draws are large: prior E x 16 x 16 normals, I E qidx rows, E x 16 exponentials, E x 16 finals
LARGE_DRAWS = dict(E=65536, N=64, P=16, K=16, H=1, A=16)


def _chi2_ok(counts):
    counts = np.asarray(counts, dtype=np.float64)
    exp = counts.sum() / counts.size
    chi = float(((counts - exp) ** 2 / exp).sum())
    return chi < stats.chi2.ppf(1 - 1e-6, counts.size - 1), chi


def test_draw_laws_normals_and_exponentials():
    lib, p, d = draw_planner(I=4, num_q=5, **LARGE_DRAWS)
    st = torch.tensor([987654321, 17], dtype=torch.int64, device="cuda")
    prior, qidx, expo, final, shift = plan_draws(p, st, d, pixel=True)
    for x in (prior.flatten().double(), final.flatten().double()):
        n = x.numel()
        assert n >= 1 << 20 and torch.isfinite(x).all()
        assert abs(float(x.mean())) < 5.0 / n ** 0.5 and abs(float(x.var()) - 1.0) < 0.01
        assert abs(float((x ** 4).mean()) - 3.0) < 0.05 and abs(float((x ** 3).mean())) < 0.02
        assert abs(float((x[:-1] * x[1:]).mean())) < 0.005
    x = expo.flatten().double()
    assert x.numel() >= 1 << 20 and torch.isfinite(x).all() and bool((x >= 0).all())
    assert abs(float(x.mean()) - 1.0) < 5.0 / x.numel() ** 0.5 and abs(float(x.var()) - 1.0) < 0.02
    s = shift.flatten()
    assert torch.equal(s, s.floor()) and int(s.min()) == 0 and int(s.max()) == 6
    ok, chi = _chi2_ok(torch.bincount(s.long(), minlength=7).numpy())
    assert ok, chi
    # deterministic for the same state; every kind changes with the counter
    again = plan_draws(p, st, d, pixel=True)
    other = plan_draws(p, torch.tensor([987654321, 18], dtype=torch.int64, device="cuda"), d, pixel=True)
    for a, b, c in zip((prior, qidx, expo, final, shift), again, other):
        assert torch.equal(a, b) and not torch.equal(a, c)
    lib.tdmpc2_planner_destroy(p)


@pytest.mark.parametrize("num_q", [5, 8])
def test_draw_laws_qidx_is_an_ordered_pair_of_distinct_heads(num_q):
    lib, p, d = draw_planner(I=8, num_q=num_q, **LARGE_DRAWS)
    st = torch.tensor([42, 3], dtype=torch.int64, device="cuda")
    q = plan_draws(p, st, d)[1].view(-1, 2).long()
    assert q.shape[0] >= 1 << 19
    assert bool((q >= 0).all()) and bool((q < num_q).all()) and bool((q[:, 0] != q[:, 1]).all())
    code = q[:, 0] * num_q + q[:, 1]
    counts = torch.bincount(code, minlength=num_q * num_q).view(num_q, num_q)
    assert int(counts.diagonal().sum()) == 0
    pairs = counts[~torch.eye(num_q, dtype=torch.bool)].numpy()          # the num_q (num_q - 1) ordered pairs
    ok, chi = _chi2_ok(pairs)
    assert ok, chi
    lib.tdmpc2_planner_destroy(p)


def test_draw_streams_are_uncorrelated_with_each_other_and_the_iteration_streams():
    lib, p, d = draw_planner(I=4, num_q=5, **LARGE_DRAWS)
    st = torch.tensor([2024, 5], dtype=torch.int64, device="cuda")
    prior, qidx, expo, final, shift = plan_draws(p, st, d, pixel=True)
    n = final.numel()
    it = []
    for s in (0, 1):                                                     # tdmpc2_plan_iter_rng's streams of iteration 0
        out = torch.empty(n, device="cuda")
        _cabi.check(lib.tdmpc2_debug_rng(st.data_ptr(), s, 0, n // 4, out.data_ptr(), cuda_stream()))
        it.append(out.cpu())
    z = lambda t: (t.flatten()[:n].double() - t.flatten()[:n].double().mean()) / t.flatten()[:n].double().std()
    series = [z(prior), z(final), z(expo), z(qidx[..., 0].float()), z(shift), z(it[0]), z(it[1])]
    for i in range(len(series)):
        for j in range(i + 1, len(series)):
            if i >= 5 and j >= 5:
                continue                                                 # the two iteration streams: test_gpu_rng.py
            m = min(series[i].numel(), series[j].numel())
            r = float((series[i][:m] * series[j][:m]).mean())
            assert abs(r) < 6.0 / m ** 0.5, (i, j, r)
    lib.tdmpc2_planner_destroy(p)


# ------------------------------------------------------------------------------------------------------------ same plan
@pytest.mark.parametrize("eval_mode", [False, True])
@pytest.mark.parametrize("E", [1, 4])
@pytest.mark.parametrize("case", list(CASES))
def test_act_is_the_python_philox_plan_bit_for_bit(case, E, eval_mode, tmp_path):
    seed = 777
    cfg, sd, path = _model(case, E, tmp_path, rng="philox", rng_seed=seed)
    m = CModel(path, seed=seed)
    assert m.E == E
    pl = planner_for(cfg, E, None, sd)
    assert pl.philox and int(pl.rng_state[0]) == seed
    obs, task = _inputs(cfg, E, 3)
    prev = torch.zeros(E, cfg.horizon, cfg.action_dim, device="cuda")
    for k in range(3):
        t0 = torch.full((E,), int(k == 0), dtype=torch.uint8, device="cuda")
        nz = alloc_noise(cfg, E, "cuda", eval_mode)
        prior, qidx, expo, final, shift = plan_draws(m.p, torch.tensor([seed, k + 1], dtype=torch.int64, device="cuda"), m.d,
                                                     eval_mode, m.pixel)
        nz.prior.copy_(prior); nz.qidx.copy_(qidx); nz.expo.copy_(expo)
        if not eval_mode:
            nz.final.copy_(final)
        if m.pixel:
            nz.shift.copy_(shift)
        want_a, prev, _ = pl.plan(obs[k], task, t0, prev, nz)
        got_a, got_prev = m.act(obs[k], t0, task, eval_mode)
        torch.cuda.synchronize()
        assert int(m.rng_state[1]) == k + 1 == int(pl.rng_state[1])
        assert torch.equal(got_a, want_a), (k, (got_a - want_a).abs().max())
        assert torch.equal(got_prev, prev), k
        assert bool((got_a.abs() <= 1).all())


# ------------------------------------------------------------------------------------------------------------ counter, graphs
def test_counter_graph_replay_sync_free_and_simt(tmp_path):
    cfg, sd, path = _model("c1", 2, tmp_path)
    m = CModel(path, seed=5)
    obs, _ = _inputs(cfg, 2, 1)
    t0 = torch.zeros(2, dtype=torch.uint8, device="cuda")
    m.act(obs[0], torch.ones_like(t0))
    torch.cuda.synchronize()
    start_state, start_prev = m.rng_state.clone(), m.prev_mean.clone()
    eager = []
    torch.cuda.set_sync_debug_mode("error")
    try:
        for k in range(4):
            _cabi.check(m.act_rc(obs[0], t0))
            eager.append(m.action.clone())
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert int(m.rng_state[1]) == int(start_state[1]) + 4
    assert not torch.equal(eager[0], eager[1])                           # fresh noise every call
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        _cabi.check(m.act_rc(obs[0], t0))
    torch.cuda.synchronize()
    m.rng_state.copy_(start_state); m.prev_mean.copy_(start_prev)
    for k in range(4):
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(m.action, eager[k]), k
    assert int(m.rng_state[1]) == int(start_state[1]) + 4
    _cabi.check(m.lib.tdmpc2_planner_set_engine(m.p, _cabi.ENGINE_SIMT))
    assert m.act_rc(obs[0], t0) == -5                                    # TDMPC2_ERR_UNSUPPORTED
    assert b"tensor-core" in m.lib.tdmpc2_last_error()


# ------------------------------------------------------------------------------------------------------------ the C host
def _compile_c_act(tmp_path):
    from tdmpc2_b200.build import find_nvcc
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no gcc")
    cuda = os.path.dirname(os.path.dirname(os.path.realpath(find_nvcc())))
    libdir = os.path.dirname(_cabi.LIB_PATH)
    cudalib = next(p for p in (os.path.join(cuda, "lib64"), os.path.join(cuda, "lib"), os.path.join(cuda, "targets", "x86_64-linux", "lib"))
                   if os.path.exists(os.path.join(p, "libcudart.so")))
    exe = str(tmp_path / "c_act")
    subprocess.run([gcc, "-std=c11", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(cuda, "include"),
                    os.path.join(ROOT, "examples", "c_act.c"), "-L" + libdir, "-ltdmpc2_b200", "-L" + cudalib, "-lcudart",
                    "-Wl,-rpath," + libdir, "-Wl,-rpath," + cudalib, "-o", exe], check=True)
    return exe


@pytest.mark.parametrize("case,E", [("c1", 1), ("c1", 4), ("tiny-rgb", 4)])
def test_c_host_acts_like_the_ctypes_calls(case, E, tmp_path):
    exe = _compile_c_act(tmp_path)
    steps, seed = 3, 31
    cfg, sd, path = _model(case, 1, tmp_path)                            # exported for one environment: --envs overrides
    obs, _ = _inputs(cfg, E, steps)
    obs_path, act_path = str(tmp_path / "obs.bin"), str(tmp_path / "act.bin")
    np.concatenate([o.cpu().numpy().astype("<f4").ravel() for o in obs]).tofile(obs_path)
    res = subprocess.run([exe, path, obs_path, act_path, "--envs", str(E), "--steps", str(steps), "--seed", str(seed), "--graph", "5"],
                         capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "graph: 5 replays" in res.stdout
    got = torch.from_numpy(np.fromfile(act_path, dtype="<f4")).view(steps, E, cfg.action_dim)
    m = CModel(path, num_envs=E, seed=seed)
    for k in range(steps):
        a, _ = m.act(obs[k], torch.full((E,), int(k == 0), dtype=torch.uint8, device="cuda"))
        assert torch.equal(got[k], a.cpu()), k
