"""The model file a C host plans from (tdmpc2_b200/export.py, tdmpc2_model_file_* of include/tdmpc2_b200.h), on the host
alone: agent.export writes the state dict's tensors and the planner's dims, tdmpc2_model_file_open reads them back field
for field, and every malformed file is refused with a message naming the problem."""
import ctypes as C
import json
import os
import struct

import numpy as np
import pytest
import torch

from tdmpc2_b200.config import workload
from tdmpc2_b200.synth import synth_state_dict

CASES = {"c1": ("c1", {}), "tiny-mt": ("tiny-mt", {}), "episodic": ("tiny", {"episodic": True}), "tiny-rgb": ("tiny-rgb", {}),
         "legacy": ("tiny", {})}
ERR_INVALID = -1


@pytest.fixture(scope="module")
def lib():
    from tdmpc2_b200 import build, _cabi
    build.build()
    return _cabi.load()


def _open(lib, path):
    """-> (rc, message, handle or None)"""
    h = C.c_void_p()
    rc = lib.tdmpc2_model_file_open(str(path).encode(), C.byref(h))
    return rc, lib.tdmpc2_last_error().decode(), (h if rc == 0 else None)


def _read(path):
    """(header dict, data bytes) of a safetensors file, parsed with json + struct."""
    b = open(path, "rb").read()
    n = struct.unpack("<Q", b[:8])[0]
    return json.loads(b[8:8 + n]), b[8 + n:]


def _write(path, header, data, pad=True):
    h = json.dumps(header).encode()
    if pad:
        h += b" " * (-len(h) % 8)
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", len(h)) + h + data)


def _legacy(sd):
    """The pre-compile-API checkpoint layout of sd: _Qs.params.<n> / _target_Qs.params.<n> (layers.py:167-221)."""
    out = {k: v for k, v in sd.items() if "Qs" not in k}
    for layer in range(3):
        for j, nm in enumerate(("weight", "bias", "ln.weight", "ln.bias")):
            key = f"{layer}.{nm}"
            if "_Qs.params." + key in sd:
                out[f"_Qs.params.{4 * layer + j}"] = sd["_Qs.params." + key]
                out[f"_target_Qs.params.{4 * layer + j}"] = sd["_target_Qs_params." + key]
    return out


def _f32(x):
    return struct.unpack("<f", struct.pack("<f", float(x)))[0]


def _exported(case, tmp_path):
    from tdmpc2_b200.tdmpc2 import TDMPC2
    wl, over = CASES[case]
    cfg = workload(wl, **over)
    agent = TDMPC2(cfg, device="cpu")
    sd = synth_state_dict(agent.cfg, seed=4, perturb=True)
    agent.load(_legacy(sd) if case == "legacy" else sd)
    path = tmp_path / f"{case}.tdmpc2"
    agent.export(str(path))
    return agent.cfg, sd, path


@pytest.mark.parametrize("case", list(CASES))
def test_export_round_trips_through_the_c_reader(lib, case, tmp_path):
    from tdmpc2_b200 import _cabi
    from tdmpc2_b200.config import get_discount
    cfg, sd, path = _exported(case, tmp_path)
    rc, msg, h = _open(lib, path)
    assert rc == 0, msg
    d, pd, isp = _cabi.Dims(), _cabi.PixelDims(), C.c_int32()
    assert lib.tdmpc2_model_file_dims(h, C.byref(d), C.byref(pd), C.byref(isp)) == 0
    rgb = cfg.get("obs", "state") == "rgb"
    want = dict(num_envs=cfg.num_envs, num_samples=cfg.num_samples, num_pi_trajs=cfg.num_pi_trajs, num_elites=cfg.num_elites,
                horizon=cfg.horizon, iterations=cfg.iterations, obs_dim=1 if rgb else cfg.obs_shape["state"][0],
                action_dim=cfg.action_dim, latent_dim=cfg.latent_dim, mlp_dim=cfg.mlp_dim, enc_dim=cfg.enc_dim,
                num_enc_layers=0 if rgb else cfg.num_enc_layers, task_dim=cfg.task_dim if cfg.multitask else 0,
                num_tasks=len(cfg.tasks) if cfg.multitask else 1, num_q=cfg.num_q, num_bins=cfg.num_bins,
                simnorm_dim=cfg.simnorm_dim, episodic=int(bool(cfg.episodic)), temperature=_f32(cfg.temperature),
                min_std=_f32(cfg.min_std), max_std=_f32(cfg.max_std), log_std_min=_f32(cfg.log_std_min),
                log_std_dif=_f32(float(cfg.log_std_max) - float(cfg.log_std_min)))
    assert {n: getattr(d, n) for n, _ in d._fields_} == want
    assert cfg.iterations_effective and (case != "c1" or cfg.iterations == 8)       # tdmpc2.py:34's += 2 for A >= 20
    assert isp.value == int(rgb)
    if rgb:
        assert (pd.in_channels, pd.num_channels, pd.simnorm_dim) == (cfg.obs_shape["rgb"][0], cfg.num_channels, cfg.simnorm_dim)
    nb = C.c_size_t()
    assert lib.tdmpc2_model_file_device_bytes(h, C.byref(d), C.byref(nb)) == 0 and nb.value > 0
    lib.tdmpc2_model_file_close(h)

    header, data = _read(path)
    meta = header.pop("__metadata__")
    assert meta["format"] == "tdmpc2_b200.model" and meta["version"] == "1" and meta["obs"] == ("rgb" if rgb else "state")
    assert all(isinstance(v, str) for v in meta.values())
    model_keys = {k for k in sd if not k.startswith(("_detach_", "_target_", "log_std"))}
    assert set(header) == model_keys | {"tdmpc2.bins", "tdmpc2.discount"} | ({"tdmpc2.grid_base"} if rgb else set())
    for k in model_keys:                                                 # every tensor's bytes are the state dict's
        e = header[k]
        assert e["dtype"] == "F32" and e["shape"] == list(sd[k].shape), k
        assert data[e["data_offsets"][0]:e["data_offsets"][1]] == sd[k].float().contiguous().numpy().astype("<f4").tobytes(), k
    e = header["tdmpc2.discount"]
    disc = np.frombuffer(data[e["data_offsets"][0]:e["data_offsets"][1]], dtype="<f8")
    eps = cfg.episode_lengths if cfg.multitask else [cfg.episode_length]
    assert e["dtype"] == "F64" and disc.tolist() == [get_discount(cfg, ep) for ep in eps]
    e = header["tdmpc2.bins"]
    bins = np.frombuffer(data[e["data_offsets"][0]:e["data_offsets"][1]], dtype="<f4")
    assert bins.shape == (cfg.num_bins,) and bins[0] == cfg.vmin and bins[-1] == cfg.vmax
    np.testing.assert_allclose(bins, np.linspace(cfg.vmin, cfg.vmax, cfg.num_bins), rtol=0, atol=1e-6)

    try:
        from safetensors import safe_open
    except ImportError:
        return
    with safe_open(str(path), framework="pt") as f:
        assert set(f.keys()) == set(header) and f.metadata() == meta
        for k in model_keys:
            assert torch.equal(f.get_tensor(k), sd[k].float()), k


def test_device_bytes_take_planning_overrides_but_not_model_changes(lib, tmp_path):
    from tdmpc2_b200 import _cabi
    cfg, sd, path = _exported("tiny-mt", tmp_path)
    rc, msg, h = _open(lib, path)
    d = _cabi.Dims()
    assert lib.tdmpc2_model_file_dims(h, C.byref(d), None, None) == 0
    nb, nb2 = C.c_size_t(), C.c_size_t()
    assert lib.tdmpc2_model_file_device_bytes(h, C.byref(d), C.byref(nb)) == 0
    for field, value in (("num_envs", 64), ("num_samples", 256), ("num_pi_trajs", 0), ("num_elites", 8), ("iterations", 9),
                         ("temperature", 2.0), ("min_std", 0.1), ("max_std", 1.0)):
        d2 = _cabi.Dims.from_buffer_copy(d)
        setattr(d2, field, value)
        assert lib.tdmpc2_model_file_device_bytes(h, C.byref(d2), C.byref(nb2)) == 0, field
        assert nb2.value == nb.value, field
    d2 = _cabi.Dims.from_buffer_copy(d)
    d2.horizon = d.horizon + 60                                          # discount_pow grows with the horizon
    assert lib.tdmpc2_model_file_device_bytes(h, C.byref(d2), C.byref(nb2)) == 0 and nb2.value > nb.value
    for field, value in (("latent_dim", 128), ("mlp_dim", 32), ("num_q", 2), ("num_bins", 51), ("task_dim", 8), ("obs_dim", 12),
                         ("episodic", 1), ("log_std_min", -5.0)):
        d2 = _cabi.Dims.from_buffer_copy(d)
        setattr(d2, field, value)
        assert lib.tdmpc2_model_file_device_bytes(h, C.byref(d2), C.byref(nb2)) == ERR_INVALID, field
        assert (field in lib.tdmpc2_last_error().decode()) or field == "log_std_min", lib.tdmpc2_last_error()
    lib.tdmpc2_model_file_close(h)


def _malformed(tmp_path):
    """(name, bytes-editing function, expected message fragment) for each way a file can be malformed."""
    def edit_header(fn):
        def go(path):
            header, data = _read(path)
            fn(header, data)
            _write(path, header, data)
        return go

    def truncate(n):
        def go(path):
            b = open(path, "rb").read()
            open(path, "wb").write(b[:n] if n >= 0 else b[:len(b) + n])
        return go

    def header_len(path):
        b = bytearray(open(path, "rb").read())
        b[:8] = struct.pack("<Q", len(b))
        open(path, "wb").write(bytes(b))

    def setmeta(k, v):
        return edit_header(lambda h, d: h["__metadata__"].__setitem__(k, v))

    def overlap(h, d):
        a, b = h["_pi.0.bias"]["data_offsets"], h["_pi.0.ln.bias"]["data_offsets"]
        h["_pi.0.ln.bias"]["data_offsets"] = [a[0] + 4, a[0] + 4 + (b[1] - b[0])]

    def out_of_range(h, d):
        e = h["_reward.1.bias"]["data_offsets"]
        h["_reward.1.bias"]["data_offsets"] = [len(d) - 4, len(d) - 4 + (e[1] - e[0])]

    def reversed_offsets(h, d):
        e = h["_reward.1.bias"]["data_offsets"]
        h["_reward.1.bias"]["data_offsets"] = [e[1], e[0]]

    def transpose(h, d):
        h["_reward.2.weight"]["shape"] = h["_reward.2.weight"]["shape"][::-1]

    return [
        ("short", truncate(5), "truncated file: 5 bytes"),
        ("cut data", truncate(-100), "out of range"),
        ("header length", header_len, "runs past the end of the file"),
        ("dtype", edit_header(lambda h, d: h["_dynamics.0.weight"].__setitem__("dtype", "F16")), "dtype F16, expected F32"),
        ("discount dtype", edit_header(lambda h, d: h["tdmpc2.discount"].__setitem__("dtype", "F32")), "dtype F32, expected F64"),
        ("overlap", edit_header(overlap), "overlap"),
        ("out of range", edit_header(out_of_range), "out of range"),
        ("reversed", edit_header(reversed_offsets), "out of range"),
        ("format", setmeta("format", "pytorch"), "not a tdmpc2_b200 model file"),
        ("no format", edit_header(lambda h, d: h["__metadata__"].pop("format")), "not a tdmpc2_b200 model file"),
        ("version", setmeta("version", "2"), "version '2' is not supported"),
        ("missing tensor", edit_header(lambda h, d: h.pop("_dynamics.1.weight")), "missing tensor '_dynamics.1.weight'"),
        ("missing bins", edit_header(lambda h, d: h.pop("tdmpc2.bins")), "missing tensor 'tdmpc2.bins'"),
        ("missing dims field", edit_header(lambda h, d: h["__metadata__"].pop("latent_dim")), "missing __metadata__ field 'latent_dim'"),
        ("shape", edit_header(transpose), "tensor '_reward.2.weight' has shape [64, 101], the dims need [101, 64]"),
        ("dims vs shapes", setmeta("mlp_dim", "32"), "the dims need"),
        ("json", lambda p: open(p, "r+b").write(struct.pack("<Q", 2) + b"{["), "malformed JSON header"),
    ]


@pytest.mark.parametrize("name", [m[0] for m in _malformed(None)])
def test_malformed_files_are_refused_with_the_reason(lib, name, tmp_path):
    _, _, path = _exported("episodic", tmp_path)
    rc, msg, h = _open(lib, path)
    assert rc == 0, msg
    lib.tdmpc2_model_file_close(h)
    edit, want = {m[0]: m[1:] for m in _malformed(tmp_path)}[name]
    edit(str(path))
    rc, msg, h = _open(lib, path)
    assert rc == ERR_INVALID and h is None, (rc, msg)
    assert want in msg, msg
    assert str(path) in msg


def test_missing_file_is_refused(lib, tmp_path):
    rc, msg, _ = _open(lib, tmp_path / "nope.tdmpc2")
    assert rc == ERR_INVALID and "cannot open" in msg
