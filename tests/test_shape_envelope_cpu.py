"""The model shapes tdmpc2_planner_create accepts, at each limit and one step past it.  tests/test_gpu_shape_envelope.py
runs the kernels at these limits; this module pins that the limits are where it says they are.

Validation runs before the device check: on a machine without an H100 an accepted shape fails with
TDMPC2_ERR_NO_DEVICE, a rejected one with TDMPC2_ERR_INVALID / TDMPC2_ERR_UNSUPPORTED.  On an H100 an accepted shape
creates a planner (which is destroyed again)."""
import ctypes as C

import pytest
import torch

OK, INVALID, NO_DEVICE, UNSUPPORTED = 0, -1, -2, -5
BASE = dict(num_envs=1, num_samples=128, num_pi_trajs=8, num_elites=16, horizon=3, iterations=2, obs_dim=8,
            action_dim=4, latent_dim=64, mlp_dim=64, enc_dim=64, num_enc_layers=2, task_dim=0, num_tasks=1,
            num_q=2, num_bins=101, simnorm_dim=8, episodic=0, temperature=0.5, min_std=0.05, max_std=2.0,
            log_std_min=-10.0, log_std_dif=12.0)

# (field overrides, accepted?): each limit the GPU envelope tests reach, and the first shape past it
ENVELOPE = [
    (dict(action_dim=128), True),            # pad32(128) + 128 = 256 = kMaxHeadCols
    (dict(action_dim=129), False),           # pad32(129) + 129 = 289
    (dict(num_bins=256), True),
    (dict(num_bins=257), False),
    (dict(num_bins=2), True),
    (dict(num_bins=1), False),               # the reference's scalar regression head: not built
    (dict(latent_dim=8), True),              # one SimNorm group
    (dict(latent_dim=12), False),            # not a multiple of simnorm_dim
    (dict(num_enc_layers=8), True),          # 7 hidden + 1 output layer = TDMPC2_MAX_ENC_LAYERS
    (dict(num_enc_layers=9), False),
    (dict(num_pi_trajs=128), True),
    (dict(num_pi_trajs=129, num_samples=256), False),
    (dict(num_samples=4096), True),
    (dict(num_samples=4097), False),
    (dict(num_samples=2048, num_elites=1024), True),
    (dict(num_samples=2048, num_elites=1025), False),
    (dict(num_elites=1), True),
    (dict(num_samples=1, num_elites=1, num_pi_trajs=0), True),
    (dict(num_samples=1, num_elites=1, num_pi_trajs=1), True),   # every sample a policy-prior sample
    (dict(num_samples=1, num_elites=2, num_pi_trajs=0), False),  # more elites than samples
]


@pytest.fixture(scope="module")
def lib():
    from tdmpc2_b200 import build, _cabi
    build.build()
    return _cabi.load()


def _create(lib, **over):
    from tdmpc2_b200 import _cabi
    d = _cabi.Dims(**dict(BASE, **over))
    h = C.c_void_p()
    rc = lib.tdmpc2_planner_create(C.byref(d), C.byref(h))
    if rc == OK:
        lib.tdmpc2_planner_destroy(h)
    return rc, lib.tdmpc2_last_error().decode()


@pytest.mark.parametrize("over,accepted", ENVELOPE, ids=[",".join(f"{k}={v}" for k, v in o.items()) for o, _ in ENVELOPE])
def test_create_accepts_exactly_the_envelope(lib, over, accepted):
    rc, msg = _create(lib, **over)
    if accepted:
        assert rc == (OK if torch.cuda.is_available() else NO_DEVICE), (rc, msg)
    else:
        assert rc in (INVALID, UNSUPPORTED), (rc, msg)


def test_envelope_limits_compose(lib):
    """Every limit at once: the widest heads, the deepest encoder, the most prior trajectories and samples."""
    rc, msg = _create(lib, action_dim=128, num_bins=256, latent_dim=8, num_enc_layers=8, num_pi_trajs=128,
                      num_samples=4096, num_elites=1024)
    assert rc == (OK if torch.cuda.is_available() else NO_DEVICE), (rc, msg)
