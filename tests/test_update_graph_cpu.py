"""cfg.compile without a GPU: the option is off by default, and with it on a CPU agent's `_update` refuses exactly as it
does without it (there is no CPU fallback, graphed or not)."""
import pytest
import torch

from tdmpc2_b200.config import workload
from tdmpc2_b200.tdmpc2 import TDMPC2


def test_compile_defaults_to_false():
    assert workload("tiny").compile is False
    assert workload("c1").compile is False
    assert TDMPC2(workload("tiny"), device="cpu")._compile is False


@pytest.mark.parametrize("kw", [{}, {"td_eps": torch.zeros(2, 4, 6)}])
def test_compiled_cpu_agent_refuses_as_before(kw):
    H, B = 2, 4
    for compile_ in (False, True):
        cfg = workload("tiny", compile=compile_)
        agent = TDMPC2(cfg, device="cpu")
        args = (torch.zeros(H + 1, B, cfg.obs_shape["state"][0]), torch.zeros(H, B, cfg.action_dim), torch.zeros(H, B, 1),
                torch.zeros(H, B, 1))
        with pytest.raises(RuntimeError, match="_update runs on the sm_90a kernels: the agent needs a CUDA device"):
            agent._update(*args, **kw)
        rgb = workload("tiny", obs="rgb", num_channels=4, latent_dim=64, compile=compile_)
        pix = TDMPC2(rgb, device="cpu")
        with pytest.raises(NotImplementedError, match="pixel `_update` runs on the sm_90a conv encoder kernels"):
            pix._update(torch.zeros(H + 1, B, 3, 64, 64), *args[1:])
        assert agent._planner is None and pix._planner is None
