"""`RunningScale`: the running trimmed scale of the Q values that agent.update_pi divides by (reference
common/scale.py, restated from its behaviour).

`update(x)` takes the 5th and 95th percentiles of x over its first dimension (linear interpolation between the sorted
values, per remaining column), clamps their difference to at least 1 and moves `value` towards it by `cfg.tau`
(lerp).  `forward(x)` returns x / value.  The scale is a buffer outside any autograd graph.  `state_dict()` has the
reference's keys `value` and `percentiles`.
"""
from __future__ import annotations

import torch


class RunningScale(torch.nn.Module):
    def __init__(self, cfg, device=None):
        super().__init__()
        self.cfg = cfg
        dev = torch.device("cuda:0" if device is None else device)
        self.value = torch.nn.Buffer(torch.ones(1, dtype=torch.float32, device=dev))
        self._percentiles = torch.nn.Buffer(torch.tensor([5, 95], dtype=torch.float32, device=dev))

    def state_dict(self, *args, **kwargs):
        if args or kwargs:       # an enclosing module's state_dict() walking its children
            return super().state_dict(*args, **kwargs)
        return dict(value=self.value, percentiles=self._percentiles)

    def load_state_dict(self, state_dict):
        self.value.copy_(state_dict["value"])
        self._percentiles.copy_(state_dict["percentiles"])

    def _percentile(self, x: torch.Tensor) -> torch.Tensor:
        """[2, *x.shape[1:]]: the two percentiles of x along dim 0."""
        shape, n = x.shape, x.shape[0]
        xs = torch.sort(x.flatten(1), dim=0).values
        pos = self._percentiles * (n - 1) / 100
        lo = torch.floor(pos)
        hi = torch.clamp(lo + 1, max=n - 1)
        w_hi = (pos - lo).unsqueeze(1)
        out = xs[lo.long()] * (1.0 - w_hi) + xs[hi.long()] * w_hi
        return out.reshape(-1, *shape[1:]).to(x.dtype)

    @torch.no_grad()
    def update(self, x: torch.Tensor) -> None:
        p = self._percentile(x.detach())
        self.value.lerp_(torch.clamp(p[1] - p[0], min=1.0), self.cfg.tau)

    def forward(self, x, update=False):
        if update:
            self.update(x)
        return x / self.value

    def __repr__(self):
        return f"RunningScale(S: {self.value})"
