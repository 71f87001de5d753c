"""tf.train.AdamOptimizer (TF 1.3, training_posenet.py:67 / training_handsegnet.py:67) over the project's multi-tensor Adam kernel
(h3d_adam_step).

    opt = Adam(ctx.variables("PoseNet2D").values(), lr=1e-4)
    loss.backward(); opt.step(); opt.zero_grad()

The update is TF's ApplyAdam, the "epsilon-hat" form p -= lr sqrt(1 - b2^t) / (1 - b1^t) m / (sqrt(v) + eps), evaluated in fp32 in TF's
operation order.  torch.optim.Adam adds eps after the bias correction instead, which differs visibly for small gradients.  The learning
rate and the beta powers live on the device, so one step (every parameter in one launch) can be captured into a CUDA graph and
replayed; set_lr() rewrites the device learning rate between replays.
"""
from __future__ import annotations

import torch

from . import _lib, runtime


class Adam(torch.optim.Optimizer):
    """Adam with TF 1.3 semantics on CUDA fp32 contiguous parameters of one device (one parameter group).

    zero_grad() zeroes the gradients in place rather than dropping them: the kernel's table holds their addresses, and a captured
    step needs them to stay put.  state_dict() / load_state_dict() carry m, v and the beta powers."""

    def __init__(self, params, lr, beta1=0.9, beta2=0.999, epsilon=1e-8):
        super().__init__(params, dict(lr=float(lr), beta1=float(beta1), beta2=float(beta2), epsilon=float(epsilon)))
        if len(self.param_groups) != 1:
            raise ValueError("hand3d_b200.optim.Adam takes one parameter group")
        ps = self.param_groups[0]["params"]
        if not ps:
            raise ValueError("hand3d_b200.optim.Adam got no parameters")
        dev = ps[0].device
        for p in ps:
            if not p.is_cuda or p.dtype != torch.float32 or not p.is_contiguous() or p.device != dev:
                raise TypeError("hand3d_b200.optim.Adam takes contiguous float32 CUDA parameters of one device, got %s %s on %s"
                                % (p.dtype, tuple(p.shape), p.device))
        self._ctx = runtime.default_context(dev)
        for p in ps:
            self.state[p]["m"] = torch.zeros_like(p)
            self.state[p]["v"] = torch.zeros_like(p)
        # [lr, beta1_power, beta2_power, ticket]: the accumulators start at beta1 and beta2 (AdamOptimizer._create_slots)
        self._dev_state = torch.zeros(_lib.ADAM_STATE_WORDS, dtype=torch.float32, device=dev)
        g = self.param_groups[0]
        self._ctx.adam_state_set(self._dev_state, g["lr"], g["beta1"], g["beta2"])
        self._table, self._table_key = None, None

    def _params(self):
        return self.param_groups[0]["params"]

    def set_lr(self, lr):
        """Writes the learning rate of the following steps to the device (e.g. LearningRateScheduler.get_lr(step))."""
        self.param_groups[0]["lr"] = float(lr)
        self._ctx.adam_set_lr(self._dev_state, float(lr))

    def zero_grad(self, set_to_none=False):
        if set_to_none:
            raise ValueError("hand3d_b200.optim.Adam zeroes gradients in place (its kernel table holds their addresses)")
        for p in self._params():
            if p.grad is not None:
                p.grad.zero_()

    def _table_for(self, ps):
        key = tuple((p.data_ptr(), p.grad.data_ptr(), self.state[p]["m"].data_ptr(), self.state[p]["v"].data_ptr(), p.numel()) for p in ps)
        if key != self._table_key:        # rebuilt only when an address changed (never between the replays of a captured step)
            self._table = torch.tensor(key, dtype=torch.int64).to(ps[0].device)
            self._table_key = key
        return self._table

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        ps = self._params()
        for p in ps:
            if p.grad is None:
                raise RuntimeError("hand3d_b200.optim.Adam: a parameter of shape %s has no gradient (TF's minimize updates every "
                                   "variable it differentiates)" % (tuple(p.shape),))
            if p.grad.dtype != torch.float32 or not p.grad.is_contiguous():
                raise TypeError("hand3d_b200.optim.Adam: gradients must be contiguous float32")
        g = self.param_groups[0]
        self._ctx.adam_step(self._table_for(ps), len(ps), self._dev_state, g["beta1"], g["beta2"], g["epsilon"])
        return loss

    def beta_powers(self):
        """(beta1^t, beta2^t) as the device holds them (a host read)."""
        return tuple(self._dev_state[1:3].tolist())

    def state_dict(self):
        sd = super().state_dict()
        sd["beta_powers"] = self.beta_powers()
        return sd

    def load_state_dict(self, state_dict):
        sd = dict(state_dict)
        powers = sd.pop("beta_powers")
        super().load_state_dict(sd)
        for p in self._params():          # own, contiguous copies: the kernel writes m and v in place
            for k in ("m", "v"):
                self.state[p][k] = self.state[p][k].to(device=p.device, dtype=torch.float32).clone(memory_format=torch.contiguous_format)
        self._table_key = None
        self._ctx.adam_state_set(self._dev_state, self.param_groups[0]["lr"], powers[0], powers[1])
