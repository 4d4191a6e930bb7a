"""RAdam with the reference's constructor surface (ZEGGS/optimizers.py) backed by one fused kernel.

All parameters are re-homed into ONE flat fp32 buffer (each nn.Parameter becomes a view of it), with a
matching flat gradient buffer: the optimizer step is one zeggs_radam_step_dev call (two launches) and the
data-parallel gradient exchange is a single NCCL all-reduce of `flat_grad`."""
import torch

from . import _lib
from . import ops


class RAdam(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, degenerated_to_sgd=True):
        if weight_decay != 0 or not degenerated_to_sgd:
            raise _lib.ZeggsError("fused RAdam implements weight_decay=0, degenerated_to_sgd=True (train.py:160)")
        params = list(params)
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=0))
        ps = [p for g in self.param_groups for p in g["params"]]
        dev = ps[0].device
        if dev.type != "cuda":
            raise _lib.ZeggsError("fused RAdam needs CUDA parameters (no CPU fallback)")
        n = sum(p.numel() for p in ps)
        self.flat_param = torch.empty(n, dtype=torch.float32, device=dev)
        self.flat_grad = torch.zeros(n, dtype=torch.float32, device=dev)
        self.exp_avg = torch.zeros(n, dtype=torch.float32, device=dev)
        self.exp_avg_sq = torch.zeros(n, dtype=torch.float32, device=dev)
        off = 0
        for p in ps:
            k = p.numel()
            self.flat_param[off:off + k].copy_(p.data.reshape(-1))
            p.data = self.flat_param[off:off + k].view(p.shape)
            p.grad = self.flat_grad[off:off + k].view(p.shape)
            off += k
        self._step = 0
        self.grad_scale = 1.0
        # step-dependent scalars live in DEVICE memory (zeggs_radam_step_dev) so a captured CUDA graph of the step can be replayed:
        # hyper = [lr, beta1, beta2, eps, grad_scale, <scratch x3>] in float64 (the kernel forms 1 - beta and the rectification terms
        # from the host's doubles, as the reference does), step_dev = steps taken so far (incremented by the kernel)
        self.hyper = torch.zeros(8, dtype=torch.float64, device=dev)
        self.step_dev = torch.zeros(1, dtype=torch.int32, device=dev)
        self._hyper_host = None

    def sync_hyper(self):
        """Push lr / betas / eps / grad_scale to the device when they changed (call OUTSIDE graph capture; train() changes lr every
        1000 iterations through param_groups like the reference's ExponentialLR, train.py:431-432)."""
        g = self.param_groups[0]
        h = (float(g["lr"]), float(g["betas"][0]), float(g["betas"][1]), float(g["eps"]), float(self.grad_scale))
        if h != self._hyper_host:
            self.hyper[:5].copy_(torch.tensor(h, dtype=torch.float64))
            self._hyper_host = h

    def zero_grad(self, set_to_none=False):
        self.flat_grad.zero_()

    @torch.no_grad()
    def step(self, closure=None):
        loss = closure() if closure is not None else None
        capturing = torch.cuda.is_current_stream_capturing()
        if not capturing:
            self.sync_hyper()
            self._step += 1          # host mirror of step_dev (a graph replay wrapper keeps it in step, see train.GraphedStep)
        _lib.check(_lib.lib().zeggs_radam_step_dev(
            self.flat_param.data_ptr(), self.flat_grad.data_ptr(), self.exp_avg.data_ptr(), self.exp_avg_sq.data_ptr(),
            self.flat_param.numel(), self.hyper.data_ptr(), self.step_dev.data_ptr(), _lib.stream_ptr()), "zeggs_radam_step_dev")
        ops.bump_weights_epoch()     # parameters changed behind autograd's back: invalidate packed-weight caches
        return loss

    def state_dict(self):
        d = super().state_dict()
        d["zeggs"] = dict(step=self._step, exp_avg=self.exp_avg, exp_avg_sq=self.exp_avg_sq)
        return d

    def _restore_groups(self, state_dict):
        """lr / betas / eps of the checkpoint (the reference's optimizer.load_state_dict restores the DECAYED lr and its
        ExponentialLR continues from it, train.py:165-175)."""
        for g, sg in zip(self.param_groups, state_dict.get("param_groups", [])):
            for k in ("lr", "betas", "eps"):
                if k in sg:
                    g[k] = tuple(sg[k]) if k == "betas" else sg[k]
        self._hyper_host = None

    def load_state_dict(self, state_dict):
        self._restore_groups(state_dict)
        z = state_dict.get("zeggs")
        if z is not None:
            self._step = int(z["step"])
            self.step_dev.fill_(self._step)
            self.exp_avg.copy_(z["exp_avg"])
            self.exp_avg_sq.copy_(z["exp_avg_sq"])
            return
        # reference checkpoint (per-parameter state, optimizers.py:47-56)
        ps = [p for g in self.param_groups for p in g["params"]]
        off = 0
        for i, p in enumerate(ps):
            st = state_dict["state"].get(i)
            k = p.numel()
            if st is not None:
                self._step = int(st["step"])
                self.exp_avg[off:off + k].copy_(st["exp_avg"].reshape(-1))
                self.exp_avg_sq[off:off + k].copy_(st["exp_avg_sq"].reshape(-1))
            off += k
        self.step_dev.fill_(self._step)
