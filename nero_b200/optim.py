"""Adam over the flat parameter / gradient buffers of a nero_b200 renderer: ONE kernel per step.

The reference trains with `torch.optim.Adam(network.parameters(), lr=1e-3)` and sets the learning rate of
`param_groups[0]` every step (train/trainer.py:73-76, 160-166; train/lr_common_manager.py).  `FlatAdam` keeps that
surface (`param_groups[0]['lr']`, `step()`, `zero_grad()`, torch-compatible `state_dict()` / `load_state_dict()`) but
re-homes all parameters as views of one flat fp32 buffer, matching the flat gradient buffer the engines already own
(`engine.Grads`), and updates it with `nero_adam_flat`.  Arithmetic follows torch's Adam (amsgrad=False) operation by
operation; results agree with `torch.optim.Adam` to rounding.
"""
import math

import torch

from . import ops


class FlatAdam(torch.optim.Optimizer):
    def __init__(self, net, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0):
        params = [p for p in net.parameters()]
        assert params and all(p.dtype == torch.float32 for p in params)
        dev = params[0].device
        ops.require_cuda(dev, 'FlatAdam')
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        self.net = net
        self.params = params
        self.sizes = [p.numel() for p in params]
        total = sum(self.sizes)
        self.flat_p = torch.empty(total, dtype=torch.float32, device=dev)
        off = 0
        with torch.no_grad():
            for p, n in zip(params, self.sizes):
                self.flat_p[off:off + n].copy_(p.detach().reshape(-1))
                p.data = self.flat_p[off:off + n].view(p.shape)      # parameters become views of the flat buffer
                off += n
        self.exp_avg = torch.zeros_like(self.flat_p)
        self.exp_avg_sq = torch.zeros_like(self.flat_p)
        self.t = 0
        self._flat_g = None

    # ------------------------------------------------------------------ gradients
    def _gather_grads(self):
        """The engines hand out every .grad as a view of one flat buffer in parameter order (engine.Grads); use it in place
        when that holds, otherwise pack the gradients (e.g. after an external backward that created its own tensors)."""
        g = getattr(self.net.engine.grads, 'flat', None)
        if g is not None and g.numel() == self.flat_p.numel():
            off, ok = 0, True
            for p, n in zip(self.params, self.sizes):
                if p.grad is None or p.grad.data_ptr() != g.data_ptr() + 4 * off:
                    ok = False
                    break
                off += n
            if ok:
                return g
        if self._flat_g is None:
            self._flat_g = torch.zeros_like(self.flat_p)
        off = 0
        for p, n in zip(self.params, self.sizes):
            if p.grad is None:
                self._flat_g[off:off + n].zero_()
            else:
                self._flat_g[off:off + n].copy_(p.grad.reshape(-1))
            off += n
        return self._flat_g

    def zero_grad(self, set_to_none=True):
        # dropping the views lets the engine allocate one zeroed flat buffer on the next backward (one memset)
        for p in self.params:
            p.grad = None

    @torch.no_grad()
    def step(self, closure=None):
        assert closure is None
        grp = self.param_groups[0]
        b1, b2 = grp['betas']
        self.t += 1
        bc1 = 1.0 - b1 ** self.t
        bc2 = 1.0 - b2 ** self.t
        g = self._gather_grads()
        ops.K('nero_adam_flat', self.flat_p, g, self.exp_avg, self.exp_avg_sq, self.flat_p.numel(), float(grp['lr'] / bc1), float(b1),
              float(b2), float(grp['eps']), float(1.0 / math.sqrt(bc2)), float(grp['weight_decay']))

    # ------------------------------------------------------------------ torch.optim.Adam-compatible checkpoints
    def state_dict(self):
        st, off = {}, 0
        for i, n in enumerate(self.sizes):
            shp = self.params[i].shape
            st[i] = {'step': torch.tensor(float(self.t)), 'exp_avg': self.exp_avg[off:off + n].view(shp).clone(),
                     'exp_avg_sq': self.exp_avg_sq[off:off + n].view(shp).clone()}
            off += n
        grp = {k: v for k, v in self.param_groups[0].items() if k != 'params'}
        grp['params'] = list(range(len(self.params)))
        return {'state': st if self.t > 0 else {}, 'param_groups': [grp]}

    def load_state_dict(self, sd):
        grp = sd['param_groups'][0]
        for k in ('lr', 'betas', 'eps', 'weight_decay'):
            if k in grp:
                self.param_groups[0][k] = grp[k]
        off = 0
        for i, n in enumerate(self.sizes):
            s = sd['state'].get(i, sd['state'].get(str(i)))
            if s is not None:
                self.exp_avg[off:off + n].copy_(s['exp_avg'].reshape(-1))
                self.exp_avg_sq[off:off + n].copy_(s['exp_avg_sq'].reshape(-1))
                self.t = int(float(s['step']))
            off += n
