"""The optimizers of train.py:123-128 on the device.

`Adam` and `SGD` are `torch.optim.Optimizer`s with torch's constructor signature (for the supported subset), parameter
groups and state keys, so the reference's `get_params` (utils/solver.py) and its schedulers drive them unchanged and their
`state_dict()` loads into `torch.optim.Adam` / `torch.optim.SGD` and back.  `step()` runs two launches of csrc/optim.cu over
every parameter that has a gradient: a check of all gradients for inf / NaN, then, unless one was found, the update of all
tensors at once.  A step with a non-finite gradient changes nothing and sets `found_inf`; `LossScaler` turns that into the
dynamic loss scaling of the reference's fp16 mode (apex O1, train.py:136-137, 342-345)."""
import numpy as np
import torch

from . import _lib as L

_ROW = np.dtype(L.step_optim_tensor)
_BLOCK = np.dtype(L.step_optim_block)


class _DeviceTables:
    """Per-device launch buffers: the row table (pinned host staging + device copy), the block map (rebuilt only when the
    tensor sizes change) and the non-finite flag."""

    def __init__(self, dev):
        self.dev = dev
        self.flag = torch.zeros((1,), dtype=torch.int32, device=dev)
        self.rows = 0
        self.numels = None
        self.copied = None

    def host_rows(self, n):
        """Structured numpy view (step_optim_tensor rows) of pinned memory, safe to overwrite."""
        if n > self.rows:
            self.rows = max(n, 2 * self.rows)
            self.pinned = torch.empty((self.rows * _ROW.itemsize,), dtype=torch.uint8, pin_memory=True)
            self.table = torch.empty((self.rows * _ROW.itemsize,), dtype=torch.uint8, device=self.dev)
            self.copied = None
        if self.copied is not None:
            self.copied.synchronize()             # the previous step's upload has left the staging buffer
        arr = self.pinned.numpy().view(_ROW)[:n]
        arr[:] = np.zeros((), dtype=_ROW)
        return arr

    def upload(self, n):
        nbytes = n * _ROW.itemsize
        self.table[:nbytes].copy_(self.pinned[:nbytes], non_blocking=True)
        self.copied = torch.cuda.Event()
        self.copied.record()

    def block_map(self, numels):
        if numels != self.numels:
            chunk = L.lib().step_multi_tensor_chunk()
            counts = (np.asarray(numels, dtype=np.int64) + chunk - 1) // chunk
            first = np.repeat(np.cumsum(counts) - counts, counts)
            m = np.zeros((int(counts.sum()),), dtype=_BLOCK)
            m["tensor"] = np.repeat(np.arange(len(numels), dtype=np.int32), counts)
            m["chunk"] = np.arange(m.shape[0], dtype=np.int64) - first
            self.blocks = torch.from_numpy(m.view(np.uint8).copy()).to(self.dev)
            self.n_blocks = m.shape[0]
            self.numels = numels
        return self.blocks, self.n_blocks


class _MultiTensorOptimizer(torch.optim.Optimizer):
    _REJECT = {}        # option -> default; other values raise ValueError (construction, and each step for loaded groups)
    _IGNORED = {}       # torch's implementation switches: rejected at construction, carried as-is in loaded groups

    def __init__(self, params, defaults):
        for k, d in {**self._REJECT, **self._IGNORED}.items():
            if defaults[k] != d:
                raise ValueError("%s: %s=%r is not supported (only %r)" % (type(self).__name__, k, defaults[k], d))
        super().__init__(params, defaults)
        self.found_inf = False
        self._tables = {}

    def __setstate__(self, state):
        super().__setstate__(state)
        for group in self.param_groups:
            for k, d in {**self._REJECT, **self._IGNORED}.items():
                group.setdefault(k, d)
        self.__dict__.setdefault("found_inf", False)
        self.__dict__.setdefault("_tables", {})

    def _fill(self, arr, rows):
        """Fills the optimizer's columns of the row table; returns the state of parameters updated for the first time
        (kept only if the step is applied)."""
        raise NotImplementedError

    def _commit(self, rows, new_state):
        raise NotImplementedError

    def _launch(self, lib):
        raise NotImplementedError

    @torch.no_grad()
    def step(self, closure=None):
        """One update of every parameter that has a gradient, or none if any gradient holds inf or NaN (then `found_inf`
        is True and parameters, state and step counts are unchanged)."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        rows = []
        for group in self.param_groups:
            for k, d in self._REJECT.items():
                if group.get(k, d) != d:
                    raise ValueError("%s: %s=%r is not supported (only %r)" % (type(self).__name__, k, group[k], d))
            for p in group["params"]:
                if p.grad is not None:
                    rows.append((group, p))
        self.found_inf = False
        if not rows:
            return loss
        dev = L.same_device(*[t for _, p in rows for t in (p, p.grad)])
        grads = []
        for _, p in rows:
            if p.dtype != torch.float32 or p.grad.dtype != torch.float32 or p.grad.is_sparse:
                raise RuntimeError("%s: fp32 dense parameters and gradients only (got %s / %s)"
                                   % (type(self).__name__, p.dtype, p.grad.dtype))
            if not p.is_contiguous() or p.grad.shape != p.shape:
                raise RuntimeError("%s: parameters must be contiguous and match their gradient's shape" % type(self).__name__)
            grads.append(p.grad if p.grad.is_contiguous() else p.grad.contiguous())
        tables = self._tables.get(dev)
        if tables is None:
            tables = self._tables[dev] = _DeviceTables(dev)
        lib = L.lib()
        with torch.cuda.device(dev):
            n = len(rows)
            arr = tables.host_rows(n)
            arr["param"] = [p.data_ptr() for _, p in rows]
            arr["grad"] = [g.data_ptr() for g in grads]
            arr["numel"] = [p.numel() for _, p in rows]
            new_state = self._fill(arr, rows)
            tables.upload(n)
            blocks, nb = tables.block_map(tuple(int(x) for x in arr["numel"]))
            table = L.c_void_p(tables.table.data_ptr())
            L.check(lib.step_multi_tensor_nonfinite_f32(table, n, L.ptr(blocks), nb, L.ptr(tables.flag), L.stream()))
            if int(tables.flag.item()) != 0:
                self.found_inf = True
                return loss
            self._commit(rows, new_state)
            L.check(self._launch(lib)(table, n, L.ptr(blocks), nb, L.stream()))
        torch.autograd.graph.increment_version([p for _, p in rows])   # the fp16 / permuted weight caches key on _version
        return loss


class Adam(_MultiTensorOptimizer):
    """torch.optim.Adam with amsgrad=False, maximize=False and L2 weight decay added to the gradient (not AdamW), for fp32
    CUDA parameters.  State: `step` (CPU float32 scalar tensor), `exp_avg`, `exp_avg_sq`, as torch's non-capturable path."""
    _REJECT = {"amsgrad": False, "maximize": False, "decoupled_weight_decay": False}
    _IGNORED = {"foreach": None, "capturable": False, "differentiable": False, "fused": None}

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False, *, foreach=None,
                 maximize=False, capturable=False, differentiable=False, fused=None, decoupled_weight_decay=False):
        if not 0.0 <= lr:
            raise ValueError("Invalid learning rate: %r" % lr)
        if not 0.0 <= eps:
            raise ValueError("Invalid epsilon value: %r" % eps)
        if not 0.0 <= betas[0] < 1.0 or not 0.0 <= betas[1] < 1.0:
            raise ValueError("Invalid beta parameters: %r" % (betas,))
        if not 0.0 <= weight_decay:
            raise ValueError("Invalid weight_decay value: %r" % weight_decay)
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=amsgrad,
                                      foreach=foreach, maximize=maximize, capturable=capturable, differentiable=differentiable,
                                      fused=fused, decoupled_weight_decay=decoupled_weight_decay))

    def _fill(self, arr, rows):
        new_state, m, v, steps = {}, [], [], []
        for group, p in rows:
            st = self.state.get(p)
            if not st:
                st = new_state[p] = dict(step=torch.tensor(0.0, dtype=torch.float32),
                                         exp_avg=torch.zeros_like(p, memory_format=torch.preserve_format),
                                         exp_avg_sq=torch.zeros_like(p, memory_format=torch.preserve_format))
            for k in ("exp_avg", "exp_avg_sq"):
                if st[k].device != p.device or st[k].dtype != torch.float32 or not st[k].is_contiguous() or st[k].shape != p.shape:
                    raise RuntimeError("Adam: state %s of a %s parameter is not a contiguous fp32 tensor of its shape on %s"
                                       % (k, tuple(p.shape), p.device))
            m.append(st["exp_avg"].data_ptr())
            v.append(st["exp_avg_sq"].data_ptr())
            steps.append(st["step"])
        arr["exp_avg"], arr["exp_avg_sq"] = m, v
        t = torch.stack(steps).to(torch.float64).add_(1).tolist()
        cols = []
        for (group, _), ti in zip(rows, t):
            # in double as torch's _single_tensor_adam, rounded to float where its kernels take them
            beta1, beta2 = (float(b) for b in group["betas"])
            # torch divides by the host scalar bias_correction2_sqrt as a multiply by its reciprocal, taken in double
            cols.append((float(group["lr"]) / (1 - beta1 ** ti), 1.0 / (1 - beta2 ** ti) ** 0.5, 1 - beta1, beta2, 1 - beta2))
        for k, col in zip(("step_size", "inv_bias_correction2_sqrt", "one_minus_beta1", "beta2", "one_minus_beta2"), zip(*cols)):
            arr[k] = col
        arr["weight_decay"] = [float(g["weight_decay"]) for g, _ in rows]
        arr["eps"] = [float(g["eps"]) for g, _ in rows]
        return new_state

    def _commit(self, rows, new_state):
        self.state.update(new_state)
        torch._foreach_add_([self.state[p]["step"] for _, p in rows], 1.0)

    def _launch(self, lib):
        return lib.step_multi_tensor_adam_f32


class SGD(_MultiTensorOptimizer):
    """torch.optim.SGD with dampening=0, nesterov=False and maximize=False, for fp32 CUDA parameters.  State:
    `momentum_buffer` (when momentum != 0), set to the first step's gradient as torch does."""
    _REJECT = {"dampening": 0, "nesterov": False, "maximize": False}
    _IGNORED = {"foreach": None, "differentiable": False, "fused": None}

    def __init__(self, params, lr=1e-3, momentum=0, dampening=0, weight_decay=0, nesterov=False, *, maximize=False,
                 foreach=None, differentiable=False, fused=None):
        if not 0.0 <= lr:
            raise ValueError("Invalid learning rate: %r" % lr)
        if not 0.0 <= momentum:
            raise ValueError("Invalid momentum value: %r" % momentum)
        if not 0.0 <= weight_decay:
            raise ValueError("Invalid weight_decay value: %r" % weight_decay)
        super().__init__(params, dict(lr=lr, momentum=momentum, dampening=dampening, weight_decay=weight_decay,
                                      nesterov=nesterov, maximize=maximize, foreach=foreach, differentiable=differentiable,
                                      fused=fused))

    def _fill(self, arr, rows):
        new_state, bufs, init = {}, [], []
        for group, p in rows:
            if float(group["momentum"]) == 0.0:
                bufs.append(0)
                init.append(0)
                continue
            b = self.state.get(p, {}).get("momentum_buffer")
            if b is None:
                b = torch.empty_like(p, memory_format=torch.preserve_format)
                new_state[p] = b
            elif b.device != p.device or b.dtype != torch.float32 or not b.is_contiguous() or b.shape != p.shape:
                raise RuntimeError("SGD: momentum_buffer of a %s parameter is not a contiguous fp32 tensor of its shape on %s"
                                   % (tuple(p.shape), p.device))
            bufs.append(b.data_ptr())
            init.append(int(p in new_state))
        arr["exp_avg"], arr["buf_uninit"] = bufs, init
        arr["step_size"] = [float(g["lr"]) for g, _ in rows]
        arr["momentum"] = [float(g["momentum"]) for g, _ in rows]
        arr["weight_decay"] = [float(g["weight_decay"]) for g, _ in rows]
        return new_state

    def _commit(self, rows, new_state):
        for p, b in new_state.items():
            self.state[p]["momentum_buffer"] = b

    def _launch(self, lib):
        return lib.step_multi_tensor_sgd_f32


class LossScaler:
    """Dynamic loss scaling with torch.amp.GradScaler's policy and defaults: the scale halves after a step whose gradients
    overflowed (the optimizer skipped it) and doubles after `growth_interval` consecutive clean steps."""

    def __init__(self, init_scale=2.0 ** 16, growth_factor=2.0, backoff_factor=0.5, growth_interval=2000):
        self.scale = float(init_scale)
        self._growth_factor, self._backoff_factor = float(growth_factor), float(backoff_factor)
        self._growth_interval = int(growth_interval)
        self._clean = 0

    def update(self, found_inf):
        if found_inf:
            self.scale *= self._backoff_factor
            self._clean = 0
        else:
            self._clean += 1
            if self._clean == self._growth_interval:
                self.scale *= self._growth_factor
                self._clean = 0
