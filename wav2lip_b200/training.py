"""Host side of the training step (scope row f1) above the C-ABI of include/w2l.h (w2l_train_*):

* the autograd bridge that lets the reference's training scripts run unchanged — `model.train(); g = model(indiv_mels, x);
  loss = ...; loss.backward(); optimizer.step()` (wav2lip_train.py:210-231, color_syncnet_train.py:146-163,
  hq_wav2lip_train.py:213-255): in train mode the mirrors' forward goes through `w2l_train_forward` (BatchNorm on batch
  statistics, running averages updated in place) and registers one autograd node whose backward is `w2l_train_backward`
  (dgrad / wgrad / BatchNorm-ReLU-residual kernels); torch only sees the loss arithmetic and the optimizer;
* `Wav2LipTrainStep`: the same iteration as ONE native call (`w2l_wav2lip_train_step`: generator forward, the frozen
  expert in train mode as the scripts leave it, both losses and their gradients, backward, bucketed gradient all-reduce
  over NCCL overlapped with the backward, multi-tensor Adam) — what bench.py --workload train times;
* `HQWav2LipTrainStep` (`w2l_hq_wav2lip_train_step`, hq_wav2lip_train.py:212-256, with the quality discriminator and its
  own step) and `SyncNetTrainStep` (`w2l_syncnet_train_step`, color_syncnet_train.py:149-163): the other two scripts'
  iterations as one native call each;
* the fused steps' Adam state as `torch.optim.Adam(...).state_dict()` gives it (`optimizer_state_dict()` /
  `load_optimizer_state_dict()`), so checkpoints move between the reference's scripts and the fused steps;
* `init_data_parallel`: hands every rank's context the NCCL communicator (unique id from rank 0, broadcast with
  torch.distributed).

Training runs with bf16 operands and fp32 master weights / gradients / statistics on its own bf16 context per module;
there is no CPU path."""
import ctypes as C

import torch

from . import _lib

_P = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None   # noqa: E731


class _Binding:
    """One module's tensors bound to a training context: fp32 master parameters and BatchNorm buffers by reference,
    gradients in ONE contiguous fp32 arena in state_dict order (so the all-reduce runs over three large buckets)."""

    def __init__(self, module, device_index: int, ctx=None):
        # (ctx: bind into another module's context — the expert and the discriminator inside a generator step)
        self.ctx = ctx if ctx is not None else _lib.Context(device_index, _lib.PREC_BF16)
        self.device = torch.device("cuda", device_index)
        self.module = module
        self.key = None
        self.arena = None
        self.grads = {}
        self.nbt = []

    def _tensors(self):
        return [(n, t) for n, t in self.module.state_dict(keep_vars=True).items()]

    def ensure(self):
        ts = self._tensors()
        key = tuple((n, t.data_ptr(), bool(getattr(t, "requires_grad", False))) for n, t in ts)
        if key == self.key:
            return self
        names, values, grads, numels = [], [], [], []
        total = sum(t.numel() for _, t in ts if t.dtype.is_floating_point and getattr(t, "requires_grad", False))
        self.arena = torch.zeros(max(total, 1), device=self.device, dtype=torch.float32)
        self.grads, self.nbt, off = {}, [], 0
        for n, t in ts:
            if not t.dtype.is_floating_point:
                if n.endswith("num_batches_tracked"):
                    self.nbt.append(t)
                continue
            if not t.is_cuda or t.device != self.device:
                raise _lib.W2LError(f"{n} is on {t.device}, expected {self.device}: move the module with .to('cuda') first")
            if t.dtype != torch.float32 or not t.is_contiguous():
                raise _lib.W2LError(f"{n}: training binds fp32 contiguous master tensors, got {t.dtype}")
            names.append(n.encode())
            values.append(t.data_ptr())
            numels.append(t.numel())
            if getattr(t, "requires_grad", False):
                g = self.arena[off:off + t.numel()].view(t.shape)
                off += t.numel()
                self.grads[n] = g
                grads.append(g.data_ptr())
            else:
                grads.append(None)
        k = len(names)
        _lib.check(self.ctx.lib.w2l_train_bind(self.ctx.h, self.module.NET, k, (C.c_char_p * k)(*names),
                                               (C.c_void_p * k)(*values), (C.c_void_p * k)(*grads), (C.c_int64 * k)(*numels)))
        self.key = key
        return self

    def bump_batches_tracked(self):
        if self.nbt:
            torch._foreach_add_(self.nbt, 1)


def binding_of(module, ref: torch.Tensor) -> _Binding:
    if not ref.is_cuda:
        raise _lib.W2LError(f"{type(module).__name__} trains on a CUDA (sm_90) device only; got a {ref.device} tensor")
    idx = ref.device.index if ref.device.index is not None else torch.cuda.current_device()
    b = module.__dict__.get("_w2l_binding")
    if b is None or b.device.index != idx:
        b = _Binding(module, idx)
        module.__dict__["_w2l_binding"] = b
    return b.ensure()


def _check(b: _Binding, *tensors):
    for t in tensors:
        if t is not None and (not t.is_cuda or t.device != b.device):
            raise _lib.W2LError(f"expected every input on {b.device}, got a tensor on {t.device}")


def _f32(t):
    return t.detach().contiguous().float()


def _stream(b: _Binding):
    return C.c_void_p(torch.cuda.current_stream(b.device).cuda_stream)


def _param_list(module):
    return [p for p in module.parameters()]


class _TrainFn(torch.autograd.Function):
    """One network's train-mode forward as a single autograd node.  Inputs after the fixed arguments are the module's
    parameters (so that autograd routes gradients to them); the C side writes parameter gradients into the binding's
    arena, of which fresh copies are returned (autograd then accumulates into .grad as for any other op)."""

    @staticmethod
    def forward(ctx, module, b, kind, in0, in1, *params):
        lib, h, net = b.ctx.lib, b.ctx.h, module.NET
        want_param_grads = any(p.requires_grad for p in params)
        if net == _lib.NET_GENERATOR:
            want_input_grad = False      # mel and face windows are data (wav2lip_train.py:214-217)
        elif net == _lib.NET_SYNCNET:
            want_input_grad = bool(in1.requires_grad)
        else:
            want_input_grad = bool(in0.requires_grad)
        flags = (_lib.TRAIN_WGRAD if want_param_grads else 0) | (_lib.TRAIN_INPUT_GRAD if want_input_grad else 0)
        a0 = _f32(in0)
        a1 = _f32(in1) if in1 is not None else None
        if net == _lib.NET_GENERATOR:
            if a1.dim() > 4:
                B, T = a1.shape[0], a1.shape[2]
                out = torch.empty((B, 3, T, 96, 96), device=b.device, dtype=torch.float32)
            else:
                B, T = a1.shape[0], 0
                out = torch.empty((B, 3, 96, 96), device=b.device, dtype=torch.float32)
            outs = (out,)
            _lib.check(lib.w2l_train_forward(h, net, _P(a0), _P(a1), _P(out), None, B, T, flags, _stream(b)))
        elif net == _lib.NET_SYNCNET:
            B = a1.shape[0]
            T = 5 if kind == "frames" else 0
            a = torch.empty((B, 512), device=b.device, dtype=torch.float32)
            v = torch.empty((B, 512), device=b.device, dtype=torch.float32)
            outs = (a, v)
            _lib.check(lib.w2l_train_forward(h, net, _P(a0), _P(a1), _P(a), _P(v), B, T, flags, _stream(b)))
        else:
            B, T = a0.shape[0], a0.shape[2]
            out = torch.empty((B * T, 1), device=b.device, dtype=torch.float32)
            outs = (out,)
            _lib.check(lib.w2l_train_forward(h, net, _P(a0), None, _P(out), None, B, T, flags, _stream(b)))
        b.bump_batches_tracked()
        ctx.module, ctx.b, ctx.flags, ctx.net = module, b, flags, net
        ctx.in_shape = tuple((in1 if net != _lib.NET_DISC else in0).shape)
        ctx.n_params = len(params)
        ctx.save_for_backward(*outs)     # the generator's head backward re-reads its output: keep it alive
        return outs if len(outs) > 1 else outs[0]

    @staticmethod
    def backward(ctx, *douts):
        b, net, module = ctx.b, ctx.net, ctx.module
        lib, h = b.ctx.lib, b.ctx.h
        d = [_f32(x) if x is not None else None for x in douts]
        if net == _lib.NET_SYNCNET:
            zeros = None
            for i in range(2):
                if d[i] is None:
                    zeros = zeros if zeros is not None else torch.zeros((ctx.in_shape[0], 512), device=b.device)
                    d[i] = zeros
        dinput = None
        if ctx.flags & _lib.TRAIN_INPUT_GRAD:
            dinput = torch.empty(ctx.in_shape, device=b.device, dtype=torch.float32)
        _lib.check(lib.w2l_train_backward(h, net, _P(d[0]), _P(d[1]) if len(d) > 1 else None, _P(dinput), ctx.flags, _stream(b)))
        pgrads = []
        names = [n for n, _ in module.named_parameters()]
        for n, p in zip(names, module.parameters()):
            g = b.grads.get(n) if (p.requires_grad and (ctx.flags & _lib.TRAIN_WGRAD)) else None
            pgrads.append(g.clone() if g is not None else None)
        if net == _lib.NET_DISC:
            return (None, None, None, dinput, None, *pgrads)
        return (None, None, None, None, dinput, *pgrads)


def train_forward(module, kind, in0, in1):
    """Entry used by the mirrors' forward() in train mode."""
    ref = in1 if in1 is not None else in0
    b = binding_of(module, ref)
    _check(b, in0, in1)
    module.mark_weights_dirty()          # the inference plan's packed weights are stale once training touches the module
    return _TrainFn.apply(module, b, kind, in0, in1, *_param_list(module))


# ----------------------------------------------------------------------------------------------------------------------
# the fused native steps
# ----------------------------------------------------------------------------------------------------------------------
ADAM_BETAS = (0.9, 0.999)          # wav2lip_train.py:357-360, color_syncnet_train.py:270-271 (torch's default)
HQ_ADAM_BETAS = (0.5, 0.999)       # hq_wav2lip_train.py:421-424


def _bind_expert(b: _Binding, syncnet):
    """The frozen expert (wav2lip_train.py:188-189) bound into the generator's context: its input gradient feeds the
    generator's backward on the device."""
    if syncnet is None:
        return None
    for q in syncnet.parameters():
        q.requires_grad_(False)
    return _Binding(syncnet, b.device.index, ctx=b.ctx).ensure()


def _generator_batch(b: _Binding, x, indiv_mels, mel, gt, want_mel: bool):
    """The generator steps' inputs, checked and made fp32 contiguous: (x, indiv_mels, mel or None, gt, B, T)."""
    _check(b, x, indiv_mels, mel, gt)
    x, indiv_mels, gt = _f32(x), _f32(indiv_mels), _f32(gt)
    B, T = x.shape[0], x.shape[2] if x.dim() == 5 else 0
    if tuple(x.shape) != (B, 6, T, 96, 96) or tuple(indiv_mels.shape) != (B, T, 1, 80, 16) or tuple(gt.shape) != (B, 3, T, 96, 96):
        raise ValueError(f"expected x (B,6,T,96,96), indiv_mels (B,T,1,80,16), gt (B,3,T,96,96); got {tuple(x.shape)}, "
                         f"{tuple(indiv_mels.shape)}, {tuple(gt.shape)}")
    mel = _f32(mel) if want_mel and mel is not None else None
    if mel is not None:
        if tuple(mel.shape) != (B, 1, 80, 16):
            raise ValueError(f"expected mel (B,1,80,16), got {tuple(mel.shape)}")
    return x, indiv_mels, mel, gt, B, T


# ---- optimizer state: torch.optim.Adam's state_dict() <-> the moments of the fused steps, mapped by parameter name ----
def adam_param_names(module) -> list:
    """Names of `[p for p in module.parameters() if p.requires_grad]`, the list the reference scripts hand to
    torch.optim.Adam: entry i of its state_dict()['state'] belongs to names[i]."""
    return [n for n, p in module.named_parameters() if p.requires_grad]


def adam_state_to_named(sd: dict, names: list) -> dict:
    """torch.optim.Adam(params).state_dict() (one param group over `names`) -> {'step': int, 'exp_avg': {name: t},
    'exp_avg_sq': {name: t}, 'param_groups': [...]}.  Every state entry shares one step count (one optimizer, one
    iteration counter); a state without entries (no step taken) has step 0."""
    groups = sd["param_groups"]
    if len(groups) != 1 or list(groups[0]["params"]) != list(range(len(names))):
        raise ValueError(f"expected one Adam param group over {len(names)} parameters, got "
                         f"{[len(g['params']) for g in groups]}")
    steps = {float(st["step"]) for st in sd["state"].values()}
    if len(steps) > 1:
        raise ValueError(f"Adam state entries with different step counts {sorted(steps)}")
    for i in sd["state"]:
        if not 0 <= int(i) < len(names):
            raise ValueError(f"Adam state entry {i} is outside the {len(names)} parameters")
    step = int(steps.pop()) if steps else 0
    return {"step": step,
            "exp_avg": {names[int(i)]: st["exp_avg"] for i, st in sd["state"].items()},
            "exp_avg_sq": {names[int(i)]: st["exp_avg_sq"] for i, st in sd["state"].items()},
            "param_groups": groups}


def adam_state_from_named(named: dict, names: list) -> dict:
    """The inverse of adam_state_to_named: the state_dict() torch.optim.Adam would give."""
    index = {n: i for i, n in enumerate(names)}
    unknown = set(named["exp_avg"]) - set(index)
    if unknown:
        raise ValueError(f"moments of unknown parameters: {sorted(unknown)[:4]}")
    state = {}
    for n in sorted(named["exp_avg"], key=index.get):
        state[index[n]] = {"step": torch.tensor(float(named["step"]), dtype=torch.float32),
                           "exp_avg": named["exp_avg"][n], "exp_avg_sq": named["exp_avg_sq"][n]}
    return {"state": state, "param_groups": named["param_groups"]}


def _adam_call(b: _Binding, net: int, direction: int, names: list, m: list, v: list, step: int) -> int:
    k = len(names)
    s = C.c_int64(step)
    _lib.check(b.ctx.lib.w2l_adam_state(b.ctx.h, net, direction, k, (C.c_char_p * k)(*[n.encode() for n in names]),
                                        (C.c_void_p * k)(*[t.data_ptr() for t in m]), (C.c_void_p * k)(*[t.data_ptr() for t in v]),
                                        C.byref(s), _stream(b)))
    return int(s.value)


def _export_adam(b: _Binding, module, lr: float, betas) -> dict:
    b.ensure()
    names = adam_param_names(module)
    params = dict(module.named_parameters())
    m = [torch.empty_like(params[n]) for n in names]
    v = [torch.empty_like(params[n]) for n in names]
    step = _adam_call(b, module.NET, 0, names, m, v, 0)
    groups = torch.optim.Adam([params[n] for n in names], lr=lr, betas=betas).state_dict()["param_groups"]
    named = {"step": step, "exp_avg": dict(zip(names, m)) if step else {}, "exp_avg_sq": dict(zip(names, v)) if step else {},
             "param_groups": groups}
    return adam_state_from_named(named, names)


def _import_adam(b: _Binding, module, sd: dict, betas) -> float:
    """Loads sd into the context's Adam of `module`; returns the saved learning rate."""
    b.ensure()
    names = adam_param_names(module)
    named = adam_state_to_named(sd, names)
    group = named["param_groups"][0]
    if tuple(group["betas"]) != tuple(betas):
        raise ValueError(f"optimizer state with betas {tuple(group['betas'])}, this step runs Adam with {tuple(betas)}")
    params = dict(module.named_parameters())
    if named["step"] and set(named["exp_avg"]) != set(names):
        raise ValueError(f"optimizer state has moments for {len(named['exp_avg'])} of {len(names)} parameters")

    def moment(which, n):
        t = named[which].get(n)
        if t is None:
            return torch.zeros_like(params[n])
        if t.numel() != params[n].numel():
            raise ValueError(f"{which} of {n}: {tuple(t.shape)}, parameter {tuple(params[n].shape)}")
        return t.detach().to(device=b.device, dtype=torch.float32).reshape(params[n].shape).contiguous()
    m = [moment("exp_avg", n) for n in names]
    v = [moment("exp_avg_sq", n) for n in names]
    _adam_call(b, module.NET, 1, names, m, v, named["step"])
    return float(group["lr"])


class Wav2LipTrainStep:
    """wav2lip_train.py:210-231 as one native call per iteration.

        step = Wav2LipTrainStep(model, syncnet, lr=1e-4, syncnet_wt=0.03)
        losses = step(x, indiv_mels, mel, gt)      # device tensor [sync_loss, l1, 0, loss]

    `model` (wav2lip_b200.models.Wav2Lip) holds the fp32 master parameters, updated in place by the fused Adam; its
    BatchNorm running averages (and the frozen expert's: the scripts leave it in train mode, :187-189) move as in the
    reference.  With torch.distributed initialised (backend nccl) and `init_data_parallel(step)` called, gradients are
    averaged over the ranks inside the step."""

    def __init__(self, model, syncnet=None, lr: float = 1e-4, syncnet_wt: float = 0.0):
        self.model, self.syncnet, self.lr, self.syncnet_wt = model, syncnet, float(lr), float(syncnet_wt)
        p = next(model.parameters())
        if not p.is_cuda:
            raise _lib.W2LError("move the model to a CUDA device first: wav2lip_b200 has no CPU path")
        self.b = binding_of(model, p)
        self.losses = torch.zeros(4, device=p.device, dtype=torch.float32)
        self.eb = _bind_expert(self.b, syncnet)

    def __call__(self, x, indiv_mels, mel, gt):
        b = self.b.ensure()
        wt = self.syncnet_wt if self.syncnet is not None else 0.0
        x, indiv_mels, m, gt, B, T = _generator_batch(b, x, indiv_mels, mel, gt, wt > 0)
        if self.eb is not None:
            self.eb.ensure()
        _lib.check(b.ctx.lib.w2l_wav2lip_train_step(b.ctx.h, _P(indiv_mels), _P(x), _P(m), _P(gt), B, T, wt, self.lr,
                                                    _P(self.losses), _stream(b)))
        b.bump_batches_tracked()
        if wt > 0:
            self.eb.bump_batches_tracked()
        self.model.mark_weights_dirty()
        return self.losses

    def optimizer_state_dict(self) -> dict:
        """`optimizer.state_dict()` of wav2lip_train.py's `optim.Adam([p for p in model.parameters() if p.requires_grad],
        lr)` after the steps run so far."""
        return _export_adam(self.b, self.model, self.lr, ADAM_BETAS)

    def load_optimizer_state_dict(self, sd: dict) -> None:
        """`optimizer.load_state_dict(sd)` (load_checkpoint(..., reset_optimizer=False)); takes the saved lr, as torch does."""
        self.lr = _import_adam(self.b, self.model, sd, ADAM_BETAS)

    def last_output(self, B: int, T: int) -> torch.Tensor:
        """g of the last step, (B,3,T,96,96) fp32 (a copy)."""
        out = torch.empty((B, 3, T, 96, 96), device=self.b.device, dtype=torch.float32)
        _lib.check(self.b.ctx.lib.w2l_train_last_output(self.b.ctx.h, _P(out), out.numel(), _stream(self.b)))
        return out


class HQWav2LipTrainStep:
    """hq_wav2lip_train.py:212-256 as one native call per iteration.

        step = HQWav2LipTrainStep(model, disc, syncnet, lr=1e-4, disc_lr=1e-4, syncnet_wt=0.0, disc_wt=0.07)
        losses = step(x, indiv_mels, mel, gt)   # device tensor [sync, l1, perceptual, loss, disc_real, disc_fake]

    The generator, the frozen expert and the discriminator share one training context; both networks' parameters are
    updated in place by their Adam (betas 0.5, 0.999).  `syncnet_wt` / `disc_wt` may be changed between calls (the script
    switches the sync loss on with hparams.set_hparam('syncnet_wt', ...)).  With `init_data_parallel(step)` both networks'
    gradients are averaged over the ranks inside the step."""

    def __init__(self, model, disc, syncnet=None, lr: float = 1e-4, disc_lr: float = 1e-4, syncnet_wt: float = 0.0,
                 disc_wt: float = 0.07):
        self.model, self.disc, self.syncnet = model, disc, syncnet
        self.lr, self.disc_lr, self.syncnet_wt, self.disc_wt = float(lr), float(disc_lr), float(syncnet_wt), float(disc_wt)
        p = next(model.parameters())
        if not p.is_cuda:
            raise _lib.W2LError("move the model to a CUDA device first: wav2lip_b200 has no CPU path")
        self.b = binding_of(model, p)
        self.db = _Binding(disc, self.b.device.index, ctx=self.b.ctx).ensure()
        self.eb = _bind_expert(self.b, syncnet)
        self.losses = torch.zeros(6, device=p.device, dtype=torch.float32)
        self._shape = None

    def __call__(self, x, indiv_mels, mel, gt):
        b = self.b.ensure()
        self.db.ensure()
        wt = self.syncnet_wt if self.syncnet is not None else 0.0
        x, indiv_mels, mel, gt, B, T = _generator_batch(b, x, indiv_mels, mel, gt, wt > 0)
        if self.eb is not None:
            self.eb.ensure()
        _lib.check(b.ctx.lib.w2l_hq_wav2lip_train_step(b.ctx.h, _P(indiv_mels), _P(x), _P(mel), _P(gt), B, T,
                                                       wt, self.disc_wt, self.lr, self.disc_lr, _P(self.losses), _stream(b)))
        b.bump_batches_tracked()
        if wt > 0:
            self.eb.bump_batches_tracked()
        self.model.mark_weights_dirty()
        self.disc.mark_weights_dirty()
        self._shape = (B, T)
        return self.losses

    def last_output(self, B: int = None, T: int = None) -> torch.Tensor:
        """g of the last step, (B,3,T,96,96) fp32 (a copy)."""
        B, T = (B, T) if B is not None else self._shape
        out = torch.empty((B, 3, T, 96, 96), device=self.b.device, dtype=torch.float32)
        _lib.check(self.b.ctx.lib.w2l_train_last_output(self.b.ctx.h, _P(out), out.numel(), _stream(self.b)))
        return out

    def optimizer_state_dict(self) -> dict:
        """`optimizer.state_dict()` of the generator's Adam (hq_wav2lip_train.py:421-422)."""
        return _export_adam(self.b, self.model, self.lr, HQ_ADAM_BETAS)

    def load_optimizer_state_dict(self, sd: dict) -> None:
        self.lr = _import_adam(self.b, self.model, sd, HQ_ADAM_BETAS)

    def disc_optimizer_state_dict(self) -> dict:
        """`disc_optimizer.state_dict()` (hq_wav2lip_train.py:423-424), saved in its own checkpoint file (:280-282)."""
        return _export_adam(self.db, self.disc, self.disc_lr, HQ_ADAM_BETAS)

    def load_disc_optimizer_state_dict(self, sd: dict) -> None:
        self.disc_lr = _import_adam(self.db, self.disc, sd, HQ_ADAM_BETAS)


class SyncNetTrainStep:
    """color_syncnet_train.py:149-163 as one native call per iteration.

        step = SyncNetTrainStep(model, lr=1e-4)
        loss = step(x, mel, y)      # x (B,15,48,96), mel (B,1,80,16), y (B,1) in {0,1} (SyncNetBatches); device tensor [loss]

    Adam with torch's default betas (:270-271) updates the parameters in place; with `init_data_parallel(step)` the
    gradients are averaged over the ranks inside the step."""

    def __init__(self, model, lr: float = 1e-4):
        self.model, self.lr = model, float(lr)
        p = next(model.parameters())
        if not p.is_cuda:
            raise _lib.W2LError("move the model to a CUDA device first: wav2lip_b200 has no CPU path")
        self.b = binding_of(model, p)
        self.loss = torch.zeros(1, device=p.device, dtype=torch.float32)

    def __call__(self, x, mel, y):
        b = self.b.ensure()
        _check(b, x, mel, y)
        x, mel, y = _f32(x), _f32(mel), _f32(y)
        B = x.shape[0]
        if tuple(x.shape) != (B, 15, 48, 96) or tuple(mel.shape) != (B, 1, 80, 16) or tuple(y.shape) != (B, 1):
            raise ValueError(f"expected x (B,15,48,96), mel (B,1,80,16), y (B,1); got {tuple(x.shape)}, {tuple(mel.shape)}, "
                             f"{tuple(y.shape)}")
        _lib.check(b.ctx.lib.w2l_syncnet_train_step(b.ctx.h, _P(mel), _P(x), _P(y), B, self.lr, _P(self.loss), _stream(b)))
        b.bump_batches_tracked()
        self.model.mark_weights_dirty()
        return self.loss

    def optimizer_state_dict(self) -> dict:
        """`optimizer.state_dict()` of color_syncnet_train.py's Adam."""
        return _export_adam(self.b, self.model, self.lr, ADAM_BETAS)

    def load_optimizer_state_dict(self, sd: dict) -> None:
        self.lr = _import_adam(self.b, self.model, sd, ADAM_BETAS)


def init_data_parallel(step_or_binding) -> int:
    """Create the NCCL communicator of a data-parallel run on this rank's context: rank 0 makes the unique id, it is
    broadcast through torch.distributed (must be initialised), every rank joins.  Returns the world size."""
    import torch.distributed as dist
    b = step_or_binding.b if hasattr(step_or_binding, "b") else step_or_binding
    if not dist.is_initialized():
        _lib.check(b.ctx.lib.w2l_comm_init(b.ctx.h, b"\0" * 128, 0, 1))
        return 1
    rank, world = dist.get_rank(), dist.get_world_size()
    buf = C.create_string_buffer(128)
    if rank == 0:
        _lib.check(b.ctx.lib.w2l_comm_unique_id(b.ctx.h, buf))
    box = [bytes(buf.raw)]
    dist.broadcast_object_list(box, src=0)
    _lib.check(b.ctx.lib.w2l_comm_init(b.ctx.h, box[0], rank, world))
    return world
