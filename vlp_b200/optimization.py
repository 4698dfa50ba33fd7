"""BertAdam on H100 — same constructor, param-group keys, state keys and schedule functions as the reference's
pytorch_pretrained_bert/optimization.py:32-182 (imported by vlp/run_img2txt_dist.py:25, built at :422-426), with `step()`
executed by two launches of libvlpk.so (`vlpk_bertadam_step`, csrc/optim.cu) over ALL parameters instead of the reference's
Python loop of ~400 tensors x (norm + host read-back + 6 elementwise kernels).

Differences a caller can observe, all deliberate:
  * bf16 parameters are supported: state['master'] holds an fp32 copy that carries the arithmetic (what the reference's --fp16
    branch delegates to apex FP16_Optimizer, run_img2txt_dist.py:403-420); moments are always fp32.  fp32 parameters are
    updated exactly like the reference (no master copy).
  * gradient clipping does not rescale p.grad in place (the clip factor is applied inside the update kernel).
  * CUDA only — there is no CPU path; a parameter that lives on the CPU raises.
"""
import ctypes as C
import math

import numpy as np
import torch
from torch.optim import Optimizer
from torch.optim.optimizer import required

from . import _lib as L
from . import ops


def warmup_cosine(x, warmup=0.002):
    if x < warmup:
        return x / warmup
    return 0.5 * (1.0 + math.cos(math.pi * x))


def warmup_constant(x, warmup=0.002):
    if x < warmup:
        return x / warmup
    return 1.0


def warmup_linear(x, warmup=0.002):
    if x < warmup:
        return x / warmup
    return max((x - 1.) / (warmup - 1.), 0)


SCHEDULES = {'warmup_cosine': warmup_cosine, 'warmup_constant': warmup_constant, 'warmup_linear': warmup_linear}

_TENSOR_DTYPE = np.dtype([("param", "<u8"), ("grad", "<u8"), ("master", "<u8"), ("m", "<u8"), ("v", "<u8"), ("n", "<i8"),
                          ("weight_decay", "<f4"), ("param_dtype", "<i4"), ("grad_dtype", "<i4"), ("reserved", "<i4")])
assert _TENSOR_DTYPE.itemsize == C.sizeof(L.VlpkAdamTensor) == 64
_DT = {torch.bfloat16: 0, torch.float32: 1}     # VLPK_BF16 / VLPK_F32


class BertAdam(Optimizer):
    """BERT version of Adam with decoupled weight decay, per-tensor gradient clipping and no bias correction.
    Params (optimization.py:58-71): lr; warmup: portion of t_total, -1 = none; t_total: total steps, -1 = constant lr;
    schedule; b1; b2; e; weight_decay; max_grad_norm (-1 = no clipping)."""

    def __init__(self, params, lr=required, warmup=-1, t_total=-1, schedule='warmup_linear', b1=0.9, b2=0.999, e=1e-6, weight_decay=0.01,
                 max_grad_norm=1.0):
        if lr is not required and lr < 0.0:
            raise ValueError("Invalid learning rate: {} - should be >= 0.0".format(lr))
        if schedule not in SCHEDULES:
            raise ValueError("Invalid schedule parameter: {}".format(schedule))
        if not 0.0 <= warmup < 1.0 and not warmup == -1:
            raise ValueError("Invalid warmup: {} - should be in [0.0, 1.0[ or -1".format(warmup))
        if not 0.0 <= b1 < 1.0:
            raise ValueError("Invalid b1 parameter: {} - should be in [0.0, 1.0[".format(b1))
        if not 0.0 <= b2 < 1.0:
            raise ValueError("Invalid b2 parameter: {} - should be in [0.0, 1.0[".format(b2))
        if not e >= 0.0:
            raise ValueError("Invalid epsilon value: {} - should be >= 0.0".format(e))
        defaults = dict(lr=lr, schedule=schedule, warmup=warmup, t_total=t_total, b1=b1, b2=b2, e=e, weight_decay=weight_decay,
                        max_grad_norm=max_grad_norm)
        super(BertAdam, self).__init__(params, defaults)
        self._keep = None     # device tables of the last step (kept alive until the next one)
        self._plan = None     # cached per-group descriptor tables (see step())
        self._plan_sig = None
        self._pinned = {}     # (device, n tensors) -> rotating pinned host tables

    @staticmethod
    def _scheduled_lr(group, step):
        if group['t_total'] != -1:
            return group['lr'] * SCHEDULES[group['schedule']](step / group['t_total'], group['warmup'])
        return group['lr']

    def get_lr(self):
        lr = []
        for group in self.param_groups:
            for p in group['params']:
                state = self.state[p]
                if len(state) == 0:
                    return [0]
                lr.append(self._scheduled_lr(group, state['step']))
        return lr

    def _init_state(self, p):
        state = self.state[p]
        if len(state) == 0:
            state['step'] = 0
            state['next_m'] = torch.zeros(p.shape, dtype=torch.float32, device=p.device)
            state['next_v'] = torch.zeros(p.shape, dtype=torch.float32, device=p.device)
        if p.dtype == torch.bfloat16 and 'master' not in state:
            state['master'] = p.detach().float().contiguous()
        return state

    _FP32_STATE = ('next_m', 'next_v', 'master')

    def load_state_dict(self, state_dict):
        """torch's Optimizer.load_state_dict casts every floating-point state tensor to the PARAMETER dtype: with bf16 parameters the
        moments and the fp32 master copy would come back as bf16 (half the bytes the update kernel addresses, and the master's extra
        precision lost).  The kernel's state is fp32 by contract, so the saved tensors are re-installed from the checkpoint itself
        — fp32, contiguous, on the parameter's device — after the base class has rebuilt the param <-> state mapping.  A reference
        checkpoint (fp32 moments, no master) loads the same way; its master copy is then created from the parameter on first use
        (run_img2txt_dist.py:430-434 loads optimizer state after the model weights)."""
        saved_groups = state_dict['param_groups']
        saved_state = state_dict['state']
        super(BertAdam, self).load_state_dict(state_dict)
        self._plan = None
        ids = [i for g in saved_groups for i in g['params']]
        params = [p for g in self.param_groups for p in g['params']]
        for i, p in zip(ids, params):
            src = saved_state.get(i)
            if src is None:
                continue
            st = self.state[p]
            for key in self._FP32_STATE:
                if key in src and torch.is_tensor(src[key]):
                    st[key] = src[key].detach().to(device=p.device, dtype=torch.float32).contiguous().clone()
            if 'step' in st and torch.is_tensor(st['step']):
                st['step'] = int(st['step'])
            if p.dtype != torch.bfloat16:
                st.pop('master', None)

    @torch.no_grad()
    def resync_master(self):
        """Re-derive the fp32 master copies from the current bf16 parameters.  Call after the parameters were changed behind the
        optimizer's back once training has started (model.load_state_dict of weights only, a parameter broadcast, manual
        re-initialisation): step() writes the parameters from the master copy, which would otherwise undo that change."""
        for group in self.param_groups:
            for p in group['params']:
                st = self.state.get(p)
                if st and 'master' in st:
                    st['master'].copy_(p.detach().float())

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        # Host side of a step = O(#tensors) pointer gathering only: everything that does not change between steps (parameter / state
        # pointers, sizes, weight decay, dtype tags, chunk prefix, validation) is cached in a plan, rebuilt when the set of parameters
        # that carry a gradient changes or state is (re)loaded.  One launch pair per distinct (device, scheduled lr, b1, b2, e,
        # max_grad_norm); in practice a single one: the two weight-decay groups of run_img2txt_dist.py:394-401 differ only in the
        # per-tensor weight_decay field.  The schedule is evaluated at each tensor's own state['step'] (optimization.py:164-172): a
        # tensor that had no gradient on some steps keeps a smaller count than its group and gets its own learning rate.
        sig = tuple((id(p), p.grad is None) for group in self.param_groups for p in group['params'])
        if self._plan is not None and self._plan_sig == sig:
            # state tensors replaced behind the plan's back (a hand-rolled state load, dtype casts): re-validate
            for _, _, states, tab in self._plan:
                if [st['next_m'].data_ptr() for st in states] != tab["m"].tolist() or [st['next_v'].data_ptr() for st in states] != tab["v"].tolist():
                    self._plan = None
                    break
        if self._plan is None or self._plan_sig != sig:
            self._build_plan()
            self._plan_sig = sig
        buckets = {}
        for group, ps, states, tab in self._plan:
            if not ps:
                continue
            grads = []
            for i, p in enumerate(ps):
                g = p.grad
                if g.dtype not in _DT or g.is_sparse:
                    raise RuntimeError(f"vlp_b200 BertAdam: gradients must be dense bf16 or fp32, got {g.dtype}")
                if not g.is_contiguous():
                    g = g.contiguous()
                grads.append(g)
            tab["grad"] = [g.data_ptr() for g in grads]
            tab["grad_dtype"] = [_DT[g.dtype] for g in grads]
            rest = (group['b1'], group['b2'], group['e'], group['max_grad_norm'])
            steps = [st['step'] for st in states]
            if steps.count(steps[0]) == len(steps):
                buckets.setdefault((ps[0].device, self._scheduled_lr(group, steps[0])) + rest, []).append((tab, grads, states))
            else:
                lrs = [self._scheduled_lr(group, s) for s in steps]
                for lr_s in dict.fromkeys(lrs):
                    idx = [i for i, l in enumerate(lrs) if l == lr_s]
                    buckets.setdefault((ps[0].device, lr_s) + rest, []).append((tab[idx], [grads[i] for i in idx], [states[i] for i in idx]))
        keep = []
        for (device, lr_s, b1, b2, e, max_norm), parts in buckets.items():
            tab = parts[0][0] if len(parts) == 1 else np.concatenate([t for t, _, _ in parts])
            keep.append(self._launch(device, tab, lr_s, b1, b2, e, max_norm) + ([g for _, gs, _ in parts for g in gs],))
            for _, _, states in parts:
                for state in states:
                    state['step'] += 1
        self._keep = keep
        return loss

    def _build_plan(self):
        plan = []
        for group in self.param_groups:
            ps, states = [], []
            for p in group['params']:
                if p.grad is None or p.numel() == 0:
                    continue
                if p.grad.is_sparse:
                    raise RuntimeError('Adam does not support sparse gradients, please consider SparseAdam instead')
                if p.dtype not in _DT or p.grad.dtype not in _DT:
                    raise RuntimeError(f"vlp_b200 BertAdam: parameters / gradients must be bf16 or fp32, got {p.dtype} / {p.grad.dtype}")
                ops._require_cuda(p, "BertAdam parameters")
                if not p.is_contiguous():
                    raise RuntimeError("vlp_b200 BertAdam: parameters must be contiguous")
                state = self._init_state(p)
                for key in ('next_m', 'next_v', 'master'):
                    t = state.get(key)
                    if t is not None and not (t.dtype == torch.float32 and t.is_contiguous() and t.numel() == p.numel() and t.device == p.device):
                        raise RuntimeError(f"vlp_b200 BertAdam: state['{key}'] must be a contiguous fp32 tensor of the parameter's size on its "
                                           f"device (got {t.dtype}, {tuple(t.shape)}, {t.device}); state loaded without BertAdam.load_state_dict?")
                ps.append(p)
                states.append(state)
            tab = np.zeros(len(ps), dtype=_TENSOR_DTYPE)
            wd = float(group['weight_decay'])
            for i, (p, state) in enumerate(zip(ps, states)):
                master = state.get('master')
                tab[i] = (p.data_ptr(), 0, 0 if master is None else master.data_ptr(), state['next_m'].data_ptr(), state['next_v'].data_ptr(),
                          p.numel(), wd, _DT[p.dtype], 0, 0)
            plan.append((group, ps, states, tab))
        self._plan = plan

    def _launch(self, device, tab, lr_s, b1, b2, e, max_norm):
        n = len(tab)
        chunk = L.lib().vlpk_bertadam_chunk()
        # The descriptor table travels through PINNED host memory: an asynchronous copy from pageable memory synchronises the host
        # with the stream, i.e. with the whole backward that is still in flight — a pipeline bubble every step.
        # Three rotating slots.  The host may run ahead of the device (a GPU-bound step, a graph replay followed by step()), so a slot
        # is only rewritten once the event recorded after its copies has completed: this waits only when the device is three
        # launches behind, and otherwise costs an event query.
        slot = self._pinned.setdefault((device, n), {"i": 0, "bufs": [None, None, None], "copied": [None, None, None]})
        k = slot["i"] = (slot["i"] + 1) % 3
        if slot["copied"][k] is not None:
            slot["copied"][k].synchronize()
        if slot["bufs"][k] is None:
            pin = (lambda t: t.pin_memory()) if torch.cuda.is_available() else (lambda t: t)     # (CPU dry-run tests marshal without a GPU)
            slot["bufs"][k] = (pin(torch.empty(n * _TENSOR_DTYPE.itemsize, dtype=torch.uint8)), pin(torch.empty(n + 1, dtype=torch.int32)))
        tab_pin, prefix_pin = slot["bufs"][k]
        tab_np = tab_pin.numpy().view(_TENSOR_DTYPE)
        tab_np[:] = tab
        prefix = prefix_pin.numpy()
        prefix[0] = 0
        np.cumsum((tab["n"] + chunk - 1) // chunk, out=prefix[1:])
        tab_dev = tab_pin.to(device, non_blocking=True)
        prefix_dev = prefix_pin.to(device, non_blocking=True)
        if device.type == "cuda":
            if slot["copied"][k] is None:
                slot["copied"][k] = torch.cuda.Event()
            slot["copied"][k].record()
        sqnorm = torch.empty(n, dtype=torch.float32, device=device)
        L.call("vlpk_bertadam_step", tab_np.ctypes.data, tab_dev.data_ptr(), prefix.ctypes.data, prefix_dev.data_ptr(), n, sqnorm.data_ptr(),
               float(lr_s), float(b1), float(b2), float(e), float(max_norm), L.stream())
        return tab_dev, prefix_dev, sqnorm
