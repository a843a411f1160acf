"""Fused Adam step of the hash table (libsdb200: sdb_adam_step) and its zero-edit hook.

The reference trains `hash_encoder.embeddings` ([8388608, 8] fp32, 268 MB) with torch.optim.Adam
(imaginaire/utils/trainer.py:297-323; configs/scenedreamer_train.yaml:36-61: lr 1e-4, eps 1e-7, betas (0, 0.999)): about ten
element-wise passes over four 268 MB arrays per step although a view touches a few per cent of the rows.  `adam_step_`
does the same arithmetic in one kernel and one pass and leaves exactly torch's optimizer state behind
(`step`, `exp_avg`, `exp_avg_sq`), so checkpoints stay interchangeable with the reference.

Zero-edit route: `install_step_hook()` registers a global optimizer-step pre-hook (torch.optim.optimizer.
register_optimizer_step_pre_hook).  When a torch.optim.Adam is about to step, parameters tagged by the integration layer
(`param._sdb200_table`, set on the generator's `hash_encoder.embeddings`) are stepped by the fused kernel with that
optimizer's own hyper-parameters and state, and their `.grad` is cleared so that the optimizer skips them.  The hook runs
at `optimizer.step()` time, i.e. after DDP has all-reduced the dense gradient.
"""
import ctypes

import torch

from . import _lib

_hook_handle = None
stats = {'fused_steps': 0}


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr())


def adam_step_(param, grad, exp_avg, exp_avg_sq, step, lr, beta1, beta2, eps):
    """In place, on param's device; `step` = step count AFTER the increment (torch's state['step'])."""
    for t in (param, grad, exp_avg, exp_avg_sq):
        if not t.is_cuda or t.dtype != torch.float32 or not t.is_contiguous():
            raise RuntimeError('adam_step_: contiguous float32 CUDA tensors expected')
    if not (param.numel() == grad.numel() == exp_avg.numel() == exp_avg_sq.numel()) or param.numel() % 4:
        raise RuntimeError('adam_step_: sizes must match and be a multiple of 4')
    with torch.cuda.device(param.device):
        code = _lib.lib().sdb_adam_step(_ptr(param), _ptr(grad), _ptr(exp_avg), _ptr(exp_avg_sq), int(param.numel()), float(lr),
                                        float(beta1), float(beta2), float(eps), int(step),
                                        ctypes.c_void_p(torch.cuda.current_stream(param.device).cuda_stream))
    _lib.check(code, 'sdb_adam_step')


def _eligible(opt, group, p):
    return (getattr(p, '_sdb200_table', False) and p.grad is not None and p.is_cuda and p.dtype == torch.float32 and
            p.is_contiguous() and p.grad.is_contiguous() and not p.grad.is_sparse and p.numel() % 4 == 0 and
            not group.get('amsgrad', False) and group.get('weight_decay', 0) == 0 and not group.get('maximize', False) and
            not group.get('capturable', False) and not torch.is_tensor(group['lr']))


def _step_pre_hook(opt, args, kwargs):
    if type(opt) is not torch.optim.Adam:
        return None
    # Under torch.amp.GradScaler a plain Adam is stepped only when every gradient is finite, and after unscale_: the hook then
    # sees the true gradients and is not called on a skipped step.  A fused Adam (`_step_supports_amp_scaling`) is stepped
    # with its gradients still scaled, also on a step to be skipped: GradScaler hands it the scale and the inf flag as the
    # optimizer attributes `grad_scale` / `found_inf` for the length of the call, and the fused kernel unscales and skips by
    # itself.  Leave the table to it then.
    if getattr(opt, 'grad_scale', None) is not None or getattr(opt, 'found_inf', None) is not None:
        return None
    for group in opt.param_groups:
        for p in group['params']:
            if not _eligible(opt, group, p):
                continue
            st = opt.state[p]
            if len(st) == 0:                                    # what Adam._init_group creates
                st['step'] = torch.zeros((), dtype=torch.float32, device=p.device) if group.get('fused') else torch.tensor(0.0)
                st['exp_avg'] = torch.zeros_like(p, memory_format=torch.preserve_format)
                st['exp_avg_sq'] = torch.zeros_like(p, memory_format=torch.preserve_format)
            st['step'] += 1
            b1, b2 = group['betas']
            with torch.no_grad():
                adam_step_(p.data, p.grad.data, st['exp_avg'], st['exp_avg_sq'], int(st['step'].item()), group['lr'], b1, b2, group['eps'])
            p.grad = None                                       # torch's Adam now skips this parameter
            stats['fused_steps'] += 1
    return None


def install_step_hook():
    global _hook_handle
    if _hook_handle is None:
        from torch.optim.optimizer import register_optimizer_step_pre_hook
        _hook_handle = register_optimizer_step_pre_hook(_step_pre_hook)
    return _hook_handle


def remove_step_hook():
    global _hook_handle
    if _hook_handle is not None:
        _hook_handle.remove()
        _hook_handle = None


def tag_table(param):
    """Mark a Parameter as 'the hash table': the step hook takes over its Adam step."""
    param._sdb200_table = True
    return param
