"""Optimizer step of the training loop on the engine.

The reference's loop (tools/train.py:193-196) clamps every gradient (``utils.clip_gradient``, captioning/utils/misc.py:156-160) and
then calls ``torch.optim.Adam.step()`` (``build_optimizer``, misc.py:186-205).  On the stock path that is ~125 small launches and
about ten passes over the parameters.  ``FusedAdam`` is ``torch.optim.Adam`` with ``step()``
replaced by one launch of ``capb200_adam_step`` (csrc/optim.cu): same constructor, same ``state_dict`` layout (``step`` / ``exp_avg`` /
``exp_avg_sq`` per parameter, so checkpoints written by either load into the other -- tools/train.py:74-77 resumes ``optimizer.pth``),
same arithmetic term by term; ``clip_value`` folds ``clip_gradient`` into the same pass.

    optimizer = b200.optim.FusedAdam(model.parameters(), opt.learning_rate, (opt.optim_alpha, opt.optim_beta), opt.optim_epsilon,
                                     weight_decay=opt.weight_decay, clip_value=opt.grad_clip_value)     # replaces build_optimizer + clip_gradient

CUDA fp32 parameters only (the engine's parameters); anything else raises -- there is no CPU path.
"""
from __future__ import annotations

import torch

from . import _lib


class FusedAdam(torch.optim.Adam):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, clip_value=None, write_clamped_grad=True):
        super().__init__(params, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=False)
        self.clip_value = clip_value
        self.write_clamped_grad = write_clamped_grad
        self._tables = {}
        self.launches = 0

    def _table(self, gi, params, grads, ms, vs):
        key = (gi, tuple(t.data_ptr() for t in params), tuple(t.data_ptr() for t in grads), tuple(t.data_ptr() for t in ms))
        hit = self._tables.get(gi)
        if hit is not None and hit[0] == key:
            return hit[1]
        dev = params[0].device
        chunk = _lib.load().capb200_adam_chunk_elems()
        rows, numel, chunks = [], [], []
        for i, (p, g, m, v) in enumerate(zip(params, grads, ms, vs)):
            rows.append([p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr()])
            numel.append(p.numel())
            chunks.extend([i, c] for c in range((p.numel() + chunk - 1) // chunk))
        # pointers are < 2^63, so int64 storage round-trips them
        tab = (torch.tensor(rows, dtype=torch.int64).to(dev), torch.tensor(numel, dtype=torch.int64).to(dev),
               torch.tensor(chunks, dtype=torch.int32).to(dev), len(chunks))
        self._tables[gi] = (key, tab)
        return tab

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        lib = _lib.load()
        for gi, group in enumerate(self.param_groups):
            if group.get('amsgrad') or group.get('maximize'):
                raise NotImplementedError('capb200 FusedAdam: amsgrad / maximize are not implemented')
            by_dev = {}
            for p in group['params']:
                if p.grad is None:
                    continue
                if not (p.is_cuda and p.dtype == torch.float32 and p.is_contiguous() and p.grad.is_contiguous() and p.grad.dtype == torch.float32
                        and not p.grad.is_sparse):
                    raise RuntimeError('capb200 FusedAdam: parameters and gradients must be contiguous fp32 CUDA tensors (no CPU path)')
                st = self.state[p]
                if len(st) == 0:
                    st['step'] = torch.tensor(0.0, dtype=torch.float32)         # torch.optim.Adam's default (host scalar tensor)
                    st['exp_avg'] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    st['exp_avg_sq'] = torch.zeros_like(p, memory_format=torch.preserve_format)
                by_dev.setdefault((p.device, float(st['step'])), []).append(p)
            beta1, beta2 = group['betas']
            for (dev, step0), ps in by_dev.items():
                step = int(step0) + 1
                torch._foreach_add_([self.state[p]['step'] for p in ps], 1)
                grads = [p.grad for p in ps]
                ms = [self.state[p]['exp_avg'] for p in ps]
                vs = [self.state[p]['exp_avg_sq'] for p in ps]
                table, numel, chunks, n_chunks = self._table((gi, str(dev), len(by_dev) > 1 and step), ps, grads, ms, vs)
                with torch.cuda.device(dev):
                    _lib.check(lib.capb200_adam_step(_lib.ptr(table), _lib.ptr(numel), _lib.ptr(chunks), n_chunks, float(group['lr']), float(beta1),
                                                     float(beta2), float(group['eps']), float(group['weight_decay']), step,
                                                     float(self.clip_value) if self.clip_value else 0.0, 1 if self.write_clamped_grad else 0,
                                                     _lib.current_stream()), 'adam_step')
                self.launches += 1
                # the kernel writes the parameters through raw pointers: bump their version counters as an in-place torch op would, so the
                # engines see new weights and re-bind their derived copies (fp16 planes, bias sums) before the next call
                for p in ps:
                    torch.autograd.graph.increment_version(p)
        return loss
