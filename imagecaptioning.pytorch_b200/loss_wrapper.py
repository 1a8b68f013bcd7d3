"""Mirror of captioning/modules/loss_wrapper.py (LossWrapper) and losses.RewardCriterion for the SCST branch.

    B200LossWrapper(model, opt).forward(fc_feats, att_feats, labels, masks, att_masks, gts, gt_indices,
                                        sc_flag, struc_flag, drop_worst_flag) -> {'loss', 'reward'}

sc_flag=True follows loss_wrapper.py:56-73 exactly: the eval-mode baseline (opt.sc_sample_method), the train-mode samples
(opt.train_sample_method: 'sample', 'greedy', 'gumbel', 'top<k>' or 'top<p>'), the self-critical
reward (``cider_reward_weight * CIDEr-D + bleu_reward_weight * BLEU-4``) and RewardCriterion -- every stage on the device through the C ABI.  sc_flag=False is the XE stage
(loss_wrapper.py:54-55: teacher-forced forward + LanguageModelCriterion / LabelSmoothing) and struc_flag=True the structure-loss
branch (loss_wrapper.py:25-53) with ``structure_loss_type='new_self_critical'`` (losses.py:168-187), the recipe of the reference's
best models; both run as one fused device step incl. the backward pass (UpDown, Att2in2, NewFC, AoANet, Transformer).
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import _lib
from .rewards import cider_scores, get_scores, get_self_critical_reward, reward_weights, weighted_scores


class RewardCriterion(nn.Module):
    """losses.py:18-37 on the device: -logp[seq] * reward * mask, mask = tokens up to and including the first EOS."""

    def forward(self, input, seq, reward, reduction='mean'):
        N, L = seq.shape
        V1 = input.shape[2]
        lp = input.detach().to(torch.float32).contiguous()
        sq = seq.detach().to(torch.long).contiguous()
        rw = reward.detach().to(torch.float32).contiguous()
        dev = lp.device
        loss = torch.empty(1, dtype=torch.float32, device=dev)
        rows = torch.empty(N, dtype=torch.float32, device=dev)
        msum = torch.empty(1, dtype=torch.float32, device=dev)
        _lib.check(_lib.load().capb200_reward_criterion_forward(_lib.ptr(lp), _lib.ptr(sq), _lib.ptr(rw), N, L, V1, _lib.ptr(loss), _lib.ptr(rows),
                                                                _lib.ptr(msum), _lib.current_stream()), 'reward_criterion_forward')
        self.mask_sum = msum
        return rows if reduction == 'none' else loss[0]

    def backward_logprobs(self, seq, reward, V1, upstream=1.0):
        """d loss_mean / d logprobs as a dense [N, L, V1] tensor (what autograd hands to the reference's log-softmax)."""
        N, L = seq.shape
        grad = torch.zeros(N, L, V1, dtype=torch.float32, device=seq.device)
        sq = seq.detach().to(torch.long).contiguous()
        rw = reward.detach().to(torch.float32).contiguous()
        _lib.check(_lib.load().capb200_reward_criterion_backward(_lib.ptr(sq), _lib.ptr(rw), N, L, V1, _lib.ptr(self.mask_sum), float(upstream),
                                                                 _lib.ptr(grad), _lib.current_stream()), 'reward_criterion_backward')
        return grad


_FUSED_SAMPLERS = "'sample', 'greedy', 'gumbel', 'top<k>' or 'top<p>' with beam size 1"


def _fused_sampler(method):
    """Whether the fused steps draw with ``method`` (CaptionModel.sample_next_word's methods; beam search and the others are not)."""
    if method in ('sample', 'greedy', 'gumbel'):
        return True
    if not (isinstance(method, str) and method.startswith('top')):
        return False
    try:
        return float(method[3:]) > 0
    except ValueError:
        return False


def _shifted_mask(seq):
    # tokens up to and including the first EOS (losses.py:28-29, :57-58)
    m = (seq > 0).to(torch.float32)
    return torch.cat([m.new_ones(m.shape[0], 1), m[:, :-1]], 1)


class LanguageModelCriterion(nn.Module):
    """losses.py:204-225: masked negative log-likelihood of the target tokens (host-level torch ops; the training path uses the fused
    kernels of the capb200_*_xe_step entry points, this module serves evaluation and the parity tests)."""

    def forward(self, input, target, mask, reduction='mean'):
        if target.ndim == 3:
            target, mask = target.reshape(-1, target.shape[2]), mask.reshape(-1, mask.shape[2])
        L = input.shape[1]
        target, mask = target[:, :L], mask[:, :L].to(input)
        nll = -torch.gather(input, 2, target.unsqueeze(2)).squeeze(2) * mask
        return nll.sum(1) / mask.sum(1) if reduction == 'none' else nll.sum() / mask.sum()


class LabelSmoothing(nn.Module):
    """losses.py:228-265: KL divergence to the smoothed target distribution (smoothing / (V1 - 1) off-target, 1 - smoothing on it)."""

    def __init__(self, size=0, padding_idx=0, smoothing=0.0):
        super().__init__()
        self.smoothing, self.confidence = smoothing, 1.0 - smoothing

    def forward(self, input, target, mask, reduction='mean'):
        N, L, V1 = input.shape
        target, mask = target[:, :L].reshape(-1), mask[:, :L].reshape(-1).to(input)
        flat = input.reshape(-1, V1)
        dist = torch.full_like(flat, self.smoothing / (V1 - 1))
        dist.scatter_(1, target.unsqueeze(1), self.confidence)
        kl = (torch.xlogy(dist, dist) - dist * flat).sum(1) * mask
        if reduction == 'none':
            return kl.view(N, L).sum(1) / mask.view(N, L).sum(1)
        return kl.sum() / mask.sum()


class StructureLosses(nn.Module):
    """losses.py:38-200 for ``structure_loss_type='new_self_critical'``: every sample is rewarded with its score (cider_reward_weight *
    CIDEr-D + bleu_reward_weight * BLEU-4) minus the mean score of the image's other samples.  Scores come from the device kernels
    (rewards.get_scores)."""

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        self.loss_type = opt.structure_loss_type
        if self.loss_type != 'new_self_critical':
            raise NotImplementedError("structure_loss_type %r: the engine implements 'new_self_critical'" % self.loss_type)

    def forward(self, input, seq, data_gts, reduction='mean'):
        n = input.shape[0] // len(data_gts)
        assert n == self.opt.train_sample_n, n
        if getattr(self.opt, 'entropy_reward_weight', 0) > 0 or getattr(self.opt, 'self_cider_reward_weight', 0) > 0:
            raise NotImplementedError('entropy / self-CIDEr rewards are out of scope of the engine')
        mask = _shifted_mask(seq)
        scores = get_scores(data_gts, seq, self.opt).to(input).view(-1, n)
        out = {'reward': scores}
        adv = scores - (scores.sum(1, keepdim=True) - scores) / (n - 1)
        picked = torch.gather(input, 2, seq.unsqueeze(2)).squeeze(2)
        term = -picked * mask * adv.reshape(-1, 1)
        out['loss'] = term.sum(1) / mask.sum(1) if reduction == 'none' else term.sum() / mask.sum()
        return out


class _ScstLoss(torch.autograd.Function):
    """Connects the engine-computed loss to the parameters: the gradients were produced by the engine's own BPTT during the forward
    call (into the model's persistent flat gradient buffer); backward hands them (scaled by the upstream gradient) to autograd, so
    loss.backward(), DDP hooks, clip_grad_value_ and the optimizers of tools/train.py:189-196 work unchanged.

    With B200LossWrapper.enable_gradient_sync() the wrapper itself plays DDP's role: the flat buffer has been all-reduced in chunks while
    the step was still running; backward waits for that, scales the buffer in place and makes ``param.grad`` VIEWS of it (no copy; a second
    backward before zero_grad accumulates like autograd would)."""

    @staticmethod
    def forward(ctx, loss_value, grad_list, sync, flat, *params):
        ctx.grad_list = grad_list
        ctx.sync = sync
        ctx.flat = flat
        ctx.params = params
        return loss_value.clone()

    @staticmethod
    def backward(ctx, grad_out):
        if ctx.flat is None:
            # through autograd (nn.DataParallel replicas, torch DDP hooks): one new tensor per parameter
            return (None, None, None, None) + tuple(g * grad_out for g in ctx.grad_list)
        _deliver_views(ctx, grad_out)
        return (None, None, None, None) + tuple(None for _ in ctx.params)


def _deliver_views(ctx, scale):
    """The direct path of the fused steps: the engine's flat gradient buffer is scaled in place by the upstream gradient (ONE launch) and
    every ``param.grad`` becomes a view of it -- no per-parameter kernels, no allocation, and stable gradient addresses from step to step
    (what lets optim.FusedAdam keep its pointer table).  Gradients are NOT accumulated over several fused steps in this mode -- the next
    step overwrites the buffer the views point into, exactly what the reference loop's optimizer.zero_grad() per iteration (tools/train.py:184)
    makes of them anyway; B200LossWrapper.direct_grads = False restores autograd's accumulate-into-.grad behaviour."""
    if ctx.sync is not None:
        ctx.sync.wait()
    ctx.flat.mul_(scale)
    for p_, g in zip(ctx.params, ctx.grad_list):
        if p_.grad is None:
            p_.grad = g
        elif p_.grad.data_ptr() == g.data_ptr():
            pass        # still the view of an earlier step (optimizer.zero_grad(set_to_none=False)): the engine has overwritten it with this step's gradient
        else:
            p_.grad.add_(g)


class _DropWorstLoss(torch.autograd.Function):
    """drop_worst (tools/train.py:187-191): LossWrapper returns one loss per caption row (reduction 'none') and the TRAINER averages the
    k = int(rows * (1 - drop_worst_rate)) smallest.  The fused step has already applied exactly that selection on the device (its gradients
    are those of the mean over the kept rows); backward checks that the upstream gradient is the selection the step assumed -- 1/k on the
    kept rows, 0 elsewhere -- and refuses anything else instead of handing out gradients of a different objective."""

    @staticmethod
    def forward(ctx, row_loss, keep, grad_list, sync, flat, *params):
        ctx.grad_list, ctx.sync, ctx.flat, ctx.params, ctx.keep = grad_list, sync, flat, params, keep
        ctx.save_for_backward(row_loss)
        return row_loss.clone()

    @staticmethod
    def backward(ctx, grad_out):
        (row_loss,) = ctx.saved_tensors
        k = ctx.keep
        kept = torch.zeros_like(row_loss)
        kept[torch.topk(row_loss, k, largest=False).indices] = 1.0 / k
        scale = grad_out.sum()                         # the trainer may multiply the mean by a constant
        if not torch.allclose(grad_out, kept * scale, rtol=1e-4, atol=1e-8):
            raise NotImplementedError('drop_worst: the fused step computed the gradients of the mean over the %d smallest row losses '
                                      '(tools/train.py:191); a different reduction of out[\'loss\'] is not supported' % k)
        if ctx.flat is None:
            return (None, None, None, None, None) + tuple(g * scale for g in ctx.grad_list)
        _deliver_views(ctx, scale)
        return (None, None, None, None, None) + tuple(None for _ in ctx.params)


class B200LossWrapper(nn.Module):
    def __init__(self, model, opt):
        super().__init__()
        self.opt = opt
        self.model = model
        smoothing = getattr(opt, 'label_smoothing', 0)
        self.crit = LabelSmoothing(smoothing=smoothing) if smoothing > 0 else LanguageModelCriterion()      # loss_wrapper.py:10-13
        self.rl_crit = RewardCriterion()
        self.struc_crit = None
        self._sync = None
        self.last_sync_bytes = 0
        # True: backward() points param.grad at views of the engine's flat gradient buffer (fast path).  Set False under torch DDP (its
        # reducer listens to autograd's per-parameter hooks) or for gradient accumulation; nn.DataParallel replicas always go through autograd.
        self.direct_grads = True

    # -- data-parallel gradient synchronisation (the role DDP plays for the reference, tools/train_pl.py:479) -------------------------
    def enable_gradient_sync(self, process_group=None):
        """One process per GPU: after every fused training step the engine's flat gradient buffer is averaged over the ranks with one NCCL
        all-reduce per gradient group, issued on a communication stream as soon as the engine has finished that group (logit first, then the
        decoder, then the refiner layers), i.e. overlapped with the rest of the backward pass.  ``loss.backward()`` then waits for the
        reduced buffer and points ``param.grad`` at it."""
        from .grad_sync import GradSync
        self._sync = GradSync(process_group)
        self.model._grad_sync_on = True            # the engine now records an event per finished gradient group
        return self

    @property
    def last_sync_exposed_ms(self):
        """Device time the last backward() spent waiting for the all-reduce (the part that did not overlap); synchronises."""
        return 0.0 if self._sync is None else self._sync.exposed_ms()

    # -- fused device steps ------------------------------------------------------------------------------------------
    def _bridge(self, res):
        params = list(res['grads'].keys())
        fg = res.get('flat')
        sync = None
        if self._sync is not None and fg is not None:
            self._sync.launch(fg)
            self.last_sync_bytes = self._sync.bytes
            sync = self._sync
        direct = fg is not None and (sync is not None or (self.direct_grads and all(p_.is_leaf for p_ in params)))
        flat = fg.flat if direct else None
        if res.get('row_loss') is not None:          # drop_worst: the per-row vector is what the reference returns as out['loss']
            return _DropWorstLoss.apply(res['row_loss'], int(res['keep_rows']), [res['grads'][p_] for p_ in params], sync, flat, *params)
        return _ScstLoss.apply(res['loss'], [res['grads'][p_] for p_ in params], sync, flat, *params)

    def _keep_rows(self, rows, drop_worst_flag):
        """int(loss.shape[0] * (1 - opt.drop_worst_rate)), the trainer's own arithmetic (tools/train.py:191); 0 when the flag is off."""
        if not drop_worst_flag:
            return 0
        k = int(rows * (1 - float(getattr(self.opt, 'drop_worst_rate', 0))))
        if k < 1:
            raise ValueError('drop_worst_rate leaves no caption rows')
        return k

    def _scorer(self):
        from . import rewards as _rw
        if _rw.CiderD_scorer is None:
            raise RuntimeError('init_scorer(cached_tokens) must be called before the SCST reward (tools/train.py:150-152)')
        return _rw.CiderD_scorer

    def _xe_loss(self, fc_feats, att_feats, labels, masks, att_masks, drop_worst_flag, snapshot=False):
        """loss_wrapper.py:54-55: crit(model(fc, att, labels[..., :-1], att_masks), labels[..., 1:], masks[..., 1:])."""
        if torch.is_grad_enabled() and self.model.training:
            if not hasattr(self.model, 'xe_step'):
                raise NotImplementedError('the fused XE step covers the UpDown, Att2in2, NewFC, AoANet and Transformer families')
            rows = labels.shape[0] * (labels.shape[1] if labels.dim() == 3 else 1)
            keep = self._keep_rows(rows, drop_worst_flag)
            res = self.model.xe_step(fc_feats, att_feats, labels, masks, label_smoothing=getattr(self.opt, 'label_smoothing', 0), att_masks=att_masks,
                                     keep_rows=keep)
            res['keep_rows'] = keep
            if snapshot:        # another fused step will reuse the model's flat gradient buffer before this loss is back-propagated
                res = dict(res, grads={p_: g.clone() for p_, g in res['grads'].items()}, flat=None)
            self.last_step = res
            return self._bridge(res)
        # evaluation (no gradients): the teacher-forced forward of the engine plus the criterion as host-level ops
        reduction = 'none' if drop_worst_flag else 'mean'
        return self.crit(self.model(fc_feats, att_feats, labels[..., :-1], att_masks), labels[..., 1:], masks[..., 1:], reduction=reduction)

    def _weights(self):
        """(cider_reward_weight, bleu_reward_weight), or None for the CIDEr-D reward of the default weights (1, 0)."""
        w = reward_weights(self.opt)
        return None if w == (1.0, 0.0) else w

    def _sampled_step(self, fc_feats, att_feats, gts, baseline, att_masks=None, drop_worst_flag=False):
        opt = self.opt
        self.model.train()
        keep = self._keep_rows(len(gts) * opt.train_sample_n, drop_worst_flag)
        # the reference's training-time _sample call passes no temperature (loss_wrapper.py:63-67): 1.0, whatever opt.temperature says
        w = self._weights()
        extra = {} if w is None else {'reward_weights': w}          # the default weights and samplers call the step exactly as before
        if opt.train_sample_method != 'sample':
            extra['sample_method'] = opt.train_sample_method
        if baseline == 'greedy' and opt.sc_sample_method != 'greedy':
            extra['baseline_method'] = opt.sc_sample_method
        res = self.model.scst_step(fc_feats, att_feats, gts, self._scorer(), opt.train_sample_n, temperature=1.0, baseline=baseline, att_masks=att_masks,
                                   keep_rows=keep, **extra)
        res['keep_rows'] = keep
        self.last_step = res
        return res

    def forward(self, fc_feats, att_feats, labels, masks, att_masks, gts, gt_indices, sc_flag, struc_flag, drop_worst_flag):
        opt = self.opt
        out = {}
        reduction = 'none' if drop_worst_flag else 'mean'
        can_fuse = (hasattr(self.model, 'scst_step') and torch.is_grad_enabled() and
                    _fused_sampler(opt.train_sample_method) and opt.train_beam_size == 1)
        if struc_flag:
            w = opt.structure_loss_weight
            lm_loss = self._xe_loss(fc_feats, att_feats, labels, masks, att_masks, drop_worst_flag, snapshot=w > 0) if w < 1 else \
                torch.zeros((), device=fc_feats.device)
            if w > 0:
                if getattr(opt, 'use_ppo', 0) or opt.structure_loss_type != 'new_self_critical' or not can_fuse:
                    raise NotImplementedError("the structure-loss branch covers structure_loss_type='new_self_critical' on the fused SCST steps")
                if getattr(opt, 'entropy_reward_weight', 0) > 0 or getattr(opt, 'self_cider_reward_weight', 0) > 0:
                    raise NotImplementedError('entropy / self-CIDEr rewards are out of scope of the engine')
                gts = [gts[_] for _ in gt_indices.tolist()]
                if drop_worst_flag and 0 < w < 1:
                    raise NotImplementedError('drop_worst with a mixed XE / structure loss: the two fused steps would select rows independently')
                res = self._sampled_step(fc_feats, att_feats, gts, 'leave_one_out', att_masks, drop_worst_flag)
                rw = self._weights()
                # out['reward'] is the score the step rewarded, in fp32 as losses.py:61-62 casts it
                scores = cider_scores(gts, res['sample_seq']) if rw is None else weighted_scores(gts, res['sample_seq'], rw)
                struc = {'loss': self._bridge(res), 'reward': scores.float().view(-1, opt.train_sample_n)}
            else:
                struc = {'loss': torch.zeros((), device=fc_feats.device), 'reward': torch.zeros((), device=fc_feats.device)}
            out['lm_loss'], out['struc_loss'], out['reward'] = lm_loss, struc['loss'], struc['reward']
            out['loss'] = (1 - w) * lm_loss + w * struc['loss']
            return out
        if not sc_flag:
            out['loss'] = self._xe_loss(fc_feats, att_feats, labels, masks, att_masks, drop_worst_flag)
            return out
        if can_fuse and _fused_sampler(opt.sc_sample_method) and opt.sc_beam_size == 1:
            # whole step on the device incl. the backward pass; dropout as in model.train()
            gts = [gts[_] for _ in gt_indices.tolist()]
            res = self._sampled_step(fc_feats, att_feats, gts, 'greedy', att_masks, drop_worst_flag)
            out['loss'] = self._bridge(res)
            out['reward'] = res['reward'][:, 0].mean()
            return out
        if torch.is_grad_enabled():
            # a differentiable loss exists only on the fused device step: refuse up front instead of returning a detached loss that fails (or
            # silently trains nothing) at backward()
            why = []
            if not hasattr(self.model, 'scst_step'):
                why.append('model family %r has no fused SCST step (UpDown, Att2in2, NewFC, AoANet and Transformer do)' % getattr(self.model, 'family_name', type(self.model).__name__))
            if not _fused_sampler(opt.train_sample_method) or opt.train_beam_size != 1:
                why.append('train_sample_method / train_beam_size other than ' + _FUSED_SAMPLERS)
            if not _fused_sampler(opt.sc_sample_method) or opt.sc_beam_size != 1:
                why.append('sc_sample_method / sc_beam_size other than a baseline drawn by ' + _FUSED_SAMPLERS)
            raise NotImplementedError('self-critical training step outside the fused engine path: ' + '; '.join(why or ['unsupported configuration']))
        # no-grad evaluation of the sc branch (reward monitoring): host-level composition of the engine calls, dropout off
        self.model.eval()
        with torch.no_grad():
            greedy_res, _ = self.model(fc_feats, att_feats, att_masks, mode='sample',
                                       opt={'sample_method': opt.sc_sample_method, 'beam_size': opt.sc_beam_size})
        self.model.train()
        gen_result, sample_logprobs = self.model(fc_feats, att_feats, att_masks,
                                                 opt={'sample_method': opt.train_sample_method, 'beam_size': opt.train_beam_size,
                                                      'sample_n': opt.train_sample_n}, mode='sample')
        gts = [gts[_] for _ in gt_indices.tolist()]
        reward = get_self_critical_reward(greedy_res, gts, gen_result, opt)
        loss = self.rl_crit(sample_logprobs, gen_result, reward, reduction=reduction)
        out['reward'] = reward[:, 0].mean()
        out['loss'] = loss
        return out
