"""The selectable samplers of the fused self-critical steps on the H100, for all five families: train_sample_method ('greedy', 'top<k>',
'top<p>') draws only inside the kept set of the step's own log-prob rows and fits the truncated distribution; sc_sample_method draws the
eval-mode baseline the same way from its own seed; replayed (forced) baseline captions give the oracle's loss, reward and gradients; and
the captured step graph is keyed on the samplers."""
import numpy as np
import pytest
import torch

from helpers import LOGP_TOL, co, family_opt

pytestmark = pytest.mark.gpu

FAMILIES = ['updown', 'att2in2', 'newfc', 'aoa', 'transformer']
CFGS = {'updown': dict(V=40, E=32, H=48, A=24, F_fc=40, F_att=40, T=9),
        'att2in2': dict(V=40, E=32, H=48, A=24, F_fc=32, F_att=40, T=9),
        'newfc': dict(V=40, E=32, H=48, A=24, F_fc=40, F_att=40, T=9),
        'aoa': dict(V=40, E=32, H=64, A=0, F_fc=32, F_att=40, T=7),
        'transformer': dict(V=40, E=32, H=64, A=2, F_fc=32, F_att=40, T=7)}
HEADS = {'aoa': 8, 'transformer': 4}
NO_DROPOUT = {'updown': {}, 'att2in2': {}, 'newfc': {}, 'aoa': dict(drop_attn=0.0, drop_aoa=0.0, drop_sublayer=0.0),
              'transformer': dict(dropout=0.0)}


def _model(family, mode='tc_f16x3', seed=31, logit_scale=2.0):
    import imagecaptioning.pytorch_b200 as b200
    c = CFGS[family]
    dims = (c['V'], c['E'], c['H'], c['A'], c['F_fc'], c['F_att'])
    W = co.make_weights(family, *dims, seed=seed, logit_scale=logit_scale)
    m = b200.setup(family_opt(family, *dims, c['T'], heads=HEADS.get(family, 8)), numeric_mode=mode)
    m.load_state_dict(W, strict=True)
    return m.cuda().train(), W


def _inputs(family, B, R=6, seed=4, same=False):
    c = CFGS[family]
    fc, att = co.make_inputs(1 if same else B, R, c['F_fc'], c['F_att'], seed=seed)
    if same:                         # every image identical: the first-step rows of all B * n samples share one distribution
        fc, att = fc.expand(B, -1).contiguous(), att.expand(B, -1, -1).contiguous()
    if family == 'newfc':
        att = fc.new_zeros(B, 0, 0)
    return fc.cuda(), att.cuda()


def _table(V, B):
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    gts = cdo.make_refs(B, V, seed=2)
    df, ref_len = cdo.build_document_frequency(cdo.make_refs(50, V, seed=3))
    return gts, b200.rewards.CiderDTable(df, ref_len), df, ref_len


def _live(seq):
    """[N, T] bool: the steps that drew a word (the first step, and every step after a non-zero word)."""
    live = torch.ones_like(seq, dtype=torch.bool)
    live[:, 1:] = torch.cumprod((seq[:, :-1] > 0).to(torch.int64), 1).bool()
    return live


def _kept(lp, method):
    """[rows, V1] bool: the words the reference's sampler keeps from log-prob rows `lp` (float64), CaptionModel.py:387-404 at T = 1 --
    top-k: every word at least as likely as the k-th (ties at the threshold kept); nucleus: the words whose strictly more likely words hold
    less than p of the mass."""
    lp = lp.double()
    top = float(method[3:])
    if top >= 1:
        kth = lp.topk(int(top), dim=1).values[:, -1:]
        return lp >= kth
    p = lp.exp()
    above = (p.unsqueeze(1) * (lp.unsqueeze(1) > lp.unsqueeze(2))).sum(2)      # [rows, v]: mass of the words more likely than v
    return above < top * p.sum(1, keepdim=True)


def _check_in_kept(seq, lp, method):
    live = _live(seq)
    rows, steps = live.nonzero(as_tuple=True)
    kept = _kept(lp[rows, steps], method)
    ok = kept.gather(1, seq[rows, steps].unsqueeze(1)).squeeze(1)
    assert bool(ok.all()), (method, int((~ok).sum()), int(ok.numel()))
    return kept


@pytest.mark.parametrize('method', ['top1', 'top5', 'top0.5', 'top0.9'])
@pytest.mark.parametrize('family', FAMILIES)
def test_train_samples_fit_truncated_distribution(family, method):
    from scipy import stats
    model, _ = _model(family)
    B, n, V = 640, 16, CFGS[family]['V']
    fc, att = _inputs(family, B, same=True)
    gts, table, _, _ = _table(V, B)
    res = model.scst_step(fc, att, gts, table, n, drop_prob=0.0, seed=99, sample_method=method, **NO_DROPOUT[family])
    seq, lp = res['sample_seq'].cpu(), res['sample_logprobs'].cpu()
    N = B * n
    assert N >= 10 ** 4
    live = _live(seq)
    # the criterion reads the full log-softmax rows (AttModel.py:337,347), not the truncated ones
    assert float(torch.logsumexp(lp.double()[live], 1).abs().max()) < 1e-5
    _check_in_kept(seq, lp, method)
    # first word: every row shares one distribution; the empirical frequencies fit its truncation
    row0 = lp[:, 0].double()
    assert float((row0 - row0[:1]).abs().max()) < 1e-5
    kept = _kept(row0[:1], method)[0]
    probs = row0[0].exp() * kept
    probs = (probs / probs.sum()).numpy()
    counts = np.bincount(seq[:, 0].numpy(), minlength=V + 1)
    assert counts[~kept.numpy()].sum() == 0
    idx = np.flatnonzero(kept.numpy())
    if len(idx) == 1:
        assert counts[idx[0]] == N
        return
    chi2, pval = stats.chisquare(counts[idx], probs[idx] * N)
    assert pval > 1e-4, (method, len(idx), chi2, pval)


@pytest.mark.parametrize('family', FAMILIES)
def test_greedy_train_rows_are_argmax(family):
    model, _ = _model(family)
    B, n, V = 4, 5, CFGS[family]['V']
    fc, att = _inputs(family, B)
    gts, table, _, _ = _table(V, B)
    res = model.scst_step(fc, att, gts, table, n, seed=5, sample_method='greedy')
    seq, lp = res['sample_seq'].cpu(), res['sample_logprobs'].cpu()
    live = _live(seq)
    picked = lp.gather(2, seq.unsqueeze(2)).squeeze(2)
    assert torch.equal(picked[live], lp.max(2).values[live])
    # dropout is on: the n rows of one image differ through their masks only, and greedy rows of different masks do differ
    assert not all(torch.equal(seq[i * n], seq[i * n + j]) for i in range(B) for j in range(1, n))


def _baseline_logprobs(model, fc, att, seq):
    """The eval-mode decode's log-prob rows along the baseline captions `seq` (replayed), for the kept-set check."""
    model.eval()
    with torch.no_grad():
        _, lp = model._sample(fc, att, None, opt={'sample_n': 1}, forced_tokens=seq)
    model.train()
    return lp.cpu()


@pytest.mark.parametrize('method', ['top3', 'top0.6', 'sample', 'gumbel'])
@pytest.mark.parametrize('family', FAMILIES)
def test_sampled_baseline(family, method):
    model, _ = _model(family)
    B, n, V = 64, 2, CFGS[family]['V']
    fc, att = _inputs(family, B)
    gts, table, _, _ = _table(V, B)
    greedy = model.scst_step(fc, att, gts, table, n, seed=7)['greedy_seq'].clone().cpu()
    res = model.scst_step(fc, att, gts, table, n, seed=7, baseline_method=method)
    base, samples = res['greedy_seq'].clone().cpu(), res['sample_seq'].clone().cpu()
    blp = _baseline_logprobs(model, fc, att, base.cuda())
    if method.startswith('top'):
        _check_in_kept(base, blp, method)
    assert not torch.equal(base, greedy)                 # drawn, not the argmax
    # its own seed: another step seed draws other baseline captions, the same seed the same ones
    other = model.scst_step(fc, att, gts, table, n, seed=8, baseline_method=method)['greedy_seq'].clone().cpu()
    again = model.scst_step(fc, att, gts, table, n, seed=7, baseline_method=method)['greedy_seq'].clone().cpu()
    assert not torch.equal(other, base) and torch.equal(again, base)
    # the train samples do not depend on how the baseline is drawn
    assert torch.equal(samples, model.scst_step(fc, att, gts, table, n, seed=7)['sample_seq'].cpu())


def _snapshot(res):
    return {'seq': res['sample_seq'].clone().cpu(), 'base': None if res['greedy_seq'] is None else res['greedy_seq'].clone().cpu(),
            'loss': res['loss'].clone().cpu(), 'reward': res['reward'].clone().cpu(), 'lp': res['sample_logprobs'].clone().cpu(),
            'grads': [g.clone().cpu() for g in res['grads'].values()]}


def _same(a, b):
    """Words, baseline captions, log-probs, reward and loss bit for bit; gradients to 1e-5 of their largest entry."""
    for k in ('seq', 'base', 'loss', 'reward', 'lp'):
        if a[k] is None:
            assert b[k] is None
            continue
        assert torch.equal(a[k], b[k]), k
    # the weight gradients' split-K reductions are not bitwise reproducible from run to run, even for one setting and seed
    for x, y in zip(a['grads'], b['grads']):
        assert float((x - y).abs().max()) <= 1e-5 * float(y.abs().max()) + 1e-9


SETTINGS = [dict(sample_method='top5', baseline_method='top0.9'), dict(sample_method='greedy', baseline_method='sample'),
            dict(), dict(sample_method='top0.5'), dict(baseline_method='top2')]


@pytest.mark.parametrize('family', FAMILIES)
def test_graph_replay_matches_eager_and_is_keyed_on_samplers(family):
    """Each call's outputs equal those of a fresh engine's eager step for the same setting and seed, through eager first sightings,
    captures and replays, while the samplers switch between calls."""
    model, W = _model(family)
    B, n, V = 3, 4, CFGS[family]['V']
    fc, att = _inputs(family, B)
    gts, table, _, _ = _table(V, B)
    calls = [(0, 11), (0, 11), (0, 11), (0, 12), (1, 13), (1, 13), (1, 14), (0, 15), (2, 16), (2, 16), (3, 17), (3, 17), (3, 18), (4, 19),
             (4, 19), (4, 20), (0, 21)]
    eager = {}
    for s, seed in calls:
        got = _snapshot(model.scst_step(fc, att, gts, table, n, seed=seed, **SETTINGS[s]))
        if (s, seed) not in eager:
            fresh, _ = _model(family)
            eager[(s, seed)] = _snapshot(fresh.scst_step(fc, att, gts, table, n, seed=seed, **SETTINGS[s]))
            del fresh
        _same(got, eager[(s, seed)])


@pytest.mark.parametrize('family', FAMILIES)
def test_sampler_settings_launch_the_same_kernels(family):
    """A sampler only changes the vocabulary step's selection and the baseline's method: every setting launches what the default step
    launches, and a replayed baseline adds one word-column load per step."""
    import imagecaptioning.pytorch_b200 as b200
    lib = b200._lib.load()
    count = {'aoa': lib.capb200_aoa_launch_count, 'transformer': lib.capb200_tfm_launch_count}.get(family, lib.capb200_engine_launch_count)
    B, n, V, T = 3, 4, CFGS[family]['V'], CFGS[family]['T']
    fc, att = _inputs(family, B)
    gts, table, _, _ = _table(V, B)
    per_setting = []
    for kw in (dict(), dict(sample_method='sample', baseline_method='greedy'), dict(sample_method='top5', baseline_method='top0.9'),
               dict(sample_method='greedy', baseline_method='gumbel')):
        model, _ = _model(family)
        model.scst_step(fc, att, gts, table, n, seed=3, **kw)                 # eager first sighting
        c0 = count(model._engine)
        model.scst_step(fc, att, gts, table, n, seed=3, **kw)                 # capture
        per_setting.append(count(model._engine) - c0)
    assert len(set(per_setting)) == 1, per_setting
    model, _ = _model(family)
    res = model.scst_step(fc, att, gts, table, n, seed=3)
    base = res['greedy_seq'].clone()
    c0 = count(model._engine)
    model.scst_step(fc, att, gts, table, n, seed=3, forced_baseline=base)
    assert count(model._engine) - c0 == per_setting[0] + T


@pytest.mark.parametrize('family', FAMILIES)
def test_forced_baseline_replays_the_greedy_step(family):
    """Replaying the step's own samples and greedy captions as forced tokens and forced baseline captions reproduces the default step."""
    model, _ = _model(family)
    B, n, V = 3, 4, CFGS[family]['V']
    fc, att = _inputs(family, B)
    gts, table, _, _ = _table(V, B)
    ref = _snapshot(model.scst_step(fc, att, gts, table, n, seed=41))
    got = _snapshot(model.scst_step(fc, att, gts, table, n, seed=41, forced_baseline=ref['base'].cuda(), forced_tokens=ref['seq'].cuda()))
    _same(got, ref)


@pytest.mark.parametrize('baseline_method', ['top5', 'top0.9', 'gumbel'])
@pytest.mark.parametrize('mode', ['tc_f16x3', 'simt_fp32'])
def test_updown_parity_with_oracle_baseline_draw(mode, baseline_method):
    """The oracle draws the train samples and the eval-mode baseline; the engine, set to other samplers, replays both: loss, reward and every
    gradient match torch autograd through the oracle (dropout off, so that the oracle needs no masks).  The samplers choose words only."""
    from oracle import ciderd_oracle as cdo
    model, W = _model('updown', mode=mode, logit_scale=5.0)
    B, R, n, T, V = 5, 11, 4, CFGS['updown']['T'], CFGS['updown']['V']
    fc, att = co.make_inputs(B, R, CFGS['updown']['F_fc'], CFGS['updown']['F_att'], seed=4)
    gts, table, df, ref_len = _table(V, B)
    fam0 = co.Family('updown', W, T)
    torch.manual_seed(3)
    with torch.no_grad():
        o_base, _ = co.sample(fam0, fc, att, sample_method='sample')
        o_seq, _ = co.sample(fam0, fc, att, sample_method='sample', sample_n=n)
    res = model.scst_step(fc.cuda(), att.cuda(), gts, table, n, drop_prob=0.0, seed=1, sample_method='top5', baseline_method=baseline_method,
                          forced_tokens=o_seq.cuda(), forced_baseline=o_base.cuda())
    torch.cuda.synchronize()
    assert torch.equal(res['greedy_seq'].cpu(), o_base) and torch.equal(res['sample_seq'].cpu(), o_seq)
    Wg = {k: v.clone().requires_grad_(True) for k, v in W.items()}
    _, lp = co.sample(co.Family('updown', Wg, T), fc, att, sample_method='sample', sample_n=n, forced_tokens=o_seq)
    reward, _ = cdo.self_critical_reward(o_base.numpy(), gts, o_seq.numpy(), df, ref_len)
    reward = torch.from_numpy(reward).float()
    loss = co.reward_criterion(lp, o_seq, reward)
    loss.backward()
    assert float((res['sample_logprobs'].cpu() - lp.detach()).abs().max()) < LOGP_TOL
    assert float((res['reward'].cpu() - reward).abs().max()) < LOGP_TOL
    assert abs(float(res['loss']) - float(loss)) < LOGP_TOL and abs(float(loss)) > 1e-3
    name_of = {id(p): k for k, p in model.state_dict(keep_vars=True).items()}
    for p, g in res['grads'].items():
        ref = Wg[name_of[id(p)]].grad
        scale = float(ref.abs().max())
        assert float((g.cpu() - ref).abs().max()) <= 5e-4 * scale + 2e-9, name_of[id(p)]


@pytest.mark.parametrize('family', ['updown', 'aoa', 'transformer'])
def test_loss_wrapper_runs_fused_with_samplers(family):
    """B200LossWrapper reads opt.train_sample_method / opt.sc_sample_method and runs the fused step (SCST and new_self_critical)."""
    import argparse
    import imagecaptioning.pytorch_b200 as b200
    model, _ = _model(family)
    B, n, V = 3, 4, CFGS[family]['V']
    fc, att = _inputs(family, B)
    gts, table, _, _ = _table(V, B)
    b200.rewards.reset_scorer()
    b200.rewards.init_scorer(table)
    opt = argparse.Namespace(sc_sample_method='top0.9', sc_beam_size=1, train_sample_method='top3', train_beam_size=1, train_sample_n=n,
                             cider_reward_weight=1, bleu_reward_weight=0, structure_loss_weight=1.0, structure_loss_type='new_self_critical',
                             label_smoothing=0.0)
    lw = b200.B200LossWrapper(model, opt)
    out = lw(fc, att, None, None, None, gts, torch.arange(B), True, False, False)
    assert out['loss'].requires_grad
    step = lw.last_step
    _check_in_kept(step['sample_seq'].cpu(), step['sample_logprobs'].cpu(), 'top3')
    _check_in_kept(step['greedy_seq'].cpu(), _baseline_logprobs(model, fc, att, step['greedy_seq'].clone()), 'top0.9')
    out['loss'].backward()
    assert any(float(p.grad.abs().max()) > 0 for p in model.parameters() if p.grad is not None)
    model.zero_grad(set_to_none=True)
    opt.train_sample_method = 'top0.5'
    out = lw(fc, att, None, None, None, gts, torch.arange(B), False, True, False)
    assert out['loss'].requires_grad and lw.last_step['greedy_seq'] is None
    _check_in_kept(lw.last_step['sample_seq'].cpu(), lw.last_step['sample_logprobs'].cpu(), 'top0.5')
    b200.rewards.reset_scorer()
