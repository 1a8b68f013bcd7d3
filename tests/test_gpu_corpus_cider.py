"""Corpus-mode CIDEr-D on the H100 (init_scorer('corpus') -> CiderD(df='corpus')): the document-frequency table is rebuilt on the device
by every reward call from its own references.  The standalone rewards and every family's fused SCST / new_self_critical step, replaying
the golden's captions, match the reference's own corpus-mode rewards and scores at configs[3] size (tests/golden/corpus_cider.npz, with and
without the BLEU term); the step graph replays a corpus table faithfully and never replays a graph captured for the other table kind."""
import os

import numpy as np
import pytest
import torch

from helpers import co, family_opt

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'corpus_cider.npz')
TOL = 1e-4
FAMILIES = ['updown', 'att2in2', 'newfc', 'aoa', 'transformer']
DIMS = {'updown': (32, 32, 16), 'att2in2': (32, 32, 16), 'newfc': (32, 32, 16), 'aoa': (32, 64, 0), 'transformer': (32, 64, 2)}


def _golden():
    g = np.load(GOLD)
    V, B, n, T = (int(x) for x in g['meta'])
    return g, V, B, n, T, [g['gts'][i] for i in range(B)]


def _loo(scores, n):
    s = torch.from_numpy(scores).float().view(-1, n)
    return (s - (s.sum(1, keepdim=True) - s) / (n - 1)).reshape(-1)


def test_standalone_rewards_match_reference():
    import argparse
    import imagecaptioning.pytorch_b200 as b200
    g, V, B, n, T, gts = _golden()
    b200.rewards.reset_scorer()
    table = b200.rewards.init_scorer('corpus')
    assert isinstance(table, b200.rewards.CorpusCiderDTable)
    sampled, greedy = torch.from_numpy(g['sampled']).cuda(), torch.from_numpy(g['greedy']).cuda()
    try:
        for j, (wc, wb) in enumerate(g['weights']):
            opt = argparse.Namespace(cider_reward_weight=float(wc), bleu_reward_weight=float(wb))
            reward = b200.rewards.get_self_critical_reward(greedy, gts, sampled, opt).cpu().double().numpy()
            assert np.abs(reward - g['reward_%d' % j]).max() < TOL, (wc, wb)
            scores = b200.rewards.get_scores(gts, sampled, opt).cpu().numpy()
            assert np.abs(scores - g['scores_%d' % j]).max() < TOL, (wc, wb)
        # the other entry points read the same kind of table; the entry counts differ between the calls (n + 1 with greedy captions, n without)
        scores, reward = b200.rewards.cider_scores(gts, sampled, with_reward=True)
        assert np.abs(scores.cpu().numpy() - g['scores_0']).max() < TOL
        assert float((reward[:, 0].cpu() - _loo(g['scores_0'], n)).abs().max()) < TOL
        sc, _ = b200.rewards.cider_scores_and_reward(greedy, gts, sampled)
        assert np.abs(sc[:B * n].cpu().numpy() - g['scores_0']).max() > 1e-3          # n + 1 entries per image, not n
    finally:
        b200.rewards.reset_scorer()


def _model(family, V, T):
    import imagecaptioning.pytorch_b200 as b200
    E, H, A = DIMS[family]
    W = co.make_weights(family, V, E, H, A, 24, 24, seed=5, logit_scale=2.0)
    m = b200.setup(family_opt(family, V, E, H, A, 24, 24, T, heads=4 if family == 'transformer' else 8), numeric_mode='tc_f16x3')
    m.load_state_dict(W, strict=True)
    return m.cuda().train()


def _feats(family, B):
    fc, att = co.make_inputs(B, 5, 24, 24, seed=3)
    if family == 'newfc':
        att = fc.new_zeros(B, 0, 0)
    return fc.cuda(), att.cuda()


@pytest.mark.parametrize('family', FAMILIES)
def test_fused_steps_match_reference_corpus_rewards(family):
    import imagecaptioning.pytorch_b200 as b200
    g, V, B, n, T, gts = _golden()
    model = _model(family, V, T)
    fc, att = _feats(family, B)
    table = b200.rewards.CorpusCiderDTable()
    sampled, greedy = torch.from_numpy(g['sampled']).cuda(), torch.from_numpy(g['greedy']).cuda()
    for j, (wc, wb) in enumerate(g['weights']):
        w = None if (wc, wb) == (1.0, 0.0) else (float(wc), float(wb))
        res = model.scst_step(fc, att, gts, table, n, seed=1, forced_tokens=sampled, forced_baseline=greedy, reward_weights=w)
        assert float((res['reward'].cpu().double() - torch.from_numpy(g['reward_%d' % j])).abs().max()) < TOL, (wc, wb)
        res = model.scst_step(fc, att, gts, table, n, seed=1, forced_tokens=sampled, baseline='leave_one_out', reward_weights=w)
        assert float((res['reward'][:, 0].cpu() - _loo(g['scores_%d' % j], n)).abs().max()) < TOL, (wc, wb)


def _launches(model):
    import imagecaptioning.pytorch_b200 as b200
    return b200._lib.load().capb200_engine_launch_count(model._engine)


def test_step_graph_with_corpus_and_pickle_tables():
    """Calls alternate between a pickle table and a corpus table, with the step graph capturing and replaying each: every call equals a
    fresh engine's eager call of the same table and seed, and a replayed corpus step launches exactly the three build kernels more."""
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    g, V, B, n, T, gts = _golden()
    fc, att = _feats('updown', B)
    corpus = b200.rewards.CorpusCiderDTable()
    pickle_table = b200.rewards.CiderDTable(*cdo.build_document_frequency(cdo.make_refs(60, V, seed=3, L=T)))
    tables = {'corpus': corpus, 'pickle': pickle_table}
    model = _model('updown', V, T)
    eager, per_call = {}, {}
    for kind, seed in [('pickle', 1), ('pickle', 1), ('pickle', 2), ('corpus', 3), ('corpus', 3), ('corpus', 4), ('corpus', 5), ('pickle', 6),
                       ('corpus', 7)]:
        c0 = _launches(model)
        res = model.scst_step(fc, att, gts, tables[kind], n, seed=seed)
        per_call[(kind, seed)] = _launches(model) - c0
        got = (res['sample_seq'].clone().cpu(), res['greedy_seq'].clone().cpu(), res['reward'].clone().cpu(), res['loss'].clone().cpu())
        if (kind, seed) not in eager:
            fresh = _model('updown', V, T)
            r = fresh.scst_step(fc, att, gts, tables[kind], n, seed=seed)
            eager[(kind, seed)] = (r['sample_seq'].clone().cpu(), r['greedy_seq'].clone().cpu(), r['reward'].clone().cpu(), r['loss'].clone().cpu())
            del fresh
        for a, b in zip(got, eager[(kind, seed)]):
            assert torch.equal(a, b), (kind, seed)
    # replays (the first sighting of a configuration also pays one-time set-up launches)
    assert per_call[('corpus', 4)] == per_call[('corpus', 5)] == per_call[('pickle', 2)] + 3
