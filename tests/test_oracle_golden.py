"""CPU: the oracle restatement must reproduce the vectors the live reference produced (tests/golden, made by
oracle/make_golden.py).  This is what pins the oracle; every GPU parity test then compares against the oracle."""
import os

import numpy as np
import pytest
import torch

from oracle import caption_oracle as co
from oracle import ciderd_oracle as cdo

TOL = 1e-4   # north_star: log-probs and CIDEr-D rewards within 1e-4 fp32


def _load(golden_dir, name):
    return np.load(os.path.join(golden_dir, name))


def _family(g, name, scale):
    V, E, H, A, F_fc, F_att, T = (int(x) for x in g['cfg'])
    B, R, b, seed = (int(x) for x in g['meta'])
    W = co.make_weights(name, V, E, H, A, F_fc, F_att, seed=seed, logit_scale=scale)
    fc, att = co.make_inputs(B, R, F_fc, F_att, seed=seed)
    return co.Family(name, W, T), fc, att, b


def test_updown_small_greedy_and_beam(golden_dir):
    g = _load(golden_dir, 'updown_small.npz')
    fam, fc, att, b = _family(g, 'updown', 20.0)
    seq, lp = co.sample(fam, fc, att)
    assert np.array_equal(seq.numpy(), g['greedy_seq'])
    assert np.abs(lp.numpy() - g['greedy_lp']).max() < TOL
    seq, lp, done = co.sample_beam(fam, fc, att, beam_size=b)
    assert np.array_equal(seq.numpy(), g['beam_seq'])
    assert np.abs(lp.numpy() - g['beam_lp']).max() < TOL
    for i, lst in enumerate(done):
        for j, rec in enumerate(lst):
            L = int(g['done_len'][i, j])
            assert rec['seq'].tolist() == g['done_seq'][i, j, :L].tolist()
            assert abs(rec['p'] - g['done_p'][i, j]) < 1e-3
    seq, _, _ = co.sample_beam(fam, fc, att, beam_size=b, sample_n=b)
    assert np.array_equal(seq.numpy(), g['beamn_seq'])


def test_updown_small_masks_teacher_sample(golden_dir):
    g = _load(golden_dir, 'updown_small.npz')
    fam, fc, att, b = _family(g, 'updown', 20.0)
    masks = torch.from_numpy(g['masks'])
    seq, lp = co.sample(fam, fc, att, masks)
    assert np.array_equal(seq.numpy(), g['masked_greedy_seq'])
    assert np.abs(lp.numpy() - g['masked_greedy_lp']).max() < TOL
    seq, _, _ = co.sample_beam(fam, fc, att, masks, beam_size=b)
    assert np.array_equal(seq.numpy(), g['masked_beam_seq'])
    out = co.forward_teacher(fam, fc, att, torch.from_numpy(g['teacher_in']))
    assert np.abs(out.numpy() - g['teacher_lp']).max() < TOL
    # the reference's random stream is torch.multinomial's; replay its tokens and compare the stored rows
    forced = torch.from_numpy(g['sample_seq'])
    seq, lp = co.sample(fam, fc, att, sample_method='sample', sample_n=3, forced_tokens=forced)
    assert np.array_equal(seq.numpy(), g['sample_seq'])
    assert np.abs(lp.numpy() - g['sample_lp']).max() < TOL


def test_newfc_config1(golden_dir):
    """BASELINE.json configs[0]: newfc greedy, batch 4, 2048-d fc feats, seq_len 16, CPU."""
    g = _load(golden_dir, 'newfc_cfg1.npz')
    fam, fc, att, _ = _family(g, 'newfc', 12.0)
    seq, lp = co.sample(fam, fc, att)
    assert np.array_equal(seq.numpy(), g['greedy_seq'])
    picked = lp.gather(2, seq.unsqueeze(2)).squeeze(2)
    assert np.abs(picked.numpy() - g['greedy_picked_lp']).max() < TOL
    seq, _, done = co.sample_beam(fam, fc, att, beam_size=3)
    assert np.array_equal(seq.numpy(), g['beam_seq'])
    assert np.abs(np.array([[r['p'] for r in d] for d in done]) - g['done_p']).max() < 1e-3


@pytest.mark.slow
def test_updown_full_dims(golden_dir):
    g = _load(golden_dir, 'updown_full.npz')
    fam, fc, att, b = _family(g, 'updown', 12.0)
    seq, lp = co.sample(fam, fc, att)
    assert np.array_equal(seq.numpy(), g['greedy_seq'])
    picked = lp.gather(2, seq.unsqueeze(2)).squeeze(2)
    assert np.abs(picked.numpy() - g['greedy_picked_lp']).max() < TOL
    seq, lp, done = co.sample_beam(fam, fc, att, beam_size=b)
    assert np.array_equal(seq.numpy(), g['beam_seq'])
    assert np.abs(np.array([[r['p'] for r in d] for d in done]) - g['done_p']).max() < 1e-3


def _df_from_golden(g):
    return {tuple(int(t) for t in k if t >= 0): float(v) for k, v in zip(g['df_keys'], g['df_vals'])}


def test_ciderd_scores_and_reward(golden_dir):
    g = _load(golden_dir, 'ciderd.npz')
    df = _df_from_golden(g)
    V, B, n, T = (int(x) for x in g['meta'])
    gts = [g['gts'][i] for i in range(B)]
    reward, scores = cdo.self_critical_reward(g['greedy'], gts, g['sampled'], df, float(g['ref_len']))
    assert np.abs(reward - g['reward']).max() < 1e-9
    assert np.abs(scores[:B * n] - g['sample_scores']).max() < 1e-9
    # the DF builder reproduces the table the reference's compute_doc_freq produced
    df2, n_img = cdo.build_document_frequency(cdo.make_refs(300, V, seed=3))
    assert df2 == df and n_img == int(g['ref_len'])


def test_reward_criterion(golden_dir):
    g = _load(golden_dir, 'reward_criterion.npz')
    lp, seq, reward = (torch.from_numpy(g[k]) for k in ('lp', 'seq', 'reward'))
    assert abs(float(co.reward_criterion(lp, seq, reward)) - float(g['loss'])) < 1e-6
    assert np.abs(co.reward_criterion(lp, seq, reward, 'none').numpy() - g['loss_none']).max() < 1e-6
    assert np.abs(co.reward_criterion_grad(seq, reward, lp.shape[2]).numpy() - g['grad']).max() < 1e-7


def _family_small(golden_dir, fname, family, scale):
    g = _load(golden_dir, fname)
    V, E, H, A, F_fc, F_att, T = (int(x) for x in g['cfg'])
    B, R, b, seed, heads = (int(x) for x in g['meta'])
    W = co.make_weights(family, V, E, H, A, F_fc, F_att, seed=seed, logit_scale=scale)
    fc, att = co.make_inputs(B, R, F_fc, F_att, seed=seed)
    return g, co.Family(family, W, T, heads=heads), fc, att, b


@pytest.mark.parametrize('fname,family,scale', [('transformer_small.npz', 'transformer', 10.0), ('aoa_small.npz', 'aoa', 20.0)])
def test_transformer_and_aoa_small(golden_dir, fname, family, scale):
    g, fam, fc, att, b = _family_small(golden_dir, fname, family, scale)
    seq, lp = co.sample(fam, fc, att)
    assert np.array_equal(seq.numpy(), g['greedy_seq'])
    assert np.abs(lp.numpy() - g['greedy_lp']).max() < TOL
    seq, lp, done = co.sample_beam(fam, fc, att, beam_size=b)
    assert np.array_equal(seq.numpy(), g['beam_seq'])
    assert np.abs(lp.numpy() - g['beam_lp']).max() < TOL
    assert np.abs(np.array([[r['p'] for r in d] for d in done]) - g['done_p']).max() < 1e-3
    masks = torch.from_numpy(g['masks'])
    seq, lp = co.sample(fam, fc, att, masks)
    assert np.array_equal(seq.numpy(), g['masked_greedy_seq'])
    assert np.abs(lp.numpy() - g['masked_greedy_lp']).max() < TOL
    seq, _, _ = co.sample_beam(fam, fc, att, masks, beam_size=b)
    assert np.array_equal(seq.numpy(), g['masked_beam_seq'])
    out = co.forward_teacher(fam, fc, att, torch.from_numpy(g['teacher_in']))
    assert np.abs(out.numpy() - g['teacher_lp']).max() < TOL
    seq, lp = co.sample(fam, fc, att, sample_method='sample', sample_n=3, forced_tokens=torch.from_numpy(g['sample_seq']))
    assert np.abs(lp.numpy() - g['sample_lp']).max() < TOL


def test_xe_criteria_and_structure_loss(golden_dir):
    """LanguageModelCriterion, LabelSmoothing and StructureLosses('new_self_critical') restatements against the live reference's values."""
    g = _load(golden_dir, 'xe_struct.npz')
    labels, masks = torch.from_numpy(g['crit_labels']), torch.from_numpy(g['crit_masks'])
    for name, fn in (('lm', co.language_model_criterion), ('ls', lambda a, b, c, r='mean': co.label_smoothing_loss(a, b, c, 0.2, r))):
        x = torch.from_numpy(g['crit_lp']).clone().requires_grad_(True)
        loss = fn(x, labels[:, 1:], masks[:, 1:])
        loss.backward()
        assert abs(float(loss) - float(g[name + '_loss'])) < 1e-6
        assert np.abs(x.grad.numpy() - g[name + '_grad']).max() < 1e-7
        assert np.abs(fn(x.detach(), labels[:, 1:], masks[:, 1:], 'none').numpy() - g[name + '_loss_none']).max() < 1e-6
    c = _load(golden_dir, 'ciderd.npz')
    V, B, n, T = (int(x) for x in c['meta'])
    gts = [c['gts'][i] for i in range(B)]
    scores = cdo.get_scores(gts, c['sampled'], _df_from_golden(c), float(c['ref_len']))
    assert np.abs(scores - g['struc_scores']).max() < 1e-9
    x = torch.from_numpy(g['struc_lp']).clone().requires_grad_(True)
    loss = co.new_self_critical_loss(x, torch.from_numpy(c['sampled']), torch.from_numpy(scores), n)
    loss.backward()
    assert abs(float(loss) - float(g['struc_loss'])) < 1e-6
    assert np.abs(x.grad.numpy() - g['struc_grad']).max() < 1e-7
    assert np.abs(scores.reshape(B, n) - g['struc_reward']).max() < 1e-6


@pytest.mark.parametrize('name,smoothing', [('xe', 0.0), ('xels', 0.1)])
def test_xe_step_of_the_reference_model(golden_dir, name, smoothing):
    """Teacher-forced forward (train mode, no dropout) + criterion + autograd through the oracle reproduce the reference model's XE loss
    and parameter gradients; the labels end before the last column, so the data-dependent early break (AttModel.py:158-159) is covered."""
    g = _load(golden_dir, 'xe_struct.npz')
    V, E, H, A, F_fc, F_att, T, B, R, spi, seed = (int(x) for x in g['xe_cfg'])
    W = co.make_weights('updown', V, E, H, A, F_fc, F_att, seed=seed, logit_scale=20.0)
    Wg = {k: v.clone().requires_grad_(True) for k, v in W.items()}
    fc, att = co.make_inputs(B, R, F_fc, F_att, seed=seed)
    labels, masks = torch.from_numpy(g['xe_labels']), torch.from_numpy(g['xe_masks'])
    lp = co.forward_teacher(co.Family('updown', Wg, T), fc, att, labels[..., :-1])
    if smoothing == 0:
        assert np.abs(lp.detach().numpy() - g['xe_logprobs']).max() < TOL
        assert float(lp[:, -1].abs().max()) == 0.0                       # columns after the early break stay zero
        loss = co.language_model_criterion(lp, labels[..., 1:], masks[..., 1:])
    else:
        loss = co.label_smoothing_loss(lp, labels[..., 1:], masks[..., 1:], smoothing)
    loss.backward()
    assert abs(float(loss) - float(g[name + '_loss'])) < 1e-5
    for k in g.files:
        if k.startswith(name + '_grad_'):
            ref = g[k]
            got = Wg[k[len(name) + 6:]].grad.numpy()
            assert np.abs(got - ref).max() < 1e-5 * max(1.0, np.abs(ref).max()), k


def test_ciderd_on_real_captions(golden_dir):
    """CIDEr-D restatement against the live reference scorer on real text: 60 PASCAL-50S images with 50 references each and their
    candidate captions (cider/data/pascal50S.json, pascal_candsB.json), document frequencies from the reference's compute_doc_freq."""
    g = _load(golden_dir, 'ciderd_pascal.npz')
    df = _df_from_golden(g)
    refs, cands = g['refs'].astype(np.int64), g['cands'].astype(np.int64)
    gts = [refs[i] for i in range(refs.shape[0])]
    scores = cdo.get_scores(gts, cands, df, float(g['ref_len']))
    assert np.abs(scores - g['scores']).max() < 1e-9
    assert abs(float(scores.mean()) - float(g['mean'])) < 1e-9 and float(g['mean']) > 0.3
    # the document-frequency builder reproduces the reference's table on real text too
    df2, n_img = cdo.build_document_frequency(gts)
    assert df2 == df and n_img == int(g['ref_len'])


@pytest.mark.parametrize('tag,pen', [('wu', 'wu_0.5'), ('avg', 'avg_0'), ('wu2', 'wu_1.5')])
def test_beam_length_penalties(golden_dir, tag, pen):
    """misc.penalty_builder (length_wu / length_average) only re-ranks the finished beams ('p'): ids, log-probs and penalised scores of
    the reference's beam search with each penalty."""
    g = _load(golden_dir, 'updown_penalty.npz')
    V, E, H, A, F_fc, F_att, T = (int(x) for x in g['cfg'])
    B, R, b, seed = (int(x) for x in g['meta'])
    W = co.make_weights('updown', V, E, H, A, F_fc, F_att, seed=seed, logit_scale=20.0)
    fc, att = co.make_inputs(B, R, F_fc, F_att, seed=seed)
    seq, lp, done = co.sample_beam(co.Family('updown', W, T), fc, att, beam_size=b, length_penalty=pen)
    assert np.array_equal(seq.numpy(), g[tag + '_seq'])
    assert np.abs(lp.numpy() - g[tag + '_lp']).max() < TOL
    assert np.abs(np.array([[r['p'] for r in d] for d in done]) - g[tag + '_done_p']).max() < 1e-3


def test_aoa_scst_step_at_config_dims(golden_dir):
    """The oracle at BASELINE configs[3]'s own size (AoANet H = 1024, V = 9487, 10 images x 5 samples): loss, reward and the gradient
    fingerprints of the reference's LossWrapper(sc_flag=True) step (tests/golden/aoa_scst_full.npz), with the reference's samples replayed."""
    g = _load(golden_dir, 'aoa_scst_full.npz')
    V, E, H, A, F_fc, F_att, T = (int(x) for x in g['cfg'])
    B, R, n, seed, heads = (int(x) for x in g['meta'])
    W = co.make_weights('aoa', V, E, H, A, F_fc, F_att, seed=seed, logit_scale=6.0)
    fc, att = co.make_inputs(B, R, F_fc, F_att, seed=seed)
    og, _ = co.sample(co.Family('aoa', W, T, heads=heads), fc, att)
    assert np.array_equal(og.numpy(), g['greedy_seq'].astype(np.int64))
    df = {tuple(int(t) for t in k if t >= 0): float(v) for k, v in zip(g['df_keys'], g['df_vals'])}
    gts = [g['gts'][i].astype(np.int64) for i in range(B)]
    sample_seq = torch.from_numpy(g['sample_seq'].astype(np.int64))
    reward, _ = cdo.self_critical_reward(og.numpy(), gts, sample_seq.numpy(), df, float(g['ref_len']))
    assert np.abs(reward[:, 0] - g['reward']).max() < 1e-9
    Wg = {k: v.clone().requires_grad_(True) for k, v in W.items()}
    fam = co.Family('aoa', Wg, T, heads=heads)
    _, lp = co.sample(fam, fc, att, sample_method='sample', sample_n=n, forced_tokens=sample_seq)
    loss = co.reward_criterion(lp, sample_seq, torch.from_numpy(reward).float())
    loss.backward()
    assert abs(float(loss) - float(g['loss'])) < TOL * abs(float(g['loss']))
    largest = max(float(g['t_' + k][3]) for k in g['names'])
    for k in g['names']:
        a = Wg[str(k)].grad.numpy()
        step, stats = g['s_' + k], g['t_' + k]
        sub = a if a.size <= 8192 else (a[::int(step[0])] if a.ndim == 1 else a[::int(step[0]), ::int(step[1])])
        assert np.abs(sub - g['g_' + k]).max() <= 2e-4 * float(stats[3]) + 1e-7 * largest, k


def test_transformer_training_steps_of_the_reference(golden_dir):
    """The oracle's Transformer training path (teacher-forced pass with the pad/eos + causal mask; sampled prefixes with the causal mask only)
    against the LIVE reference's LossWrapper + backward() (transformer_train_small.npz: XE with both criteria, the sc branch with the
    reference's own draw): losses, log-probs, rewards and all 93 gradients."""
    g = np.load(os.path.join(golden_dir, 'transformer_train_small.npz'))
    cfg = dict(zip(('V', 'E', 'H', 'A', 'F_fc', 'F_att', 'T'), (int(v) for v in g['cfg'])))
    B, R, n, seed, heads, spi, _ = (int(x) for x in g['meta'])
    W = co.make_weights('transformer', cfg['V'], cfg['E'], cfg['H'], cfg['A'], cfg['F_fc'], cfg['F_att'], seed=seed, logit_scale=float(g['logit_scale']))
    fc, att = co.make_inputs(B, R, cfg['F_fc'], cfg['F_att'], seed=seed)
    labels, masks = torch.from_numpy(g['xe_labels'].astype(np.int64)), torch.from_numpy(g['xe_masks'])
    N = B * spi

    def grads_of(loss, Wg, prefix):
        loss.backward()
        largest = max(float(np.abs(g[prefix + 'g_' + k]).max()) for k in g['names'])
        for k in g['names']:
            ref = g[prefix + 'g_' + k]
            # key biases have a true gradient of zero (softmax is shift invariant): held to 1e-6 of the step's largest gradient
            assert np.abs(Wg[k].grad.numpy() - ref).max() <= 2e-5 * np.abs(ref).max() + 1e-6 * largest, (prefix, k)

    for prefix, smoothing in (('xe_', 0.0), ('xels_', 0.1)):
        Wg = {k: (v.clone().requires_grad_(True) if k in set(g['names']) else v) for k, v in W.items()}
        fam = co.Family('transformer', Wg, cfg['T'], heads=heads)
        lp = co.forward_teacher(fam, fc, att, labels[..., :-1])
        fl, fm = labels.reshape(N, -1), masks.reshape(N, -1)
        loss = co.label_smoothing_loss(lp, fl[:, 1:], fm[:, 1:], smoothing) if smoothing > 0 else co.language_model_criterion(lp, fl[:, 1:], fm[:, 1:])
        assert abs(float(loss) - float(g[prefix + 'loss'])) < 1e-5 * max(1.0, abs(float(loss)))
        if prefix == 'xe_':
            assert np.abs(lp.detach().numpy() - g['xe_logprobs']).max() < 1e-5
        grads_of(loss, Wg, prefix)
    Wg = {k: (v.clone().requires_grad_(True) if k in set(g['names']) else v) for k, v in W.items()}
    fam = co.Family('transformer', Wg, cfg['T'], heads=heads)
    seq = torch.from_numpy(g['sample_seq'].astype(np.int64))
    seq_in = torch.cat([torch.zeros(seq.shape[0], 1, dtype=torch.long), seq[:, :-1]], 1)
    lp = co.forward_teacher(fam, fc, att, seq_in, None, pad_keys_masked=False)          # one causal pass == the reference's step-by-step prefixes
    lp = lp * torch.cat([torch.ones(seq.shape[0], 1, dtype=torch.bool), seq[:, :-1] > 0], 1).unsqueeze(2)
    df = _df_from_golden(g)
    gts = [g['gts'][i].astype(np.int64) for i in range(B)]
    with torch.no_grad():
        og, _ = co.sample(co.Family('transformer', W, cfg['T'], heads=heads), fc, att)
    assert np.array_equal(og.numpy(), g['greedy_seq'].astype(np.int64))
    reward, _ = cdo.self_critical_reward(og.numpy(), gts, seq.numpy(), df, float(g['ref_len']))
    assert np.abs(reward[:, 0] - g['reward']).max() < 1e-9
    loss = co.reward_criterion(lp, seq, torch.from_numpy(reward).float())
    assert abs(float(loss) - float(g['sc_loss'])) < 1e-5
    grads_of(loss, Wg, 'sc_')


@pytest.mark.parametrize('family', ['updown', 'att2in2', 'aoa'])
def test_oracle_runs_in_float64(family):
    """Given float64 weights and features the oracle computes in float64 throughout (its state, sampled and teacher-forced log-prob
    buffers follow the inputs' dtype), and agrees with its float32 self within 1e-5 of each tensor's largest entry."""
    import att2in2_oracle as ao
    V, E, H, A, F_fc, F_att, T, B, R, n = 30, 16, 24, 12, 20, 20, 6, 3, 5, 2
    W = co.make_weights(family, V, E, H, A, F_fc, F_att, seed=3, logit_scale=3.0)
    fc, att = co.make_inputs(B, R, F_fc, F_att, seed=2)
    masks = torch.ones(B, R)
    masks[1, 3:] = 0
    tok = torch.randint(1, V + 1, (B * n, T), generator=torch.Generator().manual_seed(1))
    tok[0, 2:] = 0
    reward = torch.randn(B * n, 1, generator=torch.Generator().manual_seed(4)).expand(-1, T)
    out = {}
    for dt in (torch.float32, torch.float64):
        Wg = {k: v.to(dt, copy=True).requires_grad_(True) for k, v in W.items()}
        fam = ao.Att2in2Family(Wg, T) if family == 'att2in2' else co.Family(family, Wg, T, heads=4)
        _, lp = co.sample(fam, fc.to(dt), att.to(dt), masks, sample_method='sample', sample_n=n, forced_tokens=tok)
        tf = co.forward_teacher(fam, fc.to(dt), att.to(dt), torch.cat([torch.zeros(B * n, 1, dtype=torch.long), tok], 1).view(B, n, -1), masks)
        assert lp.dtype == dt and tf.dtype == dt
        (co.reward_criterion(lp, tok, reward.to(dt)) + tf.sum() * 1e-3).backward()
        assert all(v.grad is not None and v.grad.dtype == dt for v in Wg.values())
        out[dt] = (lp.detach(), {k: v.grad for k, v in Wg.items()})
    (lp32, g32), (lp64, g64) = out[torch.float32], out[torch.float64]
    assert float((lp64 - lp32.double()).abs().max()) <= 1e-5 * float(lp64.abs().max())
    largest = max(float(v.abs().max()) for v in g64.values())
    for k in g64:          # tensors whose true gradient is zero (alpha_net.bias, attention key biases) hold fp32 noise of the step's size
        assert float((g64[k] - g32[k].double()).abs().max()) <= 1e-5 * float(g64[k].abs().max()) + 1e-7 * largest, k
