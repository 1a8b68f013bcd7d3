"""Decoding with vocabularies above 51 199 words (V + 1 > 51 200: the vocabulary step runs on a thread-block cluster) for all five
families at small dimensions (E = H = 32), against the oracle run live on the CPU: greedy ids bit-exact wherever the oracle's decision
is clear and log-probs within 1e-4, beam search, teacher forcing, and greedy decoding with decoding_constraint and block_trigrams
(the edited rows are what is stored and what the next word is chosen from).  V = 60 000 makes V + 1 odd (the scalar paths of the
kernels); V = 131 071 spreads each row over three CTAs."""
import pytest
import torch

from helpers import LOGP_TOL, build_pair, check_decode, co
import att2in2_oracle as ao

pytestmark = pytest.mark.gpu

FAMILIES = ['updown', 'att2in2', 'newfc', 'aoa', 'transformer']
# weight seeds whose greedy decisions (the oracle's top-1 / top-2 gaps) are all clear by more than 1e-3, so that the ids are compared bit
# for bit; the others are 0
SEED_SHIFT = {('updown', 60000): 2, ('updown', 131071): 4, ('transformer', 131071): 1}
B, R = 3, 5


def _pair(family, V, seed):
    cfg = dict(V=V, E=32, H=32, A=16, F_fc=48, F_att=48, T=8)
    if family == 'transformer':
        cfg = dict(cfg, H=64, A=2)
    if family == 'att2in2':
        import imagecaptioning.pytorch_b200 as b200
        from helpers import family_opt
        W = co.make_weights('att2in2', V, cfg['E'], cfg['H'], cfg['A'], cfg['F_fc'], cfg['F_att'], seed=seed, logit_scale=8.0)
        model = b200.setup(family_opt('att2in2', **cfg), numeric_mode='tc_f16x3')
        model.load_state_dict(W, strict=True)
        return model.cuda().eval(), ao.Att2in2Family(W, cfg['T']), cfg
    model, fam = build_pair(family, seed=seed, logit_scale=8.0, mode='tc_f16x3', heads=4, **cfg)
    return model, fam, cfg


def _inputs(family, cfg, seed):
    fc, att = co.make_inputs(B, R, cfg['F_fc'], cfg['F_att'], seed=seed)
    return fc, att


def _edited(seq, lp, constraint, trigrams, trigram_rows=None):
    """The reference's edits of the log-prob rows of a replayed sequence (AttModel.py:294-332): the previous word to -inf, then every word
    that completed an earlier trigram with the last two words lowered by 0.693 * 2 per occurrence -- in the first `trigram_rows` rows only
    (the reference's loop runs over the batch size before the sample_n expansion).  Finished rows stay zero."""
    lp = lp.clone().double()
    N, T = seq.shape
    for n in range(N):
        for t in range(1, T):
            if int(seq[n, t - 1]) == 0:
                break
            if constraint:
                lp[n, t, int(seq[n, t - 1])] = float('-inf')
            if trigrams and t >= 3 and (trigram_rows is None or n < trigram_rows):
                p0, p1 = int(seq[n, t - 2]), int(seq[n, t - 1])
                counts = {}
                for i in range(t - 2):
                    if int(seq[n, i]) == p0 and int(seq[n, i + 1]) == p1:
                        w = int(seq[n, i + 2])
                        counts[w] = counts.get(w, 0) + 1
                for w, c in counts.items():
                    lp[n, t, w] += c * -0.693 * 2.0
    return lp


@pytest.mark.parametrize('V', [60000, 131071])
@pytest.mark.parametrize('family', FAMILIES)
def test_greedy_beam_and_teacher_forcing(family, V):
    model, fam, cfg = _pair(family, V, seed=V % 97 + len(family) + 100 * SEED_SHIFT.get((family, V), 0))
    fc, att = _inputs(family, cfg, seed=V % 31)
    fcd, attd = fc.cuda(), att.cuda()
    with torch.no_grad():
        margins = []
        seq, lp = model(fcd, attd, None, opt={'sample_method': 'greedy', 'beam_size': 1}, mode='sample')
        oseq, olp = co.sample(fam, fc, att, record_margin=margins)
        assert lp.shape[-1] == V + 1
        assert check_decode(fam, fc, att, seq, lp, oseq, olp, margins), ('greedy ids were not compared bit for bit', min(margins))

        margins = []
        seq_b, lp_b = model(fcd, attd, None, opt={'beam_size': 3, 'sample_n': 1}, mode='sample')
        oseq_b, olp_b, odone = co.sample_beam(fam, fc, att, beam_size=3, record_margin=margins)
        done_p = [[model.done_beams[i][j]['p'] for j in range(3)] for i in range(B)]
        check_decode(fam, fc, att, seq_b, lp_b, oseq_b, olp_b, margins, done_p=done_p, odone=odone)

        labels = torch.cat([torch.zeros(B, 1, dtype=torch.long), oseq[:, :-1]], 1)
        labels2 = torch.stack([labels, labels.flip(0)], 1)                       # [B, 2, T]
        out = model(fcd, attd, labels2.cuda(), None).cpu()
        ref = co.forward_teacher(fam, fc, att, labels2)
        assert float((out.reshape(ref.shape) - ref).abs().max()) < LOGP_TOL


@pytest.mark.parametrize('V', [60000, 131071])
@pytest.mark.parametrize('family', ['updown', 'transformer'])
def test_greedy_with_decoding_constraint_and_block_trigrams(family, V):
    model, fam, cfg = _pair(family, V, seed=V % 89 + 3)
    fc, att = _inputs(family, cfg, seed=V % 29 + 1)
    fcd, attd = fc.cuda(), att.cuda()
    with torch.no_grad():
        for constraint, trigrams in ((1, 0), (0, 1), (1, 1)):
            opt = {'sample_method': 'greedy', 'beam_size': 1, 'decoding_constraint': constraint, 'block_trigrams': trigrams}
            seq, lp = model(fcd, attd, None, opt=opt, mode='sample')
            seq, lp = seq.cpu(), lp.cpu()
            _, olp = co.sample(fam, fc, att, forced_tokens=seq)
            ref = _edited(seq, olp, constraint, trigrams)
            assert torch.equal(torch.isinf(lp), torch.isinf(ref)), (constraint, trigrams)
            fin = torch.isfinite(ref)
            assert float((lp.double()[fin] - ref[fin]).abs().max()) < LOGP_TOL
            top2 = ref.topk(2, -1).values
            live = torch.ones_like(seq, dtype=torch.bool)
            live[:, 1:] = (seq[:, :-1] != 0).long().cumprod(1).bool()
            clear = live & ((top2[..., 0] - top2[..., 1]) > 1e-3)
            assert torch.equal(seq[clear], ref.argmax(-1)[clear])
            if constraint:
                assert not bool(((seq[:, 1:] == seq[:, :-1]) & (seq[:, 1:] != 0)).any())


def _kept_clearly(ref_row, w, method):
    """Word w of a float64 edited row is inside the kept set of `method` ('top<k>' or 'top<p>'), by more than the fp32 rounding."""
    if method.startswith('top') and '.' not in method:
        return int((ref_row > ref_row[w] + 1e-5).sum()) < int(method[3:])
    p = float(method[3:])
    q = torch.softmax(ref_row, 0)
    return float(q[ref_row > ref_row[w] + 1e-5].sum()) < p + 1e-4


@pytest.mark.parametrize('method', ['sample', 'top5', 'top0.9'])
@pytest.mark.parametrize('V', [60000, 131071])
def test_sampling_with_decoding_constraint_and_block_trigrams(V, method):
    """Sampling (multinomial, top-k, nucleus) with both edits: the stored rows are the oracle's rows of the drawn words, edited; every
    drawn word is one the edited row keeps (so never the previous word)."""
    model, fam, cfg = _pair('updown', V, seed=V % 83 + 5)
    fc, att = _inputs('updown', cfg, seed=V % 23 + 2)
    opt = {'sample_method': method, 'beam_size': 1, 'sample_n': 4, 'decoding_constraint': 1, 'block_trigrams': 1}
    with torch.no_grad():
        torch.manual_seed(11)
        seq, lp = model(fc.cuda(), att.cuda(), None, opt=opt, mode='sample')
    seq, lp = seq.cpu(), lp.cpu()
    _, olp = co.sample(fam, fc, att, sample_n=4, forced_tokens=seq)
    ref = _edited(seq, olp, 1, 1, trigram_rows=B)
    assert torch.equal(torch.isinf(lp), torch.isinf(ref))
    fin = torch.isfinite(ref)
    assert float((lp.double()[fin] - ref[fin]).abs().max()) < LOGP_TOL
    live = torch.ones_like(seq, dtype=torch.bool)
    live[:, 1:] = (seq[:, :-1] != 0).long().cumprod(1).bool()
    for n, t in live.nonzero().tolist():
        w = int(seq[n, t])
        assert torch.isfinite(ref[n, t, w]), (n, t, w)
        if method != 'sample':
            assert _kept_clearly(ref[n, t], w, method), (n, t, w)
    assert not bool(((seq[:, 1:] == seq[:, :-1]) & (seq[:, 1:] != 0)).any())
