"""CPU tests of the host-side mirrors: the criterion modules against the live-reference goldens, the option guards, and the
"fail loudly without CUDA" contract of the product path (no CPU fallback anywhere)."""
import argparse
import os

import numpy as np
import pytest
import torch

from helpers import co, family_opt

GOLD = os.path.join(os.path.dirname(__file__), 'golden')


def test_criterion_modules_match_reference_golden():
    """loss_wrapper.LanguageModelCriterion / LabelSmoothing (host-level torch ops) reproduce the reference's losses and gradients."""
    from imagecaptioning.pytorch_b200.loss_wrapper import LabelSmoothing, LanguageModelCriterion
    g = np.load(os.path.join(GOLD, 'xe_struct.npz'))
    labels, masks = torch.from_numpy(g['crit_labels']), torch.from_numpy(g['crit_masks'])
    for name, crit in (('lm', LanguageModelCriterion()), ('ls', LabelSmoothing(smoothing=0.2))):
        x = torch.from_numpy(g['crit_lp']).clone().requires_grad_(True)
        loss = crit(x, labels[:, 1:], masks[:, 1:])
        loss.backward()
        assert abs(float(loss.detach()) - float(g[name + '_loss'])) < 1e-6
        assert np.abs(x.grad.numpy() - g[name + '_grad']).max() < 1e-7
        none = crit(x.detach(), labels[:, 1:], masks[:, 1:], reduction='none')
        assert np.abs(none.numpy() - g[name + '_loss_none']).max() < 1e-6


@pytest.mark.parametrize('family', ['updown', 'newfc', 'transformer', 'aoa'])
def test_product_path_refuses_cpu_tensors(family):
    """Every family's decode raises instead of computing on the CPU (the engine has no CPU or PyTorch-op fallback)."""
    import imagecaptioning.pytorch_b200 as b200
    cfg = dict(V=30, E=16, H=16, A=8, F_fc=16, F_att=16, T=5)
    if family == 'transformer':
        cfg = dict(cfg, E=16, H=32, A=1)
    model = b200.setup(family_opt(family, heads=2, **cfg))
    fc, att = co.make_inputs(2, 3, 16, 16, seed=1)
    with pytest.raises(RuntimeError, match='CUDA'):
        model(fc, att, None, opt={'sample_method': 'greedy', 'beam_size': 1}, mode='sample')


def test_loss_wrapper_option_guards():
    """Unsupported LossWrapper configurations raise NotImplementedError before any device work (structure losses other than
    new_self_critical, PPO) and the reward needs init_scorer."""
    import imagecaptioning.pytorch_b200 as b200
    model = b200.setup(family_opt('updown', V=30, E=16, H=16, A=8, F_fc=16, F_att=16, T=5))
    opt = argparse.Namespace(sc_sample_method='greedy', sc_beam_size=1, train_sample_method='sample', train_beam_size=1, train_sample_n=2,
                             cider_reward_weight=1, bleu_reward_weight=0, label_smoothing=0.0, structure_loss_weight=1.0,
                             structure_loss_type='softmax_margin', use_ppo=0)
    lw = b200.B200LossWrapper(model, opt)
    fc, att = co.make_inputs(2, 3, 16, 16, seed=1)
    gts = [np.zeros((5, 7), np.int64)] * 2
    with pytest.raises(NotImplementedError):
        lw(fc, att, None, None, None, gts, torch.arange(2), False, True, False)
    b200.rewards.reset_scorer()
    opt.structure_loss_type = 'new_self_critical'
    with pytest.raises(RuntimeError, match='init_scorer'):
        lw(fc, att, None, None, None, gts, torch.arange(2), True, False, False)
    with pytest.raises(NotImplementedError):
        b200.loss_wrapper.StructureLosses(argparse.Namespace(structure_loss_type='risk'))


def test_bench_gpu_arm_does_not_import_the_oracle():
    """Only bench.py's CPU-baseline legs (cpu_reference_rate / cpu_reference_scst_rate) may touch oracle/ (or the test helpers that import it); the measured GPU arms build their synthetic
    model and inputs from the package's own generators."""
    import ast
    src = open(os.path.join(os.path.dirname(os.path.dirname(__file__)), 'bench.py')).read()
    tree = ast.parse(src)
    offenders = []
    for fn in [n for n in ast.walk(tree) if isinstance(n, ast.FunctionDef)] + [tree]:
        for node in ast.walk(fn):
            names = []
            if isinstance(node, ast.Import):
                names = [a.name for a in node.names]
            elif isinstance(node, ast.ImportFrom):
                names = [node.module or '']
            for nm in names:
                if nm.split('.')[0] in ('oracle', 'helpers') and getattr(fn, 'name', '<module>') not in ('cpu_reference_rate', 'cpu_reference_scst_rate'):
                    if isinstance(fn, ast.Module) and any(node in ast.walk(f) for f in ast.walk(tree) if isinstance(f, ast.FunctionDef)):
                        continue                      # counted with its enclosing function
                    offenders.append((getattr(fn, 'name', '<module>'), nm))
    assert offenders == [], offenders


def test_product_and_tools_never_import_the_oracle():
    """The package (the product path) and the profiling tools must not import oracle/ or the test helpers: the oracle is test infrastructure."""
    import ast
    root = os.path.dirname(os.path.dirname(__file__))
    files = []
    for sub in ('imagecaptioning.pytorch_b200', 'tools'):
        d = os.path.join(root, sub)
        files += [os.path.join(d, f) for f in os.listdir(d) if f.endswith('.py')]
    files.append(os.path.join(root, '__graft_entry__.py'))
    offenders = []
    for path in files:
        tree = ast.parse(open(path).read())
        scopes = [tree] if not path.endswith('__graft_entry__.py') else [n for n in ast.walk(tree) if isinstance(n, ast.FunctionDef) and n.name != 'smoke'] + [
            ast.Module(body=[n for n in tree.body if not isinstance(n, ast.FunctionDef)], type_ignores=[])]
        for scope in scopes:
            for node in ast.walk(scope):
                names = [a.name for a in node.names] if isinstance(node, ast.Import) else ([node.module or ''] if isinstance(node, ast.ImportFrom) else [])
                for nm in names:
                    # __graft_entry__.build() may compile the oracle's reference copy (oracle.build_ref): building the checker is not using it
                    if nm.split('.')[0] in ('oracle', 'helpers') and not (path.endswith('__graft_entry__.py') and nm.endswith('build_ref')):
                        offenders.append((os.path.relpath(path, root), nm))
    assert offenders == [], offenders


def test_synthetic_document_frequency_matches_oracle_builder():
    from imagecaptioning.pytorch_b200 import synthetic as syn
    from oracle import ciderd_oracle as cdo
    refs = syn.make_refs(40, 120, seed=4)
    assert syn.document_frequency(refs) == cdo.build_document_frequency(refs)


def test_decode_sequence_matches_reference(monkeypatch):
    """utils.decode_sequence against strings produced by the reference's misc.decode_sequence (incl. REMOVE_BAD_ENDINGS and BPE merges)."""
    import json
    from imagecaptioning.pytorch_b200.utils import decode_sequence
    g = json.load(open(os.path.join(GOLD, 'decode_sequence.json')))
    seq = torch.tensor(g['seq'])
    for flag in ('0', '1'):
        monkeypatch.setenv('REMOVE_BAD_ENDINGS', flag)
        assert decode_sequence(g['vocab'], seq) == g['out'][flag]
    monkeypatch.delenv('REMOVE_BAD_ENDINGS')
    assert decode_sequence(g['vocab'], seq.numpy()) == g['out']['0']


def test_decode_option_guards():
    """SURVEY appendix A items 2 and 15 plus the section 8(f) 'later' options: unsupported decode options raise before any device work,
    the reference's own assertions on beam_size / sample_n hold."""
    import imagecaptioning.pytorch_b200 as b200
    cfg = dict(V=30, E=16, H=16, A=8, F_fc=16, F_att=16, T=5)
    model = b200.setup(family_opt('updown', **cfg))
    fc, att = co.make_inputs(2, 3, 16, 16, seed=1)
    for bad in ({'group_size': 2, 'beam_size': 2}, {'output_logsoftmax': 0}, {'sample_method': 'nonsense'}):
        with pytest.raises(NotImplementedError):
            model(fc, att, None, opt=dict({'beam_size': 1}, **bad), mode='sample')
    with pytest.raises(ValueError):
        model(fc, att, None, opt={'beam_size': 1, 'sample_method': 'top0'}, mode='sample')
    with pytest.raises(AssertionError):        # AttModel.py:223: sample_n must be 1 or beam_size when beam searching
        model(fc, att, None, opt={'beam_size': 3, 'sample_n': 2}, mode='sample')
    with pytest.raises(AssertionError):        # AttModel.py:228: beam_size <= vocab_size + 1
        model(fc, att, None, opt={'beam_size': 40, 'sample_n': 1}, mode='sample')
    opt_unk = family_opt('updown', **cfg)
    opt_unk.vocab = dict(opt_unk.vocab)
    opt_unk.vocab[str(cfg['V'])] = 'UNK'
    unk_model = b200.setup(opt_unk)
    with pytest.raises(RuntimeError, match='CUDA'):   # CaptionModel.py:120,161-162: UNK suppression runs on the engine (stops at the no-CPU check)
        unk_model(fc, att, None, opt={'beam_size': 2, 'sample_n': 1, 'suppress_UNK': 1}, mode='sample')
    with pytest.raises(NotImplementedError):           # 15 beams + 2 edit kinds exceed the 16 candidates a row keeps
        unk_model(fc, att, None, opt={'beam_size': 15, 'sample_n': 1, 'suppress_UNK': 1, 'decoding_constraint': 1}, mode='sample')


def test_switch_table_matches_the_sources():
    """Every CAPB200_* environment variable INTEGRATION.md documents is read somewhere in the package or bench.py (no stale documentation),
    and every one the package reads is in INTEGRATION.md's switch table (no hidden switches)."""
    import re
    root = os.path.dirname(os.path.dirname(__file__))
    doc = open(os.path.join(root, 'INTEGRATION.md')).read()
    documented = set(re.findall(r'`(CAPB200_[A-Z0-9_]+)', doc))
    table = doc.split('### Switches', 1)[1].split('\n#', 1)[0]
    in_table = set(re.findall(r'^\| `(CAPB200_[A-Z0-9_]+)', table, re.M))
    blob = open(os.path.join(root, 'bench.py')).read()
    read = set()
    pkg = os.path.join(root, 'imagecaptioning.pytorch_b200')
    for d, _, files in os.walk(pkg):
        if os.path.basename(d) == 'build':
            continue
        for f in files:
            if f.endswith(('.py', '.cu', '.cuh')):
                src = open(os.path.join(d, f)).read()
                blob += src
                read |= set(re.findall(r'getenv\(\s*"(CAPB200_[A-Z0-9_]+)"', src))
                read |= set(re.findall(r'''os\.(?:environ(?:\.get|\.setdefault|\.pop)?|getenv)\s*[\[(]\s*['"](CAPB200_[A-Z0-9_]+)''', src))
    assert 'CAPB200_SCST_GRAPH' in read, sorted(read)        # the patterns still find the reads
    missing = sorted(v for v in documented if v not in blob)
    assert missing == [], missing
    undocumented = sorted(read - in_table)
    assert undocumented == [], undocumented


def test_fused_adam_is_a_torch_adam():
    """FusedAdam keeps torch.optim.Adam's constructor, param groups and state_dict layout (optimizer.pth round-trips, tools/train.py:74-77), and
    refuses CPU tensors instead of falling back."""
    import imagecaptioning.pytorch_b200 as b200
    ps = [torch.nn.Parameter(torch.randn(7, 3)), torch.nn.Parameter(torch.randn(5))]
    ref = torch.optim.Adam([torch.nn.Parameter(p.detach().clone()) for p in ps], lr=5e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01)
    for p in ref.param_groups[0]['params']:
        p.grad = torch.randn_like(p)
    ref.step()
    opt = b200.optim.FusedAdam(ps, lr=5e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01, clip_value=0.1)
    assert isinstance(opt, torch.optim.Adam) and opt.defaults['lr'] == 5e-4 and opt.clip_value == 0.1
    opt.load_state_dict(ref.state_dict())                     # a checkpoint written by the stock optimizer loads
    sd = opt.state_dict()
    assert set(sd['state'][0]) == {'step', 'exp_avg', 'exp_avg_sq'} and float(sd['state'][0]['step']) == 1.0
    ref.load_state_dict(sd)                                   # and the other way round
    for p in ps:
        p.grad = torch.randn_like(p)
    with pytest.raises(RuntimeError, match='CUDA'):
        opt.step()


def test_loss_wrapper_gradient_delivery_paths(monkeypatch):
    """B200LossWrapper's bridge between a fused step and autograd, on a stand-in model (CPU tensors, no engine): the direct path scales the
    flat gradient buffer once and makes param.grad views of it; direct_grads = False (and non-leaf parameters, i.e. DataParallel replicas)
    hand fresh tensors to autograd so that hooks and accumulation work; drop_worst checks the upstream selection."""
    import imagecaptioning.pytorch_b200 as b200

    class Flat:
        def __init__(self, params):
            self.flat = torch.zeros(sum(p.numel() for p in params))
            self.views, off = {}, 0
            for p in params:
                self.views[p] = self.flat[off:off + p.numel()].view(p.shape)
                off += p.numel()

    class Fake(torch.nn.Module):
        family_name = 'fake'

        def __init__(self):
            super().__init__()
            self.a = torch.nn.Parameter(torch.randn(3, 4))
            self.b = torch.nn.Parameter(torch.randn(5))
            self.fg = Flat([self.a, self.b])
            self.calls = 0

        def scst_step(self, fc, att, gts, table, n, temperature=1.0, baseline='greedy', att_masks=None, keep_rows=0):
            self.calls += 1
            g = torch.Generator().manual_seed(self.calls)
            self.fg.flat.copy_(torch.randn(self.fg.flat.shape, generator=g))
            rows = len(gts) * n
            res = {'loss': torch.tensor(0.25 * self.calls), 'reward': torch.ones(rows, 4), 'sample_seq': torch.ones(rows, 4, dtype=torch.long),
                   'grads': dict(self.fg.views), 'flat': self.fg, 'seed': 1, 'row_loss': torch.arange(rows, dtype=torch.float32) if keep_rows else None}
            return res

    monkeypatch.setattr(b200.rewards, 'CiderD_scorer', object())
    opt = argparse.Namespace(sc_sample_method='greedy', sc_beam_size=1, train_sample_method='sample', train_beam_size=1, train_sample_n=2, cider_reward_weight=1,
                             bleu_reward_weight=0, label_smoothing=0.0, drop_worst_rate=0.5)
    model = Fake()
    lw = b200.B200LossWrapper(model, opt)
    fc, att, gts = torch.zeros(2, 4), torch.zeros(2, 3, 4), [np.zeros((1, 4), dtype=np.int64)] * 2
    args = (fc, att, None, None, None, gts, torch.arange(2), True, False)
    # direct path: views of the flat buffer, scaled in place by the upstream gradient
    out = lw(*args, False)
    engine = {p: g.clone() for p, g in lw.last_step['grads'].items()}
    (2.0 * out['loss']).backward()
    for p, g in lw.last_step['grads'].items():
        assert p.grad.data_ptr() == g.data_ptr() and torch.allclose(p.grad, 2.0 * engine[p])
    # the next step's gradients land in the same views (zero_grad(set_to_none=False) keeps them attached)
    model.zero_grad(set_to_none=False)
    out = lw(*args, False)
    engine = {p: g.clone() for p, g in lw.last_step['grads'].items()}
    out['loss'].backward()
    assert all(torch.allclose(p.grad, engine[p]) for p in engine)
    # through autograd: fresh tensors, accumulated over two steps, hooks fire
    model.zero_grad(set_to_none=True)
    lw.direct_grads = False
    fired = []
    h = model.a.register_hook(lambda g_: fired.append(g_.clone()))
    total = {p: torch.zeros_like(p) for p in model.parameters()}
    for k in (1.0, 3.0):
        out = lw(*args, False)
        for p, g in lw.last_step['grads'].items():
            total[p] += k * g
        (k * out['loss']).backward()
    h.remove()
    assert len(fired) == 2 and all(p.grad.data_ptr() != lw.last_step['grads'][p].data_ptr() and torch.allclose(p.grad, total[p]) for p in total)
    # drop_worst: the per-row loss vector goes out, the trainer's top-k mean must be the selection the step assumed
    lw.direct_grads = True
    model.zero_grad(set_to_none=True)
    out = lw(*args, True)
    rows = out['loss']
    assert rows.shape == (4,) and lw.last_step['keep_rows'] == 2
    engine = {p: g.clone() for p, g in lw.last_step['grads'].items()}
    torch.topk(rows, k=2, largest=False)[0].mean().backward()             # tools/train.py:191
    assert all(torch.allclose(p.grad, engine[p]) for p in engine)
    out = lw(*args, True)
    model.zero_grad(set_to_none=True)
    with pytest.raises(NotImplementedError, match='drop_worst'):
        out['loss'].mean().backward()                                        # a different reduction than the step's selection


def test_fused_adam_pointer_table_layout():
    """The device table capb200_adam_step walks: one row of four pointers per tensor, its element count, and one (tensor, chunk) pair per
    capb200_adam_chunk_elems() elements; cached while every address stays the same (the flat gradient buffer guarantees that for the grads)."""
    import imagecaptioning.pytorch_b200 as b200
    chunk = b200._lib.load().capb200_adam_chunk_elems()
    sizes = [2 * chunk + 5, 1, 100, chunk]
    ps = [torch.nn.Parameter(torch.zeros(n)) for n in sizes]
    opt = b200.optim.FusedAdam(ps, lr=1e-3)
    gs = [torch.zeros(n) for n in sizes]
    ms = [torch.zeros(n) for n in sizes]
    vs = [torch.zeros(n) for n in sizes]
    table, numel, chunks, n_chunks = opt._table((0, 'cpu'), ps, gs, ms, vs)
    assert table.shape == (4, 4) and numel.tolist() == sizes and n_chunks == 3 + 1 + 1 + 1
    assert table[:, 0].tolist() == [p.data_ptr() for p in ps] and table[:, 1].tolist() == [g.data_ptr() for g in gs]
    assert chunks.tolist() == [[0, 0], [0, 1], [0, 2], [1, 0], [2, 0], [3, 0]]
    again = opt._table((0, 'cpu'), ps, gs, ms, vs)
    assert again[0] is table                                   # cache hit: nothing is rebuilt or uploaded
    gs[1] = torch.zeros(1)                                     # one gradient moved: the table is rebuilt
    assert opt._table((0, 'cpu'), ps, gs, ms, vs)[0] is not table
