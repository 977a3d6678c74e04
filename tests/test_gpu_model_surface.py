"""The shared surface of the seven model classes: every entry point that takes caller ids raises nn.Embedding's IndexError on
an out-of-range user, item or negative id before any launch (the kernels index raw tables) and leaves the parameters
untouched; state round-trips through to() / load_state_dict; empty test loaders and Item2Vec's empty batches keep their
results."""
import contextlib
import logging

import numpy as np
import pytest
import scipy.sparse as sp
import torch

pytestmark = pytest.mark.gpu

U, I, F = 50, 60, 8
CLASSES = ('MF', 'FM', 'LightGCN', 'NGCF', 'NFM', 'NeuMF', 'Item2Vec')


def _model(name):
    from daisyrec_b200 import model
    rng = np.random.default_rng(0)
    r, c = rng.integers(0, U, 300), rng.integers(0, I, 300)
    ur = {}
    for a, b in zip(r.tolist(), c.tolist()):
        ur.setdefault(a, set()).add(b)
    cfg = dict(gpu='0', logger=logging.getLogger('surface'), progress=False, lr=0.01, reg_1=0.001, reg_2=0.001, epochs=1,
               topk=5, user_num=U, item_num=I, factors=F, loss_type='BPR', optimizer='default', init_method='default',
               early_stop=False, inter_matrix=sp.coo_matrix((np.ones(300, np.float32), (r, c)), shape=(U, I)), num_layers=2,
               node_dropout=0.0, mess_dropout=0.1, hidden_size_list=[8, 8], act_function='relu', batch_norm=True,
               dropout=0.5, model_name='NeuMF', train_ur=ur)
    torch.manual_seed(0)
    return getattr(model, name)(cfg)


def _snapshot(m):
    return {k: v.detach().clone() for k, v in m.state_dict().items()}


def _same(m, snap):
    sd = m.state_dict()
    return sd.keys() == snap.keys() and all(torch.equal(sd[k], snap[k]) for k in snap)


def _batch(name, col, bad, device='cpu'):
    """A valid (user, pos, neg) -- for Item2Vec (target, context, label) -- batch of 8 with `bad` written into column col."""
    g = torch.Generator().manual_seed(1)
    first = I if name == 'Item2Vec' else U
    cols = [torch.randint(0, first, (8,), generator=g), torch.randint(0, I, (8,), generator=g),
            torch.randint(0, 2 if name == 'Item2Vec' else I, (8,), generator=g)]
    cols[col][3] = bad
    return [c.to(device) for c in cols]


def _bad_calls(name, m):
    """(label, callable) for every id-taking entry point, each with one out-of-range id."""
    calls = []
    cols = (0, 1) if name == 'Item2Vec' else (0, 1, 2)                       # Item2Vec's third column is a 0/1 label
    for col in cols:
        top = I if (col > 0 or name == 'Item2Vec') else U
        for bad, dev in ((top, 'cpu'), (-1, 'cpu'), (top + 7, 'cuda')):
            b = _batch(name, col, bad, dev)
            calls += [(f'calc_loss col{col} {bad} {dev}', lambda b=b: m.calc_loss(b)),
                      (f'train_step col{col} {bad} {dev}', lambda b=b: m.train_step(b)),
                      (f'fit col{col} {bad} {dev}', lambda b=b: m.fit([tuple(b)]))]
    if name not in ('LightGCN', 'NGCF'):                                    # their forward() takes no ids
        calls += [('forward user', lambda: m.forward([1, U], [2, 3])),
                  ('forward item', lambda: m.forward(torch.tensor([1, 2], device='cuda'), torch.tensor([3, -2], device='cuda')))]
    calls += [('predict user', lambda: m.predict(U, 1)), ('predict item', lambda: m.predict(1, I)),
              ('rank user', lambda: m.rank([(torch.tensor([1, U]), torch.tensor([[1, 2], [3, 4]]))])),
              ('rank candidate', lambda: m.rank([(torch.tensor([1, 2]), torch.tensor([[1, 2], [3, I]]))])),
              ('rank negative candidate', lambda: m.rank([(torch.tensor([1]), torch.tensor([[-1, 2]]))])),
              ('full_rank', lambda: m.full_rank(U)), ('full_rank negative', lambda: m.full_rank(-1))]
    return calls


@pytest.mark.parametrize('name', CLASSES)
def test_out_of_range_ids_raise_before_any_launch(name):
    m = _model(name)
    m.fit([tuple(_batch(name, 0, 0))])                                      # optimiser state and caches exist
    for label, call in _bad_calls(name, m):
        snap = _snapshot(m)
        with pytest.raises(IndexError, match='index out of range in self'):
            call()
        torch.cuda.synchronize()
        assert _same(m, snap), label


@pytest.mark.parametrize('name', CLASSES)
def test_state_round_trip(name):
    m = _model(name)
    assert m.to('cuda') is m
    m.fit([tuple(_batch(name, 0, 0))])
    sd = {k: v.detach().cpu().numpy().copy() for k, v in m.state_dict().items()}
    params = m.parameters()
    assert len(params) <= len(sd) and all(any(p is t for t in m.state_dict().values()) for p in params)
    other = _model(name)
    other.load_state_dict(sd)                                               # host arrays are copied in, reshaped
    assert all(np.array_equal(v.detach().cpu().numpy(), sd[k]) for k, v in other.state_dict().items())
    users, cands = torch.tensor([0, 7]), torch.tensor([[1, 2, 3, 4, 5, 6], [9, 8, 7, 6, 5, 4]])
    m.eval(), other.eval()
    if name == 'NGCF':                                                      # message dropout: same masks for both
        torch.manual_seed(3); a = m.rank([(users, cands)])
        torch.manual_seed(3); b = other.rank([(users, cands)])
    else:
        a, b = m.rank([(users, cands)]), other.rank([(users, cands)])
    assert np.array_equal(a, b)
    with pytest.raises(KeyError) if name != 'NFM' else contextlib.nullcontext():     # NFM's keys are optional
        other.load_state_dict({})


@pytest.mark.parametrize('name', CLASSES)
def test_empty_inputs_keep_their_results(name):
    from daisyrec_b200.utils.dataset import CandidatesDataset, get_dataloader
    m = _model(name)
    for loader in ([], get_dataloader(CandidatesDataset([]), 4, False)):
        out = m.rank(loader)
        assert out.dtype == np.float32 and out.shape == (0,)
    if name == 'Item2Vec':                                                  # an empty skip-gram batch launches nothing
        snap = _snapshot(m)
        assert float(m.calc_loss([[], [], []])) == 0.0 and m.train_step([[], [], []]) == 0.0
        assert m._opt_steps == 0 and _same(m, snap)
