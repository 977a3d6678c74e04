"""Multi-VAE host side and oracle against the reference's own runs (tests/golden/vae.npz), without a GPU."""
import logging

import numpy as np
import pandas as pd
import pytest
import torch

from conftest import golden
from oracle import vae_oracle as vo


def _case(c):
    g = golden("vae")
    p = f's{c}_'
    U, I, lat, ep, bs, uv, tot = (int(x) for x in g[p + 'meta'])
    dr, lr, cap = (float(x) for x in g[p + 'fl'])
    df = pd.DataFrame({'user': g[p + 'df'][0], 'item': g[p + 'df'][1], 'rating': g[p + 'rating']})
    return g, p, df, dict(U=U, I=I, lat=lat, epochs=ep, bs=bs, use_value=bool(uv), total=tot, dropout=dr, lr=lr, cap=cap,
                          hidden=[int(h) for h in g[p + 'hidden']], opt=str(g[p + 'opt'][0]))


@pytest.mark.parametrize("case", ["a", "b"])
def test_oracle_fit_matches_reference(case):
    g, p, df, c = _case(case)
    keys = list(g[p + 'keys'])
    torch.manual_seed(2019)
    np.random.seed(2019)
    init = vo.init_state(c['I'], c['hidden'], c['lat'])
    for j, k in enumerate(keys):
        assert np.array_equal(init[k], g[p + f'init{j}']), k
    m = vo.Vae(init, c['hidden'], c['lat'], c['I'], c['opt'], c['lr'], c['dropout'], c['cap'], c['total'])
    X = vo.input_rows(g[p + 'hist_id'], g[p + 'hist_val'], c['I'])
    losses = vo.fit(m, X, df['user'].unique(), c['bs'], c['epochs'])
    ref = g[p + 'losses']
    assert np.max(np.abs(losses - ref) / np.abs(ref)) <= 1e-5
    st = m.state()
    for j, k in enumerate(keys):
        assert np.abs(st[k] - g[p + f'final{j}']).max() <= 1e-4, k
    # the host draws leave the global RNG where the reference's fit leaves it
    assert np.array_equal(torch.get_rng_state().numpy(), g[p + 'rng_after'])
    assert np.abs(m.scores(torch.from_numpy(X)) - g[p + 'logits']).max() <= 1e-4


@pytest.mark.parametrize("case", ["a", "b"])
def test_history_matrix_and_input_rule(case):
    from daisyrec_b200.utils.utils import get_history_matrix
    g, p, df, c = _case(case)
    cfg = dict(logger=logging.getLogger('t'), UID_NAME='user', IID_NAME='item', INTER_NAME='rating', user_num=c['U'],
               item_num=c['I'])
    hid, hval, hlen = get_history_matrix(df, cfg, row='user', use_config_value_name=c['use_value'])
    assert hid.dtype == torch.int64 and hval.dtype == torch.float32 and hlen.dtype == torch.int64
    assert np.array_equal(hid.numpy(), g[p + 'hist_id']) and np.array_equal(hval.numpy(), g[p + 'hist_val'])
    assert np.array_equal(hlen.numpy(), np.bincount(df['user'], minlength=c['U']))
    # the last-write rule equals index_put_ on the CPU, the reference's get_user_rating_matrix
    X = vo.input_rows(hid, hval, c['I'])
    R = torch.zeros(c['U'], c['I'])
    rows = torch.arange(c['U']).repeat_interleave(hid.shape[1])
    R.index_put_((rows, hid.flatten()), hval.flatten())
    assert np.array_equal(X, R.numpy().astype(np.float64))
    if case == 'a':
        lens = hlen.numpy()
        full = int(np.argmax(lens))
        short = [u for u in range(c['U']) if 0 in hid[u, :lens[u]].tolist() and lens[u] < hid.shape[1]]
        assert X[full, 0] != 0 and short and all(X[u, 0] == 0 for u in short)


def test_host_draws_are_the_reference_stream():
    """VAECF._host_draws consumes the global generator exactly as the reference's forward() does, and packs the mask."""
    from types import SimpleNamespace
    from daisyrec_b200.model.VAECFRecommender import VAECF
    shim = SimpleNamespace(item_num=37, lat_dim=9, dropout=0.5, device='cpu')
    torch.manual_seed(5)
    bits, eps = VAECF._host_draws(shim, 6, 2)
    after = torch.get_rng_state()
    torch.manual_seed(5)
    for s in range(2):
        keep, e = vo.host_draws(6, 37, 4, 0.5)
        flat = keep.numpy().reshape(-1).astype(bool)
        w = bits.numpy().reshape(2, -1)[s].view(np.uint32)
        got = (w[np.arange(flat.size) >> 5] >> (np.arange(flat.size) & 31)) & 1
        assert np.array_equal(got.astype(bool), flat)
        assert torch.equal(eps[s], e)
    assert torch.equal(torch.get_rng_state(), after)
    shim.dropout = 0.0
    torch.manual_seed(5)
    bits, eps = VAECF._host_draws(shim, 6, 1)
    torch.manual_seed(5)
    assert bits is None and torch.equal(eps[0], torch.randn(6, 4))


def test_loader_plan_decodes_both_aedatasets():
    from torch.utils.data import DataLoader
    from daisyrec_b200.model.AbstractRecommender import loader_plan
    from daisyrec_b200.model.VAECFRecommender import _int_rows
    from daisyrec_b200.utils.dataset import AEDataset, get_dataloader
    from oracle import ref_harness as rh
    g, p, df, c = _case('a')
    ours = get_dataloader(AEDataset(df, yield_col='user'), batch_size=16, shuffle=True)
    plan = loader_plan(ours, _int_rows)
    assert plan is not None and np.array_equal(plan[0], df['user'].unique()) and plan[1:4] == (16, True, False)
    assert ours.num_workers == 0
    assert loader_plan(ours) is None                                  # not a triple table
    if rh.available():
        rh.import_reference()
        from daisy.utils.dataset import AEDataset as RefAE
        ref = DataLoader(RefAE(df, yield_col='user'), batch_size=8, shuffle=False)
        plan = loader_plan(ref, _int_rows)
        assert plan is not None and np.array_equal(plan[0], df['user'].unique()) and plan[1:3] == (8, False)
