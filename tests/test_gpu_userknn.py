"""UserKNNCF on the GPU path (csrc/userknn.cu, the panel entry points of csrc/ease.cu / csrc/itemknn.cu,
daisyrec_b200/model/KNNCFRecommender.py) against the numpy restatement in oracle/userknn_oracle.py and the reference's own runs
in tests/golden/userknn.npz."""
import logging

import numpy as np
import pandas as pd
import pytest
import torch

from conftest import golden
from oracle import knn_oracle as ko
from oracle import userknn_oracle as uo
from test_itemknn_cpu import CENTRED, EXACT_DATA, N_CFG, _cfg, _data, _gold_w, compare_columns, same_ranking

pytestmark = pytest.mark.gpu


def _model(U, I, sim='cosine', normalize=True, shrink=0, maxk=10, topk=10, panel=None):
    from daisyrec_b200.model import UserKNNCF
    m = UserKNNCF(dict(user_num=U, item_num=I, maxk=maxk, shrink=shrink, normalize=normalize, similarity=sim, topk=topk,
                       logger=logging.getLogger('t')))
    m._panel = panel
    return m


def _df(u, i, v):
    return pd.DataFrame({'user': np.asarray(u, np.int64), 'item': np.asarray(i, np.int64), 'rating': np.asarray(v, np.float64)})


def _same_w(m, W, U, where):
    """Device lists equal to the oracle's, ids included (both break ties at the cut by lower id)."""
    cnt = m._W.cnt.cpu().numpy()
    assert np.array_equal(cnt, W.cnt), where
    idx, val = m._W.idx.cpu().numpy(), m._W.val.cpu().numpy()
    for c in range(U):
        assert np.array_equal(idx[c, :cnt[c]], W.idx[c, :cnt[c]]), (where, c)
        assert np.array_equal(val[c, :cnt[c]], W.val[c, :cnt[c]]), (where, c)


def _host_w(m, cut=None):
    """The device's forward lists as knn_oracle.Neighbours (``cut``: the oracle's first weight left out per column)."""
    return ko.Neighbours(m._W.idx.cpu().numpy(), m._W.val.cpu().numpy(), m._W.cnt.cpu().numpy(), cut)


class _Loader:
    def __init__(self, users, cands, bs=16):
        self.users, self.cands, self.bs = users, cands, bs

    def __iter__(self):
        for s in range(0, len(self.users), self.bs):
            yield torch.from_numpy(self.users[s:s + self.bs]), torch.from_numpy(self.cands[s:s + self.bs])


@pytest.mark.parametrize("d", [0, 1, 2])
def test_w_sparse_against_fixtures_and_oracle(d):
    """The device's W for every configuration: against the reference's w_sparse (ties at the cut allowed for), and against
    the oracle -- ids and values bitwise on star / binary data for the non-centred similarities, within ItemKNN's tolerance
    for adjusted / pearson and for real values (d2, the fp64 DMMA panel path)."""
    g = golden("userknn")
    U, I, topk, u, i, v = _data(g, d)
    for k in range(N_CFG):
        sim, nrm, sh, maxk = _cfg(g, k)
        m = _model(U, I, sim, nrm, sh, maxk)
        m.fit(_df(u, i, v))
        _, W = uo.fit(u, i, v, U, I, sim, nrm, sh, maxk)
        where = f"d{d} {sim} {nrm} {sh} {maxk}"
        exact = d in EXACT_DATA and sim not in CENTRED
        got = _host_w(m, W.cut)
        compare_columns(got, _gold_w(g, f"d{d}_c{k}", U), exact, where)
        compare_columns(got, W.csc(U), exact, where + " oracle")
        ws = m.w_sparse
        assert ws.shape == (U, U) and ws.dtype == np.float32
        if exact:
            _same_w(m, W, U, where)
            assert (ws != W.csc(U)).nnz == 0, where


@pytest.mark.parametrize("U,I,panel", [(37, 20, 128), (300, 90, 128), (523, 70, 256), (1000, 150, 128)])
@pytest.mark.parametrize("values", ['binary', 'stars', 'real'])
def test_panel_edges_same_w_every_panel(U, I, panel, values):
    rng = np.random.default_rng(U + I)
    nnz = 6 * U
    u, i = rng.integers(0, U - 3, nnz), rng.integers(0, I - 2, nnz)     # cold users and items at the ends
    k = rng.integers(0, nnz, nnz // 10)
    u, i = np.concatenate([u, u[k]]), np.concatenate([i, i[k]])           # duplicate rows
    v = {'binary': np.ones(len(u)), 'stars': rng.integers(1, 6, len(u)).astype(float), 'real': rng.random(len(u)) * 3 + .01}[values]
    ref = None
    for p in (panel, (U + 127) // 128 * 128):
        m = _model(U, I, 'cosine', True, 10, 20, panel=p)
        m.fit(_df(u, i, v))
        got = (m._W.idx.cpu().numpy(), m._W.val.cpu().numpy(), m._W.cnt.cpu().numpy())
        if ref is None:
            ref = got
        else:
            assert all(np.array_equal(a, b) for a, b in zip(got, ref))
    X, W = uo.fit(u, i, v, U, I, 'cosine', True, 10, 20)
    if values != 'real':
        _same_w(m, W, U, (U, I, panel))
    else:
        compare_columns(_host_w(m, W.cut), W.csc(U), False, (U, I, panel))
    users = np.arange(U)
    cands = np.stack([rng.choice(I, 15, replace=False) for _ in users]).astype(np.int64)
    dev = lambda a: torch.from_numpy(a).cuda()
    from daisyrec_b200 import ops
    ids, sc = ops.userknn_rank(m._X, m._R, dev(users), dev(cands), 5, scores=True)
    if values != 'real':
        assert np.array_equal(sc.cpu().numpy(), uo.scores(X, W, users, cands))
    else:   # on the device's own W: the fp64 summation alone
        assert np.allclose(sc.cpu().numpy(), uo.scores(X, _host_w(m), users, cands), rtol=1e-12, atol=1e-14)


def test_maxk_ge_users_and_two_fits_bitwise():
    u, i, v = np.random.default_rng(2).integers(0, 50, 400), np.random.default_rng(3).integers(0, 30, 400), np.ones(400)
    a, b = _model(50, 30, maxk=600), _model(50, 30, maxk=600)
    a.fit(_df(u, i, v)); b.fit(_df(u, i, v))
    for x, y in ((a._W.idx, b._W.idx), (a._W.val, b._W.val), (a._R.r_col, b._R.r_col), (a._R.r_val, b._R.r_val)):
        assert torch.equal(x, y)
    _, W = uo.fit(u, i, v, 50, 30, 'cosine', True, 0, 600)
    _same_w(a, W, 50, 'maxk 600')


def test_ties_at_the_cut_kept_by_lower_id():
    # user 0 shares one item with users 1..8 alike: all eight weights are equal, maxk 3 keeps users 1, 2, 3
    u = np.array([0] + list(range(1, 9)))
    i = np.zeros(9, np.int64)
    m = _model(9, 2, 'cosine', False, 0, 3)
    m.fit(_df(u, i, np.ones(9)))
    assert m._W.idx[0, :3].tolist() == [1, 2, 3] and int(m._W.cnt[0]) == 3


def test_hub_user_reverse_list_has_every_other_user():
    U, I = 700, 40
    rng = np.random.default_rng(9)
    u = np.concatenate([rng.integers(1, U, 2000), np.zeros(I, np.int64)])
    i = np.concatenate([rng.integers(0, I, 2000), np.arange(I)])     # user 0 holds every item: every user's top neighbour
    key = np.unique(u * I + i)                                         # one row per pair: every g_v,0 is v's largest
    u, i = key // I, key % I
    v = np.ones(len(u))
    m = _model(U, I, 'cosine', False, 0, 5, panel=128)
    m.fit(_df(u, i, v))
    rp = m._R.r_ptr.cpu().numpy()
    warm = np.unique(u[u > 0])
    assert rp[1] - rp[0] == len(warm)
    X, W = uo.fit(u, i, v, U, I, 'cosine', False, 0, 5)
    users = np.array([0, 1, 2, 699])
    from daisyrec_b200 import ops
    full, fs = ops.userknn_full_rank(m._X, m._R, torch.from_numpy(users).cuda(), 10, scores=True)
    assert np.array_equal(fs.cpu().numpy(), uo.scores(X, W, users))
    for uu in users:
        assert np.array_equal(m.full_rank(int(uu)), uo.full_rank(X, W, [uu], 10)[0][0])
    assert m.predict(0, 3) == uo.scores(X, W, [0], np.array([[3]]))[0, 0]


def test_fixture_scores_rank_full_rank_predict():
    """rank (the public method, through a loader), full_rank and predict on the synthetic sets: against the oracle on the
    device's own W, and against the reference's runs wherever the device's W is the reference's."""
    from daisyrec_b200 import ops
    g = golden("userknn")
    for d in range(int(g["n_data"])):
        U, I, topk, u, i, v = _data(g, d)
        cands = g[f"d{d}_cands"].astype(np.int64)
        users = np.arange(U)
        for k in range(N_CFG):
            p = f"d{d}_c{k}"
            if p + "_rank" not in g.files:
                continue
            sim, nrm, sh, maxk = _cfg(g, k)
            exact = d in EXACT_DATA and sim not in CENTRED
            m = _model(U, I, sim, nrm, sh, maxk, topk)
            m.fit(_df(u, i, v))
            X, _ = uo.fit(u, i, v, U, I, sim, nrm, sh, maxk)
            Wd = _host_w(m)
            s = uo.scores(X, Wd, users, cands)
            ids = m.rank(_Loader(users, cands))
            assert ids.dtype == np.int64 and ids.shape == (U, topk)
            sc = ops.userknn_scores(m._X, m._R, torch.from_numpy(users).cuda(), torch.from_numpy(cands).cuda()).cpu().numpy()
            fs = uo.scores(X, Wd, users[:6])
            full = np.stack([m.full_rank(a) for a in range(6)])
            assert full.dtype == np.int64 and full.shape == (6, topk)
            pred = np.array([m.predict(int(a), int(b)) for a, b in zip(users, cands[:, 0])])
            if exact:                                             # integer data: fp64 sums exact, every id decided
                assert np.array_equal(sc, s), p
                assert np.array_equal(ids, np.take_along_axis(cands, ko.topk_order(s, topk), 1)), p
                assert np.array_equal(full, ko.topk_order(fs, topk)), p
                assert np.array_equal(pred, s[:, 0]), p
            else:
                assert np.allclose(sc, s, rtol=1e-12, atol=1e-14), p
                assert np.allclose(np.take_along_axis(fs, full, 1), -np.sort(-fs, axis=1)[:, :topk], rtol=1e-12, atol=1e-14), p
                assert np.allclose(pred, s[:, 0], rtol=1e-12, atol=1e-14), p
            ref, gw, ws = g[p + "_scores"], _gold_w(g, p, U), m.w_sparse
            if exact and (ws != gw).nnz == 0:                      # no tie at a cut went the other way
                assert np.array_equal(sc[:24], ref), p
                same_ranking(ids, s, cands, g[p + "_rank"].astype(np.int64))
                assert np.array_equal(pred, g[p + "_predict"]), p
            elif not exact and np.array_equal(ws.indptr, gw.indptr) and np.array_equal(ws.indices, gw.indices):
                # the same neighbours, weights within ItemKNN's tolerance: every entry within it too
                assert np.allclose(sc[:24], ref, rtol=1e-5, atol=1e-6 * np.abs(ref).max()), p
                assert np.allclose(pred, g[p + "_predict"], rtol=1e-5, atol=1e-6 * np.abs(ref).max()), p


def test_class_surface():
    """w_sparse's content, predict's type, a second fit replacing the first, and the refusals."""
    import scipy.sparse as sp
    from daisyrec_b200.model import UserKNNCF
    U, I = 400, 300
    rng = np.random.default_rng(11)
    u, i = rng.integers(0, U, 6000), rng.integers(0, I, 6000)
    v = rng.integers(1, 6, 6000).astype(float)
    df = _df(u, i, v)
    m = _model(U, I, 'cosine', True, 100, 40, 50)
    m.fit(df)
    X, W = uo.fit(u, i, v, U, I, 'cosine', True, 100, 40)
    w = m.w_sparse
    assert isinstance(w, sp.csc_matrix) and w.shape == (U, U) and (w != W.csc(U)).nnz == 0
    p = m.predict(3, 4)
    assert isinstance(p, np.float64) and p == uo.scores(X, W, [3], np.array([[4]]))[0, 0]
    m.similarity, m.k = 'jaccard', 7
    m.fit(df)
    assert m._W.maxk == 7 and (m.w_sparse != uo.fit(u, i, v, U, I, 'jaccard', True, 100, 7)[1].csc(U)).nnz == 0
    for a, b in ((U, 0), (0, I)):
        with pytest.raises(ValueError, match='unkown'):
            m.predict(a, b)
    with pytest.raises(IndexError):
        m.full_rank(-1)
    with pytest.raises(IndexError):
        m.rank(_Loader(np.arange(4), np.full((4, 5), I, np.int64)))
    with pytest.raises(ValueError, match='not recognized'):
        _model(U, I, 'euclid').fit(df)
    with pytest.raises(NotImplementedError):
        _model(U, I, maxk=2000).fit(df)
    with pytest.raises(RuntimeError):
        _model(U, I).full_rank(0)
    free = torch.cuda.mem_get_info()[0]
    with pytest.raises(MemoryError, match='bytes'):
        UserKNNCF(dict(user_num=U, item_num=int(free // U) + 1000, maxk=10, shrink=0, normalize=True, similarity='cosine',
                       topk=10, logger=logging.getLogger('t'))).fit(df)


def test_ml100k_driver_sequence():
    """test.py's itemknn-style sequence for UserKNNCF on config 1's ml-100k split through the drop-in classes:
    UserKNNCF(config).fit(train_set) -> build_candidates_set -> rank -> calc_ranking_results, and full_rank / predict,
    against the reference's run.  30 columns have equal weights at the maxk cut, which the reference breaks its own way; the
    users whose weight equals such a cut are the only ones whose reverse lists may differ from the reference's, so scores,
    lists and predictions are compared bitwise on every other test user, and the KPIs allow for the rows whose ids differ."""
    import hashlib
    import tempfile
    import scipy.sparse as sp
    from daisyrec_b200.model import UserKNNCF
    from daisyrec_b200.utils.dataset import CandidatesDataset, get_dataloader
    from daisyrec_b200.utils.metrics import calc_ranking_results
    from daisyrec_b200.utils.utils import build_candidates_set, get_ur
    from test_itemknn_cpu import ml100k_inputs, sorted_columns
    _, cu, ci, test_ur = ml100k_inputs()
    g = golden("userknn")
    U, I, topk, seed, stride, maxk, shrink = (int(x) for x in g["ml_meta"])
    train_set = pd.DataFrame({'user': cu, 'item': ci, 'rating': 1.0})
    cfg = dict(gpu='0', user_num=U, item_num=I, topk=topk, maxk=maxk, shrink=shrink, normalize=True, similarity='cosine',
               cand_num=1000, seed=seed, logger=logging.getLogger('t'))
    np.random.seed(seed); torch.manual_seed(seed)
    train_ur = get_ur(train_set)
    model = UserKNNCF(cfg)
    model.fit(train_set)
    W = model.w_sparse
    _, val = sorted_columns(W)
    sha = lambda *a: hashlib.sha256(b"".join(np.ascontiguousarray(x).tobytes() for x in a)).digest()
    assert W.shape == (U, U)
    assert np.array_equal(W.indptr, g["ml_W_indptr"])
    assert sha(W.indptr.astype(np.int64), val) == g["ml_W_val_sha"].tobytes()
    X, full = uo.fit(cu, ci, np.ones(len(cu)), U, I, 'cosine', True, shrink, maxk)
    _same_w(model, full, U, "ml-100k")
    cols = np.arange(0, U, stride)
    ref = sp.csc_matrix((g["ml_Wc_data"], g["ml_Wc_indices"].astype(np.int32), g["ml_Wc_indptr"]), shape=(U, len(cols)))
    sub = ko.Neighbours(*(t.cpu().numpy()[cols] for t in (model._W.idx, model._W.val, model._W.cnt)), full.cut[cols])
    compare_columns(sub, ref, True, "ml-100k")
    Xt = X.T.tocsr()
    Xt.sort_indices()
    T = ko.transform(Xt, 'cosine')
    w = ko.column_weights(ko.gram_columns(T), ko.sum_of_squared(T, 'cosine'), np.arange(U), 'cosine', True, shrink)
    tied = np.zeros(U, bool)
    for c in range(U):
        if not np.isnan(full.cut[c]) and full.cut[c] != 0 and (full.val[c, :full.cnt[c]] == full.cut[c]).any():
            tied[w[:, c] == full.cut[c]] = True
    test_u, test_ucands = build_candidates_set(test_ur, train_ur, cfg)
    cands = np.stack([np.asarray(c[1], np.int64) for c in test_ucands])
    assert sha(cands) == g["ml_cands_sha"].tobytes()
    preds = model.rank(get_dataloader(CandidatesDataset(test_ucands), batch_size=128, shuffle=False, num_workers=0))
    assert preds.dtype == np.int64 and preds.shape == g["ml_rank"].shape
    tu = np.array(test_u)
    s = uo.scores(X, full, tu, cands)
    assert np.array_equal(preds, np.take_along_axis(cands, ko.topk_order(s, topk), 1))
    clear = ~tied[tu]
    assert clear.sum() >= 290
    assert np.array_equal(-np.sort(-s[clear], axis=1)[:, :20], g["ml_rank_scores"][clear])
    same_ranking(preds[clear], s[clear], cands[clear], g["ml_rank"].astype(np.int64)[clear])
    for k, a in enumerate(g["ml_full_u"]):
        f = model.full_rank(int(a))
        assert f.dtype == np.int64 and f.shape == (topk,)
        fs = uo.scores(X, full, [a])
        assert np.array_equal(f, ko.topk_order(fs, topk)[0])
        if not tied[a]:
            assert np.array_equal(fs[0, f], fs[0, g["ml_full"][k].astype(np.int64)])
    for (a, b), want in zip(g["ml_predict_pairs"], g["ml_predict"]):
        p = model.predict(int(a), int(b))
        assert isinstance(p, np.float64) and p == uo.scores(X, full, [a], np.array([[b]]))[0, 0]
        if not tied[a]:
            assert p == want
    kcfg = dict(logger=logging.getLogger('t'), res_path=tempfile.mkdtemp() + '/', metrics=["recall", "mrr", "ndcg", "hit", "precision"],
                item_num=I, topk=topk)
    res = calc_ranking_results(test_ur, preds, test_u, kcfg)
    assert [int(c) for c in res.columns[1:]] == g["ml_kpi_ks"].tolist()
    # each test user moves each KPI by at most 1 / n_test_users, and only the rows whose ids differ from the reference's can
    differ = int((preds != g["ml_rank"]).any(1).sum())
    assert differ <= 40
    np.testing.assert_allclose(res.values[:, 1:].astype(np.float64), g["ml_kpi"], rtol=0, atol=differ / len(tu) + 1e-12)


@pytest.mark.parametrize("sim", ['cosine', 'pearson'])
def test_ml20m_shape_sampled_columns(sim):
    """ML-20M's shape (138 493 users, 26 744 items, 20M rows; binary for cosine, which takes the s8 path, and stars for pearson,
    whose centred values take the fp64 path): peak memory under the stated bound, and 64 sampled user columns against the
    oracle."""
    U, I, nnz = 138493, 26744, 20_000_263
    rng = np.random.default_rng(20)
    u = rng.integers(0, U, nnz)
    i = np.minimum(rng.zipf(1.3, nnz) - 1, I - 1)
    v = np.ones(nnz) if sim == 'cosine' else rng.integers(1, 6, nnz).astype(np.float64)
    m = _model(U, I, sim, True, 100, 100)
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    m.fit(_df(u, i, v))
    from daisyrec_b200 import ops
    lib = ops.L.lib()
    peak = torch.cuda.max_memory_allocated() - base
    bound = (m._need_resident(nnz) + m._need_rest(100, lib.drb_gram_image_bytes(I, U, 0 if sim == 'cosine' else -1))
             + ops.USERKNN_PANEL_BYTES)
    assert peak <= bound, (peak, bound)
    cols = rng.choice(U, 64, replace=False)
    _, W = uo.fit(u, i, v, U, I, sim, True, 100, 100, cols=cols)
    idx, val, cnt = m._W.idx.cpu().numpy(), m._W.val.cpu().numpy(), m._W.cnt.cpu().numpy()
    for c, col in enumerate(cols):
        assert cnt[col] == W.cnt[c], col
        if sim == 'cosine':
            assert np.array_equal(idx[col, :cnt[col]], W.idx[c, :W.cnt[c]]), col
            assert np.array_equal(val[col, :cnt[col]], W.val[c, :W.cnt[c]]), col
        else:
            assert np.allclose(np.sort(val[col, :cnt[col]]), np.sort(W.val[c, :W.cnt[c]]), rtol=1e-5, atol=1e-7), col
