"""ItemKNNCF on the GPU path (csrc/itemknn.cu, daisyrec_b200/model/KNNCFRecommender.py) against the numpy restatement in
oracle/knn_oracle.py and the reference's own runs in tests/golden/itemknn.npz."""
import logging

import numpy as np
import pandas as pd
import pytest
import torch

from oracle import knn_oracle as ko

pytestmark = pytest.mark.gpu

CENTRED = ('adjusted', 'pearson')


def _coo(U, I, nnz, seed, values='binary', dups=0):
    rng = np.random.default_rng(seed)
    u = rng.integers(U, size=nnz)
    i = rng.integers(I, size=nnz)
    if dups:
        k = rng.integers(nnz, size=dups)
        u, i = np.concatenate([u, u[k]]), np.concatenate([i, i[k]])
    n = len(u)
    if values == 'binary':
        v = np.ones(n)
    elif values == 'stars':
        v = rng.integers(1, 6, size=n).astype(np.float64)
    else:
        v = rng.random(n) * 3.0 + 0.01
    return u, i, v


def _X(u, i, v, U, I):
    from daisyrec_b200 import ops
    d = lambda a, t: torch.from_numpy(np.ascontiguousarray(a, t)).cuda()
    return ops.ease_csr(d(u, np.int32), d(i, np.int32), d(v, np.float64), U, I)


def _host_x(X):
    import scipy.sparse as sp
    return sp.csr_matrix((X.val.cpu().numpy(), X.col.cpu().numpy(), X.row_ptr.cpu().numpy()), shape=(X.user_num, X.item_num))


def _gram(X, sim):
    from daisyrec_b200 import ops
    Xt, ss, _ = ops.itemknn_transform(X, sim)
    ws = ops.ease_workspace(Xt)
    return ops.ease_gram(Xt, 0.0, ws), ss, Xt


def _neighbours(X, sim, nrm, sh, maxk, G=None):
    from daisyrec_b200 import ops
    G, ss, Xt = _gram(X, sim) if G is None else G
    W = ops.itemknn_neighbours(G, ss, sim, nrm, sh, maxk)
    return W, Xt.scale


def _same(W, ref, cols=None, bitwise=True):
    idx, val, cnt = (t.cpu().numpy() for t in (W.idx, W.val, W.cnt))
    if cols is not None:
        idx, val, cnt = idx[cols], val[cols], cnt[cols]
    if bitwise:
        assert np.array_equal(cnt, ref.cnt)
        assert np.array_equal(idx, ref.idx)
        assert np.array_equal(val, ref.val)
    else:                                   # mean-centred values: the Gram sums round, weights agree to fp32 accuracy
        a, b = -np.sort(-val, axis=1), -np.sort(-ref.val, axis=1)
        assert np.all(np.abs(a - b) <= 2e-6 * np.abs(b).max() + 1e-6 * np.abs(b))
        assert np.all(np.abs(cnt - ref.cnt) <= 1)


CONFIGS = ([(s, n, sh) for s in ('cosine', 'asymmetric', 'adjusted', 'pearson') for n in (True, False) for sh in (0, 100)]
           + [(s, False, sh) for s in ('jaccard', 'tanimoto', 'dice', 'tversky') for sh in (0, 100)])


# ------------------------------------------------------------------ neighbours
@pytest.mark.parametrize("U,I,values", [(300, 1, "binary"), (1000, 129, "stars"), (2000, 515, "binary"), (900, 200, "real")])
def test_neighbours_every_configuration(U, I, values):
    u, i, v = _coo(U, I, min(U * I // 3, 25 * U), 7, values, 200)
    u[u == U - 2] = U - 1
    if I > 1:
        i[i == I - 1] = 0                                   # a cold item
    X = _X(u, i, v, U, I)
    Xh = _host_x(X)
    grams = {}
    for sim, nrm, sh in CONFIGS:
        tr = (sim in CENTRED and sim) or (sim in ko.BINARY and 'bin') or 'plain'
        key = (tr, sim in ko.BINARY)
        if key not in grams:
            grams[key] = _gram(X, sim)
        for maxk in (1, 40, 600):
            W, scale = _neighbours(X, sim, nrm, sh, maxk, grams[key])
            ref = ko.neighbours(Xh, sim, nrm, sh, maxk)
            exact = values != "real" and sim not in CENTRED
            if sim not in CENTRED:
                assert (scale >= 0) == (exact or sim in ko.BINARY)
            _same(W, ref, bitwise=exact or sim in ko.BINARY)
            assert W.idx.dtype == torch.int32 and W.val.dtype == torch.float32 and W.idx.shape == (I, maxk)


def test_neighbours_large_binary():
    U, I = 70000, 9000
    u, i, v = _coo(U, I, 60 * U, 3)
    X = _X(u, i, v, U, I)
    Xh = _host_x(X)
    cols = np.random.default_rng(0).choice(I, 128, replace=False)
    for sim, nrm, sh in (("cosine", True, 100), ("jaccard", False, 0), ("tversky", False, 100), ("cosine", False, 0)):
        W, scale = _neighbours(X, sim, nrm, sh, 40)
        assert scale == 0
        _same(W, ko.neighbours(Xh, sim, nrm, sh, 40, cols), cols)


def test_ties_follow_value_then_id_and_repeat():
    # 40 groups of 12 identical item columns: every column has 11 equal weights at the top and many equal ones below
    U, I, grp = 400, 480, 12
    rng = np.random.default_rng(2)
    base_u = rng.integers(U, size=3000)
    base_g = rng.integers(I // grp, size=3000)
    u = np.repeat(base_u, grp)
    i = (base_g[:, None] * grp + np.arange(grp)[None, :]).ravel()
    X = _X(u, i, np.ones(len(u)), U, I)
    Xh = _host_x(X)
    for maxk in (5, 11, 30):
        W, _ = _neighbours(X, "cosine", True, 10, maxk)
        ref = ko.neighbours(Xh, "cosine", True, 10, maxk)
        if maxk == 5:                                             # the cut falls inside the run of 11 equal weights
            assert sum((ref.val[c, :ref.cnt[c]] == ref.cut[c]).any() for c in range(I)) > I // 2
        _same(W, ref)
        W2, _ = _neighbours(X, "cosine", True, 10, maxk)
        assert torch.equal(W.idx, W2.idx) and torch.equal(W.val, W2.val) and torch.equal(W.cnt, W2.cnt)


def _config(**kw):
    cfg = dict(gpu='0', topk=50, user_num=600, item_num=700, maxk=40, shrink=100, normalize=True, similarity='cosine',
               logger=logging.getLogger('t'))
    cfg.update(kw)
    return cfg


def test_ml20m_shape():
    from daisyrec_b200.model import ItemKNNCF
    from daisyrec_b200.utils import synthetic
    U, I, nnz = 138493, 26744, 20_000_263
    d = synthetic.make_interactions(U, I, nnz, device="cuda")
    df = pd.DataFrame({'user': d["coo_u"].cpu().numpy().astype(np.int64), 'item': d["coo_i"].cpu().numpy().astype(np.int64),
                       'rating': 1.0})
    del d
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    m = ItemKNNCF(_config(user_num=U, item_num=I))
    m.fit(df)
    assert torch.cuda.max_memory_allocated() - base < 8 * I * I + (2 << 30)
    W1 = m._W
    cols = np.random.default_rng(1).choice(I, 64, replace=False)
    _same(W1, ko.neighbours(_host_x(m._X), "cosine", True, 100, 40, cols), cols)
    m.fit(df)
    assert torch.equal(W1.idx, m._W.idx) and torch.equal(W1.val, m._W.val) and torch.equal(W1.cnt, m._W.cnt)


# ------------------------------------------------------------------ scoring
def _host_w(W):
    return ko.Neighbours(W.idx.cpu().numpy(), W.val.cpu().numpy(), W.cnt.cpu().numpy(), None)


def _check_ranking(ids, s, cands, k):
    """ids against the scores s they were ranked by: the scores of the returned ids are the sorted top scores, and on rows
    whose top k + 1 scores are distinct the ids are the stable order's."""
    top = -np.sort(-s, axis=1)
    pos = np.stack([np.argsort(c)[np.searchsorted(c, w, sorter=np.argsort(c))] for c, w in zip(cands, ids)])
    assert np.array_equal(np.take_along_axis(cands, pos, 1), ids)
    assert np.array_equal(np.take_along_axis(s, pos, 1), top[:, :k])
    assert np.array_equal(ids, np.take_along_axis(cands, ko.topk_order(s, k), 1))   # and the tie order is by position


@pytest.mark.parametrize("values,sim", [("stars", "cosine"), ("binary", "jaccard"), ("real", "pearson")])
def test_rank_full_rank_predict_against_oracle(values, sim):
    from daisyrec_b200 import ops
    U, I = 600, 700
    u, i, v = _coo(U, I, 15 * U, 5, values, 100)
    u[u < 10] = 10                                        # users 0..9 have no rows
    X = _X(u, i, v, U, I)
    W, _ = _neighbours(X, sim, True, 20, 40)
    Xh, Wh = _host_x(X), _host_w(W)
    rng = np.random.default_rng(0)
    users = rng.integers(U, size=300)
    users[:5] = np.arange(5)
    cands = np.stack([rng.choice(I, 120, replace=False) for _ in range(300)])
    ids, sc = ops.itemknn_rank(X, W, torch.from_numpy(users).cuda(), torch.from_numpy(cands).cuda(), 50, scores=True)
    ids, sc = ids.cpu().numpy(), sc.cpu().numpy()
    want = ko.scores(Xh, Wh, users, cands)
    if values == "real":
        assert np.all(np.abs(sc - want) <= 1e-12 * ko.scores(Xh, Wh, users, cands, absolute=True))
    else:
        assert np.array_equal(sc, want)
    _check_ranking(ids, sc, cands, 50)
    assert np.array_equal(ids[:5], cands[:5, :50])        # all-zero rows: the first positions
    fr, fsc = ops.itemknn_full_rank(X, W, torch.from_numpy(users[:40]).cuda(), 50, scores=True)
    fr, fsc = fr.cpu().numpy(), fsc.cpu().numpy()
    fwant = ko.scores(Xh, Wh, users[:40])
    assert np.array_equal(fsc, fwant) if values != "real" else np.allclose(fsc, fwant, rtol=1e-12, atol=1e-14)
    _check_ranking(fr, fsc, np.tile(np.arange(I), (40, 1)), 50)
    assert np.array_equal(fr[:5], np.tile(np.arange(50), (5, 1)))
    pr = ops.itemknn_predict(X, W, torch.from_numpy(users).cuda(), torch.from_numpy(cands[:, 0].copy()).cuda()).cpu().numpy()
    assert np.array_equal(pr, sc[:, 0])


class _Loader:
    def __init__(self, users, cands, bs=128):
        self.users, self.cands, self.bs = users, cands, bs

    def __iter__(self):
        for s in range(0, len(self.users), self.bs):
            yield torch.from_numpy(self.users[s:s + self.bs]), torch.from_numpy(self.cands[s:s + self.bs])


def test_class_surface():
    import scipy.sparse as sp
    from daisyrec_b200.model import ItemKNNCF
    U, I = 600, 700
    u, i, v = _coo(U, I, 9000, 11, "stars", 200)
    df = pd.DataFrame({'user': u, 'item': i, 'rating': v})
    m = ItemKNNCF(_config())
    m.fit(df)
    Xh, ref = ko.fit(u, i, v, U, I, "cosine", True, 100, 40)
    w = m.w_sparse
    assert isinstance(w, sp.csc_matrix) and w.dtype == np.float32 and w.shape == (I, I)
    assert (w != ref.csc(I)).nnz == 0
    rng = np.random.default_rng(1)
    users = rng.integers(U, size=200)
    cands = np.stack([rng.choice(I, 100, replace=False) for _ in range(200)])
    got = m.rank(_Loader(users, cands))
    assert got.dtype == np.int64 and got.shape == (200, 50)
    assert np.array_equal(got, ko.rank(Xh, ref, users, cands, 50)[0])
    fr = m.full_rank(3)
    assert fr.dtype == np.int64 and fr.shape == (50,)
    assert np.array_equal(fr, ko.full_rank(Xh, ref, np.array([3]), 50)[0][0])
    p = m.predict(3, 4)
    assert isinstance(p, np.float64) and p == ko.scores(Xh, ref, np.array([3]), np.array([[4]]))[0, 0]
    # a second fit replaces the first
    m.similarity, m.k = 'jaccard', 7
    m.fit(df)
    assert m._W.maxk == 7 and (m.w_sparse != ko.fit(u, i, v, U, I, "jaccard", True, 100, 7)[1].csc(I)).nnz == 0
    # refusals
    for a, b in ((U, 0), (0, I)):
        with pytest.raises(ValueError, match='unkown'):
            m.predict(a, b)
    with pytest.raises(IndexError):
        m.predict(-1, 0)
    with pytest.raises(IndexError):
        m.full_rank(-1)
    with pytest.raises(IndexError):
        m.rank(_Loader(users, np.where(cands == cands[0, 0], I, cands)))
    for col, bad in (('item', I), ('user', -1)):
        d2 = df.copy()
        d2.loc[0, col] = bad
        with pytest.raises(ValueError):
            ItemKNNCF(_config()).fit(d2)
    with pytest.raises(ValueError, match='not recognized'):
        ItemKNNCF(_config(similarity='euclid')).fit(df)
    with pytest.raises(NotImplementedError):
        ItemKNNCF(_config(maxk=2000)).fit(df)
    with pytest.raises(RuntimeError):
        ItemKNNCF(_config()).full_rank(0)
    free = torch.cuda.mem_get_info()[0]
    n_big = int((free / 8) ** 0.5) + 1000
    with pytest.raises(MemoryError, match='bytes'):
        ItemKNNCF(_config(item_num=n_big)).fit(df)


# ------------------------------------------------------------------ against the reference's runs (tests/golden/itemknn.npz)
def test_synthetic_cases_vs_reference():
    from conftest import golden
    from daisyrec_b200.model import ItemKNNCF
    from test_itemknn_cpu import N_CFG, _cfg, _data, _gold_w, compare_columns, same_ranking
    g = golden("itemknn")
    for d in range(int(g["n_data"])):
        U, I, topk, u, i, v = _data(g, d)
        df = pd.DataFrame({'user': u, 'item': i, 'rating': v})
        users, cands = np.arange(U), g[f"d{d}_cands"].astype(np.int64)
        for k in range(N_CFG):
            sim, nrm, sh, maxk = _cfg(g, k)
            m = ItemKNNCF(_config(user_num=U, item_num=I, topk=topk, similarity=sim, normalize=nrm, shrink=sh, maxk=maxk))
            m.fit(df)
            p = f"d{d}_c{k}"
            exact = d < 2 and sim not in CENTRED
            full = ko.neighbours(ko.interaction_matrix(u, i, v, U, I), sim, nrm, sh, maxk)
            got = _host_w(m._W)
            got.cut = full.cut
            compare_columns(got, _gold_w(g, p, I), exact, p)
            if p + "_rank" in g and exact:
                ids = m.rank(_Loader(users, cands, bs=16))
                s = ko.scores(_host_x(m._X), got, users, cands)
                if (m.w_sparse != _gold_w(g, p, I)).nnz == 0:          # no tie at a cut went the other way
                    assert np.array_equal(s[:24], g[p + "_scores"])
                    same_ranking(ids, s, cands, g[p + "_rank"].astype(np.int64))
                    pred = np.array([m.predict(int(a), int(b)) for a, b in zip(users[:24], cands[:24, 0])])
                    assert np.array_equal(pred, g[p + "_predict"][:24])


def test_ml100k_driver_sequence():
    """test.py's itemknn branch on config 1's ml-100k split through the drop-in classes: ItemKNNCF(config).fit(train_set) ->
    build_candidates_set -> rank -> calc_ranking_results, and full_rank / predict, against the reference's run."""
    import hashlib
    import tempfile
    from daisyrec_b200.model import ItemKNNCF
    from daisyrec_b200.utils.dataset import CandidatesDataset, get_dataloader
    from daisyrec_b200.utils.metrics import calc_ranking_results
    from daisyrec_b200.utils.utils import get_ur, build_candidates_set
    from test_itemknn_cpu import ml100k_inputs, sorted_columns
    g, cu, ci, test_ur = ml100k_inputs()
    U, I, topk, seed, stride, maxk, shrink = (int(v) for v in g["ml_meta"])
    train_set = pd.DataFrame({'user': cu, 'item': ci, 'rating': 1.0})
    cfg = _config(user_num=U, item_num=I, topk=topk, maxk=maxk, shrink=shrink, cand_num=1000, seed=seed)
    np.random.seed(seed); torch.manual_seed(seed)
    train_ur = get_ur(train_set)
    model = ItemKNNCF(cfg)
    model.fit(train_set)
    W = model.w_sparse
    idx, val = sorted_columns(W)
    sha = lambda *a: hashlib.sha256(b"".join(np.ascontiguousarray(x).tobytes() for x in a)).digest()
    assert np.array_equal(W.indptr, g["ml_W_indptr"])
    assert sha(W.indptr.astype(np.int64), val) == g["ml_W_val_sha"].tobytes()
    # 23 columns have equal weights at the cut, which the reference's argpartition breaks its own way: ids are compared on
    # every 64th column outside such ties, and the lists and KPIs below allow for the rows those columns and score ties reach
    from test_itemknn_cpu import compare_columns
    import scipy.sparse as sp
    cols = np.arange(0, I, stride)
    ref = sp.csc_matrix((g["ml_Wc_data"], g["ml_Wc_indices"].astype(np.int32), g["ml_Wc_indptr"]), shape=(I, len(cols)))
    full = ko.neighbours(_host_x(model._X), "cosine", True, shrink, maxk, cols)
    sub = ko.Neighbours(*(t.cpu().numpy()[cols] for t in (model._W.idx, model._W.val, model._W.cnt)), full.cut)
    compare_columns(sub, ref, True, "ml-100k")
    test_u, test_ucands = build_candidates_set(test_ur, train_ur, cfg)
    cands = np.stack([np.asarray(c[1], np.int64) for c in test_ucands])
    assert sha(cands) == g["ml_cands_sha"].tobytes()
    preds = model.rank(get_dataloader(CandidatesDataset(test_ucands), batch_size=128, shuffle=False, num_workers=0))
    assert preds.dtype == np.int64 and preds.shape == g["ml_rank"].shape
    s = ko.scores(_host_x(model._X), _host_w(model._W), np.array(test_u), cands)
    assert np.array_equal(-np.sort(-s, axis=1)[:, :20], g["ml_rank_scores"])
    assert np.array_equal(preds, np.take_along_axis(cands, ko.topk_order(s, topk), 1))
    assert (preds == g["ml_rank"]).all(1).sum() >= 300
    for k, u in enumerate(g["ml_full_u"]):
        f = model.full_rank(int(u))
        assert f.dtype == np.int64 and f.shape == (topk,)
        assert np.array_equal(f, g["ml_full"][k])
    for (a, b), want in zip(g["ml_predict_pairs"], g["ml_predict"]):
        p = model.predict(int(a), int(b))
        assert isinstance(p, np.float64) and p == want
    kcfg = dict(logger=logging.getLogger('t'), res_path=tempfile.mkdtemp() + '/', metrics=["recall", "mrr", "ndcg", "hit", "precision"],
                item_num=I, topk=topk)
    res = calc_ranking_results(test_ur, preds, test_u, kcfg)
    assert [int(c) for c in res.columns[1:]] == g["ml_kpi_ks"].tolist()
    # one user's list differs in its zero-score tail (the reference's argsort is unstable): at most 1 / 304 per KPI
    np.testing.assert_allclose(res.values[:, 1:].astype(np.float64), g["ml_kpi"], rtol=0, atol=1.0 / 304 + 1e-12)
