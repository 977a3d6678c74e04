"""MostPop on the GPU path (csrc/mostpop.cu, daisyrec_b200/model/PopRecommender.py) against oracle/userknn_oracle.mostpop and
the reference's own runs in tests/golden/mostpop.npz."""
import logging

import numpy as np
import pandas as pd
import pytest
import torch

from conftest import golden
from oracle import userknn_oracle as uo

pytestmark = pytest.mark.gpu


def _model(I, topk=10, col='item'):
    from daisyrec_b200.model import MostPop
    return MostPop(dict(item_num=I, topk=topk, IID_NAME=col, logger=logging.getLogger('t')))


class _Loader:
    def __init__(self, users, cands, bs=128):
        self.users, self.cands, self.bs = users, cands, bs

    def __iter__(self):
        for s in range(0, len(self.users), self.bs):
            yield torch.from_numpy(self.users[s:s + self.bs]), torch.from_numpy(self.cands[s:s + self.bs])


def _tie_aware(score, cands, ours, ref):
    """Equal score sequences; ids outside the last tie group at the cut equal as a set per score level; the ids in that group
    drawn from the reference's candidates of that score."""
    for r in range(len(ours)):
        so, sr = score[ours[r]], score[ref[r]]
        assert np.array_equal(so, sr), r
        last = so[-1]
        for lv in np.unique(so[so != last]):
            assert set(ours[r][so == lv]) == set(ref[r][sr == lv]), r
        pool = set(cands[r][score[cands[r]] == last])
        assert set(ours[r][so == last]) <= pool, r


def test_fit_bitwise_and_rank_against_fixtures():
    g = golden("mostpop")
    U, I, topk = (int(x) for x in g["s_meta"])
    m = _model(I, topk)
    m.fit(pd.DataFrame({'user': g["s_u"].astype(np.int64), 'item': g["s_i"].astype(np.int64)}))
    assert np.array_equal(m.item_cnt_ref, g["s_cnt"]) and np.array_equal(m.item_score, g["s_score"])
    cnt, score = uo.mostpop(g["s_i"], I)
    assert np.array_equal(m.item_score, score)
    cands = g["s_cands"].astype(np.int64)
    got = m.rank(_Loader(np.arange(U), cands, 16))
    assert got.dtype == np.float32 and got.shape == g["s_rank"].shape
    _tie_aware(score, cands, got.astype(np.int64), g["s_rank"].astype(np.int64))
    # this path's rule: (score desc, position asc) / (score desc, id asc)
    ref = np.take_along_axis(cands, np.argsort(-score[cands], axis=1, kind='stable')[:, :topk], 1)
    assert np.array_equal(got.astype(np.int64), ref)
    full = m.full_rank(3)
    assert full.dtype == np.int64 and np.array_equal(full, np.argsort(-score, kind='stable')[:topk])
    assert m.predict(0, 5) == score[5]


def test_ml100k_mostpop_branch():
    g = golden("mostpop")
    gs = golden("ml100k_sampler")
    U, I, topk, _ = (int(x) for x in g["ml_meta"])
    m = _model(I, topk)
    m.fit(pd.DataFrame({'user': gs["coo_u"], 'item': gs["coo_i"]}))
    assert np.array_equal(m.item_score, g["ml_score"]) and np.array_equal(m.item_cnt_ref, g["ml_cnt"])
    cands = g["ml_cands"].astype(np.int64)
    got = m.rank(_Loader(g["ml_test_u"].astype(np.int64), cands))
    _tie_aware(m.item_score, cands, got.astype(np.int64), g["ml_rank"].astype(np.int64))
    full = m.full_rank(0)
    _tie_aware(m.item_score, np.arange(I)[None], full[None], g["ml_full"][None])
    assert np.array_equal([m.predict(0, i) for i in range(0, I, 97)], g["ml_predict"])
    # test.py's KPI table: rows whose ids differ from the reference's (only inside its tie groups) move each KPI by at most
    # 1 / n_test_users
    import tempfile
    from daisyrec_b200.utils.metrics import calc_ranking_results
    from test_itemknn_cpu import ml100k_inputs
    _, _, _, test_ur = ml100k_inputs()
    test_u = g["ml_test_u"].tolist()
    assert sorted(test_ur) == sorted(test_u)
    kcfg = dict(logger=logging.getLogger('t'), res_path=tempfile.mkdtemp() + '/', metrics=["recall", "mrr", "ndcg", "hit", "precision"],
                item_num=I, topk=topk)
    res = calc_ranking_results(test_ur, got.astype(np.int64), test_u, kcfg)
    assert [int(c) for c in res.columns[1:]] == g["ml_kpi_ks"].tolist()
    differ = int((got != g["ml_rank"]).any(1).sum())
    np.testing.assert_allclose(res.values[:, 1:].astype(np.float64), g["ml_kpi"], rtol=0, atol=differ / len(test_u) + 1e-12)


def test_ids_out_of_range_and_edges():
    m = _model(10, 20, col='iid')
    with pytest.raises(IndexError):
        m.fit(pd.DataFrame({'iid': np.array([1, 2, 10])}))
    with pytest.raises(IndexError):
        m.fit(pd.DataFrame({'iid': np.array([1, -1])}))
    m.fit(pd.DataFrame({'iid': np.array([3, 3, 3, 1, 1, 7])}))             # duplicates counted, topk > I
    assert m.item_cnt_ref.tolist() == [0, 2, 0, 3, 0, 0, 0, 1, 0, 0]
    assert m.full_rank(0).tolist()[:4] == [3, 1, 7, 0] and len(m.full_rank(0)) == 10
    assert m.rank(_Loader(np.zeros(0, np.int64), np.zeros((0, 4), np.int64))).shape == (0,)
    rng = np.random.default_rng(1)
    big = rng.integers(0, 26744, 20_000_263)
    m = _model(26744, 50)
    m.fit(pd.DataFrame({'item': big}))
    assert np.array_equal(m.item_score, uo.mostpop(big, 26744)[1])
