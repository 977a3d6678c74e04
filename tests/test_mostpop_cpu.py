"""The restatement of MostPop (oracle/userknn_oracle.mostpop) against tests/golden/mostpop.npz, the reference's own runs
(oracle/gen_mostpop.py): item_cnt_ref and item_score bitwise, and the reference's rankings equal to a tie-aware
(score descending) order of its own scores."""
import numpy as np

from conftest import golden
from oracle import userknn_oracle as uo


def test_item_score_bitwise():
    g = golden("mostpop")
    U, I, _ = (int(x) for x in g["s_meta"])
    cnt, score = uo.mostpop(g["s_i"], I)
    assert np.array_equal(cnt, g["s_cnt"]) and np.array_equal(score, g["s_score"])
    gs = golden("ml100k_sampler")
    cnt, score = uo.mostpop(gs["coo_i"], int(g["ml_meta"][1]))
    assert np.array_equal(cnt, g["ml_cnt"]) and np.array_equal(score, g["ml_score"])


def test_reference_rank_is_a_score_order():
    g = golden("mostpop")
    for sc, cands, rank in ((g["s_score"], g["s_cands"], g["s_rank"]), (g["ml_score"], g["ml_cands"].astype(np.int64), g["ml_rank"])):
        assert rank.dtype == np.float32
        k = rank.shape[1]
        ours = np.take_along_axis(cands, np.argsort(-sc[cands], axis=1, kind="stable")[:, :k], 1)
        assert np.array_equal(sc[ours], sc[rank.astype(np.int64)])
    full = g["ml_full"]
    assert np.array_equal(g["ml_score"][full], -np.sort(-g["ml_score"])[:len(full)])
