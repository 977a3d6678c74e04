"""Generates tests/golden/item2vec.npz from the reference's own Item2Vec and SkipGramNegativeSampler
(daisy/model/Item2VecRecommender.py, daisy/utils/sampler.py:105-160), imported through oracle/ref_harness.py.

The reference sampler calls ``Series.iteritems`` (sampler.py:136), which pandas >= 2 no longer has; this generator adds
``Series.iteritems = Series.items`` in process before sampling.  It affects no other fixture.

    python oracle/gen_item2vec.py
"""
import copy
import hashlib
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_harness as rh  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
EDGE = 1024   # first / last rows of the ml-100k sampler output kept verbatim
STRIDE = 8    # the step tables and the user table are kept for every STRIDE-th row (the fixture stays small)


def _shim():
    import pandas as pd
    if not hasattr(pd.Series, "iteritems"):
        pd.Series.iteritems = pd.Series.items


def _np_state():
    s = np.random.get_state()
    return np.concatenate([s[1].astype(np.int64), [int(s[2])]])


# (users, items) of the synthetic cases.  Case 0: user 1 has one row, user 0 repeats item 3 inside the window, user 3 has
# train rows but no sequence (absent from df).  Case 1: larger, window 3, discard=True.  Case 2: a near-full user.
def _cases():
    rng = np.random.default_rng(11)
    c0 = ([0, 0, 1, 0, 2, 0, 2, 2, 4, 4, 0, 4], [3, 5, 7, 3, 1, 9, 2, 1, 0, 11, 6, 4])
    u1 = rng.integers(0, 40, 900)
    i1 = np.minimum(rng.zipf(1.4, 900) - 1, 59)
    u2 = np.concatenate([np.full(15, 2), rng.choice([0, 1, 3, 4, 5], 40)])    # user 2: all items but one
    i2 = np.concatenate([np.arange(15), rng.integers(0, 16, 40)])
    return [
        dict(U=6, I=12, users=np.array(c0[0]), items=np.array(c0[1]), window=2, discard=False, seed=2022,
             extra_ur={3: {2, 8}}),
        dict(U=40, I=60, users=u1, items=i1, window=3, discard=True, seed=7, extra_ur={}),
        dict(U=6, I=16, users=u2, items=i2, window=2, discard=False, seed=99, extra_ur={}),
    ]


def gen_synthetic(out):
    import pandas as pd
    from daisy.utils.sampler import SkipGramNegativeSampler
    from daisy.utils.utils import get_ur
    for k, c in enumerate(_cases()):
        df = pd.DataFrame({"user": c["users"].astype(np.int64), "item": c["items"].astype(np.int64), "rating": 1.0,
                           "timestamp": np.arange(len(c["users"]))})
        ur = get_ur(df)
        ur.update(c["extra_ur"])
        cfg = rh.make_config("item2vec", user_num=c["U"], item_num=c["I"], train_ur=ur, context_window=c["window"])
        np.random.seed(c["seed"])
        rows = SkipGramNegativeSampler(df, cfg, discard=c["discard"]).sampling()
        out[f"s{k}_users"] = c["users"].astype(np.int32)
        out[f"s{k}_items"] = c["items"].astype(np.int32)
        out[f"s{k}_extra_ur"] = np.array([[u, i] for u, s in c["extra_ur"].items() for i in sorted(s)], np.int32).reshape(-1, 2)
        out[f"s{k}_meta"] = np.array([c["U"], c["I"], c["window"], int(c["discard"]), c["seed"]], np.int64)
        out[f"s{k}_rows"] = rows.astype(np.int32)
        out[f"s{k}_state"] = _np_state()
    out["n_synthetic"] = np.array(len(_cases()))


def gen_ml100k(out):
    import torch
    from daisy.model.Item2VecRecommender import Item2Vec
    from daisy.utils.sampler import SkipGramNegativeSampler
    from daisy.utils.dataset import BasicDataset, CandidatesDataset, get_dataloader
    from daisy.utils.utils import build_candidates_set
    cfg = rh.make_config("item2vec", factors=32, epochs=1)
    rh.seed_everything(cfg["seed"])
    art = rh.load_ml100k(cfg)
    train_set, test_ur, train_ur = art["train_set"], art["test_ur"], art["train_ur"]
    # the split is config 1's: its train rows and test sets are those of ml100k_sampler.npz / ml100k_rank.npz
    gs, gr = np.load(os.path.join(GOLD, "ml100k_sampler.npz")), np.load(os.path.join(GOLD, "ml100k_rank.npz"))
    assert np.array_equal(train_set["user"].values, gs["coo_u"]) and np.array_equal(train_set["item"].values, gs["coo_i"])
    off = np.concatenate([[0], np.cumsum(gr["gt_len"])])
    assert list(test_ur) == gr["test_u"].tolist()
    assert all(list(test_ur[u]) == gr["gt_flat"][off[k]:off[k + 1]].tolist() for k, u in enumerate(gr["test_u"].tolist()))
    model = Item2Vec(cfg)                                          # test.py:98
    out["ml_P0_sha"] = np.frombuffer(hashlib.sha256(model.user_embedding.weight.detach().numpy().tobytes()).digest(), np.uint8)
    out["ml_Q0_sha"] = np.frombuffer(hashlib.sha256(model.shared_embedding.weight.detach().numpy().tobytes()).digest(), np.uint8)
    rows = SkipGramNegativeSampler(train_set, cfg).sampling()      # test.py:99-100
    assert rows.dtype == np.int64
    out["ml_meta"] = np.array([cfg["user_num"], cfg["item_num"], cfg["factors"], cfg["context_window"], cfg["seed"],
                               cfg["batch_size"], rows.shape[0], STRIDE], np.int64)
    out["ml_lr"] = np.array(cfg["lr"], np.float64)
    out["ml_rows_sha"] = np.frombuffer(hashlib.sha256(np.ascontiguousarray(rows).tobytes()).digest(), np.uint8)
    out["ml_rows_head"] = rows[:EDGE].astype(np.int16)
    out["ml_rows_tail"] = rows[-EDGE:].astype(np.int16)
    out["ml_state"] = _np_state()

    # three steps of each optimiser on the first rows, in order (AbstractRecommender.py:116-128)
    B = cfg["batch_size"]
    for opt in ("sgd", "adam"):
        m = copy.deepcopy(model)
        m.criterion = m._build_criterion(m.loss_type)
        optimizer = m._build_optimizer(optimizer=opt, lr=m.lr)
        losses = []
        for s in range(3):
            batch = torch.from_numpy(rows[s * B:(s + 1) * B])
            m.zero_grad()
            loss = m.calc_loss((batch[:, 0], batch[:, 1], batch[:, 2]))
            loss.backward()
            optimizer.step()
            losses.append(float(loss.item()))
        out[f"ml_{opt}_losses"] = np.array(losses, np.float64)
        out[f"ml_{opt}_Q3"] = m.shared_embedding.weight.detach().numpy()[::STRIDE].copy()

    # one fit epoch in the DataLoader's order, recording the step losses
    step_losses = []
    orig = model.calc_loss

    def rec_loss(batch):
        loss = orig(batch)
        step_losses.append(float(loss.item()))
        return loss

    model.calc_loss = rec_loss
    loader = get_dataloader(BasicDataset(rows), batch_size=B, shuffle=True, num_workers=0)
    model.fit(loader)                                              # test.py:102
    out["ml_fit_losses"] = np.array(step_losses, np.float64)
    out["ml_fit_Q"] = model.shared_embedding.weight.detach().numpy().copy()
    out["ml_fit_P"] = model.user_embedding.weight.detach().numpy()[::STRIDE].copy()

    test_u, test_ucands = build_candidates_set(test_ur, train_ur, cfg)
    loader_t = get_dataloader(CandidatesDataset(test_ucands), batch_size=128, shuffle=False, num_workers=0)
    cands = np.stack([c[1] for c in test_ucands]).astype(np.int64)
    out["ml_cands_sha"] = np.frombuffer(hashlib.sha256(cands.tobytes()).digest(), np.uint8)
    out["ml_preds"] = model.rank(loader_t).astype(np.int16)
    out["ml_full"] = np.stack([model.full_rank(int(u)) for u in test_u[:4]])
    out["ml_predict"] = np.array([model.predict(int(test_u[0]), int(test_ucands[0][1][-1]))], np.float64)


def main():
    rh.import_reference()
    _shim()
    out = {}
    gen_synthetic(out)
    gen_ml100k(out)
    path = os.path.join(GOLD, "item2vec.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}  ({os.path.getsize(path) / 1024:.1f} KiB)")


if __name__ == "__main__":
    main()
