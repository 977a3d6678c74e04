"""Restatement of the reference's Item2Vec path (daisy/utils/sampler.py:105-160, daisy/model/Item2VecRecommender.py:16-107)
in numpy -- TEST INFRASTRUCTURE ONLY, the checker of the GPU path and of tests/golden/item2vec.npz.

* skipgram_rows: the sampler, drawing its negatives with the same RandomState.choice calls in the same order (exact);
* i2v_step:      one tied-table BCEWithLogitsLoss(sum) step in fp64, then SGD or torch's Adam in fp64;
* user_embedding: the per-user row sums, in fp64.
"""
import numpy as np


def group_sequences(users, items):
    """groupby(user)[item].agg(list): {user: item list}, users ascending, row order kept."""
    users = np.asarray(users, np.int64)
    items = np.asarray(items, np.int64)
    order = np.argsort(users, kind="stable")
    su, si = users[order], items[order]
    bounds = np.flatnonzero(np.diff(su)) + 1
    return {int(g[0]): i.tolist() for g, i in zip(np.split(su, bounds), np.split(si, bounds)) if len(g)}


def discard_rows(users, items, rho, rs=np.random):
    """discard=True (sampler.py:125-131): drop a row when uniform() < 1 - sqrt(rho / count(item))."""
    items = np.asarray(items, np.int64)
    cnt = np.bincount(items)
    u01 = rs.uniform(low=0., high=1., size=len(items))
    keep = u01 >= 1 - np.sqrt(rho / cnt[items])
    return np.asarray(users)[keep], items[keep]


def skipgram_rows(seqs, ur, item_num, window, rs=np.random):
    """int64 [T, 3] rows of SkipGramNegativeSampler.sampling() for the sequences ``seqs``."""
    out = []
    for u in sorted(seqs):
        seq = seqs[u]
        cands = np.setdiff1d(np.arange(item_num), list(ur[u]))
        L = len(seq)
        for i in range(L):
            ctx = [seq[j] for j in range(max(0, i - window), min(L - 1, i + window) + 1) if j != i]
            block = np.empty((2 * len(ctx), 3), np.int64)
            block[:len(ctx), 0] = seq[i]
            block[:len(ctx), 1] = ctx
            block[:len(ctx), 2] = 1
            block[len(ctx):, 0] = seq[i]
            block[len(ctx):, 1] = rs.choice(cands, size=len(ctx))
            block[len(ctx):, 2] = 0
            out.append(block)
    return np.concatenate(out) if out else np.zeros((0, 3), np.int64)


def i2v_step(Q, rows, lr, opt="sgd", adam=None, step=1, apply=True, betas=(0.9, 0.999), eps=1e-8):
    """One step on the fp64 table Q (updated in place) -> loss.  adam = (m, v) fp64 state, updated in place."""
    t, c = rows[:, 0].astype(np.int64), rows[:, 1].astype(np.int64)
    y = rows[:, 2].astype(np.float64)
    x = np.einsum("bf,bf->b", Q[t], Q[c])
    loss = float(np.sum(np.maximum(x, 0) - x * y + np.log1p(np.exp(-np.abs(x)))))
    if not apply:
        return loss
    d = 1.0 / (1.0 + np.exp(-x)) - y                               # d loss / d x
    g = np.zeros_like(Q)
    np.add.at(g, t, d[:, None] * Q[c])
    np.add.at(g, c, d[:, None] * Q[t])
    if opt == "sgd":
        Q -= lr * g
    else:
        m, v = adam
        b1, b2 = betas
        m[:] = b1 * m + (1 - b1) * g
        v[:] = b2 * v + (1 - b2) * g * g
        Q -= (lr / (1 - b1 ** step)) * m / (np.sqrt(v) / np.sqrt(1 - b2 ** step) + eps)
    return loss


def user_embedding(Q, ur, P):
    """P[u] = sum of Q[train_ur[u]] for every u in train_ur (fp64); other rows unchanged."""
    P = np.array(P, np.float64)
    for u, items in ur.items():
        P[u] = np.asarray(Q, np.float64)[sorted(items)].sum(0)
    return P


def build_candidates_set(test_ur, train_ur, item_num, cand_num, rs=np.random):
    """daisy/utils/utils.py:53-85 (drop_past_inter=True) -> (test_u, int64 [n_users, cand_num] candidates)."""
    test_u, cands = [], []
    for u, r in test_ur.items():
        sample_num = cand_num - len(r) if len(r) <= cand_num else 0
        if sample_num == 0:
            samples = rs.choice(list(r), cand_num)
        else:
            neg_items = np.setdiff1d(np.arange(item_num), list(r) + list(train_ur.get(u, ())))   # get_ur is a defaultdict(set)
            samples = np.concatenate((rs.choice(neg_items, size=sample_num), list(r)), axis=None)
        test_u.append(u)
        cands.append(np.asarray(samples, np.int64))
    return test_u, np.stack(cands)
