"""Generates tests/golden/vae.npz from the reference's own Multi-VAE (daisy/model/VAECFRecommender.py), imported through
oracle/ref_harness.py.

Synthetic cases, each fitted through the reference's driver sequence (get_history_matrix -> VAECF -> AEDataset loader -> fit):
  a  one hidden layer [16], latent 8, dropout 0.5, Adam, 3 epochs of batches 16 over 37 users (a ragged last batch); users
     0..2 cold; duplicate (user, item) rows with differing values; item 0 held by the longest user (kept) and by a shorter one
     (erased by the padding slot)
  b  hidden [48, 24], latent 9 (odd: the middle column is in neither mu nor logvar), SGD, dropout 0, real-valued ratings
Each case stores the history tensors, the init and final state, the per-step losses, rank on 12 candidates of every user,
full_rank of 4 users, predict on 6 pairs and the global torch RNG state after fit.
ml-100k on config 1's split at multi-vae.yaml: per-step losses, per final tensor its digest, every 8th row and its column sums,
rank on all test users with their top-(k+1) candidate scores, full_rank of 4 users, predict on 8 pairs, the KPI table, and the
KPI tables of the reference's fits from seeds 1..5 (the spread a fit with another random stream should land in), and the steps
and (user, item) pairs where the reference's own rating matrix broke the last-write rule (its CPU index_put_ runs in parallel
chunks; a row that straddles a chunk boundary can have an earlier slot written after a later one).

    python oracle/gen_vae.py
"""
import hashlib
import os
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_harness as rh  # noqa: E402
from oracle import vae_oracle  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
ROW_STRIDE = 8
KEYS = ('encoder.0.weight', 'encoder.0.bias', 'encoder.2.weight', 'encoder.2.bias', 'encoder.4.weight', 'encoder.4.bias',
        'decoder.0.weight', 'decoder.0.bias', 'decoder.2.weight', 'decoder.2.bias', 'decoder.4.weight', 'decoder.4.bias')


def sha(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return np.frombuffer(h.digest(), np.uint8)


def synthetic_frames():
    """-> {case: (DataFrame, U, I, config overrides)}"""
    import pandas as pd
    rng = np.random.default_rng(2024)
    out = {}
    U, I = 37, 50
    u = rng.integers(3, U, 400)
    i = rng.integers(1, I, 400)
    k = rng.integers(0, 400, 40)                                   # duplicate pairs
    u, i = np.concatenate([u, u[k]]), np.concatenate([i, i[k]])
    cnt = np.bincount(u, minlength=U)
    longest, shortest = cnt.argmax(), 3 + cnt[3:].argmin()
    u, i = np.concatenate([u, [longest, shortest]]), np.concatenate([i, [0, 0]])   # item 0: the longest and a short user
    v = rng.integers(1, 6, len(u)).astype(np.float64)
    out['a'] = (pd.DataFrame({'user': u, 'item': i, 'rating': v}), U, I,
                dict(mlp_hidden_size=[16], latent_dim=8, dropout=0.5, optimizer='adam', lr=0.01, epochs=3, batch_size=16,
                     total_anneal_steps=4, anneal_cap=0.2))
    U, I = 30, 40
    u, i = rng.integers(0, U, 300), rng.integers(0, I, 300)
    v = (rng.random(len(u)) * 3 + 0.5).astype(np.float32).astype(np.float64)
    out['b'] = (pd.DataFrame({'user': u, 'item': i, 'rating': v}), U, I,
                dict(mlp_hidden_size=[48, 24], latent_dim=9, dropout=0.0, optimizer='sgd', lr=0.05, epochs=2, batch_size=8,
                     total_anneal_steps=0, anneal_cap=0.3, use_value=True))
    return out


def ref_fit(cfg, train_set, use_value=False, bs=None):
    """The driver of run_examples/test.py:79-85 -> (model, per-step losses, history tensors)."""
    import torch
    from daisy.model.VAECFRecommender import VAECF
    from daisy.utils.dataset import AEDataset, get_dataloader
    from daisy.utils.utils import get_history_matrix
    if use_value:
        cfg['INTER_NAME'] = 'rating'
    hid, hval, _ = get_history_matrix(train_set, cfg, row='user', use_config_value_name=use_value)
    cfg['history_item_id'], cfg['history_item_value'] = hid, hval
    model = VAECF(cfg)
    init = {k: v.detach().clone().numpy() for k, v in model.state_dict().items()}
    losses, broken = [], []
    calc, rows = model.calc_loss, model.get_user_rating_matrix
    rule = vae_oracle.input_rows(hid.numpy(), hval.numpy(), cfg['item_num'])

    def rating(user):
        # the reference's CPU index_put_ runs in parallel chunks: where a row straddles a chunk boundary, an earlier slot can
        # land after a later one.  Record the (user, item) pairs where this batch's matrix breaks the last-write rule.
        R = rows(user)
        d = np.nonzero(R.numpy() != rule[user.numpy()])
        broken.append(np.stack([user.numpy()[d[0]], d[1]], 1))
        return R

    def rec(batch):
        loss = calc(batch)
        losses.append(float(loss.item()))
        return loss

    model.calc_loss, model.get_user_rating_matrix = rec, rating
    loader = get_dataloader(AEDataset(train_set, yield_col=cfg['UID_NAME']), batch_size=bs or cfg['batch_size'], shuffle=True,
                            num_workers=0)
    model.fit(loader)
    model.calc_loss, model.get_user_rating_matrix = calc, rows
    rng_after = torch.get_rng_state().numpy().copy()
    model.broken = broken
    return model, np.array(losses, np.float64), hid.numpy(), hval.numpy(), init, rng_after


class _Loader:
    def __init__(self, users, cands, bs=16):
        self.users, self.cands, self.bs = users, cands, bs

    def __iter__(self):
        import torch
        for s in range(0, len(self.users), self.bs):
            yield torch.from_numpy(self.users[s:s + self.bs]), torch.from_numpy(self.cands[s:s + self.bs])


def gen_synthetic(out):
    import torch
    for name, (df, U, I, over) in synthetic_frames().items():
        over = dict(over)
        use_value = over.pop('use_value', False)
        cfg = rh.make_config('multi-vae', user_num=U, item_num=I, UID_NAME='user', IID_NAME='item', **over)
        rh.seed_everything(2019)
        model, losses, hid, hval, init, rng_after = ref_fit(cfg, df, use_value)
        sd = {k: v.detach().numpy().copy() for k, v in model.state_dict().items()}
        p = f's{name}_'
        out[p + 'df'] = np.stack([df['user'].values, df['item'].values]).astype(np.int64)
        out[p + 'rating'] = df['rating'].values.astype(np.float64)
        out[p + 'meta'] = np.array([U, I, over['latent_dim'], over['epochs'], over['batch_size'], int(use_value),
                                    over['total_anneal_steps']], np.int64)
        out[p + 'hidden'] = np.array(over['mlp_hidden_size'], np.int64)
        out[p + 'fl'] = np.array([over['dropout'], over['lr'], over['anneal_cap']], np.float64)
        out[p + 'opt'] = np.array([over['optimizer']])
        out[p + 'hist_id'] = hid
        out[p + 'hist_val'] = hval
        out[p + 'keys'] = np.array(list(sd))
        for j, k in enumerate(sd):
            out[p + f'init{j}'] = init[k]
            out[p + f'final{j}'] = sd[k]
        out[p + 'losses'] = losses
        assert all(len(b) == 0 for b in model.broken)
        out[p + 'rng_after'] = rng_after
        rs = np.random.default_rng(7)
        users = np.arange(U, dtype=np.int64)
        cands = np.stack([rs.permutation(I)[:12] for _ in users]).astype(np.int64)
        out[p + 'cands'] = cands
        out[p + 'rank'] = model.rank(_Loader(users, cands)).astype(np.int64)
        model.eval()
        with torch.no_grad():
            logits = model.forward(model.get_user_rating_matrix(torch.from_numpy(users)))[0].numpy()
        out[p + 'logits'] = logits
        fu = np.array([0, 3, 5, U - 1], np.int64)
        out[p + 'full_u'] = fu
        out[p + 'full'] = np.stack([model.full_rank(int(u)) for u in fu]).astype(np.int64)
        pairs = np.stack([rs.integers(0, U, 6), rs.integers(0, I, 6)], 1).astype(np.int64)
        out[p + 'predict_pairs'] = pairs
        out[p + 'predict'] = np.array([model.predict(int(a), int(b)) for a, b in pairs], np.float64)


def gen_ml100k(out):
    import torch
    from daisy.utils.dataset import CandidatesDataset, get_dataloader
    from daisy.utils.utils import build_candidates_set
    from daisy.utils.metrics import calc_ranking_results

    def run(seed, full):
        cfg = rh.make_config('multi-vae', seed=seed)
        rh.seed_everything(cfg['seed'])
        art = rh.load_ml100k(cfg)
        train_set, test_ur, train_ur = art['train_set'], art['test_ur'], art['train_ur']
        model, losses, hid, hval, init, _ = ref_fit(cfg, train_set)
        test_u, test_ucands = build_candidates_set(test_ur, train_ur, cfg)
        loader = get_dataloader(CandidatesDataset(test_ucands), batch_size=128, shuffle=False, num_workers=0)
        preds = model.rank(loader)
        cfg['res_path'] = tempfile.mkdtemp() + '/'
        res = calc_ranking_results(test_ur, preds, test_u, cfg)
        if not full:
            return res.values[:, 1:].astype(np.float64)
        U, I = cfg['user_num'], cfg['item_num']
        cands = np.stack([c[1] for c in test_ucands]).astype(np.int64)
        sd = {k: v.detach().numpy().copy() for k, v in model.state_dict().items()}
        out['ml_meta'] = np.array([U, I, cfg['topk'], cfg['seed'], ROW_STRIDE, cfg['batch_size'], cfg['epochs'],
                                   hid.shape[1]], np.int64)
        out['ml_hist_sha'] = sha(hid, hval)
        out['ml_losses'] = losses
        out['ml_broken_steps'] = np.array([len(b) > 0 for b in model.broken])
        out['ml_broken_pairs'] = np.concatenate(model.broken).astype(np.int64).reshape(-1, 2)
        out['ml_keys'] = np.array(list(sd))
        for j, k in enumerate(sd):
            t = sd[k]
            out[f'ml_sha{j}'] = sha(t)
            out[f'ml_rows{j}'] = t[::ROW_STRIDE]
            out[f'ml_colsum{j}'] = t.sum(0)
        out['ml_cands_sha'] = sha(cands)
        out['ml_test_u'] = np.array(test_u, np.int32)
        out['ml_rank'] = preds.astype(np.int16)
        model.eval()
        with torch.no_grad():
            logits = model.forward(model.get_user_rating_matrix(torch.as_tensor(np.array(test_u))))[0].numpy()
        cs = np.take_along_axis(logits, cands, 1)
        out['ml_top_scores'] = -np.sort(-cs, 1)[:, :cfg['topk'] + 1]
        fu = np.array(test_u[:4], np.int64)
        out['ml_full_u'] = fu
        out['ml_full'] = np.stack([model.full_rank(int(u)) for u in fu]).astype(np.int16)
        pairs = np.array([[test_u[k], cands[k][-1 - k]] for k in range(8)], np.int64)
        out['ml_predict_pairs'] = pairs
        out['ml_predict'] = np.array([model.predict(int(u), int(i)) for u, i in pairs], np.float64)
        out['ml_kpi'] = res.values[:, 1:].astype(np.float64)
        out['ml_kpi_ks'] = np.array([int(c) for c in res.columns[1:]], np.int32)
        return out['ml_kpi']

    run(rh.make_config('multi-vae')['seed'], True)
    out['ml_kpi_seeds'] = np.stack([run(s, False) for s in range(1, 6)])


def main():
    rh.import_reference()
    out = {}
    gen_synthetic(out)
    gen_ml100k(out)
    path = os.path.join(GOLD, 'vae.npz')
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
