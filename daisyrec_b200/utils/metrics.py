"""Ranking KPIs with the reference's entry points (daisy/utils/metrics.py:5-96), computed by ONE
device launch over rank()'s output instead of a Python loop over test users per metric and cut-off.

``calc_ranking_results(test_ur, pred_ur, test_u, config)`` returns the same DataFrame (column
'KPI@K' + one column per cut-off of common_ks, :41-56) and logs the @10 rows; ``Metric(config).run``
returns the list of KPIs of one rank list.  ``pred_ur`` is rank()'s numpy array, or a float32 CUDA
tensor (ops.mf_rank's output) to skip the round trip through the host.  Numbers are fp64 like the reference's; the per-user
values are reduced in a fixed order on the device, np.mean sums pairwise: agreement ~1e-15 relative.

Reference quirks kept: duplicate ids in a rank list each count as a hit (np.in1d); Recall can exceed
1 for that reason; NDCG's ideal DCG uses the number of hits INSIDE the list (:230), not |gt|;
'f1' / 'auc' cannot be reached through Metric.run (:87-90 compare the previous KPI, not the name) and
raise ValueError here too; 'map' runs in Metric.run but has no display name, so calc_ranking_results
raises KeyError on it exactly like :38.  'diversity' (item categories) is outside the GPU path.
"""
import os

import numpy as np
import pandas as pd
import torch

from .. import ops
from .._lib import KPI_NAMES

metrics_name_config = {
    "recall": 'Recall',
    "mrr": 'MRR',
    "ndcg": 'NDCG',
    "hit": 'Hit Ratio',
    "precision": 'Precision',
    "f1": 'F1-score',
    "auc": 'AUC',
    "coverage": 'Coverage',
    "diversity": 'Diversity',
    "popularity": 'Average Popularity',
}

_DEVICE_KPIS = ("recall", "mrr", "ndcg", "hit", "precision", "map", "coverage", "popularity")


def ground_truth_csr(test_ur, test_u):
    """test_ur[u] (set) for u in test_u -> (gt_ptr int64[n+1], gt_idx int32, ascending inside a row)."""
    n = len(test_u)
    lens = np.fromiter((len(test_ur[u]) for u in test_u), np.int64, n)
    ptr = np.zeros(n + 1, np.int64)
    np.cumsum(lens, out=ptr[1:])
    flat = np.fromiter((i for u in test_u for i in test_ur[u]), np.int64, int(ptr[-1]))
    key = np.repeat(np.arange(n, dtype=np.int64), lens) * (1 << 32) + flat
    key.sort()
    return ptr, (key & 0xFFFFFFFF).astype(np.int32)


def _kpi_table(test_ur, pred_ur, test_u, ks, item_num, item_pop):
    """-> float64 [len(ks), 8] (KPI_NAMES order) for the cut-offs ks of the rank lists pred_ur."""
    ops.require_cuda()
    ptr, idx = ground_truth_csr(test_ur, test_u)
    ks = [min(int(k), int(pred_ur.shape[1])) for k in ks]          # pred_ur[:, :topk] of a shorter list (:49)
    dev = pred_ur if isinstance(pred_ur, torch.Tensor) else None   # ops.mf_rank's output left on the device
    if dev is not None and dev.is_cuda and dev.dtype == torch.float32 and dev.is_contiguous():
        d_pop = None if item_pop is None else torch.from_numpy(np.ascontiguousarray(item_pop, np.float64)).to(dev.device)
        out = ops.rank_metrics(dev, torch.from_numpy(ptr).to(dev.device), torch.from_numpy(idx).to(dev.device), ks,
                               item_num, d_pop)
        return out.cpu().numpy()
    pred = np.asarray(pred_ur.cpu() if isinstance(pred_ur, torch.Tensor) else pred_ur)
    if pred.ndim != 2:
        raise ValueError(f'rank list must be [n_users, topk], got shape {pred.shape}')
    return ops.rank_metrics_host(pred.astype(np.float32, copy=False), ptr, idx, ks, item_num, item_pop)


def _check_names(names):
    for mc in names:
        if mc == 'diversity':
            raise NotImplementedError("'diversity' needs config['i_categories']; it is outside the GPU evaluation path")
        if mc not in _DEVICE_KPIS:
            raise ValueError(f'Invalid metric name {mc}')          # metrics.py:91-92 (also where 'f1' / 'auc' end up)


def calc_ranking_results(test_ur, pred_ur, test_u, config):
    '''
    calculate metrics with prediction results and candidates sets (daisy/utils/metrics.py:18-57)

    Parameters
    ----------
    test_ur : defaultdict(set)
        groud truths for user in test set
    pred_ur : np.array
        rank list for user in test set
    test_u : list
        the user in order from test set
    '''
    logger = config['logger']
    path = config['res_path']
    if not os.path.exists(path):
        os.makedirs(path)

    names = list(config['metrics'])
    res = pd.DataFrame({'KPI@K': [metrics_name_config[kpi_name] for kpi_name in names]})
    _check_names(names)

    common_ks = [1, 5, 10, 20, 30, 50]
    if config['topk'] not in common_ks:
        common_ks.append(config['topk'])
    ks = [k for k in common_ks if k <= config['topk']]
    metric = Metric(config)
    table = _kpi_table(test_ur, pred_ur, test_u, ks, metric.item_num, metric.item_pop)
    cols = [KPI_NAMES.index(mc) for mc in names]
    for row, topk in enumerate(ks):
        kpis = [float(table[row, c]) for c in cols]
        if topk == 10:
            for kpi_name, kpi_res in zip(names, kpis):
                logger.info(f'{metrics_name_config[kpi_name]}@{topk}: {kpi_res:.4f}')
        res[topk] = np.array(kpis)

    return res


class Metric(object):
    def __init__(self, config) -> None:
        self.metrics = config['metrics']
        self.item_num = config['item_num']
        # the reference keys item_pop on 'coverage' (:63) although 'popularity' is its only consumer (:72)
        self.item_pop = config['item_pop'] if 'popularity' in self.metrics else None

    def run(self, test_ur, pred_ur, test_u):
        _check_names(self.metrics)
        k = pred_ur.shape[1]
        table = _kpi_table(test_ur, pred_ur, test_u, [k], self.item_num, self.item_pop)
        return [float(table[0, KPI_NAMES.index(mc)]) for mc in self.metrics]
