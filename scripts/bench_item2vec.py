"""Item2Vec throughput on one GPU: prints one JSON line.

    python scripts/bench_item2vec.py [--shape ml-20m] [--steps 20] [--ref-steps 20]

* sampler: SkipGramNegativeSampler.sampling() at the given synthetic shape (utils/synthetic.py), window 2; host draw time
  (the sequential MT19937 replay) and device time (grouping, offsets, emission) reported apart, rows/s over their sum;
* step:    drb_i2v_train_steps, event-timed over persistent launches at B = 1 048 576, F = 100, Adam; the algorithmic bytes
  per row (16 F + 12: two row reads and two gradient reductions of F floats, three int32 indices) plus the per-step dense
  Adam sweep of the item table (5 table-sized fp32 reads and 4 writes: theta, g, m, v) against the 3.35 TB/s data-sheet HBM3
  bandwidth of the H100 SXM (labelled data-sheet: not a measured peak);
* e2e:     one fit() epoch (default config: B = 256, Adam, F = 100) over the first --e2e-rows of the sampler's rows;
* reference: the reference's own SkipGramNegativeSampler + K fit steps on ml-100k on the host, from oracle/_ref when it
  was installed by build(); labelled as such.
"""
import argparse
import json
import logging
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from daisyrec_b200 import ops  # noqa: E402
from daisyrec_b200.utils import synthetic  # noqa: E402

HBM_DATASHEET = 3.35e12


def device_info():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(out.splitlines()[0])
    except Exception:  # noqa: BLE001
        power = None
    return name, power


def bench_sampler(shape, window):
    U, I, nnz = synthetic.SHAPES[shape]
    d = synthetic.make_interactions(U, I, nnz, device="cuda")
    row_ptr, col = d["row_ptr"], d["col"]
    coo_u, coo_i = d["coo_u"], d["coo_i"]
    h_row_ptr = row_ptr.cpu().numpy()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    seq_ptr, ctx_ptr, order = ops.skipgram_group(coo_u, U, window)
    seq_len = np.diff(seq_ptr.cpu().numpy())
    total = int(ctx_ptr[-1].item())
    t1 = time.perf_counter()
    draws = ops.skipgram_draws_mt19937(ops.mt19937_seed(2022), I - np.diff(h_row_ptr), seq_len, window, total)
    t2 = time.perf_counter()
    d_draws = torch.from_numpy(draws).cuda()
    rows = ops.skipgram_emit(coo_u, coo_i, order, window, seq_ptr, ctx_ptr, row_ptr, col, d_draws, total)
    torch.cuda.synchronize()
    t3 = time.perf_counter()
    host_s, dev_s = t2 - t1, (t1 - t0) + (t3 - t2)
    return dict(shape=shape, window=window, nnz=int(d["nnz"]), rows=int(rows.shape[0]), host_draw_s=host_s, device_s=dev_s,
                rows_per_s=rows.shape[0] / (host_s + dev_s)), rows, I


def bench_step(rows, I, F=100, B=1 << 20, steps=20):
    Q = (torch.randn(I, F, device="cuda") * 0.01).contiguous()
    ws = ops.I2VWorkspace(I, F, "adam", Q.device)
    n = min(rows.shape[0], B * steps)
    bt, bc, bl = (rows[:n, k].contiguous() for k in range(3))
    hp = ops.hyper(0.001, 0., 0., "adam", loss="CL")
    k = (n + B - 1) // B
    ops.i2v_train_steps(Q, ws, bt, bc, bl, B, 0, min(k, 2), hp)           # warm-up
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    ops.i2v_train_steps(Q, ws, bt, bc, bl, B, 0, k, hp, adam_step0=2)
    e1.record()
    torch.cuda.synchronize()
    s = e0.elapsed_time(e1) / 1e3
    bytes_row = 16 * F + 12
    sweep = 9 * 4 * I * F
    algo = n * bytes_row + k * sweep
    return dict(batch=B, factors=F, steps=k, rows=n, seconds=s, rows_per_s=n / s, bytes_per_row=bytes_row,
                sweep_bytes_per_step=sweep, algorithmic_GBps=algo / s / 1e9,
                share_of_datasheet_hbm=algo / s / HBM_DATASHEET)


def bench_e2e(rows_dev, U, I, F=100):
    from daisyrec_b200.model.Item2VecRecommender import Item2Vec
    from daisyrec_b200.utils.dataset import BasicDataset, get_dataloader
    from daisyrec_b200.utils.sampler import TripleArray
    cfg = dict(gpu='', user_num=U, item_num=I, factors=F, train_ur={}, lr=0.001, epochs=1, optimizer='default',
               init_method='default', early_stop=False, topk=50, logger=logging.getLogger('bench'), progress=False)
    model = Item2Vec(cfg)
    host = TripleArray.attach(np.empty((rows_dev.shape[0], 3), np.int32), rows_dev)
    loader = get_dataloader(BasicDataset(host), batch_size=256, shuffle=True, num_workers=0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    model.fit(loader)
    torch.cuda.synchronize()
    s = time.perf_counter() - t0
    return dict(rows=int(rows_dev.shape[0]), batch=256, seconds=s, rows_per_s=rows_dev.shape[0] / s)


def bench_reference(steps):
    from oracle import ref_harness as rh
    rh.use_root(rh.INSTALLED_ROOT)
    if not rh.available() or not os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "data", "ml-100k")):
        return dict(status="not measured: oracle/_ref with ml-100k absent")
    rh.import_reference()
    import pandas as pd
    if not hasattr(pd.Series, "iteritems"):
        pd.Series.iteritems = pd.Series.items
    from daisy.model.Item2VecRecommender import Item2Vec
    from daisy.utils.sampler import SkipGramNegativeSampler
    from daisy.utils.dataset import BasicDataset, get_dataloader
    cfg = rh.make_config("item2vec", data_path=os.path.join(rh.INSTALLED_ROOT, "data") + "/")
    rh.seed_everything(cfg["seed"])
    art = rh.load_ml100k(cfg)
    model = Item2Vec(cfg)
    t0 = time.perf_counter()
    rows = SkipGramNegativeSampler(art["train_set"], cfg).sampling()
    t1 = time.perf_counter()
    model.epochs = 1
    loader = get_dataloader(BasicDataset(rows[:steps * cfg["batch_size"]]), batch_size=cfg["batch_size"], shuffle=True,
                            num_workers=0)
    model.fit(loader)
    t2 = time.perf_counter()
    return dict(label="reference daisyRec on the host CPU, ml-100k", rows=int(rows.shape[0]), sampling_s=t1 - t0,
                fit_steps=steps, fit_s=t2 - t1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", default="ml-20m")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--ref-steps", type=int, default=20)
    ap.add_argument("--e2e-rows", type=int, default=1 << 23)
    a = ap.parse_args()
    ops.require_cuda()
    torch.cuda.set_device(0)
    name, power = device_info()
    res = dict(bench="item2vec", device=name, power_limit_w=power)
    res["sampler"], rows, I = bench_sampler(a.shape, 2)
    res["step"] = bench_step(rows, I, steps=a.steps)
    res["e2e"] = bench_e2e(rows[:a.e2e_rows], synthetic.SHAPES[a.shape][0], I)
    res["reference"] = bench_reference(a.ref_steps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
