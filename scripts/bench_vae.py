"""Multi-VAE timings on the device: the step at the ML-20M shape (synthetic, utils.synthetic.make_interactions(138493, 26744,
20_000_000)) at B = 256 and 4 096 under both dropout engines, one epoch through VAECF(config).fit, rank 4 096 x 1 000 and
full_rank per user; then, in a run of its own under torch.profiler, the per-phase split of 20 steps at B = 256 ('philox'), each
phase against its computed bound; and the ml-100k fit at multi-vae.yaml (config 1's split, tests/golden/ml100k_sampler.npz)
on the device and, when oracle/_ref holds an installed reference, the reference's own fit on the host cores.  Prints one JSON
line per measurement, with the card's name and power limit read in the same run.

    python scripts/bench_vae.py [--users 138493 --items 26744 --rows 20000000]
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

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f"unknown ({e})"
    return q


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=138493)
    ap.add_argument("--items", type=int, default=26744)
    ap.add_argument("--rows", type=int, default=20_000_000)
    args = ap.parse_args()
    import pandas as pd
    from daisyrec_b200.model.VAECFRecommender import VAECF
    from daisyrec_b200.utils.dataset import AEDataset, get_dataloader
    from daisyrec_b200.utils.synthetic import make_interactions
    from daisyrec_b200.utils.utils import get_history_matrix
    gpu = card()
    out = lambda **kw: print(json.dumps(dict(kw, gpu=gpu)), flush=True)  # noqa: E731
    U, I = args.users, args.items
    inter = make_interactions(U, I, args.rows)
    u, i = inter['coo_u'].numpy(), inter['coo_i'].numpy()
    df = pd.DataFrame({'user': np.asarray(u), 'item': np.asarray(i)})
    cfg = dict(mlp_hidden_size=[600], latent_dim=128, dropout=0.5, lr=0.001, total_anneal_steps=100000, anneal_cap=0.2,
               epochs=1, optimizer='default', init_method='default', early_stop=False, topk=50, gpu='0', user_num=U,
               item_num=I, logger=logging.getLogger('bench'), UID_NAME='user', IID_NAME='item', progress=False)
    t = time.perf_counter()
    hid, hval, _ = get_history_matrix(df, cfg)
    out(what="get_history_matrix", seconds=time.perf_counter() - t, max_len=int(hid.shape[1]))
    cfg['history_item_id'], cfg['history_item_value'] = hid, hval
    users = torch.from_numpy(df['user'].unique().astype(np.int64))
    for engine in ('philox', 'torch'):
        model = VAECF(dict(cfg, dropout_engine=engine))
        model.train()
        for B in (256, 4096):
            model._hp = None
            batch = users[:B]
            reps = 20 if engine == 'philox' else 2
            s = timed(lambda: model.train_step(batch), reps)
            out(what="train_step", engine=engine, batch=B, ms=s * 1e3,
                decoder_gemm_gflop=6 * B * 600 * I / 1e9, adam_gb=32 * model.net.numel() / 1e9)
        del model
        torch.cuda.empty_cache()
    model = VAECF(dict(cfg, dropout_engine='philox'))
    loader = get_dataloader(AEDataset(df), batch_size=256, shuffle=True)
    torch.cuda.synchronize()
    t = time.perf_counter()
    model.fit(loader)
    torch.cuda.synchronize()
    out(what="fit_epoch", engine='philox', batch=256, seconds=time.perf_counter() - t)
    rs = np.random.default_rng(0)
    tu = rs.integers(0, U, 4096)
    cands = rs.integers(0, I, (4096, 1000))
    data = [[int(a), c] for a, c in zip(tu, cands)]
    loader = type('L', (), {'dataset': type('D', (), {'data': data})()})()
    out(what="rank", users=4096, cands=1000, ms=timed(lambda: model.rank(loader), 5) * 1e3)
    out(what="full_rank", ms_per_user=timed(lambda: model.full_rank(int(tu[0])), 20) * 1e3)
    phases(model, users, I, out)
    del model
    torch.cuda.empty_cache()
    ml100k(out, cfg)


PHASES = (   # kernel name fragments -> phase
    ("input", ("vae_batch_len", "vae_exscan", "vae_input_kernel", "vae_widen", "vae_group", "vae_clear_stale", "Memset")),
    ("sparse layer 0 (enc0 + dW0)", ("vae_enc0", "vae_dw0")),
    ("dense GEMMs", ("sgemm_kernel",)),
    ("fused CE + loss", ("vae_ce_kernel", "vae_loss_kernel")),
    ("element-wise (bias, tanh, reparam, slice sums, column sums)", ("vae_bias_act", "vae_tanh_back", "vae_slice_sum",
                                                                       "vae_colsum", "vae_reparam")),
    ("Adam", ("dense_update_kernel",)),
)


def phases(model, users, I, out, B=256, steps=20):
    """per-phase device time of `steps` steps (torch.profiler, CUDA activities), each against its bound: the dense GEMMs
    against 6 B H I + the hidden layers' FLOPs at 67 TFLOP/s (FP32 data sheet), Adam against 32 bytes per parameter at
    3.35 TB/s; the other phases are reported as time only"""
    from torch.profiler import ProfilerActivity, profile
    model._hp = None
    batch = users[:B]
    model.train_step(batch)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            model.train_step(batch)
        torch.cuda.synchronize()
    tot = {name: 0.0 for name, _ in PHASES}
    other = 0.0
    for ev in prof.key_averages():
        t = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        for name, frags in PHASES:
            if any(f in ev.key for f in frags):
                tot[name] += t
                break
        else:
            other += t
    H, lat = model.layers[0], model.lat_dim
    gflop = 6 * B * H * I + 6 * B * (H * lat + lat // 2 * H)
    nW = model.net.numel()
    bounds = {"dense GEMMs": (gflop / 67e12 * 1e3, "FP32 67 TFLOP/s"), "Adam": (32 * nW / 3.35e12 * 1e3, "HBM 3.35 TB/s")}
    step_ms = sum(tot.values()) / 1e3 / steps + other / 1e3 / steps
    for name, t in tot.items():
        ms = t / 1e3 / steps
        rec = dict(what="phase", phase=name, batch=B, ms_per_step=ms, share_of_step=ms / step_ms)
        if name in bounds:
            rec.update(bound_ms=bounds[name][0], bound=bounds[name][1], fraction_of_bound=bounds[name][0] / ms if ms else None)
        out(**rec)
    out(what="phase", phase="other kernels", batch=B, ms_per_step=other / 1e3 / steps)


def ml100k(out, base_cfg):
    """the ml-100k fit at multi-vae.yaml through the driver sequence: ours on the device, the reference on the host cores"""
    import pandas as pd
    from daisyrec_b200.model.VAECFRecommender import VAECF
    from daisyrec_b200.utils.dataset import AEDataset, get_dataloader
    from daisyrec_b200.utils.utils import get_history_matrix
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    gs = np.load(os.path.join(root, "tests", "golden", "ml100k_sampler.npz"))
    df = pd.DataFrame({'user': gs["coo_u"].astype(np.int64), 'item': gs["coo_i"].astype(np.int64), 'rating': 1.0})
    U, I = int(df.user.max()) + 1, 1152
    cfg = dict(base_cfg, user_num=U, item_num=I, epochs=10, dropout_engine='auto')
    cfg.pop('history_item_id', None)
    cfg.pop('history_item_value', None)

    def ours():
        torch.manual_seed(2022)
        hid, hval, _ = get_history_matrix(df, cfg)
        m = VAECF(dict(cfg, history_item_id=hid, history_item_value=hval))
        m.fit(get_dataloader(AEDataset(df), batch_size=256, shuffle=True))
        torch.cuda.synchronize()

    ours()
    t = time.perf_counter()
    ours()
    out(what="ml100k_fit", impl="device ('auto': host masks)", seconds=time.perf_counter() - t)
    from oracle import ref_harness as rh
    if not os.path.isdir(os.path.join(rh.INSTALLED_ROOT, "daisy")):
        out(what="ml100k_fit", impl="reference", seconds=None, note="oracle/_ref absent: not measured")
        return
    rh.use_root(rh.INSTALLED_ROOT)
    rh.import_reference()
    from daisy.model.VAECFRecommender import VAECF as RefVAECF
    from daisy.utils.dataset import AEDataset as RefAE, get_dataloader as ref_loader
    from daisy.utils.utils import get_history_matrix as ref_hist
    rcfg = rh.make_config('multi-vae', user_num=U, item_num=I, UID_NAME='user', IID_NAME='item')

    def ref():
        rh.seed_everything(2022)
        hid, hval, _ = ref_hist(df, rcfg, row='user')
        m = RefVAECF(dict(rcfg, history_item_id=hid, history_item_value=hval))
        m.fit(ref_loader(RefAE(df, yield_col='user'), batch_size=256, shuffle=True, num_workers=0))

    ref()
    t = time.perf_counter()
    ref()
    out(what="ml100k_fit", impl="reference (host cores, torch CPU)", threads=torch.get_num_threads(),
        seconds=time.perf_counter() - t)


if __name__ == "__main__":
    main()
