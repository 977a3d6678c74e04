"""Host side of the GPU-path recommenders: the reference's plug-in surface
(daisy/model/AbstractRecommender.py:10-137) without nn.Module / autograd / torch.optim.

``GeneralRecommender.fit(train_loader)`` keeps the reference contract -- a
``torch.utils.data.DataLoader`` over ``BasicDataset(samples)``, ``batch_size`` and ``shuffle`` read
from the loader, epoch loss accumulated from per-step losses, ``ValueError`` on a NaN loss, early
stop on |delta epoch loss| < 1e-5 -- but runs each epoch as ONE persistent kernel launch:
the epoch's permutation is produced with the DataLoader's own RNG protocol (so batches are the
reference's batches), gathered into SoA index planes on the device, and consumed by
``drb_mf_bpr_train_steps``.
"""
import functools
import os

import numpy as np
import torch
from torch.utils.data import RandomSampler, SequentialSampler, BatchSampler
from tqdm import tqdm

from .. import ops
from ..utils.sampler import fingerprint


# 'torch': the DataLoader's own permutation -- the reference's batches bit for bit -- computed ON THE DEVICE
#          (drb_randperm_torch: MT19937 stream + parallel Fisher-Yates, same result as torch.randperm on the CPU generator);
# 'torch-cpu': the same permutation from torch.randperm on the host (what the line above is tested against);
# 'device': torch.randperm on the GPU, seeded from the global RNG (same distribution, another order)
DEFAULT_SHUFFLE_ENGINE = 'torch'
RANDPERM_DEVICE_MAX = 0xFFFFFFFF // 20          # ATen switches algorithm above this n; the host path covers it


class _Table:
    """Stand-in for nn.Embedding: ``.weight`` is the raw fp32 [rows, factors] table."""

    def __init__(self, weight):
        self.weight = weight

    @property
    def num_embeddings(self):
        return self.weight.shape[0]

    @property
    def embedding_dim(self):
        return self.weight.shape[1]


def _init_table(rows, cols, method):
    """Reproduce the reference's CPU init stream: nn.Embedding's own N(0,1) reset first
    (torch/nn/modules/sparse.py reset_parameters), re-initialised later by ``_apply_init``."""
    return torch.empty(rows, cols, dtype=torch.float32).normal_(0.0, 1.0)


_INIT = {
    # AbstractRecommender.py:19-31 (initializer_param_config / initializer_config)
    'normal': lambda w: torch.nn.init.normal_(w, mean=0.0, std=0.01),
    'uniform': lambda w: torch.nn.init.uniform_(w, a=0.0, b=1.0),
    'xavier_normal': lambda w: torch.nn.init.xavier_normal_(w, gain=1.0),
    'xavier_uniform': lambda w: torch.nn.init.xavier_uniform_(w, gain=1.0),
}


def epoch_seed(shuffle, generator=None):
    """The DataLoader's RNG protocol for one epoch (torch/utils/data/dataloader.py:706-710 draws ``_base_seed``;
    sampler.py RandomSampler.__iter__ draws the seed of a private generator).  Consumes the global torch RNG exactly as
    iterating the loader would.  -> the RandomSampler's seed, or None without shuffling."""
    torch.empty((), dtype=torch.int64).random_(generator=generator)           # _base_seed (discarded)
    if not shuffle:
        return None
    return int(torch.empty((), dtype=torch.int64).random_().item())


def epoch_permutation(n, shuffle, generator=None, seed=None):
    """Index order of one DataLoader epoch: ``torch.randperm(n, generator)`` of a private generator seeded as
    RandomSampler.__iter__ seeds it (``seed`` given: already drawn with epoch_seed)."""
    if seed is None:
        seed = epoch_seed(shuffle, generator)
    if not shuffle or seed is None:
        return None
    g = torch.Generator()
    g.manual_seed(seed)
    return torch.randperm(n, generator=g)


def loader_plan(train_loader, rows_ok=lambda data: data.ndim == 2 and data.shape[1] == 3):
    """Decode a DataLoader into (rows ndarray, batch_size, shuffle, drop_last, generator), or None when it is not the
    plain ``DataLoader(BasicDataset(int[T,3]), batch_size, shuffle)`` of run_examples/test.py:93-94 -- or another dataset whose
    ``.data`` passes ``rows_ok`` -- (then fit() falls back to iterating it batch by batch)."""
    ds = getattr(train_loader, 'dataset', None)
    data = getattr(ds, 'data', None)
    bs = getattr(train_loader, 'batch_size', None)
    if not isinstance(data, np.ndarray) or not rows_ok(data) or bs is None:
        return None
    sampler = getattr(train_loader, 'sampler', None)
    if not isinstance(getattr(train_loader, 'batch_sampler', None), BatchSampler):
        return None
    if isinstance(sampler, RandomSampler) and not sampler.replacement and sampler._num_samples is None:
        shuffle, gen = True, sampler.generator
    elif isinstance(sampler, SequentialSampler):
        shuffle, gen = False, None
    else:
        return None
    if gen is not None:
        return None
    return data, int(bs), shuffle, bool(train_loader.drop_last), train_loader.generator


class AbstractRecommender(object):
    def __init__(self):
        self.optimizer = None
        self.initializer = None
        self.loss_type = None
        self.lr = 0.01
        self.logger = None
        self.training = False

    # -- reference surface (AbstractRecommender.py:33-46)
    def calc_loss(self, batch):
        raise NotImplementedError

    def fit(self, train_loader):
        raise NotImplementedError

    def rank(self, test_loader):
        raise NotImplementedError

    def full_rank(self, u):
        raise NotImplementedError

    def predict(self, u, i):
        raise NotImplementedError

    # -- nn.Module look-alikes used by drivers
    def train(self, mode=True):
        self.training = mode
        return self

    def eval(self):
        return self.train(False)

    SUPPORTED_OPTIMIZERS = ('sgd', 'adam')

    def _optimizer_name(self):
        """AbstractRecommender.py:48-67: unknown names fall back to Adam with a log line."""
        name = str(self.optimizer).lower()
        if name in self.SUPPORTED_OPTIMIZERS:
            return name
        if name == 'sparse_adam':       # what optim.SparseAdam.step() raises on nn.Embedding's dense gradients (:61-62)
            raise RuntimeError('SparseAdam does not support dense gradients, please consider Adam instead')
        if name in ('adagrad', 'rmsprop'):
            raise NotImplementedError(f"optimizer '{name}' is outside the GPU hot path of {type(self).__name__} "
                                      f"(native: {', '.join(self.SUPPORTED_OPTIMIZERS)})")
        if self.logger is not None:
            self.logger.info('Received unrecognized optimizer, set default Adam optimizer')
        return 'adam'

    SUPPORTED_LOSSES = ('BPR',)

    def _check_loss_type(self):
        lt = str(self.loss_type).upper()
        if lt in self.SUPPORTED_LOSSES:
            return
        if lt in ('CL', 'SL', 'HL', 'TL', 'BPR'):
            raise NotImplementedError(f"loss_type '{lt}' is outside the GPU hot path of {type(self).__name__} "
                                      f"(native: {', '.join(self.SUPPORTED_LOSSES)})")
        raise NotImplementedError(f'Invalid loss type: {self.loss_type}...')


def packed_bias(user_num, item_num, device):
    """FM's first-order terms as ONE device vector [u_bias (U), i_bias (I), bias_ (1)], zeroed as the reference's _init_weight
    leaves them -> (vector, u_bias table, i_bias table, bias_ view); the three are views of the vector."""
    bias = torch.zeros(user_num + item_num + 1, dtype=torch.float32, device=device)
    return (bias, _Table(bias[:user_num].view(user_num, 1)), _Table(bias[user_num:user_num + item_num].view(item_num, 1)),
            bias[user_num + item_num:])


def ragged_split(n, batch, first, n_steps):
    """Steps [first, first + n_steps) over n rows in batches of ``batch`` -> (full, last): ``full`` steps of whole batches, then,
    when the last of them is ragged, one step of ``last`` rows (else last = 0).  Host-drawn dropout masks are sized per step,
    so the ragged batch gets its own masks and launch."""
    full = n_steps if (first + n_steps) * batch <= n else n_steps - 1
    return full, (n - (first + full) * batch if full < n_steps else 0)


class DeviceRecommender(AbstractRecommender):
    """What every GPU-path model shares, trained or not: the device set-up of the reference's GeneralRecommender
    (AbstractRecommender.py:96-101), the multi-GPU policy, the caller-id range checks and the test-loader decoder."""
    MULTI_GPU = '{} runs as independent replicas only (DESIGN.md, multi-GPU section)'   # None: the class shards under torchrun

    def __init__(self, config):
        super().__init__()
        gpu = str(config.get('gpu', '') or '')
        if gpu and not torch.cuda.is_initialized() and 'LOCAL_RANK' not in os.environ:
            os.environ['CUDA_VISIBLE_DEVICES'] = gpu             # AbstractRecommender.py:99
        ops.require_cuda()
        local = int(os.environ.get('LOCAL_RANK', torch.cuda.current_device()))
        self.device = torch.device('cuda', local if local < torch.cuda.device_count() else 0)
        torch.cuda.set_device(self.device)
        self.logger = config['logger']
        # one process per GPU (torchrun): user-sharded training / ranking, see daisyrec_b200/parallel.py
        import torch.distributed as dist
        self.world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        self.rank_id = dist.get_rank() if self.world > 1 else 0
        if self.world > 1 and self.MULTI_GPU is not None:
            raise NotImplementedError(self.MULTI_GPU.format(type(self).__name__))

    # ------------------------------------------------------------------ caller ids
    def _check_ids(self, cols, bounds, names):
        """nn.Embedding's IndexError when a column of caller ids leaves [0, bounds[c]): the kernels index raw tables.  Host
        columns are checked on the host (no device sync), device columns in one ops.check_index_range launch."""
        dev = []
        for ids, hi, what in zip(cols, bounds, names):
            t = torch.as_tensor(ids)
            if t.is_cuda:
                dev.append((t.reshape(-1).to(torch.int64), hi, what))
            elif t.numel():
                h = t.reshape(-1).to(torch.int64)
                bad = int(((h < 0) | (h >= hi)).sum())
                if bad:
                    raise IndexError(f"index out of range in self: {bad} {what} id(s) outside [0, {int(hi)})")
        if dev:
            ids, bounds, names = zip(*dev)
            ops.check_index_range(torch.stack(ids, 1).contiguous(), bounds, names)

    def _rank_inputs(self, test_loader):
        """The test loader's (users int64 [n], candidates int64 [n, C], topk) on the host, range-checked; None when it is
        empty.  Reads ``dataset.data`` of a CandidatesDataset loader in bulk, else iterates (us, cands_ids) batches."""
        data = getattr(getattr(test_loader, 'dataset', None), 'data', None)
        if isinstance(data, (list, tuple)) and len(data) and len(data[0]) == 2:
            users = np.fromiter((int(r[0]) for r in data), np.int64, len(data))
            cands = np.stack([np.asarray(r[1], dtype=np.int64) for r in data])
        else:
            us, cs = [], []
            for b_us, b_c in test_loader:
                us.append(torch.as_tensor(b_us).reshape(-1).to(torch.int64))
                cs.append(torch.as_tensor(b_c).to(torch.int64).reshape(us[-1].numel(), -1))
            if not us:
                return None
            users, cands = torch.cat(us).numpy(), torch.cat(cs).numpy()
        if len(users) == 0:
            return None
        self._check_ids((users, cands), (self.user_num, self.item_num), ('test user', 'candidate item'))
        return users, np.ascontiguousarray(cands), min(self.topk, cands.shape[1])


class NeighbourScorer(DeviceRecommender):
    """The neighbourhood models whose prediction is a product with W kept as at most ``maxk`` neighbours per column
    (ops.KnnNeighbours): ItemKNNCF and SLiM (X W), and UserKNNCF (W X, through ``_scoring``).  Subclasses set ``self._X`` (ops.EaseX), ``self._W`` and ``self._w_host = None`` in ``fit``.  Entries of
    X W are summed on demand in fp64 over ascending neighbour ids, the order scipy's product adds in; the product itself is not
    materialised."""

    def _neighbour_csc(self, n=None):
        """W as scipy csc_matrix float32 [n, n] (n: item_num unless given), column c holding the neighbours of c (None before
        fit)."""
        if self._W is None:
            return None
        import scipy.sparse as sp
        n = self.item_num if n is None else n
        cnt = self._W.cnt.cpu().numpy().astype(np.int64)
        keep = np.arange(self._W.maxk)[None, :] < cnt[:, None]
        return sp.csc_matrix((self._W.val.cpu().numpy()[keep], self._W.idx.cpu().numpy()[keep],
                              np.concatenate([[0], np.cumsum(cnt)])), shape=(n, n))

    def _scoring(self):
        """(the neighbour structure, rank op, full_rank op, predict op) the scoring methods call: W's forward lists with the
        ItemKNN scoring kernels; UserKNNCF, whose product sums over reverse neighbours, supplies its own."""
        return self._W, ops.itemknn_rank, ops.itemknn_full_rank, ops.itemknn_predict

    def _predict_score(self, u, i):
        us, its = self._ids((u,), (i,))
        nb, _, _, predict = self._scoring()
        return np.float64(predict(self._X, nb, us, its).item())

    def rank(self, test_loader):
        """-> int64 ndarray [n_test_users, topk] of candidate ids by (X W)[u, c], ties by candidate position; None for an empty
        loader."""
        ins = self._rank_inputs(test_loader)
        if ins is None:
            return None
        users, cands, k = ins
        self._ids(())
        nb, rank, _, _ = self._scoring()
        return rank(self._X, nb, torch.from_numpy(users).to(self.device), torch.from_numpy(cands).to(self.device), k).cpu().numpy()

    def full_rank(self, u):
        """-> int64 ndarray [topk] of the top items of user u; no masking of train items."""
        users = self._ids((u,))[0]
        nb, _, full_rank, _ = self._scoring()
        return full_rank(self._X, nb, users, min(self.topk, self.item_num))[0].cpu().numpy()

    def _ids(self, users, items=None):
        if self._W is None:
            raise RuntimeError(f'{type(self).__name__}: fit() must run before scoring')
        cols, bounds, names = [users], [self.user_num], ['user']
        if items is not None:
            cols, bounds, names = cols + [items], bounds + [self.item_num], names + ['item']
        self._check_ids(cols, bounds, names)
        return [torch.as_tensor(np.asarray(c, dtype=np.int64)).reshape(-1).to(self.device) for c in cols]


class GeneralRecommender(DeviceRecommender):
    """Shared plumbing of the trained GPU-path models.  A subclass declares its defaults and state as class data, builds its
    tables in ``__init__`` and supplies ``_workspace(opt, rows)`` and ``_launch(bu, bi, bj, batch, first, n_steps, apply)``."""
    DEFAULT_OPTIMIZER = 'sgd'                   # config['optimizer'] == 'default'
    DEFAULT_INIT = 'normal'                     # config['init_method'] == 'default'
    LOSS_TYPE = None                            # a fixed, unregularised loss: loss_type, reg_1 and reg_2 are not read
    PARAMS = ('embed_user.weight', 'embed_item.weight')     # parameters() in order; attribute paths
    BUFFERS = ()                                # in state_dict() after PARAMS, not in parameters()
    STRICT_STATE = True                         # load_state_dict: every key of state_dict() must be given
    SCRATCH_KEY = None                          # config key of the row count of a batch-sized scratch (built at first step)

    def __init__(self, config):
        super().__init__(config)
        self.steps_per_launch = int(config.get('steps_per_launch', 0))   # 0 = whole epoch in one launch
        self.show_progress = bool(config.get('progress', True))
        # 'torch' (default): the DataLoader's own CPU permutation -> the reference's batches bit for bit;
        # 'device': torch.randperm on the GPU seeded from the global RNG (same distribution, no 8-byte/triple H2D)
        self.shuffle_engine = str(config.get('shuffle_engine', DEFAULT_SHUFFLE_ENGINE))
        # the reference's common keys (e.g. MFRecommender.py:46-59)
        self.lr, self.epochs, self.topk = config['lr'], config['epochs'], config['topk']
        self.user_num, self.item_num, self.factors = config['user_num'], config['item_num'], config['factors']
        if self.LOSS_TYPE is None:
            self.loss_type, self.reg_1, self.reg_2 = config['loss_type'], config['reg_1'], config['reg_2']
        else:
            self.loss_type, self.reg_1, self.reg_2 = self.LOSS_TYPE, 0., 0.
        self.optimizer = config['optimizer'] if config['optimizer'] != 'default' else self.DEFAULT_OPTIMIZER
        self.initializer = config['init_method'] if config['init_method'] != 'default' else self.DEFAULT_INIT
        self.early_stop = config['early_stop']
        if self.SCRATCH_KEY is not None:
            self._rows = int(config.get(self.SCRATCH_KEY, 1 << 16))
        self._hp = self._ws = None
        self._opt_steps = 0

    # ------------------------------------------------------------------ state
    def state_dict(self):
        return {k: functools.reduce(getattr, k.split('.'), self) for k in self.PARAMS + self.BUFFERS}

    def parameters(self):
        sd = self.state_dict()
        return [sd[k] for k in self.PARAMS]

    def load_state_dict(self, sd):
        for k, t in self.state_dict().items():
            if self.STRICT_STATE or k in sd:
                t.copy_(torch.as_tensor(sd[k]).reshape(t.shape))
        self._drop_cache()

    def _drop_cache(self):
        """Forget whatever was computed from the parameters (the graph models' propagated tables)."""

    def to(self, device):
        return self

    # ------------------------------------------------------------------ steps
    def _hyper(self, opt=None):
        opt = opt or self._optimizer_name()
        if self.SUPPORTED_LOSSES == ('BPR',):                     # the BPR-only steps take the default loss kind
            return ops.hyper(self.lr, self.reg_1, self.reg_2, opt)
        return ops.hyper(self.lr, self.reg_1, self.reg_2, opt, loss=str(self.loss_type).upper())

    def _begin_fit(self, opt):
        """fit() builds a fresh optimizer (AbstractRecommender.py:105): fresh optimiser state and step count.  A batch-sized
        scratch waits for the first step, which knows the batch size."""
        self._hp = self._hyper(opt)
        self._opt_steps = 0
        self._fit_opt = opt
        self._ws = None if self.SCRATCH_KEY is not None else self._workspace(opt)

    def _ensure(self, rows=0):
        """Optimiser state and scratch for a step of ``rows`` scratch rows; a step outside fit() starts a fresh optimiser."""
        if self._hp is None:
            self._begin_fit(self._optimizer_name())
        if self.SCRATCH_KEY is None:
            return
        rows = max(int(rows), self._rows)
        if self._ws is None:
            self._ws = self._workspace(self._fit_opt, rows)
        elif self._ws.max_rows < rows:
            # growing the scratch would drop the optimiser state: size it up front instead
            raise RuntimeError(f'{type(self).__name__} scratch too small; set config["{self.SCRATCH_KEY}"] >= 2 * batch_size')

    def _train_steps(self, bu, bi, bj, batch, first, n_steps):
        self._ensure(2 * batch)
        losses = self._launch(bu, bi, bj, batch, first, n_steps, apply=True)
        self._opt_steps += n_steps
        return losses

    def calc_loss(self, batch):
        """0-d fp32 loss of one (user, pos, neg) -- or (user, item, label) -- batch; no update."""
        self._check_loss_type()
        bu, bi, bj = self._batch_ids(batch)
        self._ensure(2 * bu.numel())
        return self._launch(bu, bi, bj, bu.numel(), 0, 1, apply=False).to(torch.float32).reshape(())

    def train_step(self, batch):
        """zero_grad + calc_loss + backward + optimizer.step on one batch, in train mode (AbstractRecommender.py:119-128)
        -> loss.item()."""
        self._check_loss_type()
        bu, bi, bj = self._batch_ids(batch)
        self._ensure(2 * bu.numel())
        was = self.training
        self.train()
        try:
            return float(self._train_steps(bu, bi, bj, bu.numel(), 0, 1).item())
        finally:
            self.train(was)

    # ------------------------------------------------------------------ caller ids
    def _device_ids(self, cols, bounds, names, dtype=torch.int32):
        """Range-checked caller ids -> one contiguous 1-D device tensor of ``dtype`` per column."""
        self._check_ids(cols, bounds, names)
        return [torch.as_tensor(c).to(self.device, dtype).reshape(-1).contiguous() for c in cols]

    def _batch_ids(self, batch):
        return self._device_ids(batch[:3], *self._index_bounds())

    def _pair_ids(self, user, item, dtype=torch.int32):
        return self._device_ids((user, item), (self.user_num, self.item_num), ('user', 'item'), dtype)

    # ------------------------------------------------------------------ ranking
    def _dot_tables(self):
        """(P, Q) of the dot-product scorers (MF's rank kernels)."""
        return self.embed_user.weight, self.embed_item.weight

    def _pair_scores(self, user, item):
        """pred = (P[user] * Q[item]).sum(-1) for index tensors (MFRecommender.py:63-68)."""
        u, i = self._pair_ids(user, item)
        return ops.mf_predict(*self._dot_tables(), u, i)

    def forward(self, user, item):
        return self._pair_scores(user, item)

    def __call__(self, *args):
        return self.forward(*args)

    def predict(self, u, i):
        """-> python float (MFRecommender.py:99-104)."""
        return float(self._pair_scores([u], [i]).item())

    def rank(self, test_loader):
        """-> float32 ndarray [n_test_users, topk] of the top candidates, rows in loader order (MFRecommender.py:106-123)."""
        P, Q = self._dot_tables()
        ins = self._rank_inputs(test_loader)
        if ins is None:
            return np.zeros((0,), np.float32)
        users, cands, k = ins
        return ops.mf_rank(P, Q, torch.from_numpy(users).to(self.device), torch.from_numpy(cands).to(self.device), k).cpu().numpy()

    def full_rank(self, u):
        """-> int64 ndarray [topk] of the top items of user u; no masking of train items (MFRecommender.py:126-133)."""
        P, Q = self._dot_tables()
        users = self._device_ids(([int(u)],), (self.user_num,), ('user',), torch.int64)[0]
        return ops.mf_full_rank(P, Q, users, min(self.topk, self.item_num))[0].cpu().numpy()

    def _loader_plan(self, train_loader):
        return loader_plan(train_loader)

    def fit(self, train_loader):
        self._check_loss_type()
        opt = self._optimizer_name()
        self._begin_fit(opt)
        plan = self._loader_plan(train_loader)
        last_loss = 0.
        for epoch in range(1, self.epochs + 1):
            self.train()
            if plan is not None and self.world > 1:
                current_loss = self._fit_epoch_sharded(plan, epoch)
            elif plan is not None:
                current_loss = self._fit_epoch_bulk(plan, epoch)
            else:
                current_loss = self._fit_epoch_generic(train_loader, epoch)
            self.eval()
            delta_loss = float(current_loss - last_loss)
            if (abs(delta_loss) < 1e-5) and self.early_stop:
                self.logger.info('Satisfy early stop mechanism')
                break
            else:
                last_loss = current_loss

    def _fit_epoch_bulk(self, plan, epoch):
        data, bs, shuffle, drop_last, gen = plan
        T = data.shape[0]
        # the epoch's order is computed on a side stream while the rows upload (first epoch) / are stamped: the one-CTA
        # MT19937 stream leaves the copy engines and 147 SMs free
        exact_on_device = shuffle and self.shuffle_engine == 'torch' and T < RANDPERM_DEVICE_MAX
        if exact_on_device:
            # buffers are allocated on the main stream and kept for the model's lifetime (no cross-stream allocator traffic)
            if getattr(self, '_perm_bufs', None) is None or self._perm_bufs[0].numel() < T:
                self._perm_bufs = ops.randperm_workspace(T, self.device)
            main = torch.cuda.current_stream(self.device)
            if getattr(self, '_side_stream', None) is None:
                self._side_stream = torch.cuda.Stream(self.device)
            self._side_stream.wait_stream(main)
            with torch.cuda.stream(self._side_stream):
                d_perm = self._device_permutation(T, shuffle, gen)
            d_triples = self._device_triples(data)
            main.wait_stream(self._side_stream)
        else:
            d_triples = self._device_triples(data)
            d_perm = self._device_permutation(T, shuffle, gen)
        bu, bi, bj = ops.gather_triples(d_triples, d_perm)
        n_use = (T // bs) * bs if drop_last else T
        nsteps = (n_use + bs - 1) // bs
        if n_use != T:
            bu, bi, bj = bu[:n_use], bi[:n_use], bj[:n_use]
        chunk = self.steps_per_launch if self.steps_per_launch > 0 else nsteps
        pbar = tqdm(total=nsteps, disable=not self.show_progress)
        pbar.set_description(f'[Epoch {epoch:03d}]')
        current_loss = 0.
        for first in range(0, nsteps, chunk):
            k = min(chunk, nsteps - first)
            losses = self._train_steps(bu, bi, bj, bs, first, k)           # raises ValueError on NaN
            current_loss += float(losses.sum().item())
            pbar.update(k)
        pbar.set_postfix(loss=current_loss)
        pbar.close()
        return current_loss

    def _device_permutation(self, T, shuffle, gen, seed=None):
        """The epoch's index order as a device int64 tensor (None = sequential); consumes the global RNG like the DataLoader."""
        if seed is None:
            seed = epoch_seed(shuffle, gen)
        if not shuffle:
            return None
        if self.shuffle_engine == 'device':
            g = torch.Generator(device=self.device)
            g.manual_seed(seed)
            return torch.randperm(T, generator=g, device=self.device)
        if self.shuffle_engine == 'torch' and T < RANDPERM_DEVICE_MAX:
            return ops.randperm_torch(seed, T, self.device, out=getattr(self, '_perm_bufs', None))
        return epoch_permutation(T, shuffle, gen, seed=seed).to(self.device, non_blocking=False)

    def _device_triples(self, data):
        """Device copy of the loader's [T,3] rows: the sampler's own device twin when the host array still carries the stamp
        it was attached with, else an upload cached per (array, stamp) -- an in-place edit of the host rows re-uploads."""
        stamp = fingerprint(data)
        d_triples = getattr(data, '_drb_device', None)
        if not (d_triples is not None and d_triples.device == self.device and getattr(data, '_drb_stamp', None) == stamp):
            if getattr(self, '_triples_key', None) != (id(data), stamp):
                host = np.ascontiguousarray(data, dtype=np.int32)
                self._triples_dev = torch.from_numpy(host if host.flags.writeable else host.copy()).to(self.device)
                self._triples_key = (id(data), stamp)
            d_triples = self._triples_dev
        if d_triples.is_cuda and getattr(self, '_range_ok', None) != (id(data), stamp):
            # nn.Embedding's IndexError (the kernels index raw tables): one pass over the ids per uploaded array
            ops.check_index_range(d_triples, *self._index_bounds())
            self._range_ok = (id(data), stamp)
        return d_triples

    def _index_bounds(self):
        """(upper bounds, names) of the three columns of the loader's rows."""
        pointwise = str(self.loss_type).upper() in ('CL', 'SL')
        return ((self.user_num, self.item_num, (1 << 62) if pointwise else self.item_num),
                ('user', 'item', 'label' if pointwise else 'negative item'))

    def _fit_epoch_sharded(self, plan, epoch):
        """N > 1: same global batches as the single-GPU run; this rank trains the triples of its users."""
        data, bs, shuffle, drop_last, gen = plan
        T = data.shape[0]
        d_triples = self._device_triples(data)
        trainer = self._sharded_trainer(d_triples)
        # every rank advances its own RNG as the DataLoader would, but rank 0's seed decides the epoch's order: the ranks
        # keep disjoint shares of ONE permutation whatever their RNG histories were
        from ..parallel import broadcast_int
        seed = epoch_seed(shuffle, gen)
        if shuffle:
            seed = broadcast_int(seed, self.device)
        d_perm = self._device_permutation(T, shuffle, gen, seed=seed if shuffle else 0)
        nsteps = trainer.prepare_epoch(d_triples, d_perm, bs)
        if drop_last and T % bs:
            nsteps -= 1
        pbar = tqdm(total=nsteps, disable=not self.show_progress or self.rank_id != 0)
        pbar.set_description(f'[Epoch {epoch:03d}]')
        losses = trainer.train_steps(0, nsteps)
        trainer.check_nan()
        current_loss = float(losses.sum().item())
        pbar.update(nsteps)
        pbar.set_postfix(loss=current_loss)
        pbar.close()
        return current_loss

    def _fit_epoch_generic(self, train_loader, epoch):
        """Any other iterable of (user, pos, neg) batches: one end-to-end step per batch."""
        current_loss = 0.
        pbar = tqdm(train_loader, disable=not self.show_progress)
        pbar.set_description(f'[Epoch {epoch:03d}]')
        for batch in pbar:
            current_loss += self.train_step(batch)
        pbar.set_postfix(loss=current_loss)
        return current_loss
