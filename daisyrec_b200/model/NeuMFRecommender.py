"""NeuMF + BPR on the GPU path, with the reference's class name, config keys and methods
(daisy/model/NeuMFRecommender.py:15-232; model_name 'NeuMF', 'GMF', 'MLP' and 'NeuMF-pre').

Four raw fp32 embedding tables (``embed_user_GMF/embed_item_GMF/embed_user_MLP/embed_item_MLP`` ``.weight``)
and the tower as one flat fp32 block (``tower``; per layer weight then bias, then predict weight and bias).
No nn.Module in the compute path, no autograd, no torch.optim: fit / calc_loss / rank / full_rank / predict
forward to ``drb_neumf_*`` (include/daisyrec_b200.h).  torch.nn is touched at construction time only, to
consume the global CPU RNG exactly as the reference's constructor does (bit-identical initial weights).
"""
import numpy as np
import torch

from .. import ops
from .AbstractRecommender import GeneralRecommender, _Table, _INIT, ragged_split


class NeuMF(GeneralRecommender):
    DEFAULT_OPTIMIZER, DEFAULT_INIT = 'adam', 'xavier_normal'
    PARAMS = ('embed_user_GMF.weight', 'embed_item_GMF.weight', 'embed_user_MLP.weight', 'embed_item_MLP.weight', 'tower')
    SCRATCH_KEY = 'neumf_scratch_rows'

    def __init__(self, config):
        super().__init__(config)
        self.dropout = config['dropout']
        self.model = config['model_name']
        self.num_layers = config['num_layers']
        if self.model not in ops.NEUMF_MODE:
            raise ValueError(f"model_name={self.model!r}: expected one of {sorted(ops.NEUMF_MODE)}")
        self._mode = ops.NEUMF_MODE[self.model]                       # 0 NeuMF / NeuMF-pre, 1 GMF, 2 MLP
        self.GMF_model = config.get('GMF_model', None)
        self.MLP_model = config.get('MLP_model', None)
        self.dropout = float(self.dropout or 0.0)
        if not (0.0 <= self.dropout < 1.0):
            raise ValueError(f'dropout must be in [0, 1), got {self.dropout}')
        if self.factors % 4 != 0:
            raise NotImplementedError('NeuMF on the GPU path needs factors to be a multiple of 4 (128-bit rows)')
        F, Ln = self.factors, self.num_layers
        D = F * (2 ** (Ln - 1))
        self.mlp_dim = D

        # ---- reference RNG stream (NeuMFRecommender.py:52-71 constructors, :81-96 _init_weight) on the CPU
        import torch.nn as nn
        embs = [nn.Embedding(self.user_num, F), nn.Embedding(self.item_num, F),
                nn.Embedding(self.user_num, D), nn.Embedding(self.item_num, D)]
        linears = [nn.Linear(F * (2 ** (Ln - i)), F * (2 ** (Ln - i)) // 2) for i in range(Ln)]
        predict = nn.Linear(F if self.model in ('MLP', 'GMF') else 2 * F, 1)          # :63-68
        init = _INIT[self.initializer]
        with torch.no_grad():
            if self.model != 'NeuMF-pre':
                for e in embs:
                    init(e.weight)
                bare = {'normal': torch.nn.init.normal_, 'uniform': torch.nn.init.uniform_,
                        'xavier_normal': torch.nn.init.xavier_normal_, 'xavier_uniform': torch.nn.init.xavier_uniform_}
                for lin in linears:
                    bare[self.initializer](lin.weight)  # :88-90 passes NO param config to the hidden layers: 'normal' is N(0, 1)
                init(predict.weight)
                for lin in linears + [predict]:
                    lin.bias.zero_()
            else:
                self._load_pretrained(embs, linears, predict)
            parts = []
            for lin in linears:
                parts += [lin.weight.reshape(-1), lin.bias.reshape(-1)]
            parts += [predict.weight.reshape(-1), predict.bias.reshape(-1)]
            tower = torch.cat(parts).contiguous()
        assert tower.numel() == ops.neumf_param_count(F, Ln, self._mode)
        self.embed_user_GMF = _Table(embs[0].weight.detach().to(self.device).contiguous())
        self.embed_item_GMF = _Table(embs[1].weight.detach().to(self.device).contiguous())
        self.embed_user_MLP = _Table(embs[2].weight.detach().to(self.device).contiguous())
        self.embed_item_MLP = _Table(embs[3].weight.detach().to(self.device).contiguous())
        self.tower = tower.to(self.device)
        # optional GPU-path key: 'fp32' (CUDA cores, parity path, default) | 'bf16' (wgmma tensor cores, BASELINE config 3)
        #                   | 'fused' (bf16 wgmma, the whole tower step of a 64-triple tile inside one CTA: activations stay in
        #                     shared memory, accumulators in registers; factors = 32, num_layers = 2, dropout 0 -- other shapes run as 'bf16')
        td = str(config.get('tower_dtype', 'fp32')).lower()
        if td not in ('fp32', 'bf16', 'fused'):
            raise ValueError(f"tower_dtype must be 'fp32', 'bf16' or 'fused', got {td!r}")
        self._tower_dtype = {'fp32': 0, 'bf16': 1, 'fused': 2}[td]
        # optional GPU-path key: how nn.Dropout's masks (:61) are produced in train mode.
        #   'torch'  : torch itself draws them on the host, in the reference's order (per step: the pos forward's L masks, then
        #              the neg forward's), from the global CPU generator; they are bit-packed and uploaded -- the reference's
        #              masks bit for bit.  Costs one host bernoulli_ per layer and forward: meant for small batches.
        #   'philox' : counter-based masks generated inside the kernels (same distribution, another stream).
        #   'auto'   : 'torch' while a step's masks stay under 4 M elements (the reference's default batch of 256 is 74 K),
        #              'philox' above (throughput).
        self.dropout_engine = str(config.get('dropout_engine', 'auto')).lower()
        if self.dropout_engine not in ('auto', 'torch', 'philox'):
            raise ValueError(f"dropout_engine must be 'auto', 'torch' or 'philox', got {self.dropout_engine!r}")

    def _load_pretrained(self, embs, linears, predict):
        """'NeuMF-pre' (NeuMFRecommender.py:97-116): tables and tower copied from config['GMF_model'] / config['MLP_model'];
        predict weight and bias as the reference leaves them -- :115 writes 0.5 * cat(w_gmf, w_mlp) into the weight and :116
        overwrites it with 0.5 * (b_gmf + b_mlp) broadcast over all 2F entries, while the bias keeps nn.Linear's own
        initial draw (mirrored: the quirk is what the reference trains from)."""
        g, m = self.GMF_model, self.MLP_model
        if g is None or m is None:
            raise ValueError("model_name='NeuMF-pre' needs config['GMF_model'] and config['MLP_model']")

        def cpu(t):
            return torch.as_tensor(t).detach().to('cpu', torch.float32)

        def tower_parts(model):
            """(per-layer (weight, bias) list, predict weight [1, k], predict bias [1]) of a GPU-path NeuMF or an nn.Module one."""
            if hasattr(model, 'tower'):
                flat, F, Ln = cpu(model.tower), model.factors, model.num_layers
                out, o = [], 0
                for i in range(Ln):
                    n_in = F * (2 ** (Ln - i))
                    w = flat[o:o + n_in * (n_in // 2)].view(n_in // 2, n_in); o += n_in * (n_in // 2)
                    b = flat[o:o + n_in // 2]; o += n_in // 2
                    out.append((w, b))
                pw = flat[o:-1].view(1, -1)
                return out, pw, flat[-1:]
            lins = [mod for mod in model.MLP_layers if isinstance(mod, torch.nn.Linear)]
            return [(cpu(l.weight), cpu(l.bias)) for l in lins], cpu(model.predict_layer.weight), cpu(model.predict_layer.bias)

        embs[0].weight.copy_(cpu(g.embed_user_GMF.weight)); embs[1].weight.copy_(cpu(g.embed_item_GMF.weight))
        embs[2].weight.copy_(cpu(m.embed_user_MLP.weight)); embs[3].weight.copy_(cpu(m.embed_item_MLP.weight))
        m_layers, m_pw, m_pb = tower_parts(m)
        _, g_pw, g_pb = tower_parts(g)
        for lin, (w, b) in zip(linears, m_layers):
            lin.weight.copy_(w); lin.bias.copy_(b)
        predict.weight.copy_(0.5 * torch.cat([g_pw, m_pw], dim=1))
        predict.weight.copy_((0.5 * (g_pb + m_pb)).expand_as(predict.weight))        # :116 (bias into weight)

    # ------------------------------------------------------------------ plumbing
    def _tabs(self):
        return (self.embed_user_GMF.weight, self.embed_item_GMF.weight, self.embed_user_MLP.weight,
                self.embed_item_MLP.weight)

    def _workspace(self, opt, rows):
        return ops.NeumfWorkspace(self.user_num, self.item_num, self.factors, self.num_layers, opt, rows, self.device)

    def _begin_fit(self, opt):
        self._philox_seed = None                                     # drawn lazily: the host-mask engine must not move the RNG here
        super()._begin_fit(opt)

    def _host_masks(self, rows_per_step):
        """Parity dropout: the keep-masks nn.Dropout would draw for steps of rows_per_step[k] triples, drawn by torch on the CPU
        generator in the reference's order and bit-packed (layout: drb_neumf_mask_words) -> int32 CUDA tensor."""
        F, Ln, keep = self.factors, self.num_layers, 1.0 - self.dropout
        widths = [F * (2 ** (Ln - i)) for i in range(Ln)]
        words = []
        for B in rows_per_step:
            per_layer = [[None, None] for _ in range(Ln)]
            for side in (0, 1):                                           # forward(user, pos) draws first, then forward(user, neg)
                for l, n in enumerate(widths):
                    per_layer[l][side] = torch.empty(B, n, dtype=torch.float32).bernoulli_(keep).numpy() != 0
            for l in range(Ln):
                bits = np.packbits(np.concatenate(per_layer[l]).reshape(-1), bitorder='little')
                pad = (-len(bits)) % 4
                words.append(np.pad(bits, (0, pad)).view(np.int32))
        return torch.from_numpy(np.concatenate(words)).to(self.device)

    def _drop_seed(self):
        """Key of the counter-based (Philox) masks: drawn from torch's global RNG the first time a fit needs it, so that
        torch.manual_seed makes runs reproducible."""
        if self.dropout <= 0.0 or not self.training or self._mode == 1:
            return 0                                                      # 'GMF' never calls a Dropout module: no draw at all
        if getattr(self, '_philox_seed', None) is None:
            self._philox_seed = int(torch.empty((), dtype=torch.int64).random_().item())
        return self._philox_seed

    def _use_host_masks(self, batch):
        if not self.training or self.dropout <= 0.0 or self._mode == 1:
            return False                                                  # 'GMF' never runs the tower: no Dropout is called
        if self.dropout_engine == 'auto':
            return 2 * batch * (4 * self.mlp_dim - 2 * self.factors) <= (1 << 22)
        return self.dropout_engine == 'torch'

    def _launch(self, bu, bi, bj, batch, first, n_steps, apply=True):
        kw = dict(apply=apply, tower_dtype=self._tower_dtype, dropout=self.dropout if self.training else 0.0, mode=self._mode)
        if not self._use_host_masks(batch):
            return ops.neumf_bpr_train_steps(self._tabs(), self.tower, self._ws, bu, bi, bj, batch, first, n_steps, self._hp,
                                             adam_step0=self._opt_steps, dropout_seed=self._drop_seed(), **kw)
        full, last = ragged_split(bu.numel(), batch, first, n_steps)
        out = []
        if full > 0:
            out.append(ops.neumf_bpr_train_steps(self._tabs(), self.tower, self._ws, bu, bi, bj, batch, first, full, self._hp,
                                                 adam_step0=self._opt_steps, drop_masks=self._host_masks([batch] * full), **kw))
        if last:
            base = (first + full) * batch
            out.append(ops.neumf_bpr_train_steps(self._tabs(), self.tower, self._ws, bu[base:], bi[base:], bj[base:], last, 0, 1,
                                                 self._hp, adam_step0=self._opt_steps + full, drop_masks=self._host_masks([last]),
                                                 **kw))
        return torch.cat(out)

    # ------------------------------------------------------------------ reference surface
    def _scores(self, users, items, per_user):
        self._ensure(1)
        return ops.neumf_scores(self._tabs(), self.tower, self._ws, users, items, per_user, self._tower_dtype, self._mode)

    def _pair_scores(self, user, item):
        u, i = self._pair_ids(user, item, torch.int64)
        return self._scores(u, i.reshape(-1, 1), 1).reshape(-1)

    def rank(self, test_loader):
        ins = self._rank_inputs(test_loader)
        if ins is None:
            return np.zeros((0,), np.float32)
        users, cands, k = ins
        d_cands = torch.from_numpy(cands).to(self.device)
        scores = self._scores(torch.from_numpy(users).to(self.device), d_cands, cands.shape[1])
        return ops.topk_from_scores(scores, d_cands, k).cpu().numpy()

    def full_rank(self, u):
        users = self._device_ids(([int(u)],), (self.user_num,), ('user',), torch.int64)[0]
        scores = self._scores(users, None, self.item_num)
        return ops.topk_from_scores(scores, None, min(self.topk, self.item_num))[0].cpu().numpy()
