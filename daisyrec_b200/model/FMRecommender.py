"""FM on the GPU path, with the reference's class name, config keys and methods
(daisy/model/FMRecommender.py:16-131).

FM here is MF's factor product plus first-order terms: ``pred = <p_u, q_i> + (u_bias[u] + i_bias[i]) + bias_``
(:61-68); the regulariser covers the factor rows only (:76-95), so the step is the MF step kernel
(``csrc/mf_bpr.cu``, GEN instantiation) with three extra scalar loads per score, three scalar ``RED``s per triple
and a sweep over the ``U + I + 1`` bias scalars in phase 2.  The biases live in ONE packed device vector
``[u_bias (U), i_bias (I), bias_ (1)]``; ``u_bias.weight`` / ``i_bias.weight`` / ``bias_`` are views of it.

    fit -> drb_gather_triples + drb_fm_train_steps     calc_loss -> drb_fm_train_steps(apply=0)
    rank -> drb_fm_rank     full_rank -> drb_fm_full_rank     predict / forward -> drb_fm_predict
"""
import numpy as np
import torch

from .. import ops
from .AbstractRecommender import GeneralRecommender, _Table, _init_table, _INIT, packed_bias


class FM(GeneralRecommender):
    SUPPORTED_LOSSES = ('BPR', 'HL', 'TL', 'CL', 'SL')               # AbstractRecommender.py:79-88
    SUPPORTED_OPTIMIZERS = ('sgd', 'adam', 'adagrad', 'rmsprop')     # AbstractRecommender.py:53-60
    MULTI_GPU = 'FM runs as independent replicas only (the sharded step covers MF)'
    PARAMS = ('embed_user.weight', 'embed_item.weight', 'u_bias.weight', 'i_bias.weight', 'bias_')

    def __init__(self, config):
        """Same keys as the reference (FMRecommender.py:38-56): epochs, lr, reg_1, reg_2, user_num, item_num, factors,
        loss_type, optimizer ('default' -> sgd), init_method ('default' -> normal), early_stop, topk (+ gpu, logger)."""
        super().__init__(config)
        # The reference's CPU RNG consumption (:43-59): four nn.Embedding constructors (N(0,1) each, in this order), then
        # self.apply(_init_weight) re-initialises all four in registration order, then the two bias tables are zeroed.
        U, I, F = self.user_num, self.item_num, self.factors
        wu, wi = _init_table(U, F, None), _init_table(I, F, None)
        bu_, bi_ = _init_table(U, 1, None), _init_table(I, 1, None)
        for w in (wu, wi, bu_, bi_):
            _INIT[self.initializer](w)
        self.embed_user = _Table(wu.to(self.device))
        self.embed_item = _Table(wi.to(self.device))
        self.bias, self.u_bias, self.i_bias, self.bias_ = packed_bias(U, I, self.device)

    def _workspace(self, opt, rows=None):
        return ops.FMWorkspace(self.user_num, self.item_num, self.factors, opt, self.device)

    def _launch(self, bu, bi, bj, batch, first, n_steps, apply=True):
        return ops.fm_train_steps(self.embed_user.weight, self.embed_item.weight, self.bias, self._ws, bu, bi, bj, max(1, batch),
                                  first, n_steps, self._hp, adam_step0=self._opt_steps, apply=apply)

    # ------------------------------------------------------------------ reference surface (FMRecommender.py:61-131)
    def _pair_scores(self, user, item):
        u, i = self._pair_ids(user, item)
        return ops.fm_predict(self.embed_user.weight, self.embed_item.weight, self.bias, u, i)

    def rank(self, test_loader):
        ins = self._rank_inputs(test_loader)
        if ins is None:
            return np.zeros((0,), np.float32)
        users, cands, k = ins
        return ops.fm_rank(self.embed_user.weight, self.embed_item.weight, self.bias, torch.from_numpy(users).to(self.device),
                           torch.from_numpy(cands).to(self.device), k).cpu().numpy()

    def full_rank(self, u):
        users = self._device_ids(([int(u)],), (self.user_num,), ('user',), torch.int64)[0]
        k = min(self.topk, self.item_num)
        return ops.fm_full_rank(self.embed_user.weight, self.embed_item.weight, self.bias, users, k)[0].cpu().numpy()
