"""daisyrec_b200 -- H100-native (sm_90a) BPR training / ranking path behind daisyRec's plug-in API.

Drop-in surface (same names and call signatures as AmazingDD/daisyRec v2.3.0):
    daisyrec_b200.model.MFRecommender.MF                 <- daisy/model/MFRecommender.py
    daisyrec_b200.utils.sampler.BasicNegtiveSampler      <- daisy/utils/sampler.py
    daisyrec_b200.utils.dataset.{BasicDataset, CandidatesDataset, get_dataloader}
    daisyrec_b200.utils.utils.build_candidates_set       <- daisy/utils/utils.py
All compute runs in hand-written CUDA (daisyrec_b200/csrc) behind the C ABI of
include/daisyrec_b200.h; there is no CPU or PyTorch fallback.
"""
__version__ = "0.1.0"
