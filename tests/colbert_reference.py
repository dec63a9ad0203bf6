"""fp64 reference of ColBERT late interaction (colbert.modeling): transformers.BertModel with ColBERT's attention mask (the
query's [MASK] rows are no keys unless attend_to_mask_tokens), the projection W h without bias, x / max(|x|, 1e-12) per token
row, and MaxSim = sum over query rows of the max over kept passage rows.  Also the fp32 twin (the yardstick) and a bf16
autocast one (the fp16 mode's bar).  Test infrastructure only."""
import copy

import numpy as np


class Fp64ColBERT:
    def __init__(self, cfg, state, weight):
        import torch
        from transformers import BertConfig, BertModel
        from transformers.initialization import no_init_weights
        with no_init_weights():
            self.m64 = BertModel(BertConfig(**cfg, attn_implementation="eager"), add_pooling_layer=False).double().eval()
        missing, _ = self.m64.load_state_dict({k: torch.from_numpy(np.asarray(v, np.float64)) for k, v in state.items()}, strict=False)
        assert not missing, missing
        self.w64 = torch.from_numpy(np.asarray(weight, np.float64))
        self.m32, self.w32 = copy.deepcopy(self.m64).float(), self.w64.float()

    def _vectors(self, m, w, ids, keys, autocast=False):
        import torch
        ids = np.asarray(ids, np.int64)
        mask = (np.arange(len(ids)) < keys).astype(np.int64)
        with torch.no_grad(), torch.autocast("cpu", dtype=torch.bfloat16, enabled=autocast):
            h = m(input_ids=torch.tensor(ids[None]), attention_mask=torch.tensor(mask[None])).last_hidden_state[0]
            v = h @ w.T.to(h.dtype) if not autocast else torch.nn.functional.linear(h, w)
        v = v.double()
        return (v / v.norm(dim=1, keepdim=True).clamp_min(1e-12)).numpy()

    def vectors(self, ids, keys=None):
        """(fp64, fp32) unit token vectors of one sequence whose first `keys` rows are keys (None: all)"""
        k = len(ids) if keys is None else keys
        return self._vectors(self.m64, self.w64, ids, k), self._vectors(self.m32, self.w32, ids, k)

    def vectors_bf16(self, ids, keys=None):
        k = len(ids) if keys is None else keys
        return self._vectors(self.m32, self.w32, ids, k, autocast=True)


def maxsim(qv, dv, keep):
    """sum over query rows of the max over kept passage rows of q . d"""
    s = np.asarray(qv, np.float64) @ np.asarray(dv, np.float64)[np.asarray(keep, bool)].T
    return float(s.max(axis=1).sum())
