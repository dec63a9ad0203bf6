"""fp64 reference of ColBERT late interaction (colbert.modeling): transformers.BertModel with ColBERT's attention mask (the
query's [MASK] rows are no keys unless attend_to_mask_tokens), the projection W h without bias, x / max(|x|, 1e-12) per token
row, and MaxSim = sum over query rows of the max over kept passage rows.  Also the fp32 twin (the yardstick) and a bf16
autocast one (the fp16 mode's bar); and maxsim_kernel's own fp32 arithmetic restated (maxsim_fp32_order), which K5's scores
equal bit for bit given K5's token vectors.  Test infrastructure only."""
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
        self._hidden = {}                 # (model, ids, keys, autocast) -> last_hidden_state, shared by with_weight

    def with_weight(self, weight):
        """the same encoder under another projection; the last hidden states computed so far are shared, so a dim sweep
        runs each encoder forward once"""
        import torch
        o = copy.copy(self)
        o.w64 = torch.from_numpy(np.asarray(weight, np.float64))
        o.w32 = o.w64.float()
        return o

    def _vectors(self, m, w, ids, keys, autocast=False):
        import torch
        ids = np.asarray(ids, np.int64)
        mask = (np.arange(len(ids)) < keys).astype(np.int64)
        key = (id(m), ids.tobytes(), int(keys), autocast)
        with torch.no_grad(), torch.autocast("cpu", dtype=torch.bfloat16, enabled=autocast):
            h = self._hidden.get(key)
            if h is None:
                h = self._hidden[key] = m(input_ids=torch.tensor(ids[None]), attention_mask=torch.tensor(mask[None])).last_hidden_state[0]
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


# ------------------------------------------------------------------------------------ maxsim_kernel's fp32 order
def exact_fmaf_available():
    """fmaf below is exact up to double rounding only with a 64-bit long double significand (x86's 80-bit format)"""
    return np.finfo(np.longdouble).nmant >= 63


def fmaf(a, b, c):
    """fp32 fmaf(a, b, c) elementwise, as float32(longdouble(a) * longdouble(b) + longdouble(c)): the product of two
    24-bit significands is exact in 64 bits, so the only departure from one rounding is the sum's double rounding, which
    can move a result only when the exact sum lies within 2^-40 of its ulp of an fp32 midpoint"""
    L = np.longdouble
    return (np.asarray(a, np.float32).astype(L) * np.asarray(b, np.float32).astype(L) + np.asarray(c, np.float32).astype(L)).astype(np.float32)


def maxsim_fp32_order(qv, dv, keep):
    """MaxSim in maxsim_kernel's arithmetic: for every (query row i, kept passage row j) one fmaf chain over k = 0 .. dim - 1
    from 0, the exact max over the kept rows, then one fp32 += of the q_rows maxima in row order.  Returns np.float32."""
    q = np.asarray(qv, np.float32)
    d = np.asarray(dv, np.float32)[np.asarray(keep, bool)]
    acc = np.zeros((len(q), len(d)), np.float32)
    for k in range(q.shape[1]):
        acc = fmaf(q[:, k, None], d[None, :, k], acc)
    s = np.float32(0.0)
    for m in acc.max(axis=1):
        s = np.float32(s + m)
    return s


def selection(scores, top_k):
    """krag_late_rerank's order of one query's pair scores: descending, the lower position first among equal scores;
    (positions int32 [top_k], scores float32 [top_k]) with -1 / NaN past the pair count"""
    scores = np.asarray(scores, np.float32)
    n = min(len(scores), top_k)
    pos = np.full(top_k, -1, np.int32)
    sc = np.full(top_k, np.nan, np.float32)
    order = np.lexsort((np.arange(len(scores)), -scores.astype(np.float64)))[:n]
    pos[:n] = order
    sc[:n] = scores[order]
    return pos, sc
