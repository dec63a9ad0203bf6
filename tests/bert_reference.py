"""fp64 reference of the K5 forward (BERT encoder, CLS or mean pooling, L2 normalisation; the cross-encoder's pooler and
classifier head) and the yardstick its error is judged by.  Test infrastructure only.

K5 packs sequences without padding, so the reference runs transformers.BertModel in fp64 (eager attention) on each
sequence alone.  Sequences are independent, so a test checks a sample of a batch: `sample()` keeps the first and last
sequences and those that straddle a 128-row GEMM tile.  The same sample through torch fp32 gives the yardstick: K5 is held
to a multiple F of torch fp32's own distance from fp64.  Forward hooks record the largest |value| at every Linear input and
output, because K5 carries GEMM operands as split fp16 pairs, which saturate at 65504."""
import copy

import numpy as np

RANGE_LIMIT = 6.0e4        # split-fp16 operands saturate at 65504
TILE = 128                 # GEMM rows per tile


def random_state(cfg, seed):
    """BertModel weights (Hugging Face names) with non-trivial biases and LayerNorm parameters, so every term of the forward
    is exercised: embeddings N(0, 0.02), other matrices N(0, 0.06), biases N(0, 0.05), LayerNorm gamma N(1, 0.1)."""
    g = np.random.default_rng(seed)
    d, i, L = cfg["hidden_size"], cfg["intermediate_size"], cfg["num_hidden_layers"]
    n = lambda std, *s, mean=0.0: (mean + std * g.standard_normal(s, dtype=np.float32)).astype(np.float32)  # noqa: E731
    st = {"embeddings.word_embeddings.weight": n(0.02, cfg["vocab_size"], d),
          "embeddings.position_embeddings.weight": n(0.02, cfg.get("max_position_embeddings", 512), d),
          "embeddings.token_type_embeddings.weight": n(0.02, 2, d)}
    for ln in _ln_names(cfg):
        st[ln + ".weight"], st[ln + ".bias"] = n(0.1, d, mean=1.0), n(0.05, d)
    for l in range(L):
        p = f"encoder.layer.{l}."
        for nm, shape in (("attention.self.query", (d, d)), ("attention.self.key", (d, d)), ("attention.self.value", (d, d)),
                          ("attention.output.dense", (d, d)), ("intermediate.dense", (i, d)), ("output.dense", (d, i))):
            st[p + nm + ".weight"], st[p + nm + ".bias"] = n(0.06, *shape), n(0.05, shape[0])
    return st


def _ln_names(cfg):
    names = ["embeddings.LayerNorm"]
    for l in range(cfg["num_hidden_layers"]):
        names += [f"encoder.layer.{l}.attention.output.LayerNorm", f"encoder.layer.{l}.output.LayerNorm"]
    return names


def stressed_state(cfg, seed, score_std=12.0, n_outliers=3):
    """(state, its Fp64Bert): random_state with the two features that stress K5's arithmetic:
    - outlier hidden channels: every LayerNorm has gamma 10-20 on the same few channels, like the outlier features of
      trained BERTs, so the residual stream and every GEMM operand row mixes O(10) values with O(1) ones;
    - sharp attention: each layer's query and key weights are scaled so that the attention scores have a standard
      deviation of about `score_std`.  The softmax is then nearly one-hot, and the running maximum of the online
      softmax moves between key blocks, so its rescaling of the partial sums decides the result.
    The outlier channels dominate the LayerNorm statistics, so the score scale is measured, layer by layer on two
    calibration sequences, rather than derived: scaling Wq, bq, Wk, bk by c scales the layer's scores by c^2."""
    import torch
    st = random_state(cfg, seed)
    g = np.random.default_rng(seed + 1000)
    ch = g.choice(cfg["hidden_size"], n_outliers, replace=False)
    for nm in _ln_names(cfg):
        st[nm + ".weight"][ch] = g.uniform(10.0, 20.0, n_outliers).astype(np.float32)
    ref = Fp64Bert(cfg, st)
    calib = [g.integers(0, cfg["vocab_size"], 48) for _ in range(2)]
    for l in range(cfg["num_hidden_layers"]):
        c = np.sqrt(score_std / ref.attention_score_std(calib, l))
        att = ref.m64.encoder.layer[l].attention.self
        for n in ("query", "key"):
            for what in ("weight", "bias"):
                k = f"encoder.layer.{l}.attention.self.{n}.{what}"
                st[k] = (st[k] * c).astype(np.float32)
                with torch.no_grad():
                    getattr(getattr(att, n), what).copy_(torch.from_numpy(st[k].astype(np.float64)))
    return st, ref


def sample(lens, n, seed=0):
    """Indices of up to n sequences of a packed batch: the first and the last, up to half of n among those whose tokens
    straddle a 128-row tile boundary (evenly spread), the rest drawn at random."""
    B = len(lens)
    if B <= n:
        return np.arange(B)
    off = np.concatenate([[0], np.cumsum(lens)])
    straddle = [i for i in range(B) if off[i] // TILE != (off[i + 1] - 1) // TILE]
    pick = {0, B - 1}
    if straddle:
        pick.update(straddle[j] for j in np.linspace(0, len(straddle) - 1, min(len(straddle), n // 2)).astype(int))
    rest = np.setdiff1d(np.arange(B), sorted(pick))
    pick.update(np.random.default_rng(seed).choice(rest, n - len(pick), replace=False).tolist())
    return np.array(sorted(pick))


class Fp64Bert:
    """transformers.BertModel in fp64 with eager attention, and on request its fp32 twin (the yardstick)."""

    def __init__(self, cfg, state):
        import torch
        from transformers import BertConfig, BertModel
        from transformers.initialization import no_init_weights
        self.cfg = cfg
        with no_init_weights():                     # every parameter comes from `state`
            self.m64 = BertModel(BertConfig(**cfg, attn_implementation="eager"), add_pooling_layer=False).double().eval()
        missing, _ = self.m64.load_state_dict({k: torch.from_numpy(np.asarray(v, np.float64)) for k, v in state.items()}, strict=False)
        assert not missing, missing
        self._m32 = None
        self.range_max = 0.0          # largest |value| at any Linear input or output seen by the fp64 forwards
        for mod in self.m64.modules():
            if isinstance(mod, torch.nn.Linear):
                mod.register_forward_hook(self._record)

    def _record(self, mod, inp, out):
        self.range_max = max(self.range_max, float(inp[0].abs().max()), float(out.abs().max()))

    def _embed(self, m, token_lists):
        import torch
        out = []
        with torch.no_grad():
            for t in token_lists:
                h = m(input_ids=torch.tensor(np.asarray(t, np.int64)[None])).last_hidden_state[0, 0]
                out.append(torch.nn.functional.normalize(h, dim=0).double().numpy())
        return np.stack(out)

    def embed(self, token_lists):
        """CLS row, L2-normalised, of each sequence run alone in fp64"""
        return self._embed(self.m64, token_lists)

    def embed_fp32(self, token_lists):
        return self._embed(self._fp32(), token_lists)

    def _fp32(self):
        if self._m32 is None:
            self._m32 = copy.deepcopy(self.m64).float()
        return self._m32

    def pooled(self, token_lists):
        """(CLS fp64, mean fp64, CLS fp32, mean fp32, largest Linear operand of the fp64 forwards) of each sequence run
        alone: one forward per sequence and precision gives both poolings"""
        self.range_max = 0.0
        c64, m64 = _pools(self.m64, token_lists)
        c32, m32 = _pools(self._fp32(), token_lists)
        return c64, m64, c32, m32, self.range_max

    def embed_padded(self, token_lists):
        """fp64, all sequences in one zero-padded batch with an attention mask (checks that running them alone is the same)"""
        import torch
        L = max(len(t) for t in token_lists)
        ids = torch.zeros((len(token_lists), L), dtype=torch.int64)
        mask = torch.zeros((len(token_lists), L), dtype=torch.int64)
        for i, t in enumerate(token_lists):
            ids[i, :len(t)] = torch.as_tensor(np.asarray(t, np.int64)); mask[i, :len(t)] = 1
        with torch.no_grad():
            h = self.m64(input_ids=ids, attention_mask=mask).last_hidden_state[:, 0]
        return torch.nn.functional.normalize(h, dim=1).numpy()

    def attention_score_std(self, token_lists, layer=0):
        """standard deviation of the scaled attention scores q.k / sqrt(dh) of one layer over the given sequences"""
        import torch
        att = self.m64.encoder.layer[layer].attention.self
        heads = self.cfg["num_attention_heads"]
        got = {}
        hq = att.query.register_forward_hook(lambda m, i, o: got.__setitem__("q", o))
        hk = att.key.register_forward_hook(lambda m, i, o: got.__setitem__("k", o))
        scores = []
        enc = self.m64.encoder
        layers, enc.layer = enc.layer, enc.layer[:layer + 1]      # the layers above do not change this one's input
        try:
            with torch.no_grad():
                for t in token_lists:
                    self.m64(input_ids=torch.tensor(np.asarray(t, np.int64)[None]))
                    q, k = (got[n][0].view(len(t), heads, -1).transpose(0, 1) for n in ("q", "k"))
                    scores.append((q @ k.transpose(1, 2) / np.sqrt(q.shape[-1])).flatten())
        finally:
            enc.layer = layers
            hq.remove(); hk.remove()
        return float(torch.cat(scores).std())


def _pools(model, token_lists):
    """(CLS rows, token means) of last_hidden_state, each x / max(|x|, 1e-12) in the model's precision"""
    import torch
    cls, mean = [], []
    with torch.no_grad():
        for t in token_lists:
            h = model(input_ids=torch.tensor(np.asarray(t, np.int64)[None])).last_hidden_state[0].numpy()
            m = h.mean(axis=0)
            cls.append(h[0] / max(np.linalg.norm(h[0]), 1e-12))
            mean.append(m / max(np.linalg.norm(m), 1e-12))
    return np.stack(cls).astype(np.float64), np.stack(mean).astype(np.float64)


def mean_pool(model, token_lists):
    """mean of last_hidden_state over every token ([CLS] and [SEP] included), then x / max(|x|, 1e-12), in the model's
    precision: sentence-transformers' mean pooling and Normalize"""
    return _pools(model, token_lists)[1]


def head_state(cfg, state, seed):
    """state + the head of a one-label BertForSequenceClassification: pooler N(0, 0.06) / N(0, 0.05), classifier
    N(0, 0.06) / N(0, 0.05)"""
    g = np.random.default_rng(seed + 77)
    d = cfg["hidden_size"]
    st = dict(state)
    st["pooler.dense.weight"] = (0.06 * g.standard_normal((d, d))).astype(np.float32)
    st["pooler.dense.bias"] = (0.05 * g.standard_normal(d)).astype(np.float32)
    st["classifier.weight"] = (0.06 * g.standard_normal((1, d))).astype(np.float32)
    st["classifier.bias"] = (0.05 * g.standard_normal(1)).astype(np.float32)
    return st


class Fp64CrossEncoder:
    """transformers.BertForSequenceClassification (one label, eager attention) in fp64 and its fp32 twin"""

    def __init__(self, cfg, state):
        import torch
        from transformers import BertConfig, BertForSequenceClassification
        from transformers.initialization import no_init_weights
        with no_init_weights():
            m = BertForSequenceClassification(BertConfig(**cfg, num_labels=1, attn_implementation="eager"))
        m = m.double().eval()
        sd = {(k if k.startswith("classifier.") else "bert." + k): torch.from_numpy(np.asarray(v, np.float64)) for k, v in state.items()}
        missing, _ = m.load_state_dict(sd, strict=False)
        assert not [k for k in missing if not k.endswith("position_ids")], missing
        self.m64, self.m32 = m, copy.deepcopy(m).float()

    @staticmethod
    def _logits(m, pairs):
        import torch
        out = []
        with torch.no_grad():
            for ids, seg in pairs:
                tt = (np.arange(len(ids)) >= seg).astype(np.int64)
                out.append(float(m(input_ids=torch.tensor(np.asarray(ids, np.int64)[None]),
                                   token_type_ids=torch.tensor(tt[None])).logits[0, 0]))
        return np.asarray(out, np.float64)

    def logits(self, pairs):
        """(fp64 logits, fp32 logits) of (token ids, index of the first segment-B token) pairs, each run alone"""
        return self._logits(self.m64, pairs), self._logits(self.m32, pairs)


def check_range(range_max):
    assert range_max < RANGE_LIMIT, f"a Linear input/output reaches {range_max:.3g}: outside the split-fp16 operand range"


def l2_deviation(got, ref, seed=0):
    """largest change of the L2^2 score against 64 random unit rows (what /retrieve returns)"""
    y = np.random.default_rng(seed).standard_normal((64, got.shape[1]))
    y /= np.linalg.norm(y, axis=1, keepdims=True)
    l2_got = ((np.asarray(got, np.float64)[:, None, :] - y[None]) ** 2).sum(-1)
    l2_ref = ((np.asarray(ref, np.float64)[:, None, :] - y[None]) ** 2).sum(-1)
    return float(np.abs(l2_got - l2_ref).max())


def yardstick(got, ref64, ref32):
    """K5's max error against fp64, torch fp32's max error against fp64 on the same rows, and their ratio (the torch
    error floored at 2^-23, the fp32 unit roundoff, so a lucky fp32 run cannot make the bound vanish)"""
    k5 = float(np.abs(np.asarray(got, np.float64) - ref64).max())
    t32 = float(np.abs(ref32 - ref64).max())
    return k5, t32, k5 / max(t32, 2.0 ** -23)
