"""XLM-RoBERTa fixtures: SentencePiece Unigram tokenizers trained offline from a seeded corpus and converted to the
tokenizer.json an XLM-R snapshot carries, bge-reranker-shaped snapshots, and the fp64 transformers reference of an
XLMRobertaForSequenceClassification cross-encoder.  Test infrastructure only."""
import copy
import json
import os

import numpy as np

from tests import bert_reference as br

# XLMRobertaConfig of the bge-reranker checkpoints (one label, pad_token_id 1, one token-type row)
BGE_RERANKERS = {
    "bge-reranker-base": dict(num_hidden_layers=12, hidden_size=768, num_attention_heads=12, intermediate_size=3072,
                              max_position_embeddings=514),
    "bge-reranker-large": dict(num_hidden_layers=24, hidden_size=1024, num_attention_heads=16, intermediate_size=4096,
                               max_position_embeddings=514),
    "bge-reranker-v2-m3": dict(num_hidden_layers=24, hidden_size=1024, num_attention_heads=16, intermediate_size=4096,
                               max_position_embeddings=8194),
}
VOCAB = 250002
PAD = 1


def config_json(shape: str, **change) -> dict:
    """the config.json of a bge-reranker snapshot"""
    cfg = dict(BGE_RERANKERS[shape], model_type="xlm-roberta", architectures=["XLMRobertaForSequenceClassification"],
               id2label={"0": "LABEL_0"}, label2id={"LABEL_0": 0}, vocab_size=VOCAB, type_vocab_size=1, pad_token_id=PAD,
               bos_token_id=0, eos_token_id=2, hidden_act="gelu", position_embedding_type="absolute", layer_norm_eps=1e-5,
               hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1, initializer_range=0.02)
    cfg.update(change)
    return cfg


# ------------------------------------------------------------------------------------------------ tokenizers
WORDS = ["the", "quick", "brown", "fox", "gpu", "token", "retrieval", "engine", "passage", "query", "rerank", "café", "naïve",
         "über", "émigré", "ß", "москва", "привет", "日本語", "中文", "한국어", "ＦＵＬＬ", "Ä", "ﬁle", "½", "x²", "straße",
         "résumé", "ångström", "données", "Ελληνικά", "العربية", "हिन्दी"]


def corpus(seed: int, n_lines: int = 3000) -> list[str]:
    g = np.random.default_rng(seed)
    return [" ".join(g.choice(WORDS, int(g.integers(3, 14)))) for _ in range(n_lines)]


def train_tokenizer(out_dir: str, seed: int = 0, normalization: str = "nmt_nfkc", vocab_size: int = 400) -> str:
    """a seeded SentencePiece Unigram model converted by transformers' XLMRobertaTokenizer into out_dir (tokenizer.json,
    tokenizer_config.json); returns out_dir.  character_coverage < 1 leaves the rarest characters to <unk>."""
    import sentencepiece as spm
    from transformers import XLMRobertaTokenizer
    spm_dir = os.path.join(out_dir, "spm")
    os.makedirs(spm_dir, exist_ok=True)
    path = os.path.join(spm_dir, "corpus.txt")
    with open(path, "w", encoding="utf-8") as f:
        f.write("\n".join(corpus(seed)) + "\n")
    spm.SentencePieceTrainer.train(input=path, model_prefix=os.path.join(spm_dir, "sentencepiece.bpe"), vocab_size=vocab_size,
                                   model_type="unigram", normalization_rule_name=normalization, character_coverage=0.995,
                                   hard_vocab_limit=False, num_threads=1, seed_sentencepiece_size=100000,
                                   minloglevel=2)
    if normalization == "identity":
        # an identity model has an empty charsmap, which the converter cannot parse: build the same vocabulary (XLM-R's
        # four specials, the pieces after SentencePiece's three, <mask>) with no normaliser
        sp = spm.SentencePieceProcessor(model_file=os.path.join(spm_dir, "sentencepiece.bpe.model"))
        vocab = [("<s>", 0.0), ("<pad>", 0.0), ("</s>", 0.0), ("<unk>", 0.0)]
        vocab += [(sp.id_to_piece(i), float(sp.get_score(i))) for i in range(3, sp.get_piece_size())] + [("<mask>", 0.0)]
        XLMRobertaTokenizer(vocab=vocab).save_pretrained(out_dir)
    else:
        XLMRobertaTokenizer.from_pretrained(spm_dir).save_pretrained(out_dir)
    return out_dir


def legacy_form(src: str, dst: str, lstrip_mask: bool = True) -> str:
    """the same tokenizer.json in the form older hub snapshots carry: normalizer Sequence[Precompiled, Replace " {2,}"],
    a bare Metaspace pre-tokenizer, <mask> with lstrip"""
    tj = json.load(open(src, encoding="utf-8"))
    steps = [tj["normalizer"]] if tj.get("normalizer") else []
    tj["normalizer"] = {"type": "Sequence", "normalizers": steps + [{"type": "Replace", "pattern": {"Regex": " {2,}"}, "content": " "}]}
    pre = tj["pre_tokenizer"]
    tj["pre_tokenizer"] = pre["pretokenizers"][-1] if pre.get("type") == "Sequence" else pre
    for t in tj["added_tokens"]:
        if t["content"] == "<mask>":
            t["lstrip"] = lstrip_mask
    with open(dst, "w", encoding="utf-8") as f:
        json.dump(tj, f, ensure_ascii=False)
    return dst


def write_snapshot(path: str, config: dict, tokenizer_dir: str | None, tokenizer_config=None, state=None) -> str:
    """a bge-reranker-shaped snapshot: config.json, tokenizer.json (copied from tokenizer_dir; None leaves it out),
    tokenizer_config.json, and model.safetensors given an XLMRobertaForSequenceClassification state"""
    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump(config, f)
    tc = tokenizer_config if tokenizer_config is not None else {"model_max_length": config["max_position_embeddings"] - 2,
                                                                 "tokenizer_class": "XLMRobertaTokenizer"}
    with open(os.path.join(path, "tokenizer_config.json"), "w") as f:
        json.dump(tc, f)
    if tokenizer_dir is not None:
        with open(os.path.join(tokenizer_dir, "tokenizer.json"), "rb") as f, open(os.path.join(path, "tokenizer.json"), "wb") as o:
            o.write(f.read())
    if state is not None:
        from safetensors.numpy import save_file
        save_file({k: np.ascontiguousarray(v, np.float32) for k, v in state.items()}, os.path.join(path, "model.safetensors"))
    return path


# ------------------------------------------------------------------------------------------------ weights and fp64 model
def encoder_config(shape: str, **change) -> dict:
    """the encoder fields bert_reference's generators read, for a bge-reranker shape"""
    return dict(BGE_RERANKERS[shape], vocab_size=VOCAB, type_vocab_size=1, **change)


def k5_state(cfg, regime: str, seed: int = 0):
    """(K5-named state with the head as pooler.dense / classifier, its fp64 reference): bert_reference's random or
    stressed weights with one token-type row, plus a one-label head"""
    if regime == "stressed":
        st = br.stressed_state(dict(cfg, type_vocab_size=2), seed)[0]
    else:
        st = br.random_state(cfg, seed)
    st["embeddings.token_type_embeddings.weight"] = st["embeddings.token_type_embeddings.weight"][:1].copy()
    st = br.head_state(cfg, st, seed)
    return st


def hf_state(state: dict) -> dict:
    """K5 names -> XLMRobertaForSequenceClassification names (what a checkpoint on disk holds)"""
    out = {}
    for k, v in state.items():
        if k.startswith("pooler.dense."):
            out["classifier.dense." + k[len("pooler.dense."):]] = v
        elif k.startswith("classifier."):
            out["classifier.out_proj." + k[len("classifier."):]] = v
        else:
            out["roberta." + k] = v
    return out


class Fp64XlmrCrossEncoder:
    """transformers.XLMRobertaForSequenceClassification (one label, eager attention) in fp64, its fp32 twin and, on
    request, torch bf16 autocast; on `device`.  Positions come from transformers' own rule (pad_token_id + 1 on), so the
    pairs must not contain the pad id.  Forward hooks record the largest |value| at every Linear input and output."""

    def __init__(self, cfg, state, device="cpu"):
        import torch
        from transformers import XLMRobertaConfig, XLMRobertaForSequenceClassification
        from transformers.initialization import no_init_weights
        with no_init_weights():
            m = XLMRobertaForSequenceClassification(XLMRobertaConfig(**cfg, num_labels=1, pad_token_id=PAD, layer_norm_eps=1e-5,
                                                                     attn_implementation="eager"))
        m = m.double().eval()
        sd = {k: torch.from_numpy(np.asarray(v, np.float64)) for k, v in hf_state(state).items()}
        missing, _ = m.load_state_dict(sd, strict=False)
        assert not [k for k in missing if not k.endswith(("position_ids", "token_type_ids"))], missing
        self.device = device
        self.m64 = m.to(device)
        self._m32 = None
        self.range_max = 0.0
        for mod in self.m64.modules():
            if isinstance(mod, torch.nn.Linear):
                mod.register_forward_hook(self._record)

    def _record(self, mod, inp, out):
        self.range_max = max(self.range_max, float(inp[0].abs().max()), float(out.abs().max()))

    def _logits(self, m, pairs, autocast=False):
        import torch
        out = []
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            for ids in pairs:
                ids = np.asarray(ids, np.int64)
                assert not (ids == PAD).any()
                out.append(float(m(input_ids=torch.tensor(ids[None], device=self.device)).logits[0, 0].float()))
        return np.asarray(out, np.float64)

    def _fp32(self):
        if self._m32 is None:
            self._m32 = copy.deepcopy(self.m64).float()
        return self._m32

    def logits(self, pairs):
        """(fp64 logits, fp32 logits) of each pair's token ids, run alone"""
        return self._logits(self.m64, pairs), self._logits(self._fp32(), pairs)

    def logits_bf16(self, pairs):
        """logits under torch bf16 autocast (the device must be cuda)"""
        return self._logits(self._fp32(), pairs, autocast=True)
