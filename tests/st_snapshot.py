"""Sentence-transformers model snapshots written to a directory, laid out like the published ones (BAAI/bge-small-en-v1.5:
CLS pooling, 512 tokens; sentence-transformers/all-MiniLM-L6-v2: mean pooling, 256 tokens): config.json, vocab.txt,
tokenizer_config.json, sentence_bert_config.json, modules.json, 1_Pooling/config.json, and model.safetensors when weights
are given.  Test infrastructure only."""
import json
import os

VOCAB = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]", "the", "The", "quick", "brown", "fox", "Fox", "jump", "##s", "##ed", "over",
         "lazy", "dog", ",", ".", "!", "?", "'", "-", ":", "cafe", "Cafe", "café", "Café", "naive", "naïve", "##ly", "中", "文", "日",
         "本", "語", "token", "##izer", "gpu", "GPU", "re", "##present", "this", "question", "for", "search", "relevant", "passage",
         "##e", "x", "a", "b", "c", "##a", "##b", "##c", "é", "##é", "e", "E", "ü", "Ü", "##ü"]

BGE_SMALL = dict(architectures=["BertModel"], attention_probs_dropout_prob=0.1, hidden_act="gelu", hidden_dropout_prob=0.1,
                 hidden_size=384, initializer_range=0.02, intermediate_size=1536, layer_norm_eps=1e-12, max_position_embeddings=512,
                 model_type="bert", num_attention_heads=12, num_hidden_layers=12, pad_token_id=0, position_embedding_type="absolute",
                 type_vocab_size=2, use_cache=True, vocab_size=30522)
MINILM_L6 = dict(BGE_SMALL, num_hidden_layers=6)

POOL_FLAGS = ("pooling_mode_cls_token", "pooling_mode_mean_tokens", "pooling_mode_max_tokens", "pooling_mode_mean_sqrt_len_tokens")


def pooling_config(dim, mode):
    return dict({"word_embedding_dimension": dim}, **{f: f == f"pooling_mode_{mode}" for f in POOL_FLAGS})


def layout(kind, config=None):
    """{file name: JSON content} of a bge-small-en-v1.5 ("bge") or all-MiniLM-L6-v2 ("minilm") snapshot; `config` replaces
    the model's config.json"""
    cfg = dict(config or (BGE_SMALL if kind == "bge" else MINILM_L6))
    mean = kind == "minilm"
    return {
        "config.json": cfg,
        "tokenizer_config.json": {"clean_up_tokenization_spaces": True, "cls_token": "[CLS]", "do_basic_tokenize": True,
                                  "do_lower_case": True, "mask_token": "[MASK]", "model_max_length": 512, "never_split": None,
                                  "pad_token": "[PAD]", "sep_token": "[SEP]", "strip_accents": None, "tokenize_chinese_chars": True,
                                  "tokenizer_class": "BertTokenizer", "unk_token": "[UNK]"},
        "sentence_bert_config.json": {"max_seq_length": 256, "do_lower_case": False} if mean else
                                     {"max_seq_length": 512, "do_lower_case": True},
        "modules.json": [{"idx": 0, "name": "0", "path": "", "type": "sentence_transformers.models.Transformer"},
                         {"idx": 1, "name": "1", "path": "1_Pooling", "type": "sentence_transformers.models.Pooling"},
                         {"idx": 2, "name": "2", "path": "2_Normalize", "type": "sentence_transformers.models.Normalize"}],
        "1_Pooling/config.json": pooling_config(cfg["hidden_size"], "mean_tokens" if mean else "cls_token"),
    }


def write(path, files, vocab=VOCAB, state=None):
    """write `files` ({relative name: JSON content, or None to leave the file out}), vocab.txt and, given a BertModel state
    dict, model.safetensors"""
    os.makedirs(path, exist_ok=True)
    for name, content in files.items():
        if content is None:
            continue
        p = os.path.join(path, name)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, "w", encoding="utf-8") as f:
            json.dump(content, f)
    if vocab is not None:
        with open(os.path.join(path, "vocab.txt"), "w", encoding="utf-8") as f:
            f.write("\n".join(vocab) + "\n")
    if state is not None:
        import numpy as np
        from safetensors.numpy import save_file
        save_file({k: np.ascontiguousarray(v, np.float32) for k, v in state.items()}, os.path.join(path, "model.safetensors"))
    return str(path)
