"""Host-side text pipeline for the sparse side of /retrieve.

The reference tokenises inside `BM25Retriever.from_defaults` (hybrid_retriever.py:122-125) with
bm25s + PyStemmer, neither vendored nor installable offline [3P-unverified]; this module
restates that pipeline from the published algorithms:

  bm25s.tokenize(texts, stopwords="english", stemmer=Stemmer.Stemmer("english")):
    lower-case, regex r"(?u)\\b\\w\\w+\\b", drop the 33-word English stop list, then stem
    each remaining token with the Snowball English ("Porter2") stemmer.

Term ids are assigned by `Vocabulary` in first-seen order; they are what the C ABI takes
(`term_ids`, `q_terms` in include/kaito_rag.h).  Text stays on the host (SURVEY.md section 8 b3).
"""
from __future__ import annotations

import re
from collections import Counter

import numpy as np

TOKEN_PATTERN = re.compile(r"(?u)\b\w\w+\b")

# bm25s.stopwords.STOPWORDS_EN
STOPWORDS_EN = frozenset((
    "a", "an", "and", "are", "as", "at", "be", "but", "by", "for", "if", "in", "into", "is", "it", "no", "not", "of",
    "on", "or", "such", "that", "the", "their", "then", "there", "these", "they", "this", "to", "was", "will", "with",
))

# ---------------------------------------------------------------- Snowball English stemmer
_VOWELS = "aeiouy"
_DOUBLES = ("bb", "dd", "ff", "gg", "mm", "nn", "pp", "rr", "tt")
_LI_ENDING = "cdeghkmnrt"
_EXCEPTIONS = {"skis": "ski", "skies": "sky", "dying": "die", "lying": "lie", "tying": "tie", "idly": "idl",
               "gently": "gentl", "ugly": "ugli", "early": "earli", "only": "onli", "singly": "singl", "sky": "sky",
               "news": "news", "howe": "howe", "atlas": "atlas", "cosmos": "cosmos", "bias": "bias", "andes": "andes"}
_EXCEPTIONS_1A = frozenset(("inning", "outing", "canning", "herring", "earring", "proceed", "exceed", "succeed"))
_STEP2 = (("ization", "ize"), ("ational", "ate"), ("fulness", "ful"), ("ousness", "ous"), ("iveness", "ive"),
          ("tional", "tion"), ("biliti", "ble"), ("lessli", "less"), ("entli", "ent"), ("ation", "ate"),
          ("alism", "al"), ("aliti", "al"), ("ousli", "ous"), ("iviti", "ive"), ("fulli", "ful"), ("enci", "ence"),
          ("anci", "ance"), ("abli", "able"), ("izer", "ize"), ("ator", "ate"), ("alli", "al"), ("bli", "ble"),
          ("ogi", "og"), ("li", ""))
_STEP3 = (("ational", "ate"), ("tional", "tion"), ("alize", "al"), ("icate", "ic"), ("iciti", "ic"), ("ative", ""),
          ("ical", "ic"), ("ness", ""), ("ful", ""))
_STEP4 = ("ement", "ance", "ence", "able", "ible", "ment", "ant", "ent", "ism", "ate", "iti", "ous", "ive", "ize",
          "ion", "al", "er", "ic")


def _is_vowel(w: str, i: int) -> bool:
    return w[i] in _VOWELS


def _region_after_vc(w: str, start: int) -> int:
    """index after the first non-vowel that follows a vowel, searching from `start`"""
    for i in range(start + 1, len(w)):
        if not _is_vowel(w, i) and _is_vowel(w, i - 1):
            return i + 1
    return len(w)


def _r1_r2(w: str):
    if w.startswith(("gener", "arsen")):
        r1 = 5
    elif w.startswith("commun"):
        r1 = 6
    else:
        r1 = _region_after_vc(w, 0)
    return r1, _region_after_vc(w, r1)


def _ends_short_syllable(w: str) -> bool:
    n = len(w)
    if n == 2:
        return _is_vowel(w, 0) and not _is_vowel(w, 1)
    if n >= 3:
        return (not _is_vowel(w, n - 3)) and _is_vowel(w, n - 2) and (not _is_vowel(w, n - 1)) and w[-1] not in "wxY"
    return False


def _contains_vowel(w: str) -> bool:
    return any(c in _VOWELS for c in w)


def stem(word: str) -> str:
    """Snowball English (Porter2) stem of a lower-case token."""
    if len(word) <= 2:
        return word
    if word in _EXCEPTIONS:
        return _EXCEPTIONS[word]
    w = word[1:] if word.startswith("'") else word
    # mark consonant y
    chars = list(w)
    for i, c in enumerate(chars):
        if c == "y" and (i == 0 or chars[i - 1] in _VOWELS):
            chars[i] = "Y"
    w = "".join(chars)
    r1, r2 = _r1_r2(w)

    # step 0
    for suf in ("'s'", "'s", "'"):
        if w.endswith(suf):
            w = w[: -len(suf)]
            break
    # step 1a
    if w.endswith("sses"):
        w = w[:-2]
    elif w.endswith(("ied", "ies")):
        w = w[:-2] if len(w) > 4 else w[:-1]
    elif w.endswith(("us", "ss")):
        pass
    elif w.endswith("s"):
        if _contains_vowel(w[:-2]):
            w = w[:-1]
    if w in _EXCEPTIONS_1A:
        return w.replace("Y", "y")
    # step 1b
    if w.endswith("eedly"):
        if len(w) - 5 >= r1:
            w = w[:-3]
    elif w.endswith("eed"):
        if len(w) - 3 >= r1:
            w = w[:-1]
    else:
        for suf in ("ingly", "edly", "ing", "ed"):
            if w.endswith(suf):
                stem_part = w[: -len(suf)]
                if _contains_vowel(stem_part):
                    w = stem_part
                    if w.endswith(("at", "bl", "iz")):
                        w += "e"
                    elif w.endswith(_DOUBLES):
                        w = w[:-1]
                    elif _ends_short_syllable(w) and r1 >= len(w):
                        w += "e"
                break
    # step 1c
    if len(w) > 2 and w[-1] in "yY" and w[-2] not in _VOWELS:
        w = w[:-1] + "i"
    # step 2
    for suf, rep in _STEP2:
        if w.endswith(suf):
            if len(w) - len(suf) >= r1:
                if suf == "ogi":
                    if w[: -len(suf)].endswith("l"):
                        w = w[: -len(suf)] + rep
                elif suf == "li":
                    if len(w) > 2 and w[-3] in _LI_ENDING:
                        w = w[:-2]
                else:
                    w = w[: -len(suf)] + rep
            break
    # step 3
    for suf, rep in _STEP3:
        if w.endswith(suf):
            if len(w) - len(suf) >= r1:
                if suf == "ative":
                    if len(w) - len(suf) >= r2:
                        w = w[: -len(suf)]
                else:
                    w = w[: -len(suf)] + rep
            break
    # step 4
    for suf in _STEP4:
        if w.endswith(suf):
            if len(w) - len(suf) >= r2:
                if suf == "ion":
                    if len(w) > 3 and w[-4] in "st":
                        w = w[:-3]
                else:
                    w = w[: -len(suf)]
            break
    # step 5
    if w.endswith("e"):
        if len(w) - 1 >= r2 or (len(w) - 1 >= r1 and not _ends_short_syllable(w[:-1])):
            w = w[:-1]
    elif w.endswith("l"):
        if len(w) - 1 >= r2 and w[:-1].endswith("l"):
            w = w[:-1]
    return w.replace("Y", "y")


# ------------------------------------------------------------------------------ tokenise
def tokenize_py(text: str) -> list[str]:
    """bm25s-style tokens of one text: lower-case, \\w\\w+ words, stop words removed, stemmed.  Pure Python: the
    Unicode-complete restatement and the spec of the native path."""
    return [stem(t) for t in TOKEN_PATTERN.findall(text.lower()) if t not in STOPWORDS_EN]


_lib = None


def _native_lib():
    """libkaito_rag.so for the host-side analysis functions (csrc/text_native.cpp); False when it cannot be loaded -- the
    analysis is host code, so unlike the search path it may run in pure Python."""
    global _lib
    if _lib is None:
        try:
            from . import _native
            _lib = _native.load()
        except Exception:
            _lib = False
    return _lib


def tokenize(text: str) -> list[str]:
    """tokenize_py, through the native analyser (same output, ~20x faster) when the text is ASCII."""
    L = _native_lib()
    if not L or not text.isascii():
        return tokenize_py(text)
    import ctypes as C
    raw = text.encode("ascii")
    cap = len(raw) + 16                       # stems are never longer than their tokens plus one 'e' per token... see below
    n_len, n_tok = C.c_int64(0), C.c_int32(0)
    buf = C.create_string_buffer(cap)
    if L.krag_text_analyze(raw, len(raw), buf, cap, C.byref(n_len), C.byref(n_tok)) != 0:
        return tokenize_py(text)
    if n_len.value > cap:                     # (a token of >= 2 chars yields a stem of at most len + 1 chars and a separator)
        cap = n_len.value
        buf = C.create_string_buffer(cap)
        L.krag_text_analyze(raw, len(raw), buf, cap, C.byref(n_len), C.byref(n_tok))
    return buf.raw[: n_len.value].decode("ascii").split("\n") if n_tok.value else []


class Vocabulary:
    """term string <-> dense u32 id in first-seen order (the host owns the vocabulary)."""

    def __init__(self):
        self.ids: dict[str, int] = {}
        self.terms: list[str] = []

    def __len__(self):
        return len(self.terms)

    def add(self, term: str) -> int:
        i = self.ids.get(term)
        if i is None:
            i = len(self.terms)
            self.ids[term] = i
            self.terms.append(term)
        return i

    def doc_terms(self, text: str):
        """(unique term ids u32, tf u16, doc_len) of one node; grows the vocabulary."""
        toks = tokenize(text)
        cnt = Counter(toks)                     # C-speed counting of the strings; keys keep first-occurrence order, so new terms
        get, add = self.ids.get, self.add       # get their ids in exactly the order a token-by-token pass would hand them out
        known = [get(t) for t in cnt]
        if None in known:
            known = [add(t) if i is None else i for t, i in zip(cnt, known)]
        ids = np.array(known, np.uint32)
        tf = np.minimum(np.fromiter(cnt.values(), np.int64, len(cnt)), 65535).astype(np.uint16)
        return ids, tf, len(toks)

    def query_terms(self, text: str) -> np.ndarray:
        """term ids of a query in token order, duplicates kept, unknown terms dropped (bm25s semantics)."""
        return np.asarray([self.ids[t] for t in tokenize(text) if t in self.ids], np.uint32)


# ------------------------------------------------------------------ WordPiece (BERT / bge tokeniser)
import unicodedata  # noqa: E402


def _is_punct(ch: str) -> bool:
    cp = ord(ch)
    if (33 <= cp <= 47) or (58 <= cp <= 64) or (91 <= cp <= 96) or (123 <= cp <= 126):
        return True
    return unicodedata.category(ch).startswith("P")


def _is_cjk(cp: int) -> bool:
    return ((0x4E00 <= cp <= 0x9FFF) or (0x3400 <= cp <= 0x4DBF) or (0x20000 <= cp <= 0x2A6DF) or (0x2A700 <= cp <= 0x2B73F)
            or (0x2B740 <= cp <= 0x2B81F) or (0x2B820 <= cp <= 0x2CEAF) or (0xF900 <= cp <= 0xFAFF) or (0x2F800 <= cp <= 0x2FA1F))


class WordPieceTokenizer:
    """BertTokenizer (uncased) restated: BasicTokenizer (clean, CJK spacing, lower-case, accent strip,
    punctuation split) + greedy longest-match WordPiece with "##" continuations.  Produces the ids the
    embedder takes: [CLS] tokens [SEP], truncated to max_length.  The reference reaches the same
    tokenizer through sentence-transformers (embedding/huggingface_local_embedding.py:34-53)."""

    def __init__(self, vocab: dict[str, int] | list[str], do_lower_case: bool = True, max_length: int = 512,
                 cls_token: str = "[CLS]", sep_token: str = "[SEP]", unk_token: str = "[UNK]"):
        """cls_token / sep_token / unk_token: the specials (MPNet: <s>, </s>, [UNK]); a special typed in a text is text"""
        tokens = None
        if not isinstance(vocab, dict):
            tokens = list(vocab)
            vocab = {t: i for i, t in enumerate(tokens)}
        self.vocab, self.lower, self.max_length = vocab, do_lower_case, max_length
        self.unk, self.cls, self.sep = vocab[unk_token], vocab[cls_token], vocab[sep_token]
        # native encoder (csrc/text_native.cpp) for ASCII text; needs the ordered token list and tokens without newlines
        self._nat = None
        L = _native_lib()
        if L and tokens is not None and all("\n" not in t for t in tokens):
            import ctypes as C
            blob = "\n".join(tokens).encode("utf-8")
            h = C.c_void_p()
            if L.krag_wordpiece_create_specials(blob, len(blob), 1 if do_lower_case else 0, unk_token.encode("utf-8"),
                                                cls_token.encode("utf-8"), sep_token.encode("utf-8"), C.byref(h)) == 0:
                self._nat = h

    def __del__(self):
        if getattr(self, "_nat", None):
            try:
                _native_lib().krag_wordpiece_destroy(self._nat)
            except Exception:
                pass
            self._nat = None

    @classmethod
    def from_file(cls, path: str, **kw):
        with open(path, encoding="utf-8") as f:
            return cls([line.rstrip("\n") for line in f], **kw)

    def _basic(self, text: str) -> list[str]:
        out = []
        for ch in text:
            cp = ord(ch)
            if cp == 0 or cp == 0xFFFD or (unicodedata.category(ch) in ("Cc", "Cf") and ch not in "\t\n\r"):
                continue
            if _is_cjk(cp):
                out.append(f" {ch} ")
            elif ch in " \t\n\r" or unicodedata.category(ch) == "Zs":
                out.append(" ")
            else:
                out.append(ch)
        toks = []
        for tok in "".join(out).split():
            if self.lower:
                tok = tok.lower()
                tok = "".join(c for c in unicodedata.normalize("NFD", tok) if unicodedata.category(c) != "Mn")
            cur = []
            for ch in tok:
                if _is_punct(ch):
                    if cur:
                        toks.append("".join(cur)); cur = []
                    toks.append(ch)
                else:
                    cur.append(ch)
            if cur:
                toks.append("".join(cur))
        return toks

    def _wordpiece(self, word: str) -> list[int]:
        if len(word) > 100:
            return [self.unk]
        ids, start = [], 0
        while start < len(word):
            end, cur = len(word), None
            while start < end:
                sub = word[start:end] if start == 0 else "##" + word[start:end]
                if sub in self.vocab:
                    cur = self.vocab[sub]
                    break
                end -= 1
            if cur is None:
                return [self.unk]
            ids.append(cur)
            start = end
        return ids

    def encode_py(self, text: str) -> list[int]:
        ids = [i for w in self._basic(text) for i in self._wordpiece(w)]
        return [self.cls] + ids[: self.max_length - 2] + [self.sep]

    def encode(self, text: str) -> list[int]:
        return self.encode_batch([text])[0]

    def encode_batch_flat(self, texts: list[str]):
        """(flat int32 ids, int32 offsets [n + 1]) of every text -- what the embedder's C entry point takes.  All-ASCII batches
        (the common case for queries) never become Python lists: one native call, one masked gather."""
        if self._nat is not None and texts and all(t.isascii() for t in texts):
            import ctypes as C
            raws = [t.encode("ascii") for t in texts]
            offs = np.zeros(len(raws) + 1, np.int64)
            np.cumsum([len(r) for r in raws], out=offs[1:])
            ids = np.empty((len(raws), self.max_length), np.int32)
            cnt = np.empty(len(raws), np.int32)
            rc = _native_lib().krag_wordpiece_encode_batch(self._nat, len(raws), b"".join(raws), offs.ctypes.data_as(C.c_void_p),
                                                           self.max_length, ids.ctypes.data_as(C.c_void_p), cnt.ctypes.data_as(C.c_void_p))
            if rc == 0:
                width = int(cnt.max())
                flat = ids[:, :width][np.arange(width, dtype=np.int32)[None, :] < cnt[:, None]]
                toff = np.zeros(len(raws) + 1, np.int32)
                np.cumsum(cnt, out=toff[1:])
                return np.ascontiguousarray(flat, np.int32), toff
        lists = self.encode_batch(texts)
        toff = np.zeros(len(lists) + 1, np.int32)
        np.cumsum([len(t) for t in lists], out=toff[1:])
        flat = np.fromiter((i for t in lists for i in t), np.int32, int(toff[-1]))
        return flat, toff

    def encode_batch_plain(self, texts: list[str]) -> list[np.ndarray]:
        """int32 ids of every text without [CLS] / [SEP] and without truncation (the halves of a sentence pair).  ASCII
        texts go through the native encoder in one call: a WordPiece token covers at least one character, so a budget of
        the longest text's length + 2 never truncates."""
        out: list = [None] * len(texts)
        idx = [i for i, t in enumerate(texts) if self._nat is not None and t.isascii()]
        if idx:
            import ctypes as C
            raws = [texts[i].encode("ascii") for i in idx]
            offs = np.zeros(len(raws) + 1, np.int64)
            np.cumsum([len(r) for r in raws], out=offs[1:])
            width = max(len(r) for r in raws) + 2
            ids = np.empty((len(raws), width), np.int32)
            cnt = np.empty(len(raws), np.int32)
            rc = _native_lib().krag_wordpiece_encode_batch(self._nat, len(raws), b"".join(raws), offs.ctypes.data_as(C.c_void_p),
                                                           width, ids.ctypes.data_as(C.c_void_p), cnt.ctypes.data_as(C.c_void_p))
            if rc == 0:
                for j, i in enumerate(idx):
                    out[i] = ids[j, 1: cnt[j] - 1].copy()
        for i, t in enumerate(texts):
            if out[i] is None:
                out[i] = np.asarray([k for w in self._basic(t) for k in self._wordpiece(w)], np.int32)
        return out

    def encode_batch(self, texts: list[str]) -> list[list[int]]:
        """ids of every text; ASCII texts go through the native, multi-threaded encoder in one call, the rest through encode_py"""
        out: list = [None] * len(texts)
        idx = [i for i, t in enumerate(texts) if self._nat is not None and t.isascii()]
        if idx:
            import ctypes as C
            raws = [texts[i].encode("ascii") for i in idx]
            offs = np.zeros(len(raws) + 1, np.int64)
            np.cumsum([len(r) for r in raws], out=offs[1:])
            ids = np.empty((len(raws), self.max_length), np.int32)
            cnt = np.empty(len(raws), np.int32)
            rc = _native_lib().krag_wordpiece_encode_batch(self._nat, len(raws), b"".join(raws), offs.ctypes.data_as(C.c_void_p),
                                                           self.max_length, ids.ctypes.data_as(C.c_void_p), cnt.ctypes.data_as(C.c_void_p))
            if rc == 0:
                for j, i in enumerate(idx):
                    out[i] = ids[j, : cnt[j]].tolist()
        for i, t in enumerate(texts):
            if out[i] is None:
                out[i] = self.encode_py(t)
        return out


# ------------------------------------------------------ Unigram (XLM-RoBERTa / bge-reranker tokeniser)
# What the Rust `tokenizers` library does with the tokenizer.json of an XLM-R snapshot, restated: added tokens matched in the
# raw text, the SentencePiece `Precompiled` normaliser (optionally followed by Replace " {2,}" -> " "), the `Metaspace`
# pre-tokeniser (alone or after `WhitespaceSplit`) and the `Unigram` model's Viterbi.  The native path
# (krag_text_unigram_*, csrc/text_native.cpp) runs the same tables for ASCII text.
import base64  # noqa: E402
import json  # noqa: E402

_METASPACE = "▁"
# Rust char::is_whitespace (the Unicode White_Space property), which WhitespaceSplit and an added token's lstrip / rstrip use
_WHITE_SPACE = frozenset(chr(c) for c in (*range(0x09, 0x0E), 0x20, 0x85, 0xA0, 0x1680, *range(0x2000, 0x200B), 0x2028,
                                          0x2029, 0x202F, 0x205F, 0x3000))
_UNK_PENALTY = 10.0                       # an uncovered character scores min_score - 10 (sentencepiece's kUnkPenalty)


class _Charsmap:
    """The `precompiled_charsmap` of a SentencePiece normaliser: a little-endian u32 trie size, a darts-clone double-array
    trie of that many bytes whose values index the NUL-terminated replacement strings that follow it."""

    def __init__(self, blob: bytes, where: str):
        if len(blob) < 4:
            raise ValueError(f"{where}: normalizer.precompiled_charsmap: {len(blob)} bytes, too short for its trie size")
        n = int.from_bytes(blob[:4], "little")
        if n % 4 or 4 + n > len(blob):
            raise ValueError(f"{where}: normalizer.precompiled_charsmap: trie size {n} does not fit its {len(blob)} bytes")
        self.blob = blob
        self.units = np.frombuffer(blob, "<u4", n // 4, 4).tolist()
        self.strings = blob[4 + n:]
        self._memo: dict[str, str | None] = {}

    def lookup(self, key: str):
        """the replacement of the shortest key that prefixes `key` (what the Rust normaliser takes: results[0] of the
        common-prefix search), or None"""
        r = self._memo.get(key, 0)
        if r != 0:
            return r
        r, units, node = None, self.units, 0
        try:
            unit = units[0]
            node ^= (unit >> 10) << ((unit & (1 << 9)) >> 6)
            for c in key.encode("utf-8"):
                if c == 0:
                    break
                node ^= c
                unit = units[node]
                if unit & ((1 << 31) | 0xFF) != c:
                    break
                node ^= (unit >> 10) << ((unit & (1 << 9)) >> 6)
                if (unit >> 8) & 1:
                    v = units[node] & ((1 << 31) - 1)
                    end = self.strings.find(b"\0", v)
                    r = self.strings[v: end if end >= 0 else len(self.strings)].decode("utf-8")
                    break
        except IndexError:
            r = None
        self._memo[key] = r
        return r


def _ws_split(s: str) -> list[tuple[str, int]]:
    """WhitespaceSplit: (word, its index in s) of every maximal run of non-White_Space characters"""
    out, start = [], None
    for i, ch in enumerate(s):
        if ch in _WHITE_SPACE:
            if start is not None:
                out.append((s[start:i], start)); start = None
        elif start is None:
            start = i
    if start is not None:
        out.append((s[start:], start))
    return out


def read_unigram_json(path: str) -> dict:
    """the tables of an XLM-R tokenizer.json, or a ValueError naming the file and the field that asks for something this
    restatement does not do.  Returns pieces, scores, unk_id, charsmap (bytes or None), collapse_spaces, ws_split,
    prepend ("always" | "first") and added [(content, id, lstrip, rstrip)]"""
    try:
        with open(path, encoding="utf-8") as f:
            tj = json.load(f)
    except OSError as ex:
        raise ValueError(f"{path}: cannot be read ({ex.strerror})") from None
    except ValueError as ex:
        raise ValueError(f"{path}: not JSON ({ex})") from None
    model = tj.get("model") or {}
    if model.get("type") != "Unigram":
        raise ValueError(f"{path}: model.type {model.get('type')!r}: the XLM-R reranker path reads Unigram models only")
    if model.get("byte_fallback"):
        raise ValueError(f"{path}: model.byte_fallback true: byte-fallback pieces are not restated")
    vocab = model.get("vocab")
    if not isinstance(vocab, list) or not vocab or not all(isinstance(v, list) and len(v) == 2 for v in vocab):
        raise ValueError(f"{path}: model.vocab: expected a non-empty list of [piece, score]")
    unk = model.get("unk_id")
    if not isinstance(unk, int) or not 0 <= unk < len(vocab):
        raise ValueError(f"{path}: model.unk_id {unk!r}: must index model.vocab")
    # normaliser: null, Precompiled, Replace(" {2,}" -> " "), or a Sequence of those
    norm = tj.get("normalizer")
    steps = [] if norm is None else (norm.get("normalizers") if norm.get("type") == "Sequence" else [norm])
    charsmap, collapse = None, False
    for i, st in enumerate(steps or []):
        kind = st.get("type") if isinstance(st, dict) else None
        if kind == "Precompiled" and charsmap is None and not collapse:
            raw = st.get("precompiled_charsmap") or ""
            charsmap = _Charsmap(base64.b64decode(raw), path) if raw else None
        elif (kind == "Replace" and st.get("pattern") == {"Regex": " {2,}"} and st.get("content") == " " and not collapse):
            collapse = True
        else:
            raise ValueError(f"{path}: normalizer {kind!r} (step {i}): only Precompiled, optionally followed by Replace "
                             f"' {{2,}}' -> ' ', is restated")
    # pre-tokeniser: Metaspace, alone or after WhitespaceSplit
    pre = tj.get("pre_tokenizer") or {}
    seq = pre.get("pretokenizers") if pre.get("type") == "Sequence" else [pre]
    ws = len(seq or []) == 2 and isinstance(seq[0], dict) and seq[0].get("type") == "WhitespaceSplit"
    meta = seq[-1] if seq and isinstance(seq[-1], dict) else {}
    if len(seq or []) != (2 if ws else 1) or meta.get("type") != "Metaspace":
        raise ValueError(f"{path}: pre_tokenizer {pre.get('type')!r}: expected Metaspace, alone or after WhitespaceSplit")
    scheme = meta.get("prepend_scheme") or ("always" if meta.get("add_prefix_space", True) else "never")
    if meta.get("replacement", _METASPACE) != _METASPACE or scheme not in ("always", "first") or meta.get("split", True) is not True:
        raise ValueError(f"{path}: pre_tokenizer Metaspace (replacement {meta.get('replacement')!r}, prepend_scheme {scheme!r}, "
                         f"split {meta.get('split', True)!r}): expected '▁', 'always' or 'first', split true")
    added = []
    for t in tj.get("added_tokens") or []:
        if t.get("normalized") or t.get("single_word"):
            raise ValueError(f"{path}: added_tokens {t.get('content')!r}: normalized / single_word tokens are not restated")
        added.append((t["content"], int(t["id"]), bool(t.get("lstrip")), bool(t.get("rstrip"))))
    return {"pieces": [str(v[0]) for v in vocab], "scores": [float(v[1]) for v in vocab], "unk_id": unk, "charsmap": charsmap,
            "collapse_spaces": collapse, "ws_split": ws, "prepend": scheme, "added": added}


class UnigramTokenizer:
    """XLM-RoBERTa's SentencePiece Unigram tokeniser (bge-reranker-*), read from tokenizer.json.  encode_batch_plain gives
    what `tokenizers.Tokenizer.encode(text, add_special_tokens=False).ids` gives; `cls` / `sep` are <s> / </s>.  All-ASCII
    batches go through the native encoder; other text through this restatement."""

    def __init__(self, tables: dict, max_length: int = 512):
        self.max_length = max_length
        self.pieces, self.scores, self.unk = tables["pieces"], tables["scores"], tables["unk_id"]
        self.charsmap, self.collapse, self.ws_split = tables["charsmap"], tables["collapse_spaces"], tables["ws_split"]
        self.prepend_first = tables["prepend"] == "first"
        self.added = tables["added"]
        self.ids = {p: i for i, p in enumerate(self.pieces)}          # a repeated piece keeps its last id, as in Rust
        self.min_score = min(self.scores)
        self.max_piece = max(len(p) for p in self.pieces)
        amap = {c: i for c, i, _, _ in self.added}
        try:
            self.cls, self.sep = amap.get("<s>", self.ids["<s>"]), amap.get("</s>", self.ids["</s>"])
        except KeyError:
            raise ValueError("tokenizer.json: <s> / </s> missing from added_tokens and model.vocab") from None
        self._added_re = (re.compile("|".join(re.escape(c) for c, *_ in sorted(self.added, key=lambda a: -len(a[0]))))
                          if self.added else None)
        self._added = {c: (i, l, r) for c, i, l, r in self.added}
        self._nat = None
        L = _native_lib()
        if L:
            import ctypes as C
            enc = [p.encode("utf-8") for p in self.pieces]
            poff = np.zeros(len(enc) + 1, np.int64)
            np.cumsum([len(b) for b in enc], out=poff[1:])
            sc = np.asarray(self.scores, np.float64)
            cm = self.charsmap.blob if self.charsmap else b""
            aenc = [c.encode("utf-8") for c, *_ in self.added]
            aoff = np.zeros(len(aenc) + 1, np.int64)
            np.cumsum([len(b) for b in aenc], out=aoff[1:])
            aid = np.asarray([i for _, i, _, _ in self.added] or [0], np.int32)
            afl = np.asarray([int(l) | 2 * int(r) for _, _, l, r in self.added] or [0], np.int32)
            flags = int(self.collapse) | 2 * int(self.ws_split) | 4 * int(self.prepend_first)
            h = C.c_void_p()
            if L.krag_text_unigram_create(b"".join(enc), poff.ctypes.data_as(C.c_void_p), sc.ctypes.data_as(C.c_void_p), len(enc),
                                          self.unk, cm, len(cm), flags, b"".join(aenc), aoff.ctypes.data_as(C.c_void_p),
                                          aid.ctypes.data_as(C.c_void_p), afl.ctypes.data_as(C.c_void_p), len(aenc),
                                          C.byref(h)) == 0:
                self._nat = h

    def __del__(self):
        if getattr(self, "_nat", None):
            try:
                _native_lib().krag_text_unigram_destroy(self._nat)
            except Exception:
                pass
            self._nat = None

    @classmethod
    def from_file(cls, path: str, max_length: int = 512):
        """tokenizer.json of an XLM-R snapshot; a ValueError naming the file and field it refuses"""
        return cls(read_unigram_json(path), max_length=max_length)

    # ---- the restatement (any text)
    def _split_added(self, text: str) -> list[tuple[str, int | None, int]]:
        """(segment, added-token id or None, segment's start in text): the added tokens' leftmost-longest matches, an lstrip
        token taking the White_Space before it (not past the previous match), an rstrip one the White_Space after it"""
        if self._added_re is None or not text:
            return [(text, None, 0)]
        out, pos = [], 0
        for m in self._added_re.finditer(text):
            start, stop = m.start(), m.end()
            tid, lstrip, rstrip = self._added[m.group()]
            if lstrip:
                j = start
                while j > 0 and text[j - 1] in _WHITE_SPACE:
                    j -= 1
                start = max(j, pos)
            if rstrip:
                while stop < len(text) and text[stop] in _WHITE_SPACE:
                    stop += 1
            if pos < start:
                out.append((text[pos:start], None, pos))
            out.append((text[start:stop], tid, start))
            pos = stop
        if pos < len(text):
            out.append((text[pos:], None, pos))
        return out

    def _normalize(self, s: str) -> str:
        if self.charsmap is not None:
            import regex
            look, out = self.charsmap.lookup, []
            for g in regex.findall(r"\X", s):
                if len(g.encode("utf-8")) < 6:
                    r = look(g)
                    if r is not None:
                        out.append(r)
                        continue
                for ch in g:
                    r = look(ch)
                    out.append(ch if r is None else r)
            s = "".join(out)
        if self.collapse:
            s = re.sub(" {2,}", " ", s)
        return s

    def _pre_tokenize(self, s: str, at_origin: bool) -> list[str]:
        """Metaspace (after WhitespaceSplit when configured): ' ' -> U+2581, prepended to every word ("always") or to the one
        that starts the input ("first"), then split before every U+2581"""
        words = _ws_split(s) if self.ws_split else [(s, 0)]
        out = []
        for w, at in words:
            w = w.replace(" ", _METASPACE)
            if w and not w.startswith(_METASPACE) and (not self.prepend_first or (at_origin and at == 0)):
                w = _METASPACE + w
            out += [p for p in re.split(f"(?={_METASPACE})", w) if p]
        return out

    def _viterbi(self, w: str) -> list[int]:
        """the Unigram model's best segmentation of one pre-token (Rust encode_optimized): a later path replaces an earlier
        one only with a strictly higher score; an uncovered character is unk at min_score - 10; adjacent unks fuse"""
        n, ids, scores, maxp = len(w), self.ids, self.scores, self.max_piece
        if n == 0:
            return []
        unk_score = self.min_score - _UNK_PENALTY
        best = [0.0] * (n + 1)
        start = [-1] * (n + 1)
        tok = [0] * (n + 1)
        start[0] = 0
        for i in range(n):
            base = best[i]
            single = False
            for j in range(i + 1, min(n, i + maxp) + 1):
                t = ids.get(w[i:j])
                if t is None:
                    continue
                c = scores[t] + base
                if start[j] < 0 or c > best[j]:
                    best[j], start[j], tok[j] = c, i, t
                if j == i + 1:
                    single = True
            if not single:
                c = unk_score + base
                if start[i + 1] < 0 or c > best[i + 1]:
                    best[i + 1], start[i + 1], tok[i + 1] = c, i, self.unk
        # back from the end; a run of unk nodes becomes one piece, looked up as a whole (not found: unk)
        out, end, run_end = [], n, -1
        while end > 0:
            b = start[end]
            if tok[end] == self.unk:
                if run_end < 0:
                    run_end = end
            else:
                if run_end >= 0:
                    out.append(self.ids.get(w[end:run_end], self.unk)); run_end = -1
                out.append(tok[end])
            end = b
        if run_end >= 0:
            out.append(self.ids.get(w[0:run_end], self.unk))
        out.reverse()
        return out

    def encode_py(self, text: str) -> list[int]:
        """ids of one text without <s> / </s>, untruncated"""
        ids = []
        for seg, tid, at in self._split_added(text):
            if tid is not None:
                ids.append(tid)
                continue
            for w in self._pre_tokenize(self._normalize(seg), at == 0):
                ids += self._viterbi(w)
        return ids

    # ---- batch entry points
    def encode_batch_plain(self, texts: list[str]) -> list[np.ndarray]:
        """int32 ids of every text without <s> / </s> and without truncation (the halves of a sentence pair); all-ASCII
        texts in one native call"""
        out: list = [None] * len(texts)
        idx = [i for i, t in enumerate(texts) if self._nat is not None and t.isascii()]
        if idx:
            import ctypes as C
            raws = [texts[i].encode("ascii") for i in idx]
            offs = np.zeros(len(raws) + 1, np.int64)
            np.cumsum([len(r) for r in raws], out=offs[1:])
            blob = b"".join(raws)
            cap = max(len(r) for r in raws) + 8
            for _ in range(2):                 # the count of a text longer than cap is reported; grow once and redo
                ids = np.empty((len(raws), cap), np.int32)
                cnt = np.empty(len(raws), np.int32)
                rc = _native_lib().krag_text_unigram_encode_batch(self._nat, len(raws), blob, offs.ctypes.data_as(C.c_void_p), cap,
                                                                  ids.ctypes.data_as(C.c_void_p), cnt.ctypes.data_as(C.c_void_p))
                if rc != 0 or int(cnt.max()) <= cap:
                    break
                cap = int(cnt.max())
            if rc == 0 and int(cnt.max()) <= cap:
                for j, i in enumerate(idx):
                    out[i] = ids[j, : cnt[j]].copy()
        for i, t in enumerate(texts):
            if out[i] is None:
                out[i] = np.asarray(self.encode_py(t), np.int32)
        return out
