// text_native.cpp -- host-side text analysis of the /index and /retrieve paths in native code (SURVEY.md section 8 f1):
//   * the bm25s analysis chain the reference reaches through BM25Retriever.from_defaults (hybrid_retriever.py:122-125):
//     lower-case, r"(?u)\b\w\w+\b" tokens, bm25s's 33 English stop words, Snowball English ("Porter2") stems -- PyStemmer
//     is C in the reference's stack too;
//   * BertTokenizer (uncased) as sentence-transformers runs it for bge (huggingface_local_embedding.py:34-53): BasicTokenizer
//     clean-up / lower-casing / punctuation split + greedy longest-match WordPiece -- HF tokenizers is native (Rust) there.
// Contract: the input is ASCII.  kaito_b200/text.py holds the Unicode-complete Python restatement, which is also the spec
// these functions are tested against (tests/test_text_native.py); the host calls the native path for ASCII text only.
// No CUDA in this file; it is part of libkaito_rag.so so that a cgo host gets the same analysis as the Python host.
#include <stdint.h>
#include <stddef.h>
#include <string.h>

#include <algorithm>
#include <memory>
#include <stdexcept>
#include <string>
#include <thread>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "../../include/kaito_rag.h"

namespace {

// ------------------------------------------------------------------------------------------ Snowball English
inline bool is_vowel(char c) { return c == 'a' || c == 'e' || c == 'i' || c == 'o' || c == 'u' || c == 'y'; }
inline bool ends_with(const std::string& w, const char* suf)
{
    const size_t n = strlen(suf);
    return w.size() >= n && memcmp(w.data() + w.size() - n, suf, n) == 0;
}
inline bool starts_with(const std::string& w, const char* pre)
{
    const size_t n = strlen(pre);
    return w.size() >= n && memcmp(w.data(), pre, n) == 0;
}
size_t region_after_vc(const std::string& w, size_t start)
{
    for (size_t i = start + 1; i < w.size(); ++i)
        if (!is_vowel(w[i]) && is_vowel(w[i - 1])) return i + 1;
    return w.size();
}
bool contains_vowel(const std::string& w, size_t n)   // over w[0, n)
{
    for (size_t i = 0; i < n && i < w.size(); ++i) if (is_vowel(w[i])) return true;
    return false;
}
bool ends_short_syllable(const std::string& w)
{
    const size_t n = w.size();
    if (n == 2) return is_vowel(w[0]) && !is_vowel(w[1]);
    if (n >= 3) {
        const char l = w[n - 1];
        return !is_vowel(w[n - 3]) && is_vowel(w[n - 2]) && !is_vowel(l) && l != 'w' && l != 'x' && l != 'Y';
    }
    return false;
}
bool ends_with_double(const std::string& w)
{
    static const char* D[] = {"bb", "dd", "ff", "gg", "mm", "nn", "pp", "rr", "tt"};
    for (const char* d : D) if (ends_with(w, d)) return true;
    return false;
}
std::string unmark(std::string w)
{
    for (char& c : w) if (c == 'Y') c = 'y';
    return w;
}

const std::unordered_map<std::string, std::string>& exceptions()
{
    static const std::unordered_map<std::string, std::string> m = {
        {"skis", "ski"}, {"skies", "sky"}, {"dying", "die"}, {"lying", "lie"}, {"tying", "tie"}, {"idly", "idl"},
        {"gently", "gentl"}, {"ugly", "ugli"}, {"early", "earli"}, {"only", "onli"}, {"singly", "singl"}, {"sky", "sky"},
        {"news", "news"}, {"howe", "howe"}, {"atlas", "atlas"}, {"cosmos", "cosmos"}, {"bias", "bias"}, {"andes", "andes"}};
    return m;
}
const std::unordered_set<std::string>& exceptions_1a()
{
    static const std::unordered_set<std::string> s = {"inning", "outing", "canning", "herring", "earring", "proceed", "exceed", "succeed"};
    return s;
}

std::string stem(const std::string& word)
{
    if (word.size() <= 2) return word;
    auto ex = exceptions().find(word);
    if (ex != exceptions().end()) return ex->second;
    std::string w = word[0] == '\'' ? word.substr(1) : word;
    for (size_t i = 0; i < w.size(); ++i)
        if (w[i] == 'y' && (i == 0 || is_vowel(w[i - 1]))) w[i] = 'Y';
    size_t r1;
    if (starts_with(w, "gener") || starts_with(w, "arsen")) r1 = 5;
    else if (starts_with(w, "commun")) r1 = 6;
    else r1 = region_after_vc(w, 0);
    const size_t r2 = region_after_vc(w, r1);

    // step 0
    if (ends_with(w, "'s'")) w.resize(w.size() - 3);
    else if (ends_with(w, "'s")) w.resize(w.size() - 2);
    else if (ends_with(w, "'")) w.resize(w.size() - 1);
    // step 1a
    if (ends_with(w, "sses")) w.resize(w.size() - 2);
    else if (ends_with(w, "ied") || ends_with(w, "ies")) w.resize(w.size() > 4 ? w.size() - 2 : w.size() - 1);
    else if (ends_with(w, "us") || ends_with(w, "ss")) { /* unchanged */ }
    else if (ends_with(w, "s")) { if (w.size() >= 2 && contains_vowel(w, w.size() - 2)) w.resize(w.size() - 1); }
    if (exceptions_1a().count(w)) return unmark(w);
    // step 1b
    if (ends_with(w, "eedly")) { if (w.size() - 5 >= r1) w.resize(w.size() - 3); }
    else if (ends_with(w, "eed")) { if (w.size() - 3 >= r1) w.resize(w.size() - 1); }
    else {
        static const char* S[] = {"ingly", "edly", "ing", "ed"};
        for (const char* suf : S) {
            if (!ends_with(w, suf)) continue;
            const size_t n = w.size() - strlen(suf);
            if (contains_vowel(w, n)) {
                w.resize(n);
                if (ends_with(w, "at") || ends_with(w, "bl") || ends_with(w, "iz")) w += 'e';
                else if (ends_with_double(w)) w.resize(w.size() - 1);
                else if (ends_short_syllable(w) && r1 >= w.size()) w += 'e';
            }
            break;
        }
    }
    // step 1c
    if (w.size() > 2 && (w.back() == 'y' || w.back() == 'Y') && !is_vowel(w[w.size() - 2])) w.back() = 'i';
    // step 2
    {
        static const char* S[][2] = {{"ization", "ize"}, {"ational", "ate"}, {"fulness", "ful"}, {"ousness", "ous"}, {"iveness", "ive"},
                                     {"tional", "tion"}, {"biliti", "ble"}, {"lessli", "less"}, {"entli", "ent"}, {"ation", "ate"},
                                     {"alism", "al"}, {"aliti", "al"}, {"ousli", "ous"}, {"iviti", "ive"}, {"fulli", "ful"}, {"enci", "ence"},
                                     {"anci", "ance"}, {"abli", "able"}, {"izer", "ize"}, {"ator", "ate"}, {"alli", "al"}, {"bli", "ble"},
                                     {"ogi", "og"}, {"li", ""}};
        for (auto& p : S) {
            if (!ends_with(w, p[0])) continue;
            const size_t ls = strlen(p[0]);
            if (w.size() - ls >= r1) {
                if (strcmp(p[0], "ogi") == 0) {
                    if (w.size() > ls && w[w.size() - ls - 1] == 'l') { w.resize(w.size() - ls); w += p[1]; }
                } else if (strcmp(p[0], "li") == 0) {
                    if (w.size() > 2 && strchr("cdeghkmnrt", w[w.size() - 3]) != nullptr) w.resize(w.size() - 2);
                } else {
                    w.resize(w.size() - ls); w += p[1];
                }
            }
            break;
        }
    }
    // step 3
    {
        static const char* S[][2] = {{"ational", "ate"}, {"tional", "tion"}, {"alize", "al"}, {"icate", "ic"}, {"iciti", "ic"}, {"ative", ""},
                                     {"ical", "ic"}, {"ness", ""}, {"ful", ""}};
        for (auto& p : S) {
            if (!ends_with(w, p[0])) continue;
            const size_t ls = strlen(p[0]);
            if (w.size() - ls >= r1) {
                if (strcmp(p[0], "ative") == 0) { if (w.size() - ls >= r2) w.resize(w.size() - ls); }
                else { w.resize(w.size() - ls); w += p[1]; }
            }
            break;
        }
    }
    // step 4
    {
        static const char* S[] = {"ement", "ance", "ence", "able", "ible", "ment", "ant", "ent", "ism", "ate", "iti", "ous", "ive", "ize",
                                  "ion", "al", "er", "ic"};
        for (const char* suf : S) {
            if (!ends_with(w, suf)) continue;
            const size_t ls = strlen(suf);
            if (w.size() - ls >= r2) {
                if (strcmp(suf, "ion") == 0) { if (w.size() > 3 && (w[w.size() - 4] == 's' || w[w.size() - 4] == 't')) w.resize(w.size() - 3); }
                else w.resize(w.size() - ls);
            }
            break;
        }
    }
    // step 5
    if (ends_with(w, "e")) {
        const std::string head = w.substr(0, w.size() - 1);
        if (w.size() - 1 >= r2 || (w.size() - 1 >= r1 && !ends_short_syllable(head))) w.resize(w.size() - 1);
    } else if (ends_with(w, "l")) {
        if (w.size() - 1 >= r2 && w.size() >= 2 && w[w.size() - 2] == 'l') w.resize(w.size() - 1);
    }
    return unmark(w);
}

const std::unordered_set<std::string>& stopwords()
{
    static const std::unordered_set<std::string> s = {
        "a", "an", "and", "are", "as", "at", "be", "but", "by", "for", "if", "in", "into", "is", "it", "no", "not", "of",
        "on", "or", "such", "that", "the", "their", "then", "there", "these", "they", "this", "to", "was", "will", "with"};
    return s;
}
inline bool is_word_char(unsigned char c) { return (c >= '0' && c <= '9') || (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z') || c == '_'; }
inline char lower(char c) { return (c >= 'A' && c <= 'Z') ? (char)(c + 32) : c; }

// stems of one ASCII text, '\n'-separated
void analyze(const char* text, int64_t len, std::string& out, int32_t& n)
{
    n = 0;
    std::string tok;
    for (int64_t i = 0; i <= len; ++i) {
        const bool wc = i < len && is_word_char((unsigned char)text[i]);
        if (wc) { tok += lower(text[i]); continue; }
        if (tok.size() >= 2 && !stopwords().count(tok)) {
            if (n) out += '\n';
            out += stem(tok);
            ++n;
        }
        tok.clear();
    }
}

// ------------------------------------------------------------------------------------------ WordPiece
inline bool is_ascii_punct(unsigned char c) { return (c >= 33 && c <= 47) || (c >= 58 && c <= 64) || (c >= 91 && c <= 96) || (c >= 123 && c <= 126); }

}  // namespace

struct krag_wordpiece {
    std::unordered_map<std::string, int32_t> vocab;
    int32_t unk = -1, cls = -1, sep = -1;
    bool lower_case = true;

    void piece(const std::string& word, std::vector<int32_t>& ids) const
    {
        if (word.size() > 100) { ids.push_back(unk); return; }
        const size_t mark = ids.size();
        size_t start = 0;
        std::string sub;
        while (start < word.size()) {
            size_t end = word.size();
            int32_t cur = -1;
            while (start < end) {
                sub.assign(start == 0 ? "" : "##");
                sub.append(word, start, end - start);
                auto it = vocab.find(sub);
                if (it != vocab.end()) { cur = it->second; break; }
                --end;
            }
            if (cur < 0) { ids.resize(mark); ids.push_back(unk); return; }
            ids.push_back(cur);
            start = end;
        }
    }
    // BasicTokenizer on ASCII + WordPiece; [CLS] ids[:max_len-2] [SEP]
    void encode(const char* text, int64_t len, int32_t max_len, std::vector<int32_t>& out) const
    {
        std::vector<int32_t> ids;
        std::string word;
        auto flush = [&] { if (!word.empty()) { piece(word, ids); word.clear(); } };
        for (int64_t i = 0; i < len; ++i) {
            const unsigned char c = (unsigned char)text[i];
            if (c == ' ' || c == '\t' || c == '\n' || c == '\r') { flush(); continue; }
            if (c < 0x20 || c == 0x7F) continue;                       // other control characters are dropped
            if (is_ascii_punct(c)) { flush(); word.assign(1, (char)c); flush(); continue; }
            word += lower_case ? lower((char)c) : (char)c;
        }
        flush();
        out.clear();
        out.push_back(cls);
        const size_t keep = max_len > 2 ? (size_t)(max_len - 2) : 0;
        out.insert(out.end(), ids.begin(), ids.begin() + (ids.size() < keep ? ids.size() : keep));
        out.push_back(sep);
    }
};

// ------------------------------------------------------------------------------------------ Unigram (XLM-R)
// The tokenizer.json of an XLM-R snapshot as the Rust `tokenizers` library runs it, over the tables kaito_b200/text.py
// (UnigramTokenizer, the spec) parsed: added tokens split out of the raw text, the Precompiled normaliser per grapheme
// cluster (for ASCII input every character is a cluster of its own except "\r\n"), Replace " {2,}" -> " ", Metaspace
// (after WhitespaceSplit when configured) and the Unigram Viterbi.
namespace {
inline int utf8_len(unsigned char c) { return c < 0x80 ? 1 : c < 0xE0 ? 2 : c < 0xF0 ? 3 : 4; }
uint32_t utf8_cp(const std::string& s, size_t i, int n)
{
    const unsigned char* p = (const unsigned char*)s.data() + i;
    if (n == 1) return p[0];
    if (n == 2) return ((p[0] & 0x1Fu) << 6) | (p[1] & 0x3Fu);
    if (n == 3) return ((p[0] & 0x0Fu) << 12) | ((p[1] & 0x3Fu) << 6) | (p[2] & 0x3Fu);
    return ((p[0] & 0x07u) << 18) | ((p[1] & 0x3Fu) << 12) | ((p[2] & 0x3Fu) << 6) | (p[3] & 0x3Fu);
}
// Rust char::is_whitespace: the Unicode White_Space property
inline bool white_space(uint32_t c)
{
    return (c >= 0x09 && c <= 0x0D) || c == 0x20 || c == 0x85 || c == 0xA0 || c == 0x1680 || (c >= 0x2000 && c <= 0x200A) ||
           c == 0x2028 || c == 0x2029 || c == 0x202F || c == 0x205F || c == 0x3000;
}
const char kMeta[] = "\xE2\x96\x81";   // U+2581, Metaspace's replacement
constexpr double kUnkPenalty = 10.0;
}  // namespace

struct krag_unigram {
    enum { COLLAPSE_SPACES = 1, WS_SPLIT = 2, PREPEND_FIRST = 4 };
    // pieces: a byte trie with one hash table of edges (node << 8 | byte) -> child; node_id[node] = piece id or -1
    std::unordered_map<uint64_t, int32_t> edge;
    std::vector<int32_t> node_id{-1};
    std::unordered_map<std::string, int32_t> ids;   // for a fused run of unknowns, looked up as a whole
    std::vector<double> score;
    int32_t unk = 0;
    double min_score = 0.0;
    // darts-clone double array of the precompiled charsmap and the NUL-terminated replacements after it
    std::vector<uint32_t> units;
    std::string repl;
    int flags = 0;
    struct Added { std::string s; int32_t id; bool lstrip, rstrip; };
    std::vector<Added> added;       // longest first: the first that matches at a position is the leftmost-longest match

    // replacement of the shortest charsmap key that prefixes key[0, n) (the Rust normaliser's results[0]), or null
    const char* charsmap(const char* key, size_t n) const
    {
        if (units.empty()) return nullptr;
        auto offset = [](uint32_t u) { return (size_t)((u >> 10) << ((u & (1u << 9)) >> 6)); };
        size_t node = offset(units[0]);
        for (size_t i = 0; i < n; ++i) {
            const unsigned char c = (unsigned char)key[i];
            if (c == 0) break;
            node ^= c;
            if (node >= units.size()) return nullptr;
            const uint32_t u = units[node];
            if ((u & ((1u << 31) | 0xFFu)) != c) return nullptr;
            node ^= offset(u);
            if ((u >> 8) & 1) {
                if (node >= units.size()) return nullptr;
                const size_t v = units[node] & ((1u << 31) - 1);
                return v < repl.size() ? repl.c_str() + v : nullptr;
            }
        }
        return nullptr;
    }
    void normalize(const char* s, size_t n, std::string& out) const
    {
        out.clear();
        for (size_t i = 0; i < n;) {
            const size_t g = (s[i] == '\r' && i + 1 < n && s[i + 1] == '\n') ? 2 : 1;   // ASCII grapheme clusters
            const char* r = charsmap(s + i, g);
            if (r) { out += r; i += g; continue; }
            for (size_t k = 0; k < g; ++k, ++i) {
                const char* rc = g > 1 ? charsmap(s + i, 1) : nullptr;
                if (rc) out += rc; else out += s[i];
            }
        }
        if (flags & COLLAPSE_SPACES) {
            size_t w = 0;
            for (size_t i = 0; i < out.size(); ++i)
                if (!(out[i] == ' ' && i > 0 && out[i - 1] == ' ')) out[w++] = out[i];   // out[i - 1] is still the input byte
            out.resize(w);
        }
    }
    void viterbi(const std::string& w, std::vector<int32_t>& ids_out) const
    {
        const size_t n = w.size();
        if (n == 0) return;
        struct Node { double best; int64_t start; int32_t id; };
        std::vector<Node> nodes(n + 1, Node{0.0, -1, 0});
        nodes[0].start = 0;
        const double unk_score = min_score - kUnkPenalty;
        for (size_t i = 0; i < n;) {
            const size_t mb = (size_t)utf8_len((unsigned char)w[i]);
            const double base = nodes[i].best;
            bool single = false;
            int32_t node = 0;
            for (size_t j = i; j < n; ++j) {
                auto it = edge.find(((uint64_t)node << 8) | (unsigned char)w[j]);
                if (it == edge.end()) break;
                node = it->second;
                const int32_t id = node_id[(size_t)node];
                if (id < 0) continue;
                Node& t = nodes[j + 1];
                const double c = score[(size_t)id] + base;
                if (t.start < 0 || c > t.best) { t.best = c; t.start = (int64_t)i; t.id = id; }
                if (j + 1 - i == mb) single = true;
            }
            if (!single) {
                Node& t = nodes[i + mb];
                const double c = unk_score + base;
                if (t.start < 0 || c > t.best) { t.best = c; t.start = (int64_t)i; t.id = unk; }
            }
            i += mb;
        }
        const size_t mark = ids_out.size();
        int64_t end = (int64_t)n, run_end = -1;
        auto flush_run = [&](int64_t from) {
            auto it = ids.find(w.substr((size_t)from, (size_t)(run_end - from)));
            ids_out.push_back(it == ids.end() ? unk : it->second);
            run_end = -1;
        };
        while (end > 0) {
            const Node& t = nodes[(size_t)end];
            if (t.id == unk) { if (run_end < 0) run_end = end; }
            else {
                if (run_end >= 0) flush_run(end);
                ids_out.push_back(t.id);
            }
            end = t.start;
        }
        if (run_end >= 0) flush_run(0);
        std::reverse(ids_out.begin() + (ptrdiff_t)mark, ids_out.end());
    }
    // Metaspace over one normalised segment (after WhitespaceSplit when configured), then the Viterbi of every piece
    void pre_tokenize(const std::string& s, bool at_origin, std::vector<int32_t>& out) const
    {
        std::string word, piece;
        auto emit = [&](size_t from, size_t to) {
            word.clear();
            for (size_t i = from; i < to; ++i) { if (s[i] == ' ') word += kMeta; else word += s[i]; }
            if (word.empty()) return;
            const bool prepend = word.compare(0, 3, kMeta) != 0 && (!(flags & PREPEND_FIRST) || (at_origin && from == 0));
            if (prepend) word.insert(0, kMeta);
            size_t p0 = 0;
            for (size_t i = 3; i + 3 <= word.size(); ++i)
                if (word.compare(i, 3, kMeta) == 0) { viterbi(word.substr(p0, i - p0), out); p0 = i; i += 2; }
            viterbi(word.substr(p0), out);
        };
        if (!(flags & WS_SPLIT)) { emit(0, s.size()); return; }
        size_t start = SIZE_MAX;
        for (size_t i = 0; i < s.size();) {
            const int m = utf8_len((unsigned char)s[i]);
            const bool ws = white_space(utf8_cp(s, i, m));
            if (ws && start != SIZE_MAX) { emit(start, i); start = SIZE_MAX; }
            else if (!ws && start == SIZE_MAX) start = i;
            i += (size_t)m;
        }
        if (start != SIZE_MAX) emit(start, s.size());
    }
    // ids of one ASCII text without <s> / </s>
    void encode(const char* t, size_t n, std::vector<int32_t>& out) const
    {
        out.clear();
        std::string norm;
        auto segment = [&](size_t a, size_t b) {
            normalize(t + a, b - a, norm);
            pre_tokenize(norm, a == 0, out);
        };
        auto ws = [&](char c) { return c == ' ' || (c >= 0x09 && c <= 0x0D); };
        size_t pos = 0;
        for (size_t i = 0; i < n;) {
            const Added* m = nullptr;
            for (const Added& a : added)
                if (a.s.size() <= n - i && memcmp(t + i, a.s.data(), a.s.size()) == 0) { m = &a; break; }
            if (!m) { ++i; continue; }
            size_t start = i, stop = i + m->s.size();
            if (m->lstrip) { while (start > pos && ws(t[start - 1])) --start; }
            if (m->rstrip) { while (stop < n && ws(t[stop])) ++stop; }
            if (pos < start) segment(pos, start);
            out.push_back(m->id);
            pos = i = stop;
        }
        if (pos < n) segment(pos, n);
    }
};

namespace {
thread_local std::string g_text_err;
template <class F>
int32_t text_guard(F&& f)
{
    try { f(); return KRAG_OK; }
    catch (const std::bad_alloc&) { return KRAG_E_OOM; }
    catch (const std::exception&) { return KRAG_E_INVALID; }
}
template <class F>
void parallel_for(int64_t n, int64_t total_bytes, F&& body)
{
    unsigned hw = std::thread::hardware_concurrency();
    int64_t nt = hw ? hw : 4;
    if (nt > n / 8) nt = n / 8;          // a thread per >= 8 texts ...
    if (nt > total_bytes / 32768) nt = total_bytes / 32768;   // ... and per >= 32 KB of text: a batch of queries is not worth a thread
    if (nt <= 1) { for (int64_t i = 0; i < n; ++i) body(i); return; }
    std::vector<std::thread> th;
    for (int64_t t = 0; t < nt; ++t)
        th.emplace_back([&, t] { for (int64_t i = t; i < n; i += nt) body(i); });
    for (auto& x : th) x.join();
}
}  // namespace

extern "C" {

int32_t krag_text_analyze(const char* text, int64_t len, char* out, int64_t cap, int64_t* out_len, int32_t* n_terms)
{
    return text_guard([&] {
        if (!text || !out_len || !n_terms || len < 0) throw std::invalid_argument("null argument");
        std::string s;
        int32_t n = 0;
        analyze(text, len, s, n);
        *out_len = (int64_t)s.size();
        *n_terms = n;
        if (out && (int64_t)s.size() <= cap) memcpy(out, s.data(), s.size());
    });
}

int32_t krag_wordpiece_create(const char* vocab, int64_t len, int32_t lower_case, krag_wordpiece** out)
{
    return krag_wordpiece_create_specials(vocab, len, lower_case, "[UNK]", "[CLS]", "[SEP]", out);
}

int32_t krag_wordpiece_create_specials(const char* vocab, int64_t len, int32_t lower_case, const char* unk_token,
                                       const char* cls_token, const char* sep_token, krag_wordpiece** out)
{
    return text_guard([&] {
        if (!vocab || !out || len < 0 || !unk_token || !cls_token || !sep_token) throw std::invalid_argument("null argument");
        krag_wordpiece* w = new krag_wordpiece();
        w->lower_case = lower_case != 0;
        // one token per line, exactly like "\n".join(tokens).split("\n"); a repeated token keeps its LAST id (dict semantics)
        int32_t id = 0;
        const char* p = vocab; const char* e = vocab + len;
        for (;;) {
            const char* nl = (const char*)memchr(p, '\n', (size_t)(e - p));
            const char* q = nl ? nl : e;
            w->vocab[std::string(p, q)] = id++;
            if (!nl) break;
            p = nl + 1;
        }
        auto need = [&](const char* t) { auto it = w->vocab.find(t); if (it == w->vocab.end()) { delete w; throw std::invalid_argument(t); } return it->second; };
        w->unk = need(unk_token); w->cls = need(cls_token); w->sep = need(sep_token);
        *out = w;
    });
}

int32_t krag_wordpiece_encode_batch(const krag_wordpiece* w, int64_t n, const char* texts, const int64_t* offsets /*[n+1]*/,
                                    int32_t max_len, int32_t* out_ids /*[n * max_len]*/, int32_t* out_n /*[n]*/)
{
    return text_guard([&] {
        if (!w || !texts || !offsets || !out_ids || !out_n || n < 0 || max_len < 2) throw std::invalid_argument("bad argument");
        parallel_for(n, offsets[n] - offsets[0], [&](int64_t i) {
            std::vector<int32_t> ids;
            w->encode(texts + offsets[i], offsets[i + 1] - offsets[i], max_len, ids);
            out_n[i] = (int32_t)ids.size();
            memcpy(out_ids + i * (int64_t)max_len, ids.data(), ids.size() * sizeof(int32_t));
        });
    });
}

int32_t krag_wordpiece_destroy(krag_wordpiece* w)
{
    delete w;
    return KRAG_OK;
}

int32_t krag_text_unigram_create(const char* pieces, const int64_t* piece_off, const double* scores, int64_t n_pieces, int32_t unk_id,
                                 const char* charsmap, int64_t charsmap_len, int32_t flags, const char* added, const int64_t* added_off,
                                 const int32_t* added_ids, const int32_t* added_strip, int32_t n_added, krag_unigram** out)
{
    return text_guard([&] {
        if (!pieces || !piece_off || !scores || !out || n_pieces < 1 || unk_id < 0 || unk_id >= n_pieces || charsmap_len < 0 ||
            n_added < 0 || (n_added && (!added || !added_off || !added_ids || !added_strip)) || (charsmap_len && !charsmap))
            throw std::invalid_argument("bad argument");
        auto u = std::make_unique<krag_unigram>();
        u->unk = unk_id;
        u->flags = flags;
        u->score.assign(scores, scores + n_pieces);
        u->min_score = *std::min_element(u->score.begin(), u->score.end());
        for (int64_t p = 0; p < n_pieces; ++p) {
            const std::string s(pieces + piece_off[p], (size_t)(piece_off[p + 1] - piece_off[p]));
            u->ids[s] = (int32_t)p;                     // a repeated piece keeps its last id
            int32_t node = 0;
            for (unsigned char c : s) {
                auto it = u->edge.find(((uint64_t)node << 8) | c);
                if (it == u->edge.end()) {
                    it = u->edge.emplace(((uint64_t)node << 8) | c, (int32_t)u->node_id.size()).first;
                    u->node_id.push_back(-1);
                }
                node = it->second;
            }
            if (node) u->node_id[(size_t)node] = (int32_t)p;
        }
        if (charsmap_len) {
            uint32_t n = 0;
            memcpy(&n, charsmap, 4);                    // little-endian hosts only (x86-64, aarch64)
            if (charsmap_len < 4 || n % 4 || 4 + (int64_t)n > charsmap_len) throw std::invalid_argument("charsmap");
            u->units.resize(n / 4);
            memcpy(u->units.data(), charsmap + 4, n);
            u->repl.assign(charsmap + 4 + n, (size_t)(charsmap_len - 4 - n));
        }
        for (int32_t a = 0; a < n_added; ++a)
            u->added.push_back({std::string(added + added_off[a], (size_t)(added_off[a + 1] - added_off[a])), added_ids[a],
                                (added_strip[a] & 1) != 0, (added_strip[a] & 2) != 0});
        std::stable_sort(u->added.begin(), u->added.end(), [](const krag_unigram::Added& x, const krag_unigram::Added& y) {
            return x.s.size() > y.s.size();
        });
        u->added.erase(std::remove_if(u->added.begin(), u->added.end(), [](const krag_unigram::Added& x) { return x.s.empty(); }),
                       u->added.end());
        *out = u.release();
    });
}

int32_t krag_text_unigram_encode_batch(const krag_unigram* u, int64_t n, const char* texts, const int64_t* offsets /*[n+1]*/,
                                       int32_t cap, int32_t* out_ids /*[n * cap]*/, int32_t* out_n /*[n]*/)
{
    return text_guard([&] {
        if (!u || !texts || !offsets || !out_ids || !out_n || n < 0 || cap < 1) throw std::invalid_argument("bad argument");
        parallel_for(n, offsets[n] - offsets[0], [&](int64_t i) {
            std::vector<int32_t> ids;
            u->encode(texts + offsets[i], (size_t)(offsets[i + 1] - offsets[i]), ids);
            out_n[i] = (int32_t)ids.size();
            memcpy(out_ids + i * (int64_t)cap, ids.data(), std::min(ids.size(), (size_t)cap) * sizeof(int32_t));
        });
    });
}

int32_t krag_text_unigram_destroy(krag_unigram* u)
{
    delete u;
    return KRAG_OK;
}

}  // extern "C"
