// Character n-gram LM (plain-text ARPA) for the CTC prefix beam search: host loader, packed tables and the query kernel.
// Replaces the external decoder's Scorer (masr/decoders/swig_wrapper.py:4-18) for character-based LMs; semantics
// oracle/lm.py.  The real LMs are gigabytes of ARPA, so the file is parsed here in C++ (one pass, no per-line Python).
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <unordered_map>
#include <vector>

#include "common.cuh"
#include "lm.cuh"

namespace masr {
namespace {

struct Gram {
    uint32_t k0, k1, k2;
    float p, bo;
    uint32_t k3;                   // word tables only (24-bit ids fill 4 words)
};

struct LmHandle {
    int order = 0, char_based = 1, V = 0, bos = 0, eos = 0;
    int64_t dict_size = 0;
    int64_t read[LM_MAX_ORDER + 1] = {0}, kept[LM_MAX_ORDER + 1] = {0}, slots[LM_MAX_ORDER + 1] = {0};
    int64_t off[LM_MAX_ORDER + 1] = {0};
    std::vector<uint32_t> keys;    // 4 per slot
    std::vector<float> vals;       // 2 per slot
    std::vector<int> tok2lm;
    // word LM (masr_word_lm_load_arpa): the <space> token and the lexicon trie in CSR form
    int word = 0, space = -1;
    std::vector<int> lex_off, lex_tok, lex_next, lex_word;
};

// UTF-8 code points of s -> their first model token ids; false if one is not a model token
bool spell(const std::string& s, const std::unordered_map<std::string, int>& vid, std::vector<int>& out) {
    out.clear();
    for (size_t i = 0; i < s.size();) {
        const unsigned char c = (unsigned char)s[i];
        size_t n = c < 0x80 ? 1 : (c >> 5) == 6 ? 2 : (c >> 4) == 14 ? 3 : 4;
        if (i + n > s.size()) n = s.size() - i;
        auto it = vid.find(s.substr(i, n));
        if (it == vid.end()) return false;
        out.push_back(it->second);
        i += n;
    }
    return !out.empty();
}

// The lexicon of a word LM: every unigram except <s>, </s>, <unk> that spells as model tokens, ids in file order;
// fills H.lex_* (CSR, arcs ascending by token), H.dict_size and lmw (word -> id, -1 = not in the lexicon).
void build_lexicon(const std::vector<std::string>& uni, const std::unordered_map<std::string, int>& vid, LmHandle& H,
                   std::unordered_map<std::string, int>& lmw) {
    std::vector<std::vector<std::pair<int, int>>> arcs(1);
    std::vector<int> wend(1, -1);
    std::vector<int> toks;
    int nwords = 0;
    for (const std::string& w : uni) {
        if (w == "<s>" || w == "</s>" || w == "<unk>" || lmw.count(w)) continue;
        if (!spell(w, vid, toks)) { lmw[w] = -1; continue; }
        int n = 0;
        for (int t : toks) {
            int nxt = -1;
            for (const auto& a : arcs[n]) if (a.first == t) { nxt = a.second; break; }
            if (nxt < 0) {
                nxt = (int)arcs.size();
                arcs[n].push_back({t, nxt});
                arcs.emplace_back();
                wend.push_back(-1);
            }
            n = nxt;
        }
        wend[n] = nwords;
        lmw[w] = nwords++;
    }
    H.dict_size = nwords;
    H.bos = nwords;
    H.eos = nwords + 1;
    lmw["<s>"] = H.bos;
    lmw["</s>"] = H.eos;
    lmw["<unk>"] = -1;
    H.lex_off.assign(1, 0);
    for (auto& a : arcs) {
        std::sort(a.begin(), a.end());
        for (const auto& e : a) { H.lex_tok.push_back(e.first); H.lex_next.push_back(e.second); }
        H.lex_off.push_back((int)H.lex_tok.size());
    }
    H.lex_word = std::move(wend);
}

int utf8_code_points(const char* s, size_t n) {
    int c = 0;
    for (size_t i = 0; i < n; ++i) c += ((unsigned char)s[i] & 0xC0) != 0x80;
    return c;
}

float to_ln(double log10v) { return (float)(log10v * 2.302585092994046); }   // float32(double(v) * ln 10)

// strip trailing '\r' / '\n' / blanks and leading blanks in place; returns the trimmed start
char* trim(char* s) {
    size_t n = strlen(s);
    while (n && (s[n - 1] == '\n' || s[n - 1] == '\r' || s[n - 1] == ' ' || s[n - 1] == '\t')) s[--n] = 0;
    while (*s == ' ' || *s == '\t') ++s;
    return s;
}

struct LineReader {
    FILE* f;
    char* buf = nullptr;
    size_t cap = 0;
    int64_t lineno = 0;
    char* cur = nullptr;
    bool next() {
        if (getline(&buf, &cap, f) < 0) return false;
        ++lineno;
        cur = trim(buf);
        return true;
    }
    ~LineReader() { free(buf); }
};

#define LM_FAIL(...)                     \
    do {                                 \
        set_last_error(__VA_ARGS__);     \
        return MASR_ERR_INVALID_ARGUMENT; \
    } while (0)

int parse_arpa(const char* path, const char* vocab, int V, LmHandle& H, bool word = false) {
    const char* fn = word ? "masr_word_lm_load_arpa" : "masr_lm_load_arpa";
    H.word = word;
    FILE* f = fopen(path, "rb");
    if (!f) LM_FAIL("%s: cannot open %s", fn, path);
    char head[8] = {0};
    const size_t nh = fread(head, 1, 7, f);
    if (nh == 7 && memcmp(head, "mmap lm", 7) == 0) {
        fclose(f);
        LM_FAIL("%s: %s is a KenLM binary (mmap lm); only plain-text ARPA is supported", fn, path);
    }
    rewind(f);
    struct Closer { FILE* f; ~Closer() { fclose(f); } } closer{f};
    // model vocabulary: string -> first token id
    std::unordered_map<std::string, int> vid;
    {
        const char* s = vocab;
        for (int i = 0; i < V; ++i) {
            const char* e = strchr(s, '\n');
            const size_t n = e ? (size_t)(e - s) : strlen(s);
            vid.emplace(std::string(s, n), i);
            if (!e && i + 1 < V) LM_FAIL("%s: vocabulary has fewer than %d entries", fn, V);
            s = e ? e + 1 : s + n;
        }
    }
    H.V = V;
    H.bos = V;
    H.eos = V + 1;
    if (word) {
        auto it = vid.find("<space>");
        if (it == vid.end()) LM_FAIL("%s: the vocabulary has no <space> token: a word LM needs one", fn);
        H.space = it->second;
    }
    LineReader R{f};
    bool found = false;
    while (R.next())
        if (strcmp(R.cur, "\\data\\") == 0) { found = true; break; }
    if (!found) LM_FAIL("%s: %s: missing \\data\\ section", fn, path);
    int64_t counts[LM_MAX_ORDER + 2] = {0};
    int order = 0;
    bool have_line = R.next();
    while (have_line && strncmp(R.cur, "ngram ", 6) == 0) {
        int k = 0;
        long long c = -1;
        char tail = 0;
        if (sscanf(R.cur + 6, "%d=%lld%c", &k, &c, &tail) != 2)
            LM_FAIL("%s: %s:%lld: malformed line '%s'", fn, path, (long long)R.lineno, R.cur);
        if (k != order + 1 || c < 0) LM_FAIL("%s: %s:%lld: count mismatch '%s'", fn, path, (long long)R.lineno, R.cur);
        if (k > LM_MAX_ORDER) LM_FAIL("%s: %s: order %d > %d is not supported", fn, path, k, LM_MAX_ORDER);
        order = k;
        counts[k] = c;
        have_line = R.next();
    }
    if (order == 0) LM_FAIL("%s: %s: \\data\\ section declares no n-gram counts", fn, path);
    if (word && order > WLM_MAX_ORDER) LM_FAIL("%s: %s: word LM order %d > %d is not supported", fn, path, order, WLM_MAX_ORDER);
    if (word && counts[1] > (int64_t)WLM_MAX_IDS)
        LM_FAIL("%s: %s: %lld unigrams exceed the 24-bit word ids of the word LM tables (at most %lld)", fn, path,
                (long long)counts[1], (long long)WLM_MAX_IDS);
    H.order = order;
    std::unordered_map<std::string, int> lmw;     // LM word -> LM id (-1: not a model token -> n-grams with it are dropped)
    std::vector<std::vector<Gram>> grams(order + 1);
    bool has_bos = false, has_eos = false;
    std::vector<std::string> uni;                 // word LM: unigrams in file order (ids are assigned after the section)
    for (int n = 1; n <= order; ++n) {
        while (have_line && R.cur[0] == 0) have_line = R.next();
        char want[32];
        snprintf(want, sizeof(want), "\\%d-grams:", n);
        if (!have_line || strcmp(R.cur, want) != 0) LM_FAIL("%s: %s: section mismatch: expected %s", fn, path, want);
        int64_t nread = 0;
        grams[n].reserve((size_t)counts[n]);
        while ((have_line = R.next()) && R.cur[0] != 0 && R.cur[0] != '\\') {
            char* fields[LM_MAX_ORDER + 3];
            int nf = 0;
            for (char* p = R.cur; *p;) {
                while (*p == ' ' || *p == '\t') ++p;
                if (!*p) break;
                if (nf == n + 2) { nf = n + 3; break; }
                fields[nf++] = p;
                while (*p && *p != ' ' && *p != '\t') ++p;
                if (*p) *p++ = 0;
            }
            if (nf != n + 1 && nf != n + 2)
                LM_FAIL("%s: %s:%lld: malformed line (%d fields in a %d-gram)", fn, path, (long long)R.lineno, nf, n);
            char* end = nullptr;
            const double p = strtod(fields[0], &end);
            if (end == fields[0] || *end) LM_FAIL("%s: %s:%lld: malformed probability '%s'", fn, path, (long long)R.lineno, fields[0]);
            double bo = 0.0;
            if (nf == n + 2) {
                bo = strtod(fields[n + 1], &end);
                if (end == fields[n + 1] || *end) LM_FAIL("%s: %s:%lld: malformed backoff '%s'", fn, path, (long long)R.lineno, fields[n + 1]);
            }
            ++nread;
            Gram g{0, 0, 0, to_ln(p), to_ln(bo), 0};
            bool keep = true;
            if (word && n == 1) {
                const char* w = fields[1];
                const bool special = !strcmp(w, "<s>") || !strcmp(w, "</s>") || !strcmp(w, "<unk>");
                if (!special && utf8_code_points(w, strlen(w)) != 1) H.char_based = 0;
                has_bos |= !strcmp(w, "<s>");
                has_eos |= !strcmp(w, "</s>");
                uni.emplace_back(w);
                grams[1].push_back(g);                // keys filled in once the lexicon is built
                continue;
            }
            for (int j = 0; j < n; ++j) {
                int id;
                if (n == 1) {
                    const char* w = fields[1];
                    const size_t len = strlen(w);
                    const bool special = !strcmp(w, "<s>") || !strcmp(w, "</s>") || !strcmp(w, "<unk>");
                    if (!special && utf8_code_points(w, len) != 1) H.char_based = 0;
                    if (!strcmp(w, "<s>")) { id = H.bos; has_bos = true; }
                    else if (!strcmp(w, "</s>")) { id = H.eos; has_eos = true; }
                    else if (!strcmp(w, "<unk>")) id = -1;
                    else {
                        auto it = vid.find(std::string(w, len));
                        id = it == vid.end() ? -1 : it->second;
                    }
                    lmw[std::string(w, len)] = id;
                } else {
                    auto it = lmw.find(fields[1 + j]);
                    id = it == lmw.end() ? -1 : it->second;
                }
                if (id < 0) { keep = false; break; }
                if (word) {
                    uint32_t k[4] = {g.k0, g.k1, g.k2, g.k3};
                    wlm_put(k, j, (uint32_t)id);
                    g.k0 = k[0]; g.k1 = k[1]; g.k2 = k[2]; g.k3 = k[3];
                } else if (j < 2) g.k0 |= (uint32_t)id << (16 * j);
                else if (j < 4) g.k1 |= (uint32_t)id << (16 * (j - 2));
                else g.k2 |= (uint32_t)id << (16 * (j - 4));
            }
            if (keep) grams[n].push_back(g);
        }
        if (nread != counts[n])
            LM_FAIL("%s: %s: count mismatch: \\%d-grams: has %lld entries, \\data\\ says %lld", fn, path, n,
                    (long long)nread, (long long)counts[n]);
        H.read[n] = nread;
        if (n == 1) H.dict_size = nread;
        if (word && n == 1) {
            build_lexicon(uni, vid, H, lmw);
            std::vector<Gram> kept;
            for (size_t i = 0; i < uni.size(); ++i) {
                const int id = lmw[uni[i]];
                if (id < 0) continue;
                Gram g = grams[1][i];
                uint32_t k[4] = {0, 0, 0, 0};
                wlm_put(k, 0, (uint32_t)id);
                g.k0 = k[0]; g.k1 = k[1]; g.k2 = k[2]; g.k3 = k[3];
                kept.push_back(g);
            }
            grams[1].swap(kept);
        }
    }
    while (have_line && R.cur[0] == 0) have_line = R.next();
    if (!have_line || strcmp(R.cur, "\\end\\") != 0) LM_FAIL("%s: %s: section mismatch: expected \\end\\", fn, path);
    if (!has_bos || !has_eos) LM_FAIL("%s: %s: %s is not a unigram", fn, path, has_bos ? "</s>" : "<s>");
    if (word && H.char_based) LM_FAIL("%s: %s is a character-based LM, not a word LM (use masr_lm_load_arpa)", fn, path);
    // model token -> LM id: the token's string is an LM unigram other than <unk>
    // (duplicate token strings share the first token's id)
    H.tok2lm.assign(V, -1);
    if (!word) {
        const char* s = vocab;
        for (int i = 0; i < V; ++i) {
            const char* e = strchr(s, '\n');
            const size_t n = e ? (size_t)(e - s) : strlen(s);
            auto it = lmw.find(std::string(s, n));
            H.tok2lm[i] = it == lmw.end() ? -1 : it->second;
            s = e ? e + 1 : s + n;
        }
    }
    // open-addressing tables, load <= 1/2
    int64_t total = 0;
    for (int n = 1; n <= order; ++n) {
        int64_t cap = 16;
        while (cap < 2 * (int64_t)grams[n].size()) cap <<= 1;
        H.kept[n] = (int64_t)grams[n].size();
        H.slots[n] = cap;
        H.off[n] = total;
        total += cap;
    }
    H.keys.assign((size_t)total * 4, 0);
    H.vals.assign((size_t)total * 2, 0.f);
    for (int64_t s = 0; s < total; ++s) H.keys[s * 4] = LM_EMPTY;
    for (int n = 1; n <= order; ++n) {
        const uint64_t mask = (uint64_t)H.slots[n] - 1;
        for (const Gram& g : grams[n]) {
            uint64_t s = (word ? wlm_hash(g.k0, g.k1, g.k2, g.k3) : lm_hash(g.k0, g.k1, g.k2)) & mask;
            for (;;) {
                uint32_t* k = &H.keys[(H.off[n] + s) * 4];
                if (k[0] == LM_EMPTY || (k[0] == g.k0 && k[1] == g.k1 && k[2] == g.k2 && k[3] == g.k3)) {   // a repeated n-gram: the last wins
                    k[0] = g.k0; k[1] = g.k1; k[2] = g.k2; k[3] = g.k3;
                    H.vals[(H.off[n] + s) * 2] = g.p;
                    H.vals[(H.off[n] + s) * 2 + 1] = g.bo;
                    break;
                }
                s = (s + 1) & mask;
            }
        }
        std::vector<Gram>().swap(grams[n]);
    }
    return MASR_OK;
}

// ---------------------------------------------------------------------------------------------------------------
__global__ void lm_score_kernel(const masr_lm_tables lm, const int* __restrict__ ctx, const int* __restrict__ word, int Q,
                                float* __restrict__ out) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= Q) return;
    const int n1 = lm.order - 1;
    auto id = [&](int t) -> uint16_t { return t == -1 ? (uint16_t)lm.bos : t == -2 ? (uint16_t)lm.eos : lm_word(lm, t); };
    uint16_t h[LM_CTX];
    for (int j = 0; j < n1; ++j) h[j] = id(ctx[(int64_t)q * n1 + j]);
    out[q] = lm_lnp(lm, h, id(word[q]));
}

__global__ void word_lm_score_kernel(const masr_word_lm_tables lm, const int* __restrict__ ctx, const int* __restrict__ word,
                                     int Q, float* __restrict__ out) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= Q) return;
    const int n1 = lm.order - 1;
    const int nid = lm.dict_size + 2;
    auto id = [&](int w) -> uint32_t { return w < 0 || w >= nid ? WLM_OOV : (uint32_t)w; };
    uint32_t h[WLM_CTX];
    for (int j = 0; j < n1; ++j) h[j] = id(ctx[(int64_t)q * n1 + j]);
    out[q] = wlm_lnp(lm, h, id(word[q]));
}

}  // namespace
}  // namespace masr

using namespace masr;

extern "C" int masr_lm_load_arpa(const char* path_host, const char* vocab_host, int V, void** handle_host) {
    MASR_REQUIRE(path_host && vocab_host && handle_host, "masr_lm_load_arpa: null pointer");
    MASR_REQUIRE(V >= 1 && V <= 0xFFFF - 3, "masr_lm_load_arpa: vocabulary size %d out of range (1..65532)", V);
    *handle_host = nullptr;
    LmHandle* H = new LmHandle();
    const int rc = parse_arpa(path_host, vocab_host, V, *H);
    if (rc != MASR_OK) { delete H; return rc; }
    *handle_host = H;
    return MASR_OK;
}

extern "C" int masr_lm_info(const void* handle_host, int64_t* info_host) {
    MASR_REQUIRE(handle_host && info_host, "masr_lm_info: null pointer");
    const LmHandle& H = *static_cast<const LmHandle*>(handle_host);
    for (int i = 0; i < 32; ++i) info_host[i] = 0;
    info_host[MASR_LM_INFO_ORDER] = H.order;
    info_host[MASR_LM_INFO_CHAR_BASED] = H.char_based;
    info_host[MASR_LM_INFO_DICT_SIZE] = H.dict_size;
    info_host[MASR_LM_INFO_VOCAB] = H.V;
    info_host[MASR_LM_INFO_KEY_WORDS] = (int64_t)H.keys.size();
    info_host[MASR_LM_INFO_VAL_FLOATS] = (int64_t)H.vals.size();
    info_host[MASR_LM_INFO_BOS] = H.bos;
    info_host[MASR_LM_INFO_EOS] = H.eos;
    for (int n = 1; n <= LM_MAX_ORDER; ++n) {
        info_host[MASR_LM_INFO_READ + n - 1] = H.read[n];
        info_host[MASR_LM_INFO_KEPT + n - 1] = H.kept[n];
        info_host[MASR_LM_INFO_SLOTS + n - 1] = H.slots[n];
    }
    info_host[MASR_LM_INFO_TABLE_BYTES] = (int64_t)(H.keys.size() * 4 + H.vals.size() * 4 + H.tok2lm.size() * 4);
    return MASR_OK;
}

extern "C" int masr_lm_export(const void* handle_host, uint32_t* keys_host, float* vals_host, int* tok2lm_host,
                              masr_lm_tables* layout_host) {
    MASR_REQUIRE(handle_host && keys_host && vals_host && tok2lm_host && layout_host, "masr_lm_export: null pointer");
    const LmHandle& H = *static_cast<const LmHandle*>(handle_host);
    memcpy(keys_host, H.keys.data(), H.keys.size() * sizeof(uint32_t));
    memcpy(vals_host, H.vals.data(), H.vals.size() * sizeof(float));
    memcpy(tok2lm_host, H.tok2lm.data(), H.tok2lm.size() * sizeof(int));
    memset(layout_host, 0, sizeof(*layout_host));
    layout_host->order = H.order;
    layout_host->bos = H.bos;
    layout_host->eos = H.eos;
    layout_host->vocab = H.V;
    for (int n = 1; n <= H.order; ++n) {
        layout_host->off[n] = H.off[n];
        layout_host->mask[n] = H.slots[n] - 1;
    }
    return MASR_OK;
}

extern "C" int masr_lm_free(void* handle_host) {
    delete static_cast<LmHandle*>(handle_host);
    return MASR_OK;
}

extern "C" int masr_lm_score_f32(const masr_lm_tables* lm_host, const int* ctx, const int* word, int Q, float* out, void* stream) {
    if (Q == 0) return MASR_OK;
    MASR_REQUIRE(lm_host && lm_host->keys && lm_host->vals && lm_host->tok2lm && word && out && (ctx || lm_host->order == 1),
                 "masr_lm_score_f32: null pointer");
    MASR_REQUIRE(lm_host->order >= 1 && lm_host->order <= LM_MAX_ORDER, "masr_lm_score_f32: order %d out of range", lm_host->order);
    lm_score_kernel<<<(Q + 255) / 256, 256, 0, (cudaStream_t)stream>>>(*lm_host, ctx, word, Q, out);
    return check_launch("lm_score_kernel");
}

// ---- word LM ----------------------------------------------------------------------------------------------------
extern "C" int masr_word_lm_load_arpa(const char* path_host, const char* vocab_host, int V, void** handle_host) {
    MASR_REQUIRE(path_host && vocab_host && handle_host, "masr_word_lm_load_arpa: null pointer");
    MASR_REQUIRE(V >= 1, "masr_word_lm_load_arpa: vocabulary size %d out of range", V);
    *handle_host = nullptr;
    LmHandle* H = new LmHandle();
    const int rc = parse_arpa(path_host, vocab_host, V, *H, true);
    if (rc != MASR_OK) { delete H; return rc; }
    *handle_host = H;
    return MASR_OK;
}

extern "C" int masr_word_lm_info(const void* handle_host, int64_t* info_host) {
    MASR_REQUIRE(handle_host && info_host, "masr_word_lm_info: null pointer");
    const LmHandle& H = *static_cast<const LmHandle*>(handle_host);
    MASR_REQUIRE(H.word, "masr_word_lm_info: not a word LM handle");
    const int rc = masr_lm_info(handle_host, info_host);
    if (rc != MASR_OK) return rc;
    info_host[MASR_LM_INFO_TABLE_BYTES] =
        (int64_t)(H.keys.size() + H.vals.size() + H.lex_off.size() + 2 * H.lex_tok.size() + H.lex_word.size()) * 4;
    info_host[MASR_WORD_LM_INFO_NODES] = (int64_t)H.lex_word.size();
    info_host[MASR_WORD_LM_INFO_ARCS] = (int64_t)H.lex_tok.size();
    info_host[MASR_WORD_LM_INFO_SPACE] = H.space;
    return MASR_OK;
}

extern "C" int masr_word_lm_export(const void* handle_host, uint32_t* keys_host, float* vals_host, int* lex_off_host,
                                   int* lex_tok_host, int* lex_next_host, int* lex_word_host, masr_word_lm_tables* layout_host) {
    MASR_REQUIRE(handle_host && keys_host && vals_host && lex_off_host && lex_word_host && layout_host &&
                 ((lex_tok_host && lex_next_host) || static_cast<const LmHandle*>(handle_host)->lex_tok.empty()),
                 "masr_word_lm_export: null pointer");
    const LmHandle& H = *static_cast<const LmHandle*>(handle_host);
    MASR_REQUIRE(H.word, "masr_word_lm_export: not a word LM handle");
    memcpy(keys_host, H.keys.data(), H.keys.size() * sizeof(uint32_t));
    memcpy(vals_host, H.vals.data(), H.vals.size() * sizeof(float));
    memcpy(lex_off_host, H.lex_off.data(), H.lex_off.size() * sizeof(int));
    if (!H.lex_tok.empty()) {
        memcpy(lex_tok_host, H.lex_tok.data(), H.lex_tok.size() * sizeof(int));
        memcpy(lex_next_host, H.lex_next.data(), H.lex_next.size() * sizeof(int));
    }
    memcpy(lex_word_host, H.lex_word.data(), H.lex_word.size() * sizeof(int));
    memset(layout_host, 0, sizeof(*layout_host));
    layout_host->order = H.order;
    layout_host->bos = H.bos;
    layout_host->eos = H.eos;
    layout_host->vocab = H.V;
    layout_host->space = H.space;
    layout_host->root = 0;
    layout_host->nodes = (int)H.lex_word.size();
    layout_host->dict_size = (int)H.dict_size;
    for (int n = 1; n <= H.order; ++n) {
        layout_host->off[n] = H.off[n];
        layout_host->mask[n] = H.slots[n] - 1;
    }
    return MASR_OK;
}

extern "C" int masr_word_lm_score_f32(const masr_word_lm_tables* lm_host, const int* ctx, const int* word, int Q, float* out,
                                      void* stream) {
    if (Q == 0) return MASR_OK;
    MASR_REQUIRE(lm_host && lm_host->keys && lm_host->vals && word && out && (ctx || lm_host->order == 1),
                 "masr_word_lm_score_f32: null pointer");
    MASR_REQUIRE(lm_host->order >= 1 && lm_host->order <= WLM_MAX_ORDER, "masr_word_lm_score_f32: order %d out of range",
                 lm_host->order);
    word_lm_score_kernel<<<(Q + 255) / 256, 256, 0, (cudaStream_t)stream>>>(*lm_host, ctx, word, Q, out);
    return check_launch("word_lm_score_kernel");
}
