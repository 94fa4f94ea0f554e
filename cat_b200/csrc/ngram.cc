// ARPA text loader for the beam search's token n-gram LM (ngram.h).  Host only.
#include "ngram.h"

#include <algorithm>
#include <cctype>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <numeric>
#include <unordered_map>

namespace ccb {

namespace {

struct Order {   // the n-grams of order k: words [k*i, k*i + k), log10 p (NaN: inserted by the closure), bow
    int k = 0;
    std::vector<int> words;
    std::vector<float> p, bow;
    long size() const { return (long)p.size(); }
    const int *at(long i) const { return words.data() + (size_t)k * i; }
};

// index of the k words w in the lexicographically sorted order o, or -1
long Find(const Order &o, const int *w) {
    long lo = 0, hi = o.size();
    while (lo < hi) {
        const long mid = (lo + hi) >> 1;
        const int *x = o.at(mid);
        int c = 0;
        for (int j = 0; j < o.k && c == 0; ++j) c = x[j] < w[j] ? -1 : (x[j] > w[j] ? 1 : 0);
        if (c == 0) return mid;
        if (c < 0) lo = mid + 1; else hi = mid;
    }
    return -1;
}

// sort an order lexicographically; of n-grams listed twice the first is kept
void SortOrder(Order *o) {
    std::vector<long> idx(o->size());
    std::iota(idx.begin(), idx.end(), 0L);
    const int k = o->k;
    std::stable_sort(idx.begin(), idx.end(), [&](long a, long b) {
        return std::lexicographical_compare(o->at(a), o->at(a) + k, o->at(b), o->at(b) + k);
    });
    Order s;
    s.k = k;
    for (size_t i = 0; i < idx.size(); ++i) {
        const int *w = o->at(idx[i]);
        if (i > 0 && std::equal(w, w + k, o->at(idx[i - 1]))) continue;
        s.words.insert(s.words.end(), w, w + k);
        s.p.push_back(o->p[idx[i]]);
        s.bow.push_back(o->bow[idx[i]]);
    }
    *o = std::move(s);
}

struct Tok {
    const char *b;
    size_t n;
    bool is(const char *s) const { return strlen(s) == n && memcmp(b, s, n) == 0; }
    std::string str() const { return std::string(b, n); }
};

bool ParseNumber(const Tok &t, float *v) {
    const std::string s = t.str();
    char *end = nullptr;
    const double d = strtod(s.c_str(), &end);
    if (end != s.c_str() + s.size() || !std::isfinite(d)) return false;
    *v = (float)d;
    return true;
}

}  // namespace

bool LoadArpa(const char *path, const char *const *labels, int V, NGramHost *out, std::string *err) {
    const std::string where = std::string(path ? path : "(null)") + ": ";
    auto fail = [&](const std::string &m) { *err = where + m; return false; };
    auto at = [](long line) { return "line " + std::to_string(line) + ": "; };
    if (!path || !labels || V < 1) return fail("bad arguments");
    FILE *f = fopen(path, "rb");
    if (!f) return fail("cannot open the file");
    std::string text;
    char buf[1 << 16];
    for (size_t r; (r = fread(buf, 1, sizeof buf, f)) > 0;) text.append(buf, r);
    fclose(f);
    static const char kKenlm[] = "mmap lm http://kheafield.com/code";
    if (text.compare(0, sizeof kKenlm - 1, kKenlm) == 0)
        return fail("this is a KenLM binary; pass the ARPA text that `ngram.sh --arpa` (lmplz) writes");

    // the words the labels name (an empty label names <unk>)
    std::vector<std::string> label_word(V);
    std::unordered_map<std::string, int> named;
    for (int i = 1; i < V; ++i) {
        std::string w = labels[i] ? labels[i] : "";
        if (w == "<s>" || w == "</s>") return fail("label " + std::to_string(i) + " is " + w + ", which the LM cannot score");
        if (w.empty()) w = "<unk>";
        label_word[i] = w;
        named.emplace(w, 1);
    }

    // the text: \data\, ngram k=count, then \k-grams: sections, \end\ .
    int order = 0;
    long counts[kNgramMaxOrder + 1] = {};
    std::vector<Order> ord(1);          // ord[k], k = 1 .. order
    std::unordered_map<std::string, int> vocab;
    std::vector<float> uni_p, uni_bow;
    int section = -1;                   // -1 before \data\, 0 in \data\, k in \k-grams:
    long section_line = 0, listed = 0, line = 0;
    bool ended = false;
    std::vector<Tok> tk;
    std::vector<int> ws;
    auto close_section = [&]() -> bool {
        if (section >= 1 && listed != counts[section])
            return fail(at(section_line) + "\\" + std::to_string(section) + "-grams: lists " + std::to_string(listed) +
                        " n-grams, \\data\\ declares " + std::to_string(counts[section]));
        return true;
    };
    size_t pos = 0;
    while (!ended && pos < text.size()) {
        size_t e = text.find('\n', pos);
        if (e == std::string::npos) e = text.size();
        const char *b = text.data() + pos, *end = text.data() + e;
        pos = e + 1;
        ++line;
        tk.clear();
        for (const char *c = b; c < end;) {
            while (c < end && isspace((unsigned char)*c)) ++c;
            const char *s = c;
            while (c < end && !isspace((unsigned char)*c)) ++c;
            if (c > s) tk.push_back(Tok{s, (size_t)(c - s)});
        }
        if (tk.empty()) continue;
        if (section < 0) {
            if (!tk[0].is("\\data\\") || tk.size() != 1) return fail(at(line) + "an ARPA file starts with \\data\\");
            section = 0;
            continue;
        }
        if (tk[0].b[0] == '\\') {   // a section header
            if (!close_section()) return false;
            if (section == 0 && order == 0) return fail(at(line) + "\\data\\ declares no n-gram counts");
            const std::string h = tk[0].str();
            if (tk.size() == 1 && h == "\\end\\") {
                if (section < order)
                    return fail(at(line) + "\\end\\ before the \\" + std::to_string(section + 1) + "-grams: section");
                ended = true;
                continue;
            }
            if (tk.size() != 1 || h != "\\" + std::to_string(section + 1) + "-grams:" || section + 1 > order)
                return fail(at(line) + "unknown section '" + h + "' (expected " +
                            (section < order ? "\\" + std::to_string(section + 1) + "-grams:" : std::string("\\end\\")) + ")");
            section += 1;
            section_line = line;
            listed = 0;
            ord.emplace_back();
            ord.back().k = section;
            continue;
        }
        if (section == 0) {   // ngram k=count
            const std::string s = tk.size() == 2 && tk[0].is("ngram") ? tk[1].str() : std::string();
            const size_t eq = s.find('=');
            char *e1 = nullptr, *e2 = nullptr;
            const long k = eq == std::string::npos ? -1 : strtol(s.c_str(), &e1, 10);
            const long c = eq == std::string::npos ? -1 : strtol(s.c_str() + eq + 1, &e2, 10);
            if (eq == std::string::npos || e1 != s.c_str() + eq || e2 != s.c_str() + s.size() || eq == 0 || c < 0)
                return fail(at(line) + "expected 'ngram k=count' in \\data\\");
            if (k != order + 1) return fail(at(line) + "the counts must be listed for orders 1, 2, ... in turn");
            if (k > kNgramMaxOrder) return fail(at(line) + "orders above " + std::to_string(kNgramMaxOrder) + " are not supported");
            order = (int)k;
            counts[k] = c;
            continue;
        }
        // an n-gram: log10 p, `section` words, an optional back-off weight
        const int k = section;
        ++listed;
        if ((int)tk.size() != k + 1 && (int)tk.size() != k + 2)
            return fail(at(line) + "a " + std::to_string(k) + "-gram line has log10 p, " + std::to_string(k) +
                        " words and an optional back-off weight, not " + std::to_string(tk.size()) + " fields");
        float p = 0.f, bw = 0.f;
        if (!ParseNumber(tk[0], &p)) return fail(at(line) + "'" + tk[0].str() + "' is not a number");
        if ((int)tk.size() == k + 2 && !ParseNumber(tk[k + 1], &bw)) return fail(at(line) + "'" + tk[k + 1].str() + "' is not a number");
        if (k == 1) {
            // a word no label names is unreachable (and so is every n-gram that contains it)
            const std::string w = tk[1].str();
            if (!named.count(w) && w != "<s>" && w != "</s>" && w != "<unk>") continue;
            if (!vocab.emplace(w, (int)uni_p.size()).second) continue;
            uni_p.push_back(p);
            uni_bow.push_back(bw);
            continue;
        }
        ws.clear();
        for (int j = 1; j <= k; ++j) {
            auto it = vocab.find(tk[j].str());
            if (it == vocab.end()) break;
            ws.push_back(it->second);
        }
        if ((int)ws.size() < k) continue;
        Order &o = ord[k];
        o.words.insert(o.words.end(), ws.begin(), ws.end());
        o.p.push_back(p);
        o.bow.push_back(bw);
    }
    if (section < 0) return fail(at(line) + "an ARPA file starts with \\data\\");
    if (!ended) return fail("the file ends at line " + std::to_string(line) + " without \\end\\");

    NGramHost &m = *out;
    m = NGramHost();
    m.order = order;
    m.V = V;
    for (int k = 1; k <= order; ++k) m.counts[k - 1] = counts[k];
    if (!vocab.count("<unk>")) {   // KenLM's substitution: log10 p = -100, no context
        vocab.emplace("<unk>", (int)uni_p.size());
        uni_p.push_back(-100.f);
        uni_bow.push_back(0.f);
        m.unk_substituted = true;
    }
    const int W = (int)uni_p.size(), unk = vocab["<unk>"];
    m.W = W;
    m.tok2word.assign(V, -1);
    for (int i = 1; i < V; ++i) {
        auto it = vocab.find(label_word[i]);
        m.tok2word[i] = it == vocab.end() ? unk : it->second;
    }
    ord[1].words.resize(W);
    std::iota(ord[1].words.begin(), ord[1].words.end(), 0);
    ord[1].p = uni_p;
    ord[1].bow = uni_bow;
    for (int k = 2; k <= order; ++k) SortOrder(&ord[k]);

    // prefix closure, from the highest order down: a missing prefix is inserted with bow 0 and probability NaN, which tells
    // the walk to take the arc's destination and the back-off value (bow of the history plus the next shorter history's
    // value), so that the value is the textbook one to the last bit rather than its fp32 rounding
    for (int k = order; k >= 3; --k) {
        Order &lo = ord[k - 1];
        const long n0 = lo.size();
        for (long i = 0; i < ord[k].size(); ++i)
            if (Find(lo, ord[k].at(i)) < 0) {   // the first k-1 words of the k-gram
                lo.words.insert(lo.words.end(), ord[k].at(i), ord[k].at(i) + k - 1);
                lo.p.push_back(NAN);
                lo.bow.push_back(0.f);
            }
        if (lo.size() > n0) SortOrder(&lo);
    }

    // states: the root, then the n-grams of orders 1 .. order-1
    std::vector<int> base(order + 1, 0);
    int S = 1;
    for (int k = 1; k < order; ++k) { base[k] = S; S += (int)ord[k].size(); }
    auto state_of_suffix = [&](const int *w, int k, int from) {   // longest suffix w[j..k), j >= from, that is a state
        for (int j = from; j < k; ++j) {
            const int len = k - j;
            if (len >= order) continue;
            const long i = Find(ord[len], w + j);
            if (i >= 0) return base[len] + (int)i;
        }
        return 0;
    };
    m.bow.assign(S, 0.f);
    m.back.assign(S, -1);
    for (int k = 1; k < order; ++k)
        for (long i = 0; i < ord[k].size(); ++i) {
            const int s = base[k] + (int)i;
            m.bow[s] = ord[k].bow[i];
            m.back[s] = state_of_suffix(ord[k].at(i), k, 1);
        }
    m.root_p = uni_p;
    m.root_dst.resize(W);
    for (int w = 0; w < W; ++w) m.root_dst[w] = order >= 2 ? base[1] + w : 0;
    // arcs: the n-grams of orders 2 .. order, from the state of their history
    m.arc_off.assign(S + 1, 0);
    std::vector<int> src;
    for (int k = 2; k <= order; ++k)
        for (long i = 0; i < ord[k].size(); ++i) {
            const long h = Find(ord[k - 1], ord[k].at(i));
            src.push_back(base[k - 1] + (int)h);
            ++m.arc_off[base[k - 1] + (int)h + 1];
        }
    for (int s = 0; s < S; ++s) m.arc_off[s + 1] += m.arc_off[s];
    const size_t A = src.size();
    m.arc_word.resize(A); m.arc_dst.resize(A); m.arc_p.resize(A);
    std::vector<int> cur(m.arc_off.begin(), m.arc_off.end() - 1);
    size_t a = 0;
    for (int k = 2; k <= order; ++k)
        for (long i = 0; i < ord[k].size(); ++i, ++a) {
            const int *w = ord[k].at(i);
            const int slot = cur[src[a]]++;
            m.arc_word[slot] = w[k - 1];
            m.arc_p[slot] = ord[k].p[i];
            m.arc_dst[slot] = state_of_suffix(w, k, 0);
        }
    auto bos = vocab.find("<s>");
    m.bos = bos != vocab.end() && order >= 2 ? base[1] + bos->second : 0;
    m.bos_word = bos != vocab.end() ? bos->second : -1;
    auto eos = vocab.find("</s>");
    m.eos = eos != vocab.end() ? eos->second : unk;
    m.eos_listed = eos != vocab.end();
    return true;
}

}  // namespace ccb
