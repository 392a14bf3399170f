// constraint.cpp — the automaton compiler (see constraint.h).
#include "constraint.h"
#include <algorithm>
#include <limits.h>
#include <numeric>

namespace mg4 {

int Constraint::next(int s, int32_t id) const {
    const int32_t *r = row(s);
    int lo = 0, hi = row_size(s);
    while (lo < hi) {   // first pair with id >= the wanted one
        const int mid = (lo + hi) / 2;
        if (r[2 * mid] < id) lo = mid + 1;
        else hi = mid;
    }
    return lo < row_size(s) && r[2 * lo] == id ? r[2 * lo + 1] : -1;
}

namespace {

// a byte trie of the vocabulary's texts: every state's walk visits each shared prefix once instead of once per id
struct Trie {
    struct Node { int first_child = -1, sibling = -1, id_begin = 0, id_end = 0; unsigned char byte = 0; };
    std::vector<Node> nodes;   // node 0 is the root (the empty text)
    std::vector<int32_t> ids;  // the ids of node k are ids[id_begin, id_end), ascending

    explicit Trie(const std::vector<std::string> &texts) {
        // ids other than 2 with a non-empty text, in byte order of their texts (then by id): equal texts end up adjacent, and every node's
        // children are created in ascending byte order, so a new byte is always the node's last child so far
        for (int32_t id = 0; id < (int32_t)texts.size(); ++id) if (id != 2 && !texts[(size_t)id].empty()) ids.push_back(id);
        std::stable_sort(ids.begin(), ids.end(), [&](int32_t a, int32_t b) {
            const std::string &x = texts[(size_t)a], &y = texts[(size_t)b];
            return std::lexicographical_compare(x.begin(), x.end(), y.begin(), y.end(),
                                                [](char p, char q) { return (unsigned char)p < (unsigned char)q; });
        });
        nodes.emplace_back();
        std::vector<int> last_child(1, -1);
        for (size_t k = 0; k < ids.size(); ++k) {
            const std::string &t = texts[(size_t)ids[k]];
            int n = 0;
            for (unsigned char b : t) {
                const int lc = last_child[(size_t)n];
                if (lc >= 0 && nodes[(size_t)lc].byte == b) { n = lc; continue; }
                Node c; c.byte = b; c.id_begin = c.id_end = (int)k;
                nodes.push_back(c);
                last_child.push_back(-1);
                const int ci = (int)nodes.size() - 1;
                if (lc >= 0) nodes[(size_t)lc].sibling = ci;
                else nodes[(size_t)n].first_child = ci;
                last_child[(size_t)n] = ci;
                n = ci;
            }
            if (nodes[(size_t)n].id_end == nodes[(size_t)n].id_begin) nodes[(size_t)n].id_begin = (int)k;
            nodes[(size_t)n].id_end = (int)k + 1;
        }
    }

    // every id whose walk from state s never meets -1: emit(id, state at the end of its text)
    template <class Emit> void walk(const int32_t *next, int s, std::vector<std::pair<int, int>> &stack, Emit emit) const {
        stack.clear();
        for (int c = nodes[0].first_child; c >= 0; c = nodes[(size_t)c].sibling) stack.emplace_back(c, s);
        while (!stack.empty()) {
            const std::pair<int, int> top = stack.back();
            stack.pop_back();
            const Node &nd = nodes[(size_t)top.first];
            const int t = next[(size_t)top.second * 256 + nd.byte];
            if (t < 0) continue;
            for (int k = nd.id_begin; k < nd.id_end; ++k) emit(ids[(size_t)k], t);
            for (int c = nd.first_child; c >= 0; c = nodes[(size_t)c].sibling) stack.emplace_back(c, t);
        }
    }
};

}  // namespace

bool compile_constraint(const std::vector<std::string> &texts, int n_states, const int32_t *next, const uint8_t *accept, Constraint &out,
                        std::string *why) {
    auto fail = [&](const char *m) { if (why) *why = m; return false; };
    if (!next || !accept || n_states < 1 || n_states > 65536) return fail("n_states outside 1..65536");
    const size_t S = (size_t)n_states;
    for (size_t i = 0; i < S * 256; ++i) if (next[i] < -1 || next[i] >= n_states) return fail("a transition outside -1 .. n_states - 1");
    const Trie trie(texts);
    std::vector<std::pair<int, int>> stack;

    // pass 1: the states each state's ids lead to, and from them liveness, to a fixed point (a backward search from the accepting states)
    std::vector<std::vector<int>> preds(S);
    std::vector<int> seen(S, -1);
    for (int s = 0; s < n_states; ++s)
        trie.walk(next, s, stack, [&](int32_t, int t) { if (seen[(size_t)t] != s) { seen[(size_t)t] = s; preds[(size_t)t].push_back(s); } });
    std::vector<char> live(S, 0);
    std::vector<int> queue;
    for (int s = 0; s < n_states; ++s) if (accept[s]) { live[(size_t)s] = 1; queue.push_back(s); }
    for (size_t q = 0; q < queue.size(); ++q)
        for (int p : preds[(size_t)queue[q]]) if (!live[(size_t)p]) { live[(size_t)p] = 1; queue.push_back(p); }
    if (!live[0]) return fail("the start state is not live");

    // pass 2: each live state's ids that end in a live state (id 2 if it accepts), ascending; the finished state's row last
    out.n_states = n_states;
    out.off.assign(S + 2, 0);
    out.pairs.clear();
    std::vector<std::pair<int32_t, int32_t>> row;
    long long total = 0;
    for (int s = 0; s <= n_states; ++s) {
        row.clear();
        if (s == n_states) row.emplace_back(2, n_states);
        else if (live[(size_t)s]) {
            trie.walk(next, s, stack, [&](int32_t id, int t) { if (live[(size_t)t]) row.emplace_back(id, t); });
            if (accept[s]) row.emplace_back(2, n_states);
            std::sort(row.begin(), row.end());
        }
        total += (long long)row.size();
        if (total > INT_MAX) return fail("more than 2^31 - 1 transitions");
        for (const auto &p : row) { out.pairs.push_back(p.first); out.pairs.push_back(p.second); }
        out.off[(size_t)s + 1] = (int32_t)total;
    }
    return true;
}

}  // namespace mg4
