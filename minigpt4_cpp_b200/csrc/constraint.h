// constraint.h — constrained replies (minigpt4_b200_constraint_*, DESIGN.md §4.12): a deterministic automaton over bytes compiled
// against a vocabulary into the ids each state allows.
//
// allowed(s): every id other than 2 whose text (the C string minigpt4_end_chat returns for it), walked byte by byte from s, never meets
// -1 and ends in a live state; and id 2 if s accepts.  A state is live if some sequence of allowed ids leads from it to an accepting
// state (a fixed point over the token transitions, not the byte graph).  Id 2 moves to the finished state, which allows only id 2.
//
// The compiled form is a CSR table over n_states + 1 rows, the last one the finished state (row n_states): row s is the pairs
// (id, next state) off[s] .. off[s + 1] - 1 in ascending id order.  A state that is not live has an empty row.  Only this module builds
// the table; the host Sampler, the engine and the device sampler take its arrays.
#pragma once
#include <memory>
#include <stdint.h>
#include <string>
#include <vector>

namespace mg4 {

struct LlamaGroup;
struct SharedTable;

struct Constraint {
    int n_states = 0;             // the caller's states; row n_states is the finished state
    std::vector<int32_t> off;     // [n_states + 2]
    std::vector<int32_t> pairs;   // [2 off[n_states + 1]]: id, next state
    const LlamaGroup *group = nullptr;      // the contexts it attaches to
    std::shared_ptr<SharedTable> dev;       // off then pairs on the device (LlamaDevice::upload_table)

    int finished() const { return n_states; }
    int row_size(int s) const { return off[(size_t)s + 1] - off[(size_t)s]; }
    const int32_t *row(int s) const { return pairs.data() + 2 * (size_t)off[(size_t)s]; }
    // the state id leads to from s, -1 if s does not allow it (a binary search in the row)
    int next(int s, int32_t id) const;
};

// Compile the automaton (next: [n_states][256], -1 rejects; accept: [n_states]) against texts[id]; false, with the reason in *why, for
// n_states outside 1..65536, next[] outside -1 .. n_states - 1, a start state that is not live, or more than 2^31 - 1 transitions.
bool compile_constraint(const std::vector<std::string> &texts, int n_states, const int32_t *next, const uint8_t *accept, Constraint &out,
                        std::string *why);

}  // namespace mg4
