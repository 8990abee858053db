// Declarations shared by the trie coprocessor witness kernels (trie.cu) and the fold context.
#pragma once
#include "common.cuh"

namespace lurk {

// Input elements of one call: root, key, path[H][8] (lookup); root, key, value, old_path[H][8], new_path[H][8] (insert).
inline size_t trie_n_inputs(int op, int height) {
    return op == LURK_TRIE_INSERT ? 3 + (size_t)16 * height : 2 + (size_t)8 * height;
}
// Aux block of one call in field F: D + 403 H (lookup), D + 799 H (insert); 0 for an unsupported op or height.
template <class F>
size_t trie_block_len(int op, int height);
// count calls, count * trie_n_inputs elements in in_fmt; block k is written at element offset d_offs[k] of d_out
// (k * block length when d_offs is null) in out_fmt.  Two launches: the Poseidon levels, then root, key bits and picks.
template <class F>
int launch_trie_witness(int op, int height, const void *d_in, size_t count, void *d_out, const uint64_t *d_offs, int in_fmt, int out_fmt,
                        cudaStream_t s);

}  // namespace lurk
