// Declarations shared by the per-field Poseidon translation units and the C-ABI front end (poseidon.cu).
#pragma once
#include "common.cuh"
#include "poseidon_params.h"

namespace lurk {

struct PoseidonLayout {
    int rf, rp;
    int off_mds, off_pre, off_sw, off_sv, flat_len;   // in elements
    int block_elems;                                   // witness block size (arity + aux + 1)
};

// Where sponge h of a launch reads its preimage and writes its witness block.  Without one (a plain batch) preimage h
// starts at element h * arity and block h at d_offsets[h] (h * block elements without offsets).  Coprocessor calls
// group `per_call` sponges: sponge h is level l = h % per_call of call c = h / per_call, its preimage starts at element
// c * in_stride + in_first + arity * l, its block at base + (l < split ? out0 + step0 * l : out1 + step1 * (l - split)),
// base = d_offsets[c] (c * out_stride without offsets).
struct PoseidonGather {
    int per_call, split;
    uint64_t in_stride, in_first, out_stride;
    int64_t out0, step0, out1, step1;
};

// defined (explicitly instantiated) in poseidon_f{0..3}.cu
template <class F, bool WITNESS>
int launch_poseidon(int arity, const void *d_pre, size_t n, void *d_out, int in_fmt, int out_fmt, cudaStream_t s,
                    const uint64_t *d_offsets = nullptr,       // optional element offset of every witness block (call)
                    const PoseidonGather *gather = nullptr);
template <class F>
int poseidon_instance_info(int arity, const PoseidonParams<F> **params, PoseidonLayout *layout);
template <class F>
int launch_bitdecomp(const void *d_values, size_t n, void *d_blocks, int blk, int fmt, cudaStream_t s, const uint64_t *d_offsets = nullptr);
int bitdecomp_block_host(const uint32_t mod[8]);

}  // namespace lurk
