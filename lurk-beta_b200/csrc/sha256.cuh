// Declarations shared by the SHA-256 coprocessor witness kernel (sha256.cu) and the fold context.
#pragma once
#include "common.cuh"

namespace lurk {

// Aux block of one synthesize_sha256 call with n pointers in field F (0 for n out of range); the allocation schedule
// behind it is built once per (field, n).
template <class F>
size_t sha256_block_len(int n);
// count calls, count * 2n input elements (per pointer: tag, then hash) in in_fmt; block k is written at element offset
// d_offs[k] of d_out (k * block length when d_offs is null) in out_fmt.
template <class F>
int launch_sha256_witness(const void *d_in, size_t count, int n, void *d_out, const uint64_t *d_offs, int in_fmt, int out_fmt,
                          cudaStream_t s);

}  // namespace lurk
