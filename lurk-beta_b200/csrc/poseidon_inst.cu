// One (field, arity, digest|witness) instance of the Poseidon kernels per object file: the Makefile compiles this file 32
// times with -DLURK_F=<field params> -DLURK_A=<arity> -DLURK_W=<0|1> so that the build runs in parallel.
#include "poseidon_kernel.cuh"
namespace lurk {
template int launch_arity<Fe<LURK_F>, LURK_A, (LURK_W != 0)>(const void *, size_t, void *, const uint64_t *, const PoseidonGather *, int, int, cudaStream_t);
}
