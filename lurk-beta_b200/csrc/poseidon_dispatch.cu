// Arity dispatch, constant cache access and bit-decomposition launches for the four fields; the per-arity kernels are
// compiled in poseidon_inst.cu instances (extern templates here).
#include "poseidon_kernel.cuh"
namespace lurk {
#define LURK_EXTERN_ARITY(F, A)                                                                                          \
    extern template int launch_arity<F, A, false>(const void *, size_t, void *, const uint64_t *, const PoseidonGather *, int, int, cudaStream_t); \
    extern template int launch_arity<F, A, true>(const void *, size_t, void *, const uint64_t *, const PoseidonGather *, int, int, cudaStream_t);
#define LURK_FIELD_DISPATCH(F)                                                                                           \
    LURK_EXTERN_ARITY(F, 3) LURK_EXTERN_ARITY(F, 4) LURK_EXTERN_ARITY(F, 6) LURK_EXTERN_ARITY(F, 8)                      \
    template int launch_poseidon<F, false>(int, const void *, size_t, void *, int, int, cudaStream_t, const uint64_t *, const PoseidonGather *); \
    template int launch_poseidon<F, true>(int, const void *, size_t, void *, int, int, cudaStream_t, const uint64_t *, const PoseidonGather *);  \
    template int poseidon_instance_info<F>(int, const PoseidonParams<F> **, PoseidonLayout *);                          \
    template int launch_bitdecomp<F>(const void *, size_t, void *, int, int, cudaStream_t, const uint64_t *);
LURK_FIELD_DISPATCH(Fe<Bn254Fr>)
LURK_FIELD_DISPATCH(Fe<Bn254Fq>)
LURK_FIELD_DISPATCH(Fe<PallasFq>)
LURK_FIELD_DISPATCH(Fe<PallasFp>)
}  // namespace lurk
