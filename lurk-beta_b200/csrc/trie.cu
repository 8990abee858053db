// Witness of the trie coprocessor's lookup and insert circuits (reference src/coprocessor/trie/mod.rs:118-156 and
// 226-268 -> synthesize_lookup_at_path 668-714, synthesize_modify_value_at_path 846-880) on the GPU.
//
// One call's block, with D = the bit-decomposition block of the field and S = the arity-8 slot block (8 preimage
// elements, 387 Poseidon aux, the digest):
//   [allocated_root | the D - 1 aux of key.to_bits_le_strict | per level L = 0..H-1: S of path[L], then select's 7 picks]
// and for an insert, after that, per level L = H-1 down to 0: S of new_path[L].
// The inputs carry every preimage (the reference's witness generation reads them from the inverse Poseidon cache), so
// the 85 or 170 hashes of a call are independent: launch 1 is the arity-8 Poseidon witness kernel over all of them,
// gathered from the inputs and scattered into the blocks (PoseidonGather); launch 2 writes the root, the key's bits
// (bitdecomp_aux) and the picks, one thread per (call, root-and-bits | level).
#include "trie.cuh"
#include "poseidon_kernel.cuh"

#include <cstring>

namespace lurk {

#define LURK_TRIE_POSEIDON_EXTERN(F)                                                                                                   \
    extern template int launch_poseidon<F, true>(int, const void *, size_t, void *, int, int, cudaStream_t, const uint64_t *,          \
                                                 const PoseidonGather *);                                                               \
    extern template int poseidon_instance_info<F>(int, const PoseidonParams<F> **, PoseidonLayout *);
LURK_TRIE_POSEIDON_EXTERN(Fe<Bn254Fr>)
LURK_TRIE_POSEIDON_EXTERN(Fe<Bn254Fq>)
LURK_TRIE_POSEIDON_EXTERN(Fe<PallasFq>)
LURK_TRIE_POSEIDON_EXTERN(Fe<PallasFp>)

namespace {

constexpr int ARITY = 8, PICKS = 7;

template <class F>
int bitdecomp_len() {
    uint32_t mod[8];
    for (int i = 0; i < 8; i++) mod[i] = F::Params::MOD(i);
    return bitdecomp_block_host(mod);
}

template <class F>
int slot_len() {
    PoseidonLayout L;
    poseidon_instance_info<F>(ARITY, nullptr, &L);
    return L.block_elems;
}

template <class F>
__device__ __forceinline__ F convert(const F &raw, int in_fmt, int out_fmt) {
    if (in_fmt == out_fmt) return raw;
    return out_fmt == LURK_FMT_MONTGOMERY ? F::from_canonical(raw) : raw.to_canonical();
}

// item = call * (H + 1) + j: j = 0 writes allocated_root and the key's bits, j = L + 1 the 7 picks of level L
template <class F>
__global__ void __launch_bounds__(128) trie_witness_kernel(const F *__restrict__ in, size_t count, int height, int first, size_t n_in,
                                                           int D, int slot, size_t blk, F *__restrict__ out,
                                                           const uint64_t *__restrict__ offs, int in_fmt, int out_fmt) {
    const size_t per = (size_t)height + 1, items = count * per;
    for (size_t it = (size_t)blockIdx.x * blockDim.x + threadIdx.x; it < items; it += (size_t)gridDim.x * blockDim.x) {
        const size_t c = it / per;
        const int j = (int)(it - c * per);
        const F *x = in + c * n_in;
        F *o = out + (offs ? offs[c] : c * blk);
        F key = load_fe<F>(x + 1);
        if (in_fmt == LURK_FMT_MONTGOMERY) key = key.to_canonical();
        if (j == 0) {
            store_fe(o, convert(load_fe<F>(x), in_fmt, out_fmt));   // allocated_root_value
            bitdecomp_aux(key, o + 1, out_fmt);                     // key.to_bits_le_strict
            continue;
        }
        // synthesize_path: level L's chunk is key bits 3(H-1-L) .. +2 (bit 254 is Constant(false) on the 254-bit
        // fields, and 0 in every key below p); select consumes the most significant bit first
        const int L = j - 1, lo = 3 * (height - 1 - L);
        uint32_t k = 0;
        for (int t = 0; t < 3; t++) k |= ((key.v[(lo + t) >> 5] >> ((lo + t) & 31)) & 1) << t;
        const F *pre = x + first + (size_t)ARITY * L;
        F *po = o + D + (size_t)(slot + PICKS) * L + slot;
        // pick i, j: bit ? state[half + j] : state[j]; after the top bit the state is pre[(k & 4) + 0..3], and so on
        int q = 0;
        for (int half = 4, hi = 2; half >= 1; half >>= 1, hi--) {
            const uint32_t sel = (k >> hi) << hi;   // the bits consumed so far
            for (int m = 0; m < half; m++) store_fe(po + q++, convert(load_fe<F>(pre + sel + m), in_fmt, out_fmt));
        }
    }
}

}  // namespace

template <class F>
size_t trie_block_len(int op, int height) {
    if ((op != LURK_TRIE_LOOKUP && op != LURK_TRIE_INSERT) || height < 1 || height > LURK_TRIE_MAX_HEIGHT) return 0;
    const size_t lvl = (size_t)slot_len<F>() + PICKS;
    return (size_t)bitdecomp_len<F>() + lvl * height + (op == LURK_TRIE_INSERT ? (size_t)slot_len<F>() * height : 0);
}

constexpr int TRIE_THREADS = 128, TRIE_CTAS_PER_SM = 2;

template <class F>
int launch_trie_witness(int op, int height, const void *d_in, size_t count, void *d_out, const uint64_t *d_offs, int in_fmt, int out_fmt,
                        cudaStream_t st) {
    const size_t blk = trie_block_len<F>(op, height);
    if (!blk) { set_error("trie op %d / height %d: op 0 (lookup) or 1 (insert), height 1..%d", op, height, LURK_TRIE_MAX_HEIGHT); return LURK_ERR_ARG; }
    if (!count) return LURK_OK;
    const int D = bitdecomp_len<F>(), slot = slot_len<F>(), first = op == LURK_TRIE_INSERT ? 3 : 2;
    const int lvl = slot + PICKS;
    // every preimage of a call, old path then new path, is contiguous in its inputs: level l at first + 8 l
    PoseidonGather G;
    G.per_call = op == LURK_TRIE_INSERT ? 2 * height : height;
    G.split = height;
    G.in_stride = trie_n_inputs(op, height);
    G.in_first = first;
    G.out_stride = blk;
    G.out0 = D; G.step0 = lvl;                                                        // the lookup's levels
    G.out1 = (int64_t)D + (int64_t)lvl * height + (int64_t)slot * (height - 1);       // new level L = H-1 goes first
    G.step1 = -slot;
    LURK_TRY((launch_poseidon<F, true>(ARITY, d_in, count * G.per_call, d_out, in_fmt, out_fmt, st, d_offs, &G)));
    const size_t items = count * ((size_t)height + 1), cap = (size_t)sm_count() * TRIE_CTAS_PER_SM;
    size_t grid = (items + TRIE_THREADS - 1) / TRIE_THREADS;
    if (grid > cap) grid = cap;
    trie_witness_kernel<F><<<(unsigned)grid, TRIE_THREADS, 0, st>>>((const F *)d_in, count, height, first, G.in_stride, D, slot, blk, (F *)d_out,
                                                                   d_offs, in_fmt, out_fmt);
    LURK_CUDA_TRY(cudaGetLastError());
    return LURK_OK;
}

#define LURK_TRIE_INSTANTIATE(F)                    \
    template size_t trie_block_len<F>(int, int);    \
    template int launch_trie_witness<F>(int, int, const void *, size_t, void *, const uint64_t *, int, int, cudaStream_t);
LURK_TRIE_INSTANTIATE(Fe<Bn254Fr>)
LURK_TRIE_INSTANTIATE(Fe<Bn254Fq>)
LURK_TRIE_INSTANTIATE(Fe<PallasFq>)
LURK_TRIE_INSTANTIATE(Fe<PallasFp>)

namespace {

// The host call's path check, on one call's inputs and block (both in one format, so equal elements are equal bytes):
// each level's digest against the element its parent selects (level 0: the root); for an insert, the new path the same
// way, its leaf against the value.
template <class F>
int check_paths(int op, int height, const uint8_t *x, const uint8_t *o, size_t call, int fmt) {
    const int D = bitdecomp_len<F>(), slot = slot_len<F>(), lvl = slot + PICKS, first = op == LURK_TRIE_INSERT ? 3 : 2;
    F key;
    memcpy(key.v, x + 32, 32);
    if (fmt == LURK_FMT_MONTGOMERY) key = key.to_canonical();
    auto k_at = [&](int L) {
        const int lo = 3 * (height - 1 - L);
        int k = 0;
        for (int t = 0; t < 3; t++) k |= (int)((key.v[(lo + t) >> 5] >> ((lo + t) & 31)) & 1) << t;
        return k;
    };
    auto eq = [](const uint8_t *a, const uint8_t *b) { return memcmp(a, b, 32) == 0; };
    for (int L = 0; L < height; L++) {
        const uint8_t *digest = o + ((size_t)D + (size_t)lvl * L + slot - 1) * 32;
        const uint8_t *parent = L == 0 ? x : x + ((size_t)first + (size_t)ARITY * (L - 1) + k_at(L - 1)) * 32;
        if (!eq(digest, parent)) {
            set_error("trie call %zu level %d: the path's preimage does not hash to %s", call, L, L ? "the element its parent selects" : "the root");
            return LURK_ERR_ARG;
        }
    }
    if (op != LURK_TRIE_INSERT) return LURK_OK;
    const size_t new_first = (size_t)first + (size_t)ARITY * height;
    for (int L = 0; L < height; L++) {
        const uint8_t *sel = x + (new_first + (size_t)ARITY * L + k_at(L)) * 32;
        // the digest of new level L + 1: new levels are laid out from H - 1 down to 0 after the lookup's levels
        const uint8_t *want = L == height - 1 ? x + 2 * 32
                                              : o + ((size_t)D + (size_t)lvl * height + (size_t)slot * (height - 2 - L) + slot - 1) * 32;
        if (!eq(sel, want)) {
            set_error("trie call %zu level %d: the new path's element at the key is not %s", call, L,
                      L == height - 1 ? "the value" : "the digest of its child");
            return LURK_ERR_ARG;
        }
    }
    return LURK_OK;
}

}  // namespace
}  // namespace lurk

using namespace lurk;

extern "C" {

size_t lurk_trie_witness_block(int field_id, int op, int height) {
    size_t out = 0;
    dispatch_field(field_id, [&](auto f) {
        out = trie_block_len<decltype(f)>(op, height);
        return LURK_OK;
    });
    return out;
}

static int trie_args(int field_id, int op, int height, int fmt, size_t count, const void *a, const void *b) {
    if (fmt != LURK_FMT_CANONICAL && fmt != LURK_FMT_MONTGOMERY) { set_error("bad format %d", fmt); return LURK_ERR_ARG; }
    if (!lurk_trie_witness_block(field_id, op, height)) {
        set_error("unsupported field %d / trie op %d / height %d (op 0 lookup or 1 insert, height 1..%d)", field_id, op, height, LURK_TRIE_MAX_HEIGHT);
        return LURK_ERR_ARG;
    }
    if (count && (!a || !b)) { set_error("null buffer"); return LURK_ERR_ARG; }
    return LURK_OK;
}

int lurk_trie_witness_scatter_dev(int field_id, int op, int height, const void *d_inputs, size_t count, const uint64_t *d_offsets, void *d_W,
                                  int fmt, void *stream) {
    LURK_TRY(trie_args(field_id, op, height, fmt, count, d_inputs, d_W));
    if (count && !d_offsets) { set_error("null offsets"); return LURK_ERR_ARG; }
    LURK_TRY(require_gpu());
    return dispatch_field(field_id, [&](auto f) {
        return launch_trie_witness<decltype(f)>(op, height, d_inputs, count, d_W, d_offsets, fmt, fmt, (cudaStream_t)stream);
    });
}

int lurk_trie_witness_batch_dev(int field_id, int op, int height, const void *d_inputs, size_t count, void *d_aux, int fmt, void *stream) {
    LURK_TRY(trie_args(field_id, op, height, fmt, count, d_inputs, d_aux));
    LURK_TRY(require_gpu());
    return dispatch_field(field_id, [&](auto f) {
        return launch_trie_witness<decltype(f)>(op, height, d_inputs, count, d_aux, nullptr, fmt, fmt, (cudaStream_t)stream);
    });
}

int lurk_trie_witness_batch(int field_id, int op, int height, const uint8_t *inputs, size_t count, uint8_t *aux_out, int fmt) {
    LURK_TRY(trie_args(field_id, op, height, fmt, count, inputs, aux_out));
    LURK_TRY(require_gpu());
    if (!count) return LURK_OK;
    const size_t blk = lurk_trie_witness_block(field_id, op, height), in_per = trie_n_inputs(op, height) * 32, out_per = blk * 32;
    // calls per chunk: bounded device staging for any count
    size_t chunk = ((size_t)256 << 20) / out_per;
    if (chunk < 1) chunk = 1;
    if (chunk > count) chunk = count;
    return dispatch_field(field_id, [&](auto f) {
        using F = decltype(f);
        DevBuf din, dout;
        LURK_TRY(din.alloc(count * in_per));
        LURK_TRY(dout.alloc(chunk * out_per));
        LURK_CUDA_TRY(cudaMemcpy(din.p, inputs, din.bytes, cudaMemcpyHostToDevice));
        int bad = 0;
        LURK_TRY(check_reduced_dev<F>(din.p, count * trie_n_inputs(op, height), 0, &bad));
        if (bad) { set_error("%d input element(s) are not reduced below the field modulus", bad); return LURK_ERR_RANGE; }
        for (size_t first = 0; first < count; first += chunk) {
            const size_t m = count - first < chunk ? count - first : chunk;
            LURK_TRY(launch_trie_witness<F>(op, height, (const uint8_t *)din.p + first * in_per, m, dout.p, nullptr, fmt, fmt, 0));
            LURK_CUDA_TRY(cudaMemcpy(aux_out + first * out_per, dout.p, m * out_per, cudaMemcpyDeviceToHost));
        }
        for (size_t c = 0; c < count; c++) LURK_TRY(check_paths<F>(op, height, inputs + c * in_per, aux_out + c * out_per, c, fmt));
        return LURK_OK;
    });
}

}  // extern "C"
