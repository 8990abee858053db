/*
 * lurk_b200.h -- C ABI of liblurk_b200.so: the H100 (sm_90a) implementation of lurk-beta's Nova/SuperNova
 * proving hot path (SURVEY.md section 8).  Plain pointers and sizes only; no C++/torch types.
 *
 * The reference (argumentcomputer/lurk-beta @ f238d85c) has no FFI of its own: GPU work is delegated to
 * third-party crates via `--features cuda = ["neptune/cuda", "nova/cuda"]` (Cargo.toml:105-110).  Each entry
 * point below names the Rust seam it sits behind (reference file:line); INTEGRATION.md shows the
 * `extern "C"` binding a maintainer adds on the Rust side.
 *
 * Conventions
 *   - Field element: 32 bytes little-endian.  LURK_FMT_CANONICAL = the integer < p, i.e.
 *     ff::PrimeField::to_repr (src/field.rs:72-81).  LURK_FMT_MONTGOMERY = x * 2^256 mod p as 4 x u64, the
 *     in-memory form of pasta_curves (feature repr-c, Cargo.toml:42) and halo2curves field types, so Rust
 *     slices of `F` can be passed without conversion.
 *   - Affine point: x | y (64 bytes); the identity is (0, 0).  Result point: x | y | z (96 bytes) with
 *     z = 1 (finite) or x = y = z = 0 (identity), in the format asked for.
 *   - Ownership: the caller owns every buffer.  Contexts are created/destroyed by paired calls.
 *   - Errors: 0 = LURK_OK, negative = error; lurk_last_error() returns a thread-local message.  The library
 *     never aborts or unwinds (reference error style: Result<_, ProofError>, src/error.rs:8-18).
 *   - Threading: every call is re-entrant.  A `*_dev` call reads its device inputs in the order of the given CUDA stream (a
 *     cudaStream_t passed as void*; NULL = the legacy default stream): work queued on that stream before the call is complete before the
 *     call reads, also on the side streams some calls fork from it.  "Asynchronous" below: the call returns once its work is queued on the
 *     stream, and its device outputs are ready in the order of that stream.  "Returns when done": the call returns after its device work,
 *     its side streams' included, has finished, so its outputs may be read from any stream.  Every `*_dev` entry point says which.  The
 *     first call of a shape may also wait while it sets up tables or scratch (NTT twiddles, constant tables, MSM scratch growth).
 *     Host-buffer calls synchronise before returning.
 *   - Non-canonical inputs (>= p) are rejected with LURK_ERR_RANGE by the host-buffer calls (mirrors
 *     from_repr failing, src/field.rs:76-81); `*_dev` calls assume reduced inputs.
 *   - There is no CPU fallback: without a CUDA device every compute call returns LURK_ERR_NOGPU.
 */
#ifndef LURK_B200_H
#define LURK_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* LanguageField (src/field.rs:40-50) */
#define LURK_FIELD_BN254_FR 0  /* LanguageField::BN256   = halo2curves::bn256::Fr  (default, all benches) */
#define LURK_FIELD_BN254_FQ 1  /* LanguageField::Grumpkin = grumpkin::Fr = bn256::Fq                       */
#define LURK_FIELD_PALLAS_FQ 2 /* LanguageField::Pallas  = pallas::Scalar                                  */
#define LURK_FIELD_PALLAS_FP 3 /* LanguageField::Vesta   = vesta::Scalar = pallas::Base                    */

/* curves of the Nova curve cycles (src/proof/nova.rs:57-71) */
#define LURK_CURVE_BN254_G1 0 /* base Fq(1), scalars Fr(0) */
#define LURK_CURVE_GRUMPKIN 1 /* base Fr(0), scalars Fq(1) */
#define LURK_CURVE_PALLAS 2   /* base Fp(3), scalars Fq(2) */
#define LURK_CURVE_VESTA 3    /* base Fq(2), scalars Fp(3) */

#define LURK_FMT_CANONICAL 0
#define LURK_FMT_MONTGOMERY 1

#define LURK_OK 0
#define LURK_ERR_ARG (-1)
#define LURK_ERR_CUDA (-2)
#define LURK_ERR_OOM (-3)
#define LURK_ERR_RANGE (-4)
#define LURK_ERR_NOGPU (-5)
#define LURK_ERR_ORDER (-6) /* DAG nodes not topologically ordered */

const char *lurk_last_error(void);
int lurk_version(void);
int lurk_device_count(void);
/* modulus of a field as 32 bytes LE */
int lurk_field_modulus(int field_id, uint8_t out[32]);

/* ---------------------------------------------------------------------------------------------------
 * S1  Poseidon digests.  Replaces PoseidonCache::hash3/hash4/hash6/hash8 = neptune
 *     Poseidon::new_with_preimage(..).hash() (src/hash.rs:180-203) for a batch of independent preimages.
 *     arity in {3,4,6,8}; preimages n*arity elements, digests n elements.
 * ------------------------------------------------------------------------------------------------- */
int lurk_poseidon_hash_batch(int field_id, int arity, const uint8_t *preimages, size_t n, uint8_t *digests);
int lurk_poseidon_hash_batch_mont(int field_id, int arity, const uint8_t *preimages, size_t n, uint8_t *digests);
/* Asynchronous. */
int lurk_poseidon_hash_batch_dev(int field_id, int arity, const void *d_preimages, size_t n, void *d_digests,
                                 int fmt, void *stream);
/* Constants as PoseidonConstants::new() builds them (src/hash.rs:61-72): R_F, R_P, the t*(R_F+R_P) round
 * constants and the t*t MDS matrix (row-major), canonical form.  Buffers may be NULL to query sizes. */
int lurk_poseidon_constants(int field_id, int arity, int *full_rounds, int *partial_rounds,
                            uint8_t *round_constants, uint8_t *mds);

/* ---------------------------------------------------------------------------------------------------
 * S3  Slot witnesses.  Replaces the per-slot body of generate_slots_witnesses (src/lem/multiframe.rs:520-592):
 *     allocate_slot -> neptune circuit2 poseidon_hash_allocated in witness mode (src/lem/circuit.rs:212-315).
 *     Output block per slot = [preimage (arity) | 3 aux per S-box in Neptune's optimised-round order | digest],
 *     lurk_poseidon_witness_block() elements (= hashN_cost + N, src/lem/multiframe.rs:503-516).
 *     Bit-decomposition slots: [value | aux of AllocatedNum::to_bits_le_strict] (src/lem/circuit.rs:241-243),
 *     lurk_bitdecomp_witness_block() elements (= BIT_DECOMP_*_WITNESS_SIZE, src/lem/multiframe.rs:495-498).
 * ------------------------------------------------------------------------------------------------- */
size_t lurk_poseidon_witness_block(int field_id, int arity);
int lurk_poseidon_witness_batch(int field_id, int arity, const uint8_t *preimages, size_t n, uint8_t *blocks,
                                int fmt);
/* The _dev and _scatter_dev witness forms below are asynchronous. */
int lurk_poseidon_witness_batch_dev(int field_id, int arity, const void *d_preimages, size_t n, void *d_blocks,
                                    int fmt, void *stream);
/* In-place form for the step witness: block k is written at element offset d_offsets[k] (u64, device) of d_base.  In the
 * reference every frame's aux is [its slot blocks in slot order | LEM body aux] (synthesize_frames_parallel,
 * src/lem/multiframe.rs:635-712), so the blocks of one slot type are strided by the frame length (9119 on BN256). */
int lurk_poseidon_witness_scatter_dev(int field_id, int arity, const void *d_preimages, size_t n, void *d_base,
                                      const void *d_offsets, int fmt, void *stream);
int lurk_bitdecomp_witness_scatter_dev(int field_id, const void *d_values, size_t n, void *d_base, const void *d_offsets,
                                       int fmt, void *stream);
size_t lurk_bitdecomp_witness_block(int field_id);
int lurk_bitdecomp_witness_batch(int field_id, const uint8_t *values, size_t n, uint8_t *blocks, int fmt);
int lurk_bitdecomp_witness_batch_dev(int field_id, const void *d_values, size_t n, void *d_blocks, int fmt,
                                     void *stream);

/* SHA-256 coprocessor (synthesize_sha256, src/coprocessor/sha256.rs:27-64): the witness of one call with n pointers,
 * in allocation order: per pointer the aux of to_bits_le_strict of its tag, then of its hash; the aux of bellpepper's
 * sha256 gadget over their bits; pack_bits' element (the digest's low CAPACITY bits, equal to compute_sha256,
 * sha256.rs:66-90); allocate_constant's ExprTag::Num.  Bits are 0/1 elements in `fmt`.  The block's length depends on
 * (field, n) only and is what lurk_sha256_witness_block returns (0: unsupported field or n outside 1..MAX_N).
 * inputs: count * 2n elements in `fmt`, per pointer tag then hash.  The host call rejects elements >= p (LURK_ERR_RANGE).
 * The _dev and scatter forms are asynchronous. */
#define LURK_SHA256_MAX_N 32
size_t lurk_sha256_witness_block(int field_id, int n);
int lurk_sha256_witness_batch(int field_id, int n, const uint8_t *inputs, size_t count, uint8_t *aux_out, int fmt);
int lurk_sha256_witness_batch_dev(int field_id, int n, const void *d_inputs, size_t count, void *d_aux, int fmt, void *stream);
/* In-place form: block k is written at element offset d_offsets[k] (u64, device) of d_W. */
int lurk_sha256_witness_scatter_dev(int field_id, int n, const void *d_inputs, size_t count, const uint64_t *d_offsets, void *d_W,
                                    int fmt, void *stream);

/* Trie coprocessor (src/coprocessor/trie/mod.rs): the witness of one lookup (synthesize_lookup_aux, mod.rs:118-156) or
 * insert (synthesize_insert_aux, mod.rs:226-268) over an arity-8 trie of height H = 1..LURK_TRIE_MAX_HEIGHT (StandardTrie:
 * 85), in allocation order, with D = lurk_bitdecomp_witness_block(field_id):
 *   allocated_root_value | the D - 1 aux of key.to_bits_le_strict | per level L = 0..H-1 (root level first): the 8
 *   preimage elements, their arity-8 Poseidon aux and digest (the slot block), select's 7 picks (most significant bit
 *   first: 4, 2, 1; the last pick of level H-1 is the lookup's result)
 * and, for an insert, then per level L = H-1 down to 0: the new preimage's slot block (the last element is the new root).
 * Lookup: D + 403 H elements, insert: D + 799 H; lurk_trie_witness_block returns it (0: unsupported field, op or height).
 * inputs, per call in `fmt`, paths root level first: lookup root, key, path[H][8] (2 + 8H elements); insert root, key,
 * value, old_path[H][8], new_path[H][8] (3 + 16H) -- the reference's LookupProof / InsertProof preimages.
 * The host call rejects elements >= p (LURK_ERR_RANGE) and, after the copy back, paths that do not chain
 * (LURK_ERR_ARG, naming the call and level): each level's digest must equal the element its parent selects (level 0:
 * root), and for an insert the new path's elements at the key must equal the digest of the level below, the leaf's the
 * value.  The _dev and scatter forms do not check paths: the caller vouches for them.  They are asynchronous. */
#define LURK_TRIE_LOOKUP 0
#define LURK_TRIE_INSERT 1
#define LURK_TRIE_MAX_HEIGHT 85
size_t lurk_trie_witness_block(int field_id, int op, int height);
int lurk_trie_witness_batch(int field_id, int op, int height, const uint8_t *inputs, size_t count, uint8_t *aux_out, int fmt);
int lurk_trie_witness_batch_dev(int field_id, int op, int height, const void *d_inputs, size_t count, void *d_aux, int fmt,
                                void *stream);
/* In-place form: block k is written at element offset d_offsets[k] (u64, device) of d_W. */
int lurk_trie_witness_scatter_dev(int field_id, int op, int height, const void *d_inputs, size_t count, const uint64_t *d_offsets,
                                  void *d_W, int fmt, void *stream);

/* Device-resident trie node store (the reference's Trie over its inverse Poseidon cache, arity 8, height H = 1..
 * LURK_TRIE_MAX_HEIGHT): content-addressed nodes, digest -> 8-element preimage, only ever added.  Creation registers the
 * H empty roots; on a machine without a GPU the context is created without a store and every call that needs one returns
 * LURK_ERR_NOGPU.  capacity_nodes bounds the node count (H .. 2^31 - 1); the store takes about 300 bytes per node.
 * One context is used by one thread at a time; separate contexts may run on separate threads. */
typedef struct lurk_trie_ctx lurk_trie_ctx;
int lurk_trie_ctx_create(int field_id, int height, uint64_t capacity_nodes, lurk_trie_ctx **out);
void lurk_trie_ctx_destroy(lurk_trie_ctx *ctx);
/* the root of the empty trie of height H, in fmt */
int lurk_trie_ctx_empty_root(lurk_trie_ctx *ctx, uint8_t out[32], int fmt);
int lurk_trie_ctx_info(const lurk_trie_ctx *ctx, uint64_t *node_count, uint64_t *capacity);
/* Add n existing nodes (preimages: n x 8 elements in fmt, e.g. a host inverse cache), hashed on the GPU; their digests
 * go to digests_out (n elements in fmt, may be NULL).  A node already stored is not added again.  Returns when done. */
int lurk_trie_ctx_register(lurk_trie_ctx *ctx, const uint8_t *preimages, size_t n, uint8_t *digests_out, int fmt);
/* Apply n operations in program order, exactly as the reference's sequential Trie would.  Operation i: kinds[i]
 * LURK_TRIE_LOOKUP or LURK_TRIE_INSERT, keys[i], values[i] (read for inserts only), and its root: prev[i] = -1 names
 * roots[i], which must be stored; prev[i] = j < i names the root insert j of this batch produced.  An insert with prev =
 * j continues j's chain and j must be that chain's latest insert (no forks inside a batch; each insert with prev = -1
 * starts its own chain, forks from a stored root are fine); a lookup may name any earlier insert and reads that version.
 * A key's path is its low 3H bits, most significant 3-bit chunk first.  Arrays are host memory of n entries (elements
 * 32 bytes in fmt); roots[i] is read only where prev[i] = -1 and values[i] only for an insert, so roots may be NULL
 * when every prev[i] >= 0 and values when the batch has no insert.
 * results_out (n elements in fmt, may be NULL): a lookup's value (0 when absent), an insert's new root.  The proofs go
 * to device memory in fmt, in lurk_trie_witness_batch's input layout: the lookups' in their program order to
 * d_lookup_inputs (2 + 8H elements each), the inserts' to d_insert_inputs (3 + 16H each); either may be NULL.  New nodes
 * are registered, so later batches may start from any root produced.
 * Refused before any launch, with the operation's index in lurk_last_error(), as LURK_ERR_ARG: a bad kind or prev, a
 * fork, an element >= p, a NULL roots or values array that is read, node count + H x inserts > capacity (naming the
 * first insert that would not fit).  Then
 * LURK_ERR_NOGPU.  A root or node missing from the store (the reference's MissingPreimage) returns LURK_ERR_RANGE naming
 * the first such operation and the digest; the store, the node count and the outputs are then left as they were.
 * Ordered on `stream` after the caller's earlier work there; returns when the batch is applied. */
int lurk_trie_ctx_apply(lurk_trie_ctx *ctx, size_t n, const int *kinds, const int64_t *prev, const uint8_t *roots, const uint8_t *keys,
                        const uint8_t *values, int fmt, uint8_t *results_out, void *d_lookup_inputs, void *d_insert_inputs, void *stream);
/* Device-resident forms, for operations and preimages already in device memory (e.g. a replay batch uploaded in one copy).
 * lurk_trie_ctx_apply_dev: lurk_trie_ctx_apply with every array in device memory -- d_kinds (int32), d_prev (int64),
 * d_roots / d_keys / d_values (n elements in fmt; d_roots and d_values may be NULL when never read), d_results (n elements
 * in fmt, may be NULL) -- and the batch planned on the GPU instead of the host.  The proof buffers are sized by the
 * caller, as for lurk_trie_ctx_apply.  Refused on the host, as LURK_ERR_ARG and in this order, before LURK_ERR_NOGPU: a
 * null ctx, a bad fmt, NULL d_kinds, d_prev or d_keys with n > 0, n >= 2^31.  Every other refusal is found on the device
 * and returns the code lurk_trie_ctx_apply returns on the same arrays, naming the same operation: a bad kind or prev, a
 * prev naming a lookup, a fork, an element >= p, a NULL d_roots or d_values that would be read, the capacity (the first
 * insert that does not fit), MissingPreimage (LURK_ERR_RANGE, with the digest).  On any refusal the store, the node count,
 * d_results and the proof buffers are left as they were.
 * lurk_trie_ctx_register_dev: lurk_trie_ctx_register with d_preimages (n x 8 elements in fmt) and d_digests_out (n in
 * fmt, may be NULL) in device memory.  Refused on the host as LURK_ERR_ARG, in this order and before LURK_ERR_NOGPU: a
 * null ctx, a bad fmt, NULL d_preimages with n > 0, n over the remaining capacity; an element >= p is found on the device
 * and refused as LURK_ERR_ARG naming the preimage and the element.
 * Both are ordered on `stream` after the caller's earlier work there and return when the batch is applied (so the error
 * is exact); neither returns before its device work is done. */
int lurk_trie_ctx_apply_dev(lurk_trie_ctx *ctx, size_t n, const int32_t *d_kinds, const int64_t *d_prev, const void *d_roots, const void *d_keys,
                            const void *d_values, int fmt, void *d_results, void *d_lookup_inputs, void *d_insert_inputs, void *stream);
int lurk_trie_ctx_register_dev(lurk_trie_ctx *ctx, const void *d_preimages, size_t n, void *d_digests_out, int fmt, void *stream);

/* ---------------------------------------------------------------------------------------------------
 * S2  DAG hydration.  Replaces StoreCore::hydrate_z_cache / hash_ptr_val_unsafe (src/lem/store_core.rs:199-269)
 *     with the preimage layouts of `impl StoreHasher for PoseidonCache` (src/lem/store.rs:29-78).
 *     child[i] < n_atoms refers to atom digest child[i]; otherwise to node (child[i] - n_atoms), which must
 *     precede the referring node (children first).  out_digests: n elements, canonical.
 * ------------------------------------------------------------------------------------------------- */
#define LURK_DAG_TUPLE2 2     /* H4 [t0, d0, t1, d1]                 hash_ptrs len 2 (store.rs:31-36)  */
#define LURK_DAG_TUPLE3 3     /* H6                                   hash_ptrs len 3 (store.rs:37-50)  */
#define LURK_DAG_TUPLE4 4     /* H8                                   hash_ptrs len 4 (store.rs:51-67)  */
#define LURK_DAG_COMPACT 5    /* H4 [d0, t1, d1, d2]                  hash_compact    (store.rs:75-77)  */
#define LURK_DAG_COMMITMENT 6 /* H3 [d0 = secret, t1, d1]            hash_commitment (store.rs:70-73)  */
typedef struct lurk_dag_node {
    uint8_t kind;
    uint8_t reserved;
    uint16_t tag[4];   /* Tag::to_field = F::from(u16) (src/tag.rs:99-101) */
    uint32_t child[4];
} lurk_dag_node;
int lurk_dag_hash(int field_id, const lurk_dag_node *nodes, size_t n, const uint8_t *atom_digests,
                  size_t n_atoms, uint8_t *out_digests);
/* Routing aid, host only (works without a GPU): shape of the dependency DAG and a cost estimate.  A level costs one
 * dependent Poseidon latency on the GPU whatever its width, so deep and narrow stores (lists hashed cons by cons) are
 * faster on the caller's own CPU path (hash_ptr_val_unsafe, src/lem/store_core.rs:199-248), wide ones on the GPU.  The
 * library never hashes on the CPU itself: use_gpu == 0 means "keep this hydration on the reference's CPU path". */
typedef struct lurk_dag_plan {
    uint64_t nodes, levels, max_width;
    uint64_t est_gpu_us;       /* levels * ~170 us + nodes / 23 M/s + transfers */
    uint64_t est_cpu_core_us;  /* nodes * ~50 us on one core */
    int use_gpu;               /* est_gpu_us < the level-parallel CPU estimate on 8 cores */
} lurk_dag_plan;
int lurk_dag_hash_plan(const lurk_dag_node *nodes, size_t n, size_t n_atoms, lurk_dag_plan *plan);

/* ---------------------------------------------------------------------------------------------------
 * S4  Pedersen commitment = multi-scalar multiplication.  Replaces Arecibo
 *     CommitmentEngineTrait::commit -> DlogGroup::vartime_multiscalar_mul(scalars, bases) (called from
 *     RecursiveSNARK::prove_step, src/proof/nova.rs:287,292; supernova.rs:231-244).  The fixed commitment key
 *     is uploaded once into a context; each call streams scalars.
 * ------------------------------------------------------------------------------------------------- */
typedef struct lurk_msm_ctx lurk_msm_ctx;
/* bases_affine: n * 64 bytes, x || y per point, (0, 0) = identity.  Coordinates >= p or points off the curve are
 * rejected with LURK_ERR_RANGE (what the reference's point deserialisation checks before a key is used).  A context
 * belongs to the device that is current at creation; using it with another device current is LURK_ERR_ARG. */
int lurk_msm_ctx_create(int curve_id, const uint8_t *bases_affine, size_t n, int fmt, lurk_msm_ctx **out);
/* bases already on the current device (n * 64 bytes, Montgomery); the context borrows the pointer */
int lurk_msm_ctx_create_dev(int curve_id, const void *d_bases_mont, size_t n, lurk_msm_ctx **out);
void lurk_msm_ctx_destroy(lurk_msm_ctx *ctx);
/* curve and number of bases of a context (either output may be NULL) */
int lurk_msm_ctx_info(lurk_msm_ctx *ctx, int *curve_id, size_t *n);
/* sum_{i<n} scalars[i] * bases[i], n <= size of the key */
int lurk_msm_ctx_run(lurk_msm_ctx *ctx, const uint8_t *scalars, size_t n, int fmt, uint8_t out_xyz[96]);
/* _dev: returns when done (the point is a host output). */
int lurk_msm_ctx_run_dev(lurk_msm_ctx *ctx, const void *d_scalars, size_t n, int fmt, uint8_t out_xyz[96],
                         void *stream);
/* Fixed-base acceleration (the key never changes between folds): builds table[w][i] = 2^(c w) * bases[i] once
 * (nwin x n x 64 bytes of HBM; 1.7 GB for a 2^21-point key) so that all windows share one bucket set and a wider
 * window (c = 20) becomes affordable: ~13 instead of 16 bucket additions per scalar.  Results are unchanged.
 * Call before cloning; clones share the table. */
int lurk_msm_ctx_precompute(lurk_msm_ctx *ctx);
/* The same with a chosen window width c (10 .. 22: at most 26 windows) instead of the one the key's size suggests: the fold context builds its own tables
 * with c = 16, where one bucket set (2^15 counters) fits a CTA's shared memory and the digit sort keeps its histogram on chip.
 * LURK_ERR_ARG when the context already has a table. */
int lurk_msm_ctx_precompute_window(lurk_msm_ctx *ctx, int c);
/* Asynchronous form: `launch` enqueues the whole commitment on `stream` and returns; `finish` waits for it and
 * produces the point.  One launch may be pending per context; `clone` gives another context on the same resident key
 * (own scratch; the parent must outlive it) so that e.g. commit(W) and commit(T) of one fold overlap. */
int lurk_msm_ctx_launch_dev(lurk_msm_ctx *ctx, const void *d_scalars, size_t n, int fmt, void *stream);
int lurk_msm_ctx_finish(lurk_msm_ctx *ctx, uint8_t out_xyz[96]);
int lurk_msm_ctx_clone(lurk_msm_ctx *ctx, lurk_msm_ctx **out);
/* Measurement hooks: when enabled, every run records CUDA events around the bucket-accumulation kernel (the dominant
 * kernel) on the launching stream; last_profile returns its duration and the number of kernels the run launched. */
int lurk_msm_ctx_set_profiling(lurk_msm_ctx *ctx, int enable);
int lurk_msm_ctx_last_profile(lurk_msm_ctx *ctx, float *accumulate_ms, unsigned *kernel_launches);
/* with profiling enabled: device time of the last finished run's digit sort (first memset to the end of the scatter kernel) */
int lurk_msm_ctx_last_sort_ms(lurk_msm_ctx *ctx, float *sort_ms);
/* one-shot convenience (uploads bases every call) */
int lurk_msm(int curve_id, const uint8_t *bases_affine, const uint8_t *scalars, size_t n, int fmt,
             uint8_t out_xyz[96]);
/* Synthetic commitment key: bases_out[i] = [start + i + 1] G for the curve's standard generator, affine, n * 64 bytes
 * (host, multi-threaded).  The reference derives its key by hash-to-curve / powers of tau inside Arecibo
 * (public_params, src/proof/nova.rs:196-216) -- out of scope; this gives benches and tests a deterministic key of
 * distinct points (SURVEY.md 8(d) config 3). */
int lurk_synthetic_bases(int curve_id, uint64_t start, size_t n, int fmt, uint8_t *bases_out);
/* host-side sum of `count` result points (the per-GPU partial sums of a sharded commitment key) */
int lurk_point_sum(int curve_id, const uint8_t *points_xyz, size_t count, int fmt, uint8_t out_xyz[96]);

/* ---------------------------------------------------------------------------------------------------
 * N3  Commitment-key generation.  Replaces what `public_params` (src/proof/nova.rs:196-216, supernova.rs:117-137; cached on
 *     disk by src/public_parameters/mod.rs:20-71 because it takes minutes on the CPU) makes Arecibo do for the Pedersen key:
 *     R1CSShape::commitment_key -> CommitmentKey::setup(b"ck", n), n = next_power_of_two(max(#cons, #vars, ck_floor)) ->
 *     DlogGroup::from_label(label, n):  uniform_i = next 32 bytes of SHAKE256(label);
 *     G_i = Curve::hash_to_curve("from_uniform_bytes")(uniform_i), affine.
 *     hash_to_curve = halo2curves 0.6 (BN254 G1 / Grumpkin: BLAKE2b expand_message_xmd + Shallue-van de Woestijne, RFC 9380)
 *     or pasta_curves 0.5 (Pallas / Vesta: same hash_to_field + simplified SWU on the 3-isogenous curve + isogeny).
 *     The XOF is sequential and stays on a host thread, pipelined against the kernel that maps the points.
 * ------------------------------------------------------------------------------------------------- */
/* next_power_of_two(max(num_cons, num_vars, ck_floor)): the key length public_params asks for.  Host only. */
size_t lurk_ck_size(size_t num_cons, size_t num_vars, size_t ck_floor);
/* from_label: n affine points x | y (64 bytes each, identity = (0, 0)) in `fmt`. */
int lurk_ck_generate(int curve_id, const uint8_t *label, size_t label_len, size_t n, int fmt, uint8_t *bases_out);
/* same, written to device memory in Montgomery form -- exactly what lurk_msm_ctx_create_dev borrows: the key never crosses
 * PCIe.  Returns when the key is complete (the host thread feeds the XOF stream while the GPU works). */
int lurk_ck_generate_dev(int curve_id, const uint8_t *label, size_t label_len, size_t n, void *d_bases_mont, void *stream);
/* points first .. first + n - 1 of the same key: a rank's contiguous slice of a key sharded over GPUs (SURVEY.md 8(e)); returns when
 * complete, as lurk_ck_generate_dev */
int lurk_ck_generate_range_dev(int curve_id, const uint8_t *label, size_t label_len, size_t first, size_t n, void *d_bases_mont,
                               void *stream);
/* Curve::hash_to_curve(domain_prefix)(message) for n messages of msg_len bytes each (msg_len <= 64 and
 * msg_len + strlen(domain_prefix) <= ~80: everything must fit the single-block layout, else LURK_ERR_ARG). */
int lurk_hash_to_curve_batch(int curve_id, const char *domain_prefix, const uint8_t *messages, size_t msg_len, size_t n, int fmt,
                             uint8_t *points_out);
/* _dev: asynchronous. */
int lurk_hash_to_curve_batch_dev(int curve_id, const char *domain_prefix, const void *d_messages, size_t msg_len, size_t n,
                                 void *d_points, int fmt, void *stream);
/* Powers-of-tau key of the KZG engine (Arecibo hyperkzg CommitmentKey::setup -> UniversalKZGParam::gen_srs_for_testing; the
 * primary circuit's engine on BN256, src/proof/nova.rs:65-71): d_bases_mont[i] = beta^i * g for i < n, affine Montgomery, by
 * fixed-base windows of g.  g (64 bytes affine) and beta (32 bytes, scalar field) in `fmt`; how the reference derives them from
 * the label (a seeded RNG) and the verifier key's G2 side stay on the caller's CPU.  Returns when the key is complete. */
int lurk_ck_powers_dev(int curve_id, const uint8_t g[64], const uint8_t beta[32], size_t n, void *d_bases_mont, int fmt, void *stream);
/* SHAKE256(in) -> out_len bytes (FIPS 202).  Host only (works without a GPU); the XOF behind from_label. */
int lurk_shake256(const uint8_t *in, size_t in_len, uint8_t *out, size_t out_len);

/* ---------------------------------------------------------------------------------------------------
 * N4  The data-parallel loops of `compress` (src/proof/nova.rs:341-356, supernova.rs:293-317 -> Arecibo CompressedSNARK::prove ->
 *     spartan::snark::RelaxedR1CSSNARK::prove): sum-check prover rounds over device-resident multilinear polynomials
 *     (SumcheckProof::prove_quad / prove_cubic_with_additive_term: compute_eval_points_* + bind_poly_var_top) and the folding rounds
 *     of the inner-product argument (provider::ipa_pc::InnerProductArgument::prove), the HyperKZG opening prover
 *     (provider::hyperkzg::EvaluationEngine::prove), batch_eval_reduce (every evaluation claim of a proof reduced to one opening), plus
 *     EqPolynomial::evals and the inner product behind MultilinearPolynomial::evaluate.  The Fiat-Shamir transcript (Keccak256Transcript) stays on the caller's side:
 *     every round passes its message to `challenge` and receives the verifier's challenge.  Polynomials: 2^num_rounds elements,
 *     Montgomery form, index bit (num_rounds - 1) = the first variable (bound first), as in Arecibo's MultilinearPolynomial.
 *     The verifier's data-parallel parts are here too: the matrix evaluations of RelaxedR1CSSNARK::verify and the tensor MSM of
 *     InnerProductArgument::verify.  Not here: the transcript, proof (de)serialisation, HyperKZG's pairing check -- CPU / third-party
 *     protocol code.
 * ------------------------------------------------------------------------------------------------- */
/* message: the round's prover message in `fmt` -- sum-check: s(0) | s(1) | s(2) [| s(3)] (32 bytes each; Arecibo absorbs the
 * compressed form, i.e. the coefficients without the linear one: the caller converts);  IPA: L | R as 96-byte points.
 * Writes the challenge (32 bytes, `fmt`) and returns 0, or non-zero to abort the proof. */
typedef int (*lurk_challenge_fn)(void *user, int round, const uint8_t *message, size_t message_len, uint8_t challenge_out[32]);
#define LURK_SUMCHECK_QUAD 0  /* claim = sum_i A[i] B[i]                 d_polys = {A, B}          degree 2 */
#define LURK_SUMCHECK_CUBIC 1 /* claim = sum_i A[i] (B[i] C[i] - D[i])   d_polys = {A, B, C, D}    degree 3 */
/* Runs all num_rounds rounds.  The polynomials are consumed (bound in place; element 0 of each ends as its final evaluation).
 * round_evals: num_rounds x (degree + 1) x 32 bytes; challenges: num_rounds x 32; final_evals: 2 or 4 x 32 (any may be NULL).
 * Returns when done, as every call below that takes a challenge callback. */
int lurk_sumcheck_prove_dev(int field_id, int kind, void *const *d_polys, int num_rounds, const uint8_t claim[32],
                            lurk_challenge_fn challenge, void *user, uint8_t *round_evals, uint8_t *challenges, uint8_t *final_evals,
                            int fmt, void *stream);
/* SumcheckProof::prove_quad_batch / prove_cubic_with_additive_term_batch (BatchedRelaxedR1CSSNARK: SuperNova's `compress`,
 * src/proof/supernova.rs:293-317): n_instances (<= 60) claims proven together, the round message is sum_i coeffs[i] * s_i(X).
 * Instance i has 2 or 4 polynomials of 2^num_rounds[i] elements (d_polys instance-major) and joins in round max - num_rounds[i];
 * before that its round polynomial is the constant 2^(remaining - num_rounds[i] - 1) * claims[i].  coeffs may be NULL (all 1).
 * round_evals: max_rounds x (degree + 1) x 32; challenges: max_rounds x 32; final_evals: n_instances x (2 | 4) x 32. */
int lurk_sumcheck_prove_batch_dev(int field_id, int kind, int n_instances, void *const *d_polys, const int *num_rounds,
                                  const uint8_t *claims, const uint8_t *coeffs, lurk_challenge_fn challenge, void *user,
                                  uint8_t *round_evals, uint8_t *challenges, uint8_t *final_evals, int fmt, void *stream);
/* EqPolynomial::new(tau).evals(): d_out[i] = prod_j (bit_j(i) ? tau[j] : 1 - tau[j]), tau[0] <-> the top index bit; 2^num_vars
 * elements in `fmt` (tau: host, num_vars x 32 bytes, same fmt).  Asynchronous. */
int lurk_eq_evals_dev(int field_id, const uint8_t *tau, int num_vars, void *d_out, int fmt, void *stream);
/* <a, b> over n Montgomery elements (MultilinearPolynomial::evaluate = <Z, eq(r)>; the c_L / c_R of an IPA round).  Synchronous. */
int lurk_inner_product_dev(int field_id, const void *d_a, const void *d_b, size_t n, uint8_t out[32], int fmt, void *stream);
/* one IPA folding step, in place on the first n / 2 slots: a[i] <- x a[i] + y a[i + n/2];  G[i] <- x G[i] + y G[i + n/2]
 * (CommitmentKey::fold; bases affine Montgomery; x, y host scalars in `fmt`).  Both asynchronous. */
int lurk_ipa_fold_scalars_dev(int field_id, void *d_a, size_t n, const uint8_t x[32], const uint8_t y[32], int fmt, void *stream);
int lurk_ipa_fold_bases_dev(int curve_id, void *d_bases_mont, size_t n, const uint8_t x[32], const uint8_t y[32], int fmt, void *stream);
/* All log_n rounds of InnerProductArgument::prove on device-resident a, b (2^log_n scalars each, Montgomery, consumed) under the
 * key of context `ck` (>= 2^log_n bases; NOT consumed): per round c_L = <a_lo, b_hi>, c_R = <a_hi, b_lo>,
 * L = commit(a_lo; G_hi) + c_L ck_c, R = commit(a_hi; G_lo) + c_R ck_c, r = challenge(L | R), a' = a_lo r + a_hi / r,
 * b' = b_lo / r + b_hi r, G' = G_lo / r + G_hi r.  The folded key G' is never materialised: the prover only needs commitments under
 * it, and those are Pippenger passes over the original key with scalars weighted by the products of the earlier challenges
 * (lurk_ipa_fold_bases_dev is the explicit CommitmentKey::fold for callers that want G').  ck_c: the (already scaled) base for the
 * inner-product value, 64 bytes affine in `fmt`.  L_out / R_out: log_n x 96 bytes. */
int lurk_ipa_prove_dev(int curve_id, lurk_msm_ctx *ck, const uint8_t ck_c[64], void *d_a, void *d_b, int log_n,
                       lurk_challenge_fn challenge, void *user, uint8_t *L_out, uint8_t *R_out, uint8_t a_final[32], uint8_t b_final[32],
                       int fmt, void *stream);
/* InnerProductArgument::verify for the claim <a, b> = c with comm = commit(a): per round r_j = challenge(j, L_j | R_j) (as in the prover),
 * s[i] = prod_j (bit_j(i) ? r_j : 1 / r_j) (bit 0 = the top bit of i), ck_hat = commit(ck, s) over 2^log_n bases of `ck` (NOT consumed),
 * b_hat = <b, s>; accepted iff a_final ck_hat + a_final b_hat ck_c == comm + c ck_c + sum_j (r_j^2 L_j + r_j^-2 R_j).  d_b: 2^log_n
 * Montgomery elements on the device (not modified); ck_c: 64 bytes affine; comm, L, R (log_n x 96), ck_hat_out: 96-byte points; scalars 32
 * bytes; all in `fmt`.  Points off the curve and values >= p are LURK_ERR_RANGE; a failed check is LURK_OK with *accepted = 0.
 * ck_hat_out / b_hat_out may be NULL.  Synchronous. */
int lurk_ipa_verify_dev(int curve_id, lurk_msm_ctx *ck, const uint8_t ck_c[64], const uint8_t comm[96], const uint8_t c[32], const void *d_b,
                        int log_n, const uint8_t *L, const uint8_t *R, const uint8_t a_final[32], lurk_challenge_fn challenge, void *user,
                        int *accepted, uint8_t ck_hat_out[96], uint8_t b_hat_out[32], int fmt, void *stream);
/* provider::hyperkzg::EvaluationEngine::prove (the opening argument of the primary BN256 circuit, EE1 in src/proof/nova.rs:65-71):
 * d_poly = 2^num_vars evaluations (Montgomery, not modified), point = num_vars elements (host, `fmt`), ck = a context on the KZG key
 * (>= 2^num_vars bases).  Phase 1: P_{i+1}[j] = P_i[2j] + x_{l-1-i} (P_i[2j+1] - P_i[2j]) and com_i = commit(P_i), i = 1..l-1;
 * challenge(round 0, com) -> r; u = (r, -r, r^2); v[t][j] = P_j(u_t); challenge(round 1, v) -> q; B = sum_j q^j P_j;
 * w_t = commit(B(X) / (X - u_t)); challenge(round 2, w) is called for the transcript's sake.
 * com_out: (num_vars - 1) x 96; w_out: 3 x 96; v_out: 3 x num_vars x 32 (v[t][j] at (t * num_vars + j)). */
int lurk_hyperkzg_prove_dev(int curve_id, lurk_msm_ctx *ck, const void *d_poly, const uint8_t *point, int num_vars,
                            lurk_challenge_fn challenge, void *user, uint8_t *com_out, uint8_t *w_out, uint8_t *v_out, int fmt,
                            void *stream);
/* Arecibo's batch_eval_reduce (with PolyEvalInstance / PolyEvalWitness::batch_diff_size; public crate, not under the reference checkout):
 * reduces n_claims (1..60) evaluation claims P_i(x_i) = e_i to ONE claim about one polynomial, so that `compress` ends in a single
 * opening.  d_polys[i]: 2^num_vars[i] Montgomery elements (0 <= num_vars[i] <= 40; NOT modified); points: the x_i concatenated, num_vars[i]
 * elements each, x_i[0] <-> the top index bit (may be NULL when every num_vars[i] is 0); evals: the e_i.  m = max num_vars[i].
 *   round 0:      message e_0 | .. | e_{n-1}                 -> rho
 *   rounds 1..m:  SumcheckProof::prove_quad_batch over (P_i, eq(x_i)), claims e_i, coefficients rho^i, instance i joining late as in
 *                 lurk_sumcheck_prove_batch_dev; message s(0) | s(1) | s(2)  -> r_{j-1}
 *   round m + 1:  message L_0 | .. | L_{n-1}, L_i = P_i(r[m - n_i:])   -> gamma
 * Outputs (any but d_joint may be NULL): round_evals m x 3 x 32; r_out m x 32; claims_left the L_i; weights w_i = gamma^i (the caller
 * forms the joint commitment sum_i w_i C_i); joint_eval = sum_i gamma^i prod_{j < m - n_i} (1 - r_j) L_i; d_joint (caller-allocated,
 * 2^m Montgomery elements, not overlapping any P_i) d_joint[k] = sum_{i : k < 2^n_i} gamma^i P_i[k] -- the polynomial to open at r. */
int lurk_batch_eval_reduce_dev(int field_id, int n_claims, const void *const *d_polys, const int *num_vars,
                               const uint8_t *points, const uint8_t *evals, lurk_challenge_fn challenge, void *user,
                               uint8_t *round_evals, uint8_t *r_out, uint8_t *claims_left, uint8_t *weights,
                               uint8_t joint_eval[32], void *d_joint, int fmt, void *stream);

/* Spartan prover context: RelaxedR1CSSNARK::prove (Nova's `compress`, src/proof/nova.rs:341-356) and
 * BatchedRelaxedR1CSSNARK::prove (SuperNova's, supernova.rs:293-317) in one call each, from the fold context's running instance.
 * The context is created once per circuit shape: the same CSR-over-z = (W, u, X) description as lurk_fold_config: columns
 * < n_w + 1 + n_x, coefficients in `fmt`.  It keeps the three matrices on the device and builds there, by counting sort, the merged
 * transpose the evaluation table needs (rows = indices of the padded z = (W | 0.. | u | X | 0..) of 2 num_vars elements, entries of
 * A, B, C grouped in that order within a row).  num_vars = 2^log_vars = next power of two of max(n_w, n_x + 1) (at least 2);
 * rows are padded to 2^log_rows.  joint_len = 2^max(log_rows, log_vars): the length of the joint polynomial of a plain proof.
 * Matrices of one context are used by one call at a time. */
typedef struct lurk_spartan_ctx lurk_spartan_ctx;
int lurk_spartan_ctx_create(int field_id, uint64_t n_w, uint64_t n_x, uint64_t n_rows, const uint64_t *const row_ptr[3],
                            const uint32_t *const col[3], const uint8_t *const val[3], int fmt, lurk_spartan_ctx **out);
/* A verifier-only context: the same arguments and checks, the three CSRs uploaded and range-checked, but no merged transpose,
 * eval-table slots or tickets (the prover's).  lurk_spartan_matrix_evals_dev, lurk_spartan_verify, lurk_spartan_verify_batch and
 * lurk_recursive_verify(_dev) take it and give exactly what a full context gives; lurk_spartan_prove_dev, _prove_batch_dev,
 * _eval_table_dev and lurk_compress_ctx_create refuse it with LURK_ERR_ARG.  Destroyed by lurk_spartan_ctx_destroy. */
int lurk_spartan_ctx_create_verifier(int field_id, uint64_t n_w, uint64_t n_x, uint64_t n_rows, const uint64_t *const row_ptr[3],
                                     const uint32_t *const col[3], const uint8_t *const val[3], int fmt, lurk_spartan_ctx **out);
void lurk_spartan_ctx_destroy(lurk_spartan_ctx *ctx);
/* any output may be NULL */
int lurk_spartan_ctx_info(lurk_spartan_ctx *ctx, int *field_id, int *log_rows, int *log_vars, size_t *joint_len);
/* The transcript.  `phase` says what the message is; `round` numbers the calls of one phase.
 *   LURK_SPARTAN_TAU         plain: rounds 0 .. log_rows - 1, empty message -> tau_i;  batched: round 0, empty -> tau
 *                            (instance i's table is eq(tau, tau^2, tau^4, ..), PowPolynomial::evals_with_powers)
 *   LURK_SPARTAN_OUTER_R     batched only, round 0, empty -> outer_r (instance i's coefficient outer_r^i)
 *   LURK_SPARTAN_OUTER       each outer (cubic) sum-check round: s(0) | s(1) | s(2) | s(3) -> r_x[j]
 *   LURK_SPARTAN_CLAIMS      round 0: Az, Bz, Cz, E at rx_i, instance after instance -> r (joint_i = Az + r Bz + r^2 Cz; batched
 *                            coefficients (r^3)^i)
 *   LURK_SPARTAN_INNER       each inner (quadratic) sum-check round: s(0) | s(1) | s(2) -> r_y[j]
 *   LURK_SPARTAN_BATCH_EVAL  rounds 0 .. m + 1 of lurk_batch_eval_reduce_dev over [W_0 .. W_{n-1}, E_0 .. E_{n-1}] at
 *                            [ry_0[1:] .., rx_0 ..]
 * The caller absorbs the verifier key's digest and the instance U into its transcript before the call, as Arecibo does.
 * Writes the challenge (32 bytes, `fmt`) and returns 0, or non-zero to abort the proof. */
#define LURK_SPARTAN_TAU 0
#define LURK_SPARTAN_OUTER_R 1
#define LURK_SPARTAN_OUTER 2
#define LURK_SPARTAN_CLAIMS 3
#define LURK_SPARTAN_INNER 4
#define LURK_SPARTAN_BATCH_EVAL 5
typedef int (*lurk_spartan_challenge_fn)(void *user, int phase, int round, const uint8_t *message, size_t message_len,
                                         uint8_t challenge_out[32]);
/* Caller-owned host buffers (any may be NULL), `fmt`.  S = max log_rows, T = max log_vars + 1, m = max(S, T - 1), n instances. */
typedef struct lurk_spartan_proof {
    uint8_t *outer_rounds;  /* S x 4 x 32 */
    uint8_t *r_x;           /* S x 32; instance i's point is the last log_rows_i of them */
    uint8_t *claims;        /* n x 4 x 32: Az, Bz, Cz, E at rx_i */
    uint8_t *inner_rounds;  /* T x 3 x 32 */
    uint8_t *r_y;           /* T x 32; instance i's point is the last log_vars_i + 1 */
    uint8_t *eval_W;        /* n x 32: W_i at ry_i[1:] */
    uint8_t *reduce_rounds; /* m x 3 x 32: the reduction's sum-check */
    uint8_t *r;             /* m x 32: the point at which the joint polynomial is opened */
    uint8_t *claims_left;   /* 2n x 32 */
    uint8_t *weights;       /* 2n x 32: gamma^i; the joint commitment is sum_i weights_i C_i over [comm_W_0 .., comm_E_0 ..] */
    uint8_t *joint_eval;    /* 32 */
} lurk_spartan_proof;
/* RelaxedR1CSSNARK::prove followed by batch_eval_reduce over [W, E].  d_z = (W, u, X): n_w + 1 + n_x Montgomery elements, laid out as
 * LURK_FOLD_BUF_Z1 holds them; d_E: n_rows Montgomery elements.  Both are read, never written.  d_joint (2^m elements, not overlapping
 * d_z or d_E) receives the joint polynomial, ready for lurk_hyperkzg_prove_dev or lurk_ipa_prove_dev.  Everything runs on `stream`;
 * the call returns when the proof is complete. */
int lurk_spartan_prove_dev(lurk_spartan_ctx *ctx, const void *d_z, const void *d_E, lurk_spartan_challenge_fn challenge, void *user,
                           lurk_spartan_proof *out, void *d_joint, int fmt, void *stream);
/* BatchedRelaxedR1CSSNARK::prove over n (1..30) running instances, instance i of shape ctxs[i] (shapes may differ; one field).  Returns when
 * the proof is complete. */
int lurk_spartan_prove_batch_dev(int n, lurk_spartan_ctx *const *ctxs, const void *const *d_z, const void *const *d_E,
                                 lurk_spartan_challenge_fn challenge, void *user, lurk_spartan_proof *out, void *d_joint, int fmt,
                                 void *stream);
/* compute_eval_table_sparse alone: d_out[j] = sum_rows eq_rx[row] (A[row][j] + r B[row][j] + r^2 C[row][j]) over the padded z's
 * columns (2 num_vars elements); d_eq_rx: 2^log_rows Montgomery elements; r: 32 bytes in `fmt`.  For callers that schedule the
 * primitives themselves.  Asynchronous. */
int lurk_spartan_eval_table_dev(lurk_spartan_ctx *ctx, const void *d_eq_rx, const uint8_t r[32], void *d_out, int fmt, void *stream);
/* The verifier's side (RelaxedR1CSSNARK::verify, BatchedRelaxedR1CSSNARK::verify: CompressedSNARK::verify, src/proof/nova.rs:358-373).
 * lurk_spartan_matrix_evals_dev: the multilinear extensions of A, B, C at (r_x, r_y) -- r_x: log_rows elements, r_y: log_vars + 1
 * elements over the padded z, both `fmt`; out = A | B | C (3 x 32, `fmt`).  One pass over the context's non-zeros with eq(r_x) and
 * eq(r_y) looked up in product-tensor tables in shared memory: no O(rows) or O(columns) scratch.  Synchronous. */
int lurk_spartan_matrix_evals_dev(lurk_spartan_ctx *ctx, const uint8_t *r_x, const uint8_t *r_y, uint8_t out[96], int fmt, void *stream);
/* Round polynomials of a proof handed to the verifiers:
 *   LURK_SPARTAN_ROUNDS_EVALS       s(0) | s(1) | .. | s(d) per round, as lurk_spartan_prove_dev writes them (outer S x 4, inner T x 3,
 *                                   reduction m x 3 elements); each round must sum to the running claim.
 *   LURK_SPARTAN_ROUNDS_COMPRESSED  Arecibo's CompressedUniPoly: every coefficient but the linear one, constant first (outer S x 3,
 *                                   inner T x 2, reduction m x 2 elements); the linear one is recovered from the running claim.
 * In both cases `challenge` receives the evaluations s(0) | .. | s(d), exactly the messages of the prover. */
#define LURK_SPARTAN_ROUNDS_EVALS 0
#define LURK_SPARTAN_ROUNDS_COMPRESSED 1
/* RelaxedR1CSSNARK::verify up to the opening, then the verifier of batch_eval_reduce over [W, E] at [r_y[1:], r_x].  u (32 bytes) and
 * X (n_x x 32 bytes) are the instance's public values, in `fmt`.  Reads outer_rounds, claims, inner_rounds, eval_W, reduce_rounds and
 * claims_left of `proof`; when the proof is accepted, writes r_x, r_y, r, weights and joint_eval wherever they are non-NULL (the bytes the
 * prover wrote).  `challenge` is called with the phases, rounds and messages of lurk_spartan_prove_dev, in the same order, so one transcript
 * drives both.  What remains for the caller is the opening: the joint commitment sum_i weights_i C_i over [comm_W, comm_E] at r has value
 * joint_eval.  A proof that fails a check is not an error: LURK_OK with *accepted = 0.  Values >= p are LURK_ERR_RANGE. */
int lurk_spartan_verify(lurk_spartan_ctx *ctx, const uint8_t u[32], const uint8_t *X, lurk_spartan_proof *proof, int rounds_fmt,
                        lurk_spartan_challenge_fn challenge, void *user, int *accepted, int fmt, void *stream);
/* BatchedRelaxedR1CSSNARK::verify over n (1..30) instances of shapes ctxs[i] (distinct contexts, one field): u = n x 32 bytes, X[i] =
 * instance i's n_x_i x 32 bytes.  One matrix-evaluation launch per instance and one synchronisation. */
int lurk_spartan_verify_batch(int n, lurk_spartan_ctx *const *ctxs, const uint8_t *u, const uint8_t *const *X, lurk_spartan_proof *proof,
                              int rounds_fmt, lurk_spartan_challenge_fn challenge, void *user, int *accepted, int fmt, void *stream);

/* The satisfiability checks of RecursiveSNARK::verify (Proof::verify on a Recursive proof, src/proof/nova.rs:358-373,
 * supernova.rs:304-317) in one call: R1CSShape::is_sat_relaxed on every running instance and is_sat on the secondary's last fresh
 * instance.  Per instance, one pass over the shape's rows forms A z, B z, C z in registers and counts the rows where
 * (A z)∘(B z) != u (C z) + E (no O(rows) scratch), then commit(W) and commit(E) are recomputed on the key and compared with comm_W and
 * comm_E.  One call covers one proof: Nova [r_U_primary, r_U_secondary, l_u_secondary]; SuperNova every Some running primary, then the
 * secondary's two instances.  n = 1..32.  Shapes and keys may repeat.
 *
 * The RO hashes (num_steps, z0, the two hashes compared with l_u_secondary.X) stay with the caller. */
typedef struct lurk_recursive_instance {
    lurk_spartan_ctx *shape;  /* full or verifier-only; borrowed                                                              */
    lurk_msm_ctx *ck;         /* key on the curve whose scalar field is the shape's field, >= max(n_w, n_rows) bases; not consumed */
    const void *z;            /* (W, u, X): n_w + 1 + n_x elements, laid out as LURK_FOLD_BUF_Z1 / LURK_FOLD_BUF_W2 hold it     */
    const void *E;            /* n_rows elements; NULL = strict instance (R1CSShape::is_sat: the u slot must hold 1)          */
    const uint8_t *comm_W;    /* 96 bytes, `fmt`, x | y | 1 or 0 | 0 | 0 for the identity                                     */
    const uint8_t *comm_E;    /* 96 bytes as comm_W; NULL exactly when E is NULL                                              */
} lurk_recursive_instance;
typedef struct lurk_recursive_verdict {
    uint64_t bad_rows;        /* rows where the R1CS equation fails                                                           */
    uint64_t first_bad_row;   /* the first of them; UINT64_MAX when every row holds                                           */
    int u_ok;                 /* strict: u == 1; relaxed: 1                                                                   */
    int comm_W_ok, comm_E_ok; /* the recomputed commitments equal the given ones; comm_E_ok = 1 for a strict instance          */
} lurk_recursive_verdict;
/* _dev: z and E are Montgomery elements on the device, as the fold contexts hold them (LURK_FOLD_BUF_Z1 / _E1 for a running instance,
 * LURK_FOLD_BUF_W2 for a staged fresh one); `fmt` applies to the commitments only.  The host form: z and E are host memory in `fmt`,
 * uploaded into stream-ordered scratch and converted there.  Neither form writes the caller's vectors.
 * *accepted = 1 when every verdict holds (bad_rows == 0, u_ok, comm_W_ok, comm_E_ok); a rejected proof is LURK_OK with *accepted = 0 and
 * every verdict filled in.  An element of z or E >= p, or a commitment off the curve, is LURK_ERR_RANGE; null pointers, n out of range,
 * E without comm_E or the reverse, a key that is too short, on another device or on the curve of another field are LURK_ERR_ARG.  Every
 * argument check runs before any device work.
 * Each distinct key context gets a stream forked from `stream` and joined before the call returns, so the primary's and the secondary's
 * instances run at once; on its stream each instance runs the R1CS pass, commit(W), then commit(E), through lurk_msm_ctx_launch_dev /
 * _finish on the borrowed key.  Synchronous.  The key contexts must have no launch pending and must not be used concurrently by the
 * caller during the call. */
int lurk_recursive_verify_dev(int n, const lurk_recursive_instance *inst, lurk_recursive_verdict *out, int *accepted, int fmt, void *stream);
int lurk_recursive_verify(int n, const lurk_recursive_instance *inst, lurk_recursive_verdict *out, int *accepted, int fmt, void *stream);

/* Compress context: CompressedSNARK::prove (Nova's `compress`, src/proof/nova.rs:341-356; SuperNova's, supernova.rs:293-317) in one call
 * -- for the primary and the secondary circuit, RelaxedR1CSSNARK::prove (or BatchedRelaxedR1CSSNARK::prove for SuperNova's primary),
 * batch_eval_reduce, the joint commitment sum_i weights_i C_i and the opening of the joint polynomial -- with the two circuits proved at
 * once, each on its own library-owned host thread and CUDA stream (Arecibo's rayon::join of S1::prove and S2::prove).
 *
 * Before the call, as in Arecibo's CompressedSNARK::prove, the secondary's last fresh instance is folded into its running instance
 * (NIFS::prove of l_u_secondary into r_U_secondary): one more lurk_fold_ctx_stage_a + lurk_fold_ctx_stage_b_launch + lurk_fold_ctx_collect
 * on the secondary's fold context with that instance in the buffer (its record carries comm_T).  The call then reads the running
 * instances straight from the fold contexts' LURK_FOLD_BUF_Z1 / LURK_FOLD_BUF_E1 buffers, and takes their commitments from the last
 * records (running_comm_W, running_comm_E).
 *
 * The context borrows the Spartan contexts (n_primary of them; 1 for Nova, 1..30 for SuperNova) and, per circuit, the evaluation engine:
 *   LURK_PCS_HYPERKZG  ck = a context on the KZG key (the primary of the BN256 / Grumpkin cycle);
 *   LURK_PCS_IPA       ck = a context on the Pedersen key, ck_c = the inner-product base, 64 bytes affine, unscaled.
 * It clones each key context (the clones never share MSM scratch with a fold context on the same key; the borrowed contexts must outlive
 * the compress context), allocates on its first proof one scratch arena per circuit -- fold chain, witness polynomials, evaluation
 * partials, MSM clones, side streams -- sized for that circuit's joint polynomial, and keeps everything until destroy.  Every size, field
 * and curve is checked before any device work: each key holds >= joint_len bases, the secondary's field is the primary's cycle partner,
 * each key's scalar field is its circuit's field, and no Spartan context is passed twice. */
#define LURK_PCS_HYPERKZG 0
#define LURK_PCS_IPA 1
typedef struct lurk_compress_pcs {
    int kind;              /* LURK_PCS_* */
    lurk_msm_ctx *ck;      /* borrowed; curve = the one whose scalar field is the circuit's field */
    const uint8_t *ck_c;   /* IPA: 64 bytes affine in the create call's `fmt` (copied); HyperKZG: NULL */
} lurk_compress_pcs;
typedef struct lurk_compress_ctx lurk_compress_ctx;
int lurk_compress_ctx_create(int n_primary, lurk_spartan_ctx *const *primary, lurk_spartan_ctx *secondary, const lurk_compress_pcs *pcs_primary,
                             const lurk_compress_pcs *pcs_secondary, int fmt, lurk_compress_ctx **out);
void lurk_compress_ctx_destroy(lurk_compress_ctx *ctx);
/* device bytes the context holds (its arenas; 0 before the first proof) and the joint-polynomial lengths; any output may be NULL */
int lurk_compress_ctx_info(lurk_compress_ctx *ctx, size_t *device_bytes, size_t *joint_len_primary, size_t *joint_len_secondary);
/* The transcript: circuit 0 = primary, 1 = secondary; phase and round as lurk_spartan_challenge_fn, plus the opening's phase
 * LURK_SPARTAN_PCS:
 *   HyperKZG  rounds 0, 1, 2: the messages lurk_hyperkzg_prove_dev passes (com; v; w -- the last challenge is ignored)
 *   IPA       round 0: comm | joint_eval (96 + 32 bytes) -> r, the scale of ck_c (InnerProductInstance absorbs comm and c, not b);
 *             rounds 1 .. m: L | R of the inner-product argument's rounds 0 .. m - 1
 * For one circuit the callback is called in protocol order and never concurrently with itself; the two circuits' calls may be concurrent
 * (with LURK_COMPRESS_SEQUENTIAL they are not).  The caller absorbs each circuit's verifier-key digest and instance U into that circuit's
 * transcript before the call, as the Spartan context requires.  Returns 0, or non-zero to abort the proof. */
#define LURK_SPARTAN_PCS 6
typedef int (*lurk_compress_challenge_fn)(void *user, int circuit, int phase, int round, const uint8_t *message, size_t message_len,
                                          uint8_t challenge_out[32]);
/* One circuit's proof, every buffer caller-owned and optional (NULL = not wanted), `fmt`.  m = log2 of the circuit's joint_len. */
typedef struct lurk_compress_circuit_proof {
    lurk_spartan_proof snark;  /* as lurk_spartan_prove_dev / _batch_dev write it */
    uint8_t *comm;             /* 96: the joint commitment sum_i weights_i C_i over [comm_W_0 .., comm_E_0 ..] */
    uint8_t *com;              /* HyperKZG: (m - 1) x 96 */
    uint8_t *w;                /* HyperKZG: 3 x 96 */
    uint8_t *v;                /* HyperKZG: 3 x m x 32 */
    uint8_t *L, *R;            /* IPA: m x 96 each */
    uint8_t *a_final, *b_final;   /* IPA: 32 each */
} lurk_compress_circuit_proof;
typedef struct lurk_compress_proof {
    lurk_compress_circuit_proof primary, secondary;
} lurk_compress_proof;
#define LURK_COMPRESS_SEQUENTIAL 1  /* the secondary proof after the primary one, on the same host thread */
#define LURK_COMPRESS_BATCHED 2     /* the primary is BatchedRelaxedR1CSSNARK (SuperNova), also with n_primary = 1 */
/* d_z[i] / d_E[i]: primary instance i on the device, laid out as LURK_FOLD_BUF_Z1 / LURK_FOLD_BUF_E1 hold it (read, never written);
 * comm_W[i] / comm_E[i]: its commitments (96 bytes, `fmt`); d_z2, d_E2, comm_W2, comm_E2: the secondary's.  n_primary must be the
 * number of primary contexts.  The primary proof runs on `stream`, the secondary on the context's worker stream (after the work queued
 * on `stream` so far); both host threads are joined before the call returns, errors included: the call returns when done.  A failed
 * callback or any other error returns its code with a message naming the circuit; the context stays usable.  One call at a time per
 * context. */
int lurk_compress_prove_dev(lurk_compress_ctx *ctx, int n_primary, const void *const *d_z, const void *const *d_E, const uint8_t *const *comm_W,
                            const uint8_t *const *comm_E, const void *d_z2, const void *d_E2, const uint8_t comm_W2[96], const uint8_t comm_E2[96],
                            lurk_compress_challenge_fn challenge, void *user, int flags, lurk_compress_proof *out, int fmt, void *stream);

/* Compressed verifier: CompressedSNARK::verify (Nova's Proof::verify on a compressed proof, src/proof/nova.rs:358-373; SuperNova's,
 * supernova.rs:304-317) in one call, for the proof lurk_compress_prove_dev writes.  Per circuit, in order:
 *   1. RelaxedR1CSSNARK::verify (BatchedRelaxedR1CSSNARK::verify with LURK_COMPRESS_BATCHED) up to the opening, as lurk_spartan_verify /
 *      _batch run it (sum-checks, claims, batch_eval_reduce's verifier);
 *   2. the joint commitment sum_i weights_i C_i over [comm_W_0 .., comm_E_0 ..] on the host;
 *   3. the opening of the joint polynomial at r with value joint_eval:
 *      IPA       round 0 comm | joint_eval -> the scale of ck_c; eq(r) in stream-ordered scratch; InnerProductArgument::verify as
 *                lurk_ipa_verify_dev runs it, its rounds numbered 1 .. m;
 *      HyperKZG  round 0 com -> r; the fold consistency 2 r Y[i+1] = r (1 - x) (v0[i] + v1[i]) + x (v0[i] - v1[i]), x = point[m - 1 - i],
 *                Y = v[2] | joint_eval; round 1 v -> q; round 2 w -> d; then, with B = sum_j q^j com_j (com_0 = the joint commitment),
 *                u = (r, -r, r^2) and B(u_t) = sum_j q^j v[t][j], the two G1 points
 *                    P = sum_t d^t (B - B(u_t) G + u_t w_t),   Q = sum_t d^t w_t
 *                and the caller's pairing check e(P, H) == e(Q, beta H).  Under a key of known beta it holds exactly when P == beta Q.
 * The pairing stays with the caller, as the transcript does: `pairing` gets the circuit and P, Q (96 bytes each, `fmt`, the header's form),
 * writes *holds (0 or 1) and returns 0, or non-zero to abort.
 *
 * Not here, as in lurk_compress_prove_dev: the secondary's NIFS::verify, which folds l_u_secondary into r_U_secondary with the RO challenge.
 * u2, X2, comm_W2 and comm_E2 are f_U_secondary's, already folded by the caller; the RO hashes, the transcript, serde and the pairing too.
 *
 * The transcript is lurk_compress_challenge_fn with the calls of lurk_compress_prove_dev, in the same order, with the same messages: one
 * transcript object serves prover and verifier.  HyperKZG's round 2 returns the verifier's d (the prover ignores it).  For one circuit the
 * callbacks (transcript and pairing) come in protocol order and never concurrently with themselves; the two circuits' may run at once.
 *
 * The primary runs on the calling thread and `stream`, the secondary on a library-owned thread and a stream forked from `stream`; both are
 * joined before the call returns, errors included.  LURK_COMPRESS_SEQUENTIAL runs the secondary after the primary, on the calling thread and
 * `stream`.  Synchronous.
 *
 * Contexts: primary (n_primary, distinct) and secondary Spartan contexts, full or verifier-only, give the same results.  The IPA key contexts
 * are borrowed: they must have no launch pending and must not be used by the caller during the call (as lurk_recursive_verify).
 *
 * Inputs, `fmt`: u (n_primary x 32), X[i] (n_x_i x 32), comm_W[i] / comm_E[i] (96) of the primary instances; u2, X2, comm_W2, comm_E2 of the
 * secondary's.  proof: read are snark.outer_rounds, claims, inner_rounds, eval_W, reduce_rounds, claims_left (round polynomials in
 * `rounds_fmt`, LURK_SPARTAN_ROUNDS_*), and com, v, w (HyperKZG) or L, R, a_final (IPA); comm, b_final and the snark's derived fields are
 * neither read nor written.
 *
 * Result: out[0] primary, out[1] secondary.  snark_ok: step 1; eval_ok: HyperKZG's fold consistency, 1 for IPA; opening_ok: the pairing
 * callback's answer, or IPA's closing check.  1 = holds, 0 = fails, -1 = not reached: the first failing check ends that circuit, and the other
 * circuit is unaffected.  *accepted = 1 when all six hold.  A rejected proof is LURK_OK with *accepted = 0.
 * Errors, all raised before the first callback and before any device work: values >= p and points off the curve (u, X, the commitments, every
 * proof field read, g, ck_c) are LURK_ERR_RANGE; null pointers, n_primary out of range or not matching the contexts, mixed fields, a
 * secondary field that is not the cycle partner, a key that is too short, on the wrong curve, on another device or with a launch pending, a
 * context passed twice, HyperKZG without `pairing` are LURK_ERR_ARG.  A failing transcript or pairing callback is LURK_ERR_ARG with a message
 * naming the circuit, never a rejection.  After an error the verdicts read -1 where not reached. */
typedef struct lurk_compress_vk_pcs {
    int kind;              /* LURK_PCS_HYPERKZG | LURK_PCS_IPA                                                              */
    lurk_msm_ctx *ck;      /* IPA: the Pedersen key, >= joint_len bases, not consumed;  HyperKZG: NULL                      */
    const uint8_t *ck_c;   /* IPA: 64 bytes affine, unscaled, `fmt`;  HyperKZG: NULL                                        */
    const uint8_t *g;      /* HyperKZG: the verifier key's G1 point G (the key's first base), 64 bytes affine, `fmt`;  IPA: NULL */
} lurk_compress_vk_pcs;
/* e(P, H) == e(Q, beta H) under the caller's verifier key?  Writes *holds (0 / 1) and returns 0, or non-zero to abort. */
typedef int (*lurk_pairing_check_fn)(void *user, int circuit, const uint8_t P[96], const uint8_t Q[96], int *holds);
typedef struct lurk_compress_verdict {
    int snark_ok;     /* RelaxedR1CSSNARK / BatchedRelaxedR1CSSNARK::verify up to the opening                 */
    int eval_ok;      /* HyperKZG: the fold consistency of v;  IPA: 1;                  -1 = not reached      */
    int opening_ok;   /* HyperKZG: the pairing callback's answer;  IPA: the closing check;  -1 = not reached  */
} lurk_compress_verdict;
int lurk_compress_verify(int n_primary, lurk_spartan_ctx *const *primary, lurk_spartan_ctx *secondary, const lurk_compress_vk_pcs *pcs_primary,
                         const lurk_compress_vk_pcs *pcs_secondary, const uint8_t *u, const uint8_t *const *X, const uint8_t *const *comm_W,
                         const uint8_t *const *comm_E, const uint8_t u2[32], const uint8_t *X2, const uint8_t comm_W2[96], const uint8_t comm_E2[96],
                         const lurk_compress_proof *proof, int rounds_fmt, lurk_compress_challenge_fn challenge, lurk_pairing_check_fn pairing,
                         void *user, int flags, lurk_compress_verdict out[2], int *accepted, int fmt, void *stream);
/* sum_k scalars[k] points[k] on the host (Straus, split over host threads): the point arithmetic of the compressed verifier -- the joint
 * commitment, HyperKZG's P and Q -- for callers that compose the verifier themselves.  points: count x 96 bytes of the header's form, scalars:
 * count x 32 bytes, out: 96 bytes, all `fmt`.  Host only; works without a GPU. */
int lurk_point_combination(int curve_id, const uint8_t *points_xyz, const uint8_t *scalars, size_t count, int fmt, uint8_t out_xyz[96]);
/* n_groups independent combinations on the GPU, in order on `stream`; returns when they are done.
 * Group g has counts[g] >= 1 terms. Its terms come after the terms of groups 0..g-1 in points_xyz
 * (total x 96 bytes, host, in the header's form) and scalars (total x 32, fmt).
 * out_xyz: n_groups x 96 bytes, the same bytes lurk_point_combination writes for that group.
 * One CTA per group: Straus with 4-bit windows, the tables and window sums spread over its threads, the 252 doublings on one thread.
 * At most LURK_POINT_COMBINATION_MAX_TERMS terms per group (past it, commit through an lurk_msm_ctx instead).  n_groups < 1, a count
 * of 0 or over the limit, null pointers, an unknown curve or format are LURK_ERR_ARG; then LURK_ERR_NOGPU without a device; then a
 * point off the curve or not of the header's form, or a scalar >= r, is LURK_ERR_RANGE with lurk_point_combination's message and the
 * group's index -- all before anything is launched.  Keeps no state between calls: host threads may call it at once on their streams. */
#define LURK_POINT_COMBINATION_MAX_TERMS 4096
int lurk_point_combination_batch(int curve_id, int n_groups, const uint32_t *counts, const uint8_t *points_xyz, const uint8_t *scalars, int fmt,
                                 uint8_t *out_xyz, void *stream);

/* ---------------------------------------------------------------------------------------------------
 * S5  Fold helpers on device-resident vectors (Arecibo NIFS::prove / R1CSShape::commit_T /
 *     RelaxedR1CSWitness::fold; SURVEY.md Appendix B).  All vectors Montgomery form on the device.
 * ------------------------------------------------------------------------------------------------- */
/* All four asynchronous.
 * out[i] = a[i] + r * b[i]  (W <- W1 + r W2, E <- E1 + r T).  r: 32 bytes host, Montgomery. out may alias a. */
int lurk_axpy_dev(int field_id, const void *d_a, const void *d_b, const uint8_t r_mont[32], size_t n, void *d_out,
                  void *stream);
/* y = M z for a CSR matrix (row_ptr: rows+1 x u64, col: nnz x u32, val: nnz elements) */
int lurk_spmv_csr_dev(int field_id, const void *d_row_ptr, const void *d_col, const void *d_val, size_t rows,
                      const void *d_z, void *d_y, void *stream);
/* T = az1*bz2 + az2*bz1 - u1*cz2 - u2*cz1 */
int lurk_cross_term_dev(int field_id, const void *d_az1, const void *d_bz1, const void *d_cz1, const void *d_az2,
                        const void *d_bz2, const void *d_cz2, const uint8_t u1_mont[32], const uint8_t u2_mont[32],
                        size_t n, void *d_t, void *stream);
/* element-wise format conversion on the device (LURK_FMT_*), in place allowed */
int lurk_convert_dev(int field_id, const void *d_in, size_t n, int to_fmt, void *d_out, void *stream);

/* ---------------------------------------------------------------------------------------------------
 * S5/S6  Fold context: the GPU half of `Proof::prove_recursively` (src/proof/nova.rs:260-339, supernova.rs:207-291) for
 *     ONE running instance, i.e. what RecursiveSNARK::new / prove_step (nova.rs:286-293) do with the primary circuit's
 *     witness inside Arecibo's NIFS::prove (SURVEY.md Appendix B), on device-resident state:
 *         comm_W2 = commit(W2); T = cross term; comm_T = commit(T); r = RO(..., comm_W2, ..., comm_T);
 *         (W, u, X) += r (W2, 1, X2); E += r T; comm_W += r comm_W2; comm_E += r comm_T.
 *     The reference overlaps a witness thread with the fold thread over a bounded channel (nova.rs:297-326); here stage A
 *     (inputs, slot witnesses, commit(W2), A z2 .. C z2) of up to `depth - 1` later steps runs on its own CUDA streams while
 *     stage B -- the sequential chain -- runs without any host round trip: the commitments are finished, exchanged between
 *     GPUs (peer memory over NVLink), normalised, hashed into the challenge and consumed by the fold on the device.
 *     SuperNova / NIVC: one context per circuit index (src/lem/multiframe.rs:941), all sharing one commitment key.
 *     z = (W, u, X).  Matrices are CSR over z's columns.  All calls of one context must come from one thread at a time.
 * ------------------------------------------------------------------------------------------------- */
typedef struct lurk_fold_ctx lurk_fold_ctx;
typedef struct lurk_fold_config {
    int curve_id;            /* commitments on this curve; the witness field is its scalar field */
    int depth;               /* fresh-instance buffers, 1..4: stage A may run depth - 1 steps ahead of the fold */
    uint64_t n_w;            /* |W| of this rank's share */
    uint64_t n_x;            /* |X| (2 for Nova step circuits) */
    uint64_t n_rows;         /* constraints of this rank's share */
    const uint64_t *row_ptr[3]; /* A, B, C: rows + 1 offsets                                    (host) */
    const uint32_t *col[3];     /* column of every non-zero, < n_w + 1 + n_x                     (host) */
    const uint8_t *val[3];      /* coefficient of every non-zero, 32 bytes each, in `fmt`        (host) */
    int fmt;
    int world, rank;         /* > 1: the key is sharded; the partial commitments are exchanged every step */
    int latency_sms;         /* 0 = off; otherwise SMs reserved for the latency-shaped kernels of the chain (green
                                contexts; multiple of 8, e.g. 16): bucket accumulation and stage A get the rest */
} lurk_fold_config;
/* ck_w / ck_t: this rank's bases for W (>= n_w points) and for T / E (>= n_rows points); the same context when the key is
 * not sharded.  Fixed-base tables are built if absent.  The contexts must outlive the fold context. */
int lurk_fold_ctx_create(const lurk_fold_config *cfg, lurk_msm_ctx *ck_w, lurk_msm_ctx *ck_t, lurk_fold_ctx **out);
void lurk_fold_ctx_destroy(lurk_fold_ctx *ctx);
/* One batch per slot type of the step circuit (generate_slots_witnesses, src/lem/multiframe.rs:520-592): arity 3/4/6/8 =
 * Poseidon slots, 0 = bit-decomposition slots.  offsets[k] = element offset of block k inside W (the reference's layout:
 * every frame's aux = [its slot blocks | LEM body aux], multiframe.rs:635-712).  Returns the batch index (>= 0). */
int lurk_fold_ctx_add_slot_batch(lurk_fold_ctx *ctx, int arity, size_t count, const uint64_t *offsets);
/* One batch of `count` SHA-256 coprocessor calls with n pointers each: stage A writes their witness blocks
 * (lurk_sha256_witness_block elements) into W at element offsets offsets[k].  Its host buffer holds count * 2n inputs
 * (per pointer tag, then hash).  Returns the batch index (>= 0), an index of the same host buffers as the slot batches. */
int lurk_fold_ctx_add_sha256_batch(lurk_fold_ctx *ctx, int n, size_t count, const uint64_t *offsets);
/* One batch of `count` trie coprocessor calls (op LURK_TRIE_LOOKUP / LURK_TRIE_INSERT, height H): stage A writes their
 * witness blocks (lurk_trie_witness_block elements) into W at element offsets offsets[k].  Its host buffer holds the
 * calls' inputs (lurk_trie_witness_batch's layout).  Stage A trusts them as it trusts slot preimages: paths are not
 * checked.  Returns the batch index (>= 0), an index of the same host buffers as the slot batches. */
int lurk_fold_ctx_add_trie_batch(lurk_fold_ctx *ctx, int op, int height, size_t count, const uint64_t *offsets);
/* The parts of W2 the host produces (LEM body aux, the augmented-circuit part): up to 4 strided spans of W; the host
 * buffer LURK_FOLD_BUF_GLUE holds them densely, span after span, row after row. */
typedef struct lurk_fold_span { uint64_t first, row_elems, stride, rows; } lurk_fold_span;
int lurk_fold_ctx_set_spans(lurk_fold_ctx *ctx, int n_spans, const lurk_fold_span *spans);
/* Random oracle = Arecibo's PoseidonRO (neptune sponge, arity 24, [Absorb(n), Squeeze(1)], low `challenge_bits` bits).
 * kinds[i] says what is absorbed at position i.  Default (NIFS::prove): CONST pp_digest, W_X, W_Y, W_INF, CONST X2[0],
 * CONST X2[1], T_X, T_Y, T_INF with 128 bits.  CONST values come from the host buffer LURK_FOLD_BUF_RO of the step. */
#define LURK_FOLD_RO_CONST 0
#define LURK_FOLD_RO_W_X 1
#define LURK_FOLD_RO_W_Y 2
#define LURK_FOLD_RO_W_INF 3
#define LURK_FOLD_RO_T_X 4
#define LURK_FOLD_RO_T_Y 5
#define LURK_FOLD_RO_T_INF 6
int lurk_fold_ctx_set_ro(lurk_fold_ctx *ctx, int n_absorb, const int *kinds, int challenge_bits);
/* Pinned host buffers the caller (the CPU witness generator) fills before stage A of buffer b: `which` >= 0 = preimages
 * of that slot batch (count * arity elements; bit decomposition: count values; SHA-256: count * 2n inputs; trie: count
 * calls' inputs), or one of the names below. */
#define LURK_FOLD_BUF_GLUE (-1) /* the spans, densely                       (witness field)            */
#define LURK_FOLD_BUF_X2 (-2)   /* public IO of the fresh instance, n_x      (witness field)            */
#define LURK_FOLD_BUF_RO (-3)   /* 24 elements: position i = CONST value of RO slot i (commitment curve's base field) */
#define LURK_FOLD_BUF_W2 (-4)   /* device only: z2 of buffer b = (W2, 1, X2), Montgomery               */
#define LURK_FOLD_BUF_T (-5)    /* device only: cross term of the last step                             */
#define LURK_FOLD_BUF_Z1 (-6)   /* device only: running z = (W, u, X)                                   */
#define LURK_FOLD_BUF_E1 (-7)   /* device only: running E                                               */
/* When the device buffers may be read or written.  The context runs on non-blocking streams of its own and takes no stream, so a
 * caller's stream is ordered against it only through these calls:
 *   LURK_FOLD_BUF_Z1, _E1  after lurk_fold_ctx_collect of the step that last changed them (init_running or a fold): collect returns
 *                          once the fold has written them, so lurk_spartan_prove_dev, lurk_compress_prove_dev or
 *                          lurk_recursive_verify_dev may read them on any stream straight after it.
 *   LURK_FOLD_BUF_T        after lurk_fold_ctx_collect of the stage B that computed it.
 *   LURK_FOLD_BUF_W2       after a stage A of buffer b, only after lurk_fold_ctx_sync (collect does not cover a stage A that no
 *                          collected step consumed).
 *   Writes for LURK_FOLD_INPUTS_RESIDENT  must be complete, not merely queued on the caller's stream, before lurk_fold_ctx_stage_a
 *                          (e.g. cudaStreamSynchronize of that stream), and made after the previous step of buffer b was collected. */
int lurk_fold_ctx_host_buffer(lurk_fold_ctx *ctx, int b, int which, void **ptr, size_t *bytes);
int lurk_fold_ctx_device_buffer(lurk_fold_ctx *ctx, int b, int which, void **d_ptr, size_t *bytes);
/* Sharded key, one process per GPU: every rank publishes a 64-byte handle of its exchange buffer (any transport: e.g. a
 * torch.distributed all_gather of the bytes) and receives all `world` handles, ordered by rank. */
int lurk_fold_ctx_exchange_handle(lurk_fold_ctx *ctx, uint8_t handle[64]);
int lurk_fold_ctx_set_peers(lurk_fold_ctx *ctx, const uint8_t *handles /* world * 64 bytes */);
/* Running instance (checkpoint / resume: prove_recursively's `init: Option<RecursiveSNARK>`, src/proof/mod.rs:107-115).
 * comm_* are 96-byte points x | y | z as everywhere in this header; any output pointer of _get_ may be NULL. */
int lurk_fold_ctx_set_running(lurk_fold_ctx *ctx, const uint8_t *W, const uint8_t *E, const uint8_t u[32], const uint8_t *X,
                              const uint8_t comm_W[96], const uint8_t comm_E[96], int fmt);
int lurk_fold_ctx_get_running(lurk_fold_ctx *ctx, uint8_t *W, uint8_t *E, uint8_t u[32], uint8_t *X, uint8_t comm_W[96],
                              uint8_t comm_E[96], int fmt);
/* Stage A of the step whose inputs are in the host buffers of b (fmt = their format).  LURK_FOLD_INPUTS_RESIDENT: skip
 * the host-to-device copies and use what the device buffers hold (Montgomery). Asynchronous. */
#define LURK_FOLD_INPUTS_RESIDENT 1
int lurk_fold_ctx_stage_a(lurk_fold_ctx *ctx, int b, int flags, int fmt);
/* RecursiveSNARK::new: the running instance becomes the fresh instance of buffer b (u = 1, E = 0, comm_E = identity). */
int lurk_fold_ctx_init_running(lurk_fold_ctx *ctx, int b);
/* Stage B: enqueues the whole fold of the fresh instance in buffer b onto the running instance.  Asynchronous; call
 * stage_a for later steps and stage_b_launch for the next step without waiting. */
int lurk_fold_ctx_stage_b_launch(lurk_fold_ctx *ctx, int b);
typedef struct lurk_fold_result {
    uint8_t comm_W[96];         /* commitment to the fresh witness (whole key) */
    uint8_t comm_T[96];         /* commitment to the cross term; identity after init_running */
    uint8_t r[32];              /* the challenge as an element of the witness field */
    uint8_t running_comm_W[96]; /* after this step's fold */
    uint8_t running_comm_E[96];
    uint8_t ro_hash[32];        /* the squeezed sponge element before truncation (commitment curve's base field) */
    int status;
    uint64_t seq;               /* exchange epoch = number of commitments finished by this context */
} lurk_fold_result;
/* waits for the step enqueued on buffer b (init_running or stage_b_launch), its fold of Z1 and E1 included, and returns its record */
int lurk_fold_ctx_collect(lurk_fold_ctx *ctx, int b, lurk_fold_result *out, int fmt);
/* Verifier-side sanity of the running instance, computed on the device: rows with (A z) o (B z) != u (C z) + E, and
 * whether commit(W) / commit(E) recomputed from the vectors equal the folded commitments.  Synchronous. */
int lurk_fold_ctx_check_running(lurk_fold_ctx *ctx, uint64_t *bad_rows, int *comm_W_ok, int *comm_E_ok);
/* kernels enqueued by the last stage A / stage B, device time of the bucket-accumulation kernels of the last commit(W2) of
 * buffer 0 and of the last commit(T) (CUDA events on the launching streams).  Synchronises the context. */
int lurk_fold_ctx_stats(lurk_fold_ctx *ctx, unsigned *launches_a, unsigned *launches_b, float *accumulate_w_ms, float *accumulate_t_ms);
int lurk_fold_ctx_sync(lurk_fold_ctx *ctx);

/* ---------------------------------------------------------------------------------------------------
 * K6  Number-theoretic transform (north_star; no call site in the reference -- SURVEY.md D4).
 *     In-place length-2^log_n DFT over the field's 2-adic subgroup, natural order in and out, Montgomery form.
 *     Roots: omega = g^((p-1)/2^s) with g the multiplicative generator of halo2curves / pasta_curves.
 * ------------------------------------------------------------------------------------------------- */
/* Asynchronous (the first transform of a size and direction on a device waits while it builds that size's twiddles). */
int lurk_ntt_dev(int field_id, void *d_data, int log_n, int inverse, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* LURK_B200_H */
