//! Rust binding of liblurk_b200 (C ABI: include/lurk_b200.h).  Hand-written `extern "C"` block + thin safe wrappers, the
//! counterpart of what `pasta-msm` / `grumpkin-msm` are for sppark (SURVEY.md D5).  NOT compiled in the lurk-beta_b200
//! repository (no Rust toolchain in its build image): it is the file a maintainer drops into lurk-beta / Arecibo, next to
//! `build.rs`.  Seams (reference file:line) each wrapper serves are named on the wrapper.
#![allow(non_camel_case_types, dead_code)]
use std::ffi::CStr;
use std::os::raw::{c_char, c_int, c_uint, c_void};

pub const LURK_FIELD_BN254_FR: c_int = 0;
pub const LURK_FIELD_BN254_FQ: c_int = 1;
pub const LURK_FIELD_PALLAS_FQ: c_int = 2;
pub const LURK_FIELD_PALLAS_FP: c_int = 3;
pub const LURK_CURVE_BN254_G1: c_int = 0;
pub const LURK_CURVE_GRUMPKIN: c_int = 1;
pub const LURK_CURVE_PALLAS: c_int = 2;
pub const LURK_CURVE_VESTA: c_int = 3;
pub const LURK_FMT_CANONICAL: c_int = 0;
pub const LURK_FMT_MONTGOMERY: c_int = 1;
pub const LURK_TRIE_LOOKUP: c_int = 0;
pub const LURK_TRIE_INSERT: c_int = 1;
pub const LURK_TRIE_MAX_HEIGHT: c_int = 85;
pub const LURK_FOLD_BUF_GLUE: c_int = -1;
pub const LURK_FOLD_BUF_X2: c_int = -2;
pub const LURK_FOLD_BUF_RO: c_int = -3;

#[repr(C)]
pub struct lurk_msm_ctx { _private: [u8; 0] }
#[repr(C)]
pub struct lurk_fold_ctx { _private: [u8; 0] }
#[repr(C)]
pub struct lurk_spartan_ctx { _private: [u8; 0] }
/// caller-owned host buffers of one proof (include/lurk_b200.h: lurk_spartan_proof); null = not wanted
#[repr(C)]
pub struct lurk_spartan_proof {
    pub outer_rounds: *mut u8, pub r_x: *mut u8, pub claims: *mut u8, pub inner_rounds: *mut u8, pub r_y: *mut u8, pub eval_w: *mut u8,
    pub reduce_rounds: *mut u8, pub r: *mut u8, pub claims_left: *mut u8, pub weights: *mut u8, pub joint_eval: *mut u8,
}
pub const LURK_SPARTAN_TAU: c_int = 0;
pub const LURK_SPARTAN_OUTER_R: c_int = 1;
pub const LURK_SPARTAN_OUTER: c_int = 2;
pub const LURK_SPARTAN_CLAIMS: c_int = 3;
pub const LURK_SPARTAN_INNER: c_int = 4;
pub const LURK_SPARTAN_BATCH_EVAL: c_int = 5;
pub const LURK_SPARTAN_PCS: c_int = 6;
#[repr(C)]
pub struct lurk_compress_ctx { _private: [u8; 0] }
#[repr(C)]
pub struct lurk_trie_ctx { _private: [u8; 0] }
pub const LURK_PCS_HYPERKZG: c_int = 0;
pub const LURK_PCS_IPA: c_int = 1;
pub const LURK_COMPRESS_SEQUENTIAL: c_int = 1;
pub const LURK_COMPRESS_BATCHED: c_int = 2;
/// one circuit's evaluation engine (include/lurk_b200.h: lurk_compress_pcs); ck_c: IPA's 64-byte affine base, null for HyperKZG
#[repr(C)]
pub struct lurk_compress_pcs { pub kind: c_int, pub ck: *mut lurk_msm_ctx, pub ck_c: *const u8 }
/// one circuit's CompressedSNARK half: the Spartan proof, the joint commitment and the opening (HyperKZG: com, w, v; IPA: L, R, a/b_final)
#[repr(C)]
pub struct lurk_compress_circuit_proof {
    pub snark: lurk_spartan_proof, pub comm: *mut u8, pub com: *mut u8, pub w: *mut u8, pub v: *mut u8, pub l: *mut u8, pub r: *mut u8,
    pub a_final: *mut u8, pub b_final: *mut u8,
}
#[repr(C)]
pub struct lurk_compress_proof { pub primary: lurk_compress_circuit_proof, pub secondary: lurk_compress_circuit_proof }
/// `int (*)(void *user, int circuit, int phase, int round, const uint8_t *message, size_t message_len, uint8_t challenge_out[32])`: circuit 0 =
/// primary, 1 = secondary; the two circuits' calls may come from two threads at once (one transcript per circuit).
pub type lurk_compress_challenge_fn = unsafe extern "C" fn(user: *mut c_void, circuit: c_int, phase: c_int, round: c_int, message: *const u8,
                                                           message_len: usize, challenge_out: *mut u8) -> c_int;
/// the compressed verifier's evaluation engine (include/lurk_b200.h: lurk_compress_vk_pcs): IPA ck + ck_c (unscaled), HyperKZG g (the key's G1
/// base); the other pointers null
#[repr(C)]
pub struct lurk_compress_vk_pcs { pub kind: c_int, pub ck: *mut lurk_msm_ctx, pub ck_c: *const u8, pub g: *const u8 }
/// `int (*)(void *user, int circuit, const uint8_t P[96], const uint8_t Q[96], int *holds)`: e(P, H) == e(Q, beta H) under the verifier key
pub type lurk_pairing_check_fn = unsafe extern "C" fn(user: *mut c_void, circuit: c_int, p: *const u8, q: *const u8, holds: *mut c_int) -> c_int;
/// one circuit's verdict: 1 holds, 0 fails, -1 not reached
#[repr(C)]
#[derive(Clone, Copy, Debug, Default, PartialEq, Eq)]
pub struct lurk_compress_verdict { pub snark_ok: c_int, pub eval_ok: c_int, pub opening_ok: c_int }
/// one instance of RecursiveSNARK::verify's is_sat checks (include/lurk_b200.h: lurk_recursive_instance); e / comm_e null for a strict
/// instance (l_u_secondary)
#[repr(C)]
pub struct lurk_recursive_instance {
    pub shape: *mut lurk_spartan_ctx, pub ck: *mut lurk_msm_ctx, pub z: *const c_void, pub e: *const c_void, pub comm_w: *const u8,
    pub comm_e: *const u8,
}
/// what one instance's checks found: first_bad_row = u64::MAX when every row holds
#[repr(C)]
#[derive(Clone, Copy, Default)]
pub struct lurk_recursive_verdict { pub bad_rows: u64, pub first_bad_row: u64, pub u_ok: c_int, pub comm_w_ok: c_int, pub comm_e_ok: c_int }
#[repr(C)]
#[derive(Clone, Copy)]
pub struct lurk_dag_node { pub kind: u8, pub reserved: u8, pub tag: [u16; 4], pub child: [u32; 4] }
#[repr(C)]
pub struct lurk_fold_config {
    pub curve_id: c_int, pub depth: c_int, pub n_w: u64, pub n_x: u64, pub n_rows: u64,
    pub row_ptr: [*const u64; 3], pub col: [*const u32; 3], pub val: [*const u8; 3],
    pub fmt: c_int, pub world: c_int, pub rank: c_int, pub latency_sms: c_int,
}
#[repr(C)]
#[derive(Clone, Copy)]
pub struct lurk_fold_span { pub first: u64, pub row_elems: u64, pub stride: u64, pub rows: u64 }
#[repr(C)]
pub struct lurk_fold_result {
    pub comm_w: [u8; 96], pub comm_t: [u8; 96], pub r: [u8; 32], pub running_comm_w: [u8; 96], pub running_comm_e: [u8; 96],
    pub ro_hash: [u8; 32], pub status: c_int, pub seq: u64,
}

extern "C" {
    pub fn lurk_last_error() -> *const c_char;
    pub fn lurk_device_count() -> c_int;
    // S1 -- PoseidonCache::hash3/4/6/8 (src/hash.rs:180-203)
    pub fn lurk_poseidon_hash_batch(field_id: c_int, arity: c_int, preimages: *const u8, n: usize, digests: *mut u8) -> c_int;
    pub fn lurk_poseidon_hash_batch_mont(field_id: c_int, arity: c_int, preimages: *const u8, n: usize, digests: *mut u8) -> c_int;
    // S3 -- generate_slots_witnesses (src/lem/multiframe.rs:520-592)
    pub fn lurk_poseidon_witness_block(field_id: c_int, arity: c_int) -> usize;
    pub fn lurk_poseidon_witness_batch(field_id: c_int, arity: c_int, preimages: *const u8, n: usize, blocks: *mut u8, fmt: c_int) -> c_int;
    pub fn lurk_bitdecomp_witness_block(field_id: c_int) -> usize;
    pub fn lurk_bitdecomp_witness_batch(field_id: c_int, values: *const u8, n: usize, blocks: *mut u8, fmt: c_int) -> c_int;
    // a12 -- synthesize_lookup_aux / synthesize_insert_aux (src/coprocessor/trie/mod.rs:118-156, 226-268)
    pub fn lurk_trie_witness_block(field_id: c_int, op: c_int, height: c_int) -> usize;
    pub fn lurk_trie_witness_batch(field_id: c_int, op: c_int, height: c_int, inputs: *const u8, count: usize, aux_out: *mut u8, fmt: c_int) -> c_int;
    pub fn lurk_trie_witness_batch_dev(field_id: c_int, op: c_int, height: c_int, d_inputs: *const c_void, count: usize, d_aux: *mut c_void, fmt: c_int,
                                       stream: *mut c_void) -> c_int;
    pub fn lurk_trie_witness_scatter_dev(field_id: c_int, op: c_int, height: c_int, d_inputs: *const c_void, count: usize, d_offsets: *const u64,
                                         d_w: *mut c_void, fmt: c_int, stream: *mut c_void) -> c_int;
    // a12 -- the trie's own operations (Trie::prove_lookup / prove_insert over the inverse Poseidon cache, mod.rs:718-811) on a
    // device node store; the replay of a proved evaluation's trie calls hands (op, root, key, value) instead of packed proofs
    pub fn lurk_trie_ctx_create(field_id: c_int, height: c_int, capacity_nodes: u64, out: *mut *mut lurk_trie_ctx) -> c_int;
    pub fn lurk_trie_ctx_destroy(ctx: *mut lurk_trie_ctx);
    pub fn lurk_trie_ctx_empty_root(ctx: *mut lurk_trie_ctx, out: *mut u8, fmt: c_int) -> c_int;
    pub fn lurk_trie_ctx_info(ctx: *const lurk_trie_ctx, node_count: *mut u64, capacity: *mut u64) -> c_int;
    pub fn lurk_trie_ctx_register(ctx: *mut lurk_trie_ctx, preimages: *const u8, n: usize, digests_out: *mut u8, fmt: c_int) -> c_int;
    pub fn lurk_trie_ctx_apply(ctx: *mut lurk_trie_ctx, n: usize, kinds: *const c_int, prev: *const i64, roots: *const u8, keys: *const u8,
                               values: *const u8, fmt: c_int, results_out: *mut u8, d_lookup_inputs: *mut c_void, d_insert_inputs: *mut c_void,
                               stream: *mut c_void) -> c_int;
    // the same on operations already in device memory: a shim may upload a replay batch in one copy and plan it on the GPU
    pub fn lurk_trie_ctx_apply_dev(ctx: *mut lurk_trie_ctx, n: usize, d_kinds: *const i32, d_prev: *const i64, d_roots: *const c_void,
                                   d_keys: *const c_void, d_values: *const c_void, fmt: c_int, d_results: *mut c_void, d_lookup_inputs: *mut c_void,
                                   d_insert_inputs: *mut c_void, stream: *mut c_void) -> c_int;
    pub fn lurk_trie_ctx_register_dev(ctx: *mut lurk_trie_ctx, d_preimages: *const c_void, n: usize, d_digests_out: *mut c_void, fmt: c_int,
                                      stream: *mut c_void) -> c_int;
    // S2 -- StoreCore::hydrate_z_cache (src/lem/store_core.rs:256-269)
    pub fn lurk_dag_hash(field_id: c_int, nodes: *const lurk_dag_node, n: usize, atom_digests: *const u8, n_atoms: usize, out: *mut u8) -> c_int;
    // S4 -- Arecibo CommitmentEngineTrait::commit (call sites src/proof/nova.rs:287,292)
    pub fn lurk_msm_ctx_create(curve_id: c_int, bases: *const u8, n: usize, fmt: c_int, out: *mut *mut lurk_msm_ctx) -> c_int;
    pub fn lurk_msm_ctx_precompute(ctx: *mut lurk_msm_ctx) -> c_int;
    pub fn lurk_msm_ctx_run(ctx: *mut lurk_msm_ctx, scalars: *const u8, n: usize, fmt: c_int, out_xyz: *mut u8) -> c_int;
    pub fn lurk_msm_ctx_destroy(ctx: *mut lurk_msm_ctx);
    // S5/S6 -- Proof::prove_recursively (src/proof/nova.rs:260-339, supernova.rs:207-291)
    pub fn lurk_fold_ctx_create(cfg: *const lurk_fold_config, ck_w: *mut lurk_msm_ctx, ck_t: *mut lurk_msm_ctx, out: *mut *mut lurk_fold_ctx) -> c_int;
    pub fn lurk_fold_ctx_destroy(ctx: *mut lurk_fold_ctx);
    pub fn lurk_fold_ctx_add_slot_batch(ctx: *mut lurk_fold_ctx, arity: c_int, count: usize, offsets: *const u64) -> c_int;
    pub fn lurk_fold_ctx_add_trie_batch(ctx: *mut lurk_fold_ctx, op: c_int, height: c_int, count: usize, offsets: *const u64) -> c_int;
    pub fn lurk_fold_ctx_set_spans(ctx: *mut lurk_fold_ctx, n: c_int, spans: *const lurk_fold_span) -> c_int;
    pub fn lurk_fold_ctx_set_ro(ctx: *mut lurk_fold_ctx, n_absorb: c_int, kinds: *const c_int, challenge_bits: c_int) -> c_int;
    pub fn lurk_fold_ctx_host_buffer(ctx: *mut lurk_fold_ctx, b: c_int, which: c_int, ptr: *mut *mut c_void, bytes: *mut usize) -> c_int;
    pub fn lurk_fold_ctx_exchange_handle(ctx: *mut lurk_fold_ctx, handle: *mut u8) -> c_int;
    pub fn lurk_fold_ctx_set_peers(ctx: *mut lurk_fold_ctx, handles: *const u8) -> c_int;
    pub fn lurk_fold_ctx_set_running(ctx: *mut lurk_fold_ctx, w: *const u8, e: *const u8, u: *const u8, x: *const u8, comm_w: *const u8, comm_e: *const u8, fmt: c_int) -> c_int;
    pub fn lurk_fold_ctx_get_running(ctx: *mut lurk_fold_ctx, w: *mut u8, e: *mut u8, u: *mut u8, x: *mut u8, comm_w: *mut u8, comm_e: *mut u8, fmt: c_int) -> c_int;
    pub fn lurk_fold_ctx_stage_a(ctx: *mut lurk_fold_ctx, b: c_int, flags: c_int, fmt: c_int) -> c_int;
    pub fn lurk_fold_ctx_init_running(ctx: *mut lurk_fold_ctx, b: c_int) -> c_int;
    pub fn lurk_fold_ctx_stage_b_launch(ctx: *mut lurk_fold_ctx, b: c_int) -> c_int;
    pub fn lurk_fold_ctx_collect(ctx: *mut lurk_fold_ctx, b: c_int, out: *mut lurk_fold_result, fmt: c_int) -> c_int;
    pub fn lurk_fold_ctx_check_running(ctx: *mut lurk_fold_ctx, bad_rows: *mut u64, comm_w_ok: *mut c_int, comm_e_ok: *mut c_int) -> c_int;
    pub fn lurk_fold_ctx_stats(ctx: *mut lurk_fold_ctx, la: *mut c_uint, lb: *mut c_uint, acc_w_ms: *mut f32, acc_t_ms: *mut f32) -> c_int;
    // N3 -- public_params -> CommitmentKey::setup (src/proof/nova.rs:196-216): from_label (Pedersen engines), powers of tau (HyperKZG)
    pub fn lurk_ck_size(num_cons: usize, num_vars: usize, ck_floor: usize) -> usize;
    pub fn lurk_ck_generate(curve_id: c_int, label: *const u8, label_len: usize, n: usize, fmt: c_int, bases_out: *mut u8) -> c_int;
    pub fn lurk_ck_generate_dev(curve_id: c_int, label: *const u8, label_len: usize, n: usize, d_bases: *mut c_void, stream: *mut c_void) -> c_int;
    pub fn lurk_ck_generate_range_dev(curve_id: c_int, label: *const u8, label_len: usize, first: usize, n: usize, d_bases: *mut c_void, stream: *mut c_void) -> c_int;
    pub fn lurk_ck_powers_dev(curve_id: c_int, g: *const u8, beta: *const u8, n: usize, d_bases: *mut c_void, fmt: c_int, stream: *mut c_void) -> c_int;
    pub fn lurk_msm_ctx_create_dev(curve_id: c_int, d_bases: *const c_void, n: usize, out: *mut *mut lurk_msm_ctx) -> c_int;
    // N4 -- compress (src/proof/nova.rs:341-356): the loops of RelaxedR1CSSNARK::prove / EvaluationEngine::prove; the transcript is the callback
    pub fn lurk_sumcheck_prove_dev(field_id: c_int, kind: c_int, d_polys: *const *mut c_void, num_rounds: c_int, claim: *const u8, challenge: lurk_challenge_fn,
                                   user: *mut c_void, round_evals: *mut u8, challenges: *mut u8, final_evals: *mut u8, fmt: c_int, stream: *mut c_void) -> c_int;
    pub fn lurk_eq_evals_dev(field_id: c_int, tau: *const u8, num_vars: c_int, d_out: *mut c_void, fmt: c_int, stream: *mut c_void) -> c_int;
    pub fn lurk_inner_product_dev(field_id: c_int, d_a: *const c_void, d_b: *const c_void, n: usize, out: *mut u8, fmt: c_int, stream: *mut c_void) -> c_int;
    pub fn lurk_ipa_prove_dev(curve_id: c_int, ck: *mut lurk_msm_ctx, ck_c: *const u8, d_a: *mut c_void, d_b: *mut c_void, log_n: c_int, challenge: lurk_challenge_fn,
                              user: *mut c_void, l_out: *mut u8, r_out: *mut u8, a_final: *mut u8, b_final: *mut u8, fmt: c_int, stream: *mut c_void) -> c_int;
    pub fn lurk_hyperkzg_prove_dev(curve_id: c_int, ck: *mut lurk_msm_ctx, d_poly: *const c_void, point: *const u8, num_vars: c_int, challenge: lurk_challenge_fn,
                                   user: *mut c_void, com_out: *mut u8, w_out: *mut u8, v_out: *mut u8, fmt: c_int, stream: *mut c_void) -> c_int;
    pub fn lurk_batch_eval_reduce_dev(field_id: c_int, n_claims: c_int, d_polys: *const *const c_void, num_vars: *const c_int, points: *const u8,
                                      evals: *const u8, challenge: lurk_challenge_fn, user: *mut c_void, round_evals: *mut u8, r_out: *mut u8,
                                      claims_left: *mut u8, weights: *mut u8, joint_eval: *mut u8, d_joint: *mut c_void, fmt: c_int,
                                      stream: *mut c_void) -> c_int;
    // N4 -- RelaxedR1CSSNARK::prove / BatchedRelaxedR1CSSNARK::prove in one call (src/proof/nova.rs:341-356, supernova.rs:293-317)
    pub fn lurk_spartan_ctx_create(field_id: c_int, n_w: u64, n_x: u64, n_rows: u64, row_ptr: *const *const u64, col: *const *const u32,
                                   val: *const *const u8, fmt: c_int, out: *mut *mut lurk_spartan_ctx) -> c_int;
    pub fn lurk_spartan_ctx_create_verifier(field_id: c_int, n_w: u64, n_x: u64, n_rows: u64, row_ptr: *const *const u64, col: *const *const u32,
                                            val: *const *const u8, fmt: c_int, out: *mut *mut lurk_spartan_ctx) -> c_int;
    pub fn lurk_spartan_ctx_destroy(ctx: *mut lurk_spartan_ctx);
    pub fn lurk_spartan_ctx_info(ctx: *mut lurk_spartan_ctx, field_id: *mut c_int, log_rows: *mut c_int, log_vars: *mut c_int, joint_len: *mut usize) -> c_int;
    pub fn lurk_spartan_prove_dev(ctx: *mut lurk_spartan_ctx, d_z: *const c_void, d_e: *const c_void, challenge: lurk_spartan_challenge_fn, user: *mut c_void,
                                  out: *mut lurk_spartan_proof, d_joint: *mut c_void, fmt: c_int, stream: *mut c_void) -> c_int;
    pub fn lurk_spartan_prove_batch_dev(n: c_int, ctxs: *const *mut lurk_spartan_ctx, d_z: *const *const c_void, d_e: *const *const c_void,
                                        challenge: lurk_spartan_challenge_fn, user: *mut c_void, out: *mut lurk_spartan_proof, d_joint: *mut c_void,
                                        fmt: c_int, stream: *mut c_void) -> c_int;
    pub fn lurk_spartan_eval_table_dev(ctx: *mut lurk_spartan_ctx, d_eq_rx: *const c_void, r: *const u8, d_out: *mut c_void, fmt: c_int,
                                       stream: *mut c_void) -> c_int;
    // N4 -- the data-parallel parts of CompressedSNARK::verify (src/proof/nova.rs:358-373)
    pub fn lurk_spartan_matrix_evals_dev(ctx: *mut lurk_spartan_ctx, r_x: *const u8, r_y: *const u8, out: *mut u8, fmt: c_int, stream: *mut c_void) -> c_int;
    pub fn lurk_spartan_verify(ctx: *mut lurk_spartan_ctx, u: *const u8, x: *const u8, proof: *mut lurk_spartan_proof, rounds_fmt: c_int,
                               challenge: lurk_spartan_challenge_fn, user: *mut c_void, accepted: *mut c_int, fmt: c_int, stream: *mut c_void) -> c_int;
    pub fn lurk_spartan_verify_batch(n: c_int, ctxs: *const *mut lurk_spartan_ctx, u: *const u8, x: *const *const u8, proof: *mut lurk_spartan_proof,
                                     rounds_fmt: c_int, challenge: lurk_spartan_challenge_fn, user: *mut c_void, accepted: *mut c_int, fmt: c_int,
                                     stream: *mut c_void) -> c_int;
    pub fn lurk_ipa_verify_dev(curve_id: c_int, ck: *mut lurk_msm_ctx, ck_c: *const u8, comm: *const u8, c: *const u8, d_b: *const c_void, log_n: c_int,
                               l: *const u8, r: *const u8, a_final: *const u8, challenge: lurk_challenge_fn, user: *mut c_void, accepted: *mut c_int,
                               ck_hat_out: *mut u8, b_hat_out: *mut u8, fmt: c_int, stream: *mut c_void) -> c_int;
    // S6 -- RecursiveSNARK::verify's three is_sat* calls (Proof::verify on a Recursive proof, src/proof/nova.rs:358-373): Nova
    // [r_U_primary, r_U_secondary, l_u_secondary], SuperNova every Some running primary then the secondary's two.  The num_steps, z0 and
    // X.len() checks and the two RO hashes stay in Rust.  Host form: z = (W, u, X) and E as Arecibo's structs hold them, in `fmt`.
    pub fn lurk_recursive_verify(n: c_int, inst: *const lurk_recursive_instance, out: *mut lurk_recursive_verdict, accepted: *mut c_int, fmt: c_int,
                                 stream: *mut c_void) -> c_int;
    pub fn lurk_recursive_verify_dev(n: c_int, inst: *const lurk_recursive_instance, out: *mut lurk_recursive_verdict, accepted: *mut c_int,
                                     fmt: c_int, stream: *mut c_void) -> c_int;
    // CompressedSNARK::prove in one call.  Before it, fold l_u_secondary into r_U_secondary (Arecibo's NIFS::prove) with one more
    // lurk_fold_ctx_stage_a + lurk_fold_ctx_stage_b_launch + lurk_fold_ctx_collect on the secondary fold context; then pass both fold
    // contexts' LURK_FOLD_BUF_Z1 / _E1 pointers and the records' running commitments.
    pub fn lurk_compress_ctx_create(n_primary: c_int, primary: *const *mut lurk_spartan_ctx, secondary: *mut lurk_spartan_ctx,
                                    pcs_primary: *const lurk_compress_pcs, pcs_secondary: *const lurk_compress_pcs, fmt: c_int,
                                    out: *mut *mut lurk_compress_ctx) -> c_int;
    pub fn lurk_compress_ctx_destroy(ctx: *mut lurk_compress_ctx);
    pub fn lurk_compress_ctx_info(ctx: *mut lurk_compress_ctx, device_bytes: *mut usize, joint_len_primary: *mut usize, joint_len_secondary: *mut usize) -> c_int;
    pub fn lurk_compress_prove_dev(ctx: *mut lurk_compress_ctx, n_primary: c_int, d_z: *const *const c_void, d_e: *const *const c_void,
                                   comm_w: *const *const u8, comm_e: *const *const u8, d_z2: *const c_void, d_e2: *const c_void, comm_w2: *const u8,
                                   comm_e2: *const u8, challenge: lurk_compress_challenge_fn, user: *mut c_void, flags: c_int,
                                   out: *mut lurk_compress_proof, fmt: c_int, stream: *mut c_void) -> c_int;
    // N4 -- CompressedSNARK::verify (src/proof/nova.rs:358-373): after NIFS::verify of the secondary, which stays in Rust
    pub fn lurk_compress_verify(n_primary: c_int, primary: *const *mut lurk_spartan_ctx, secondary: *mut lurk_spartan_ctx,
                                pcs_primary: *const lurk_compress_vk_pcs, pcs_secondary: *const lurk_compress_vk_pcs, u: *const u8,
                                x: *const *const u8, comm_w: *const *const u8, comm_e: *const *const u8, u2: *const u8, x2: *const u8,
                                comm_w2: *const u8, comm_e2: *const u8, proof: *const lurk_compress_proof, rounds_fmt: c_int,
                                challenge: lurk_compress_challenge_fn, pairing: Option<lurk_pairing_check_fn>, user: *mut c_void, flags: c_int,
                                out: *mut lurk_compress_verdict, accepted: *mut c_int, fmt: c_int, stream: *mut c_void) -> c_int;
    pub fn lurk_point_combination(curve_id: c_int, points_xyz: *const u8, scalars: *const u8, count: usize, fmt: c_int, out_xyz: *mut u8) -> c_int;
}
pub const LURK_SPARTAN_ROUNDS_EVALS: c_int = 0;
pub const LURK_SPARTAN_ROUNDS_COMPRESSED: c_int = 1;
/// `int (*)(void *user, int phase, int round, const uint8_t *message, size_t message_len, uint8_t challenge_out[32])`: the phase-tagged
/// transcript of the Spartan prover context (LURK_SPARTAN_*).  The caller has absorbed the vk digest and U before the call.
pub type lurk_spartan_challenge_fn = unsafe extern "C" fn(user: *mut c_void, phase: c_int, round: c_int, message: *const u8, message_len: usize,
                                                          challenge_out: *mut u8) -> c_int;
pub unsafe extern "C" fn spartan_trampoline<F: FnMut(i32, i32, &[u8]) -> Option<[u8; 32]>>(user: *mut c_void, phase: c_int, round: c_int, message: *const u8,
                                                                                          len: usize, out: *mut u8) -> c_int {
    let f = &mut *(user as *mut F);
    let msg = if len == 0 { &[][..] } else { std::slice::from_raw_parts(message, len) };
    match f(phase, round, msg) {
        Some(r) => { std::ptr::copy_nonoverlapping(r.as_ptr(), out, 32); 0 }
        None => 1,
    }
}
/// `int (*)(void *user, int round, const uint8_t *message, size_t message_len, uint8_t challenge_out[32])`: the Fiat-Shamir transcript stays in
/// Rust.  A closure is passed as `user` and trampolined, e.g. for SumcheckProof::prove_*:
/// `|round, msg| { transcript.absorb(b"p", &UniPoly::from_evals(&elems(msg)).compress()); transcript.squeeze(b"c") }`.
pub type lurk_challenge_fn = unsafe extern "C" fn(user: *mut c_void, round: c_int, message: *const u8, message_len: usize, challenge_out: *mut u8) -> c_int;
pub unsafe extern "C" fn challenge_trampoline<F: FnMut(i32, &[u8]) -> Option<[u8; 32]>>(user: *mut c_void, round: c_int, message: *const u8, len: usize, out: *mut u8) -> c_int {
    let f = &mut *(user as *mut F);
    match f(round, std::slice::from_raw_parts(message, len)) {
        Some(r) => { std::ptr::copy_nonoverlapping(r.as_ptr(), out, 32); 0 }
        None => 1,
    }
}

#[derive(Debug)]
pub struct B200Error { pub code: c_int, pub message: String }
fn check(code: c_int) -> Result<(), B200Error> {
    if code == 0 { return Ok(()); }
    let message = unsafe { CStr::from_ptr(lurk_last_error()) }.to_string_lossy().into_owned();
    Err(B200Error { code, message })
}

/// `PoseidonCache::hashN` for a whole batch: `[F; A]` rows are `repr(C)` `[u64; 4]` Montgomery limbs for pasta_curves
/// (feature `repr-c`, Cargo.toml:42) and halo2curves, so the slices are passed as they are.
pub fn poseidon_hash_batch_mont(field_id: c_int, arity: usize, preimages: &[u8], digests: &mut [u8]) -> Result<(), B200Error> {
    let n = digests.len() / 32;
    assert_eq!(preimages.len(), n * arity * 32);
    check(unsafe { lurk_poseidon_hash_batch_mont(field_id, arity as c_int, preimages.as_ptr(), n, digests.as_mut_ptr()) })
}

/// A device-resident commitment key: what `CommitmentKey<E>` + `commit` become (Arecibo provider; src/proof/nova.rs:196-216).
pub struct MsmCtx(*mut lurk_msm_ctx);
unsafe impl Send for MsmCtx {}
impl MsmCtx {
    pub fn new(curve_id: c_int, bases_affine_mont: &[u8]) -> Result<Self, B200Error> {
        let mut p = std::ptr::null_mut();
        check(unsafe { lurk_msm_ctx_create(curve_id, bases_affine_mont.as_ptr(), bases_affine_mont.len() / 64, LURK_FMT_MONTGOMERY, &mut p) })?;
        check(unsafe { lurk_msm_ctx_precompute(p) })?;
        Ok(Self(p))
    }
    /// `vartime_multiscalar_mul(scalars, bases[..n])` -> x | y | z (z = 1, or all zero for the identity), Montgomery limbs
    pub fn commit(&self, scalars_mont: &[u8]) -> Result<[u8; 96], B200Error> {
        let mut out = [0u8; 96];
        check(unsafe { lurk_msm_ctx_run(self.0, scalars_mont.as_ptr(), scalars_mont.len() / 32, LURK_FMT_MONTGOMERY, out.as_mut_ptr()) })?;
        Ok(out)
    }
    pub fn raw(&self) -> *mut lurk_msm_ctx { self.0 }
}
impl Drop for MsmCtx { fn drop(&mut self) { unsafe { lurk_msm_ctx_destroy(self.0) } } }

/// One running instance on the device (`RecursiveSNARK`'s primary or secondary half; one per circuit index for SuperNova).
pub struct FoldCtx { raw: *mut lurk_fold_ctx, depth: usize, next: usize }
unsafe impl Send for FoldCtx {}
impl FoldCtx {
    /// # Safety: the CSR slices must stay valid for the duration of the call only; `ck` must outlive the context.
    pub unsafe fn new(cfg: &lurk_fold_config, ck_w: &MsmCtx, ck_t: &MsmCtx) -> Result<Self, B200Error> {
        let mut p = std::ptr::null_mut();
        check(lurk_fold_ctx_create(cfg, ck_w.raw(), ck_t.raw(), &mut p))?;
        Ok(Self { raw: p, depth: cfg.depth as usize, next: 0 })
    }
    /// the pinned buffer the witness thread (src/proof/nova.rs:306-318) writes this step's inputs into
    pub fn host_buffer(&mut self, b: usize, which: c_int) -> Result<&mut [u8], B200Error> {
        let (mut p, mut n) = (std::ptr::null_mut(), 0usize);
        check(unsafe { lurk_fold_ctx_host_buffer(self.raw, b as c_int, which, &mut p, &mut n) })?;
        Ok(unsafe { std::slice::from_raw_parts_mut(p as *mut u8, n) })
    }
    pub fn next_buffer(&mut self) -> usize { let b = self.next; self.next = (b + 1) % self.depth; b }
    pub fn stage_a(&mut self, b: usize) -> Result<(), B200Error> { check(unsafe { lurk_fold_ctx_stage_a(self.raw, b as c_int, 0, LURK_FMT_MONTGOMERY) }) }
    pub fn init_running(&mut self, b: usize) -> Result<(), B200Error> { check(unsafe { lurk_fold_ctx_init_running(self.raw, b as c_int) }) }
    pub fn fold(&mut self, b: usize) -> Result<(), B200Error> { check(unsafe { lurk_fold_ctx_stage_b_launch(self.raw, b as c_int) }) }
    pub fn collect(&mut self, b: usize) -> Result<lurk_fold_result, B200Error> {
        let mut r = std::mem::MaybeUninit::<lurk_fold_result>::zeroed();
        check(unsafe { lurk_fold_ctx_collect(self.raw, b as c_int, r.as_mut_ptr(), LURK_FMT_MONTGOMERY) })?;
        Ok(unsafe { r.assume_init() })
    }
}
impl Drop for FoldCtx { fn drop(&mut self) { unsafe { lurk_fold_ctx_destroy(self.raw) } } }

/// One circuit shape's Spartan prover key on the device (`ProverKey` of RelaxedR1CSSNARK): the matrices and their merged transpose, built
/// on the GPU.  `prove` runs RelaxedR1CSSNARK::prove + batch_eval_reduce straight from a fold context's running instance
/// (`lurk_fold_ctx_device_buffer(LURK_FOLD_BUF_Z1 / _E1)`), leaving the joint polynomial in `d_joint` for the EE opening.
pub struct SpartanCtx(*mut lurk_spartan_ctx);
unsafe impl Send for SpartanCtx {}
impl SpartanCtx {
    /// row_ptr / col / val: the A, B, C CSR over z = (W, u, X) as lurk_fold_config takes them (Montgomery coefficients)
    pub fn new(field_id: c_int, n_w: u64, n_x: u64, n_rows: u64, row_ptr: [&[u64]; 3], col: [&[u32]; 3], val: [&[u8]; 3]) -> Result<Self, B200Error> {
        let rp = [row_ptr[0].as_ptr(), row_ptr[1].as_ptr(), row_ptr[2].as_ptr()];
        let cl = [col[0].as_ptr(), col[1].as_ptr(), col[2].as_ptr()];
        let vl = [val[0].as_ptr(), val[1].as_ptr(), val[2].as_ptr()];
        let mut p = std::ptr::null_mut();
        check(unsafe { lurk_spartan_ctx_create(field_id, n_w, n_x, n_rows, rp.as_ptr(), cl.as_ptr(), vl.as_ptr(), LURK_FMT_MONTGOMERY, &mut p) })?;
        Ok(Self(p))
    }
    /// (log_rows, log_vars, joint length)
    pub fn info(&self) -> Result<(i32, i32, usize), B200Error> {
        let (mut lr, mut lv, mut jl) = (0, 0, 0usize);
        check(unsafe { lurk_spartan_ctx_info(self.0, std::ptr::null_mut(), &mut lr, &mut lv, &mut jl) })?;
        Ok((lr, lv, jl))
    }
    /// # Safety: d_z / d_e / d_joint are device pointers of the sizes include/lurk_b200.h gives; `out`'s buffers are large enough.
    pub unsafe fn prove<F: FnMut(i32, i32, &[u8]) -> Option<[u8; 32]>>(&mut self, d_z: *const c_void, d_e: *const c_void, transcript: &mut F,
                                                                       out: &mut lurk_spartan_proof, d_joint: *mut c_void) -> Result<(), B200Error> {
        check(lurk_spartan_prove_dev(self.0, d_z, d_e, spartan_trampoline::<F>, transcript as *mut F as *mut c_void, out, d_joint,
                                     LURK_FMT_MONTGOMERY, std::ptr::null_mut()))
    }
    /// BatchedRelaxedR1CSSNARK::prove over one running instance per circuit index (SuperNova)
    /// # Safety: as `prove`, per instance.
    pub unsafe fn prove_batch<F: FnMut(i32, i32, &[u8]) -> Option<[u8; 32]>>(ctxs: &mut [&mut SpartanCtx], d_z: &[*const c_void], d_e: &[*const c_void],
                                                                             transcript: &mut F, out: &mut lurk_spartan_proof, d_joint: *mut c_void)
                                                                             -> Result<(), B200Error> {
        let raw: Vec<*mut lurk_spartan_ctx> = ctxs.iter().map(|c| c.0).collect();
        check(lurk_spartan_prove_batch_dev(raw.len() as c_int, raw.as_ptr(), d_z.as_ptr(), d_e.as_ptr(), spartan_trampoline::<F>,
                                           transcript as *mut F as *mut c_void, out, d_joint, LURK_FMT_MONTGOMERY, std::ptr::null_mut()))
    }
    /// RelaxedR1CSSNARK::verify up to the opening, from Arecibo's proof fields with their compressed round polynomials; on acceptance `proof`'s
    /// r / weights / joint_eval say which opening remains.  Ok(false) = rejected.
    /// # Safety: `proof`'s buffers have the sizes include/lurk_b200.h gives; u is 32 bytes, x n_x x 32 bytes (Montgomery).
    pub unsafe fn verify<F: FnMut(i32, i32, &[u8]) -> Option<[u8; 32]>>(&mut self, u: &[u8], x: &[u8], transcript: &mut F, proof: &mut lurk_spartan_proof)
                                                                        -> Result<bool, B200Error> {
        let mut accepted: c_int = 0;
        check(lurk_spartan_verify(self.0, u.as_ptr(), x.as_ptr(), proof, LURK_SPARTAN_ROUNDS_COMPRESSED, spartan_trampoline::<F>,
                                  transcript as *mut F as *mut c_void, &mut accepted, LURK_FMT_MONTGOMERY, std::ptr::null_mut()))?;
        Ok(accepted != 0)
    }
    /// BatchedRelaxedR1CSSNARK::verify (SuperNova): u = n x 32 bytes, x[i] = instance i's public values.
    /// # Safety: as `verify`, per instance.
    pub unsafe fn verify_batch<F: FnMut(i32, i32, &[u8]) -> Option<[u8; 32]>>(ctxs: &mut [&mut SpartanCtx], u: &[u8], x: &[&[u8]], transcript: &mut F,
                                                                              proof: &mut lurk_spartan_proof) -> Result<bool, B200Error> {
        let raw: Vec<*mut lurk_spartan_ctx> = ctxs.iter().map(|c| c.0).collect();
        let xs: Vec<*const u8> = x.iter().map(|v| v.as_ptr()).collect();
        let mut accepted: c_int = 0;
        check(lurk_spartan_verify_batch(raw.len() as c_int, raw.as_ptr(), u.as_ptr(), xs.as_ptr(), proof, LURK_SPARTAN_ROUNDS_COMPRESSED,
                                        spartan_trampoline::<F>, transcript as *mut F as *mut c_void, &mut accepted, LURK_FMT_MONTGOMERY,
                                        std::ptr::null_mut()))?;
        Ok(accepted != 0)
    }
}

/// InnerProductArgument::verify (EE2, and EE1 on Pallas): `comm` = the joint commitment, `c` = joint_eval, `d_b` = eq(r) on the device (2^log_n
/// Montgomery elements), `l` / `r` = the proof's L_vec / R_vec as 96-byte points.  The key context is not consumed.  Ok(false) = rejected.
/// # Safety: `d_b` is a device pointer of 2^log_n elements; `l` / `r` hold log_n points each.
pub unsafe fn ipa_verify<F: FnMut(i32, &[u8]) -> Option<[u8; 32]>>(curve_id: c_int, ck: &MsmCtx, ck_c: &[u8; 64], comm: &[u8; 96], c: &[u8; 32],
                                                                   d_b: *const c_void, log_n: i32, l: &[u8], r: &[u8], a_final: &[u8; 32],
                                                                   transcript: &mut F) -> Result<bool, B200Error> {
    let mut accepted: c_int = 0;
    check(lurk_ipa_verify_dev(curve_id, ck.raw(), ck_c.as_ptr(), comm.as_ptr(), c.as_ptr(), d_b, log_n, l.as_ptr(), r.as_ptr(), a_final.as_ptr(),
                              challenge_trampoline::<F>, transcript as *mut F as *mut c_void, &mut accepted, std::ptr::null_mut(),
                              std::ptr::null_mut(), LURK_FMT_MONTGOMERY, std::ptr::null_mut()))?;
    Ok(accepted != 0)
}
impl Drop for SpartanCtx { fn drop(&mut self) { unsafe { lurk_spartan_ctx_destroy(self.0) } } }

/// CompressedSNARK::verify in one call.  `transcript(circuit, phase, round, msg)` is the prover's callback (one transcript per circuit; the two
/// circuits may call at once, so it must be Sync), `pairing(P, Q)` the HyperKZG check e(P, H) == e(Q, beta H).  `inst` = (u, X, comm_W,
/// comm_E) per primary instance, `inst2` = f_U_secondary's, already folded by NIFS::verify.  Returns (accepted, verdicts).
/// # Safety: `proof`'s buffers have the sizes include/lurk_b200.h gives; X slices hold each shape's n_x elements.
pub unsafe fn compress_verify<T, P>(primary: &[&SpartanCtx], secondary: &SpartanCtx, pcs: [&lurk_compress_vk_pcs; 2], u: &[u8], inst: &[(&[u8], &[u8; 96], &[u8; 96])],
                                    inst2: (&[u8; 32], &[u8], &[u8; 96], &[u8; 96]), proof: &lurk_compress_proof, batched: bool, transcript: &T, pairing: &P)
                                    -> Result<(bool, [lurk_compress_verdict; 2]), B200Error>
where T: Fn(i32, i32, i32, &[u8]) -> Option<[u8; 32]> + Sync, P: Fn(i32, &[u8; 96], &[u8; 96]) -> Option<bool> + Sync {
    struct User<'a, T, P> { t: &'a T, p: &'a P }
    unsafe extern "C" fn tr<T: Fn(i32, i32, i32, &[u8]) -> Option<[u8; 32]> + Sync, P>(user: *mut c_void, circuit: c_int, phase: c_int, round: c_int,
                                                                                     msg: *const u8, len: usize, out: *mut u8) -> c_int {
        let u = &*(user as *const User<T, P>);
        let m = if len == 0 { &[][..] } else { std::slice::from_raw_parts(msg, len) };
        match (u.t)(circuit, phase, round, m) { Some(r) => { std::ptr::copy_nonoverlapping(r.as_ptr(), out, 32); 0 } None => 1 }
    }
    unsafe extern "C" fn pc<T, P: Fn(i32, &[u8; 96], &[u8; 96]) -> Option<bool> + Sync>(user: *mut c_void, circuit: c_int, p: *const u8, q: *const u8,
                                                                                      holds: *mut c_int) -> c_int {
        let u = &*(user as *const User<T, P>);
        match (u.p)(circuit, &*(p as *const [u8; 96]), &*(q as *const [u8; 96])) { Some(h) => { *holds = h as c_int; 0 } None => 1 }
    }
    let user = User { t: transcript, p: pairing };
    let raw: Vec<*mut lurk_spartan_ctx> = primary.iter().map(|c| c.0).collect();
    let xs: Vec<*const u8> = inst.iter().map(|i| i.0.as_ptr()).collect();
    let cw: Vec<*const u8> = inst.iter().map(|i| i.1.as_ptr()).collect();
    let ce: Vec<*const u8> = inst.iter().map(|i| i.2.as_ptr()).collect();
    let (mut out, mut accepted) = ([lurk_compress_verdict::default(); 2], 0 as c_int);
    check(lurk_compress_verify(raw.len() as c_int, raw.as_ptr(), secondary.0, pcs[0], pcs[1], u.as_ptr(), xs.as_ptr(), cw.as_ptr(), ce.as_ptr(),
                               inst2.0.as_ptr(), inst2.1.as_ptr(), inst2.2.as_ptr(), inst2.3.as_ptr(), proof, LURK_SPARTAN_ROUNDS_COMPRESSED, tr::<T, P>,
                               Some(pc::<T, P>), &user as *const User<T, P> as *mut c_void, if batched { LURK_COMPRESS_BATCHED } else { 0 },
                               out.as_mut_ptr(), &mut accepted, LURK_FMT_MONTGOMERY, std::ptr::null_mut()))?;
    Ok((accepted != 0, out))
}
