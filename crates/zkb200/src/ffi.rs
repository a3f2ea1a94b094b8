//! `extern "C"` declarations of include/zkb200.h (the subset the shim calls; `bindgen include/zkb200.h` gives the rest).
#![allow(non_camel_case_types)]
use core::ffi::{c_char, c_int, c_uint, c_void};

#[repr(C)]
pub struct zk_ctx {
    _p: [u8; 0],
}
#[repr(C)]
pub struct zk_bases {
    _p: [u8; 0],
}
#[repr(C)]
pub struct zk_srs {
    _p: [u8; 0],
}
#[repr(C)]
pub struct zk_index_cache {
    _p: [u8; 0],
}

/// zk_index_header: the cache file's ScalarHeader and preamble fields (kimchi/src/cached_prover_index.rs:173-225)
#[repr(C)]
pub struct zk_index_header {
    pub public_inputs: u32,
    pub prev_challenges: u32,
    pub zk_rows: u64,
    pub max_poly_size: u64,
    pub domain_d1_size: u64,
    pub feature_flags: u32,
    pub optional_selectors_present: u32,
    pub lookup_selectors_present: u32,
    pub num_sections: u32,
    pub disable_gates_checks: c_int,
    pub has_verifier_index_digest: c_int,
    pub endo: [u64; 4],
    pub shift: [[u64; 4]; 7],
    pub verifier_index_digest: [u64; 4],
    pub identifier: [c_char; 512],
}

pub const ZK_FP: c_int = 0;
pub const ZK_FQ: c_int = 1;
pub const ZK_PALLAS: c_int = 0;
pub const ZK_VESTA: c_int = 1;
pub const ZK_OK: c_int = 0;
pub const ZK_ERR_LENGTH: c_int = -4;

#[repr(C)]
pub struct zk_open_poly {
    pub data: *const u64,
    pub len: usize,
    pub domain_size: usize,
    pub blinders: *const u64,
    pub n_blinders: usize,
}

#[repr(C)]
pub struct zk_open_transcript {
    pub user: *mut c_void,
    pub u_base: unsafe extern "C" fn(user: *mut c_void, cip: *const u64, out_u_xy: *mut u64) -> c_int,
    pub round: unsafe extern "C" fn(user: *mut c_void, round: c_uint, l_xy: *const u64, r_xy: *const u64, out_u: *mut u64) -> c_int,
    pub final_challenge: unsafe extern "C" fn(user: *mut c_void, delta_xy: *const u64, out_c: *mut u64) -> c_int,
}

#[repr(C)]
pub struct zk_verify_proof {
    pub lr_xy: *const u64,
    pub n_rounds: usize,
    pub delta_xy: *const u64,
    pub z1: *const u64,
    pub z2: *const u64,
    pub sg_xy: *const u64,
    pub elm: *const u64,
    pub n_elm: usize,
    pub polyscale: *const u64,
    pub evalscale: *const u64,
    pub comm_xy: *const u64,
    pub comm_chunks: *const usize,
    pub n_comms: usize,
    pub combined_inner_product: *const u64,
    pub transcript: *const zk_open_transcript,
}

pub const ZK_EXPR_CONST: u32 = 0;
pub const ZK_EXPR_CELL: u32 = 1;
pub const ZK_EXPR_DUP: u32 = 2;
pub const ZK_EXPR_POW: u32 = 3;
pub const ZK_EXPR_ADD: u32 = 4;
pub const ZK_EXPR_MUL: u32 = 5;
pub const ZK_EXPR_SUB: u32 = 6;
pub const ZK_EXPR_STORE: u32 = 7;
pub const ZK_EXPR_LOAD: u32 = 8;

#[repr(C)]
#[derive(Copy, Clone)]
pub struct zk_expr_token {
    pub op: u32,
    pub arg: u32,
}

#[repr(C)]
#[derive(Copy, Clone)]
pub struct zk_expr_column {
    pub d_evals: *const c_void,
    pub len: u64,
    pub domain_mult: u32,
    pub reserved: u32,
}

#[repr(C)]
#[derive(Copy, Clone)]
pub struct zk_eval_column {
    pub d_evals: *const c_void,
    pub len: u64,
    pub boolean: u32,
    pub reserved: u32,
}

#[repr(C)]
#[derive(Copy, Clone)]
pub struct zk_dev_poly {
    pub d_coeffs: *const c_void,
    pub len: u64,
}

/// zk_lookup_term: coeff (Montgomery) * w[column][row + next]
#[repr(C)]
#[derive(Clone, Copy)]
pub struct zk_lookup_term {
    pub coeff: [u64; 4],
    pub column: u32,
    pub next: u32,
}

/// zk_lookup_joint: one JointLookupSpec; entry e is entry_terms[e] consecutive terms from first_term on
#[repr(C)]
#[derive(Clone, Copy)]
pub struct zk_lookup_joint {
    pub table_id: i32,
    pub table_id_column: i32, // -1: Constant(table_id), else WitnessColumn
    pub n_entries: u32,
    pub entry_terms: [u32; 4],
    pub first_term: u32,
}

/// zk_lookup_info: LookupInfo lowered (patterns of lookups, each row's pattern: 0 none, p + 1 pattern p)
#[repr(C)]
pub struct zk_lookup_info {
    pub terms: *const zk_lookup_term,
    pub n_terms: usize,
    pub lookups: *const zk_lookup_joint,
    pub n_lookups: usize,
    pub pattern_first: *const u32,
    pub pattern_count: *const u32,
    pub n_patterns: usize,
    pub row_pattern: *const u8,
    pub max_per_row: c_uint,
    pub joint_combiner: [u64; 4],
    pub table_id_combiner: [u64; 4],
    pub dummy: [u64; 4],
}

#[repr(C)]
#[derive(Copy, Clone)]
pub struct zk_lin_term {
    pub d_evals: *const c_void,
    pub len: u64,
    pub coeff: [u64; 4],
}

/// zk_lookup_table: one LookupTable, its `width` columns of `len` Montgomery elements back to back (column-major)
#[repr(C)]
#[derive(Copy, Clone)]
pub struct zk_lookup_table {
    pub id: i32,
    pub width: u32,
    pub len: u64,
    pub data: *const u64,
}

/// zk_runtime_table_cfg: one RuntimeTableCfg, its first column of `len` Montgomery elements
#[repr(C)]
#[derive(Copy, Clone)]
pub struct zk_runtime_table_cfg {
    pub id: i32,
    pub len: u64,
    pub first_column: *const u64,
}

/// the LookupError kinds zk_lookup_index_build reports (kimchi/src/circuits/lookup/index.rs:23-36)
pub const ZK_LOOKUP_ERR_NONE: c_int = 0;
pub const ZK_LOOKUP_ERR_ID_COLLISION: c_int = 1;
pub const ZK_LOOKUP_ERR_TABLE_ID_ZERO: c_int = 2;
pub const ZK_LOOKUP_ERR_TOO_LONG: c_int = 3;

extern "C" {
    pub fn zk_last_error() -> *const c_char;
    pub fn zk_ctx_create(device_id: c_int, out: *mut *mut zk_ctx) -> c_int;
    pub fn zk_ctx_destroy(ctx: *mut zk_ctx);

    pub fn zk_srs_create(ctx: *mut zk_ctx, curve_id: c_int, g_xy: *const u64, n: usize, h_xy: *const u64, window_bits: c_int,
                         out: *mut *mut zk_srs) -> c_int;
    pub fn zk_srs_generate(ctx: *mut zk_ctx, curve_id: c_int, depth: usize, window_bits: c_int, g_xy_out: *mut u64, h_xy_out: *mut u64,
                           out: *mut *mut zk_srs) -> c_int;
    pub fn zk_srs_destroy(srs: *mut zk_srs);
    pub fn zk_srs_lagrange_basis(srs: *mut zk_srs, domain_size: usize, window_bits: c_int) -> c_int;
    pub fn zk_srs_lagrange_basis_chunks(srs: *const zk_srs, domain_size: usize) -> usize;
    pub fn zk_srs_get_lagrange_basis(srs: *mut zk_srs, domain_size: usize, out_xy: *mut u64, capacity_points: usize) -> c_int;
    pub fn zk_srs_commit_non_hiding(srs: *mut zk_srs, coeffs_mont: *const u64, len: usize, num_chunks: usize, out_xy: *mut u64,
                                    out_capacity: usize, out_chunks: *mut usize) -> c_int;
    pub fn zk_srs_commit_evaluations_non_hiding(srs: *mut zk_srs, domain_size: usize, evals_mont: *const u64, evals_domain_size: usize,
                                                out_xy: *mut u64) -> c_int;
    pub fn zk_srs_mask_custom(srs: *mut zk_srs, chunks_xy: *const u64, n_chunks: usize, blinders_mont: *const u64, n_blinders: usize,
                              out_xy: *mut u64) -> c_int;
    pub fn zk_srs_open(srs: *mut zk_srs, polys: *const zk_open_poly, n_polys: usize, elm_mont: *const u64, n_elm: usize,
                       polyscale: *const u64, evalscale: *const u64, rng_scalars: *const u64, n_rng_scalars: usize,
                       transcript: *const zk_open_transcript, out_lr_xy: *mut u64, lr_capacity_rounds: usize, out_rounds: *mut usize,
                       out_delta_xy: *mut u64, out_z1: *mut u64, out_z2: *mut u64, out_sg_xy: *mut u64) -> c_int;
    pub fn zk_srs_verify(srs: *mut zk_srs, batch: *const zk_verify_proof, n: usize, rng_scalars: *const u64, out_ok: *mut c_int,
                         out_sum_xyz: *mut u64) -> c_int;
    pub fn zk_srs_accumulator_check(srs: *mut zk_srs, comms_xy: *const u64, n_comms: usize, chals_mont: *const u64, n_chals: usize,
                                    r_mont: *const u64, out_ok: *mut c_int, out_sum_xyz: *mut u64) -> c_int;
    pub fn zk_srs_accumulator_generate(srs: *mut zk_srs, num_comms: usize, chals_mont: *const u64, n_chals: usize, out_xy: *mut u64,
                                       capacity_points: usize, out_points: *mut usize) -> c_int;

    pub fn zk_dev_alloc(ctx: *mut zk_ctx, bytes: usize, out: *mut *mut c_void) -> c_int;
    pub fn zk_dev_free(ctx: *mut zk_ctx, d_ptr: *mut c_void) -> c_int;
    pub fn zk_dev_upload(ctx: *mut zk_ctx, d_dst: *mut c_void, src: *const c_void, bytes: usize) -> c_int;
    pub fn zk_dev_download(ctx: *mut zk_ctx, dst: *mut c_void, d_src: *const c_void, bytes: usize) -> c_int;
    pub fn zk_expr_eval_dev(ctx: *mut zk_ctx, field_id: c_int, tokens: *const zk_expr_token, n_tokens: usize, constants_mont: *const u64,
                            n_constants: usize, cols: *const zk_expr_column, n_cols: usize, out_len: u64, out_domain_mult: c_uint,
                            accumulate: c_int, d_out: *mut c_void) -> c_int;

    pub fn zk_ntt_dev(ctx: *mut zk_ctx, field_id: c_int, d_data: *mut c_void, log_n: c_uint, batch: usize, in_len: usize, inverse: c_int,
                      coset: c_int) -> c_int;
    pub fn zk_ntt_dev_oop(ctx: *mut zk_ctx, field_id: c_int, d_in: *const c_void, in_stride: usize, in_len: usize, d_out: *mut c_void,
                          log_n: c_uint, batch: usize, inverse: c_int, coset: c_int) -> c_int;
    pub fn zk_poly_add_dev(ctx: *mut zk_ctx, field_id: c_int, d_dst: *mut c_void, d_src: *const c_void, len: usize) -> c_int;
    pub fn zk_poly_divide_by_vanishing_dev(ctx: *mut zk_ctx, field_id: c_int, d_f: *const c_void, len: usize, log_n: c_uint,
                                           d_quot: *mut c_void, remainder_is_zero: *mut c_int) -> c_int;

    pub fn zk_lagrange_evals_chunks(domain_size: usize, max_poly_size: usize) -> usize;
    pub fn zk_lagrange_evals_dev(ctx: *mut zk_ctx, field_id: c_int, log_n: c_uint, max_poly_size: usize, x_mont: *const u64,
                                 d_out: *mut c_void) -> c_int;
    pub fn zk_lagrange_evaluate_dev(ctx: *mut zk_ctx, field_id: c_int, d_bases: *const *const c_void, n_points: usize, log_n: c_uint,
                                    chunks: usize, cols: *const zk_eval_column, n_cols: usize, out: *mut u64) -> c_int;
    pub fn zk_poly_evaluate_chunks_dev(ctx: *mut zk_ctx, field_id: c_int, polys: *const zk_dev_poly, n_polys: usize, num_chunks: usize,
                                       chunk_size: usize, points_mont: *const u64, n_points: usize, out: *mut u64) -> c_int;
    pub fn zk_prover_ft_dev(ctx: *mut zk_ctx, field_id: c_int, log_n: c_uint, max_poly_size: usize, terms: *const zk_lin_term, n_terms: usize,
                            d_t: *const c_void, t_len: usize, zeta_mont: *const u64, d_ft: *mut c_void, ft_len: *mut usize,
                            ft_eval1: *mut u64) -> c_int;
    pub fn zk_lookup_joint_table_dev(ctx: *mut zk_ctx, field_id: c_int, log_n: c_uint, d_cols: *const *const c_void, n_cols: usize,
                                     d_table_ids8: *const c_void, d_runtime8: *const c_void, joint_combiner: *const u64,
                                     table_id_combiner: *const u64, d_out8: *mut c_void, d_out1: *mut c_void) -> c_int;
    pub fn zk_lookup_sorted_dev(ctx: *mut zk_ctx, field_id: c_int, log_n: c_uint, zk_rows: usize, d_w: *const *const c_void,
                                d_table: *const c_void, table_stride: c_uint, info: *const zk_lookup_info, rand: *const u64,
                                d_sorted: *const *mut c_void, not_in_table_row: *mut i64) -> c_int;
    pub fn zk_lookup_aggreg_dev(ctx: *mut zk_ctx, field_id: c_int, log_n: c_uint, zk_rows: usize, d_w: *const *const c_void,
                                d_table: *const c_void, table_stride: c_uint, info: *const zk_lookup_info, d_sorted: *const *const c_void,
                                beta: *const u64, gamma: *const u64, rand: *const u64, d_aggreg: *mut c_void, final_is_one: *mut c_int) -> c_int;
    pub fn zk_perm_aggreg_dev(ctx: *mut zk_ctx, field_id: c_int, log_n: c_uint, zk_rows: usize, d_w: *const *const c_void,
                              d_sigma: *const *const c_void, sigma_len: u64, beta: *const u64, gamma: *const u64, shifts: *const u64,
                              rand: *const u64, d_z: *mut c_void, final_is_one: *mut c_int) -> c_int;

    pub fn zk_ntt_batch(ctx: *mut zk_ctx, field_id: c_int, data: *mut u64, log_n: c_uint, batch: usize, in_len: usize, inverse: c_int,
                        coset: c_int) -> c_int;

    pub fn zk_index_cache_free(cache: *mut zk_index_cache);
    pub fn zk_index_cache_header(cache: *const zk_index_cache, out: *mut zk_index_header) -> c_int;
    pub fn zk_index_cache_section(cache: *const zk_index_cache, tag: u32, d_ptr: *mut *const c_void, n_elems: *mut usize,
                                  elem_domain_size: *mut u32) -> c_int;
    pub fn zk_index_build(ctx: *mut zk_ctx, field_id: c_int, hdr: *const zk_index_header, gates: *const c_void, n_gates: usize,
                          gate_coeffs: *const c_void, gate_coeffs_len: usize, zero_selectors: c_int, out: *mut *mut zk_index_cache) -> c_int;
    pub fn zk_index_commitments(srs: *mut zk_srs, index: *const zk_index_cache, out_xy: *mut u64, capacity_points: usize,
                                out_points: *mut usize) -> c_int;
    pub fn zk_lookup_index_build(ctx: *mut zk_ctx, field_id: c_int, domain_d1_size: u64, zk_rows: u64, gates: *const c_void, n_gates: usize,
                                 tables: *const zk_lookup_table, n_tables: usize, runtime: *const zk_runtime_table_cfg, n_runtime: usize,
                                 has_runtime: c_int, lookup_error: *mut c_int, runtime_table_offset: *mut u64,
                                 out: *mut *mut zk_index_cache) -> c_int;
    pub fn zk_lookup_index_commitments(srs: *mut zk_srs, lookup_index: *const zk_index_cache, out_xy: *mut u64, capacity_points: usize,
                                       out_points: *mut usize) -> c_int;
}
