// expr.cu — the constraint evaluator of the d8 pipeline (SURVEY.md §8f row 3): kimchi's expression framework on the device.
//
// The prover evaluates every gate's combined constraint over d4 or d8 with `Expr::evaluations(&env)`
// (kimchi/src/circuits/expr.rs:1938-2190; call sites kimchi/src/prover.rs:794-892: generic, the eleven gate arguments, the lookup
// constraints) and adds the results into t4 / t8.  The reference walks the expression TREE and materialises one array per node
// (rayon over the elements of each); here the expression arrives as the reference's own flat form — the RPN program of
// `PolishToken` (expr.rs:819-836, produced by `Expr::to_polish`) — and ONE kernel runs the program at every point of the domain:
// a thread per point, the operand stack and the `Store`/`Load` cache in the thread's local memory, every column read exactly once
// per use from where the d8 pipeline left it (zk_ntt_dev_oop, zk_index_cache_section), the result written — or accumulated into
// t4 / t8 — once.  No intermediate array exists.
//
// Semantics restated from PolishToken::evaluate (expr.rs:856-940) with the point replaced by the domain index:
//   CONST k          push constants[k]        (Literal / EndoCoefficient / Mds / Challenge terms, resolved by the caller)
//   CELL col|next    push col.evals[(scale * i + col.domain_mult * shift) % col.len], scale = col.len / out_len, shift = next ? 1 : 0
//                    — `SubEvals` indexing, expr.rs:1976-1982; VanishesOnZeroKnowledgeAndPreviousRows and
//                    UnnormalizedLagrangeBasis are columns the caller supplies (they are precomputed arrays in the reference too)
//   DUP, POW n, ADD, MUL, SUB, STORE, LOAD k     as in the reference;  SkipIf / SkipIfNot are resolved when the program is built
// The program is validated on the host (stack discipline, indices, divisibility); a malformed one never reaches the device.
#include <cstring>
#include <mutex>
#include <vector>

#include "../../include/zkb200.h"
#include "ctx.hpp"

using namespace zkb;

namespace zkb {

constexpr unsigned EXPR_MAX_STACK = 24, EXPR_MAX_CACHE = 96, EXPR_MAX_COLS = 64;

struct ExprCol {
    const fe* evals;
    uint64_t len;        // power of two
    uint32_t scale;      // len / out_len
    uint32_t mult;       // the column's domain multiple of d1 (1, 2, 4, 8)
};

struct ExprArgs {
    const zk_expr_token* tokens;   // device
    const fe* constants;           // device
    const ExprCol* cols;           // device
    fe* out;
    uint64_t out_len;
    uint32_t n_tokens;
    int accumulate;
};

template <class FS> __global__ void __launch_bounds__(128, 8) k_expr_eval(const __grid_constant__ ExprArgs a) {
    fe stack[EXPR_MAX_STACK], cache[EXPR_MAX_CACHE];
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.out_len; i += stride) {
        // the top of the stack lives in registers (`top`, valid while depth > 0); stack[0 .. depth - 2] holds what is below it: a
        // binary operator costs one local load instead of two loads and a store
        unsigned depth = 0, nc = 0;
        fe top = fe_zero();
#pragma unroll 1
        for (uint32_t t = 0; t < a.n_tokens; t++) {
            const zk_expr_token tok = a.tokens[t];          // uniform across the grid: one broadcast load
            switch (tok.op) {
            case ZK_EXPR_CONST:
                if (depth) stack[depth - 1] = top;
                top = load_fe_nc(a.constants + tok.arg); depth++;
                break;
            case ZK_EXPR_CELL: {
                const ExprCol c = a.cols[tok.arg & 0x7fffffffu];
                const uint64_t j = ((uint64_t)c.scale * i + ((tok.arg >> 31) ? c.mult : 0u)) & (c.len - 1);
                if (depth) stack[depth - 1] = top;
                top = load_fe_nc(c.evals + j); depth++;
                break;
            }
            case ZK_EXPR_DUP: stack[depth - 1] = top; depth++; break;
            case ZK_EXPR_POW: {
                // x^n: square-and-multiply from the top bit (n = 0 gives one, like ark's pow)
                const fe x = top;
                fe acc = fe_one<FS>();
                bool started = false;
                for (int b = 31 - __clz((int)(tok.arg | 1u)); b >= 0; b--) {
                    if (started) acc = fe_mul_call<FS>(acc, acc);
                    if ((tok.arg >> b) & 1u) { acc = started ? fe_mul_call<FS>(acc, x) : x; started = true; }
                }
                top = acc;
                break;
            }
            case ZK_EXPR_ADD: depth--; top = fe_add<FS>(stack[depth - 1], top); break;
            case ZK_EXPR_SUB: depth--; top = fe_sub<FS>(stack[depth - 1], top); break;
            case ZK_EXPR_MUL: depth--; top = fe_mul_call<FS>(stack[depth - 1], top); break;
            case ZK_EXPR_STORE: cache[nc++] = top; break;
            case ZK_EXPR_LOAD:
                if (depth) stack[depth - 1] = top;
                top = cache[tok.arg]; depth++;
                break;
            default: break;
            }
        }
        fe r = top;
        if (a.accumulate) r = fe_add<FS>(r, load_fe(a.out + i));
        store_fe(a.out + i, r);
    }
}

}  // namespace zkb

extern "C" int zk_expr_eval_dev(zk_ctx* ctx, int field_id, const zk_expr_token* tokens, size_t n_tokens, const uint64_t* constants_mont,
                                size_t n_constants, const zk_expr_column* cols, size_t n_cols, uint64_t out_len, unsigned out_domain_mult,
                                int accumulate, void* d_out) {
    if (!ctx || !tokens || (!constants_mont && n_constants) || (!cols && n_cols) || !d_out) { zk_set_error("expr_eval: null argument"); return ZK_ERR_INVALID; }
    if (int rc = check_field("expr_eval", field_id)) return rc;
    if (out_len == 0 || (out_len & (out_len - 1)) || out_len > ((uint64_t)1 << 30)) { zk_set_error("expr_eval: output domain size %llu is not a power of two <= 2^30", (unsigned long long)out_len); return ZK_ERR_INVALID; }
    if (out_domain_mult == 0 || (out_domain_mult & (out_domain_mult - 1)) || out_len % out_domain_mult) { zk_set_error("expr_eval: output domain multiple %u does not divide %llu", out_domain_mult, (unsigned long long)out_len); return ZK_ERR_INVALID; }
    if (n_tokens == 0 || n_tokens > (1u << 20)) { zk_set_error("expr_eval: %zu tokens outside [1, 2^20]", n_tokens); return ZK_ERR_INVALID; }
    if (n_cols > EXPR_MAX_COLS) { zk_set_error("expr_eval: %zu columns, at most %u", n_cols, EXPR_MAX_COLS); return ZK_ERR_INVALID; }
    // ---- columns: every domain is a power-of-two multiple of the same d1, at least as fine as the output's
    const uint64_t d1 = out_len / out_domain_mult;
    std::vector<ExprCol> hc(n_cols);
    for (size_t k = 0; k < n_cols; k++) {
        const zk_expr_column& c = cols[k];
        if (!c.d_evals) { zk_set_error("expr_eval: column %zu is null", k); return ZK_ERR_INVALID; }
        if (c.len == 0 || (c.len & (c.len - 1)) || c.len % out_len) { zk_set_error("expr_eval: column %zu has %llu evaluations: not a power-of-two multiple of the output domain (%llu)", k, (unsigned long long)c.len, (unsigned long long)out_len); return ZK_ERR_INVALID; }
        if (c.domain_mult == 0 || (uint64_t)c.domain_mult * d1 != c.len) { zk_set_error("expr_eval: column %zu: domain multiple %u x d1 size %llu != %llu evaluations", k, c.domain_mult, (unsigned long long)d1, (unsigned long long)c.len); return ZK_ERR_INVALID; }
        hc[k] = ExprCol{(const fe*)c.d_evals, c.len, (uint32_t)(c.len / out_len), c.domain_mult};
    }
    // ---- the program: stack discipline of PolishToken::evaluate, checked before anything runs
    unsigned sp = 0, nc = 0;
    for (size_t t = 0; t < n_tokens; t++) {
        const zk_expr_token& k = tokens[t];
        unsigned need = 0;
        int delta = 0;
        switch (k.op) {
        case ZK_EXPR_CONST: if (k.arg >= n_constants) { zk_set_error("expr_eval: token %zu: constant %u of %zu", t, k.arg, n_constants); return ZK_ERR_INVALID; } delta = 1; break;
        case ZK_EXPR_CELL: if ((k.arg & 0x7fffffffu) >= n_cols) { zk_set_error("expr_eval: token %zu: column %u of %zu", t, k.arg & 0x7fffffffu, n_cols); return ZK_ERR_INVALID; } delta = 1; break;
        case ZK_EXPR_DUP: need = 1; delta = 1; break;
        case ZK_EXPR_POW: need = 1; break;
        case ZK_EXPR_ADD: case ZK_EXPR_SUB: case ZK_EXPR_MUL: need = 2; delta = -1; break;
        case ZK_EXPR_STORE: need = 1; if (++nc > EXPR_MAX_CACHE) { zk_set_error("expr_eval: more than %u cached values", EXPR_MAX_CACHE); return ZK_ERR_INVALID; } break;
        case ZK_EXPR_LOAD: if (k.arg >= nc) { zk_set_error("expr_eval: token %zu loads cache slot %u before it is stored", t, k.arg); return ZK_ERR_INVALID; } delta = 1; break;
        default: zk_set_error("expr_eval: token %zu: unknown opcode %u", t, k.op); return ZK_ERR_INVALID;
        }
        if (sp < need) { zk_set_error("expr_eval: token %zu pops an empty stack", t); return ZK_ERR_INVALID; }   // ExprError::EmptyStack
        sp = (unsigned)((int)sp + delta);
        if (sp > EXPR_MAX_STACK) { zk_set_error("expr_eval: stack deeper than %u", EXPR_MAX_STACK); return ZK_ERR_INVALID; }
    }
    if (sp != 1) { zk_set_error("expr_eval: the program leaves %u values on the stack, not 1", sp); return ZK_ERR_INVALID; }   // assert_eq!(stack.len(), 1)

    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    // program, constants and column table in one staging buffer
    Layout lay;
    const size_t o_tok = lay.add(n_tokens * sizeof(zk_expr_token)), o_con = lay.add(std::max<size_t>(n_constants, 1) * sizeof(fe));
    const size_t o_col = lay.add(std::max<size_t>(n_cols, 1) * sizeof(ExprCol));
    if (int rc = ctx->d_expr.ensure(lay.total)) return rc;
    std::vector<uint8_t> stage(lay.total, 0);
    memcpy(stage.data() + o_tok, tokens, n_tokens * sizeof(zk_expr_token));
    if (n_constants) memcpy(stage.data() + o_con, constants_mont, n_constants * sizeof(fe));
    if (n_cols) memcpy(stage.data() + o_col, hc.data(), n_cols * sizeof(ExprCol));
    ZK_CUDA(cudaMemcpyAsync(ctx->d_expr.p, stage.data(), stage.size(), cudaMemcpyHostToDevice, st));
    ZK_CUDA(cudaStreamSynchronize(st));      // `stage` is a local
    ExprArgs a{};
    a.tokens = ctx->d_expr.at<const zk_expr_token>(o_tok);
    a.constants = ctx->d_expr.at<const fe>(o_con);
    a.cols = ctx->d_expr.at<const ExprCol>(o_col);
    a.out = (fe*)d_out; a.out_len = out_len; a.n_tokens = (uint32_t)n_tokens; a.accumulate = accumulate ? 1 : 0;
    // one resident wave of threads striding over the domain: the local-memory frames (stack + cache) are reserved per resident thread
    int sms = 0;
    ZK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, ctx->device));
    const uint64_t want = (out_len + 127) / 128;
    const unsigned blocks = (unsigned)std::min<uint64_t>(want, (uint64_t)sms * 8);
    with_field(field_id, [&](auto f) { k_expr_eval<typename decltype(f)::Dev><<<blocks, 128, 0, st>>>(a); });
    ZK_CUDA(cudaGetLastError());
    ctx->launches += 1;
    return ZK_OK;
}
