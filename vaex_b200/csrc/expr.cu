// expr.cu — device-side evaluation of simple virtual-column / filter / selection expressions and filter compaction
// (SURVEY.md section 8f row 2; the chunk-feed loop's share of section 8a row a17).
//
// Reference: per chunk the executor evaluates every expression a task needs with Python `eval` over numpy blocks
// (_BlockScope.evaluate, vaex/scopes.py:108-128), evaluates the filter to a boolean mask and compresses EVERY dependent column
// with it before the task parts see a row (ExecutorLocal.process_tasks, vaex/execution.py:516-522: `filter(v, filter_mask)`).
// Here both run on the slot's stream, so filtered / virtual-column frames never fall back to host speed:
//
//   b200_eval     a postfix program (built by vaex_b200/expression.py from the expression's Python AST, with numpy's result
//                 types decided there, NEP 50 included) is interpreted once per row: inputs are loaded with coalesced typed loads,
//                 the value stack lives in registers / local memory, every operation is a single correctly rounded IEEE operation
//                 in the node's numpy dtype class (no contraction across nodes: the interpreter's dispatch separates them), so the
//                 result is bit-identical to numpy for + - * / neg abs sqrt, the six comparisons, & | ~ on booleans, astype-style
//                 casts, and `_ordinal_values(x, hash_map_unique)` (vaex/functions.py:2454-2463: a probe of the device ordered_set).
//   b200_compact  stable stream compaction of up to 16 columns by a keep-mask: per-block counts -> one scan -> scatter.
#include <algorithm>

#include "binby.cuh"
#include "device_utils.cuh"
#include "scan.cuh"
#include "settable.cuh"

namespace b200 {
int set_fill_binner(b200_set *s, DevBinner &b); // hashset.cu
}

namespace b200 {
namespace {

constexpr int kMaxOps = 64, kMaxInputs = 8, kMaxSets = 4, kStack = 12;

union Val {
    double d;
    float s;
    long long i;
    unsigned long long u;
};

struct EvalParams {
    int nops, ninputs;
    b200_expr_op ops[kMaxOps];
    const void *in[kMaxInputs];
    int in_dtype[kMaxInputs];
    // _ordinal_values: finalized probe tables
    const SetSlot *table[kMaxSets];
    unsigned long long table_mask[kMaxSets];
    long long nan_ordinal[kMaxSets], sentinel_ordinal[kMaxSets];
    int set_dtype[kMaxSets];
    long long nrows;
    int out_dtype;
    void *out;
};

__device__ __forceinline__ Val load_input(const void *p, int dtype, long long i) {
    Val v;
    v.u = 0;
    switch (dtype) {
    case B200_F64: v.d = __ldcs(static_cast<const double *>(p) + i); break;
    case B200_F32: v.s = __ldcs(static_cast<const float *>(p) + i); break;
    case B200_I64: v.i = __ldcs(static_cast<const long long *>(p) + i); break;
    case B200_I32: v.i = __ldcs(static_cast<const int *>(p) + i); break;
    case B200_I16: v.i = __ldcs(static_cast<const short *>(p) + i); break;
    case B200_I8: v.i = __ldcs(static_cast<const signed char *>(p) + i); break;
    case B200_U64: v.u = __ldcs(static_cast<const unsigned long long *>(p) + i); break;
    case B200_U32: v.u = __ldcs(static_cast<const unsigned *>(p) + i); break;
    case B200_U16: v.u = __ldcs(static_cast<const unsigned short *>(p) + i); break;
    case B200_U8: v.u = __ldcs(static_cast<const unsigned char *>(p) + i); break;
    default: v.u = __ldcs(static_cast<const unsigned char *>(p) + i) != 0; break; // bool
    }
    return v;
}

// wrap an integer held in 64 bits to the width / signedness of `dtype` (numpy's overflow behaviour of the narrow integer types)
__device__ __forceinline__ Val wrap_int(Val v, int dtype) {
    switch (dtype) {
    case B200_I32: v.i = (int)v.u; break;
    case B200_I16: v.i = (short)v.u; break;
    case B200_I8: v.i = (signed char)v.u; break;
    case B200_U32: v.u = (unsigned)v.u; break;
    case B200_U16: v.u = (unsigned short)v.u; break;
    case B200_U8: v.u = (unsigned char)v.u; break;
    case B200_BOOL: v.u = v.u != 0; break;
    default: break;
    }
    return v;
}

__device__ __forceinline__ int dtype_class(int dtype) {
    switch (dtype) {
    case B200_F64: return B200_EXC_F64;
    case B200_F32: return B200_EXC_F32;
    case B200_I64:
    case B200_I32:
    case B200_I16:
    case B200_I8: return B200_EXC_I64;
    case B200_BOOL: return B200_EXC_BOOL;
    default: return B200_EXC_U64;
    }
}

// astype(dtype) of a value of class `from`
__device__ __forceinline__ Val cast_val(Val v, int from, int dtype) {
    const int to = dtype_class(dtype);
    Val r;
    r.u = 0;
    if (to == B200_EXC_F64) {
        switch (from) {
        case B200_EXC_F64: r.d = v.d; break;
        case B200_EXC_F32: r.d = (double)v.s; break;
        case B200_EXC_I64: r.d = __ll2double_rn(v.i); break;
        default: r.d = __ull2double_rn(v.u); break;
        }
    } else if (to == B200_EXC_F32) {
        switch (from) {
        case B200_EXC_F64: r.s = __double2float_rn(v.d); break;
        case B200_EXC_F32: r.s = v.s; break;
        case B200_EXC_I64: r.s = __ll2float_rn(v.i); break;
        default: r.s = __ull2float_rn(v.u); break;
        }
    } else if (to == B200_EXC_BOOL) {
        switch (from) {
        case B200_EXC_F64: r.u = v.d != 0.0; break;
        case B200_EXC_F32: r.u = v.s != 0.f; break;
        default: r.u = v.u != 0; break;
        }
    } else if (from == B200_EXC_F64 || from == B200_EXC_F32) {
        // floats: numpy's x86-64 casts.  int64 and uint32 take the 64-bit cvttsd2si (out of range / NaN -> INT64_MIN), then uint32
        // wraps (numpy's scalar loop; its vector loop differs out of range, DESIGN §3); uint64 takes gcc's two-step sequence; the
        // narrower types take the 32-bit cvttsd2si (out of range / NaN -> INT32_MIN), then wrap
        const double x = from == B200_EXC_F64 ? v.d : (double)v.s;
        if (dtype == B200_U64)
            r.u = f64_to_u64_x86(x);
        else if (dtype == B200_I64 || dtype == B200_U32)
            r.i = f64_to_i64_x86(x);
        else
            r.i = f64_to_i32_x86(x);
        r = wrap_int(r, dtype);
    } else {
        r.u = v.u;
        r = wrap_int(r, dtype);
    }
    return r;
}

__device__ __forceinline__ void store_output(void *out, int dtype, long long i, Val v) {
    switch (dtype) {
    case B200_F64: static_cast<double *>(out)[i] = v.d; break;
    case B200_F32: static_cast<float *>(out)[i] = v.s; break;
    case B200_I64:
    case B200_U64: static_cast<unsigned long long *>(out)[i] = v.u; break;
    case B200_I32:
    case B200_U32: static_cast<unsigned *>(out)[i] = (unsigned)v.u; break;
    case B200_I16:
    case B200_U16: static_cast<unsigned short *>(out)[i] = (unsigned short)v.u; break;
    default: static_cast<unsigned char *>(out)[i] = (unsigned char)v.u; break;
    }
}

__device__ __forceinline__ long long ordinal_lookup(const EvalParams &p, int k, Val v, int cls) {
    // the key in the set's own dtype -> canonical pattern (src/hash.hpp:50-152), NaN -> the NaN ordinal
    uint64_t raw;
    const int dt = p.set_dtype[k];
    if (dt == B200_F64) {
        if (v.d != v.d)
            return p.nan_ordinal[k];
        raw = (uint64_t)__double_as_longlong(v.d);
    } else if (dt == B200_F32) {
        if (v.s != v.s)
            return p.nan_ordinal[k];
        raw = __float_as_uint(v.s);
    } else {
        raw = v.u;
        switch (dtype_size(dt)) { // zero-extended raw bits of the storage type
        case 4: raw &= 0xffffffffull; break;
        case 2: raw &= 0xffffull; break;
        case 1: raw &= 0xffull; break;
        default: break;
        }
    }
    (void)cls;
    return set_ordinal(p.table[k], p.table_mask[k], p.sentinel_ordinal[k], key_canon(dt, raw));
}

__global__ void __launch_bounds__(256) k_eval(const __grid_constant__ EvalParams p) {
    for (long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x; row < p.nrows; row += (long long)gridDim.x * blockDim.x) {
        Val st[kStack];
        int sp = 0;
        for (int pc = 0; pc < p.nops; pc++) {
            const b200_expr_op &o = p.ops[pc];
            const int c = o.cls;
            switch (o.op) {
            case B200_EX_INPUT: st[sp++] = load_input(p.in[o.arg], p.in_dtype[o.arg], row); break;
            case B200_EX_CONST_F64:
                if (c == B200_EXC_F32)
                    st[sp].u = 0, st[sp].s = (float)o.f;
                else
                    st[sp].d = o.f;
                sp++;
                break;
            case B200_EX_CONST_I64: st[sp++].i = o.i; break;
            case B200_EX_CAST: st[sp - 1] = cast_val(st[sp - 1], c, o.arg); break;
            case B200_EX_ORDINAL: st[sp - 1].i = ordinal_lookup(p, o.arg, st[sp - 1], c); break;
            case B200_EX_NEG:
                if (c == B200_EXC_F64)
                    st[sp - 1].d = -st[sp - 1].d;
                else if (c == B200_EXC_F32)
                    st[sp - 1].s = -st[sp - 1].s;
                else
                    st[sp - 1].u = 0ull - st[sp - 1].u;
                break;
            case B200_EX_ABS:
                if (c == B200_EXC_F64)
                    st[sp - 1].d = fabs(st[sp - 1].d);
                else if (c == B200_EXC_F32)
                    st[sp - 1].s = fabsf(st[sp - 1].s);
                else if (c == B200_EXC_I64)
                    st[sp - 1].u = st[sp - 1].i < 0 ? 0ull - st[sp - 1].u : st[sp - 1].u;
                break;
            case B200_EX_SQRT:
                if (c == B200_EXC_F64)
                    st[sp - 1].d = __dsqrt_rn(st[sp - 1].d);
                else
                    st[sp - 1].s = __fsqrt_rn(st[sp - 1].s);
                break;
            case B200_EX_NOT: st[sp - 1].u = st[sp - 1].u == 0; break;
            default: { // binary operators
                const Val b = st[--sp], a = st[sp - 1];
                Val r;
                r.u = 0;
                switch (o.op) {
                case B200_EX_ADD:
                    if (c == B200_EXC_F64)
                        r.d = __dadd_rn(a.d, b.d);
                    else if (c == B200_EXC_F32)
                        r.s = __fadd_rn(a.s, b.s);
                    else
                        r.u = a.u + b.u;
                    break;
                case B200_EX_SUB:
                    if (c == B200_EXC_F64)
                        r.d = __dsub_rn(a.d, b.d);
                    else if (c == B200_EXC_F32)
                        r.s = __fsub_rn(a.s, b.s);
                    else
                        r.u = a.u - b.u;
                    break;
                case B200_EX_MUL:
                    if (c == B200_EXC_F64)
                        r.d = __dmul_rn(a.d, b.d);
                    else if (c == B200_EXC_F32)
                        r.s = __fmul_rn(a.s, b.s);
                    else
                        r.u = a.u * b.u;
                    break;
                case B200_EX_DIV:
                    if (c == B200_EXC_F64)
                        r.d = __ddiv_rn(a.d, b.d);
                    else
                        r.s = __fdiv_rn(a.s, b.s);
                    break;
                case B200_EX_AND: r.u = (a.u != 0) & (b.u != 0); break;
                case B200_EX_OR: r.u = (a.u != 0) | (b.u != 0); break;
                default: { // comparisons -> bool
                    bool lt, eq;
                    if (c == B200_EXC_F64)
                        lt = a.d < b.d, eq = a.d == b.d;
                    else if (c == B200_EXC_F32)
                        lt = a.s < b.s, eq = a.s == b.s;
                    else if (c == B200_EXC_I64)
                        lt = a.i < b.i, eq = a.i == b.i;
                    else if (c == B200_EXC_I64_U64) // a negative signed value is below every uint64
                        lt = a.i < 0 || a.u < b.u, eq = a.i >= 0 && a.u == b.u;
                    else if (c == B200_EXC_U64_I64)
                        lt = b.i >= 0 && a.u < b.u, eq = b.i >= 0 && a.u == b.u;
                    else
                        lt = a.u < b.u, eq = a.u == b.u;
                    bool gt;
                    if (c == B200_EXC_F64)
                        gt = a.d > b.d;
                    else if (c == B200_EXC_F32)
                        gt = a.s > b.s;
                    else
                        gt = !lt && !eq;
                    switch (o.op) {
                    case B200_EX_LT: r.u = lt; break;
                    case B200_EX_LE: r.u = lt || eq; break;
                    case B200_EX_GT: r.u = gt; break;
                    case B200_EX_GE: r.u = gt || eq; break;
                    case B200_EX_EQ: r.u = eq; break;
                    default: r.u = !eq; break; // NE (NaN != x is true)
                    }
                }
                }
                st[sp - 1] = r;
            }
            }
        }
        store_output(p.out, p.out_dtype, row, st[0]);
    }
}

// ---- filter compaction -----------------------------------------------------------------------------------------------------
constexpr int kCompactBlock = 1024, kMaxCompactCols = 16;

__global__ void __launch_bounds__(kCompactBlock) k_keep_count(const uint8_t *keep, long long nrows, unsigned *counts) {
    const long long i = (long long)blockIdx.x * kCompactBlock + threadIdx.x;
    const bool k = i < nrows && keep[i] != 0;
    const int n = __syncthreads_count(k);
    if (threadIdx.x == 0)
        counts[blockIdx.x] = (unsigned)n;
}

struct CompactParams {
    int ncols;
    const void *in[kMaxCompactCols];
    void *out[kMaxCompactCols];
    int isz[kMaxCompactCols];
};

__global__ void __launch_bounds__(kCompactBlock) k_compact(const uint8_t *keep, long long nrows, const unsigned *offsets, const __grid_constant__ CompactParams p) {
    __shared__ unsigned warp_counts[kCompactBlock / 32];
    const long long i = (long long)blockIdx.x * kCompactBlock + threadIdx.x;
    const bool k = i < nrows && keep[i] != 0;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned m = __ballot_sync(0xffffffffu, k);
    if (lane == 0)
        warp_counts[warp] = __popc(m);
    __syncthreads();
    if (warp == 0) { // exclusive scan of the 32 warp counts
        unsigned x = warp_counts[lane], v = x;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o)
                x += y;
        }
        warp_counts[lane] = x - v;
    }
    __syncthreads();
    if (!k)
        return;
    const unsigned long long pos = (unsigned long long)offsets[blockIdx.x] + warp_counts[warp] + __popc(m & ((1u << lane) - 1u));
    for (int c = 0; c < p.ncols; c++) {
        store1_raw(p.out[c], p.isz[c], pos, load1_raw(p.in[c], p.isz[c], i));
    }
}

} // namespace
} // namespace b200

using namespace b200;

extern "C" int b200_eval(b200_ctx *ctx, int slot, const b200_expr_op *prog, int nops, const b200_expr_input *inputs, int ninputs, b200_set *const *sets,
                         int nsets, int64_t nrows, int memspace, int out_dtype, void *out_device) {
    if (!prog || nops < 1 || nops > kMaxOps || ninputs < 0 || ninputs > kMaxInputs || nsets < 0 || nsets > kMaxSets || nrows < 0 || out_dtype < 0 ||
        out_dtype >= B200_NDTYPE || (nrows && !out_device)) {
        set_error("b200_eval: invalid argument (%d ops, %d inputs, %d sets)", nops, ninputs, nsets);
        return B200_ERR_INVALID;
    }
    CallFrame call(ctx, slot, memspace, 0, "b200_eval");
    B200_CHECK(call.rc);
    if (!nrows)
        return B200_OK;
    EvalParams p;
    memset(&p, 0, sizeof p);
    // validate the program: stack discipline, operand indices (a malformed program must not read out of bounds on the device)
    int depth = 0, maxdepth = 0;
    for (int i = 0; i < nops; i++) {
        const b200_expr_op &o = prog[i];
        int pop = 0, push = 1;
        switch (o.op) {
        case B200_EX_INPUT:
            if (o.arg < 0 || o.arg >= ninputs) {
                set_error("b200_eval: op %d reads input %d of %d", i, o.arg, ninputs);
                return B200_ERR_INVALID;
            }
            break;
        case B200_EX_CONST_F64:
        case B200_EX_CONST_I64: break;
        case B200_EX_ORDINAL:
            if (o.arg < 0 || o.arg >= nsets) {
                set_error("b200_eval: op %d uses set %d of %d", i, o.arg, nsets);
                return B200_ERR_INVALID;
            }
            pop = 1;
            break;
        case B200_EX_CAST:
            if (o.arg < 0 || o.arg >= B200_NDTYPE) {
                set_error("b200_eval: op %d casts to unknown dtype %d", i, o.arg);
                return B200_ERR_INVALID;
            }
            pop = 1;
            break;
        case B200_EX_NEG:
        case B200_EX_ABS:
        case B200_EX_SQRT:
        case B200_EX_NOT: pop = 1; break;
        default:
            if (o.op < 0 || o.op > B200_EX_ORDINAL) {
                set_error("b200_eval: unknown opcode %d", o.op);
                return B200_ERR_INVALID;
            }
            pop = 2;
            break;
        }
        if (depth < pop) {
            set_error("b200_eval: stack underflow at op %d", i);
            return B200_ERR_INVALID;
        }
        depth += push - pop;
        maxdepth = std::max(maxdepth, depth);
    }
    if (depth != 1 || maxdepth > kStack) {
        set_error("b200_eval: the program leaves %d values (stack depth %d, limit %d)", depth, maxdepth, kStack);
        return B200_ERR_INVALID;
    }
    for (int k = 0; k < ninputs; k++) {
        if (inputs[k].dtype < 0 || inputs[k].dtype >= B200_NDTYPE || !inputs[k].data) {
            set_error("b200_eval: input %d: %s", k, inputs[k].data ? "unknown dtype" : "data not set");
            return B200_ERR_INVALID;
        }
        call.plan(inputs[k].data, (size_t)nrows * dtype_size(inputs[k].dtype));
    }
    B200_CHECK(call.commit());
    p.nops = nops;
    p.ninputs = ninputs;
    memcpy(p.ops, prog, sizeof(b200_expr_op) * nops);
    for (int k = 0; k < ninputs; k++) {
        p.in[k] = call.dev(inputs[k].data);
        p.in_dtype[k] = inputs[k].dtype;
    }
    for (int k = 0; k < nsets; k++) {
        DevBinner b;
        memset(&b, 0, sizeof b);
        B200_CHECK(set_fill_binner(sets[k], b));
        p.table[k] = b.table;
        p.table_mask[k] = b.table_mask;
        p.nan_ordinal[k] = b.nan_ordinal;
        p.sentinel_ordinal[k] = b.sentinel_ordinal;
        p.set_dtype[k] = b200_set_dtype(sets[k]);
    }
    p.nrows = nrows;
    p.out_dtype = out_dtype;
    p.out = out_device;
    const long long want = (nrows + 255) / 256;
    const int blocks = (int)std::min<long long>(want, (long long)ctx->sm_count * 16);
    k_eval<<<blocks, 256, 0, call.st>>>(p);
    B200_CUDA(cudaGetLastError());
    return call.finish();
}

extern "C" int b200_compact(b200_ctx *ctx, int slot, const uint8_t *keep, int ncols, const void *const *cols, const int32_t *dtypes, int64_t nrows,
                            int memspace, void *const *outs_device, int64_t *count_out) {
    if (ncols < 0 || ncols > kMaxCompactCols || nrows < 0 || !count_out || (nrows && !keep) || (ncols && (!cols || !dtypes || !outs_device))) {
        set_error("b200_compact: invalid argument");
        return B200_ERR_INVALID;
    }
    CallFrame call(ctx, slot, memspace, 0, "b200_compact");
    B200_CHECK(call.rc);
    *count_out = 0;
    if (!nrows)
        return B200_OK;
    cudaStream_t st = call.st;
    const unsigned nblk = (unsigned)((nrows + kCompactBlock - 1) / kCompactBlock);
    call.plan(keep, (size_t)nrows);
    CompactParams p;
    memset(&p, 0, sizeof p);
    p.ncols = ncols;
    for (int c = 0; c < ncols; c++) {
        if (dtypes[c] < 0 || dtypes[c] >= B200_NDTYPE || !cols[c] || !outs_device[c]) {
            set_error("b200_compact: column %d is invalid", c);
            return B200_ERR_INVALID;
        }
        p.isz[c] = dtype_size(dtypes[c]);
        call.plan(cols[c], (size_t)nrows * p.isz[c]);
    }
    B200_CHECK(call.commit());
    for (int c = 0; c < ncols; c++) {
        p.in[c] = call.dev(cols[c]);
        p.out[c] = outs_device[c];
    }
    const uint8_t *d_keep = static_cast<const uint8_t *>(call.dev(keep));
    DevBuf<unsigned> d_counts;
    B200_CHECK(d_counts.alloc(ctx, (size_t)nblk * 4 + 16, "b200_compact", st));
    unsigned long long *d_total;
    B200_CHECK(call.out(count_out, 8, false, &d_total));
    k_keep_count<<<nblk, kCompactBlock, 0, st>>>(d_keep, nrows, d_counts);
    k_scan_u32<<<1, 1024, 0, st>>>(d_counts, nblk, d_total);
    if (ncols)
        k_compact<<<nblk, kCompactBlock, 0, st>>>(d_keep, nrows, d_counts, p);
    B200_CUDA(cudaGetLastError());
    return call.finish();
}
