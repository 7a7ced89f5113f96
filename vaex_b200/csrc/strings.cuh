// strings.cuh — staging of string columns in the arrow large_string layout (int64 offsets[nrows + 1] into a byte buffer, plus an
// optional byte mask), shared by the string key sets (hashset.cu) and the string list aggregator (list.cu via api.cu).
#pragma once
#include "common.cuh"

namespace b200 {

// string columns staged for one call: offsets (device), bytes (device, starting at offsets[0]), masks.  The string of row r is
// bytes[offsets[r] - base, offsets[r + 1] - base).
struct StrInput {
    const long long *offsets = nullptr;
    const unsigned char *bytes = nullptr;
    const uint8_t *masks = nullptr;
    long long base = 0, nbytes = 0;
};

// phase 1: read offsets[0] and offsets[nrows] (a short synchronous copy when the offsets live on the device) and plan the three
// columns on `call`; the byte column is planned as the range the call uses, so a sliced arrow array stages only its own bytes
inline int plan_strings(CallFrame &call, const int64_t *offsets, const uint8_t *bytes, const uint8_t *masks, int64_t nrows, StrInput *in) {
    long long first = 0, last = 0;
    if (nrows) {
        if (call.on_device(offsets)) {
            B200_CUDA(cudaMemcpyAsync(&first, offsets, 8, cudaMemcpyDeviceToHost, call.st));
            B200_CUDA(cudaMemcpyAsync(&last, offsets + nrows, 8, cudaMemcpyDeviceToHost, call.st));
            B200_CUDA(cudaStreamSynchronize(call.st));
        } else {
            first = offsets[0], last = offsets[nrows];
        }
    }
    if (last < first) {
        set_error("string column: offsets[nrows] (%lld) < offsets[0] (%lld)", last, first);
        return B200_ERR_INVALID;
    }
    in->base = first;
    in->nbytes = last - first;
    call.plan(offsets, (size_t)(nrows + 1) * 8);
    if (in->nbytes)
        call.plan(bytes + first, (size_t)in->nbytes);
    if (masks)
        call.plan(masks, (size_t)nrows);
    return B200_OK;
}

// phase 2, after call.commit(): the device pointers.  Device columns are used in place (CallFrame::dev returns them unchanged), so
// `bytes` + base is the row range's first byte in every memspace.
inline void resolve_strings(const CallFrame &call, const int64_t *offsets, const uint8_t *bytes, const uint8_t *masks, StrInput *in) {
    in->offsets = static_cast<const long long *>(call.dev(offsets));
    in->bytes = in->nbytes ? static_cast<const unsigned char *>(call.dev(bytes + in->base)) : bytes;
    in->masks = masks ? static_cast<const uint8_t *>(call.dev(masks)) : nullptr;
}

// both phases for a call that stages nothing else
inline int stage_strings(CallFrame &call, const int64_t *offsets, const uint8_t *bytes, const uint8_t *masks, int64_t nrows, StrInput *in) {
    B200_CHECK(plan_strings(call, offsets, bytes, masks, nrows, in));
    B200_CHECK(call.commit());
    resolve_strings(call, offsets, bytes, masks, in);
    return B200_OK;
}

// 16 bytes of the byte stream that starts `mis` (1..15) bytes into the aligned word `a`, followed by `b`
__device__ __forceinline__ uint4 shift16(uint4 a, uint4 b, int mis) {
    const int q = mis >> 2;
    const unsigned r = (unsigned)(mis & 3) * 8;
    const unsigned w0 = q == 0 ? a.x : q == 1 ? a.y : q == 2 ? a.z : a.w;
    const unsigned w1 = q == 0 ? a.y : q == 1 ? a.z : q == 2 ? a.w : b.x;
    const unsigned w2 = q == 0 ? a.z : q == 1 ? a.w : q == 2 ? b.x : b.y;
    const unsigned w3 = q == 0 ? a.w : q == 1 ? b.x : q == 2 ? b.y : b.z;
    const unsigned w4 = q == 0 ? b.x : q == 1 ? b.y : q == 2 ? b.z : b.w;
    return make_uint4(__funnelshift_r(w0, w1, r), __funnelshift_r(w1, w2, r), __funnelshift_r(w2, w3, r), __funnelshift_r(w3, w4, r));
}

// G threads copy one string: single bytes up to the first 16-byte boundary of the destination, then 16-byte stores (16-byte loads
// when source and destination are equally misaligned, else two aligned loads and a funnel shift), then the last bytes.  The source
// reads may run up to 16 bytes past the string: the pool is allocated with that much slack.
template <int G>
__device__ __forceinline__ void copy_string(char *dst, const char *src, long long len, int lane) {
    const long long head = min(len, (long long)((16 - (reinterpret_cast<uintptr_t>(dst) & 15)) & 15));
    for (long long c = lane; c < head; c += G)
        dst[c] = src[c];
    const long long chunks = (len - head) >> 4;
    uint4 *d = reinterpret_cast<uint4 *>(dst + head);
    const char *s = src + head;
    const int mis = (int)(reinterpret_cast<uintptr_t>(s) & 15);
    const uint4 *s4 = reinterpret_cast<const uint4 *>(s - mis);
    if (mis == 0) {
        for (long long c = lane; c < chunks; c += G)
            d[c] = __ldg(s4 + c);
    } else {
        for (long long c = lane; c < chunks; c += G)
            d[c] = shift16(__ldg(s4 + c), __ldg(s4 + c + 1), mis);
    }
    for (long long c = head + chunks * 16 + lane; c < len; c += G)
        dst[c] = src[c];
}

} // namespace b200
