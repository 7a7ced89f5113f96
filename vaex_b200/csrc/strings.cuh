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

} // namespace b200
