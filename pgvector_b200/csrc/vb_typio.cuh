// vb_typio.cuh -- host machinery the type I/O calls share (vb_text.cu, vb_binary.cu): offsets from per-row
// counts, and the two-slot pinned staging that pipelines the host variants.
#pragma once

#include "vb_common.cuh"

namespace vb {

// row_off[0] = 0, row_off[1 + i] = sum of count[0 .. i] (device arrays, on the library stream)
int offsets_from_counts(const int64_t* count, int64_t n, int64_t* row_off);

// the sparse table calls' check of n >= 1 device CSR rows, with their texts (vb_sparse.cu): one read of 24 bytes;
// *total (optional) is off[n]
int sparse_csr_check_dev(const char* what, int dim, int64_t n, const int64_t* off, const int32_t* idx,
                         int64_t* total = nullptr);

// pinned staging of the pipelined host variants: two slots, each with an input and an output buffer
struct Staging {
    void* in[2] = {nullptr, nullptr};
    void* out[2] = {nullptr, nullptr};
    size_t in_bytes[2] = {0, 0}, out_bytes[2] = {0, 0};
    cudaEvent_t done[2] = {nullptr, nullptr};
};
Staging& staging();
// *buf holds at least `bytes` pinned bytes afterwards (contents not kept)
int pinned_grow(void** buf, size_t* have, size_t bytes);

// Runs nch chunks through the two staging slots: enqueue(c, k) stages chunk c into slot k and enqueues its work and
// its copy back; finish(c, k) runs once slot k's copy back has landed.  While the device works on chunk c, the host
// finishes chunk c - 1 and then stages chunk c + 1.  The first failing finish ends the call, after the chunk still in
// flight has landed (its buffers are about to go).  The caller sizes the slots with pinned_grow first.
template <typename Enqueue, typename Finish>
int pipeline_chunks(int64_t nch, Enqueue enqueue, Finish finish) {
    Staging& sg = staging();
    cudaStream_t s = ctx().stream;
    for (int k = 0; k < 2 && k < nch; ++k)
        if (!sg.done[k]) VB_CUDA(cudaEventCreateWithFlags(&sg.done[k], cudaEventDisableTiming));
    for (int64_t c = 0; c < nch; ++c) {
        const int k = (int)(c & 1);
        // slot k's last user, chunk c - 2, was finished (its event waited for) in the previous iteration
        VB_TRY(enqueue(c, k));
        VB_CUDA(cudaEventRecord(sg.done[k], s));
        if (c >= 1) {
            VB_CUDA(cudaEventSynchronize(sg.done[k ^ 1]));
            const int rc = finish(c - 1, k ^ 1);
            if (rc != VB_OK) {
                cudaStreamSynchronize(s);
                return rc;
            }
        }
    }
    if (nch == 0) return VB_OK;
    const int k = (int)((nch - 1) & 1);
    VB_CUDA(cudaEventSynchronize(sg.done[k]));
    return finish(nch - 1, k);
}

}  // namespace vb
