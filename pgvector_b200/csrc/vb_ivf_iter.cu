// vb_ivf_iter.cu -- ivfflat.iterative_scan on the device (src/ivfscan.c:123-187 GetScanItems, :400-406 the loop of
// ivfflatgettuple that calls it again while lists remain).
//
// A scan handle (vb_ivf_scan, vb_ivf.cu) keeps per query the lists of its current group of `probes` lists, their
// candidate distances, the reference's listIndex and a cursor into the group's sorted sequence (the key of the last
// element returned and how many were returned).  A vb_ivf_scan_next call is a fixed sequence of launches:
//   1. ivf_iter_advance_kernel (here): a query whose group is used up moves to its next non-empty group;
//   2. ivf_build_chunks_kernel with the handle's `active` mask: candidate offsets and scan chunks of the queries that moved;
//   3. scan_kernel (the LDG chunk scan) over those chunks: the chunk count lives on the device, so a call in which no
//      query moves does no scan work;
//   4. segment_topk_floor_kernel: the next `page` keys of every query above its cursor, cursor advanced;
//   5. ivf_finish_kernel: positions to heap ids and float8 distances;
//   6. one copy of ids, distances and counts back to the host.
#include "vb_common.cuh"

namespace vb {

// One warp per query.  A query still draining its group (returned < seg_len) is left alone.  Otherwise the warp walks
// forward from listIndex over groups of `probes` consecutive lists of the probe order, summing list lengths from
// list_off, to the first non-empty group (the reference's while loop skips empty ones the same way: GetScanItems
// adds nothing and the loop calls it again).  That group's lists go to glists (-1 padded), listIndex moves past it,
// the cursor is reset and the query is marked active so that step 2 builds its scan.  When no non-empty group
// remains, listIndex = max_probes and seg_len = 0: the query is exhausted and every later page of it is empty.
__global__ void ivf_iter_advance_kernel(int64_t nq, int probes, int max_probes, const int32_t* __restrict__ probe_lists,
                                        const int64_t* __restrict__ list_off, int32_t* __restrict__ glists,
                                        int32_t* __restrict__ list_index, int32_t* __restrict__ returned,
                                        int32_t* __restrict__ seg_len, int32_t* __restrict__ active) {
    const int64_t q = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (q >= nq) return;
    if (returned[q] < seg_len[q]) {
        if (lane == 0) active[q] = 0;
        return;
    }
    const int32_t* pl = probe_lists + q * max_probes;
    int li = list_index[q], g0 = li;
    int64_t total = 0;
    while (li < max_probes) {
        g0 = li;
        const int end = min(li + probes, max_probes);
        int64_t s = 0;
        for (int j = li + lane; j < end; j += 32) {
            const int l = pl[j];
            if (l >= 0) s += list_off[l + 1] - list_off[l];
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        li = end;
        if (s > 0) {
            total = s;
            break;
        }
    }
    if (total > 0)
        for (int j = lane; j < probes; j += 32) glists[q * probes + j] = g0 + j < li ? pl[g0 + j] : -1;
    if (lane == 0) {
        list_index[q] = li;
        returned[q] = 0;
        active[q] = total > 0 ? 1 : 0;
        if (total == 0) seg_len[q] = 0;
    }
}

int launch_ivf_iter_advance(int64_t nq, int probes, int max_probes, const int32_t* probe_lists, const int64_t* list_off,
                            int32_t* glists, int32_t* list_index, int32_t* returned, int32_t* seg_len, int32_t* active) {
    if (nq <= 0) return VB_OK;
    const int threads = 256;
    const int64_t blocks = (nq * 32 + threads - 1) / threads;
    ivf_iter_advance_kernel<<<(unsigned)blocks, threads, 0, ctx().stream>>>(nq, probes, max_probes, probe_lists, list_off, glists,
                                                                           list_index, returned, seg_len, active);
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

// A filtered handle (vb_ivf_scan_begin_filtered) keeps the offset tables of its row filters side by side: list l of
// filter f is the run foff[f lists + l] .. foff[f lists + l + 1] of the concatenated allowed positions.  Renaming every
// probed list to that virtual list is all the advance, chunk and finish kernels need: they read the filter's runs
// through the list_off they already take, so they are the same kernels for both kinds of handle.
__global__ void ivf_filter_lists_kernel(int64_t n, int max_probes, int lists, const int32_t* __restrict__ fq, int32_t* __restrict__ probe_lists) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t l = probe_lists[i];
    if (l >= 0) probe_lists[i] = fq[i / max_probes] * lists + l;
}

int launch_ivf_filter_lists(int64_t nq, int max_probes, int lists, const int32_t* fq_dev, int32_t* probe_lists) {
    const int64_t n = nq * max_probes;
    if (n <= 0) return VB_OK;
    ivf_filter_lists_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx().stream>>>(n, max_probes, lists, fq_dev, probe_lists);
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

}  // namespace vb
