// vb_runtime.cu -- process-wide runtime of libvecb200: device binding, streams,
// scratch, pinned staging, resident row tables, query image upload.
#include "vb_common.cuh"

#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <algorithm>
#include <vector>

namespace vb {

// grows to hold the longest message: the type input errors echo their whole literal (16000 elements, ~250 kB)
static thread_local std::string g_err;
static thread_local std::string g_err_detail;
thread_local int g_last_status = 0;

void set_error(const char* fmt, ...) {
    va_list ap, ap2;
    va_start(ap, fmt);
    va_copy(ap2, ap);
    const int len = vsnprintf(nullptr, 0, fmt, ap);
    va_end(ap);
    std::string msg(len > 0 ? (size_t)len : 0, '\0');   // formatted apart: an argument may be the old message
    if (len > 0) vsnprintf(&msg[0], (size_t)len + 1, fmt, ap2);
    va_end(ap2);
    g_err.swap(msg);
    g_err_detail.clear();
}
// the errdetail of the error just set (the type input errors have one)
void set_error_detail(const char* detail) { g_err_detail = detail; }
const char* last_error() { return g_err.c_str(); }
const char* last_error_detail() { return g_err_detail.c_str(); }
int prof_read(int which, double* total_ms, int64_t* launches);
void prof_set(bool on);

Context& ctx() {
    static Context c;
    return c;
}

int require_init() {
    if (!ctx().inited) {
        // lazy init on device 0 (a backend's first call), still no CPU fallback
        int rc = vb_init(0);
        if (rc != VB_OK) return rc;
    }
    return VB_OK;
}

Scratch::Scratch(const char* fn) : fn_(fn), outer_(ctx().scratch), top_(outer_ ? outer_->top_ : 0) { ctx().scratch = this; }

Scratch::~Scratch() {
    Context& c = ctx();
    for (void* p : owned_) cudaFreeAsync(p, c.stream);
    c.scratch = outer_;
    if (outer_ || c.arena_peak <= c.arena_bytes) return;
    // the call needed more than the arena holds: grow it to the peak, with head-room so steady-state calls stop
    // reallocating (after the work that still reads the old arena)
    cudaStreamSynchronize(c.stream);
    cudaFree(c.arena);
    c.arena = nullptr;
    c.arena_bytes = 0;
    const size_t want = c.arena_peak + c.arena_peak / 4;
    if (cudaMalloc(&c.arena, want) == cudaSuccess) {
        c.arena_bytes = want;
    } else {
        // the arena stays empty and forgets the peak: the next call takes one-off allocations and grows the arena to
        // its own peak, so one oversized call does not make every later one allocate
        cudaGetLastError();
        c.arena = nullptr;
        c.arena_peak = 0;
    }
}

int Scratch::take(size_t bytes, void** out) {
    Context& c = ctx();
    if (c.scratch != this) {
        set_error("%s: scratch taken from an enclosing call while an inner call's scratch is live", fn_ ? fn_ : "libvecb200");
        return VB_ESTATE;
    }
    const size_t end = top_ + ((std::max<size_t>(bytes, 16) + 255) & ~(size_t)255);
    if (end <= c.arena_bytes) *out = c.arena + top_;
    else VB_TRY(own(bytes, out));   // (a range that could not be had does not raise the peak)
    top_ = end;
    c.arena_peak = std::max(c.arena_peak, end);
    return VB_OK;
}

int Scratch::own(size_t bytes, void** out) {
    void* p = nullptr;
    const cudaError_t e = cudaMallocAsync(&p, bytes ? bytes : 16, ctx().stream);
    if (e != cudaSuccess) {
        cudaGetLastError();
        set_error("%s: allocation of %zu bytes of device memory failed: %s", fn_ ? fn_ : "libvecb200", bytes, cudaGetErrorString(e));
        return VB_ENOMEM;
    }
    owned_.push_back(p);
    *out = p;
    return VB_OK;
}

static int pinned_impl(void** buf, size_t* have, size_t bytes, void** out) {
    if (*have < bytes) {
        if (*buf) {
            VB_CUDA(cudaDeviceSynchronize());
            VB_CUDA(cudaFreeHost(*buf));
            *buf = nullptr;
            *have = 0;
        }
        cudaError_t e = cudaMallocHost(buf, bytes);
        if (e != cudaSuccess) {
            set_error("cudaMallocHost(%zu) failed: %s", bytes, cudaGetErrorString(e));
            return VB_ENOMEM;
        }
        *have = bytes;
    }
    *out = *buf;
    return VB_OK;
}
int pinned_buffer(size_t bytes, void** out) { return pinned_impl(&ctx().pinned, &ctx().pinned_bytes, bytes, out); }
int pinned_buffer2(size_t bytes, void** out) { return pinned_impl(&ctx().pinned2, &ctx().pinned2_bytes, bytes, out); }

// ----------------------------------------------------------------------------- tables

int table_reserve(Table& t, int64_t rows) {
    if (rows <= t.cap) return VB_OK;
    int64_t ncap = std::max<int64_t>(rows, t.cap + t.cap / 2);
    uint8_t* nd = nullptr;
    size_t bytes = (size_t)ncap * t.stride + 16;
    cudaError_t e = cudaMalloc(&nd, bytes);
    if (e != cudaSuccess) {
        set_error("cudaMalloc(%zu) for table failed: %s", bytes, cudaGetErrorString(e));
        return VB_ENOMEM;
    }
    if (t.d) {
        VB_CUDA(cudaMemcpyAsync(nd, t.d, (size_t)t.n * t.stride, cudaMemcpyDeviceToDevice, ctx().stream));
        VB_CUDA(cudaStreamSynchronize(ctx().stream));
        VB_CUDA(cudaFree(t.d));
    }
    t.d = nd;
    t.cap = ncap;
    return VB_OK;
}

// Host rows -> pinned staging -> HBM, double buffered so the memcpy into staging of block i+1
// overlaps the DMA of block i.  Rows land at the padded stride (pad bytes zeroed).
int table_append_host(Table& t, const void* rows, int64_t n) {
    if (n <= 0) return VB_OK;
    VB_TRY(table_reserve(t, t.n + n));
    Context& c = ctx();
    const size_t raw = raw_row_bytes(t.elem, t.dim);
    uint8_t* dst = t.d + (size_t)t.n * t.stride;
    if (raw != t.stride) VB_CUDA(cudaMemsetAsync(dst, 0, (size_t)n * t.stride, c.stream));
    const size_t block_bytes = 32u << 20;
    const int64_t rows_per_block = std::min<int64_t>(1 << 20, std::max<int64_t>(1, (int64_t)(block_bytes / raw)));
    void *p0, *p1;
    VB_TRY(pinned_buffer((size_t)rows_per_block * raw, &p0));
    VB_TRY(pinned_buffer2((size_t)rows_per_block * raw, &p1));
    void* stage[2] = {p0, p1};
    cudaEvent_t ev[2];
    VB_CUDA(cudaEventCreateWithFlags(&ev[0], cudaEventDisableTiming));
    VB_CUDA(cudaEventCreateWithFlags(&ev[1], cudaEventDisableTiming));
    int b = 0;
    for (int64_t r = 0; r < n; r += rows_per_block, b ^= 1) {
        int64_t m = std::min(rows_per_block, n - r);
        VB_CUDA(cudaEventSynchronize(ev[b]));  // staging buffer b free again
        memcpy(stage[b], (const uint8_t*)rows + (size_t)r * raw, (size_t)m * raw);
        VB_CUDA(cudaMemcpy2DAsync(dst + (size_t)r * t.stride, t.stride, stage[b], raw, raw, (size_t)m,
                                  cudaMemcpyHostToDevice, c.stream));
        VB_CUDA(cudaEventRecord(ev[b], c.stream));
    }
    VB_CUDA(cudaStreamSynchronize(c.stream));
    cudaEventDestroy(ev[0]);
    cudaEventDestroy(ev[1]);
    t.n += n;
    return VB_OK;
}

int table_append_dev(Table& t, const void* rows_dev, int64_t n) {
    if (n <= 0) return VB_OK;
    VB_TRY(table_reserve(t, t.n + n));
    Context& c = ctx();
    const size_t raw = raw_row_bytes(t.elem, t.dim);
    uint8_t* dst = t.d + (size_t)t.n * t.stride;
    if (raw == t.stride) {
        VB_CUDA(cudaMemcpyAsync(dst, rows_dev, (size_t)n * raw, cudaMemcpyDeviceToDevice, c.stream));
    } else {
        VB_CUDA(cudaMemsetAsync(dst, 0, (size_t)n * t.stride, c.stream));
        // 2-D copies are issued in slabs: the height of one cudaMemcpy2D is kept well inside driver limits
        const int64_t slab = 1 << 20;
        for (int64_t r = 0; r < n; r += slab) {
            int64_t m = std::min(slab, n - r);
            VB_CUDA(cudaMemcpy2DAsync(dst + (size_t)r * t.stride, t.stride, (const uint8_t*)rows_dev + (size_t)r * raw, raw, raw, (size_t)m,
                                      cudaMemcpyDeviceToDevice, c.stream));
        }
    }
    t.n += n;
    return VB_OK;
}

void table_free(Table& t) {
    if (t.d) cudaFree(t.d);
    t.d = nullptr;
    t.n = t.cap = 0;
}

// ----------------------------------------------------------------------------- query images

// raw query rows (device) -> padded image; halfvec widened to fp32 (exact, like HalfToFloat4)
__global__ void query_image_kernel(int elem, int dim, const uint8_t* __restrict__ raw, size_t raw_stride,
                                   uint8_t* __restrict__ img, size_t img_stride, int64_t nq) {
    const int64_t q = blockIdx.x;
    if (q >= nq) return;
    const uint8_t* src = raw + (size_t)q * raw_stride;
    uint8_t* dst = img + (size_t)q * img_stride;
    if (elem == VB_BIT) {
        const int nb = (dim + 7) / 8;
        for (int i = threadIdx.x; i < (int)img_stride; i += blockDim.x) dst[i] = i < nb ? src[i] : 0;
    } else {
        const int nf = (int)(img_stride / 4);
        float* d = reinterpret_cast<float*>(dst);
        for (int i = threadIdx.x; i < nf; i += blockDim.x) {
            float v = 0.f;
            if (i < dim) {
                if (elem == VB_VECTOR) v = reinterpret_cast<const float*>(src)[i];
                else v = __half2float(reinterpret_cast<const __half*>(src)[i]);
            }
            d[i] = v;
        }
    }
}

int upload_queries(Scratch& sc, int elem, int dim, const void* queries, int64_t nq, bool host, void** out_dev,
                   size_t* qstride) {
    Context& c = ctx();
    const size_t raw = raw_row_bytes(elem, dim);
    const size_t pad = padded_row_bytes(elem, dim);
    // image stride: fp32 per element for vector/halfvec (halfvec padded to 8 elements -> 32 B of floats)
    const size_t img = elem == VB_HALFVEC ? pad * 2 : pad;
    *qstride = img;
    if (!host && elem != VB_HALFVEC && raw == pad) {
        *out_dev = const_cast<void*>(queries);  // already in image layout
        return VB_OK;
    }
    void* d_img;
    VB_TRY(sc.take(img * (size_t)nq + raw * (size_t)nq + 32, &d_img));
    uint8_t* d_raw = (uint8_t*)d_img + ((img * (size_t)nq + 15) & ~(size_t)15);
    const uint8_t* src_dev = (const uint8_t*)queries;
    if (host) {
        // a caller buffer that is already page-locked (cudaHostAlloc / cudaHostRegister) is DMA'd in place;
        // pageable memory goes through the library's pinned staging buffer
        cudaPointerAttributes attr;
        const void* src = queries;
        if (cudaPointerGetAttributes(&attr, queries) != cudaSuccess || attr.type != cudaMemoryTypeHost) {
            cudaGetLastError();   // clear the "not a registered pointer" status of older drivers
            void* pin;
            VB_TRY(pinned_buffer(raw * (size_t)nq, &pin));
            memcpy(pin, queries, raw * (size_t)nq);
            src = pin;
        }
        if (elem != VB_HALFVEC && raw == pad) {
            // rows are already in image layout: DMA straight into the image, no repack kernel
            VB_CUDA(cudaMemcpyAsync(d_img, src, raw * (size_t)nq, cudaMemcpyHostToDevice, c.stream));
            *out_dev = d_img;
            return VB_OK;
        }
        VB_CUDA(cudaMemcpyAsync(d_raw, src, raw * (size_t)nq, cudaMemcpyHostToDevice, c.stream));
        src_dev = d_raw;
    }
    query_image_kernel<<<(unsigned)nq, 128, 0, c.stream>>>(elem, dim, src_dev, raw, (uint8_t*)d_img, img, nq);
    VB_CUDA(cudaGetLastError());
    count_launch();
    *out_dev = d_img;
    return VB_OK;
}

const char* last_error();

// ----------------------------------------------------------------------------- profiling brackets
struct ProfSpan {
    int which;
    cudaEvent_t a, b;
};
static bool g_prof_on = false;
static std::vector<ProfSpan> g_spans;
static std::vector<cudaEvent_t> g_event_pool;

static cudaEvent_t prof_event() {
    if (!g_event_pool.empty()) {
        cudaEvent_t e = g_event_pool.back();
        g_event_pool.pop_back();
        return e;
    }
    cudaEvent_t e;
    cudaEventCreate(&e);
    return e;
}
void prof_begin(int which) {
    if (!g_prof_on) return;
    ProfSpan s{which, prof_event(), prof_event()};
    cudaEventRecord(s.a, ctx().stream);
    g_spans.push_back(s);
}
void prof_end(int which) {
    if (!g_prof_on) return;
    for (size_t i = g_spans.size(); i-- > 0;)
        if (g_spans[i].which == which) {
            cudaEventRecord(g_spans[i].b, ctx().stream);
            return;
        }
}
int prof_read(int which, double* total_ms, int64_t* launches) {
    VB_CUDA(cudaStreamSynchronize(ctx().stream));
    double ms = 0;
    int64_t n = 0;
    std::vector<ProfSpan> keep;
    for (auto& s : g_spans) {
        if (s.which != which) {
            keep.push_back(s);
            continue;
        }
        float f = 0;
        if (cudaEventElapsedTime(&f, s.a, s.b) == cudaSuccess) {
            ms += f;
            ++n;
        }
        g_event_pool.push_back(s.a);
        g_event_pool.push_back(s.b);
    }
    g_spans.swap(keep);
    if (total_ms) *total_ms = ms;
    if (launches) *launches = n;
    return VB_OK;
}
void prof_set(bool on) { g_prof_on = on; }

}  // namespace vb

// ----------------------------------------------------------------------------- C ABI: runtime

extern "C" {

int vb_abi_version(void) { return VB_ABI_VERSION; }

const char* vb_last_error(void) { return vb::last_error(); }
const char* vb_last_error_detail(void) { return vb::last_error_detail(); }

int vb_init(int device) {
    vb::Context& c = vb::ctx();
    if (c.inited && c.device == device) return VB_OK;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        vb::set_error("no CUDA device: %s (libvecb200 has no CPU fallback)", e == cudaSuccess ? "count is 0" : cudaGetErrorString(e));
        return VB_ENODEVICE;
    }
    if (device < 0 || device >= n) {
        vb::set_error("device %d out of range (have %d)", device, n);
        return VB_ENODEVICE;
    }
    cudaDeviceProp p;
    if (cudaGetDeviceProperties(&p, device) != cudaSuccess || p.major != 9 || p.minor != 0) {
        vb::set_error("device %d is sm_%d%d; libvecb200 is built for sm_90a only", device, p.major, p.minor);
        return VB_ENODEVICE;
    }
    if (cudaSetDevice(device) != cudaSuccess) {
        vb::set_error("cudaSetDevice(%d) failed", device);
        return VB_ENODEVICE;
    }
    if (c.inited) vb_shutdown();
    c.device = device;
    c.sm_count = p.multiProcessorCount;
    if (cudaStreamCreateWithFlags(&c.stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithFlags(&c.copy_stream, cudaStreamNonBlocking) != cudaSuccess) {
        vb::set_error("stream creation failed");
        return VB_ECUDA;
    }
    c.inited = true;
    return VB_OK;
}

int vb_shutdown(void) {
    vb::Context& c = vb::ctx();
    if (!c.inited) return VB_OK;
    cudaDeviceSynchronize();
    if (c.arena) cudaFree(c.arena);
    c.arena = nullptr;
    c.arena_bytes = c.arena_peak = 0;
    if (c.pinned) cudaFreeHost(c.pinned);
    if (c.pinned2) cudaFreeHost(c.pinned2);
    c.pinned = c.pinned2 = nullptr;
    c.pinned_bytes = c.pinned2_bytes = 0;
    if (c.stream) cudaStreamDestroy(c.stream);
    if (c.copy_stream) cudaStreamDestroy(c.copy_stream);
    c.stream = c.copy_stream = nullptr;
    c.inited = false;
    return VB_OK;
}

void* vb_stream(void) { return (void*)vb::ctx().stream; }

int vb_stream_wait_event(void* cuda_event) {
    VB_TRY(vb::require_init());
    VB_REQUIRE(cuda_event, "null event");
    VB_CUDA(cudaStreamWaitEvent(vb::ctx().stream, (cudaEvent_t)cuda_event, 0));
    return VB_OK;
}

int vb_prof_enable(int on) {
    vb::prof_set(on != 0);
    return VB_OK;
}
int vb_prof_read(int kernel, double* total_ms, int64_t* launches) {
    VB_TRY(vb::require_init());
    return vb::prof_read(kernel, total_ms, launches);
}
int64_t vb_launch_count(void) { return vb::ctx().launches; }

int vb_synchronize(void) {
    VB_TRY(vb::require_init());
    VB_CUDA(cudaStreamSynchronize(vb::ctx().stream));
    return VB_OK;
}

}  // extern "C"
