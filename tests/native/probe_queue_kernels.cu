// probe_queue_kernels.cu -- test-only harness that launches hbm_probe_queue (the health probe's kernel, hbm_probe.cuh)
// directly, for tests/test_gpu_probe_queue.py.
//
// The product reaches the kernel only through its C ABI, with its own buffers and grid.  This library launches the
// product's instantiation on caller-owned buffers (torch allocations), with any grid and any seed/delta, so a test can
// compare every result field, the whole written buffer and the control block (tile queue included) with
// oracle/probe.py at the pipeline edges.
//
// The harness refuses a launch that would read or write outside the buffers it was given (n_vec larger than either
// buffer, a pointer that is not 32-byte aligned) or whose grid is out of range: it never launches something that
// could fault.
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <string>

#include "hbm_probe.cuh"

using namespace b2dp;

namespace {

const auto kKernel = hbm_probe_queue<kQueueCW, kQueueTileVec, kQueueStages>;
constexpr int kThreads = (kQueueCW + 2) * 32;

struct Harness {
    int device = 0;
    int sms = 0;
    cudaStream_t stream = nullptr;
    ProbeCtl* ctl = nullptr;
    ProbeOut *out_h = nullptr, *out_d = nullptr;
    std::string err;
};

int fail(Harness* h, const char* what, cudaError_t e) {
    h->err = std::string(what) + ": " + cudaGetErrorName(e) + " (" + cudaGetErrorString(e) + ")";
    return 1;
}

}  // namespace

#define CK(h, x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return fail(h, #x, e_); } while (0)

extern "C" {

// Refusals (nothing launched); CUDA failures return 1 and leave the message in pq_error().
enum { PQ_OK = 0, PQ_E_CUDA = 1, PQ_E_SIZE = -2, PQ_E_ALIGN = -3, PQ_E_GRID = -4, PQ_E_SEQ = -5 };

// The kernel's shape, in the fields of tests/probe_cases.Variant.
void pq_variant(const char** name, int* vec_per_tile, int* stages, int* threads, int* ctas_per_sm) {
    *name = "queue_4_512_6";
    *vec_per_tile = kQueueTileVec; *stages = kQueueStages; *threads = kThreads; *ctas_per_sm = kQueueCtasPerSm;
}

const char* pq_error(void* hp) { return static_cast<Harness*>(hp)->err.c_str(); }

// A stream, a control block initialised the way cuda_backend_open does it, a mapped pinned result block, and the
// kernel's dynamic-smem attribute and carve-out as the product sets them.
void* pq_open(int device, char* errbuf, int errlen) {
    Harness* h = new Harness;
    h->device = device;
    auto init = [h]() -> int {
        CK(h, cudaSetDevice(h->device));
        CK(h, cudaDeviceGetAttribute(&h->sms, cudaDevAttrMultiProcessorCount, h->device));
        CK(h, cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
        CK(h, cudaMalloc(&h->ctl, sizeof(ProbeCtl)));
        ProbeCtl c{};
        c.first_bad = ~0ull; c.t_start_ns = ~0ull;
        CK(h, cudaMemcpy(h->ctl, &c, sizeof c, cudaMemcpyHostToDevice));
        CK(h, cudaHostAlloc(&h->out_h, sizeof(ProbeOut), cudaHostAllocMapped));
        memset(h->out_h, 0, sizeof(ProbeOut));
        CK(h, cudaHostGetDevicePointer(&h->out_d, h->out_h, 0));
        CK(h, cudaFuncSetAttribute(kKernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kQueueSmem));
        CK(h, cudaFuncSetAttribute(kKernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
        return PQ_OK;
    };
    if (init() != PQ_OK) {
        snprintf(errbuf, errlen, "%s", h->err.c_str());
        if (h->out_h) cudaFreeHost(h->out_h);
        if (h->ctl) cudaFree(h->ctl);
        if (h->stream) cudaStreamDestroy(h->stream);
        delete h;
        return nullptr;
    }
    return h;
}

void pq_close(void* hp) {
    Harness* h = static_cast<Harness*>(hp);
    cudaSetDevice(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    if (h->out_h) cudaFreeHost(h->out_h);
    if (h->ctl) cudaFree(h->ctl);
    if (h->stream) cudaStreamDestroy(h->stream);
    delete h;
}

int pq_sms(void* hp) { return static_cast<Harness*>(hp)->sms; }

// One launch over n_vec vectors of src into dst; grid 0 = the product shape (SMs x kQueueCtasPerSm).  Synchronises,
// copies the published result block to *res and checks that it carries this launch's seq.
int pq_run(void* hp, unsigned long long src, unsigned long long src_bytes, unsigned long long dst,
           unsigned long long dst_bytes, unsigned long long n_vec, uint32_t seed, uint32_t delta, int grid,
           unsigned long long seq, ProbeOut* res) {
    Harness* h = static_cast<Harness*>(hp);
    if (n_vec > src_bytes / 16 || n_vec > dst_bytes / 16) return PQ_E_SIZE;
    if (!src || !dst || (src | dst) % 32) return PQ_E_ALIGN;
    if (grid < 0 || grid > (1 << 20)) return PQ_E_GRID;
    const int g = grid ? grid : h->sms * kQueueCtasPerSm;
    CK(h, cudaSetDevice(h->device));
    const uint4* s = reinterpret_cast<const uint4*>(src);
    uint4* d = reinterpret_cast<uint4*>(dst);
    kKernel<<<g, kThreads, kQueueSmem, h->stream>>>(s, d, n_vec, seed, delta, h->ctl, h->out_d, seq);
    CK(h, cudaGetLastError());
    CK(h, cudaStreamSynchronize(h->stream));
    memcpy(res, (const void*)h->out_h, sizeof(ProbeOut));
    return res->seq == seq ? PQ_OK : PQ_E_SEQ;
}

// The control block as the last launch left it ({0, 0, ~0, ~0, 0, next_tile 0} after a complete launch).
int pq_read_ctl(void* hp, ProbeCtl* out) {
    Harness* h = static_cast<Harness*>(hp);
    CK(h, cudaSetDevice(h->device));
    CK(h, cudaStreamSynchronize(h->stream));
    CK(h, cudaMemcpy(out, h->ctl, sizeof(ProbeCtl), cudaMemcpyDeviceToHost));
    return PQ_OK;
}

// Resident CTAs per SM with the shared memory the launches really use (after pq_open set the attributes).
int pq_occupancy(void* hp, int* ctas) {
    Harness* h = static_cast<Harness*>(hp);
    CK(h, cudaSetDevice(h->device));
    CK(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(ctas, reinterpret_cast<const void*>(kKernel), kThreads,
                                                        kQueueSmem));
    return PQ_OK;
}

}  // extern "C"
