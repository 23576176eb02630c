// hostlink_kernels.cu -- test-only harness over the host-link self-test's SM kernel (tests/test_gpu_hostlink_test.py).
//
// The product reaches hostlink_sm only through b2dp_hostlink_test, with its own buffers, grid and seeds.  This library
// gives a test two mapped pinned host buffers of any size (cudaHostAlloc), and runs one pass of hostlink_sm over the
// first n_vec vectors of them with any seed, grid and fault hook, returning the published ProbeOut and every CTA's
// record.  The test then compares the destination buffer, a guard region past it, the checksum and the records with
// tests/hostlink_oracle.py.  A pass that would reach past the buffers is refused, never launched.
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <string>

#include "hostlink_selftest.cuh"

using namespace b2dp;

namespace {

struct Harness {
    int device = 0;
    int sms = 0;
    int grid = 0;                       // every resident CTA
    cudaStream_t stream = nullptr;
    ProbeCtl* ctl = nullptr;
    ProbeOut *out_h = nullptr, *out_d = nullptr;
    HlRecord *rec_h = nullptr, *rec_d = nullptr;
    int rec_cap = 0;
    void *src = nullptr, *dst = nullptr;
    unsigned long long buf_bytes = 0;
    std::string err;
};

int fail(Harness* h, const char* what, cudaError_t e) {
    h->err = std::string(what) + ": " + cudaGetErrorName(e) + " (" + cudaGetErrorString(e) + ")";
    return 1;
}

}  // namespace

#define CK(h, x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return fail(h, #x, e_); } while (0)

extern "C" {

enum { HK_OK = 0, HK_E_CUDA = 1, HK_E_RANGE = -1, HK_E_GRID = -2, HK_E_NOBUF = -3 };

const char* hk_error(void* hp) { return static_cast<Harness*>(hp)->err.c_str(); }
int hk_sms(void* hp) { return static_cast<Harness*>(hp)->sms; }
int hk_grid(void* hp) { return static_cast<Harness*>(hp)->grid; }
int hk_record_bytes() { return (int)sizeof(HlRecord); }

void* hk_open(int device, char* errbuf, int errlen) {
    Harness* h = new Harness;
    h->device = device;
    auto init = [h]() -> int {
        CK(h, cudaSetDevice(h->device));
        CK(h, cudaDeviceGetAttribute(&h->sms, cudaDevAttrMultiProcessorCount, h->device));
        CK(h, cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
        CK(h, cudaMalloc(&h->ctl, sizeof(ProbeCtl)));
        ProbeCtl c = {};
        c.first_bad = ~0ull;
        c.t_start_ns = ~0ull;
        CK(h, cudaMemcpy(h->ctl, &c, sizeof c, cudaMemcpyHostToDevice));
        CK(h, cudaHostAlloc(&h->out_h, sizeof(ProbeOut), cudaHostAllocMapped));
        memset(h->out_h, 0, sizeof(ProbeOut));
        CK(h, cudaHostGetDevicePointer(&h->out_d, h->out_h, 0));
        int per_sm = 0;
        CK(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, hostlink_sm<kHlThreads, kHlUnroll>, kHlThreads, 0));
        h->grid = h->sms * (per_sm > 0 ? per_sm : 1);
        h->rec_cap = 4 * h->grid;
        CK(h, cudaHostAlloc(&h->rec_h, (size_t)h->rec_cap * sizeof(HlRecord), cudaHostAllocMapped));
        memset(h->rec_h, 0, (size_t)h->rec_cap * sizeof(HlRecord));
        CK(h, cudaHostGetDevicePointer(&h->rec_d, h->rec_h, 0));
        return HK_OK;
    };
    if (init() != HK_OK) {
        snprintf(errbuf, errlen, "%s", h->err.c_str());
        if (h->rec_h) cudaFreeHost(h->rec_h);
        if (h->out_h) cudaFreeHost(h->out_h);
        if (h->ctl) cudaFree(h->ctl);
        if (h->stream) cudaStreamDestroy(h->stream);
        delete h;
        return nullptr;
    }
    return h;
}

void hk_free(void* hp) {
    Harness* h = static_cast<Harness*>(hp);
    cudaSetDevice(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    if (h->src) cudaFreeHost(h->src);
    if (h->dst) cudaFreeHost(h->dst);
    h->src = h->dst = nullptr;
    h->buf_bytes = 0;
}

void hk_close(void* hp) {
    Harness* h = static_cast<Harness*>(hp);
    hk_free(hp);
    if (h->rec_h) cudaFreeHost(h->rec_h);
    if (h->out_h) cudaFreeHost(h->out_h);
    if (h->ctl) cudaFree(h->ctl);
    if (h->stream) cudaStreamDestroy(h->stream);
    delete h;
}

// Two mapped pinned host buffers of `bytes` each (a multiple of 16), replacing any earlier pair.
int hk_alloc(void* hp, unsigned long long bytes, void** src, void** dst) {
    Harness* h = static_cast<Harness*>(hp);
    if (bytes == 0 || bytes % 16) return HK_E_RANGE;
    hk_free(hp);
    CK(h, cudaHostAlloc(&h->src, bytes, cudaHostAllocMapped));
    CK(h, cudaHostAlloc(&h->dst, bytes, cudaHostAllocMapped));
    h->buf_bytes = bytes;
    *src = h->src;
    *dst = h->dst;
    return HK_OK;
}

// One pass of hostlink_sm over the first n_vec vectors of the buffers; grid 0 = every resident CTA.  *out = the
// published result block; recs[0 .. grid) = the CTAs' records.
int hk_run(void* hp, unsigned long long n_vec, uint32_t seed, uint32_t delta, unsigned long long fault_word,
           uint32_t fault_mask, int grid, unsigned long long seq, ProbeOut* out, HlRecord* recs, int rec_cap) {
    Harness* h = static_cast<Harness*>(hp);
    if (!h->src) return HK_E_NOBUF;
    if (n_vec * 16 > h->buf_bytes) return HK_E_RANGE;
    if (grid <= 0) grid = h->grid;
    if (grid > h->rec_cap || grid > rec_cap) return HK_E_GRID;
    CK(h, cudaSetDevice(h->device));
    uint4 *s = nullptr, *d = nullptr;
    CK(h, cudaHostGetDevicePointer((void**)&s, h->src, 0));
    CK(h, cudaHostGetDevicePointer((void**)&d, h->dst, 0));
    hostlink_sm<kHlThreads, kHlUnroll><<<grid, kHlThreads, 0, h->stream>>>(s, d, n_vec, seed, delta, fault_word,
                                                                            fault_mask, h->ctl, h->out_d, seq, h->rec_d);
    CK(h, cudaGetLastError());
    CK(h, cudaStreamSynchronize(h->stream));
    memcpy(out, (const void*)h->out_h, sizeof(ProbeOut));
    memcpy(recs, (const void*)h->rec_h, (size_t)grid * sizeof(HlRecord));
    return HK_OK;
}

}  // extern "C"
