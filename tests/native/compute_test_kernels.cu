// compute_test_kernels.cu -- test-only harness that launches the tensor-core self-test kernel of tc_selftest.cuh
// directly (tests/test_gpu_compute_test.py).
//
// The product reaches tc_selftest only through b2dp_compute_test, which reports per-device tallies.  This library
// launches one format at a time with the operand images and comparison values compute_test_math.hpp builds from a
// seed, and hands back what the product never shows:
//   - ck_dump: the DUMP instantiation (CTA 0 writes its raw accumulators of repetition 0 of every tile of round 0), so
//     a test can compare every accumulator bit with tests/compute_test_oracle.py;
//   - ck_run:  the product instantiation with any duration and fault hook, and every CTA's record.
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "tc_selftest.cuh"

using namespace b2dp;

namespace {

using CtKernel = void (*)(const uint8_t*, const uint32_t*, unsigned long long, int, uint32_t, CtRecord*,
                          unsigned long long, uint32_t*);
const CtKernel kProduct[kCtFormats] = {tc_selftest<CT_BF16, false>, tc_selftest<CT_FP8, false>,
                                       tc_selftest<CT_INT8, false>};
const CtKernel kDump[kCtFormats] = {tc_selftest<CT_BF16, true>, tc_selftest<CT_FP8, true>, tc_selftest<CT_INT8, true>};
const uint32_t kSmem[kCtFormats] = {CtShape<CT_BF16>::SMEM, CtShape<CT_FP8>::SMEM, CtShape<CT_INT8>::SMEM};

struct Harness {
    int device = 0;
    int sms = 0;
    cudaStream_t stream = nullptr;
    std::string err;
};

int fail(Harness* h, const char* what, cudaError_t e) {
    h->err = std::string(what) + ": " + cudaGetErrorName(e) + " (" + cudaGetErrorString(e) + ")";
    return 1;
}

#define CK(h, x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return fail(h, #x, e_); } while (0)

// The device buffers of one launch, released on every path.
struct Launch {
    uint8_t* img = nullptr;
    uint32_t* chk = nullptr;
    uint32_t* dump = nullptr;
    CtRecord *rec_h = nullptr, *rec_d = nullptr;
    ~Launch() {
        if (img) cudaFree(img);
        if (chk) cudaFree(chk);
        if (dump) cudaFree(dump);
        if (rec_h) cudaFreeHost(rec_h);
    }
};

int upload(Harness* h, Launch& L, int fmt, uint32_t seed, int n_rec) {
    std::vector<uint8_t> images((size_t)kCtTiles * kSmem[fmt]);
    std::vector<uint32_t> checks((size_t)kCtTiles * kCtThreads);
    CtTile t;
    for (int tile = 0; tile < kCtTiles; ++tile) {
        ct_build_tile(seed, fmt, tile, t);
        memcpy(images.data() + (size_t)tile * kSmem[fmt], t.image.data(), kSmem[fmt]);
        memcpy(checks.data() + (size_t)tile * kCtThreads, t.check, sizeof t.check);
    }
    CK(h, cudaMalloc(&L.img, images.size()));
    CK(h, cudaMalloc(&L.chk, checks.size() * sizeof(uint32_t)));
    CK(h, cudaMemcpy(L.img, images.data(), images.size(), cudaMemcpyHostToDevice));
    CK(h, cudaMemcpy(L.chk, checks.data(), checks.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
    CK(h, cudaHostAlloc(&L.rec_h, (size_t)n_rec * sizeof(CtRecord), cudaHostAllocMapped));
    memset(L.rec_h, 0, (size_t)n_rec * sizeof(CtRecord));
    CK(h, cudaHostGetDevicePointer(&L.rec_d, L.rec_h, 0));
    return 0;
}

}  // namespace

extern "C" {

enum { CK_OK = 0, CK_E_CUDA = 1, CK_E_FMT = -1, CK_E_NOSPC = -2 };

const char* ck_error(void* hp) { return static_cast<Harness*>(hp)->err.c_str(); }

void* ck_open(int device, char* errbuf, int errlen) {
    Harness* h = new Harness;
    h->device = device;
    auto init = [h]() -> int {
        CK(h, cudaSetDevice(h->device));
        CK(h, cudaDeviceGetAttribute(&h->sms, cudaDevAttrMultiProcessorCount, h->device));
        CK(h, cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
        for (int f = 0; f < kCtFormats; ++f)
            for (CtKernel fn : {kProduct[f], kDump[f]}) {
                CK(h, cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmem[f]));
                CK(h, cudaFuncSetAttribute(fn, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
            }
        return CK_OK;
    };
    if (init() != CK_OK) {
        snprintf(errbuf, errlen, "%s", h->err.c_str());
        if (h->stream) cudaStreamDestroy(h->stream);
        delete h;
        return nullptr;
    }
    return h;
}

void ck_close(void* hp) {
    Harness* h = static_cast<Harness*>(hp);
    cudaSetDevice(h->device);
    if (h->stream) {
        cudaStreamSynchronize(h->stream);
        cudaStreamDestroy(h->stream);
    }
    delete h;
}

int ck_sms(void* hp) { return static_cast<Harness*>(hp)->sms; }
int ck_tiles() { return kCtTiles; }
int ck_reps() { return kCtReps; }
int ck_record_bytes() { return (int)sizeof(CtRecord); }

// Resident CTAs per SM of the product instantiation of format `fmt` with the shared memory its launches use.
int ck_occupancy(void* hp, int fmt, int* ctas) {
    Harness* h = static_cast<Harness*>(hp);
    if (fmt < 0 || fmt >= kCtFormats) return CK_E_FMT;
    CK(h, cudaSetDevice(h->device));
    CK(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(ctas, kProduct[fmt], kCtThreads, kSmem[fmt]));
    return CK_OK;
}

// One CTA of the DUMP instantiation for one round (duration 0): out receives kCtTiles x kCtThreads x kCtAcc raw
// accumulator words in fragment order, rec its record.
int ck_dump(void* hp, int fmt, uint32_t seed, uint32_t* out, CtRecord* rec) {
    Harness* h = static_cast<Harness*>(hp);
    if (fmt < 0 || fmt >= kCtFormats) return CK_E_FMT;
    CK(h, cudaSetDevice(h->device));
    Launch L;
    if (upload(h, L, fmt, seed, 1)) return CK_E_CUDA;
    const size_t words = (size_t)kCtTiles * kCtThreads * kCtAcc;
    CK(h, cudaMalloc(&L.dump, words * 4));
    CK(h, cudaMemsetAsync(L.dump, 0xFF, words * 4, h->stream));
    kDump[fmt]<<<1, kCtThreads, kSmem[fmt], h->stream>>>(L.img, L.chk, 0ull, -1, 0u, L.rec_d, 1ull, L.dump);
    CK(h, cudaGetLastError());
    CK(h, cudaStreamSynchronize(h->stream));
    CK(h, cudaMemcpy(out, L.dump, words * 4, cudaMemcpyDeviceToHost));
    memcpy(rec, (const void*)L.rec_h, sizeof(CtRecord));
    return CK_OK;
}

// The product instantiation of format `fmt` on SMs x resident CTAs per SM for duration_ns, with the fault hook:
// every CTA's record to recs (cap records), the count to *n and the CUDA-event time of the launch to *ms.
int ck_run(void* hp, int fmt, uint32_t seed, unsigned long long duration_ns, int fault_sm, uint32_t fault_mask,
           CtRecord* recs, int cap, int* n, float* ms) {
    Harness* h = static_cast<Harness*>(hp);
    if (fmt < 0 || fmt >= kCtFormats) return CK_E_FMT;
    CK(h, cudaSetDevice(h->device));
    int per_sm = 0;
    CK(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kProduct[fmt], kCtThreads, kSmem[fmt]));
    const int grid = h->sms * (per_sm > 0 ? per_sm : 1);
    *n = grid;
    if (grid > cap) return CK_E_NOSPC;
    Launch L;
    if (upload(h, L, fmt, seed, grid)) return CK_E_CUDA;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    CK(h, cudaEventCreate(&e0));
    CK(h, cudaEventCreate(&e1));
    cudaEventRecord(e0, h->stream);
    kProduct[fmt]<<<grid, kCtThreads, kSmem[fmt], h->stream>>>(L.img, L.chk, duration_ns, fault_sm, fault_mask, L.rec_d,
                                                                7ull, nullptr);
    cudaError_t e = cudaGetLastError();
    cudaEventRecord(e1, h->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
    if (e == cudaSuccess) e = cudaEventElapsedTime(ms, e0, e1);
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    if (e != cudaSuccess) return fail(h, "tc_selftest", e);
    memcpy(recs, (const void*)L.rec_h, (size_t)grid * sizeof(CtRecord));
    return CK_OK;
}

}  // extern "C"
