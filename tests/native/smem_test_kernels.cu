// smem_test_kernels.cu -- test-only harness that launches the shared-memory self-test kernel of smem_selftest.cuh
// directly (tests/test_gpu_smem_test.py).
//
// The product reaches smem_selftest only through b2dp_smem_test, which reports per-device tallies.  This library
// launches one format at a time on the product's grid (one CTA per SM; SH_DSMEM: every co-resident cluster of two)
// and hands back what the product never shows:
//   - sh_dump: the DUMP instantiation for one round: every CTA's final array image, folds and direct-compare error
//              counts of round 0, repetition 0 of every tile, and every CTA's record;
//   - sh_run:  the product instantiation for any duration, with the fault hook at a chosen word, element and mask,
//              and every CTA's record.
// Both build the seed's tables and checks with smem_test_math.hpp, as the product does.
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "smem_selftest.cuh"

using namespace b2dp;

namespace {

using ShKernel = void (*)(const uint8_t*, const uint32_t*, unsigned long long, int, uint32_t, CtRecord*,
                          unsigned long long, uint32_t*);
const ShKernel kProduct[kShFormats] = {smem_selftest<SH_WORD, false>, smem_selftest<SH_BYTE, false>,
                                       smem_selftest<SH_DSMEM, false>};
const ShKernel kDump[kShFormats] = {smem_selftest<SH_WORD, true>, smem_selftest<SH_BYTE, true>,
                                    smem_selftest<SH_DSMEM, true>};

struct Harness {
    int device = 0;
    int sms = 0;
    int clusters = 0;  // co-resident clusters of two of the SH_DSMEM product instantiation
    cudaStream_t stream = nullptr;
    std::string err;
};

int fail(Harness* h, const char* what, cudaError_t e) {
    h->err = std::string(what) + ": " + cudaGetErrorName(e) + " (" + cudaGetErrorString(e) + ")";
    return 1;
}

#define SH(h, x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return fail(h, #x, e_); } while (0)

struct Launch {
    uint32_t* tab = nullptr;
    uint32_t* chk = nullptr;
    uint32_t* dump = nullptr;
    CtRecord *rec_h = nullptr, *rec_d = nullptr;
    ~Launch() {
        if (tab) cudaFree(tab);
        if (chk) cudaFree(chk);
        if (dump) cudaFree(dump);
        if (rec_h) cudaFreeHost(rec_h);
    }
};

int grid_of(Harness* h, int fmt) { return fmt == SH_DSMEM ? 2 * h->clusters : h->sms; }

// The seed's tables with the hook at (word, element), and the checks; grid CTAs of fn for duration_ns.
int launch(Harness* h, ShKernel fn, int fmt, uint32_t seed, uint32_t hook_word, uint32_t hook_elem,
           unsigned long long duration_ns, int fault_sm, uint32_t fault_mask, CtRecord* recs, float* ms,
           uint32_t* dump_out) {
    const int grid = grid_of(h, fmt);
    std::vector<uint32_t> tables((size_t)kCtTiles * kShTableWords), checks((size_t)kCtTiles * kCtThreads);
    for (int t = 0; t < kCtTiles; ++t) {
        sh_build_tile(seed, fmt, t, tables.data() + t * kShTableWords, checks.data() + t * kCtThreads);
        tables[t * kShTableWords + 2] = hook_word;
        tables[t * kShTableWords + 3] = hook_elem;
    }
    Launch L;
    SH(h, cudaSetDevice(h->device));
    SH(h, cudaMalloc(&L.tab, tables.size() * 4));
    SH(h, cudaMemcpy(L.tab, tables.data(), tables.size() * 4, cudaMemcpyHostToDevice));
    SH(h, cudaMalloc(&L.chk, checks.size() * 4));
    SH(h, cudaMemcpy(L.chk, checks.data(), checks.size() * 4, cudaMemcpyHostToDevice));
    SH(h, cudaHostAlloc(&L.rec_h, (size_t)grid * sizeof(CtRecord), cudaHostAllocMapped));
    memset(L.rec_h, 0, (size_t)grid * sizeof(CtRecord));
    SH(h, cudaHostGetDevicePointer(&L.rec_d, L.rec_h, 0));
    const size_t dump_words = (size_t)grid * kCtTiles * kShDumpWords;
    if (dump_out) {
        SH(h, cudaMalloc(&L.dump, dump_words * 4));
        SH(h, cudaMemsetAsync(L.dump, 0xFF, dump_words * 4, h->stream));
    }
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    SH(h, cudaEventCreate(&e0));
    SH(h, cudaEventCreate(&e1));
    cudaEventRecord(e0, h->stream);
    fn<<<grid, kCtThreads, kShBytes, h->stream>>>(reinterpret_cast<const uint8_t*>(L.tab), L.chk, duration_ns, fault_sm,
                                                  fault_mask, L.rec_d, 7ull, L.dump);
    cudaError_t e = cudaGetLastError();
    cudaEventRecord(e1, h->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
    if (e == cudaSuccess) e = cudaEventElapsedTime(ms, e0, e1);
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    if (e != cudaSuccess) return fail(h, "smem_selftest", e);
    if (dump_out) SH(h, cudaMemcpy(dump_out, L.dump, dump_words * 4, cudaMemcpyDeviceToHost));
    memcpy(recs, (const void*)L.rec_h, (size_t)grid * sizeof(CtRecord));
    return 0;
}

}  // namespace

extern "C" {

enum { SH_OK = 0, SH_E_CUDA = 1, SH_E_FMT = -1, SH_E_NOSPC = -2 };

const char* sh_error(void* hp) { return static_cast<Harness*>(hp)->err.c_str(); }

void* sh_open(int device, char* errbuf, int errlen) {
    Harness* h = new Harness;
    h->device = device;
    auto init = [h]() -> int {
        SH(h, cudaSetDevice(h->device));
        SH(h, cudaDeviceGetAttribute(&h->sms, cudaDevAttrMultiProcessorCount, h->device));
        SH(h, cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
        for (int f = 0; f < kShFormats; ++f)
            for (ShKernel k : {kProduct[f], kDump[f]}) {
                SH(h, cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kShBytes));
                SH(h, cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
            }
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(2);
        cfg.blockDim = dim3(kCtThreads);
        cfg.dynamicSmemBytes = kShBytes;
        SH(h, cudaOccupancyMaxActiveClusters(&h->clusters, kProduct[SH_DSMEM], &cfg));
        return SH_OK;
    };
    if (init() != SH_OK) {
        snprintf(errbuf, errlen, "%s", h->err.c_str());
        if (h->stream) cudaStreamDestroy(h->stream);
        delete h;
        return nullptr;
    }
    return h;
}

void sh_close(void* hp) {
    Harness* h = static_cast<Harness*>(hp);
    cudaSetDevice(h->device);
    if (h->stream) {
        cudaStreamSynchronize(h->stream);
        cudaStreamDestroy(h->stream);
    }
    delete h;
}

int sh_sms(void* hp) { return static_cast<Harness*>(hp)->sms; }
int sh_clusters(void* hp) { return static_cast<Harness*>(hp)->clusters; }
int sh_grid(void* hp, int fmt) { return fmt >= 0 && fmt < kShFormats ? grid_of(static_cast<Harness*>(hp), fmt) : SH_E_FMT; }
int sh_record_bytes() { return (int)sizeof(CtRecord); }
int sh_dump_words() { return kShDumpWords; }

// What cudaOccupancyMaxActiveBlocksPerMultiprocessor says of the product instantiation of fmt with kShBytes: its
// return code (a cudaError_t) and, on success, *ctas.
int sh_occupancy(void* hp, int fmt, int* ctas) {
    Harness* h = static_cast<Harness*>(hp);
    if (fmt < 0 || fmt >= kShFormats) return SH_E_FMT;
    cudaSetDevice(h->device);
    *ctas = -1;
    const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(ctas, kProduct[fmt], kCtThreads, kShBytes);
    cudaGetLastError();
    return (int)e;
}

// The DUMP instantiation for one round on the seed's tables: out receives grid x kCtTiles x kShDumpWords words,
// recs grid records (cap), *n the grid.
int sh_dump(void* hp, int fmt, uint32_t seed, uint32_t hook_word, uint32_t hook_elem, int fault_sm, uint32_t fault_mask,
            uint32_t* out, CtRecord* recs, int cap, int* n, float* ms) {
    Harness* h = static_cast<Harness*>(hp);
    if (fmt < 0 || fmt >= kShFormats) return SH_E_FMT;
    *n = grid_of(h, fmt);
    if (*n > cap) return SH_E_NOSPC;
    return launch(h, kDump[fmt], fmt, seed, hook_word, hook_elem, 0ull, fault_sm, fault_mask, recs, ms, out) ? SH_E_CUDA
                                                                                                            : SH_OK;
}

// The product instantiation for duration_ns with the hook at (hook_word, hook_elem): every CTA's record.
int sh_run(void* hp, int fmt, uint32_t seed, unsigned long long duration_ns, uint32_t hook_word, uint32_t hook_elem,
           int fault_sm, uint32_t fault_mask, CtRecord* recs, int cap, int* n, float* ms) {
    Harness* h = static_cast<Harness*>(hp);
    if (fmt < 0 || fmt >= kShFormats) return SH_E_FMT;
    *n = grid_of(h, fmt);
    if (*n > cap) return SH_E_NOSPC;
    return launch(h, kProduct[fmt], fmt, seed, hook_word, hook_elem, duration_ns, fault_sm, fault_mask, recs, ms,
                  nullptr)
               ? SH_E_CUDA
               : SH_OK;
}

}  // extern "C"
