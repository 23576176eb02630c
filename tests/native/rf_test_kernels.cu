// rf_test_kernels.cu -- test-only harness that launches the register-file self-test kernel of rf_selftest.cuh
// directly (tests/test_gpu_regfile_test.py).
//
// The product reaches rf_selftest only through b2dp_regfile_test, which reports per-device tallies.  This library
// launches one format at a time on the product's grid (every CTA cudaOccupancyMaxActiveBlocksPerMultiprocessor allows
// on every SM) and hands back what the product never shows:
//   - rf_dump: the DUMP instantiation for one round: every CTA's held registers after the march, folds and OR of
//              direct-compare differences of round 0, repetition 0 of every tile, and every CTA's record;
//   - rf_run:  the product instantiation for any duration, with the fault hook at a chosen register, element, thread
//              and mask, and every CTA's record.
// Both build the seed's tables and checks with rf_test_math.hpp, as the product does.
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "rf_selftest.cuh"

using namespace b2dp;

namespace {

using RfKernel = void (*)(const uint8_t*, const uint32_t*, unsigned long long, int, uint32_t, CtRecord*,
                          unsigned long long, uint32_t*);
const RfKernel kProduct[kRfFormats] = {rf_selftest<RF_ALU, false>, rf_selftest<RF_LOAD, false>,
                                       rf_selftest<RF_HOLD, false>};
const RfKernel kDump[kRfFormats] = {rf_selftest<RF_ALU, true>, rf_selftest<RF_LOAD, true>, rf_selftest<RF_HOLD, true>};

struct Harness {
    int device = 0;
    int sms = 0;
    int per_sm[kRfFormats] = {};  // cudaOccupancyMaxActiveBlocksPerMultiprocessor of the product instantiations
    cudaStream_t stream = nullptr;
    std::string err;
};

int fail(Harness* h, const char* what, cudaError_t e) {
    h->err = std::string(what) + ": " + cudaGetErrorName(e) + " (" + cudaGetErrorString(e) + ")";
    return 1;
}

#define RF(h, x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return fail(h, #x, e_); } while (0)

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

int grid_of(Harness* h, int fmt) { return h->sms * (h->per_sm[fmt] > 0 ? h->per_sm[fmt] : 1); }

// The seed's tables with the hook at (reg, element, thread), and the checks; grid CTAs of fn for duration_ns.
int launch(Harness* h, RfKernel fn, int fmt, uint32_t seed, const uint32_t hook[3], unsigned long long duration_ns,
           int fault_sm, uint32_t fault_mask, CtRecord* recs, float* ms, uint32_t* dump_out) {
    const int grid = grid_of(h, fmt);
    std::vector<uint32_t> tables((size_t)kCtTiles * kRfTableWords), checks((size_t)kCtTiles * kCtThreads);
    for (int t = 0; t < kCtTiles; ++t) {
        rf_build_tile(seed, fmt, t, tables.data() + t * kRfTableWords, checks.data() + t * kCtThreads);
        for (int i = 0; i < 3; ++i) tables[t * kRfTableWords + 2 + i] = hook[i];
    }
    Launch L;
    RF(h, cudaSetDevice(h->device));
    RF(h, cudaMalloc(&L.tab, tables.size() * 4));
    RF(h, cudaMemcpy(L.tab, tables.data(), tables.size() * 4, cudaMemcpyHostToDevice));
    RF(h, cudaMalloc(&L.chk, checks.size() * 4));
    RF(h, cudaMemcpy(L.chk, checks.data(), checks.size() * 4, cudaMemcpyHostToDevice));
    RF(h, cudaHostAlloc(&L.rec_h, (size_t)grid * sizeof(CtRecord), cudaHostAllocMapped));
    memset(L.rec_h, 0, (size_t)grid * sizeof(CtRecord));
    RF(h, cudaHostGetDevicePointer(&L.rec_d, L.rec_h, 0));
    const size_t dump_words = (size_t)grid * kCtTiles * kRfDumpWords;
    if (dump_out) {
        RF(h, cudaMalloc(&L.dump, dump_words * 4));
        RF(h, cudaMemsetAsync(L.dump, 0xFF, dump_words * 4, h->stream));
    }
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    RF(h, cudaEventCreate(&e0));
    RF(h, cudaEventCreate(&e1));
    cudaEventRecord(e0, h->stream);
    fn<<<grid, kCtThreads, kRfSmemBytes, h->stream>>>(reinterpret_cast<const uint8_t*>(L.tab), L.chk, duration_ns,
                                                      fault_sm, fault_mask, L.rec_d, 7ull, L.dump);
    cudaError_t e = cudaGetLastError();
    cudaEventRecord(e1, h->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
    if (e == cudaSuccess) e = cudaEventElapsedTime(ms, e0, e1);
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    if (e != cudaSuccess) return fail(h, "rf_selftest", e);
    if (dump_out) RF(h, cudaMemcpy(dump_out, L.dump, dump_words * 4, cudaMemcpyDeviceToHost));
    memcpy(recs, (const void*)L.rec_h, (size_t)grid * sizeof(CtRecord));
    return 0;
}

}  // namespace

extern "C" {

enum { RF_OK = 0, RF_E_CUDA = 1, RF_E_FMT = -1, RF_E_NOSPC = -2 };

const char* rf_error(void* hp) { return static_cast<Harness*>(hp)->err.c_str(); }

void* rf_open(int device, char* errbuf, int errlen) {
    Harness* h = new Harness;
    h->device = device;
    auto init = [h]() -> int {
        RF(h, cudaSetDevice(h->device));
        RF(h, cudaDeviceGetAttribute(&h->sms, cudaDevAttrMultiProcessorCount, h->device));
        RF(h, cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
        for (int f = 0; f < kRfFormats; ++f) {
            for (RfKernel k : {kProduct[f], kDump[f]})
                RF(h, cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kRfSmemBytes));
            RF(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&h->per_sm[f], kProduct[f], kCtThreads, kRfSmemBytes));
        }
        return RF_OK;
    };
    if (init() != RF_OK) {
        snprintf(errbuf, errlen, "%s", h->err.c_str());
        if (h->stream) cudaStreamDestroy(h->stream);
        delete h;
        return nullptr;
    }
    return h;
}

void rf_close(void* hp) {
    Harness* h = static_cast<Harness*>(hp);
    cudaSetDevice(h->device);
    if (h->stream) {
        cudaStreamSynchronize(h->stream);
        cudaStreamDestroy(h->stream);
    }
    delete h;
}

int rf_sms(void* hp) { return static_cast<Harness*>(hp)->sms; }
int rf_per_sm(void* hp, int fmt) { return fmt >= 0 && fmt < kRfFormats ? static_cast<Harness*>(hp)->per_sm[fmt] : RF_E_FMT; }
int rf_grid(void* hp, int fmt) { return fmt >= 0 && fmt < kRfFormats ? grid_of(static_cast<Harness*>(hp), fmt) : RF_E_FMT; }
int rf_record_bytes() { return (int)sizeof(CtRecord); }
int rf_dump_words() { return kRfDumpWords; }
int rf_held() { return kRfHeld; }

// The registers per thread of an instantiation (cudaFuncGetAttributes), DUMP or product.
int rf_num_regs(int fmt, int dump) {
    if (fmt < 0 || fmt >= kRfFormats) return RF_E_FMT;
    cudaFuncAttributes a{};
    if (cudaFuncGetAttributes(&a, dump ? kDump[fmt] : kProduct[fmt]) != cudaSuccess) return -3;
    return a.numRegs;
}

// The DUMP instantiation for one round on the seed's tables: out receives grid x kCtTiles x kRfDumpWords words,
// recs grid records (cap), *n the grid.
int rf_dump(void* hp, int fmt, uint32_t seed, uint32_t hook_reg, uint32_t hook_elem, uint32_t hook_thread, int fault_sm,
            uint32_t fault_mask, uint32_t* out, CtRecord* recs, int cap, int* n, float* ms) {
    Harness* h = static_cast<Harness*>(hp);
    if (fmt < 0 || fmt >= kRfFormats) return RF_E_FMT;
    *n = grid_of(h, fmt);
    if (*n > cap) return RF_E_NOSPC;
    const uint32_t hook[3] = {hook_reg, hook_elem, hook_thread};
    return launch(h, kDump[fmt], fmt, seed, hook, 0ull, fault_sm, fault_mask, recs, ms, out) ? RF_E_CUDA : RF_OK;
}

// The product instantiation for duration_ns with the hook at (hook_reg, hook_elem, hook_thread): every CTA's record.
int rf_run(void* hp, int fmt, uint32_t seed, unsigned long long duration_ns, uint32_t hook_reg, uint32_t hook_elem,
           uint32_t hook_thread, int fault_sm, uint32_t fault_mask, CtRecord* recs, int cap, int* n, float* ms) {
    Harness* h = static_cast<Harness*>(hp);
    if (fmt < 0 || fmt >= kRfFormats) return RF_E_FMT;
    *n = grid_of(h, fmt);
    if (*n > cap) return RF_E_NOSPC;
    const uint32_t hook[3] = {hook_reg, hook_elem, hook_thread};
    return launch(h, kProduct[fmt], fmt, seed, hook, duration_ns, fault_sm, fault_mask, recs, ms, nullptr) ? RF_E_CUDA
                                                                                                         : RF_OK;
}

}  // extern "C"
