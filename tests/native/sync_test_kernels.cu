// sync_test_kernels.cu -- test-only harness that launches the synchronization self-test kernel of sync_selftest.cuh directly
// (tests/test_gpu_sync_test.py).
//
// The product reaches sync_selftest only through b2dp_sync_test, which reports per-device tallies.  This library launches
// one format at a time and hands back what the product never shows:
//   - sk_dump:       the DUMP instantiation on one CTA for one round: every result word of repetition 0 of every tile,
//                    so a test can compare every bit with tests/sync_test_oracle.py;
//   - sk_run:        the product instantiation on tables sync_test_math.hpp builds from a seed, with any duration and the
//                    fault hook, and every CTA's record;
//   - sk_run_tables: either instantiation on operand and check tables the caller built (wrong operands, wrong check
//                    values, checks computed by a fault model), on any grid up to the resident CTAs.
//                    Malformed input is refused with a code before anything is allocated or launched.
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "sync_selftest.cuh"

using namespace b2dp;

namespace {

using SyKernel = void (*)(const uint8_t*, const uint32_t*, unsigned long long, int, uint32_t, CtRecord*,
                          unsigned long long, uint32_t*);
const SyKernel kProduct[kSyFormats] = {sync_selftest<SY_ATOM, false>, sync_selftest<SY_BAR, false>,
                                       sync_selftest<SY_WARP, false>};
const SyKernel kDump[kSyFormats] = {sync_selftest<SY_ATOM, true>, sync_selftest<SY_BAR, true>, sync_selftest<SY_WARP, true>};

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

#define IK(h, x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return fail(h, #x, e_); } while (0)

// The device buffers of one launch, released on every path.
struct Launch {
    uint8_t* tab = nullptr;
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

void build_tables(int fmt, uint32_t seed, std::vector<uint8_t>& tables, std::vector<uint32_t>& checks) {
    const size_t tb = sy_table_bytes(fmt);
    tables.assign((size_t)kCtTiles * tb, 0);
    checks.assign((size_t)kCtTiles * kCtThreads, 0);
    for (int tile = 0; tile < kCtTiles; ++tile)
        sy_build_tile(seed, fmt, tile, reinterpret_cast<uint32_t*>(tables.data() + (size_t)tile * tb),
                      checks.data() + (size_t)tile * kCtThreads);
}

int upload(Harness* h, Launch& L, const uint8_t* tables, size_t table_bytes, const uint32_t* checks, int n_rec) {
    const size_t check_bytes = (size_t)kCtTiles * kCtThreads * 4;
    IK(h, cudaMalloc(&L.tab, table_bytes));
    IK(h, cudaMalloc(&L.chk, check_bytes));
    IK(h, cudaMemcpy(L.tab, tables, table_bytes, cudaMemcpyHostToDevice));
    IK(h, cudaMemcpy(L.chk, checks, check_bytes, cudaMemcpyHostToDevice));
    IK(h, cudaHostAlloc(&L.rec_h, (size_t)n_rec * sizeof(CtRecord), cudaHostAllocMapped));
    memset(L.rec_h, 0, (size_t)n_rec * sizeof(CtRecord));
    IK(h, cudaHostGetDevicePointer(&L.rec_d, L.rec_h, 0));
    return 0;
}

size_t dump_words(int fmt) { return (size_t)kCtTiles * kCtThreads * kSyWords[fmt]; }

// One launch of fn on grid CTAs with the uploaded tables; records to recs, time to *ms, DUMP words to dump_out.
int launch(Harness* h, Launch& L, SyKernel fn, int fmt, int grid, unsigned long long duration_ns, int fault_sm,
           uint32_t fault_mask, CtRecord* recs, float* ms, uint32_t* dump_out) {
    if (dump_out) {
        IK(h, cudaMalloc(&L.dump, dump_words(fmt) * 4));
        IK(h, cudaMemsetAsync(L.dump, 0xFF, dump_words(fmt) * 4, h->stream));
    }
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    IK(h, cudaEventCreate(&e0));
    IK(h, cudaEventCreate(&e1));
    cudaEventRecord(e0, h->stream);
    fn<<<grid, kCtThreads, 0, h->stream>>>(L.tab, L.chk, duration_ns, fault_sm, fault_mask, L.rec_d, 7ull, L.dump);
    cudaError_t e = cudaGetLastError();
    cudaEventRecord(e1, h->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
    if (e == cudaSuccess) e = cudaEventElapsedTime(ms, e0, e1);
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    if (e != cudaSuccess) return fail(h, "sync_selftest", e);
    if (dump_out) IK(h, cudaMemcpy(dump_out, L.dump, dump_words(fmt) * 4, cudaMemcpyDeviceToHost));
    memcpy(recs, (const void*)L.rec_h, (size_t)grid * sizeof(CtRecord));
    return 0;
}

}  // namespace

extern "C" {

enum { IK_OK = 0, IK_E_CUDA = 1, IK_E_FMT = -1, IK_E_NOSPC = -2, IK_E_SIZE = -3, IK_E_GRID = -4, IK_E_NULL = -5 };

const char* sk_error(void* hp) { return static_cast<Harness*>(hp)->err.c_str(); }

void* sk_open(int device, char* errbuf, int errlen) {
    Harness* h = new Harness;
    h->device = device;
    auto init = [h]() -> int {
        IK(h, cudaSetDevice(h->device));
        IK(h, cudaDeviceGetAttribute(&h->sms, cudaDevAttrMultiProcessorCount, h->device));
        IK(h, cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
        return IK_OK;
    };
    if (init() != IK_OK) {
        snprintf(errbuf, errlen, "%s", h->err.c_str());
        if (h->stream) cudaStreamDestroy(h->stream);
        delete h;
        return nullptr;
    }
    return h;
}

void sk_close(void* hp) {
    Harness* h = static_cast<Harness*>(hp);
    cudaSetDevice(h->device);
    if (h->stream) {
        cudaStreamSynchronize(h->stream);
        cudaStreamDestroy(h->stream);
    }
    delete h;
}

int sk_sms(void* hp) { return static_cast<Harness*>(hp)->sms; }
int sk_tiles() { return kCtTiles; }
int sk_reps() { return kCtReps; }
int sk_record_bytes() { return (int)sizeof(CtRecord); }
int sk_words(int fmt) { return fmt >= 0 && fmt < kSyFormats ? kSyWords[fmt] : IK_E_FMT; }
unsigned long long sk_table_bytes(int fmt) { return fmt >= 0 && fmt < kSyFormats ? sy_table_bytes(fmt) : 0; }

// Resident CTAs per SM of the product instantiation of format `fmt`.
int sk_occupancy(void* hp, int fmt, int* ctas) {
    Harness* h = static_cast<Harness*>(hp);
    if (fmt < 0 || fmt >= kSyFormats) return IK_E_FMT;
    IK(h, cudaSetDevice(h->device));
    IK(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(ctas, kProduct[fmt], kCtThreads, 0));
    return IK_OK;
}

// One CTA of the DUMP instantiation for one round (duration 0) on the seed's tables: out receives kCtTiles x
// kCtThreads x kSyWords[fmt] result words, rec its record.
int sk_dump(void* hp, int fmt, uint32_t seed, uint32_t* out, CtRecord* rec) {
    Harness* h = static_cast<Harness*>(hp);
    if (fmt < 0 || fmt >= kSyFormats) return IK_E_FMT;
    IK(h, cudaSetDevice(h->device));
    std::vector<uint8_t> tables;
    std::vector<uint32_t> checks;
    build_tables(fmt, seed, tables, checks);
    Launch L;
    if (upload(h, L, tables.data(), tables.size(), checks.data(), 1)) return IK_E_CUDA;
    float ms = 0;
    return launch(h, L, kDump[fmt], fmt, 1, 0ull, -1, 0u, rec, &ms, out) ? IK_E_CUDA : IK_OK;
}

// The product instantiation of format `fmt` on SMs x resident CTAs per SM for duration_ns, with the fault hook: every
// CTA's record to recs (cap records), the count to *n and the CUDA-event time of the launch to *ms.
int sk_run(void* hp, int fmt, uint32_t seed, unsigned long long duration_ns, int fault_sm, uint32_t fault_mask,
           CtRecord* recs, int cap, int* n, float* ms) {
    Harness* h = static_cast<Harness*>(hp);
    if (fmt < 0 || fmt >= kSyFormats) return IK_E_FMT;
    IK(h, cudaSetDevice(h->device));
    int per_sm = 0;
    IK(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kProduct[fmt], kCtThreads, 0));
    const int grid = h->sms * (per_sm > 0 ? per_sm : 1);
    *n = grid;
    if (grid > cap) return IK_E_NOSPC;
    std::vector<uint8_t> tables;
    std::vector<uint32_t> checks;
    build_tables(fmt, seed, tables, checks);
    Launch L;
    if (upload(h, L, tables.data(), tables.size(), checks.data(), grid)) return IK_E_CUDA;
    return launch(h, L, kProduct[fmt], fmt, grid, duration_ns, fault_sm, fault_mask, recs, ms, nullptr) ? IK_E_CUDA
                                                                                                         : IK_OK;
}

// The product (dump = 0) or DUMP (dump != 0) instantiation of format `fmt` on tables the caller built: `tables` holds
// kCtTiles operand tables of sk_table_bytes(fmt) bytes (table_bytes in all), `checks` kCtTiles x kCtThreads comparison
// values (n_checks in all).  `grid` CTAs, from 1 up to the resident CTAs, run for duration_ns (no fault hook).
int sk_run_tables(void* hp, int fmt, int dump, const uint8_t* tables, unsigned long long table_bytes,
                  const uint32_t* checks, unsigned long long n_checks, int grid, unsigned long long duration_ns,
                  CtRecord* recs, int cap, int* n, float* ms, uint32_t* dump_out) {
    Harness* h = static_cast<Harness*>(hp);
    if (fmt < 0 || fmt >= kSyFormats) return IK_E_FMT;
    if (table_bytes != (unsigned long long)kCtTiles * sy_table_bytes(fmt)) return IK_E_SIZE;
    if (n_checks != (unsigned long long)kCtTiles * kCtThreads) return IK_E_SIZE;
    if (!tables || !checks || !recs || !n || !ms || (dump && !dump_out)) return IK_E_NULL;
    const SyKernel fn = dump ? kDump[fmt] : kProduct[fmt];
    IK(h, cudaSetDevice(h->device));
    int per_sm = 0;
    IK(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, kCtThreads, 0));
    if (grid < 1 || grid > h->sms * per_sm) return IK_E_GRID;
    *n = grid;
    if (grid > cap) return IK_E_NOSPC;
    Launch L;
    if (upload(h, L, tables, (size_t)table_bytes, checks, grid)) return IK_E_CUDA;
    return launch(h, L, fn, fmt, grid, duration_ns, -1, 0u, recs, ms, dump ? dump_out : nullptr) ? IK_E_CUDA : IK_OK;
}

}  // extern "C"
