// sfu_test_kernels.cu -- test-only harness that launches the SFU self-test kernel of sfu_selftest.cuh directly
// (tests/test_gpu_sfu_test.py).
//
// The product reaches sfu_selftest only through b2dp_sfu_test, which reports per-device tallies.  This library launches
// one format at a time and hands back what the product never shows:
//   - sk_dump:       the reference launch (the DUMP instantiation, one CTA on every SM, one round) on the seed's
//                    tables: every CTA's result words and records, so a test can compare the SMs with each other and
//                    the majority with tests/sfu_test_oracle.py;
//   - sk_run:        the reference launch, sf_consensus, then the product instantiation on its checks for any
//                    duration, with the fault hook, and every CTA's record;
//   - sk_run_tables: either instantiation on operand and check tables the caller built (wrong operands, wrong check
//                    values), on any grid up to the resident CTAs.  Malformed input is refused with a code before
//                    anything is allocated or launched.
#include <cuda_runtime.h>

#include <chrono>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "sfu_selftest.cuh"

using namespace b2dp;

namespace {

using SkKernel = void (*)(const uint8_t*, const uint32_t*, unsigned long long, int, uint32_t, CtRecord*,
                          unsigned long long, uint32_t*);
const SkKernel kProduct[kSfFormats] = {sfu_selftest<SF_F32, false>, sfu_selftest<SF_ROOT, false>,
                                       sfu_selftest<SF_F16, false>};
const SkKernel kDump[kSfFormats] = {sfu_selftest<SF_F32, true>, sfu_selftest<SF_ROOT, true>,
                                    sfu_selftest<SF_F16, true>};
constexpr int kRefSmem = 120 << 10;  // more than half an SM's shared memory: one CTA per SM (as the product)

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

#define SK(h, x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return fail(h, #x, e_); } while (0)

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

std::vector<uint32_t> build_tables(int fmt, uint32_t seed) {
    std::vector<uint32_t> t((size_t)kCtTiles * kSfSlots[fmt] * kCtThreads);
    for (int tile = 0; tile < kCtTiles; ++tile) sf_build_table(seed, fmt, tile, t.data() + (size_t)tile * kSfSlots[fmt] * kCtThreads);
    return t;
}

size_t cta_words(int fmt) { return (size_t)kCtTiles * kCtThreads * kSfWords[fmt]; }

int upload(Harness* h, Launch& L, const void* tables, size_t table_bytes, const uint32_t* checks, int n_rec) {
    SK(h, cudaMalloc(&L.tab, table_bytes));
    SK(h, cudaMemcpy(L.tab, tables, table_bytes, cudaMemcpyHostToDevice));
    if (checks) {
        const size_t check_bytes = (size_t)kCtTiles * kCtThreads * 4;
        SK(h, cudaMalloc(&L.chk, check_bytes));
        SK(h, cudaMemcpy(L.chk, checks, check_bytes, cudaMemcpyHostToDevice));
    }
    SK(h, cudaHostAlloc(&L.rec_h, (size_t)n_rec * sizeof(CtRecord), cudaHostAllocMapped));
    memset(L.rec_h, 0, (size_t)n_rec * sizeof(CtRecord));
    SK(h, cudaHostGetDevicePointer(&L.rec_d, L.rec_h, 0));
    return 0;
}

// One launch of fn on grid CTAs with the uploaded tables; records to recs, time to *ms, DUMP words to dump_out.
int launch(Harness* h, Launch& L, SkKernel fn, int fmt, int grid, int smem, unsigned long long duration_ns, int fault_sm,
           uint32_t fault_mask, CtRecord* recs, float* ms, uint32_t* dump_out) {
    if (dump_out) {
        SK(h, cudaMalloc(&L.dump, grid * cta_words(fmt) * 4));
        SK(h, cudaMemsetAsync(L.dump, 0xFF, grid * cta_words(fmt) * 4, h->stream));
    }
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    SK(h, cudaEventCreate(&e0));
    SK(h, cudaEventCreate(&e1));
    cudaEventRecord(e0, h->stream);
    fn<<<grid, kCtThreads, smem, h->stream>>>(L.tab, L.chk, duration_ns, fault_sm, fault_mask, L.rec_d, 7ull, L.dump);
    cudaError_t e = cudaGetLastError();
    cudaEventRecord(e1, h->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
    if (e == cudaSuccess) e = cudaEventElapsedTime(ms, e0, e1);
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    if (e != cudaSuccess) return fail(h, "sfu_selftest", e);
    if (dump_out) SK(h, cudaMemcpy(dump_out, L.dump, grid * cta_words(fmt) * 4, cudaMemcpyDeviceToHost));
    memcpy(recs, (const void*)L.rec_h, (size_t)grid * sizeof(CtRecord));
    return 0;
}

int set_smem(Harness* h, SkKernel fn, int smem) {
    SK(h, cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    SK(h, cudaFuncSetAttribute(fn, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
    return 0;
}

}  // namespace

extern "C" {

enum { SK_OK = 0, SK_E_CUDA = 1, SK_E_FMT = -1, SK_E_NOSPC = -2, SK_E_SIZE = -3, SK_E_GRID = -4, SK_E_NULL = -5 };

const char* sk_error(void* hp) { return static_cast<Harness*>(hp)->err.c_str(); }

void* sk_open(int device, char* errbuf, int errlen) {
    Harness* h = new Harness;
    h->device = device;
    auto init = [h]() -> int {
        SK(h, cudaSetDevice(h->device));
        SK(h, cudaDeviceGetAttribute(&h->sms, cudaDevAttrMultiProcessorCount, h->device));
        SK(h, cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
        for (int f = 0; f < kSfFormats; ++f)
            if (set_smem(h, kDump[f], kRefSmem)) return SK_E_CUDA;
        return SK_OK;
    };
    if (init() != SK_OK) {
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
int sk_words(int fmt) { return fmt >= 0 && fmt < kSfFormats ? kSfWords[fmt] : SK_E_FMT; }
int sk_slots(int fmt) { return fmt >= 0 && fmt < kSfFormats ? kSfSlots[fmt] : SK_E_FMT; }

// Resident CTAs per SM of the product (dump = 0) or reference (dump != 0, with its shared memory) instantiation.
int sk_occupancy(void* hp, int fmt, int dump, int* ctas) {
    Harness* h = static_cast<Harness*>(hp);
    if (fmt < 0 || fmt >= kSfFormats) return SK_E_FMT;
    SK(h, cudaSetDevice(h->device));
    SK(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(ctas, dump ? kDump[fmt] : kProduct[fmt], kCtThreads,
                                                        dump ? kRefSmem : 0));
    return SK_OK;
}

// The seed's operand tables: kCtTiles x slots x kCtThreads words to out.
int sk_tables(int fmt, uint32_t seed, uint32_t* out) {
    if (fmt < 0 || fmt >= kSfFormats) return SK_E_FMT;
    const std::vector<uint32_t> t = build_tables(fmt, seed);
    memcpy(out, t.data(), t.size() * 4);
    return SK_OK;
}

// The reference launch on the seed's tables: SMs CTAs of the DUMP instantiation for one round, without checks.  out
// receives SMs x kCtTiles x kCtThreads x kSfWords[fmt] words, recs SMs records, *ms the launch's event time.
int sk_dump(void* hp, int fmt, uint32_t seed, int fault_sm, uint32_t fault_mask, uint32_t* out, CtRecord* recs, int cap,
            int* n, float* ms) {
    Harness* h = static_cast<Harness*>(hp);
    if (fmt < 0 || fmt >= kSfFormats) return SK_E_FMT;
    *n = h->sms;
    if (h->sms > cap) return SK_E_NOSPC;
    SK(h, cudaSetDevice(h->device));
    const std::vector<uint32_t> tables = build_tables(fmt, seed);
    Launch L;
    if (upload(h, L, tables.data(), tables.size() * 4, nullptr, h->sms)) return SK_E_CUDA;
    return launch(h, L, kDump[fmt], fmt, h->sms, kRefSmem, 0ull, fault_sm, fault_mask, recs, ms, out) ? SK_E_CUDA
                                                                                                       : SK_OK;
}

// The reference launch and sf_consensus, then the product instantiation of format `fmt` on SMs x resident CTAs per SM
// for duration_ns with the consensus checks and the fault hook (in both launches): every CTA's record of the timed
// launch to recs (cap records), the count to *n, its event time to *ms, and the consensus's flags / dissents /
// reference-plus-consensus milliseconds to info[0..2].
int sk_run(void* hp, int fmt, uint32_t seed, unsigned long long duration_ns, int fault_sm, uint32_t fault_mask,
           CtRecord* recs, int cap, int* n, float* ms, double* info) {
    Harness* h = static_cast<Harness*>(hp);
    if (fmt < 0 || fmt >= kSfFormats) return SK_E_FMT;
    SK(h, cudaSetDevice(h->device));
    int per_sm = 0;
    SK(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kProduct[fmt], kCtThreads, 0));
    const int grid = h->sms * (per_sm > 0 ? per_sm : 1);
    *n = grid;
    if (grid > cap) return SK_E_NOSPC;
    const auto t0 = std::chrono::steady_clock::now();
    const std::vector<uint32_t> tables = build_tables(fmt, seed);
    std::vector<uint32_t> dumps((size_t)h->sms * cta_words(fmt));
    std::vector<CtRecord> ref(h->sms);
    SfConsensus cons;
    {
        Launch L;
        float ref_ms = 0;
        if (upload(h, L, tables.data(), tables.size() * 4, nullptr, h->sms)) return SK_E_CUDA;
        if (launch(h, L, kDump[fmt], fmt, h->sms, kRefSmem, 0ull, fault_sm, fault_mask, ref.data(), &ref_ms, dumps.data()))
            return SK_E_CUDA;
        sf_consensus(fmt, dumps.data(), ref.data(), h->sms, 7ull, tables.data(), cons);
    }
    info[0] = cons.flags();
    info[1] = (double)cons.dissents;
    info[2] = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    Launch L;
    if (upload(h, L, tables.data(), tables.size() * 4, cons.check.data(), grid)) return SK_E_CUDA;
    return launch(h, L, kProduct[fmt], fmt, grid, 0, duration_ns, fault_sm, fault_mask, recs, ms, nullptr) ? SK_E_CUDA
                                                                                                          : SK_OK;
}

// The product (dump = 0) or DUMP (dump != 0, with the reference launch's shared memory) instantiation of format `fmt`
// on tables the caller built: `tables` holds kCtTiles operand tables of slots x kCtThreads words (table_bytes in
// all), `checks` kCtTiles x kCtThreads comparison values (n_checks in all).  `grid` CTAs, from 1 up to the resident
// CTAs, run for duration_ns (no fault hook); with dump, dump_out receives grid x kCtTiles x kCtThreads x words.
int sk_run_tables(void* hp, int fmt, int dump, const uint32_t* tables, unsigned long long table_bytes,
                  const uint32_t* checks, unsigned long long n_checks, int grid, unsigned long long duration_ns,
                  CtRecord* recs, int cap, int* n, float* ms, uint32_t* dump_out) {
    Harness* h = static_cast<Harness*>(hp);
    if (fmt < 0 || fmt >= kSfFormats) return SK_E_FMT;
    if (table_bytes != (unsigned long long)kCtTiles * sf_table_bytes(fmt)) return SK_E_SIZE;
    if (n_checks != (unsigned long long)kCtTiles * kCtThreads) return SK_E_SIZE;
    if (!tables || !checks || !recs || !n || !ms || (dump && !dump_out)) return SK_E_NULL;
    const SkKernel fn = dump ? kDump[fmt] : kProduct[fmt];
    const int smem = dump ? kRefSmem : 0;
    SK(h, cudaSetDevice(h->device));
    int per_sm = 0;
    SK(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, kCtThreads, smem));
    if (grid < 1 || grid > h->sms * per_sm) return SK_E_GRID;
    *n = grid;
    if (grid > cap) return SK_E_NOSPC;
    Launch L;
    if (upload(h, L, tables, (size_t)table_bytes, checks, grid)) return SK_E_CUDA;
    return launch(h, L, fn, fmt, grid, smem, duration_ns, -1, 0u, recs, ms, dump ? dump_out : nullptr) ? SK_E_CUDA
                                                                                                      : SK_OK;
}

}  // extern "C"
