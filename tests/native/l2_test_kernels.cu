// l2_test_kernels.cu -- test-only harness that launches the L2 self-test kernel of l2_selftest.cuh directly
// (tests/test_gpu_l2_test.py, tools/l2_span_sweep.py).
//
// The product reaches l2_selftest only through b2dp_l2_test, which reports per-device tallies and picks the span.  This
// library launches one format at a time, cooperatively on every resident CTA, and hands back what the product never
// shows: every CTA's record, the launch time, and with the DUMP instantiation the folds, error counts and window
// images (L2_WORD / L2_BYTE) or the hot block and combined folds (L2_ATOM) of round 0, so a test can compare every bit
// with tests/l2_test_oracle.py.  The span is K blocks of 2 KiB per CTA (K = 0: the product's default).
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "l2_selftest.cuh"

using namespace b2dp;

namespace {

using LkKernel = void (*)(const uint8_t*, const uint32_t*, unsigned long long, int, uint32_t, CtRecord*,
                          unsigned long long, uint32_t*);
const LkKernel kProduct[kL2Formats] = {l2_selftest<L2_WORD, false>, l2_selftest<L2_BYTE, false>,
                                       l2_selftest<L2_ATOM, false>};
const LkKernel kDump[kL2Formats] = {l2_selftest<L2_WORD, true>, l2_selftest<L2_BYTE, true>, l2_selftest<L2_ATOM, true>};

struct Harness {
    int device = 0, sms = 0, l2 = 0;
    cudaStream_t stream = nullptr;
    std::string err;
};

int fail(Harness* h, const char* what, cudaError_t e) {
    h->err = std::string(what) + ": " + cudaGetErrorName(e) + " (" + cudaGetErrorString(e) + ")";
    return 1;
}

#define LK(h, x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return fail(h, #x, e_); } while (0)

struct Launch {
    uint8_t* tab = nullptr;
    uint32_t* chk = nullptr;
    uint32_t* scratch = nullptr;
    CtRecord *rec_h = nullptr, *rec_d = nullptr;
    ~Launch() {
        if (tab) cudaFree(tab);
        if (chk) cudaFree(chk);
        if (scratch) cudaFree(scratch);
        if (rec_h) cudaFreeHost(rec_h);
    }
};

size_t data_words(int fmt, int grid, uint32_t K) {
    return fmt == L2_ATOM ? (size_t)kL2AtomHotWords : (size_t)kL2Windows * K * grid * kL2BlockWords;
}

}  // namespace

extern "C" {

enum { LK_OK = 0, LK_E_CUDA = 1, LK_E_FMT = -1, LK_E_NOSPC = -2, LK_E_NULL = -5 };

const char* lk_error(void* hp) { return static_cast<Harness*>(hp)->err.c_str(); }

void* lk_open(int device, char* errbuf, int errlen) {
    Harness* h = new Harness;
    h->device = device;
    auto init = [h]() -> int {
        LK(h, cudaSetDevice(h->device));
        LK(h, cudaDeviceGetAttribute(&h->sms, cudaDevAttrMultiProcessorCount, h->device));
        LK(h, cudaDeviceGetAttribute(&h->l2, cudaDevAttrL2CacheSize, h->device));
        LK(h, cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
        return LK_OK;
    };
    if (init() != LK_OK) {
        snprintf(errbuf, errlen, "%s", h->err.c_str());
        if (h->stream) cudaStreamDestroy(h->stream);
        delete h;
        return nullptr;
    }
    return h;
}

void lk_close(void* hp) {
    Harness* h = static_cast<Harness*>(hp);
    cudaSetDevice(h->device);
    if (h->stream) {
        cudaStreamSynchronize(h->stream);
        cudaStreamDestroy(h->stream);
    }
    delete h;
}

int lk_sms(void* hp) { return static_cast<Harness*>(hp)->sms; }
int lk_l2_bytes(void* hp) { return static_cast<Harness*>(hp)->l2; }
int lk_record_bytes() { return (int)sizeof(CtRecord); }
unsigned long long lk_table_bytes(int fmt) { return fmt >= 0 && fmt < kL2Formats ? l2_table_bytes(fmt) : 0; }

// Resident CTAs per SM of the product (dump = 0) or DUMP instantiation of `fmt`.
int lk_occupancy(void* hp, int fmt, int dump, int* ctas) {
    Harness* h = static_cast<Harness*>(hp);
    if (fmt < 0 || fmt >= kL2Formats) return LK_E_FMT;
    LK(h, cudaSetDevice(h->device));
    LK(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(ctas, dump ? kDump[fmt] : kProduct[fmt], kCtThreads, 0));
    return LK_OK;
}

// The blocks per CTA slice the product uses on this device for `fmt` (0 for L2_ATOM).
int lk_default_blocks(void* hp, int fmt, unsigned* K) {
    Harness* h = static_cast<Harness*>(hp);
    int per_sm = 0;
    if (lk_occupancy(hp, fmt, 0, &per_sm) != LK_OK) return LK_E_CUDA;
    *K = fmt == L2_ATOM ? 0u : l2_span_blocks(l2_default_span((unsigned long long)h->l2), h->sms * per_sm);
    return LK_OK;
}

// DUMP words of one launch of `fmt` on `grid` CTAs with K blocks per slice.
unsigned long long lk_dump_words(int fmt, int grid, unsigned K) {
    if (fmt == L2_ATOM) return (unsigned long long)kCtTiles * (kL2AtomHotWords + 4 * kL2AtomRet);
    return (unsigned long long)kCtTiles * grid * 2 * kCtThreads + (unsigned long long)kCtTiles * K * grid * kL2BlockWords;
}

// One cooperative launch of `fmt` (dump: the DUMP instantiation) on every resident CTA, on the seed's tables, with K
// blocks per slice (0: the product's default), for duration_ns, with the fault hook.  Every CTA's record to recs (cap
// records), the count to *n, the CUDA-event time to *ms, K to *k_used, and with dump the DUMP words to dump_out.
int lk_run(void* hp, int fmt, int dump, uint32_t seed, unsigned K, unsigned long long duration_ns, int fault_sm,
           uint32_t fault_mask, CtRecord* recs, int cap, int* n, float* ms, unsigned* k_used, uint32_t* dump_out) {
    Harness* h = static_cast<Harness*>(hp);
    if (fmt < 0 || fmt >= kL2Formats) return LK_E_FMT;
    if (!recs || !n || !ms || !k_used || (dump && !dump_out)) return LK_E_NULL;
    const LkKernel fn = dump ? kDump[fmt] : kProduct[fmt];
    LK(h, cudaSetDevice(h->device));
    int per_sm = 0, coop = 0;
    LK(h, cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, h->device));
    if (!coop) { h->err = "the device has no cooperative launch"; return LK_E_CUDA; }
    LK(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, kCtThreads, 0));
    const int grid = h->sms * (per_sm > 0 ? per_sm : 1);
    *n = grid;
    if (grid > cap || grid > kL2MaxCtas) return LK_E_NOSPC;
    if (fmt != L2_ATOM && K == 0) K = l2_span_blocks(l2_default_span((unsigned long long)h->l2), grid);
    if (fmt == L2_ATOM) K = 0;
    *k_used = K;
    const size_t tb = l2_table_bytes(fmt);
    std::vector<uint8_t> tables((size_t)kCtTiles * tb);
    std::vector<uint32_t> checks((size_t)kCtTiles * kCtThreads);
    for (int tile = 0; tile < kCtTiles; ++tile)
        l2_build_tile(seed, fmt, tile, reinterpret_cast<uint32_t*>(tables.data() + (size_t)tile * tb),
                      checks.data() + (size_t)tile * kCtThreads);
    const size_t dwords = dump ? (size_t)lk_dump_words(fmt, grid, K) : 0;
    const size_t words = kL2DataOff + data_words(fmt, grid, K) + dwords;
    Launch L;
    LK(h, cudaMalloc(&L.tab, tables.size()));
    LK(h, cudaMalloc(&L.chk, checks.size() * 4));
    LK(h, cudaMalloc(&L.scratch, words * 4));
    LK(h, cudaMemcpy(L.tab, tables.data(), tables.size(), cudaMemcpyHostToDevice));
    LK(h, cudaMemcpy(L.chk, checks.data(), checks.size() * 4, cudaMemcpyHostToDevice));
    uint32_t hdr[kL2HdrWords] = {};
    hdr[kL2HdrBlocks] = K;
    hdr[kL2HdrDump] = (uint32_t)(kL2DataOff + data_words(fmt, grid, K));
    LK(h, cudaMemset(L.scratch, 0, words * 4));
    LK(h, cudaMemcpy(L.scratch, hdr, sizeof hdr, cudaMemcpyHostToDevice));
    LK(h, cudaHostAlloc(&L.rec_h, (size_t)grid * sizeof(CtRecord), cudaHostAllocMapped));
    memset(L.rec_h, 0, (size_t)grid * sizeof(CtRecord));
    LK(h, cudaHostGetDevicePointer(&L.rec_d, L.rec_h, 0));
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    LK(h, cudaEventCreate(&e0));
    LK(h, cudaEventCreate(&e1));
    const uint8_t* a_tab = L.tab;
    const uint32_t* a_chk = L.chk;
    unsigned long long a_dur = duration_ns, a_seq = 7ull;
    CtRecord* a_rec = L.rec_d;
    uint32_t* a_scr = L.scratch;
    void* args[] = {&a_tab, &a_chk, &a_dur, &fault_sm, &fault_mask, &a_rec, &a_seq, &a_scr};
    cudaEventRecord(e0, h->stream);
    cudaError_t e = cudaLaunchCooperativeKernel((const void*)fn, dim3(grid), dim3(kCtThreads), args, 0, h->stream);
    cudaEventRecord(e1, h->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
    if (e == cudaSuccess) e = cudaEventElapsedTime(ms, e0, e1);
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    if (e != cudaSuccess) return fail(h, "l2_selftest", e);
    if (dump) LK(h, cudaMemcpy(dump_out, L.scratch + hdr[kL2HdrDump], dwords * 4, cudaMemcpyDeviceToHost));
    memcpy(recs, (const void*)L.rec_h, (size_t)grid * sizeof(CtRecord));
    return LK_OK;
}

}  // extern "C"
