// l1_test_kernels.cu -- test-only harness that launches the L1 self-test kernel of l1_selftest.cuh directly
// (tests/test_gpu_l1_test.py, tools/l1_span_sweep.py).
//
// The product reaches l1_selftest only through b2dp_l1_test, which reports per-device tallies and picks the span and the
// carve-out.  This library launches one format at a time and hands back what the product never shows:
//   - l1k_run:        the product or DUMP instantiation on tables l1_test_math.hpp builds from a seed, on every resident
//                     CTA (DUMP: CTA 0 alone), with any span (K blocks of 2 KiB per CTA; 0 = the product's default),
//                     carve-out, duration and the fault hook: every CTA's record, the launch time, the DUMP words;
//   - l1k_run_tables: the product instantiation on tables and checks the caller built, on any grid up to the resident
//                     CTAs.  Malformed tables, out-of-range indices and a zero texture handle are refused with a code
//                     before anything launches.
// The CUDA array, the texture objects and the constant bank are made by l1_bind from the seed, as the driver makes them.
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "l1_selftest.cuh"

using namespace b2dp;

namespace {

using L1Kernel = void (*)(const uint8_t*, const uint32_t*, unsigned long long, int, uint32_t, CtRecord*,
                          unsigned long long, uint32_t*);
const L1Kernel kProduct[kL1Formats] = {l1_selftest<L1_DATA, false>, l1_selftest<L1_TEX, false>,
                                       l1_selftest<L1_CONST, false>};
const L1Kernel kDump[kL1Formats] = {l1_selftest<L1_DATA, true>, l1_selftest<L1_TEX, true>,
                                    l1_selftest<L1_CONST, true>};

struct Harness {
    int device = 0, sms = 0;
    cudaStream_t stream = nullptr;
    std::string err;
};

int fail(Harness* h, const char* what, cudaError_t e) {
    h->err = std::string(what) + ": " + cudaGetErrorName(e) + " (" + cudaGetErrorString(e) + ")";
    return 1;
}

#define LK(h, x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return fail(h, #x, e_); } while (0)

// The buffers and host objects of one launch, released on every path after the stream is synchronized.
struct Launch {
    cudaStream_t stream = nullptr;
    uint8_t* tab = nullptr;
    uint32_t* chk = nullptr;
    uint32_t* scratch = nullptr;
    CtRecord *rec_h = nullptr, *rec_d = nullptr;
    L1Bound bound;
    ~Launch() {
        if (stream) cudaStreamSynchronize(stream);
        l1_unbind(bound);
        if (tab) cudaFree(tab);
        if (chk) cudaFree(chk);
        if (scratch) cudaFree(scratch);
        if (rec_h) cudaFreeHost(rec_h);
    }
};

size_t data_words(int fmt, int grid, uint32_t K) {
    return fmt == L1_DATA ? (size_t)grid * K * kL1BlockWords : fmt == L1_TEX ? (size_t)kL1Texels * 4 : 0;
}
size_t dump_words(int fmt, uint32_t K) {
    return (size_t)kCtTiles * kCtThreads * (fmt == L1_DATA ? (size_t)kL1Passes * K * 4 : (size_t)l1_words(fmt));
}

// Resident CTAs per SM at a carve-out: the 1 KiB of shared memory the runtime reserves per CTA counts against it.
int occupancy(Harness* h, L1Kernel fn, int* per_sm, int carveout = 0) {
    LK(h, cudaFuncSetAttribute(fn, cudaFuncAttributePreferredSharedMemoryCarveout, carveout));
    LK(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(per_sm, fn, kCtThreads, 0));
    if (*per_sm < 1) *per_sm = 1;
    return 0;
}

// Uploads, binds and launches fn on grid CTAs; zap >= 0 clears texture handle zap before the handle check.
int launch(Harness* h, int fmt, L1Kernel fn, uint32_t seed, const uint32_t* tables, const uint32_t* checks, int grid,
           uint32_t K, int carveout, unsigned long long duration_ns, int fault_sm, uint32_t fault_mask, int zap,
           CtRecord* recs, float* ms, uint32_t* dump_out) {
    for (int tile = 0; tile < kCtTiles; ++tile)
        if (!l1_table_ok(fmt, tables + (size_t)tile * kL1TableWords)) return -3;
    Launch L;
    L.stream = h->stream;
    const size_t dwords = dump_out ? dump_words(fmt, K) : 0;
    const size_t words = kL1DataOff + data_words(fmt, grid, K) + dwords;
    LK(h, cudaMalloc(&L.tab, (size_t)kCtTiles * kL1TableWords * 4));
    LK(h, cudaMalloc(&L.chk, (size_t)kCtTiles * kCtThreads * 4));
    LK(h, cudaMalloc(&L.scratch, words * 4));
    LK(h, cudaMemcpy(L.tab, tables, (size_t)kCtTiles * kL1TableWords * 4, cudaMemcpyHostToDevice));
    LK(h, cudaMemcpy(L.chk, checks, (size_t)kCtTiles * kCtThreads * 4, cudaMemcpyHostToDevice));
    uint32_t hdr[kL1HdrWords] = {};
    hdr[kL1HdrBlocks] = K;
    hdr[kL1HdrDump] = (uint32_t)(kL1DataOff + data_words(fmt, grid, K));
    LK(h, cudaMemset(L.scratch, 0, words * 4));
    LK(h, cudaMemcpy(L.scratch, hdr, sizeof hdr, cudaMemcpyHostToDevice));
    const char* where = "";
    cudaError_t ce = l1_bind(seed, fmt == L1_TEX ? L.scratch : nullptr, h->stream, L.bound, &where);
    if (ce != cudaSuccess) return fail(h, where, ce);
    if (fmt == L1_TEX) {
        unsigned long long hd[kL1TexObjs];
        LK(h, cudaMemcpy(hd, L.scratch + kL1HdrTex, sizeof hd, cudaMemcpyDeviceToHost));
        if (zap >= 0 && zap < kL1TexObjs) {
            hd[zap] = 0;
            LK(h, cudaMemcpy(L.scratch + kL1HdrTex, hd, sizeof hd, cudaMemcpyHostToDevice));
        }
        if (!l1_handles_ok(hd)) return -6;
    }
    LK(h, cudaFuncSetAttribute(fn, cudaFuncAttributePreferredSharedMemoryCarveout, carveout));
    LK(h, cudaHostAlloc(&L.rec_h, (size_t)grid * sizeof(CtRecord), cudaHostAllocMapped));
    memset(L.rec_h, 0, (size_t)grid * sizeof(CtRecord));
    LK(h, cudaHostGetDevicePointer(&L.rec_d, L.rec_h, 0));
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    LK(h, cudaEventCreate(&e0));
    LK(h, cudaEventCreate(&e1));
    cudaEventRecord(e0, h->stream);
    fn<<<grid, kCtThreads, 0, h->stream>>>(L.tab, L.chk, duration_ns, fault_sm, fault_mask, L.rec_d, 7ull, L.scratch);
    cudaError_t e = cudaGetLastError();
    cudaEventRecord(e1, h->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
    if (e == cudaSuccess) e = cudaEventElapsedTime(ms, e0, e1);
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    if (e != cudaSuccess) return fail(h, "l1_selftest", e);
    if (dump_out) LK(h, cudaMemcpy(dump_out, L.scratch + hdr[kL1HdrDump], dwords * 4, cudaMemcpyDeviceToHost));
    memcpy(recs, (const void*)L.rec_h, (size_t)grid * sizeof(CtRecord));
    return 0;
}

}  // namespace

extern "C" {

enum { LK_OK = 0, LK_E_CUDA = 1, LK_E_FMT = -1, LK_E_NOSPC = -2, LK_E_TABLE = -3, LK_E_GRID = -4, LK_E_NULL = -5,
       LK_E_HANDLE = -6, LK_E_SIZE = -7 };

const char* l1k_error(void* hp) { return static_cast<Harness*>(hp)->err.c_str(); }

void* l1k_open(int device, char* errbuf, int errlen) {
    Harness* h = new Harness;
    h->device = device;
    auto init = [h]() -> int {
        LK(h, cudaSetDevice(h->device));
        LK(h, cudaDeviceGetAttribute(&h->sms, cudaDevAttrMultiProcessorCount, h->device));
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

void l1k_close(void* hp) {
    Harness* h = static_cast<Harness*>(hp);
    cudaSetDevice(h->device);
    if (h->stream) {
        cudaStreamSynchronize(h->stream);
        cudaStreamDestroy(h->stream);
    }
    delete h;
}

int l1k_sms(void* hp) { return static_cast<Harness*>(hp)->sms; }
int l1k_record_bytes() { return (int)sizeof(CtRecord); }
int l1k_words(int fmt) { return fmt >= 0 && fmt < kL1Formats ? l1_words(fmt) : LK_E_FMT; }

// Resident CTAs per SM of the product (dump = 0) or DUMP instantiation of `fmt` at the product's carve-out of 0.
int l1k_occupancy(void* hp, int fmt, int dump, int* ctas) {
    Harness* h = static_cast<Harness*>(hp);
    if (fmt < 0 || fmt >= kL1Formats) return LK_E_FMT;
    LK(h, cudaSetDevice(h->device));
    return occupancy(h, dump ? kDump[fmt] : kProduct[fmt], ctas) ? LK_E_CUDA : LK_OK;
}

// The blocks per CTA span the product uses on this device for L1_DATA.
int l1k_default_blocks(void* hp, unsigned* K) {
    int per_sm = 0;
    if (l1k_occupancy(hp, L1_DATA, 0, &per_sm) != LK_OK) return LK_E_CUDA;
    *K = l1_span_blocks(kL1DefaultSpan, per_sm);
    return LK_OK;
}

// DUMP words of one launch of `fmt` with K blocks per span.
unsigned long long l1k_dump_words(int fmt, unsigned K) {
    return fmt >= 0 && fmt < kL1Formats ? (unsigned long long)dump_words(fmt, K) : 0ull;
}

// One launch of `fmt` on the seed's tables: the product instantiation on every resident CTA, or (dump) the DUMP
// instantiation on CTA 0 alone for one round.  K blocks per span (L1_DATA; 0 = the product's default), the carve-out in
// percent, duration_ns and the fault hook.  Every CTA's record to recs (cap records), the count to *n, the CUDA-event
// time to *ms, K to *k_used, and with dump the DUMP words to dump_out.
int l1k_run(void* hp, int fmt, int dump, uint32_t seed, unsigned K, int carveout, unsigned long long duration_ns,
            int fault_sm, uint32_t fault_mask, CtRecord* recs, int cap, int* n, float* ms, unsigned* k_used,
            uint32_t* dump_out) {
    Harness* h = static_cast<Harness*>(hp);
    if (fmt < 0 || fmt >= kL1Formats) return LK_E_FMT;
    if (!recs || !n || !ms || !k_used || (dump && !dump_out)) return LK_E_NULL;
    if (carveout < 0 || carveout > 100 || K > kL1MaxBlocks) return LK_E_SIZE;
    LK(h, cudaSetDevice(h->device));
    int per_sm = 0;
    if (occupancy(h, kProduct[fmt], &per_sm, carveout)) return LK_E_CUDA;
    const int grid = dump ? 1 : h->sms * per_sm;
    *n = grid;
    if (grid > cap) return LK_E_NOSPC;
    if (K == 0) K = l1_span_blocks(kL1DefaultSpan, per_sm);
    *k_used = K;
    std::vector<uint32_t> tables((size_t)kCtTiles * kL1TableWords), checks((size_t)kCtTiles * kCtThreads);
    for (int tile = 0; tile < kCtTiles; ++tile)
        l1_build_tile(seed, fmt, tile, tables.data() + (size_t)tile * kL1TableWords,
                      checks.data() + (size_t)tile * kCtThreads);
    return launch(h, fmt, dump ? kDump[fmt] : kProduct[fmt], seed, tables.data(), checks.data(), grid, K, carveout,
                  dump ? 0ull : duration_ns, dump ? -1 : fault_sm, fault_mask, -1, recs, ms, dump ? dump_out : nullptr);
}

// The product instantiation of `fmt` on tables the caller built: `tables` holds kCtTiles tables of kL1TableWords words
// (table_bytes in all), `checks` kCtTiles x kCtThreads comparison values (n_checks in all); the image and the bank come
// from `seed`.  `grid` CTAs, from 1 up to the resident CTAs, K blocks per span (0: the default), for duration_ns, no
// fault hook; zap >= 0 clears that texture handle (L1_TEX), which must be refused.
int l1k_run_tables(void* hp, int fmt, uint32_t seed, const uint32_t* tables, unsigned long long table_bytes,
                   const uint32_t* checks, unsigned long long n_checks, int grid, unsigned K,
                   unsigned long long duration_ns, int zap, CtRecord* recs, int cap, int* n, float* ms) {
    Harness* h = static_cast<Harness*>(hp);
    if (fmt < 0 || fmt >= kL1Formats) return LK_E_FMT;
    if (table_bytes != (unsigned long long)kCtTiles * l1_table_bytes(fmt)) return LK_E_SIZE;
    if (n_checks != (unsigned long long)kCtTiles * kCtThreads || K > kL1MaxBlocks) return LK_E_SIZE;
    if (!tables || !checks || !recs || !n || !ms) return LK_E_NULL;
    LK(h, cudaSetDevice(h->device));
    int per_sm = 0;
    if (occupancy(h, kProduct[fmt], &per_sm)) return LK_E_CUDA;
    if (grid < 1 || grid > h->sms * per_sm) return LK_E_GRID;
    *n = grid;
    if (grid > cap) return LK_E_NOSPC;
    if (K == 0) K = l1_span_blocks(kL1DefaultSpan, per_sm);
    return launch(h, fmt, kProduct[fmt], seed, tables, checks, grid, K, 0, duration_ns, -1, 0u, zap, recs, ms,
                  nullptr);
}

}  // extern "C"
