// probe_kernels.cu -- test-only harness that launches the kernels of hbm_probe.cuh directly (tests/test_gpu_kernels.py).
//
// The product reaches these kernels only through its C ABI, with its own buffers, grid and fault paths.  This library
// exposes each instantiation -- the product shapes, the HINT variants and the other shapes tools/probe_sweep compares --
// with caller-owned buffers (torch allocations), any grid and any seed/delta, so a test can compare every result field
// and the whole written buffer with oracle/probe.py at the pipeline edges.
//
// The harness refuses a launch that would read or write outside the buffers it was given (n_vec larger than either
// buffer, a pointer that is not 32-byte aligned): it never launches something that could fault.
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <string>

#include "hbm_probe.cuh"

using namespace b2dp;

namespace {

using ProbeFn = void (*)(const uint4*, uint4*, unsigned long long, uint32_t, uint32_t, ProbeCtl*, ProbeOut*,
                         unsigned long long);

struct Variant {
    const char* name;
    int vec_per_tile;  // vectors per TMA tile, or per register-path chunk (one grid-stride step of one CTA)
    int stages;        // TMA ring depth, 0 for the register paths
    int threads;       // threads per CTA
    int ctas_per_sm;   // the product's CTAs per SM for this kernel family (grid 0 = SMs x this)
    ProbeFn fn;
    size_t smem;       // dynamic shared memory per CTA
};

template <int CW, int TV, int ST, int HINT = 0>
constexpr Variant tma(const char* name) {
    return {name, TV, ST, (CW + 1) * 32, kTmaCtasPerSm, hbm_probe_tma<CW, TV, ST, HINT>, tma_smem_bytes(TV, ST)};
}

const Variant kVariants[] = {
    tma<kTmaCW, kTmaTileVec, kTmaStages>("tma_4_1024_3"),
    {"r128_512_2", kRegThreads * kRegUnroll, 0, kRegThreads, kRegCtasPerSm, hbm_probe_r128<kRegThreads, kRegUnroll>, 0},
    tma<4, 1024, 3, 1>("tma_4_1024_3_h1"),
    tma<4, 1024, 3, 2>("tma_4_1024_3_h2"),
    tma<4, 1024, 3, 4>("tma_4_1024_3_h4"),
    tma<4, 1024, 3, 8>("tma_4_1024_3_h8"),
    tma<4, 512, 6>("tma_4_512_6"),
    tma<2, 1024, 4>("tma_2_1024_4"),
    tma<8, 2048, 3>("tma_8_2048_3"),
    // R256 moves pairs of vectors: one grid-stride chunk is THREADS * UNROLL pairs
    {"r256_256_1", 2 * 256 * 1, 0, 256, kRegCtasPerSm, hbm_probe_r256<256, 1>, 0},
    {"r256_512_2", 2 * 512 * 2, 0, 512, kRegCtasPerSm, hbm_probe_r256<512, 2>, 0},
};
constexpr int kNumVariants = sizeof(kVariants) / sizeof(kVariants[0]);

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

// Refusals (nothing launched); CUDA failures return 1 and leave the message in pk_error().
enum { PK_OK = 0, PK_E_CUDA = 1, PK_E_VARIANT = -1, PK_E_SIZE = -2, PK_E_ALIGN = -3, PK_E_GRID = -4, PK_E_SEQ = -5 };

int pk_num_variants() { return kNumVariants; }

int pk_variant(int v, const char** name, int* vec_per_tile, int* stages, int* threads, int* ctas_per_sm) {
    if (v < 0 || v >= kNumVariants) return PK_E_VARIANT;
    const Variant& x = kVariants[v];
    *name = x.name; *vec_per_tile = x.vec_per_tile; *stages = x.stages; *threads = x.threads; *ctas_per_sm = x.ctas_per_sm;
    return PK_OK;
}

const char* pk_error(void* hp) { return static_cast<Harness*>(hp)->err.c_str(); }

// A stream, a control block initialised the way cuda_backend_open does it, and a mapped pinned result block.  Every
// TMA instantiation gets the product's dynamic-smem attribute and carve-out.
void* pk_open(int device, char* errbuf, int errlen) {
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
        for (const Variant& v : kVariants) {
            if (!v.stages) continue;
            CK(h, cudaFuncSetAttribute(v.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)v.smem));
            CK(h, cudaFuncSetAttribute(v.fn, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
        }
        return PK_OK;
    };
    if (init() != PK_OK) {
        snprintf(errbuf, errlen, "%s", h->err.c_str());
        if (h->out_h) cudaFreeHost(h->out_h);
        if (h->ctl) cudaFree(h->ctl);
        if (h->stream) cudaStreamDestroy(h->stream);
        delete h;
        return nullptr;
    }
    return h;
}

void pk_close(void* hp) {
    Harness* h = static_cast<Harness*>(hp);
    cudaSetDevice(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    if (h->out_h) cudaFreeHost(h->out_h);
    if (h->ctl) cudaFree(h->ctl);
    if (h->stream) cudaStreamDestroy(h->stream);
    delete h;
}

int pk_sms(void* hp) { return static_cast<Harness*>(hp)->sms; }

// One launch of variant v over n_vec vectors of src into dst; grid 0 = the product shape (SMs x CTAs per SM).
// Synchronises, copies the published result block to *res and checks that it carries this launch's seq.
int pk_run(void* hp, int v, unsigned long long src, unsigned long long src_bytes, unsigned long long dst,
           unsigned long long dst_bytes, unsigned long long n_vec, uint32_t seed, uint32_t delta, int grid,
           unsigned long long seq, ProbeOut* res) {
    Harness* h = static_cast<Harness*>(hp);
    if (v < 0 || v >= kNumVariants) return PK_E_VARIANT;
    if (n_vec > src_bytes / 16 || n_vec > dst_bytes / 16) return PK_E_SIZE;
    if (!src || !dst || (src | dst) % 32) return PK_E_ALIGN;
    if (grid < 0 || grid > (1 << 20)) return PK_E_GRID;
    const Variant& x = kVariants[v];
    const int g = grid ? grid : h->sms * x.ctas_per_sm;
    CK(h, cudaSetDevice(h->device));
    const uint4* s = reinterpret_cast<const uint4*>(src);
    uint4* d = reinterpret_cast<uint4*>(dst);
    void* args[] = {&s, &d, &n_vec, &seed, &delta, &h->ctl, &h->out_d, &seq};
    CK(h, cudaLaunchKernel(reinterpret_cast<const void*>(x.fn), dim3(g), dim3(x.threads), args, x.smem, h->stream));
    CK(h, cudaStreamSynchronize(h->stream));
    memcpy(res, (const void*)h->out_h, sizeof(ProbeOut));
    return res->seq == seq ? PK_OK : PK_E_SEQ;
}

// The control block as the last launch left it (the last CTA resets it to {0, 0, ~0, ~0, 0}).
int pk_read_ctl(void* hp, ProbeCtl* out) {
    Harness* h = static_cast<Harness*>(hp);
    CK(h, cudaSetDevice(h->device));
    CK(h, cudaStreamSynchronize(h->stream));
    CK(h, cudaMemcpy(out, h->ctl, sizeof(ProbeCtl), cudaMemcpyDeviceToHost));
    return PK_OK;
}

// hbm_fill over n_vec vectors of dst with the product's launch shape.
int pk_fill(void* hp, unsigned long long dst, unsigned long long dst_bytes, unsigned long long n_vec, uint32_t seed) {
    Harness* h = static_cast<Harness*>(hp);
    if (n_vec > dst_bytes / 16) return PK_E_SIZE;
    if (!dst || dst % 32) return PK_E_ALIGN;
    CK(h, cudaSetDevice(h->device));
    hbm_fill<256><<<h->sms * 8, 256, 0, h->stream>>>(reinterpret_cast<uint4*>(dst), n_vec, seed);
    CK(h, cudaGetLastError());
    CK(h, cudaStreamSynchronize(h->stream));
    return PK_OK;
}

// Resident CTAs per SM of variant v with the shared memory its launches really use (after pk_open set the attributes).
int pk_occupancy(void* hp, int v, int* ctas) {
    Harness* h = static_cast<Harness*>(hp);
    if (v < 0 || v >= kNumVariants) return PK_E_VARIANT;
    const Variant& x = kVariants[v];
    CK(h, cudaSetDevice(h->device));
    CK(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(ctas, reinterpret_cast<const void*>(x.fn), x.threads, x.smem));
    return PK_OK;
}

}  // extern "C"
