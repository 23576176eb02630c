// memtest_kernels.cu -- test-only harness that launches the march kernel of hbm_memtest.cuh directly
// (tests/test_gpu_memtest.py).
//
// The product reaches hbm_march_tma only through b2dp_memtest, with its own segments, grid and seed.  This library runs
// one march element at a time over caller-owned segments (torch allocations), with any grid and seed, so a test can
// compare every element's result block, the whole buffer after it and a guard region past each segment with
// tests/memtest_oracle.py at the pipeline edges.  It also maps one physical allocation at two virtual addresses
// (cuMemCreate + two cuMemMap) to show that aliased segments are caught.
//
// The harness refuses a launch that would touch memory outside the segments it was given (a segment that is not a
// whole number of tiles, a last segment larger than the first, a misaligned pointer): it never launches something
// that could fault.
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <string>

#include "hbm_memtest.cuh"

using namespace b2dp;

namespace {

using MarchFn = void (*)(MarchSegs, unsigned int, unsigned long long, uint32_t, uint32_t, ProbeCtl*, ProbeOut*,
                         unsigned long long);
constexpr MarchFn kModes[3] = {hbm_march_tma<kTmaCW, kTmaTileVec, kTmaStages, MARCH_WRITE>,
                               hbm_march_tma<kTmaCW, kTmaTileVec, kTmaStages, MARCH_READ_WRITE>,
                               hbm_march_tma<kTmaCW, kTmaTileVec, kTmaStages, MARCH_READ>};
// element -> (mode, inv, delta): E0 w(P), E1 r(P) w(~P), E2 r(~P) w(P), E3 r(P)
constexpr int kElemMode[kMarchElements] = {MARCH_WRITE, MARCH_READ_WRITE, MARCH_READ_WRITE, MARCH_READ};
constexpr uint32_t kElemInv[kMarchElements] = {0u, 0u, ~0u, 0u};
constexpr uint32_t kElemDelta[kMarchElements] = {0u, ~0u, ~0u, 0u};
constexpr unsigned long long kTileBytes = (unsigned long long)kTmaTileVec * 16;

struct Harness {
    int device = 0;
    int sms = 0;
    cudaStream_t stream = nullptr;
    ProbeCtl* ctl = nullptr;  // one per element
    ProbeOut *out_h = nullptr, *out_d = nullptr;
    std::string err;
};

int fail(Harness* h, const char* what, cudaError_t e) {
    h->err = std::string(what) + ": " + cudaGetErrorName(e) + " (" + cudaGetErrorString(e) + ")";
    return 1;
}

// driver entry points for the aliasing case, without linking libcuda
struct Drv {
    decltype(&cuMemCreate) create = nullptr;
    decltype(&cuMemRelease) release = nullptr;
    decltype(&cuMemAddressReserve) reserve = nullptr;
    decltype(&cuMemAddressFree) addr_free = nullptr;
    decltype(&cuMemMap) map = nullptr;
    decltype(&cuMemUnmap) unmap = nullptr;
    decltype(&cuMemSetAccess) set_access = nullptr;
    decltype(&cuMemGetAllocationGranularity) granularity = nullptr;
};

template <class F>
bool entry(const char* name, F* fn) {
    cudaDriverEntryPointQueryResult q;
    return cudaGetDriverEntryPoint(name, reinterpret_cast<void**>(fn), cudaEnableDefault, &q) == cudaSuccess &&
           q == cudaDriverEntryPointSuccess && *fn;
}

}  // namespace

#define CK(h, x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return fail(h, #x, e_); } while (0)

extern "C" {

enum { MK_OK = 0, MK_E_CUDA = 1, MK_E_ELEM = -1, MK_E_SEGS = -2, MK_E_ALIGN = -3, MK_E_GRID = -4, MK_E_SEQ = -5,
       MK_E_DRIVER = -6 };

const char* mk_error(void* hp) { return static_cast<Harness*>(hp)->err.c_str(); }

void* mk_open(int device, char* errbuf, int errlen) {
    Harness* h = new Harness;
    h->device = device;
    auto init = [h]() -> int {
        CK(h, cudaSetDevice(h->device));
        CK(h, cudaDeviceGetAttribute(&h->sms, cudaDevAttrMultiProcessorCount, h->device));
        CK(h, cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
        CK(h, cudaMalloc(&h->ctl, kMarchElements * sizeof(ProbeCtl)));
        ProbeCtl c[kMarchElements] = {};
        for (auto& x : c) { x.first_bad = ~0ull; x.t_start_ns = ~0ull; }
        CK(h, cudaMemcpy(h->ctl, c, sizeof c, cudaMemcpyHostToDevice));
        CK(h, cudaHostAlloc(&h->out_h, kMarchElements * sizeof(ProbeOut), cudaHostAllocMapped));
        memset(h->out_h, 0, kMarchElements * sizeof(ProbeOut));
        CK(h, cudaHostGetDevicePointer(&h->out_d, h->out_h, 0));
        for (MarchFn fn : kModes) {
            CK(h, cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTmaSmem));
            CK(h, cudaFuncSetAttribute(fn, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
        }
        return MK_OK;
    };
    if (init() != MK_OK) {
        snprintf(errbuf, errlen, "%s", h->err.c_str());
        if (h->out_h) cudaFreeHost(h->out_h);
        if (h->ctl) cudaFree(h->ctl);
        if (h->stream) cudaStreamDestroy(h->stream);
        delete h;
        return nullptr;
    }
    return h;
}

void mk_close(void* hp) {
    Harness* h = static_cast<Harness*>(hp);
    cudaSetDevice(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    if (h->out_h) cudaFreeHost(h->out_h);
    if (h->ctl) cudaFree(h->ctl);
    if (h->stream) cudaStreamDestroy(h->stream);
    delete h;
}

int mk_sms(void* hp) { return static_cast<Harness*>(hp)->sms; }
int mk_tile_bytes() { return (int)kTileBytes; }

// March element `elem` over n_segs segments (device addresses and sizes in bytes) keyed with `seed`; grid 0 = the
// product shape (SMs x kTmaCtasPerSm).  Synchronises, copies the element's result block to *res and checks its seq.
int mk_element(void* hp, const unsigned long long* seg_ptr, const unsigned long long* seg_bytes, int n_segs,
               uint32_t seed, int elem, int grid, unsigned long long seq, ProbeOut* res) {
    Harness* h = static_cast<Harness*>(hp);
    if (elem < 0 || elem >= kMarchElements) return MK_E_ELEM;
    if (n_segs < 1 || n_segs > kMemtestMaxSegments) return MK_E_SEGS;
    if (grid < 0 || grid > (1 << 20)) return MK_E_GRID;
    MarchSegs segs{};
    unsigned long long total = 0;
    for (int g = 0; g < n_segs; ++g) {
        const unsigned long long b = seg_bytes[g];
        // every segment a whole number of tiles; all but the last of one size; the last no larger
        if (b == 0 || b % kTileBytes || (g < n_segs - 1 && b != seg_bytes[0]) || b > seg_bytes[0]) return MK_E_SEGS;
        if (!seg_ptr[g] || seg_ptr[g] % 128) return MK_E_ALIGN;
        segs.base[g] = reinterpret_cast<uint4*>(seg_ptr[g]);
        segs.seed[g] = memtest_segment_seed(seed, (uint32_t)g);
        total += b;
    }
    const unsigned int tiles_per_seg = (unsigned int)(seg_bytes[0] / kTileBytes);
    unsigned long long n_tiles = total / kTileBytes;
    uint32_t inv = kElemInv[elem], delta = kElemDelta[elem];
    ProbeCtl* ctl = h->ctl + elem;
    ProbeOut* out = h->out_d + elem;
    const int g = grid ? grid : h->sms * kTmaCtasPerSm;
    CK(h, cudaSetDevice(h->device));
    void* args[] = {&segs, (void*)&tiles_per_seg, &n_tiles, &inv, &delta, &ctl, &out, &seq};
    CK(h, cudaLaunchKernel(reinterpret_cast<const void*>(kModes[kElemMode[elem]]), dim3(g), dim3((kTmaCW + 1) * 32), args,
                           kTmaSmem, h->stream));
    CK(h, cudaStreamSynchronize(h->stream));
    memcpy(res, (const void*)&h->out_h[elem], sizeof(ProbeOut));
    return res->seq == seq ? MK_OK : MK_E_SEQ;
}

// The control block of element `elem` as its last launch left it (reset to {0, 0, ~0, ~0, 0} by the last CTA).
int mk_read_ctl(void* hp, int elem, ProbeCtl* out) {
    Harness* h = static_cast<Harness*>(hp);
    if (elem < 0 || elem >= kMarchElements) return MK_E_ELEM;
    CK(h, cudaSetDevice(h->device));
    CK(h, cudaStreamSynchronize(h->stream));
    CK(h, cudaMemcpy(out, h->ctl + elem, sizeof(ProbeCtl), cudaMemcpyDeviceToHost));
    return MK_OK;
}

// Resident CTAs per SM of a march mode with the shared memory its launches use.
int mk_occupancy(void* hp, int mode, int* ctas) {
    Harness* h = static_cast<Harness*>(hp);
    if (mode < 0 || mode > 2) return MK_E_ELEM;
    CK(h, cudaSetDevice(h->device));
    CK(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(ctas, reinterpret_cast<const void*>(kModes[mode]),
                                                       (kTmaCW + 1) * 32, kTmaSmem));
    return MK_OK;
}

// One physical allocation of at least `bytes` (rounded up to the granularity), mapped read/write at two virtual
// addresses.  *handle identifies it for mk_alias_free.
struct Alias { Drv d; CUmemGenericAllocationHandle mem = 0; CUdeviceptr va[2] = {0, 0}; size_t size = 0; };

int mk_alias_alloc(void* hp, unsigned long long bytes, unsigned long long* va0, unsigned long long* va1,
                   unsigned long long* size, void** handle) {
    Harness* h = static_cast<Harness*>(hp);
    CK(h, cudaSetDevice(h->device));
    CK(h, cudaFree(nullptr));  // the primary context is current
    Alias* a = new Alias;
    Drv& d = a->d;
    if (!entry("cuMemCreate", &d.create) || !entry("cuMemRelease", &d.release) || !entry("cuMemAddressReserve", &d.reserve) ||
        !entry("cuMemAddressFree", &d.addr_free) || !entry("cuMemMap", &d.map) || !entry("cuMemUnmap", &d.unmap) ||
        !entry("cuMemSetAccess", &d.set_access) || !entry("cuMemGetAllocationGranularity", &d.granularity)) {
        delete a;
        h->err = "driver entry points for virtual memory management not found";
        return MK_E_DRIVER;
    }
    CUmemAllocationProp prop{};
    prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
    prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    prop.location.id = h->device;
    size_t gran = 0;
    if (d.granularity(&gran, &prop, CU_MEM_ALLOC_GRANULARITY_MINIMUM) != CUDA_SUCCESS || !gran) { delete a; return MK_E_DRIVER; }
    a->size = (bytes + gran - 1) / gran * gran;
    bool ok = d.create(&a->mem, a->size, &prop, 0) == CUDA_SUCCESS;
    CUmemAccessDesc acc{};
    acc.location = prop.location;
    acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    for (int k = 0; k < 2 && ok; ++k)
        ok = d.reserve(&a->va[k], a->size, 0, 0, 0) == CUDA_SUCCESS && d.map(a->va[k], a->size, 0, a->mem, 0) == CUDA_SUCCESS &&
             d.set_access(a->va[k], a->size, &acc, 1) == CUDA_SUCCESS;
    *handle = a;
    if (!ok) { h->err = "cuMemCreate / cuMemMap failed"; return MK_E_DRIVER; }
    *va0 = a->va[0];
    *va1 = a->va[1];
    *size = a->size;
    return MK_OK;
}

void mk_alias_free(void* hp, void* handle) {
    Harness* h = static_cast<Harness*>(hp);
    Alias* a = static_cast<Alias*>(handle);
    if (!a) return;
    cudaSetDevice(h->device);
    cudaStreamSynchronize(h->stream);
    for (CUdeviceptr va : a->va)
        if (va) { a->d.unmap(va, a->size); a->d.addr_free(va, a->size); }
    if (a->mem) a->d.release(a->mem);
    delete a;
}

}  // extern "C"
