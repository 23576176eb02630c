// l1_selftest.cuh -- sm_90a self-test kernel of the on-demand L1 self-test (b2dp_l1_test).
//
// Four warps per CTA run the SM's L1TEX unit and its constant cache on data the host built, and compare with values the
// host computed (l1_test_math.hpp).  Every access in the repetition loop is one inline-PTX statement:
//     format    accesses                                                        SASS (CUDA 12.9, DESIGN 4.16)
//     L1_DATA   st.global.v4.u32, then three passes of weak ld.global.v4.u32     STG.E.128, LDG.E.128
//               over the CTA's private span
//     L1_TEX    tex.2d.v4.u32.s32, tex.2d.v4.u32.f32 (unnormalized and in        TLD.LZ, TEX / TEX.LL, TLD4.{R,G,B,A},
//               four normalized address modes), tld4.{r,g,b,a}, ld.global.nc     LDG.E.128.CONSTANT
//     L1_CONST  ld.const.u32 at warp-uniform and lane-divergent indices,         LDC / ULDC, LDC.64, LDC.128
//               ld.const.v2.u32, ld.const.v4.u32 over one 8 KiB window
//
// The round / tile / repetition structure is the other self-tests': a round runs each of the kCtTiles tiles kCtReps
// times and a CTA repeats rounds until its %globaltimer deadline (at least one round).  One comparison is one (tile,
// repetition); the CTA counts it as one mismatch if any thread's value differs from the host's.  There is no wait and no
// barrier across CTAs: every CTA works on its own span, or reads data nothing writes during the launch.
//   L1_DATA:  the thread's sum fold must equal l1_data_want (K x the host's check, by polarity) and every value read must
//             equal P ^ inv directly (a stuck bit 31 cancels in a sum fold).
//   L1_TEX / L1_CONST:  the thread's it_fold of its result words must equal the host's check.
// The texture and read-only paths are only read: a texture read of data written in the same launch is undefined.
//
// Fault hook: in the first comparison of a CTA whose %smid == fault_sm, L1_DATA's thread 0 XORs fault_mask into word
// kL1HookWord of its span after the write (every pass then reads it wrong); L1_TEX / L1_CONST's thread 0 XORs it into its
// first result word.  DUMP (the test harness only, its area at scratch word hdr[kL1HdrDump]) makes CTA 0 write every
// value it read in round 0, repetition 0 of every tile: [tile][thread][3 K x 4] for L1_DATA (pass, step, word; raw),
// [tile][thread][l1_words(FMT)] for the others.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "hbm_probe.cuh"  // globaltimer_ns
#include "l1_test_math.hpp"

// The constant bank: the only __constant__ array of the library (ptxas: cmem[3], 32768 bytes).  At global scope, so the
// inline PTX names it unmangled; the driver loads it per call (cudaMemcpyToSymbolAsync).
__constant__ uint32_t b2dp_l1_bank[b2dp::kL1BankWords];

namespace b2dp {

__device__ __forceinline__ void l1_st128(uint32_t* p, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    asm volatile("st.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ uint4 l1_ld128(const uint32_t* p) {
    uint4 v;
    asm volatile("ld.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p)
                 : "memory");
    return v;
}
__device__ __forceinline__ uint32_t l1_ld32(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void l1_st32(uint32_t* p, uint32_t v) {
    asm volatile("st.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint4 l1_ldnc128(const uint32_t* p) {
    uint4 v;
    asm volatile("ld.global.nc.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ uint4 l1_tld(unsigned long long h, int x, int y) {
    uint4 v;
    asm volatile("tex.2d.v4.u32.s32 {%0, %1, %2, %3}, [%4, {%5, %6}];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(h), "r"(x), "r"(y));
    return v;
}
__device__ __forceinline__ uint4 l1_tex(unsigned long long h, float u, float w) {
    uint4 v;
    asm volatile("tex.2d.v4.u32.f32 {%0, %1, %2, %3}, [%4, {%5, %6}];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(h), "f"(u), "f"(w));
    return v;
}
template <int C>
__device__ __forceinline__ uint4 l1_tld4(unsigned long long h, float u, float w) {
    uint4 v;
    if constexpr (C == 0)
        asm volatile("tld4.r.2d.v4.u32.f32 {%0, %1, %2, %3}, [%4, {%5, %6}];"
                     : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(h), "f"(u), "f"(w));
    else if constexpr (C == 1)
        asm volatile("tld4.g.2d.v4.u32.f32 {%0, %1, %2, %3}, [%4, {%5, %6}];"
                     : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(h), "f"(u), "f"(w));
    else if constexpr (C == 2)
        asm volatile("tld4.b.2d.v4.u32.f32 {%0, %1, %2, %3}, [%4, {%5, %6}];"
                     : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(h), "f"(u), "f"(w));
    else
        asm volatile("tld4.a.2d.v4.u32.f32 {%0, %1, %2, %3}, [%4, {%5, %6}];"
                     : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(h), "f"(u), "f"(w));
    return v;
}
// Constant loads at word i of the bank (masked to it).
__device__ __forceinline__ uint32_t l1_ldc(uint32_t i) {
    uint32_t d;
    asm volatile("{ .reg .u64 a; mov.u64 a, b2dp_l1_bank; mad.wide.u32 a, %1, 4, a; ld.const.u32 %0, [a]; }"
                 : "=r"(d) : "r"(i & (uint32_t)(kL1BankWords - 1)));
    return d;
}
__device__ __forceinline__ uint2 l1_ldc64(uint32_t i) {
    uint2 d;
    asm volatile("{ .reg .u64 a; mov.u64 a, b2dp_l1_bank; mad.wide.u32 a, %2, 4, a; ld.const.v2.u32 {%0, %1}, [a]; }"
                 : "=r"(d.x), "=r"(d.y) : "r"(i & (uint32_t)(kL1BankWords - 2)));
    return d;
}
__device__ __forceinline__ uint4 l1_ldc128(uint32_t i) {
    uint4 d;
    asm volatile("{ .reg .u64 a; mov.u64 a, b2dp_l1_bank; mad.wide.u32 a, %4, 4, a; "
                 "ld.const.v4.u32 {%0, %1, %2, %3}, [a]; }"
                 : "=r"(d.x), "=r"(d.y), "=r"(d.z), "=r"(d.w) : "r"(i & (uint32_t)(kL1BankWords - 4)));
    return d;
}

// A thread's it_fold over result words that arrive four at a time (word j enters chain j % 4), with the fault hook on
// the first word and the DUMP.
template <bool DUMP>
struct L1Sink {
    static constexpr uint32_t i0 = kItFoldInit[0], i1 = kItFoldInit[1], i2 = kItFoldInit[2], i3 = kItFoldInit[3];
    uint32_t h[4] = {i0, i1, i2, i3};
    uint32_t inj = 0;
    uint32_t* dump = nullptr;
    __device__ __forceinline__ void take(int c, uint32_t w) {
        const uint32_t x = (h[c] ^ w) * kItMul;
        h[c] = __funnelshift_l(x, x, kItFoldRot);
    }
    __device__ __forceinline__ void emit4(uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
        a ^= inj;
        inj = 0;
        if (DUMP && dump) { dump[0] = a; dump[1] = b; dump[2] = c; dump[3] = d; dump += 4; }
        take(0, a); take(1, b); take(2, c); take(3, d);
    }
    __device__ __forceinline__ void emit4(uint4 v) { emit4(v.x, v.y, v.z, v.w); }
    __device__ __forceinline__ uint32_t value() const {
        return h[0] ^ __funnelshift_l(h[1], h[1], 8) ^ __funnelshift_l(h[2], h[2], 16) ^ __funnelshift_l(h[3], h[3], 24);
    }
};

// table: kCtTiles tables of kL1TableWords words; checks: [kCtTiles][kCtThreads]; rec: one per CTA; scratch: the header,
// then the spans (L1_DATA) or the linear copy of the texel image (L1_TEX).  Block: kCtThreads threads, no dynamic shared
// memory.  Same signature as tc_selftest.
template <int FMT, bool DUMP>
__global__ void __launch_bounds__(kCtThreads)
l1_selftest(const uint8_t* __restrict__ table, const uint32_t* __restrict__ checks, unsigned long long duration_ns,
            int fault_sm, uint32_t fault_mask, CtRecord* rec, unsigned long long seq, uint32_t* scratch) {
    const int tid = threadIdx.x;
    uint32_t smid, nsmid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    asm volatile("mov.u32 %0, %%nsmid;" : "=r"(nsmid));
    const unsigned long long t_end = globaltimer_ns() + duration_ns;
    const bool hook_sm = (int)smid == fault_sm;
    const uint32_t* hdr = scratch;
    uint32_t* data = scratch + kL1DataOff;
    uint32_t* dump = DUMP ? scratch + __ldg(hdr + kL1HdrDump) : nullptr;
    const uint32_t* tab = reinterpret_cast<const uint32_t*>(table);
    unsigned long long rounds = 0, comparisons = 0, mismatches = 0;
    int bad_tile = -1, bad_rep = -1;
    for (;;) {
        for (int tile = 0; tile < kCtTiles; ++tile) {
            const uint32_t* tt = tab + tile * kL1TableWords;
            const uint32_t want = __ldg(checks + tile * kCtThreads + tid);
            const bool dump_tile = DUMP && blockIdx.x == 0 && rounds == 0;
            if constexpr (FMT == L1_DATA) {
                const uint32_t K = __ldg(hdr + kL1HdrBlocks);
                const uint32_t kind = __ldg(tt), key = __ldg(tt + 1), linemul = __ldg(tt + 2), hook = __ldg(tt + 3);
                uint32_t* span = data + (size_t)blockIdx.x * K * kL1BlockWords;
                const uint32_t line0 = blockIdx.x * K * (kL1BlockWords / kL1LineWords);
                uint32_t pw[4], pr[kL1Passes][4];
#pragma unroll
                for (int i = 0; i < 4; ++i) pw[i] = sh_pattern(kind, key, (uint32_t)(4 * tid + i));
#pragma unroll
                for (int p = 0; p < kL1Passes; ++p)
#pragma unroll
                    for (int i = 0; i < 4; ++i)
                        pr[p][i] = sh_pattern(kind, key, (uint32_t)(4 * l1_data_writer(tid, p) + i));
                for (int rep = 0; rep < kCtReps; ++rep) {
                    const uint32_t inv = (rep & 1) ? ~0u : 0u;
#pragma unroll 4
                    for (uint32_t b = 0; b < K; ++b) {
                        const uint32_t lk = l1_line_key(linemul, line0 + b * 16u + (uint32_t)tid / 8u) ^ inv;
                        l1_st128(span + (size_t)b * kL1BlockWords + 4 * tid, pw[0] ^ lk, pw[1] ^ lk, pw[2] ^ lk,
                                 pw[3] ^ lk);
                    }
                    __syncthreads();  // the CTA's stores are visible to its loads
                    if ((rounds | (unsigned)tile | (unsigned)rep) == 0 && hook_sm) {
                        if (tid == 0) {
                            uint32_t* p = span + hook % (K * (uint32_t)kL1BlockWords);
                            l1_st32(p, l1_ld32(p) ^ fault_mask);
                        }
                        __syncthreads();
                    }
                    uint32_t h = 0, err = 0;
                    uint32_t* d = (dump_tile && rep == 0)
                                      ? dump + ((size_t)tile * kCtThreads + tid) * kL1Passes * K * 4 : nullptr;
#pragma unroll
                    for (int p = 0; p < kL1Passes; ++p) {
                        const int wr = l1_data_writer(tid, p);
#pragma unroll 1
                        for (uint32_t s0 = 0; s0 < K; s0 += 4) {
                            uint4 v[4];
                            uint32_t bl[4];
#pragma unroll
                            for (int q = 0; q < 4; ++q) {
                                bl[q] = s0 + q < K ? l1_data_block(p, s0 + q, K) : 0u;
                                if (s0 + q < K) v[q] = l1_ld128(span + (size_t)bl[q] * kL1BlockWords + 4 * wr);
                            }
#pragma unroll
                            for (int q = 0; q < 4; ++q) {
                                if (s0 + q >= K) break;
                                const uint32_t lk = l1_line_key(linemul, line0 + bl[q] * 16u + (uint32_t)wr / 8u);
                                const uint32_t got[4] = {v[q].x, v[q].y, v[q].z, v[q].w};
#pragma unroll
                                for (int i = 0; i < 4; ++i) {
                                    const uint32_t x = got[i] ^ lk;
                                    h += (uint32_t)(8 * p + 2 * i + 1) * x;
                                    err += x != (pr[p][i] ^ inv);
                                    if (DUMP && d) d[((size_t)p * K + s0 + q) * 4 + i] = got[i];
                                }
                            }
                        }
                    }
                    // an empty span (K = 0) reads nothing and folds to 0: it counts as a mismatch, never as a pass
                    const int bad = __syncthreads_or(K == 0 || err != 0 || h != l1_data_want(want, K, rep));
                    ++comparisons;
                    if (bad && mismatches++ == 0) { bad_tile = tile; bad_rep = rep; }
                }
            } else if constexpr (FMT == L1_TEX) {
                const unsigned long long* ho = reinterpret_cast<const unsigned long long*>(hdr + kL1HdrTex);
                const unsigned long long h0 = __ldg(ho), h1 = __ldg(ho + 1), h2 = __ldg(ho + 2), h3 = __ldg(ho + 3),
                                         h4 = __ldg(ho + 4);
                const uint32_t A = __ldg(tt), B = __ldg(tt + 1), D = __ldg(tt + 2);
                for (int rep = 0; rep < kCtReps; ++rep) {
                    L1Sink<DUMP> k;
                    k.inj = (rounds | (unsigned)tile | (unsigned)rep) == 0 && hook_sm && tid == 0 ? fault_mask : 0u;
                    k.dump = (dump_tile && rep == 0) ? dump + ((size_t)tile * kCtThreads + tid) * l1_words(FMT)
                                                     : nullptr;
#pragma unroll 1
                    for (int j0 = 0; j0 < kL1TexSteps; j0 += 4) {
#pragma unroll
                        for (int c = 0; c < 4; ++c) {
                            const int j = j0 + c;
                            const uint32_t i = l1_tex_index(A, B, tid, j);
                            const int x = (int)(i % kL1TexW), y = (int)(i / kL1TexW);
                            const float u = (float)x + 0.5f, w = (float)y + 0.5f;
                            const float un = u * (1.0f / kL1TexW), wn = w * (1.0f / kL1TexH);
                            const float mx = (float)l1_tex_mx(D, tid, j), my = (float)l1_tex_my(D, tid, j);
                            k.emit4(l1_tld(h0, x, y));
                            k.emit4(l1_tex(h0, u, w));
                            k.emit4(l1_tex(h1, un + mx, wn + my));
                            k.emit4(l1_tex(h2, un + mx, wn + my));
                            k.emit4(l1_tex(h3, un + mx, wn + my));
                            k.emit4(l1_tex(h4, un + mx, wn + my));
                            if (c == 0) k.emit4(l1_tld4<0>(h0, u, w));
                            else if (c == 1) k.emit4(l1_tld4<1>(h0, u, w));
                            else if (c == 2) k.emit4(l1_tld4<2>(h0, u, w));
                            else k.emit4(l1_tld4<3>(h0, u, w));
                            k.emit4(l1_ldnc128(data + 4 * (i & (uint32_t)(kL1Texels - 1))));
                        }
                    }
                    const int bad = __syncthreads_or(k.value() != want);
                    ++comparisons;
                    if (bad && mismatches++ == 0) { bad_tile = tile; bad_rep = rep; }
                }
            } else {
                const uint32_t base = (__ldg(tt) & (uint32_t)(kL1Windows - 1)) * kL1WindowWords, rot = __ldg(tt + 1);
                const int w = tid / 32, l = tid % 32;
                for (int rep = 0; rep < kCtReps; ++rep) {
                    L1Sink<DUMP> k;
                    k.inj = (rounds | (unsigned)tile | (unsigned)rep) == 0 && hook_sm && tid == 0 ? fault_mask : 0u;
                    k.dump = (dump_tile && rep == 0) ? dump + ((size_t)tile * kCtThreads + tid) * l1_words(FMT)
                                                     : nullptr;
#pragma unroll 2
                    for (int q = 0; q < kL1ConstUni; q += 4)
                        k.emit4(l1_ldc(base + l1_const_uni(rot, w, q)), l1_ldc(base + l1_const_uni(rot, w, q + 1)),
                                l1_ldc(base + l1_const_uni(rot, w, q + 2)), l1_ldc(base + l1_const_uni(rot, w, q + 3)));
#pragma unroll 2
                    for (int q = 0; q < kL1ConstDiv; q += 4)
                        k.emit4(l1_ldc(base + l1_const_div(rot, w, l, q)), l1_ldc(base + l1_const_div(rot, w, l, q + 1)),
                                l1_ldc(base + l1_const_div(rot, w, l, q + 2)),
                                l1_ldc(base + l1_const_div(rot, w, l, q + 3)));
#pragma unroll 2
                    for (int q = 0; q < kL1ConstV2; q += 2) {
                        const uint2 a = l1_ldc64(base + l1_const_v2(rot, w, l, q));
                        const uint2 b = l1_ldc64(base + l1_const_v2(rot, w, l, q + 1));
                        k.emit4(a.x, a.y, b.x, b.y);
                    }
#pragma unroll 2
                    for (int q = 0; q < kL1ConstV4; ++q) k.emit4(l1_ldc128(base + l1_const_v4(rot, w, l, q)));
                    const int bad = __syncthreads_or(k.value() != want);
                    ++comparisons;
                    if (bad && mismatches++ == 0) { bad_tile = tile; bad_rep = rep; }
                }
            }
        }
        ++rounds;
        if (__syncthreads_or(tid == 0 && globaltimer_ns() >= t_end)) break;
    }
    if (tid == 0) {
        volatile CtRecord* r = rec + blockIdx.x;
        r->smid = smid;
        r->nsmid = nsmid;
        r->rounds = rounds;
        r->comparisons = comparisons;
        r->mismatches = mismatches;
        r->first_bad_tile = bad_tile;
        r->first_bad_rep = bad_rep;
        __threadfence_system();
        r->seq = seq;
    }
}

// ---- the host objects the kernel reads: the CUDA array, its texture objects and the constant bank ------------------
// Made before the launches that read them, released after the stream is synchronized (the driver's bind / unbind and
// the test harness).
struct L1Bound {
    cudaArray_t array = nullptr;
    cudaTextureObject_t tex[kL1TexObjs] = {};
};

inline void l1_unbind(L1Bound& b) {
    for (cudaTextureObject_t& t : b.tex)
        if (t) { cudaDestroyTextureObject(t); t = 0; }
    if (b.array) { cudaFreeArray(b.array); b.array = nullptr; }
}

// Fills the array and the linear copy at tex_scratch + kL1DataOff with seed's image, writes the texture handles into
// tex_scratch's header (if tex_scratch is set) and loads the constant bank with seed's windows, all on `stream`.  On an
// error *where names the call; what was made is left in b for l1_unbind.
inline cudaError_t l1_bind(uint32_t seed, uint32_t* tex_scratch, cudaStream_t stream, L1Bound& b, const char** where) {
    std::vector<uint32_t> img((size_t)kL1Texels * 4), bank(kL1BankWords);
    l1_tex_image(seed, img.data());
    l1_bank(seed, bank.data());
    cudaError_t ce;
#define L1_TRY(x) if ((ce = (x)) != cudaSuccess) { *where = #x; return ce; }
    // The caller wrote the scratch header with cudaMemset / cudaMemcpy on the legacy stream, which a non-blocking
    // `stream` is not ordered after, and a pageable cudaMemcpy may return before its data lands: finish them first, so
    // the handles written below are not overwritten by the header's zeros.
    L1_TRY(cudaStreamSynchronize(cudaStreamLegacy));
    L1_TRY(cudaMemcpyToSymbolAsync(b2dp_l1_bank, bank.data(), bank.size() * 4, 0, cudaMemcpyHostToDevice, stream));
    if (tex_scratch) {
        const cudaChannelFormatDesc ch = cudaCreateChannelDesc<uint4>();
        L1_TRY(cudaMallocArray(&b.array, &ch, kL1TexW, kL1TexH));
        L1_TRY(cudaMemcpy2DToArrayAsync(b.array, 0, 0, img.data(), kL1TexW * 16, kL1TexW * 16, kL1TexH,
                                        cudaMemcpyHostToDevice, stream));
        L1_TRY(cudaMemcpyAsync(tex_scratch + kL1DataOff, img.data(), img.size() * 4, cudaMemcpyHostToDevice, stream));
        cudaResourceDesc rd = {};
        rd.resType = cudaResourceTypeArray;
        rd.res.array.array = b.array;
        const cudaTextureAddressMode modes[kL1TexObjs] = {cudaAddressModeClamp, cudaAddressModeWrap,
                                                          cudaAddressModeMirror, cudaAddressModeClamp,
                                                          cudaAddressModeBorder};
        for (int i = 0; i < kL1TexObjs; ++i) {
            cudaTextureDesc td = {};
            td.addressMode[0] = td.addressMode[1] = modes[i];
            td.filterMode = cudaFilterModePoint;
            td.readMode = cudaReadModeElementType;
            td.normalizedCoords = i > 0;
            L1_TRY(cudaCreateTextureObject(&b.tex[i], &rd, &td, nullptr));
        }
        unsigned long long h[kL1TexObjs];
        for (int i = 0; i < kL1TexObjs; ++i) h[i] = (unsigned long long)b.tex[i];
        if (!l1_handles_ok(h)) { *where = "cudaCreateTextureObject (a zero handle)"; return cudaErrorInvalidValue; }
        L1_TRY(cudaMemcpyAsync(tex_scratch + kL1HdrTex, h, sizeof h, cudaMemcpyHostToDevice, stream));
    }
    // the host vectors go out of scope: the copies from them must be done
    L1_TRY(cudaStreamSynchronize(stream));
#undef L1_TRY
    return cudaSuccess;
}

}  // namespace b2dp
