// probe_sweep.cu — standalone tuning harness for the hbm_probe kernel variants.
// Not part of the product path: it instantiates the kernels in hbm_probe.cuh
// over a grid of launch shapes, times each with CUDA events (3 warm-ups, K
// timed launches, inputs 1 GiB >> 50 MB L2) and checks checksum/mismatches
// against the closed-form CPU value. Output: CSV on stdout.
// --gap [ROUNDS] runs the attribution ladder instead (run_gap below, tools/README.md).
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 \
//        -I k8s-device-plugin_b200/csrc tools/probe_sweep.cu -o tools/probe_sweep
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include <algorithm>
#include "hbm_probe.cuh"

using namespace b2dp;

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { \
    fprintf(stderr, "CUDA error %s at %s:%d: %s\n", #x, __FILE__, __LINE__, cudaGetErrorString(e_)); exit(2); } } while (0)

static unsigned long long cpu_checksum(unsigned long long n_words, uint32_t seed) {
    unsigned long long s = 0;
    for (unsigned long long i = 0; i < n_words; ++i) s += (uint32_t)((uint32_t)i * kPatternMul) ^ seed;
    return s;
}

struct Bufs {
    uint4 *a, *b; unsigned long long n_vec; ProbeCtl* ctl; ProbeOut* out_h; ProbeOut* out_d;
    uint32_t seed; int cur;  // cur: which buffer holds pattern(seed)
};

using LaunchFn = void (*)(const uint4*, uint4*, unsigned long long, uint32_t, uint32_t, ProbeCtl*, ProbeOut*,
                          unsigned long long, int grid, cudaStream_t);

template <int T, int U> static void launch_r128(const uint4* s, uint4* d, unsigned long long n, uint32_t seed,
    uint32_t delta, ProbeCtl* c, ProbeOut* o, unsigned long long seq, int grid, cudaStream_t st) {
    hbm_probe_r128<T, U><<<grid, T, 0, st>>>(s, d, n, seed, delta, c, o, seq);
}
template <int T, int U> static void launch_r256(const uint4* s, uint4* d, unsigned long long n, uint32_t seed,
    uint32_t delta, ProbeCtl* c, ProbeOut* o, unsigned long long seq, int grid, cudaStream_t st) {
    hbm_probe_r256<T, U><<<grid, T, 0, st>>>(s, d, n, seed, delta, c, o, seq);
}
template <int CW, int TV, int ST, int HINT = 0> static void launch_tma(const uint4* s, uint4* d, unsigned long long n, uint32_t seed,
    uint32_t delta, ProbeCtl* c, ProbeOut* o, unsigned long long seq, int grid, cudaStream_t st) {
    constexpr size_t smem = (size_t)ST * TV * 16 + 2 * ST * 8;
    static bool once = false;
    if (!once) { CK(cudaFuncSetAttribute(hbm_probe_tma<CW, TV, ST, HINT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); once = true; }
    hbm_probe_tma<CW, TV, ST, HINT><<<grid, (CW + 1) * 32, smem, st>>>(s, d, n, seed, delta, c, o, seq);
}

static unsigned int g_period_ns = 0;
template <int CW, int TV, int ST> static void launch_phased(const uint4* s, uint4* d, unsigned long long n, uint32_t seed,
    uint32_t delta, ProbeCtl* c, ProbeOut* o, unsigned long long seq, int grid, cudaStream_t st);

__global__ void plain_copy(const uint4* __restrict__ s, uint4* __restrict__ d, unsigned long long n) {
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
         i += (unsigned long long)gridDim.x * blockDim.x) d[i] = s[i];
}

// ---- ceilings: what pure reads and pure writes reach on this part (tool-only kernels) ---------
// sink[0 .. kSinks) accumulate the sum of the words of every full chunk (the whole buffer when n is a multiple of the chunk)
constexpr int kSinks = 64;
template <int U>
__global__ void read_only(const uint4* __restrict__ s, unsigned long long n, unsigned long long* sink) {
    unsigned long long acc = 0;
    const unsigned long long chunk = (unsigned long long)blockDim.x * U, n_full = n / chunk;
    for (unsigned long long c = blockIdx.x; c < n_full; c += gridDim.x) {
        uint4 v[U];
#pragma unroll
        for (int u = 0; u < U; ++u) v[u] = ldg_na(s + c * chunk + threadIdx.x + (unsigned long long)u * blockDim.x);
#pragma unroll
        for (int u = 0; u < U; ++u) acc += (unsigned long long)v[u].x + v[u].y + v[u].z + v[u].w;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) atomicAdd(&sink[blockIdx.x % kSinks], acc);  // spread: same-address atomics serialise
}
__global__ void write_only(uint4* __restrict__ d, unsigned long long n, uint32_t seed) {
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
         i += (unsigned long long)gridDim.x * blockDim.x) {
        const uint32_t m0 = (uint32_t)(i * 4ull) * kPatternMul;
        stg_na(d + i, make_uint4(m0 ^ seed, (m0 + kPatternMul) ^ seed, (m0 + 2u * kPatternMul) ^ seed, (m0 + 3u * kPatternMul) ^ seed));
    }
}
// bulk-copy read-only: the ring is filled and drained without any store
template <int TILE_VEC, int STAGES>
__global__ void __launch_bounds__(160) read_only_tma(const uint4* __restrict__ src, unsigned long long n_vec, unsigned long long* sink) {
    constexpr uint32_t TILE_BYTES = TILE_VEC * 16u;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    uint4* tiles = reinterpret_cast<uint4*>(smem_raw);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + (size_t)STAGES * TILE_BYTES);
    uint64_t* done = full + STAGES;
    const unsigned long long n_tiles = n_vec / TILE_VEC;
    const unsigned long long my_tiles = n_tiles > blockIdx.x ? (n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&done[s], 128); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        fence_proxy_async_smem();
    }
    __syncthreads();
    unsigned long long acc = 0;
    if (threadIdx.x < 32) {
        if (threadIdx.x == 0) {
            for (unsigned long long k = 0; k < my_tiles; ++k) {
                const int slot = (int)(k % STAGES);
                if (k >= STAGES) mbar_wait(&done[slot], (uint32_t)(((k / STAGES) - 1) & 1));
                mbar_expect_tx(&full[slot], TILE_BYTES);
                bulk_g2s(tiles + (size_t)slot * TILE_VEC, src + (blockIdx.x + k * gridDim.x) * TILE_VEC, TILE_BYTES, &full[slot]);
            }
        }
    } else {
        const int ct = threadIdx.x - 32;
        for (unsigned long long k = 0; k < my_tiles; ++k) {
            const int slot = (int)(k % STAGES);
            mbar_wait(&full[slot], (uint32_t)((k / STAGES) & 1));
            const uint4* tile = tiles + (size_t)slot * TILE_VEC;
#pragma unroll
            for (int u = 0; u < TILE_VEC / 128; ++u) { uint4 v = tile[ct + u * 128]; acc += (unsigned long long)v.x + v.y + v.z + v.w; }
            mbar_arrive(&done[slot]);
        }
    }
    if (acc == 0x123456789abcdefull) *sink = acc;
}

// ---- experiment: chip-wide read/write phase separation (tool-only) ----------------------------
// Pure reads run at 7.08 TB/s and pure writes at 7.07 TB/s on this part, a mixed copy at 6.49.
// Here every CTA (1 per SM, a 12 x 16 KiB ring) alternates "load the whole ring" / "store the
// whole ring", and the two windows are aligned across the chip with %globaltimer (period_ns;
// 0 = free-running batches).  Measures whether SM-side phasing can lift the mixed-copy ceiling.
template <int CW, int TILE_VEC, int STAGES>
__global__ void __launch_bounds__((CW + 1) * 32)
hbm_probe_phased(const uint4* __restrict__ src, uint4* __restrict__ dst, unsigned long long n_vec, uint32_t seed,
                 uint32_t delta, ProbeCtl* ctl, ProbeOut* out, unsigned long long seq, unsigned int period_ns) {
    constexpr int THREADS = (CW + 1) * 32, CT = CW * 32, PER_THREAD = TILE_VEC / CT;
    constexpr uint32_t TILE_BYTES = TILE_VEC * 16u;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    uint4* tiles = reinterpret_cast<uint4*>(smem_raw);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + (size_t)STAGES * TILE_BYTES);
    uint64_t* done = full + STAGES;
    const unsigned long long t0 = globaltimer_ns();
    const unsigned long long n_tiles = n_vec / TILE_VEC;
    const unsigned long long my_tiles = n_tiles > blockIdx.x ? (n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&done[s], CT); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        fence_proxy_async_smem();
    }
    __syncthreads();
    Acc a;
    if (threadIdx.x < 32) {
        if (threadIdx.x == 0) {
            unsigned int batch = 0;
            for (unsigned long long k0 = 0; k0 < my_tiles; k0 += STAGES, ++batch) {
                const int nb = (int)(my_tiles - k0 < (unsigned long long)STAGES ? my_tiles - k0 : STAGES);
                if (period_ns) while ((globaltimer_ns() % period_ns) >= period_ns / 2) { }   // READ window
                for (int j = 0; j < nb; ++j) {
                    mbar_expect_tx(&full[j], TILE_BYTES);
                    bulk_g2s(tiles + (size_t)j * TILE_VEC, src + (blockIdx.x + (k0 + j) * gridDim.x) * TILE_VEC, TILE_BYTES, &full[j]);
                }
                if (period_ns) while ((globaltimer_ns() % period_ns) < period_ns / 2) { }    // WRITE window
                for (int j = 0; j < nb; ++j) {
                    mbar_wait(&done[j], batch & 1u);
                    bulk_s2g(dst + (blockIdx.x + (k0 + j) * gridDim.x) * TILE_VEC, tiles + (size_t)j * TILE_VEC, TILE_BYTES);
                }
                bulk_commit();
                bulk_wait_read<0>();
            }
            bulk_wait_all<0>();
        }
    } else {
        const int ct = threadIdx.x - 32;
        unsigned int batch = 0;
        for (unsigned long long k0 = 0; k0 < my_tiles; k0 += STAGES, ++batch) {
            const int nb = (int)(my_tiles - k0 < (unsigned long long)STAGES ? my_tiles - k0 : STAGES);
            for (int j = 0; j < nb; ++j) {
                mbar_wait(&full[j], batch & 1u);
                uint4* tile = tiles + (size_t)j * TILE_VEC;
                const unsigned long long t = blockIdx.x + (k0 + j) * gridDim.x;
                uint4 v[PER_THREAD];
#pragma unroll
                for (int u = 0; u < PER_THREAD; ++u) v[u] = tile[ct + u * CT];
#pragma unroll
                for (int u = 0; u < PER_THREAD; ++u) { check4(v[u], t * TILE_VEC + ct + u * CT, seed, delta, a); tile[ct + u * CT] = v[u]; }
                fence_proxy_async_smem();
                mbar_arrive(&done[j]);
            }
        }
    }
    for (unsigned long long i = n_tiles * TILE_VEC + (unsigned long long)blockIdx.x * THREADS + threadIdx.x; i < n_vec;
         i += (unsigned long long)gridDim.x * THREADS) { uint4 v = ldg_na(src + i); check4(v, i, seed, delta, a); stg_na(dst + i, v); }
    finish<THREADS>(a, ctl, out, seq, t0);
}

struct Cfg { std::string name; LaunchFn fn; int ctas_per_sm; };

template <int CW, int TV, int ST> static void launch_phased(const uint4* s, uint4* d, unsigned long long n, uint32_t seed,
    uint32_t delta, ProbeCtl* c, ProbeOut* o, unsigned long long seq, int grid, cudaStream_t st) {
    constexpr size_t smem = (size_t)ST * TV * 16 + 2 * ST * 8;
    static bool once = false;
    if (!once) { CK(cudaFuncSetAttribute(hbm_probe_phased<CW, TV, ST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); once = true; }
    hbm_probe_phased<CW, TV, ST><<<grid, (CW + 1) * 32, smem, st>>>(s, d, n, seed, delta, c, o, seq, g_period_ns);
}

// ---- --gap candidates that lost to hbm_probe_queue (tool-only; profiles/README.md has their rates) --------------
// ===========================================================================
// Variant TMA, split roles: the same ring as hbm_probe_tma, but loads and stores are issued by
// different warps, so a refill never waits behind a store.
//   warp 0 lane 0 = loader : wait empty[s] -> expect_tx full[s] -> bulk load tile into s
//   warp 1 lane 0 = storer : wait done[s]  -> bulk store s -> wait until it has read s -> arrive empty[s]
//   warps 2..CW+1 = verifiers, exactly as in hbm_probe_tma
// Dynamic smem = STAGES*TILE_VEC*16 + 3*STAGES*8.
// ===========================================================================
constexpr size_t split_smem_bytes(int tile_vec, int stages) { return (size_t)stages * tile_vec * 16 + 3 * stages * 8; }

template <int CW, int TILE_VEC, int STAGES>
__global__ void __launch_bounds__((CW + 2) * 32)
hbm_probe_split(const uint4* __restrict__ src, uint4* __restrict__ dst, unsigned long long n_vec,
                uint32_t seed, uint32_t delta, ProbeCtl* ctl, ProbeOut* out, unsigned long long seq) {
    constexpr int THREADS = (CW + 2) * 32;
    constexpr int CT = CW * 32;
    static_assert(TILE_VEC % CT == 0, "tile must be a multiple of the verifier width");
    static_assert(STAGES >= 2, "need >=2 stages");
    constexpr int PER_THREAD = TILE_VEC / CT;
    constexpr uint32_t TILE_BYTES = TILE_VEC * 16u;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    uint4* tiles = reinterpret_cast<uint4*>(smem_raw);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + (size_t)STAGES * TILE_BYTES);
    uint64_t* done = full + STAGES;
    uint64_t* empty = done + STAGES;

    const unsigned long long t0 = globaltimer_ns();
    const unsigned long long n_tiles = n_vec / TILE_VEC;
    const unsigned long long my_tiles =
        n_tiles > blockIdx.x ? (n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;

    if (threadIdx.x == 0) {
#pragma unroll
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&done[s], CT); mbar_init(&empty[s], 1); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        fence_proxy_async_smem();
    }
    __syncthreads();

    Acc a;
    if (threadIdx.x == 0) {
        for (unsigned long long k = 0; k < my_tiles; ++k) {
            const int slot = (int)(k % STAGES);
            if (k >= STAGES) mbar_wait(&empty[slot], (uint32_t)((k / STAGES - 1) & 1));
            mbar_expect_tx(&full[slot], TILE_BYTES);
            bulk_g2s(tiles + (size_t)slot * TILE_VEC, src + (blockIdx.x + k * gridDim.x) * TILE_VEC, TILE_BYTES, &full[slot]);
        }
    } else if (threadIdx.x == 32) {
        for (unsigned long long k = 0; k < my_tiles; ++k) {
            const int slot = (int)(k % STAGES);
            mbar_wait(&done[slot], (uint32_t)((k / STAGES) & 1));
            bulk_s2g(dst + (blockIdx.x + k * gridDim.x) * TILE_VEC, tiles + (size_t)slot * TILE_VEC, TILE_BYTES);
            bulk_commit();
            bulk_wait_read<0>();  // the store no longer reads the slot: hand it back to the loader
            mbar_arrive(&empty[slot]);
        }
        bulk_wait_all<0>();
    } else if (threadIdx.x >= 64) {
        const int ct = threadIdx.x - 64;
        for (unsigned long long k = 0; k < my_tiles; ++k) {
            const int slot = (int)(k % STAGES);
            const unsigned long long t = blockIdx.x + k * gridDim.x;
            mbar_wait(&full[slot], (uint32_t)((k / STAGES) & 1));
            uint4* tile = tiles + (size_t)slot * TILE_VEC;
            uint4 v[PER_THREAD];
#pragma unroll
            for (int u = 0; u < PER_THREAD; ++u) v[u] = tile[ct + u * CT];
#pragma unroll
            for (int u = 0; u < PER_THREAD; ++u) {
                check4(v[u], t * TILE_VEC + ct + u * CT, seed, delta, a);
                tile[ct + u * CT] = v[u];
            }
            fence_proxy_async_smem();
            mbar_arrive(&done[slot]);
        }
    }

    for (unsigned long long i = n_tiles * TILE_VEC + (unsigned long long)blockIdx.x * THREADS + threadIdx.x;
         i < n_vec; i += (unsigned long long)gridDim.x * THREADS) {
        uint4 v = ldg_na(src + i);
        check4(v, i, seed, delta, a);
        stg_na(dst + i, v);
    }
    finish<THREADS>(a, ctl, out, seq, t0);
}

// ===========================================================================
// Variant PIPE: register path, software-pipelined. Each thread loads chunk c+grid while it
// verifies and stores chunk c, so UNROLL 16-byte loads per thread stay in flight across the
// verify and the stores. The accesses are plain (not asm volatile): the compiler may overlap them.
// ===========================================================================
template <int THREADS, int UNROLL>
__global__ void __launch_bounds__(THREADS)
hbm_probe_pipe(const uint4* __restrict__ src, uint4* __restrict__ dst, unsigned long long n_vec,
               uint32_t seed, uint32_t delta, ProbeCtl* ctl, ProbeOut* out, unsigned long long seq) {
    const unsigned long long t0 = globaltimer_ns();
    Acc a;
    constexpr unsigned long long chunk = (unsigned long long)THREADS * UNROLL;
    const unsigned long long n_full = n_vec / chunk;
    unsigned long long c = blockIdx.x;
    uint4 v[UNROLL];
    if (c < n_full) {
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) v[u] = src[c * chunk + threadIdx.x + (unsigned long long)u * THREADS];
    }
    for (; c < n_full; c += gridDim.x) {
        const unsigned long long base = c * chunk + threadIdx.x, cn = c + gridDim.x;
        uint4 w[UNROLL];
        if (cn < n_full) {
#pragma unroll
            for (int u = 0; u < UNROLL; ++u) w[u] = src[cn * chunk + threadIdx.x + (unsigned long long)u * THREADS];
        }
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            check4(v[u], base + (unsigned long long)u * THREADS, seed, delta, a);
            dst[base + (unsigned long long)u * THREADS] = v[u];
        }
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) v[u] = w[u];
    }
    for (unsigned long long i = n_full * chunk + (unsigned long long)blockIdx.x * THREADS + threadIdx.x;
         i < n_vec; i += (unsigned long long)gridDim.x * THREADS) {
        uint4 x = src[i];
        check4(x, i, seed, delta, a);
        dst[i] = x;
    }
    finish<THREADS>(a, ctl, out, seq, t0);
}


// ---- --gap: where the probe loses against a plain copy (tool-only kernels) ---------------------
// tma_ladder is hbm_probe_tma<4,1024,3> (same ring, tile->CTA map and barriers) with the verifier step cut down:
//   MODE 1: verifiers only wait full[s] and arrive on done[s] (the bulk-copy traffic alone)
//   MODE 2: plus the LDS.128/STS.128 round trip (re-keyed with delta, no check4) and fence.proxy.async
//   MODE 3: check4 as in the product (used for the timeline only)
// tl != nullptr records a per-CTA %globaltimer timeline, kTl slots per CTA:
//   [0] CTA start, [1] first tile ready, [2 .. kTl-3] every 32nd tile done, [kTl-2] last tile done, [kTl-1] drained
constexpr int kTl = 16;
template <int MODE>
__global__ void __launch_bounds__(160)
tma_ladder(const uint4* __restrict__ src, uint4* __restrict__ dst, unsigned long long n_vec, uint32_t seed, uint32_t delta,
           ProbeCtl* ctl, ProbeOut* out, unsigned long long seq, unsigned long long* tl) {
    constexpr int TILE_VEC = 1024, STAGES = 3, THREADS = 160, CT = 128, PER_THREAD = TILE_VEC / CT;
    constexpr uint32_t TILE_BYTES = TILE_VEC * 16u;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    uint4* tiles = reinterpret_cast<uint4*>(smem_raw);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + (size_t)STAGES * TILE_BYTES);
    uint64_t* done = full + STAGES;
    const unsigned long long t0 = globaltimer_ns();
    unsigned long long* my_tl = tl ? tl + (size_t)blockIdx.x * kTl : nullptr;
    const unsigned long long n_tiles = n_vec / TILE_VEC;
    const unsigned long long my_tiles = n_tiles > blockIdx.x ? (n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&done[s], CT); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        fence_proxy_async_smem();
        if (my_tl) my_tl[0] = t0;
    }
    __syncthreads();
    Acc a;
    if (threadIdx.x < 32) {
        if (threadIdx.x == 0) {
            for (int k = 0; k < STAGES && (unsigned long long)k < my_tiles; ++k) {
                mbar_expect_tx(&full[k], TILE_BYTES);
                bulk_g2s(tiles + (size_t)k * TILE_VEC, src + (blockIdx.x + (unsigned long long)k * gridDim.x) * TILE_VEC, TILE_BYTES, &full[k]);
            }
            int stamp = 2;
            for (unsigned long long k = 0; k < my_tiles; ++k) {
                const int slot = (int)(k % STAGES);
                mbar_wait(&done[slot], (uint32_t)((k / STAGES) & 1));
                if (my_tl) {
                    if ((k & 31) == 31 && stamp < kTl - 2) my_tl[stamp++] = globaltimer_ns();
                    if (k + 1 == my_tiles) my_tl[kTl - 2] = globaltimer_ns();
                }
                bulk_s2g(dst + (blockIdx.x + k * gridDim.x) * TILE_VEC, tiles + (size_t)slot * TILE_VEC, TILE_BYTES);
                bulk_commit();
                if (k >= 1 && k - 1 + STAGES < my_tiles) {
                    const unsigned long long kn = k - 1 + STAGES;
                    bulk_wait_read<1>();
                    const int sn = (int)(kn % STAGES);
                    mbar_expect_tx(&full[sn], TILE_BYTES);
                    bulk_g2s(tiles + (size_t)sn * TILE_VEC, src + (blockIdx.x + kn * gridDim.x) * TILE_VEC, TILE_BYTES, &full[sn]);
                }
            }
            bulk_wait_all<0>();
            if (my_tl) my_tl[kTl - 1] = globaltimer_ns();
        }
    } else {
        const int ct = threadIdx.x - 32;
        for (unsigned long long k = 0; k < my_tiles; ++k) {
            const int slot = (int)(k % STAGES);
            const unsigned long long t = blockIdx.x + k * gridDim.x;
            mbar_wait(&full[slot], (uint32_t)((k / STAGES) & 1));
            if (my_tl && k == 0 && ct == 0) my_tl[1] = globaltimer_ns();
            if (MODE >= 2) {
                uint4* tile = tiles + (size_t)slot * TILE_VEC;
                uint4 v[PER_THREAD];
#pragma unroll
                for (int u = 0; u < PER_THREAD; ++u) v[u] = tile[ct + u * CT];
#pragma unroll
                for (int u = 0; u < PER_THREAD; ++u) {
                    if (MODE == 3) check4(v[u], t * TILE_VEC + ct + u * CT, seed, delta, a);
                    else { v[u].x ^= delta; v[u].y ^= delta; v[u].z ^= delta; v[u].w ^= delta; }
                    tile[ct + u * CT] = v[u];
                }
                fence_proxy_async_smem();
            }
            mbar_arrive(&done[slot]);
        }
    }
    for (unsigned long long i = n_tiles * TILE_VEC + (unsigned long long)blockIdx.x * THREADS + threadIdx.x; i < n_vec;
         i += (unsigned long long)gridDim.x * THREADS) { uint4 v = ldg_na(src + i); check4(v, i, seed, delta, a); stg_na(dst + i, v); }
    finish<THREADS>(a, ctl, out, seq, t0);
}

// hbm_probe_pipe without check4: the register-streamed copy at the same shape
template <int THREADS, int UNROLL>
__global__ void __launch_bounds__(THREADS) copy_pipe(const uint4* __restrict__ src, uint4* __restrict__ dst, unsigned long long n_vec) {
    constexpr unsigned long long chunk = (unsigned long long)THREADS * UNROLL;
    const unsigned long long n_full = n_vec / chunk;
    unsigned long long c = blockIdx.x;
    uint4 v[UNROLL];
    if (c < n_full)
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) v[u] = src[c * chunk + threadIdx.x + (unsigned long long)u * THREADS];
    for (; c < n_full; c += gridDim.x) {
        const unsigned long long cn = c + gridDim.x;
        uint4 w[UNROLL];
        if (cn < n_full)
#pragma unroll
            for (int u = 0; u < UNROLL; ++u) w[u] = src[cn * chunk + threadIdx.x + (unsigned long long)u * THREADS];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) dst[c * chunk + threadIdx.x + (unsigned long long)u * THREADS] = v[u];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) v[u] = w[u];
    }
    for (unsigned long long i = n_full * chunk + (unsigned long long)blockIdx.x * THREADS + threadIdx.x; i < n_vec;
         i += (unsigned long long)gridDim.x * THREADS) dst[i] = src[i];
}

template <int MODE> static void launch_ladder(const uint4* s, uint4* d, unsigned long long n, uint32_t seed, uint32_t delta,
    ProbeCtl* c, ProbeOut* o, unsigned long long seq, int grid, cudaStream_t st, unsigned long long* tl = nullptr) {
    static bool once = false;
    if (!once) { CK(cudaFuncSetAttribute(tma_ladder<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTmaSmem)); once = true; }
    tma_ladder<MODE><<<grid, 160, kTmaSmem, st>>>(s, d, n, seed, delta, c, o, seq, tl);
}
template <int MODE> static void launch_ladder_fn(const uint4* s, uint4* d, unsigned long long n, uint32_t seed, uint32_t delta,
    ProbeCtl* c, ProbeOut* o, unsigned long long seq, int grid, cudaStream_t st) {
    launch_ladder<MODE>(s, d, n, seed, delta, c, o, seq, grid, st);
}
template <int CW, int TV, int ST> static void launch_split(const uint4* s, uint4* d, unsigned long long n, uint32_t seed,
    uint32_t delta, ProbeCtl* c, ProbeOut* o, unsigned long long seq, int grid, cudaStream_t st) {
    constexpr size_t smem = split_smem_bytes(TV, ST);
    static bool once = false;
    if (!once) { CK(cudaFuncSetAttribute(hbm_probe_split<CW, TV, ST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); once = true; }
    hbm_probe_split<CW, TV, ST><<<grid, (CW + 2) * 32, smem, st>>>(s, d, n, seed, delta, c, o, seq);
}
template <int CW, int TV, int ST> static void launch_queue(const uint4* s, uint4* d, unsigned long long n, uint32_t seed,
    uint32_t delta, ProbeCtl* c, ProbeOut* o, unsigned long long seq, int grid, cudaStream_t st) {
    constexpr size_t smem = queue_smem_bytes(TV, ST);
    static bool once = false;
    if (!once) { CK(cudaFuncSetAttribute(hbm_probe_queue<CW, TV, ST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); once = true; }
    hbm_probe_queue<CW, TV, ST><<<grid, (CW + 2) * 32, smem, st>>>(s, d, n, seed, delta, c, o, seq);
}
template <int T, int U> static void launch_pipe(const uint4* s, uint4* d, unsigned long long n, uint32_t seed,
    uint32_t delta, ProbeCtl* c, ProbeOut* o, unsigned long long seq, int grid, cudaStream_t st) {
    hbm_probe_pipe<T, U><<<grid, T, 0, st>>>(s, d, n, seed, delta, c, o, seq);
}
template <int T, int U> static void launch_copy_pipe(const uint4* s, uint4* d, unsigned long long n, uint32_t, uint32_t,
    ProbeCtl*, ProbeOut*, unsigned long long, int grid, cudaStream_t st) {
    copy_pipe<T, U><<<grid, T, 0, st>>>(s, d, n);
}
static void launch_plain_copy(const uint4* s, uint4* d, unsigned long long n, uint32_t, uint32_t, ProbeCtl*, ProbeOut*,
                              unsigned long long, int grid, cudaStream_t st) {
    plain_copy<<<grid, 512, 0, st>>>(s, d, n);
}
static void launch_memcpy(const uint4* s, uint4* d, unsigned long long n, uint32_t, uint32_t, ProbeCtl*, ProbeOut*,
                          unsigned long long, int, cudaStream_t st) {
    CK(cudaMemcpyAsync(d, s, n * 16, cudaMemcpyDeviceToDevice, st));
}

// What one rung does to the ping-pong pair: COPY moves src to dst unchanged, PROBE re-keys it (seed advances), READ only
// reads src, WRITE writes pattern(seed) into dst.  Every kind leaves the current buffer holding pattern(seed).
enum Kind { COPY, PROBE, READ, WRITE };
struct Rung { std::string rung, name; LaunchFn fn; int grid; Kind kind; };

static int run_gap(Bufs& B, int sms, cudaStream_t st, int rounds, int iters) {
    const unsigned long long bytes = B.n_vec * 16;
    unsigned long long* sink; CK(cudaMalloc(&sink, kSinks * 8));
    static unsigned long long* g_sink; g_sink = sink;
    std::vector<Rung> rungs = {
        {"R0", "memcpy_d2d", launch_memcpy, 0, COPY},
        {"R0", "read_only_t512_u4", [](const uint4* s, uint4*, unsigned long long n, uint32_t, uint32_t, ProbeCtl*, ProbeOut*,
             unsigned long long, int grid, cudaStream_t st) { read_only<4><<<grid, 512, 0, st>>>(s, n, g_sink); }, sms * 4, READ},
        {"R0", "write_only_t512", [](const uint4*, uint4* d, unsigned long long n, uint32_t seed, uint32_t, ProbeCtl*, ProbeOut*,
             unsigned long long, int grid, cudaStream_t st) { write_only<<<grid, 512, 0, st>>>(d, n, seed); }, sms * 4, WRITE},
        {"R1", "tma_4_1024_3_bulk_only", launch_ladder_fn<1>, sms * kTmaCtasPerSm, COPY},
        {"R2", "tma_4_1024_3_lds_sts_fence", launch_ladder_fn<2>, sms * kTmaCtasPerSm, COPY},
        {"R3", "hbm_probe_tma<4,1024,3>", launch_tma<kTmaCW, kTmaTileVec, kTmaStages>, sms * kTmaCtasPerSm, PROBE},
    };
    for (int k : {4, 8, 16}) rungs.push_back({"R4", "plain_copy_t512", launch_plain_copy, sms * k, COPY});
    for (int k : {2, 4, 8}) rungs.push_back({"R4", "copy_pipe_t256_u4", launch_copy_pipe<256, 4>, sms * k, COPY});
    for (int k : {2, 4}) rungs.push_back({"R4", "copy_pipe_t512_u2", launch_copy_pipe<512, 2>, sms * k, COPY});
    for (int k : {4, 8, 16}) rungs.push_back({"R5", "hbm_probe_r128<512,1>", launch_r128<512, 1>, sms * k, PROBE});
    rungs.push_back({"R5", "hbm_probe_r128<512,2>", launch_r128<512, 2>, sms * kRegCtasPerSm, PROBE});
    // candidates for the product kernel
    for (int k : {2, 4, 8}) rungs.push_back({"C", "hbm_probe_pipe<256,4>", launch_pipe<256, 4>, sms * k, PROBE});
    for (int k : {2, 4}) rungs.push_back({"C", "hbm_probe_pipe<512,2>", launch_pipe<512, 2>, sms * k, PROBE});
    for (int k : {2, 4}) rungs.push_back({"C", "hbm_probe_pipe<256,2>", launch_pipe<256, 2>, sms * k, PROBE});
    for (int k : {2, 3}) rungs.push_back({"C", "hbm_probe_split<4,512,6>", launch_split<4, 512, 6>, sms * k, PROBE});
    rungs.push_back({"C", "hbm_probe_split<4,256,12>", launch_split<4, 256, 12>, sms * 2, PROBE});
    rungs.push_back({"C", "hbm_probe_split<4,1024,3>", launch_split<4, 1024, 3>, sms * 2, PROBE});
    // the tile queue (hbm_probe_queue, the health probe's kernel) at its shape and around it
    for (int k : {1, 2, 3}) rungs.push_back({"Q", "hbm_probe_queue<4,512,6>", launch_queue<4, 512, 6>, sms * k, PROBE});
    rungs.push_back({"Q", "hbm_probe_queue<4,512,12>", launch_queue<4, 512, 12>, sms, PROBE});
    rungs.push_back({"Q", "hbm_probe_queue<4,1024,6>", launch_queue<4, 1024, 6>, sms, PROBE});
    rungs.push_back({"Q", "hbm_probe_queue<4,1024,3>", launch_queue<4, 1024, 3>, sms * 2, PROBE});
    rungs.push_back({"Q", "hbm_probe_queue<4,256,12>", launch_queue<4, 256, 12>, sms * 2, PROBE});
    // small grids: the health test's slow stand-ins (grid 18 must stay far below the full-grid rate)
    for (int g : {18, 33}) {
        rungs.push_back({"G", "hbm_probe_queue<4,512,6>", launch_queue<4, 512, 6>, g, PROBE});
        rungs.push_back({"G", "hbm_probe_tma<4,1024,3>", launch_tma<kTmaCW, kTmaTileVec, kTmaStages>, g, PROBE});
        rungs.push_back({"G", "hbm_probe_pipe<256,4>", launch_pipe<256, 4>, g, PROBE});
        rungs.push_back({"G", "hbm_probe_pipe<512,2>", launch_pipe<512, 2>, g, PROBE});
        rungs.push_back({"G", "hbm_probe_split<4,512,6>", launch_split<4, 512, 6>, g, PROBE});
    }

    unsigned long long seq = 1ull << 40;
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    auto step = [&](const Rung& r) {
        const uint32_t next = r.kind == PROBE ? B.seed * 1664525u + 1013904223u : B.seed;
        const uint4* s = B.cur == 0 ? B.a : B.b; uint4* d = B.cur == 0 ? B.b : B.a;
        r.fn(s, d, B.n_vec, B.seed, B.seed ^ next, B.ctl, B.out_d, ++seq, r.grid, st);
        if (r.kind != READ) B.cur ^= 1;
        B.seed = next;
    };
    // the current buffer must hold pattern(seed): a verify-only product pass over it, checked against the closed form
    auto verify = [&](const Rung& r) {
        const uint4* s = B.cur == 0 ? B.a : B.b; uint4* d = B.cur == 0 ? B.b : B.a;
        CK(cudaMemsetAsync(sink, 0, kSinks * 8, st));
        if (r.kind == READ) r.fn(s, d, B.n_vec, 0, 0, nullptr, nullptr, 0, r.grid, st);
        launch_tma<kTmaCW, kTmaTileVec, kTmaStages>(s, d, B.n_vec, B.seed, 0u, B.ctl, B.out_d, ++seq, sms * kTmaCtasPerSm, st);
        CK(cudaStreamSynchronize(st));
        unsigned long long h_sink[kSinks], got_sink = 0;
        CK(cudaMemcpy(h_sink, sink, sizeof h_sink, cudaMemcpyDeviceToHost));
        for (unsigned long long x : h_sink) got_sink += x;
        const unsigned long long want = cpu_checksum(B.n_vec * 4, B.seed);
        bool ok = B.out_h->seq == seq && B.out_h->mismatches == 0 && B.out_h->checksum == want;
        if (r.kind == READ) ok = ok && got_sink == want;
        if (!ok) {
            fprintf(stderr, "# %s %s grid %d: checksum %llx want %llx mismatches %llu first_bad %llu\n", r.rung.c_str(),
                    r.name.c_str(), r.grid, B.out_h->checksum, want, B.out_h->mismatches, B.out_h->first_bad);
            hbm_fill<256><<<sms * 8, 256, 0, st>>>(B.cur == 0 ? B.a : B.b, B.n_vec, B.seed);
            CK(cudaStreamSynchronize(st));
        }
        return ok;
    };

    std::vector<std::vector<float>> ms(rungs.size());
    std::vector<int> ok(rungs.size(), 1);
    for (int round = 0; round < rounds; ++round) {
        for (size_t i = 0; i < rungs.size(); ++i) {
            const Rung& r = rungs[i];
            for (int w = 0; w < 3; ++w) step(r);
            CK(cudaStreamSynchronize(st));
            std::vector<float> t(iters);
            for (int it = 0; it < iters; ++it) {
                CK(cudaEventRecord(e0, st)); step(r); CK(cudaEventRecord(e1, st));
                CK(cudaEventSynchronize(e1)); CK(cudaEventElapsedTime(&t[it], e0, e1));
            }
            std::sort(t.begin(), t.end());
            ms[i].push_back(t[iters / 2]);
            if (round == 0 && !verify(r)) ok[i] = 0;
        }
    }
    printf("rung,name,grid,median_gbs,min_gbs,max_gbs,median_ms,ok\n");
    for (size_t i = 0; i < rungs.size(); ++i) {
        const Rung& r = rungs[i];
        std::vector<float> m = ms[i];
        std::sort(m.begin(), m.end());
        const double moved = (r.kind == READ || r.kind == WRITE ? 1.0 : 2.0) * bytes / 1e6;
        printf("%s,%s,%d,%.1f,%.1f,%.1f,%.4f,%d\n", r.rung.c_str(), r.name.c_str(), r.grid, moved / m[m.size() / 2],
               moved / m.back(), moved / m.front(), m[m.size() / 2], ok[i]);
    }

    // per-CTA timelines of R1 and R3 (the product pipeline, instrumented copy)
    const int grid = sms * kTmaCtasPerSm;
    unsigned long long* tl; CK(cudaMalloc(&tl, (size_t)grid * kTl * 8));
    std::vector<unsigned long long> h((size_t)grid * kTl);
    printf("timeline,ramp_us_med,ramp_us_max,period_ns_per_tile_med,tail_us_med,tail_us_max,end_spread_us,span_us\n");
    for (int mode : {1, 3}) {
        for (int w = 0; w < 3; ++w) {
            CK(cudaMemsetAsync(tl, 0, (size_t)grid * kTl * 8, st));
            const uint32_t next = mode == 3 ? B.seed * 1664525u + 1013904223u : B.seed;
            const uint4* s = B.cur == 0 ? B.a : B.b; uint4* d = B.cur == 0 ? B.b : B.a;
            if (mode == 1) launch_ladder<1>(s, d, B.n_vec, B.seed, 0u, B.ctl, B.out_d, ++seq, grid, st, tl);
            else launch_ladder<3>(s, d, B.n_vec, B.seed, B.seed ^ next, B.ctl, B.out_d, ++seq, grid, st, tl);
            B.cur ^= 1; B.seed = next;
        }
        CK(cudaStreamSynchronize(st));
        CK(cudaMemcpy(h.data(), tl, h.size() * 8, cudaMemcpyDeviceToHost));
        unsigned long long start = ~0ull, end_min = ~0ull, end_max = 0;
        for (int b = 0; b < grid; ++b) {
            start = std::min(start, h[(size_t)b * kTl]);
            end_min = std::min(end_min, h[(size_t)b * kTl + kTl - 1]);
            end_max = std::max(end_max, h[(size_t)b * kTl + kTl - 1]);
        }
        std::vector<double> ramp, period, tail;
        for (int b = 0; b < grid; ++b) {
            const unsigned long long* x = &h[(size_t)b * kTl];
            ramp.push_back((x[1] - start) / 1e3);
            int last = 2;
            while (last + 1 < kTl - 2 && x[last + 1]) ++last;
            if (last > 2) period.push_back((double)(x[last] - x[2]) / (32.0 * (last - 2)));
            tail.push_back((x[kTl - 1] - x[kTl - 2]) / 1e3);
        }
        auto med = [](std::vector<double> v) { std::sort(v.begin(), v.end()); return v.empty() ? 0.0 : v[v.size() / 2]; };
        auto mx = [](const std::vector<double>& v) { return v.empty() ? 0.0 : *std::max_element(v.begin(), v.end()); };
        const bool ok_t = verify({"T", mode == 1 ? "R1" : "R3", nullptr, grid, mode == 1 ? COPY : PROBE});
        printf("%s,%.2f,%.2f,%.1f,%.2f,%.2f,%.2f,%.1f%s\n", mode == 1 ? "R1" : "R3", med(ramp), mx(ramp), med(period), med(tail),
               mx(tail), (end_max - end_min) / 1e3, (end_max - start) / 1e3, ok_t ? "" : ",BAD");
    }
    return 0;
}

int main(int argc, char** argv) {
    unsigned long long bytes = 1ull << 30;
    int iters = 10, warm = 3, rounds = 0;
    const char* only = nullptr;
    for (int i = 1; i < argc; ++i) {
        if (!strcmp(argv[i], "--bytes")) bytes = strtoull(argv[++i], 0, 0);
        else if (!strcmp(argv[i], "--iters")) iters = atoi(argv[++i]);
        else if (!strcmp(argv[i], "--only")) only = argv[++i];
        else if (!strcmp(argv[i], "--gap")) rounds = i + 1 < argc && argv[i + 1][0] != '-' ? atoi(argv[++i]) : 5;
    }
    cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
    const int sms = prop.multiProcessorCount;
    fprintf(stderr, "# %s, %d SMs, bytes=%llu\n", prop.name, sms, bytes);

    Bufs B{}; B.n_vec = bytes / 16;
    CK(cudaMalloc(&B.a, bytes)); CK(cudaMalloc(&B.b, bytes));
    CK(cudaMalloc(&B.ctl, sizeof(ProbeCtl)));
    ProbeCtl init{}; init.first_bad = ~0ull; init.t_start_ns = ~0ull;
    CK(cudaMemcpy(B.ctl, &init, sizeof init, cudaMemcpyHostToDevice));
    CK(cudaHostAlloc(&B.out_h, sizeof(ProbeOut), cudaHostAllocMapped));
    CK(cudaHostGetDevicePointer(&B.out_d, B.out_h, 0));
    cudaStream_t st; CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));

    B.seed = 0x5EED0000u; B.cur = 0;
    hbm_fill<256><<<sms * 8, 256, 0, st>>>(B.a, B.n_vec, B.seed);
    CK(cudaStreamSynchronize(st));
    if (rounds) return run_gap(B, sms, st, rounds, iters);

    std::vector<Cfg> cfgs;
#define R128(T, U) for (int k : {1, 2, 4, 8, 16}) if (k * T <= 2048) cfgs.push_back({"r128_t" #T "_u" #U, launch_r128<T, U>, k});
#define R256(T, U) for (int k : {1, 2, 4, 8}) if (k * T <= 2048) cfgs.push_back({"r256_t" #T "_u" #U, launch_r256<T, U>, k});
#define TMA(CW, TV, ST) for (int k : {1, 2, 3, 4, 6}) if ((size_t)k * ((size_t)ST * TV * 16 + 1024) <= 227 * 1024 && k * (CW + 1) * 32 <= 2048) \
        cfgs.push_back({"tma_cw" #CW "_tv" #TV "_st" #ST, launch_tma<CW, TV, ST>, k});
    R128(256, 2) R128(256, 4) R128(256, 8) R128(512, 2) R128(512, 4) R128(512, 8) R128(1024, 2) R128(1024, 4)
    R256(256, 1) R256(256, 2) R256(256, 4) R256(512, 1) R256(512, 2) R256(512, 4)
#define TMAH(CW, TV, ST, H) for (int k : {1, 2, 3}) if ((size_t)k * ((size_t)ST * TV * 16 + 1024) <= 227 * 1024 && k * (CW + 1) * 32 <= 2048) \
        cfgs.push_back({"tmah" #H "_cw" #CW "_tv" #TV "_st" #ST, launch_tma<CW, TV, ST, H>, k});
    TMAH(4, 1024, 3, 1) TMAH(4, 1024, 3, 2) TMAH(4, 1024, 3, 3) TMAH(4, 512, 6, 3) TMAH(4, 768, 4, 0) TMAH(4, 768, 4, 3)
    TMAH(8, 1024, 3, 0) TMAH(8, 1024, 3, 3) TMAH(2, 1024, 3, 0) TMAH(4, 512, 6, 0) TMAH(4, 1536, 3, 0) TMAH(4, 1280, 3, 0)
    TMAH(4, 896, 3, 0) TMAH(4, 640, 5, 0) TMAH(4, 1024, 4, 3) TMAH(6, 768, 4, 0) TMAH(6, 1536, 3, 0)
    // hint bits: 1 loads evict_first, 2 stores evict_first, 4 stores evict_last, 8 loads evict_last
    TMAH(4, 1024, 3, 4) TMAH(4, 1024, 3, 5) TMAH(4, 1024, 3, 8) TMAH(4, 1024, 3, 10) TMAH(4, 1024, 3, 12)
    TMA(4, 512, 4) TMA(4, 1024, 3) TMA(4, 1024, 4) TMA(4, 1024, 6) TMA(4, 2048, 3) TMA(4, 2048, 4)
    TMA(8, 1024, 4) TMA(8, 2048, 3) TMA(8, 2048, 4) TMA(8, 4096, 3) TMA(2, 1024, 4) TMA(2, 512, 6)

    // baselines: driver D2D memcpy and a plain copy kernel (no verify)
    auto time_it = [&](auto&& body) {
        for (int w = 0; w < warm; ++w) body();
        CK(cudaStreamSynchronize(st));
        std::vector<float> ms(iters);
        for (int i = 0; i < iters; ++i) {
            CK(cudaEventRecord(e0, st)); body(); CK(cudaEventRecord(e1, st));
            CK(cudaEventSynchronize(e1)); CK(cudaEventElapsedTime(&ms[i], e0, e1));
        }
        std::sort(ms.begin(), ms.end());
        return std::pair<float, float>(ms[iters / 2], ms[0]);
    };
    printf("name,ctas_per_sm,grid,median_ms,best_ms,median_gbs,best_gbs,ok\n");
    if (!only) {
        auto r = time_it([&] { CK(cudaMemcpyAsync(B.b, B.a, bytes, cudaMemcpyDeviceToDevice, st)); });
        printf("memcpy_d2d,0,0,%.4f,%.4f,%.1f,%.1f,1\n", r.first, r.second, 2.0 * bytes / r.first / 1e6, 2.0 * bytes / r.second / 1e6);
        for (int k : {4, 8, 16}) {
            auto r2 = time_it([&] { plain_copy<<<sms * k, 512, 0, st>>>(B.a, B.b, B.n_vec); });
            printf("plain_copy_t512,%d,%d,%.4f,%.4f,%.1f,%.1f,1\n", k, sms * k, r2.first, r2.second,
                   2.0 * bytes / r2.first / 1e6, 2.0 * bytes / r2.second / 1e6);
        }
        // restore pattern in a (plain_copy/memcpy left b == a; a is intact)
        unsigned long long* sink; CK(cudaMalloc(&sink, kSinks * 8));
        for (int k : {2, 4, 8}) {
            auto rr = time_it([&] { read_only<4><<<sms * k, 512, 0, st>>>(B.a, B.n_vec, sink); });
            printf("read_only_t512_u4,%d,%d,%.4f,%.4f,%.1f,%.1f,1\n", k, sms * k, rr.first, rr.second, 1.0 * bytes / rr.first / 1e6, 1.0 * bytes / rr.second / 1e6);
            auto r8 = time_it([&] { read_only<8><<<sms * k, 256, 0, st>>>(B.a, B.n_vec, sink); });
            printf("read_only_t256_u8,%d,%d,%.4f,%.4f,%.1f,%.1f,1\n", k, sms * k, r8.first, r8.second, 1.0 * bytes / r8.first / 1e6, 1.0 * bytes / r8.second / 1e6);
        }
        {
            constexpr size_t sm3 = 3 * 1024 * 16 + 64, sm6 = 6 * 1024 * 16 + 128;
            CK(cudaFuncSetAttribute(read_only_tma<1024, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm3));
            CK(cudaFuncSetAttribute(read_only_tma<1024, 6>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm6));
            for (int k : {1, 2, 3}) {
                auto rt = time_it([&] { read_only_tma<1024, 3><<<sms * k, 160, sm3, st>>>(B.a, B.n_vec, sink); });
                printf("read_only_tma_tv1024_st3,%d,%d,%.4f,%.4f,%.1f,%.1f,1\n", k, sms * k, rt.first, rt.second, 1.0 * bytes / rt.first / 1e6, 1.0 * bytes / rt.second / 1e6);
            }
            for (int k : {1, 2}) {
                auto rt = time_it([&] { read_only_tma<1024, 6><<<sms * k, 160, sm6, st>>>(B.a, B.n_vec, sink); });
                printf("read_only_tma_tv1024_st6,%d,%d,%.4f,%.4f,%.1f,%.1f,1\n", k, sms * k, rt.first, rt.second, 1.0 * bytes / rt.first / 1e6, 1.0 * bytes / rt.second / 1e6);
            }
        }
        for (int k : {2, 4, 8, 16}) {
            auto rw = time_it([&] { write_only<<<sms * k, 512, 0, st>>>(B.b, B.n_vec, 7u); });
            printf("write_only_t512,%d,%d,%.4f,%.4f,%.1f,%.1f,1\n", k, sms * k, rw.first, rw.second, 1.0 * bytes / rw.first / 1e6, 1.0 * bytes / rw.second / 1e6);
        }
        auto rm = time_it([&] { CK(cudaMemsetAsync(B.b, 0, bytes, st)); });
        printf("memset,0,0,%.4f,%.4f,%.1f,%.1f,1\n", rm.first, rm.second, 1.0 * bytes / rm.first / 1e6, 1.0 * bytes / rm.second / 1e6);
    }

    // phased experiment: name encodes the period; ctas_per_sm field carries it to the loop below
    struct PCfg { const char* name; LaunchFn fn; };
    const PCfg pc[] = {{"phased_cw8_tv1024_st12", launch_phased<8, 1024, 12>}, {"phased_cw8_tv1024_st8", launch_phased<8, 1024, 8>},
                       {"phased_cw8_tv2048_st6", launch_phased<8, 2048, 6>}};
    unsigned long long seq = 0;
    if (!only || strstr(only, "phased")) {
        for (auto& p : pc)
            for (unsigned int per : {0u, 6000u, 7000u, 8000u, 9000u, 10000u, 12000u, 16000u}) {
                g_period_ns = per;
                auto body = [&] {
                    const uint32_t next = B.seed * 1664525u + 1013904223u;
                    const uint4* s = B.cur == 0 ? B.a : B.b; uint4* d = B.cur == 0 ? B.b : B.a;
                    p.fn(s, d, B.n_vec, B.seed, B.seed ^ next, B.ctl, B.out_d, ++seq, sms, st);
                    B.seed = next; B.cur ^= 1;
                };
                const uint32_t seed_before = B.seed;
                body();
                CK(cudaStreamSynchronize(st));
                const bool ok = B.out_h->seq == seq && B.out_h->mismatches == 0 && B.out_h->checksum == cpu_checksum(B.n_vec * 4, seed_before);
                auto r = time_it(body);
                printf("%s_period%u,1,%d,%.4f,%.4f,%.1f,%.1f,%d\n", p.name, per, sms, r.first, r.second,
                       2.0 * bytes / r.first / 1e6, 2.0 * bytes / r.second / 1e6, ok ? 1 : 0);
                fflush(stdout);
            }
    }
    for (auto& c : cfgs) {
        if (only && c.name.find(only) == std::string::npos) continue;
        const int grid = sms * c.ctas_per_sm;
        bool ok = true;
        auto body = [&] {
            const uint32_t next = B.seed * 1664525u + 1013904223u;
            const uint4* s = B.cur == 0 ? B.a : B.b; uint4* d = B.cur == 0 ? B.b : B.a;
            c.fn(s, d, B.n_vec, B.seed, B.seed ^ next, B.ctl, B.out_d, ++seq, grid, st);
            B.seed = next; B.cur ^= 1;
        };
        // one checked launch first
        const uint32_t seed_before = B.seed;
        body();
        cudaError_t le = cudaStreamSynchronize(st);
        if (le != cudaSuccess) { printf("%s,%d,%d,0,0,0,0,CUDA_%s\n", c.name.c_str(), c.ctas_per_sm, grid, cudaGetErrorName(le)); return 3; }
        const unsigned long long want = cpu_checksum(B.n_vec * 4, seed_before);
        if (B.out_h->seq != seq || B.out_h->checksum != want || B.out_h->mismatches != 0) {
            ok = false;
            fprintf(stderr, "# %s k=%d: seq %llu/%llu checksum %llx want %llx mismatches %llu first_bad %llu\n", c.name.c_str(),
                    c.ctas_per_sm, B.out_h->seq, seq, B.out_h->checksum, want, B.out_h->mismatches, B.out_h->first_bad);
            // repair so later configs start clean
            hbm_fill<256><<<sms * 8, 256, 0, st>>>(B.cur == 0 ? B.a : B.b, B.n_vec, B.seed);
            CK(cudaStreamSynchronize(st));
        }
        auto r = time_it(body);
        printf("%s,%d,%d,%.4f,%.4f,%.1f,%.1f,%d\n", c.name.c_str(), c.ctas_per_sm, grid, r.first, r.second,
               2.0 * bytes / r.first / 1e6, 2.0 * bytes / r.second / 1e6, ok ? 1 : 0);
        fflush(stdout);
    }
    return 0;
}
