// l1_test_math.hpp -- host-side arithmetic of the on-demand L1 self-test (b2dp_l1_test, l1_selftest.cuh): the SM's L1
// data cache, its texture path and read-only data path, and its constant cache.
//
// Pure C++ (no CUDA; the patterns, the layout and the coordinate schedules are also compiled for the device), so the CPU
// tests compile it as it is (tests/native/l1_test_math_test.cpp) and compare it with tests/l1_test_oracle.py:
//   - l1_pattern / l1_line_key:  the L1_DATA span's words under a tile's data background and per-line key
//   - l1_data_block / l1_data_writer / l1_data_want:  which vector a thread reads in which pass, and its comparison
//   - l1_texel / l1_tex_image:   the texel image the driver fills the CUDA array and the linear copy with
//   - l1_tex_addr / l1_tex_point / l1_tex_gather:  the address modes, point sampling and tld4's selection
//   - l1_bank / l1_const_index:  the constant bank's four windows and the index schedules
//   - l1_results / l1_build_tile:  every result word of a thread, the tile's table and its check values
// Every expected value follows from the PTX ISA and the CUDA programming guide; nothing comes from the device under test.
//
// L1_DATA.  Every CTA owns K blocks of kL1BlockWords words (2 KiB, one 16-byte vector per thread) in the scratch
// buffer: its private span, K x 2 KiB, from the per-SM span over the CTAs an SM holds (l1_span_blocks).  One comparison
// (tile, repetition): every thread writes its vector t of every block with P ^ inv (inv = ~0 on odd repetitions, so every
// bit of every line is held as 0 and as 1), a __syncthreads makes the stores visible to the CTA, then three read passes
// load every vector of the span once with weak ld.global.v4.u32 (L1-allocating), blocks ascending, descending and
// strided by four.  In pass p thread t reads the vector of writer (t - 32 (p + 1)) mod 128: never its own.
// P(w) = sh_pattern(kind, key, w % 512) ^ (global line of w + 1) x linemul: the shared-memory and L2 tests' data
// backgrounds, and in the keyed tiles (linemul != 0) a key per 128-byte line of the whole scratch, so a line that
// answers for another address reads wrong.  Every value read is compared with P ^ inv directly, and with the line key
// XORed out it enters a sum fold with weight 2j + 1 (j = 4 p + i, i the word of the vector): K x c(t) on an even
// repetition, K x (-144 - c(t)) on an odd one, c(t) being the host's check of thread t.
//
// L1_TEX.  A kL1TexW x kL1TexH 2D CUDA array of uint4 texels (128 KiB, block-linear), image row y < kL1TexH / 2 holds
// the keyed pattern P, the other half ~P.  Five texture objects over it, all point-sampled and read as elements:
// object 0 with unnormalized coordinates and clamp; objects 1..4 with normalized coordinates in wrap, mirror, clamp and
// border (border colour 0).  A linear copy of the image sits in the scratch buffer.  In step j (0..63) thread t takes
// texel i = (A (128 j + t) + B) mod 8192 of the tile's permutation (A odd), x = i % 64, y = i / 64, and runs:
//   tex.2d.v4.u32.s32 at (x, y) on object 0                        -> texel (x, y)
//   tex.2d.v4.u32.f32 at (x + 1/2, y + 1/2) on object 0            -> texel (x, y)
//   tex.2d.v4.u32.f32 at ((x + 1/2) / 64 + mx, (y + 1/2) / 128 + my) on objects 1..4, mx, my in -2..2
//   tld4.{r,g,b,a}.2d.v4.u32.f32 at (x + 1/2, y + 1/2) on object 0 (component j % 4)
//   ld.global.nc.v4.u32 of texel i of the linear copy
// All coordinates are texel centres of power-of-two dimensions: exact in f32, so no rounding question arises.
// The address modes (CUDA C++ Programming Guide, "Texture Fetching"): a normalized coordinate u becomes frac(u) (wrap);
// frac(u) if floor(u) is even, else 1 - frac(u) (mirror); 0 if u < 0, 1 - 1/N if u >= 1 (clamp); and outside [0, 1) the
// border colour (border).  Point sampling then takes texel floor(N u).  At a texel centre tld4 gathers the 2 x 2
// footprint i0 = x, i1 = x + 1, j0 = y, j1 = y + 1 (clamped), and returns its component of the texels in the PTX ISA's
// order (tld4): (i0, j1), (i1, j1), (i1, j0), (i0, j0).
//
// L1_CONST.  One __constant__ bank of kL1BankWords words (32 KiB): four 8 KiB windows, windows 0 and 1 the keyed
// pattern, windows 2 and 3 its complement.  Tile t reads window t % 4 in every repetition: each warp reads every word of
// the window once in each of four forms -- a warp-uniform index (broadcast), lane-divergent indices that touch 32
// distinct 128-byte lines per instruction, and 64- and 128-bit loads with lane-divergent indices.
#pragma once
#include <cstdint>
#include <cstring>
#include <vector>

#include "int_test_math.hpp"   // it_fold, ct_stream_key, CtRecord, kCtThreads, kCtTiles, kCtReps
#include "smem_test_math.hpp"  // sh_pattern, sh_kind, sh_key

#if defined(__CUDACC__)
#define B2DP_L1_HD __host__ __device__
#else
#define B2DP_L1_HD
#endif

namespace b2dp {

enum L1Format { L1_DATA = 0, L1_TEX = 1, L1_CONST = 2 };
constexpr int kL1Formats = 3;
static_assert(kL1Formats == kCtFormats, "the verdict and the result struct are shared with the tensor-core test");

// ---- the scratch buffer (uint32_t words): a header, then the data ---------------------------------------------------
constexpr int kL1HdrBlocks = 0;    // L1_DATA: K, blocks per CTA span (host-written)
constexpr int kL1HdrDump = 1;      // word offset of the DUMP area (the harness only)
constexpr int kL1HdrTex = 8;       // L1_TEX: the kL1TexObjs texture handles, 64 bits each
constexpr int kL1HdrWords = 64;
constexpr int kL1DataOff = kL1HdrWords;
constexpr int kL1TableWords = 4;   // every format's tile table

// ---- L1_DATA ------------------------------------------------------------------------------------------------------
constexpr int kL1LineWords = 32;                     // 128 bytes
constexpr int kL1BlockWords = 4 * kCtThreads;        // one 16-byte vector per thread: 2 KiB
constexpr uint32_t kL1BlockBytes = 4u * kL1BlockWords;
constexpr int kL1Passes = 3;
constexpr int kL1DataWords = 4 * kL1Passes;          // values per thread per block: the fold's weights 1, 3, .., 23
constexpr uint32_t kL1WeightSum = kL1DataWords * kL1DataWords;  // sum of 2j + 1 over j < 12 = 144
constexpr unsigned long long kL1DefaultSpan = 128ull << 10;     // per SM (DESIGN 4.16, profiles/l1_span_sweep_h100.txt)
constexpr uint32_t kL1LineMul = 0x9E3779B9u;
constexpr uint32_t kL1HookWord = 37;                 // the word of its span the fault hook flips after the write
constexpr uint32_t kL1MaxBlocks = 1u << 12;          // 8 MiB per CTA: far beyond any L1

B2DP_L1_HD inline uint32_t l1_line_key(uint32_t linemul, uint32_t line) { return (line + 1u) * linemul; }
// Word w of CTA c's span of K blocks: the background and the key of its line in the whole scratch buffer.
B2DP_L1_HD inline uint32_t l1_pattern(uint32_t kind, uint32_t key, uint32_t linemul, uint32_t c, uint32_t K,
                                      uint32_t w) {
    return sh_pattern(kind, key, w % (uint32_t)kL1BlockWords) ^
           l1_line_key(linemul, (c * K * kL1BlockWords + w) / kL1LineWords);
}
// The block read in step s of pass p over K blocks: ascending, descending, then strided by four.
B2DP_L1_HD inline uint32_t l1_data_block(int p, uint32_t s, uint32_t K) {
    if (p == 0) return s;
    if (p == 1) return K - 1u - s;
    const uint32_t q = K / 4u, r = K % 4u;  // residue class m holds q + (m < r) blocks
    uint32_t m = 0, base = 0;
    for (; m < 3u; ++m) {
        const uint32_t n = q + (m < r ? 1u : 0u);
        if (s < base + n) break;
        base += n;
    }
    return m + 4u * (s - base);
}
// The thread whose vector thread t reads in pass p.
B2DP_L1_HD inline int l1_data_writer(int t, int p) { return (t - 32 * (p + 1)) & (kCtThreads - 1); }
// Blocks per CTA span for a per-SM span of span_bytes and per_sm CTAs on an SM (at least one).
inline uint32_t l1_span_blocks(unsigned long long span_bytes, int per_sm) {
    const unsigned long long k = span_bytes / ((unsigned long long)(per_sm > 0 ? per_sm : 1) * kL1BlockBytes);
    return k ? (k < kL1MaxBlocks ? (uint32_t)k : kL1MaxBlocks) : 1u;
}
// The kernel's comparison value for a span of K blocks in repetition rep.
B2DP_L1_HD inline uint32_t l1_data_want(uint32_t check, uint32_t K, int rep) {
    return K * ((rep & 1) ? 0u - kL1WeightSum - check : check);
}

// ---- L1_TEX -------------------------------------------------------------------------------------------------------
constexpr int kL1TexW = 64, kL1TexH = 128;           // texels; the array is 128 KiB
constexpr int kL1Texels = kL1TexW * kL1TexH;
constexpr int kL1TexSteps = kL1Texels / kCtThreads;  // 64 texels per thread and op
constexpr int kL1TexObjs = 5;                        // unnormalized; wrap, mirror, clamp, border
enum L1TexMode { L1_WRAP = 0, L1_MIRROR = 1, L1_CLAMP = 2, L1_BORDER = 3 };
constexpr int kL1TexOps = 8;                         // tld, tex, 4 x normalized tex, tld4, ld.nc per step
constexpr int kL1TexWordsPerStep = 4 * kL1TexOps;
static_assert(kL1TexSteps % 4 == 0, "tld4's four components rotate over the steps");

// Component c of texel (x, y) of the image.
B2DP_L1_HD inline uint32_t l1_texel(uint32_t key, int x, int y, int c) {
    return sh_pattern(4u, key, (uint32_t)(4 * (y * kL1TexW + x) + c)) ^ (y >= kL1TexH / 2 ? ~0u : 0u);
}
inline uint32_t l1_tex_key(uint32_t seed) { return ct_stream_key(seed, 10, 0, 0); }
// The image as the driver uploads it: row-major texels of four words.
inline void l1_tex_image(uint32_t seed, uint32_t* img) {
    const uint32_t key = l1_tex_key(seed);
    for (int y = 0; y < kL1TexH; ++y)
        for (int x = 0; x < kL1TexW; ++x)
            for (int c = 0; c < 4; ++c) img[4 * (y * kL1TexW + x) + c] = l1_texel(key, x, y, c);
}
// Step j of thread t: the texel index and the normalized offsets mx, my (in -2..2).
B2DP_L1_HD inline uint32_t l1_tex_index(uint32_t A, uint32_t B, int t, int j) {
    return (A * (uint32_t)(kCtThreads * j + t) + B) & (uint32_t)(kL1Texels - 1);
}
B2DP_L1_HD inline int l1_tex_mx(uint32_t D, int t, int j) { return (int)((uint32_t)(t + j) + D) % 5 - 2; }
B2DP_L1_HD inline int l1_tex_my(uint32_t D, int t, int j) { return (int)((uint32_t)(t / 5 + 2 * j) + 3u * D) % 5 - 2; }
// The texel a point-sampled normalized fetch at the centre of texel x, shifted by m whole periods, resolves to along an
// axis of N texels; -1: the border colour.
inline int l1_tex_addr(int mode, int x, int m, int N) {
    switch (mode) {
        case L1_WRAP: return x;
        case L1_MIRROR: return (m & 1) ? N - 1 - x : x;
        case L1_CLAMP: return m < 0 ? 0 : m > 0 ? N - 1 : x;
        default: return m == 0 ? x : -1;
    }
}
// One normalized fetch: four words.
inline void l1_tex_point(uint32_t key, int mode, int x, int y, int mx, int my, uint32_t* out) {
    const int ix = l1_tex_addr(mode, x, mx, kL1TexW), iy = l1_tex_addr(mode, y, my, kL1TexH);
    for (int c = 0; c < 4; ++c) out[c] = ix < 0 || iy < 0 ? 0u : l1_texel(key, ix, iy, c);
}
// tld4 of component c at the centre of texel (x, y) on the unnormalized, clamped object.
inline void l1_tex_gather(uint32_t key, int x, int y, int c, uint32_t* out) {
    const int i1 = x + 1 < kL1TexW ? x + 1 : kL1TexW - 1, j1 = y + 1 < kL1TexH ? y + 1 : kL1TexH - 1;
    out[0] = l1_texel(key, x, j1, c);
    out[1] = l1_texel(key, i1, j1, c);
    out[2] = l1_texel(key, i1, y, c);
    out[3] = l1_texel(key, x, y, c);
}

// ---- L1_CONST -----------------------------------------------------------------------------------------------------
constexpr int kL1BankWords = 8192;                   // 32 KiB: the __constant__ bank
constexpr int kL1Windows = 4;
constexpr int kL1WindowWords = kL1BankWords / kL1Windows;   // 8 KiB, the guide's constant-cache working set per SM
constexpr int kL1ConstUni = kL1WindowWords;          // broadcast loads per thread
constexpr int kL1ConstDiv = kL1WindowWords / 32;     // 64 lane-divergent 32-bit loads
constexpr int kL1ConstV2 = kL1WindowWords / 64;      // 32 64-bit loads
constexpr int kL1ConstV4 = kL1WindowWords / 128;     // 16 128-bit loads
constexpr int kL1ConstWords = kL1ConstUni + kL1ConstDiv + 2 * kL1ConstV2 + 4 * kL1ConstV4;

inline uint32_t l1_const_key(uint32_t seed) { return ct_stream_key(seed, 11, 0, 0); }
B2DP_L1_HD inline uint32_t l1_bank_word(uint32_t key, int i) {
    const int w = i / kL1WindowWords, k = i % kL1WindowWords;
    return sh_pattern(4u, key, (uint32_t)((w & 1) * kL1WindowWords + k)) ^ (w >= 2 ? ~0u : 0u);
}
inline void l1_bank(uint32_t seed, uint32_t* bank) {
    const uint32_t key = l1_const_key(seed);
    for (int i = 0; i < kL1BankWords; ++i) bank[i] = l1_bank_word(key, i);
}
// The window word each form's load k of lane l of warp w reads (v2 / v4: the first of its words); rot from the table.
B2DP_L1_HD inline uint32_t l1_const_uni(uint32_t rot, int w, int k) {
    return ((uint32_t)k + 512u * (uint32_t)w + rot) & (uint32_t)(kL1WindowWords - 1);
}
B2DP_L1_HD inline uint32_t l1_const_div(uint32_t rot, int w, int l, int k) {
    return ((uint32_t)(64 * l + k) + 512u * (uint32_t)w + rot) & (uint32_t)(kL1WindowWords - 1);
}
B2DP_L1_HD inline uint32_t l1_const_v2(uint32_t rot, int w, int l, int k) {
    return (2u * (uint32_t)(32 * l + k) + 512u * (uint32_t)w + 2u * rot) & (uint32_t)(kL1WindowWords - 2);
}
B2DP_L1_HD inline uint32_t l1_const_v4(uint32_t rot, int w, int l, int k) {
    return (4u * (uint32_t)(16 * l + k) + 512u * (uint32_t)w + 4u * rot) & (uint32_t)(kL1WindowWords - 4);
}

// ---- tables, results and checks -------------------------------------------------------------------------------------
// DATA: kind, key, linemul, hook word.  TEX: A (odd), B, D, 0.  CONST: window, rot, 0, 0.
inline void l1_table(uint32_t seed, int fmt, int tile, uint32_t* table) {
    memset(table, 0, 4 * kL1TableWords);
    if (fmt == L1_DATA) {
        table[0] = sh_kind(tile);
        table[1] = sh_key(seed, 6, tile);
        table[2] = sh_kind(tile) == 4 ? kL1LineMul : 0u;
        table[3] = kL1HookWord;
    } else if (fmt == L1_TEX) {
        const uint32_t k = ct_stream_key(seed, 7, tile, 0);
        table[0] = (k | 1u) & (uint32_t)(kL1Texels - 1);
        table[1] = (k >> 13) & (uint32_t)(kL1Texels - 1);
        table[2] = (k >> 26) % 5u;
    } else {
        table[0] = (uint32_t)(tile % kL1Windows);
        table[1] = ct_stream_key(seed, 8, tile, 0) & (uint32_t)(kL1WindowWords - 1);
    }
}
// Every index a table implies stays in range: the harness and the driver refuse any other table before a launch.
inline bool l1_table_ok(int fmt, const uint32_t* table) {
    if (fmt == L1_DATA) return table[0] <= 4u && table[3] < kL1BlockWords;
    if (fmt == L1_TEX) return (table[0] & 1u) && table[0] < (uint32_t)kL1Texels && table[1] < (uint32_t)kL1Texels && table[2] < 5u;
    if (fmt == L1_CONST) return table[0] < (uint32_t)kL1Windows && table[1] < (uint32_t)kL1WindowWords;
    return false;
}
// Every texture handle the kernel reads from the scratch header is set.
inline bool l1_handles_ok(const unsigned long long* h) {
    for (int i = 0; i < kL1TexObjs; ++i)
        if (!h[i]) return false;
    return true;
}

B2DP_L1_HD inline int l1_words(int fmt) {
    return fmt == L1_TEX ? kL1TexSteps * kL1TexWordsPerStep : fmt == L1_CONST ? kL1ConstWords : kL1DataWords;
}
inline uint32_t l1_table_bytes(int) { return 4u * kL1TableWords; }

// Every result word thread t produces in one comparison, in the kernel's order (L1_DATA: one block's kL1DataWords
// values with line keys removed, of an even repetition).
inline void l1_results(uint32_t seed, int fmt, const uint32_t* table, int t, uint32_t* out) {
    if (fmt == L1_DATA) {
        for (int p = 0; p < kL1Passes; ++p)
            for (int i = 0; i < 4; ++i)
                out[4 * p + i] = sh_pattern(table[0], table[1], (uint32_t)(4 * l1_data_writer(t, p) + i));
    } else if (fmt == L1_TEX) {
        const uint32_t key = l1_tex_key(seed);
        uint32_t* o = out;
        for (int j = 0; j < kL1TexSteps; ++j) {
            const uint32_t i = l1_tex_index(table[0], table[1], t, j);
            const int x = (int)(i % kL1TexW), y = (int)(i / kL1TexW);
            for (int k = 0; k < 2; ++k)  // tld and the unnormalized tex
                for (int c = 0; c < 4; ++c) *o++ = l1_texel(key, x, y, c);
            for (int mode = 0; mode < 4; ++mode, o += 4)
                l1_tex_point(key, mode, x, y, l1_tex_mx(table[2], t, j), l1_tex_my(table[2], t, j), o);
            l1_tex_gather(key, x, y, j & 3, o);
            o += 4;
            for (int c = 0; c < 4; ++c) *o++ = l1_texel(key, x, y, c);  // the linear copy
        }
    } else {
        const uint32_t key = l1_const_key(seed), base = table[0] * kL1WindowWords, rot = table[1];
        const int w = t / 32, l = t % 32;
        uint32_t* o = out;
        auto C = [&](uint32_t k) { return l1_bank_word(key, (int)(base + k)); };
        for (int k = 0; k < kL1ConstUni; ++k) *o++ = C(l1_const_uni(rot, w, k));
        for (int k = 0; k < kL1ConstDiv; ++k) *o++ = C(l1_const_div(rot, w, l, k));
        for (int k = 0; k < kL1ConstV2; ++k)
            for (int e = 0; e < 2; ++e) *o++ = C(l1_const_v2(rot, w, l, k) + e);
        for (int k = 0; k < kL1ConstV4; ++k)
            for (int e = 0; e < 4; ++e) *o++ = C(l1_const_v4(rot, w, l, k) + e);
    }
}

// One tile: its table and every thread's check (DATA: c(t); TEX / CONST: it_fold of the thread's result words).
inline void l1_build_tile(uint32_t seed, int fmt, int tile, uint32_t* table, uint32_t* check,
                          std::vector<uint32_t>* words = nullptr) {
    l1_table(seed, fmt, tile, table);
    const int W = l1_words(fmt);
    std::vector<uint32_t> own;
    std::vector<uint32_t>& w = words ? *words : own;
    w.assign((size_t)kCtThreads * W, 0);
    for (int t = 0; t < kCtThreads; ++t) {
        uint32_t* o = &w[(size_t)t * W];
        l1_results(seed, fmt, table, t, o);
        if (fmt == L1_DATA) {
            uint32_t h = 0;
            for (int j = 0; j < W; ++j) h += (2u * (uint32_t)j + 1u) * o[j];
            check[t] = h;
        } else {
            check[t] = it_fold(o, W);
        }
    }
}

// Bytes the loads deliver to one CTA in one comparison (L1_DATA: and its stores), for a DATA span of K blocks.
inline double l1_bytes_per_comparison(int fmt, uint32_t K) {
    if (fmt == L1_DATA) return (double)K * kL1BlockBytes * (1 + kL1Passes);
    if (fmt == L1_TEX) return (double)kCtThreads * kL1TexSteps * kL1TexOps * 16;
    return (double)kCtThreads * kL1ConstWords * 4;
}

}  // namespace b2dp
