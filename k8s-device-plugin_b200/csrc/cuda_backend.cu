// cuda_backend.cu -- the `cuda:` backend: real H100s.
//
// One worker thread per GPU owns that GPU's primary context, stream, events, pinned result
// block and the two probe buffers; callers (cgo threads, ctypes, gRPC handlers) never touch
// a CUDA "current device".  The heartbeat probe enqueues one pass on every GPU's stream before
// waiting on any (so the N kernels run concurrently), either from the calling thread with event
// polling (default, lowest latency) or through the per-GPU workers (B2DP_PROBE_VIA_WORKERS); a
// device that does not finish before the deadline yields B2DP_E_TIMEOUT / Unhealthy for that
// device only and is collected later by its worker.
//
// Replaces: the node-level text check `simpleHealthCheck` (plugin.go:161-206), the exporter
// round trip `getGPUHealth` (exporter/health.go:42-82) and the kfd link `type` read
// (allocator/device.go:143-149).  Enumeration replaces GetAMDGPUs (amdgpu.go:149-268) with
// CUDA/NVML/sysfs queries; the record layout and id formats are the reference's.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <pthread.h>
#include <sched.h>
#include <sys/mman.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <algorithm>
#include <array>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <deque>
#include <functional>
#include <map>
#include <mutex>
#include <thread>

#include "gosem.hpp"
#include "hbm_memtest.cuh"
#include "hbm_probe.cuh"
#include "hostlink_math.hpp"
#include "hostlink_selftest.cuh"
#include "internal.hpp"
#include "memtest_math.hpp"
#include "nvml_dyn.hpp"
#include "pattern_math.hpp"
#include "fp_selftest.cuh"
#include "half_selftest.cuh"
#include "int_selftest.cuh"
#include "l1_selftest.cuh"
#include "l2_selftest.cuh"
#include "rf_selftest.cuh"
#include "sync_selftest.cuh"
#include "sfu_selftest.cuh"
#include "smem_selftest.cuh"
#include "tc_selftest.cuh"
#include "units_backend.hpp"

namespace b2dp {

// the kernel shapes (kTma*, kQueue*, kReg*) are defined next to the kernels in hbm_probe.cuh
constexpr unsigned long long kFloorMinBytes = 128ull << 20;  // a ring slot well above the 50 MB L2: the pass measures HBM, not the cache

// bit b of (uint32(i) * K) summed over i < n_words, for the closed-form checksum
__global__ void pattern_bit_counts(unsigned long long n_words, unsigned long long* counts /*[32]*/) {
    unsigned int c[32];  // per-thread iterations stay far below 2^32 for any buffer that fits in HBM
#pragma unroll
    for (int b = 0; b < 32; ++b) c[b] = 0;
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_words; i += stride) {
        const uint32_t m = (uint32_t)i * kPatternMul;
#pragma unroll
        for (int b = 0; b < 32; ++b) c[b] += (m >> b) & 1u;
    }
#pragma unroll
    for (int b = 0; b < 32; ++b) {
        unsigned long long v = c[b];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if ((threadIdx.x & 31) == 0 && v) atomicAdd(&counts[b], v);
    }
}

struct Completion {
    std::mutex mu;
    std::condition_variable cv;
    bool done = false;
    void signal() { { std::lock_guard<std::mutex> g(mu); done = true; } cv.notify_all(); }
    bool wait_until(std::chrono::steady_clock::time_point tp) {
        std::unique_lock<std::mutex> l(mu);
        return cv.wait_until(l, tp, [&] { return done; });
    }
    void wait() { std::unique_lock<std::mutex> l(mu); cv.wait(l, [&] { return done; }); }
};

struct Gpu {
    int ordinal = 0;
    Device dev;                 // the enumerate record
    std::string name, pci_device_id, vbios, family;
    std::string uuid;                     // "GPU-xxxxxxxx-xxxx-xxxx-xxxx-xxxxxxxxxxxx" (cudaDeviceProp.uuid == nvmlDeviceGetUUID)
    int nvml_index = -1;                  // nvmlDeviceGetIndex: what a bare integer in NVIDIA_VISIBLE_DEVICES / a CDI name means
    std::string inforom_image, inforom_oem, inforom_ecc, inforom_power, gsp_fw;
    int64_t vram = 0, sms = 0;
    bool mig_capable = false;
    float gbs_cal = 0.f;                  // best of the calibration passes at open (this device)
    int slow_streak = 0;                  // consecutive passes below the floor (slow_passes= debounce)
    // prearm=1: the NEXT pass is enqueued in advance behind a stream wait on a host-mapped doorbell; a heartbeat then
    // only stores to the doorbell (no launch on the critical path -- after seconds of idle a launch is slow to start)
    bool armed = false;
    unsigned long long armed_seq = 0;
    uint32_t armed_seed = 0;
    volatile unsigned int* bell_h = nullptr;
    unsigned long long bell_d = 0;
    cudaEvent_t done_ev = nullptr;        // recorded between pass k and the armed pass k+1: "pass k finished"
    std::atomic<float> gbs_ref{0.f};      // the ceiling the GB/s floor is a fraction of (peer group max, ref_gbs=, or b2dp_probe_set_ref)
    std::array<unsigned long long, 32> bc{};  // host closed-form bit counts for n_vec*4 words (pattern_math.hpp)
    void* nvh = nullptr;                  // NVML device handle (optional)
    unsigned long long ecc_base = 0;      // uncorrected volatile ECC count when the context was opened
    bool have_ecc = false;
    bool xid_registered = false;
    std::atomic<unsigned long long> xid_fault{0};  // first critical Xid seen on this device (sticky, like a real fault)
    std::atomic<bool> memtest_fault{false};        // a b2dp_memtest failed or timed out (sticky until b2dp_probe_reset)
    std::atomic<bool> compute_fault{false};        // a b2dp_compute_test or b2dp_fp_test failed or timed out (likewise)
    std::atomic<bool> hostlink_fault{false};       // a b2dp_hostlink_test failed or timed out (likewise)
    int last_healthy = 1;
    // worker
    std::thread th;
    std::mutex mu;
    std::condition_variable cv;
    std::deque<std::function<void()>> q;
    bool quit = false;
    // state owned by the worker thread
    std::vector<uint4*> buf;            // ring of cfg.slots buffers: pass k reads buf[cur], writes buf[next()]
    unsigned long long n_vec = 0;       // 16-byte vectors per slot on THIS GPU (cfg.bytes / 16 unless HBM was short at open)
    bool small_ring = false;            // slots had to be smaller than requested: passes carry no GB/s floor
    bool broken = false;                // per-GPU setup failed at open: listed, never probed, always Unhealthy
    std::string broken_reason;
    ProbeCtl* ctl = nullptr;
    ProbeOut *out_h = nullptr, *out_d = nullptr;
    cudaStream_t stream = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    uint32_t seed = 0;
    int cur = 0;
    int next() const { return (cur + 1) % (int)buf.size(); }
    unsigned long long seq = 0;
    std::atomic<bool> inflight{false};  // a timed-out pass is still owned by the worker
    std::vector<char> peer_enabled;
};

// launchers=2: a second launcher thread enqueues the passes of the GPUs on the OTHER NUMA node while the caller
// enqueues its own half, so the last GPU starts ~half as late.  The helper spins for `spin_us` after a fan-out (and after
// cuda_prearm(), which the library's own ListAndWatch loop calls just before a tick is due) and sleeps on a condition
// variable otherwise; woken from sleep it still does the right thing, only later.
struct ProbeJobResult;
struct Launcher {
    std::thread th;
    std::mutex mu;
    std::condition_variable cv;
    std::atomic<unsigned long long> cmd{0}, done{0};
    std::atomic<bool> sleeping{false}, quit{false}, arm{false};
    std::vector<size_t> idx;  // gpu indices this thread launches on
    // the job (written by the caller before cmd is bumped, read by the helper after it sees the new cmd)
    std::vector<std::shared_ptr<ProbeJobResult>>* res = nullptr;
    std::vector<char>* state = nullptr;
    uint32_t variant = 0;
};

class CudaBackend {
public:
    CudaConfig cfg;
    std::vector<std::unique_ptr<Gpu>> gpus;  // sorted by dev.id
    Nvml nvml;
    std::string driver_version, driver_src_version;
    std::mutex probe_mu;  // one fan-out at a time
    std::mutex bc_mu;
    std::unique_ptr<UnitsBackend> units;             // probe=helpers / probe=off / MIG: the NVML-driven half (units_backend.hpp)
    std::vector<std::unique_ptr<std::atomic<unsigned long long>>> unit_xid;  // xid=1 in units mode: one sticky latch per unit
    void* libcuda = nullptr;                         // prearm=1: cuStreamWaitValue32 from the driver API (cudart is linked statically)
    int (*wait32)(void* stream, unsigned long long addr, unsigned value, unsigned flags) = nullptr;
    std::unique_ptr<Launcher> launcher;              // launchers=2
    std::vector<size_t> caller_idx;                  // the GPUs the calling thread enqueues (all of them without a launcher)
    cpu_set_t caller_cpus;                           // pin=1: CPUs local to the caller's GPUs
    bool have_caller_cpus = false;
    void* xid_set = nullptr;                         // NVML event set (xid=1), waited on by xid_thread only
    std::thread xid_thread;
    std::atomic<bool> xid_quit{false};
    std::mutex xid_cb_mu;
    std::function<void()> on_health_event;           // e.g. "run a heartbeat now on every ListAndWatch stream"
    void fire_health_event() {
        std::function<void()> fn;
        { std::lock_guard<std::mutex> l(xid_cb_mu); fn = on_health_event; }
        if (fn) fn();
    }
    std::map<unsigned long long, std::array<unsigned long long, 32>> bitcounts;
};

static std::string cuda_err(const char* what, cudaError_t e) {
    return std::string(what) + ": " + cudaGetErrorName(e) + " (" + cudaGetErrorString(e) + ")";
}

static void worker_loop(Gpu* g) {
    cudaSetDevice(g->ordinal);
    for (;;) {
        std::function<void()> fn;
        {
            std::unique_lock<std::mutex> l(g->mu);
            g->cv.wait(l, [&] { return g->quit || !g->q.empty(); });
            if (g->q.empty()) return;  // quit
            fn = std::move(g->q.front());
            g->q.pop_front();
        }
        fn();
    }
}

// Run fn on g's worker; returns the completion to wait on.
static std::shared_ptr<Completion> post(Gpu* g, std::function<void()> fn) {
    auto c = std::make_shared<Completion>();
    {
        std::lock_guard<std::mutex> l(g->mu);
        g->q.push_back([fn = std::move(fn), c] { fn(); c->signal(); });
    }
    g->cv.notify_one();
    return c;
}
template <class F>
static void run_sync(Gpu* g, F&& fn) { post(g, std::forward<F>(fn))->wait(); }

// Closed-form checksum of a clean buffer: computed on the HOST (pattern_math.hpp) -- a health probe must not ask the
// device under test for its own reference value.  Cached per size; the per-GPU ring size is cached in Gpu::bc.
static const std::array<unsigned long long, 32>& host_bitcounts(CudaBackend* be, unsigned long long n_words) {
    std::lock_guard<std::mutex> l(be->bc_mu);
    auto it = be->bitcounts.find(n_words);
    if (it == be->bitcounts.end()) it = be->bitcounts.emplace(n_words, pattern_bit_counts_host(n_words)).first;
    return it->second;  // std::map nodes are stable
}

static std::string read_trim(const std::string& p) {
    std::string d;
    if (!go::read_file(p, d)) return "";
    return go::trim_space(d);
}

// ---- the probe fan-out -----------------------------------------------------------------------
struct ProbeJobResult {
    cudaError_t ce = cudaSuccess;
    ProbeOut out{};
    float ms = 0;
    uint32_t seed = 0;
    unsigned long long seq = 0;
    bool seq_ok = false;
    unsigned long long n_vec = 0;   // vectors this pass covers (shrunk on a busy GPU)
    bool advance = true;            // false: verify-only prefix pass, buffers/seed stay as they are
    bool timed = false;             // bracket the kernel with CUDA events (B2DP_PROBE_EVENT_TIMING)
    int grid = 0;                   // CTAs to launch (0 = the tuned shape); diagnostic hook, see b2dp_probe_opts.grid_ctas
};

static void launch_probe(Gpu* g, unsigned long long n_vec, uint32_t variant, uint32_t seed, uint32_t delta,
                         const uint4* src, uint4* dst, unsigned long long seq, int grid = 0) {
    if (variant == B2DP_PROBE_VARIANT_R128)
        hbm_probe_r128<kRegThreads, kRegUnroll><<<grid > 0 ? grid : (int)g->sms * kRegCtasPerSm, kRegThreads, 0, g->stream>>>(
            src, dst, n_vec, seed, delta, g->ctl, g->out_d, seq);
    else
        hbm_probe_queue<kQueueCW, kQueueTileVec, kQueueStages>
            <<<grid > 0 ? grid : (int)g->sms * kQueueCtasPerSm, (kQueueCW + 2) * 32, kQueueSmem, g->stream>>>(
                src, dst, n_vec, seed, delta, g->ctl, g->out_d, seq);
}

// Enqueue one pass on g's stream (caller must have made g's device current).
static void probe_issue(Gpu* g, ProbeJobResult* r, uint32_t variant) {
    const uint32_t seed = g->seed, next = seed * 1664525u + 1013904223u;
    const unsigned long long n_vec = r->n_vec ? r->n_vec : g->n_vec;
    r->n_vec = n_vec;
    r->seed = seed;
    r->seq = ++g->seq;
    if (r->timed) cudaEventRecord(g->e0, g->stream);
    launch_probe(g, n_vec, variant, seed, r->advance ? seed ^ next : 0u, g->buf[g->cur], g->buf[g->next()], r->seq, r->grid);
    r->ce = cudaGetLastError();
    if (r->timed) cudaEventRecord(g->e1, g->stream);
}

// ---- prearm=1 ---------------------------------------------------------------------------------------------------------
// While pass k runs, pass k+1 is enqueued behind `cuStreamWaitValue32(doorbell == seq)`: a stream wait occupies no SM.
// The next heartbeat rings the doorbell (one host store per GPU) instead of launching: a launch after seconds of idle
// -- the production shape, a heartbeat every few seconds -- is slow to start work (tools/doorbell_probe.cu measures
// both ways, back to back and after idle).  An armed pass that is not
// wanted (fault repair, peek/poke/reset, P2P, a pass with other options, close) is FLUSHED: rung, waited for, its
// result ignored, the ring state not advanced -- it read and re-keyed exactly what the next ordinary pass will.
// Off by default: a pending stream wait stalls every OTHER piece of work this process submits to the same GPU (other
// streams, a second context -- measured; other processes keep their latency), so it belongs in a process whose only GPU
// user is this library.
static inline void probe_ring(Gpu* g, unsigned long long seq) { __atomic_store_n(g->bell_h, (unsigned int)seq, __ATOMIC_RELEASE); }

static void probe_arm(CudaBackend* be, Gpu* g) {  // g's device is current; pass k has just been enqueued on g->stream
    if (!be->wait32 || g->armed) return;
    const uint32_t seed = g->seed * 1664525u + 1013904223u, next = seed * 1664525u + 1013904223u;  // the state AFTER pass k
    const int M = (int)g->buf.size(), src = (g->cur + 1) % M, dst = (g->cur + 2) % M;
    cudaEventRecord(g->done_ev, g->stream);
    const unsigned long long seq = g->seq + 1;
    if (be->wait32((void*)g->stream, g->bell_d, (unsigned int)seq, 1u /*CU_STREAM_WAIT_VALUE_EQ*/) != 0) return;
    g->seq = seq;
    launch_probe(g, g->n_vec, 0u, seed, seed ^ next, g->buf[src], g->buf[dst], seq);
    if (cudaGetLastError() != cudaSuccess) { probe_ring(g, seq); return; }  // release the wait; nothing follows it
    g->armed = true;
    g->armed_seq = seq;
    g->armed_seed = seed;
}

static void probe_flush(Gpu* g) {  // discard the armed pass (see above); needs no current device
    if (!g->armed) return;
    probe_ring(g, g->armed_seq);
    cudaStreamSynchronize(g->stream);
    g->armed = false;
}

// The last CTA publishes the result block and, after a system-scope fence, the launch's sequence
// number into pinned host memory (hbm_probe.cuh finish()): seeing the number means every CTA's
// stores and the whole block are done -- completion without a driver call.
static inline bool probe_published(const Gpu* g, const ProbeJobResult* r) {
    return *(volatile const unsigned long long*)&g->out_h->seq == r->seq;
}

// After the pass completed: read the published result, advance the seed / ping-pong state.
static void probe_collect(Gpu* g, ProbeJobResult* r) {
    const unsigned long long n_vec = g->n_vec;  // repairs re-fill the whole slot
    cudaError_t e = r->ce;
    if (e == cudaSuccess && r->timed) {
        e = cudaEventSynchronize(g->e1);  // the result is already published; the event follows within ~1 us
        if (e == cudaSuccess) e = cudaEventElapsedTime(&r->ms, g->e0, g->e1);
    }
    r->ce = e;
    if (e != cudaSuccess) return;
    std::atomic_thread_fence(std::memory_order_acquire);       // the sequence number was read first (probe_published)
    memcpy(&r->out, (const void*)g->out_h, sizeof(ProbeOut));  // the block is complete once its sequence number shows
    r->seq_ok = r->out.seq == r->seq;
    if (!r->advance) {
        if (r->out.mismatches != 0 || !r->seq_ok) {  // repair the source buffer in place
            cudaSetDevice(g->ordinal);
            probe_flush(g);
            hbm_fill<256><<<(int)g->sms * 8, 256, 0, g->stream>>>(g->buf[g->cur], n_vec, g->seed);
            cudaStreamSynchronize(g->stream);
        }
        return;
    }
    g->seed = g->seed * 1664525u + 1013904223u;
    g->cur = g->next();
    if (r->out.mismatches != 0 || !r->seq_ok) {
        // report once, then start the next pass from a clean pattern: a transient flip is
        // reported exactly once, a stuck cell shows up again on the next pass
        cudaSetDevice(g->ordinal);
        probe_flush(g);  // the armed pass would read the buffer about to be repaired: discard it first
        hbm_fill<256><<<(int)g->sms * 8, 256, 0, g->stream>>>(g->buf[g->cur], n_vec, g->seed);
        cudaStreamSynchronize(g->stream);
    }
}

// "0-31,64-95" -> cpu_set_t
static bool parse_cpulist(const std::string& text, cpu_set_t* set) {
    CPU_ZERO(set);
    bool any = false;
    size_t pos = 0;
    while (pos < text.size()) {
        size_t e = text.find(',', pos);
        if (e == std::string::npos) e = text.size();
        const std::string item = text.substr(pos, e - pos);
        pos = e + 1;
        if (item.empty()) continue;
        const size_t dash = item.find('-');
        const int lo = atoi(item.c_str()), hi = dash == std::string::npos ? lo : atoi(item.c_str() + dash + 1);
        for (int c = lo; c <= hi && c < CPU_SETSIZE; ++c) { if (c >= 0) { CPU_SET(c, set); any = true; } }
    }
    return any;
}

static void launcher_loop(CudaBackend* be, Launcher* L, int spin_us) {
    unsigned long long seen = 0;
    auto spin_until = std::chrono::steady_clock::now();
    for (;;) {
        // wait for the next command: spin inside the window, sleep outside it
        for (;;) {
            if (L->quit.load(std::memory_order_acquire)) return;
            if (L->cmd.load(std::memory_order_acquire) != seen) break;
            if (L->arm.exchange(false)) spin_until = std::chrono::steady_clock::now() + std::chrono::microseconds(4 * spin_us);
            if (std::chrono::steady_clock::now() < spin_until) {
#if defined(__x86_64__)
                __builtin_ia32_pause();
#endif
                continue;
            }
            std::unique_lock<std::mutex> l(L->mu);
            L->sleeping.store(true);
            L->cv.wait(l, [&] { return L->quit.load() || L->arm.load() || L->cmd.load() != seen; });
            L->sleeping.store(false);
        }
        seen = L->cmd.load(std::memory_order_acquire);
        for (size_t i : L->idx) {
            Gpu* g = be->gpus[i].get();
            if ((*L->state)[i] != 0) continue;
            if (g->inflight.load()) { (*L->state)[i] = 2; continue; }
            cudaSetDevice(g->ordinal);
            probe_issue(g, (*L->res)[i].get(), L->variant);
        }
        L->done.store(seen, std::memory_order_release);
        spin_until = std::chrono::steady_clock::now() + std::chrono::microseconds(spin_us);
    }
}

// The library's ListAndWatch loop calls this shortly before a tick is due: the helper launcher leaves its condition
// variable and spins, so the fan-out that follows finds it hot.
void cuda_prearm(CudaBackend* be) {
    Launcher* L = be->launcher.get();
    if (!L) return;
    L->arm.store(true);
    if (L->sleeping.load()) { std::lock_guard<std::mutex> l(L->mu); L->cv.notify_one(); }
}

static void xid_listener(CudaBackend* be);

int cuda_backend_open(const CudaConfig& cfg, CudaBackend** out, std::string& err) {
    auto be = std::make_unique<CudaBackend>();
    be->cfg = cfg;
    be->nvml.load();
    // MIG: CUDA shows a process ONE compute instance (and then no other GPU), so a node with any MIG-enabled GPU is
    // enumerated through NVML and probed by one helper process per unit; this process never creates a CUDA context.
    int mode = cfg.probe_mode;
    if (mode == 0 && cfg.mig_auto && be->nvml.ok && be->nvml.device_count && be->nvml.handle_by_index && be->nvml.mig_mode) {
        unsigned cnt = 0;
        if (be->nvml.device_count(&cnt) == 0)
            for (unsigned i = 0; i < cnt; ++i) {
                void* h = nullptr;
                unsigned cur = 0, pend = 0;
                if (be->nvml.handle_by_index(i, &h) == 0 && be->nvml.mig_mode(h, &cur, &pend) == 0 && cur == 1) mode = 1;
            }
    }
    if (mode != 0) {
        int rc = units_open(cfg, be->nvml, mode == 1, &be->units, err);
        if (rc != B2DP_OK) return rc;
        {
            int n_mig = 0;
            for (auto& u : be->units->units) n_mig += u.mig_slot >= 0;
            logf(0, "NVML enumeration: %zu unit(s), %d MIG instance(s), probe=%s%s", be->units->units.size(), n_mig, mode == 1 ? "helpers" : "off",
                 cfg.probe_mode == 0 ? " (forced by MIG: CUDA shows a process one compute instance)" : "");
        }
        if (be->nvml.driver_version) {
            char buf[96] = {0};
            if (be->nvml.driver_version(buf, sizeof buf) == 0) be->driver_version = buf;
        }
        if (be->driver_version.empty()) be->driver_version = read_trim(go::join(cfg.sysroot, "sys/module/nvidia/version"));
        be->driver_src_version = read_trim(go::join(cfg.sysroot, "sys/module/nvidia/srcversion"));
        for (size_t i = 0; i < be->units->units.size(); ++i) be->unit_xid.push_back(std::make_unique<std::atomic<unsigned long long>>(0));
        // xid=1 needs no CUDA: NVML delivers critical Xid events to this process for the physical GPUs the units live on
        if (cfg.check_xid && be->nvml.event_set_create && be->nvml.register_events && be->nvml.event_wait &&
            be->nvml.event_set_create(&be->xid_set) == 0) {
            std::vector<void*> seen;
            for (auto& u : be->units->units)
                if (u.nvh && std::find(seen.begin(), seen.end(), u.nvh) == seen.end()) {
                    seen.push_back(u.nvh);
                    be->nvml.register_events(u.nvh, 0x8ull /*nvmlEventTypeXidCriticalError*/, be->xid_set);
                }
            be->xid_thread = std::thread(xid_listener, be.get());
        }
        *out = be.release();
        return B2DP_OK;
    }
    int count = 0;
    cudaError_t ce = cudaGetDeviceCount(&count);
    if (ce != cudaSuccess || count == 0) {
        err = ce != cudaSuccess ? cuda_err("cudaGetDeviceCount", ce) : "no CUDA devices";
        return B2DP_E_NOGPU;
    }
    std::vector<int> ords = cfg.devices;
    if (ords.empty()) for (int i = 0; i < count; ++i) ords.push_back(i);
    for (int o : ords) if (o < 0 || o >= count) { err = "device ordinal out of range"; return B2DP_E_INVAL; }
    for (size_t a = 0; a < ords.size(); ++a)
        for (size_t b = a + 1; b < ords.size(); ++b)
            if (ords[a] == ords[b]) { err = "device ordinal listed twice"; return B2DP_E_INVAL; }

    if (be->nvml.ok && be->nvml.driver_version) {
        char buf[96] = {0};
        if (be->nvml.driver_version(buf, sizeof buf) == 0) be->driver_version = buf;
    }
    if (be->driver_version.empty()) be->driver_version = read_trim("/sys/module/nvidia/version");
    be->driver_src_version = read_trim("/sys/module/nvidia/srcversion");

    // CPU topology nodes precede GPU nodes in a kfd tree; count NUMA nodes (>= 1)
    int n_cpu = 0;
    for (auto& p : go::glob_prefixed(go::join(cfg.sysroot, "sys/devices/system/node"), "node"))
        if (p.size() > 4 && go::is_digit(p.back())) ++n_cpu;
    if (n_cpu < 1) n_cpu = 1;

    for (int o : ords) {
        auto g = std::make_unique<Gpu>();
        g->ordinal = o;
        cudaDeviceProp prop;
        if ((ce = cudaGetDeviceProperties(&prop, o)) != cudaSuccess) { err = cuda_err("cudaGetDeviceProperties", ce); return B2DP_E_CUDA; }
        char bdf[32];
        snprintf(bdf, sizeof bdf, "%04x:%02x:%02x.0", prop.pciDomainID, prop.pciBusID, prop.pciDeviceID);
        g->dev.id = bdf;  // same shape as the reference's PCI dir names (amdgpu.go:154-155)
        char devid[32];
        snprintf(devid, sizeof devid, "%04x:%02x:%02x:0", prop.pciDomainID, prop.pciBusID, prop.pciDeviceID);  // amdgpu.go:141
        g->dev.dev_id = devid;
        g->name = prop.name;
        {
            const unsigned char* u = reinterpret_cast<const unsigned char*>(prop.uuid.bytes);
            char ub[48];
            snprintf(ub, sizeof ub, "GPU-%02x%02x%02x%02x-%02x%02x-%02x%02x-%02x%02x-%02x%02x%02x%02x%02x%02x", u[0], u[1], u[2],
                     u[3], u[4], u[5], u[6], u[7], u[8], u[9], u[10], u[11], u[12], u[13], u[14], u[15]);
            g->uuid = ub;
        }
        g->vram = (int64_t)prop.totalGlobalMem;
        g->sms = prop.multiProcessorCount;
        g->family = prop.major == 10 || prop.major == 12 ? "Blackwell" : prop.major == 9 ? "Hopper"
                    : prop.major == 8 ? (prop.minor == 9 ? "Ada" : "Ampere") : "sm_" + std::to_string(prop.major * 10 + prop.minor);
        const std::string pci_dir = go::join(cfg.sysroot, std::string("sys/bus/pci/devices/") + bdf);
        g->pci_device_id = read_trim(pci_dir + "/device");
        if (g->pci_device_id.empty()) g->pci_device_id = "0x0000";
        std::string numa = read_trim(pci_dir + "/numa_node");
        int64_t nv = 0;
        g->dev.numa = (!numa.empty() && go::atoi(numa, &nv) == go::NumErr::none) ? (int)nv : 0;
        // /dev/nvidia<minor>
        g->dev.card = o;
        bool have_minor = false;
        if (be->nvml.ok && be->nvml.handle_by_bus_id && be->nvml.minor_number) {
            void* h = nullptr;
            char busid[32];
            snprintf(busid, sizeof busid, "%08x:%02x:%02x.0", prop.pciDomainID, prop.pciBusID, prop.pciDeviceID);
            if (be->nvml.handle_by_bus_id(busid, &h) == 0) {
                g->nvh = h;
                if (be->nvml.ecc_total && be->nvml.ecc_total(h, 1 /*UNCORRECTED*/, 0 /*VOLATILE*/, &g->ecc_base) == 0)
                    g->have_ecc = true;
                unsigned mn = 0;
                if (be->nvml.minor_number(h, &mn) == 0) { g->dev.card = (int)mn; have_minor = true; }
                char vb[96] = {0};
                if (be->nvml.vbios && be->nvml.vbios(h, vb, sizeof vb) == 0) g->vbios = vb;
                unsigned ni = 0;
                if (be->nvml.index_of && be->nvml.index_of(h, &ni) == 0) g->nvml_index = (int)ni;
                if (be->nvml.uuid_of && be->nvml.uuid_of(h, vb, sizeof vb) == 0 && vb[0]) g->uuid = vb;
                // firmware label sources (the analogue of libdrm's per-block firmware versions, amdgpu.go:392-437)
                if (be->nvml.inforom_image && be->nvml.inforom_image(h, vb, sizeof vb) == 0) g->inforom_image = vb;
                if (be->nvml.inforom_object) {
                    if (be->nvml.inforom_object(h, 0, vb, sizeof vb) == 0) g->inforom_oem = vb;
                    if (be->nvml.inforom_object(h, 1, vb, sizeof vb) == 0) g->inforom_ecc = vb;
                    if (be->nvml.inforom_object(h, 2, vb, sizeof vb) == 0) g->inforom_power = vb;
                }
                if (be->nvml.gsp_firmware && be->nvml.gsp_firmware(h, vb) == 0) g->gsp_fw = vb;  // NVML_GSP_FIRMWARE_VERSION_BUF_SIZE = 64
                unsigned cur = 0, pend = 0;
                if (be->nvml.mig_mode && be->nvml.mig_mode(h, &cur, &pend) == 0) g->mig_capable = true;
            }
        }
        if (!have_minor) {
            std::string info;
            if (go::read_file(std::string("/proc/driver/nvidia/gpus/") + bdf + "/information", info)) {
                size_t p = info.find("Device Minor:");
                if (p != std::string::npos) g->dev.card = atoi(info.c_str() + p + 13);
            }
        }
        be->gpus.push_back(std::move(g));
    }
    std::sort(be->gpus.begin(), be->gpus.end(), [](const auto& a, const auto& b) { return a->dev.id < b->dev.id; });
    for (size_t i = 0; i < be->gpus.size(); ++i) {
        be->gpus[i]->dev.render_d = 128 + (int)i;
        be->gpus[i]->dev.node_id = n_cpu + (int)i;
        be->gpus[i]->peer_enabled.assign(be->gpus.size(), 0);
    }

    // xid=1: one NVML event set for the node, every GPU registered for critical Xid events
    if (cfg.check_xid && be->nvml.ok && be->nvml.event_set_create && be->nvml.register_events && be->nvml.event_wait &&
        be->nvml.event_set_create(&be->xid_set) == 0) {
        for (auto& gp : be->gpus)
            if (gp->nvh && be->nvml.register_events(gp->nvh, 0x8ull /*nvmlEventTypeXidCriticalError*/, be->xid_set) == 0)
                gp->xid_registered = true;
        be->xid_thread = std::thread(xid_listener, be.get());
    }

    // start workers and allocate per-GPU state on them
    for (auto& gp : be->gpus) gp->th = std::thread(worker_loop, gp.get());
    std::vector<std::shared_ptr<Completion>> cs;
    std::vector<cudaError_t> errs(be->gpus.size(), cudaSuccess);
    std::vector<const char*> where(be->gpus.size(), "");
    for (size_t i = 0; i < be->gpus.size(); ++i) {
        Gpu* g = be->gpus[i].get();
        const unsigned long long bytes = cfg.bytes, n_vec = cfg.bytes / 16;
        const int idx = (int)i;
        const int calib = cfg.calib;
        const int seed_idx = cfg.seed_index >= 0 ? cfg.seed_index + idx : idx;  // a helper's one device stands for unit seed_index
        g->buf.assign((size_t)cfg.slots, nullptr);
        (void)n_vec;
        cs.push_back(post(g, [g, bytes, idx, calib, seed_idx, &errs, &where] {
            cudaError_t e;
#define TRY(x) if ((e = (x)) != cudaSuccess) { errs[idx] = e; where[idx] = #x; return; }
            TRY(cudaStreamCreateWithFlags(&g->stream, cudaStreamNonBlocking));
            TRY(cudaEventCreate(&g->e0));
            TRY(cudaEventCreate(&g->e1));
            // HBM may be short when the daemon restarts under running pods: rather than fail (and take the node's
            // GPUs away from the kubelet) halve the slot size until the ring fits, down to 1 MiB
            unsigned long long slot = bytes;
            for (;;) {
                e = cudaSuccess;
                for (auto& b : g->buf) if ((e = cudaMalloc(&b, slot)) != cudaSuccess) break;
                if (e == cudaSuccess) break;
                cudaGetLastError();
                for (auto& b : g->buf) { if (b) cudaFree(b); b = nullptr; }
                if (e != cudaErrorMemoryAllocation || slot <= (1ull << 20)) { errs[idx] = e; where[idx] = "cudaMalloc(probe ring)"; return; }
                slot = (slot / 2) & ~15ull;
            }
            g->n_vec = slot / 16;
            g->small_ring = slot < bytes;
            TRY(cudaMalloc(&g->ctl, sizeof(ProbeCtl)));
            ProbeCtl init{};
            init.first_bad = ~0ull; init.t_start_ns = ~0ull;
            TRY(cudaMemcpy(g->ctl, &init, sizeof init, cudaMemcpyHostToDevice));
            TRY(cudaHostAlloc(&g->out_h, sizeof(ProbeOut), cudaHostAllocMapped));
            memset(g->out_h, 0, sizeof(ProbeOut));
            TRY(cudaHostGetDevicePointer(&g->out_d, g->out_h, 0));
            {   // doorbell for prearm=1 (allocated always: 64 bytes)
                void* bell = nullptr;
                void* bell_dev = nullptr;
                TRY(cudaHostAlloc(&bell, 64, cudaHostAllocMapped));
                memset(bell, 0, 64);
                TRY(cudaHostGetDevicePointer(&bell_dev, bell, 0));
                g->bell_h = static_cast<volatile unsigned int*>(bell);
                g->bell_d = (unsigned long long)(uintptr_t)bell_dev;
                TRY(cudaEventCreateWithFlags(&g->done_ev, cudaEventDisableTiming));
            }
            TRY(cudaFuncSetAttribute(hbm_probe_tma<kTmaCW, kTmaTileVec, kTmaStages>,
                                     cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTmaSmem));
            TRY(cudaFuncSetAttribute(hbm_probe_tma<kTmaCW, kTmaTileVec, kTmaStages>,
                                     cudaFuncAttributePreferredSharedMemoryCarveout, 100));
            TRY(cudaFuncSetAttribute(hbm_probe_queue<kQueueCW, kQueueTileVec, kQueueStages>,
                                     cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kQueueSmem));
            TRY(cudaFuncSetAttribute(hbm_probe_queue<kQueueCW, kQueueTileVec, kQueueStages>,
                                     cudaFuncAttributePreferredSharedMemoryCarveout, 100));
            g->seed = 0x5EED0000u | (uint32_t)(seed_idx & 0xffff);  // SURVEY 8(d) config 2
            g->cur = 0;
            hbm_fill<256><<<(int)g->sms * 8, 256, 0, g->stream>>>(g->buf[0], g->n_vec, g->seed);
            TRY(cudaGetLastError());
            TRY(cudaStreamSynchronize(g->stream));
            // Integer self-test of THIS GPU against the host: the pattern's bit counts, computed by the SMs, must equal
            // the host's closed form (which is what every later verdict is judged against).
            g->bc = pattern_bit_counts_host(g->n_vec * 4);
            {
                unsigned long long* d = nullptr;
                std::array<unsigned long long, 32> dev_counts{};
                TRY(cudaMalloc(&d, sizeof dev_counts));
                TRY(cudaMemsetAsync(d, 0, sizeof dev_counts, g->stream));
                pattern_bit_counts<<<(int)g->sms * 4, 256, 0, g->stream>>>(g->n_vec * 4, d);
                TRY(cudaGetLastError());
                TRY(cudaMemcpyAsync(dev_counts.data(), d, sizeof dev_counts, cudaMemcpyDeviceToHost, g->stream));
                TRY(cudaStreamSynchronize(g->stream));
                cudaFree(d);
                if (dev_counts != g->bc) { errs[idx] = cudaErrorUnknown; where[idx] = "integer self-test (pattern bit counts != host closed form)"; return; }
            }
            // Calibration: best of `calib` warm, non-advancing passes (read slot 0, write slot 1 un-re-keyed; seed and
            // ring position stay where they are) = what this device streams when healthy and idle.
            for (int k = 0; k < (calib > 0 ? calib + 1 : 0); ++k) {
                ProbeJobResult r;
                r.advance = false;
                r.timed = true;
                probe_issue(g, &r, 0u);
                if (r.ce == cudaSuccess) r.ce = cudaStreamSynchronize(g->stream);
                probe_collect(g, &r);
                TRY(r.ce);
                // the verdict's clock is the in-kernel span (first CTA start .. result published): it is there on every
                // pass, event-timed or not
                const double span_ms = (double)(r.out.t_end_ns - r.out.t_start_ns) * 1e-6;
                if (k == 0 || span_ms <= 0) continue;  // first pass warms clocks, TLBs and the instruction cache
                const float gbs = (float)(2.0 * (double)g->n_vec * 16.0 / span_ms * 1e-6);
                if (gbs > g->gbs_cal) g->gbs_cal = gbs;
            }
#undef TRY
        }));
    }
    for (auto& c : cs) c->wait();
    // One GPU that cannot be set up (fallen off the bus, exclusive-process mode held by a tenant, no memory at
    // all) must not take the node's other GPUs away from the kubelet: it stays in the device list and is
    // reported Unhealthy on every heartbeat.  Only a node with no usable GPU fails to open.
    size_t n_broken = 0;
    for (size_t i = 0; i < errs.size(); ++i) {
        const bool forced = std::find(cfg.break_devices.begin(), cfg.break_devices.end(), (int)i) != cfg.break_devices.end();
        if (errs[i] == cudaSuccess && !forced) continue;
        Gpu* g = be->gpus[i].get();
        g->broken = true;
        g->broken_reason = forced ? "setup failure injected (break=)" : cuda_err(where[i], errs[i]);
        g->last_healthy = 0;
        logf(2, "%s could not be set up and will be reported Unhealthy: %s", g->dev.id.c_str(), g->broken_reason.c_str());
        err = g->broken_reason + " on " + g->dev.id;
        ++n_broken;
    }
    if (n_broken == be->gpus.size()) {
        CudaBackend* raw = be.release();
        cuda_backend_close(raw);
        return B2DP_E_CUDA;
    }
    // The ceiling a device's GB/s floor is a fraction of: ref_gbs= if given, else the best calibration of any
    // device of the same product with the same ring size -- a part that is already slow when the daemon starts is
    // judged against its siblings, not against itself.
    for (auto& g : be->gpus) {
        if (g->broken) continue;
        float ref = cfg.ref_gbs;
        if (ref <= 0)
            for (auto& o : be->gpus)
                if (!o->broken && o->name == g->name && o->n_vec == g->n_vec) ref = std::max(ref, o->gbs_cal);
        g->gbs_ref.store(ref);
        logf(0, "%s %s ring %d x %llu MiB%s, calibrated %.0f GB/s, ceiling %.0f GB/s, floor %.0f GB/s", g->dev.id.c_str(), g->name.c_str(),
             (int)g->buf.size(), (unsigned long long)(g->n_vec * 16 >> 20), g->small_ring ? " (shrunk: HBM was short)" : "", g->gbs_cal, ref,
             cfg.min_gbs > 0 ? cfg.min_gbs : cfg.min_frac * ref);
    }
    if (cfg.prearm && cfg.launchers < 2) {
        be->libcuda = dlopen("libcuda.so.1", RTLD_NOW | RTLD_LOCAL);
        if (be->libcuda) {
            void* f = dlsym(be->libcuda, "cuStreamWaitValue32_v2");
            if (!f) f = dlsym(be->libcuda, "cuStreamWaitValue32");
            be->wait32 = reinterpret_cast<int (*)(void*, unsigned long long, unsigned, unsigned)>(f);
        }
        if (!be->wait32) logf(1, "prearm=1: cuStreamWaitValue32 is not available; passes are launched at each heartbeat");
    }
    // launchers=2: split the GPUs by NUMA node (GPU 0's node stays with the caller; one NUMA node: split in halves)
    for (size_t i = 0; i < be->gpus.size(); ++i) be->caller_idx.push_back(i);
    if (cfg.launchers >= 2 && be->gpus.size() >= 2) {
        auto L = std::make_unique<Launcher>();
        be->caller_idx.clear();
        const int numa0 = be->gpus[0]->dev.numa;
        for (size_t i = 0; i < be->gpus.size(); ++i)
            (be->gpus[i]->dev.numa == numa0 ? be->caller_idx : L->idx).push_back(i);
        if (L->idx.empty()) {
            be->caller_idx.clear();
            for (size_t i = 0; i < be->gpus.size(); ++i) (i < (be->gpus.size() + 1) / 2 ? be->caller_idx : L->idx).push_back(i);
        }
        Launcher* raw = L.get();
        CudaBackend* bp = be.get();
        raw->th = std::thread(launcher_loop, bp, raw, cfg.spin_us);
        cpu_set_t set;  // keep the helper on the CPUs next to its GPUs
        if (parse_cpulist(read_trim(go::join(cfg.sysroot, "sys/bus/pci/devices/" + be->gpus[raw->idx[0]]->dev.id + "/local_cpulist")), &set))
            pthread_setaffinity_np(raw->th.native_handle(), sizeof set, &set);
        be->launcher = std::move(L);
    }
    if (cfg.pin_caller)
        be->have_caller_cpus = parse_cpulist(
            read_trim(go::join(cfg.sysroot, "sys/bus/pci/devices/" + be->gpus[be->caller_idx[0]]->dev.id + "/local_cpulist")), &be->caller_cpus);
    *out = be.release();
    return B2DP_OK;
}

void cuda_backend_close(CudaBackend* be) {
    if (!be) return;
    if (be->units) {
        be->xid_quit = true;
        if (be->xid_thread.joinable()) be->xid_thread.join();
        { std::lock_guard<std::mutex> l(be->xid_cb_mu); be->on_health_event = nullptr; }
        units_close(be->units.get());
        if (be->xid_set && be->nvml.event_set_free) be->nvml.event_set_free(be->xid_set);
        delete be;
        return;
    }
    be->xid_quit = true;
    if (be->xid_thread.joinable()) be->xid_thread.join();
    { std::lock_guard<std::mutex> l(be->xid_cb_mu); be->on_health_event = nullptr; }
    if (be->launcher) {
        be->launcher->quit.store(true);
        { std::lock_guard<std::mutex> l(be->launcher->mu); be->launcher->cv.notify_all(); }
        if (be->launcher->th.joinable()) be->launcher->th.join();
    }
    for (auto& gp : be->gpus) {
        Gpu* g = gp.get();
        if (!g->th.joinable()) continue;
        post(g, [g] {
            probe_flush(g);
            if (g->stream) cudaStreamSynchronize(g->stream);
            if (g->bell_h) cudaFreeHost(const_cast<unsigned int*>(g->bell_h));
            if (g->done_ev) cudaEventDestroy(g->done_ev);
            for (uint4* b : g->buf) if (b) cudaFree(b);
            if (g->ctl) cudaFree(g->ctl);
            if (g->out_h) cudaFreeHost(g->out_h);
            if (g->e0) cudaEventDestroy(g->e0);
            if (g->e1) cudaEventDestroy(g->e1);
            if (g->stream) cudaStreamDestroy(g->stream);
        })->wait();
        { std::lock_guard<std::mutex> l(g->mu); g->quit = true; }
        g->cv.notify_all();
        g->th.join();
    }
    if (be->xid_set && be->nvml.event_set_free) be->nvml.event_set_free(be->xid_set);
    if (be->libcuda) dlclose(be->libcuda);
    delete be;
}

int cuda_device_count(CudaBackend* be) { return be->units ? (int)be->units->units.size() : (int)be->gpus.size(); }
float cuda_min_gbs(CudaBackend* be) { return be->cfg.min_gbs; }
void cuda_set_health_event_callback(CudaBackend* be, std::function<void()> fn) {
    std::lock_guard<std::mutex> l(be->xid_cb_mu);
    be->on_health_event = std::move(fn);
}

int cuda_enumerate(CudaBackend* be, std::vector<Device>& out, std::string&) {
    out.clear();
    if (be->units) { for (auto& u : be->units->units) out.push_back(u.dev); return B2DP_OK; }
    for (auto& g : be->gpus) out.push_back(g->dev);
    return B2DP_OK;
}

int cuda_node_health(CudaBackend* be) {
    // the analogue of "a GPU node exists in the kfd topology" (plugin.go:198-201):
    // the driver still answers and reports the devices this context was opened on
    if (be->units) {  // no CUDA in this process: NVML must still count the physical GPUs the units live on
        unsigned cnt = 0;
        return be->nvml.device_count && be->nvml.device_count(&cnt) == 0 && cnt > 0 && !be->units->units.empty() ? 1 : 0;
    }
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess) return 0;
    return count >= (int)be->gpus.size() && !be->gpus.empty() ? 1 : 0;
}

void cuda_label_source(CudaBackend* be, LabelSource& src) {
    src.native = true;
    src.driver_version = be->driver_version;
    src.driver_src_version = be->driver_src_version;
    if (be->units) {
        bool migc = !be->units->units.empty();
        for (auto& u : be->units->units) {
            src.family.push_back(u.family);
            src.product_name.push_back(u.name);
            src.device_id.push_back(u.pci_device_id);
            src.vbios.push_back(u.vbios);
            src.firmware.push_back(u.firmware);
            src.vram_bytes.push_back(u.vram);
            src.sm_count.push_back(u.sms);
            migc = migc && u.mig_capable;
        }
        src.part_supported[0] = src.part_supported[1] = migc;
        return;
    }
    bool mig = !be->gpus.empty();
    for (auto& g : be->gpus) {
        src.family.push_back(g->family);
        src.product_name.push_back(g->name);
        src.device_id.push_back(g->pci_device_id);
        src.vbios.push_back(g->vbios);
        // per-block firmware versions, the key scheme of main.go:116-144 ("<block>.fw.<version>")
        std::vector<std::pair<std::string, std::string>> fw;
        if (!g->vbios.empty()) fw.push_back({"vbios", g->vbios});
        if (!g->inforom_image.empty()) fw.push_back({"inforom-img", g->inforom_image});
        if (!g->inforom_oem.empty()) fw.push_back({"inforom-oem", g->inforom_oem});
        if (!g->inforom_ecc.empty()) fw.push_back({"inforom-ecc", g->inforom_ecc});
        if (!g->inforom_power.empty()) fw.push_back({"inforom-pwr", g->inforom_power});
        if (!g->gsp_fw.empty()) fw.push_back({"gsp", g->gsp_fw});
        src.firmware.push_back(std::move(fw));
        src.vram_bytes.push_back(g->vram);
        src.sm_count.push_back(g->sms);
        mig = mig && g->mig_capable;
    }
    src.part_supported[0] = src.part_supported[1] = mig;
}

// Xids that report an application's own fault (bad kernel, MMU fault of a user context, preemption,
// user-stopped) rather than a broken device -- the list NVIDIA's own device plugin ignores.
static bool xid_is_application_error(unsigned long long xid) {
    switch (xid) { case 13: case 31: case 43: case 45: case 68: case 109: return true; default: return false; }
}

static void latch_xid(Gpu* g, unsigned long long xid) {
    unsigned long long none = 0;
    if (!xid_is_application_error(xid)) g->xid_fault.compare_exchange_strong(none, xid ? xid : 999);
}

// xid=1: the only thread that waits on the NVML event set.  A device-level Xid is latched on its device and
// reported at once (on_health_event), not at the next pulse.
static void xid_listener(CudaBackend* be) {
    Nvml::EventData d{};
    while (!be->xid_quit.load()) {
        const int rc = be->nvml.event_wait(be->xid_set, &d, 200);  // ms; NVML_ERROR_TIMEOUT (10) when idle
        if (rc != 0) {
            if (rc != 10) std::this_thread::sleep_for(std::chrono::milliseconds(200));  // a failing set must not spin
            continue;
        }
        if (d.type != 0x8ull) continue;  // nvmlEventTypeXidCriticalError
        bool hit = false;
        for (auto& g : be->gpus)
            if (g->nvh == d.device && !xid_is_application_error(d.data)) { latch_xid(g.get(), d.data); hit = true; }
        if (be->units && !xid_is_application_error(d.data))
            for (size_t i = 0; i < be->units->units.size(); ++i) {
                const Unit& u = be->units->units[i];
                // a MIG-attributed Xid names its GPU instance; 0xFFFFFFFF = the whole GPU (every instance on it)
                if (u.nvh != d.device || (u.mig_slot >= 0 && d.gi != 0xffffffffu && d.gi != u.gi)) continue;
                unsigned long long none = 0;
                be->unit_xid[i]->compare_exchange_strong(none, d.data ? d.data : 999);
                hit = true;
            }
        if (hit) { logf(2, "critical Xid %llu reported by NVML: device(s) latched Unhealthy", d.data); be->fire_health_event(); }
    }
}

int cuda_probe(CudaBackend* be, const b2dp_probe_opts* opts, std::vector<b2dp_probe_result>& out, std::string& err) {
    std::lock_guard<std::mutex> pl(be->probe_mu);
    if (be->units) {
        if (!be->units->helpers) { err = "probe=off: this context enumerates only"; return B2DP_E_UNSUPPORTED; }
        const int rc = units_probe(be->units.get(), opts, out, err);
        if (rc == B2DP_OK && be->cfg.check_xid)
            for (size_t i = 0; i < out.size() && i < be->unit_xid.size(); ++i)
                if (be->unit_xid[i]->load()) { out[i].flags |= B2DP_RES_XID; out[i].healthy = 0; be->units->units[i].last_healthy = 0; }
        return rc;
    }
    int rc = B2DP_OK;
    const uint32_t variant = opts ? (opts->flags & B2DP_PROBE_VARIANT_MASK) : 0;
    const bool via_workers = opts && (opts->flags & B2DP_PROBE_VIA_WORKERS);
    const bool timed = opts && (opts->flags & B2DP_PROBE_EVENT_TIMING);
    const uint32_t timeout_ms = opts && opts->timeout_ms ? opts->timeout_ms : 5000;  // health.go:37
    // GB/s floor: an absolute one if the call or the context names it (min_gbs), else min_frac (default 0.8,
    // BASELINE.json's ">= 80 % of HBM peak") of the device's calibrated ceiling
    const float abs_floor = opts && opts->min_gbs > 0 ? opts->min_gbs : be->cfg.min_gbs;
    const int grid = opts ? (int)std::min<uint32_t>(opts->grid_ctas, 1u << 16) : 0;  // diagnostic hook, bounded
    const size_t n = be->gpus.size();
    std::vector<std::shared_ptr<ProbeJobResult>> res(n);
    std::vector<std::shared_ptr<Completion>> cs(n);
    std::vector<char> state(n, 0);  // 0 pending, 1 done, 2 timed out / busy
    std::vector<char> rung_any(n, 0);  // prearm=1: this pass was already enqueued and only had its doorbell rung
    const auto deadline = std::chrono::steady_clock::now() + std::chrono::milliseconds(timeout_ms);
    for (size_t i = 0; i < n; ++i) { res[i] = std::make_shared<ProbeJobResult>(); res[i]->timed = timed; res[i]->grid = grid; }
    for (size_t i = 0; i < n; ++i) if (be->gpus[i]->broken) state[i] = 4;  // never launched on
    // busy policy (tenant workloads): a 2 GiB-traffic probe steals bandwidth from a pod that owns the
    // GPU; `busy=skip` keeps the last verdict, `busy=shrink` verifies a small prefix without re-keying
    std::vector<uint32_t> rflags(n, 0);
    if (be->cfg.busy_policy != 0 && be->nvml.ok && be->nvml.running_procs) {
        for (size_t i = 0; i < n; ++i) {
            Gpu* g = be->gpus[i].get();
            if (!g->nvh || state[i] != 0) continue;
            unsigned cnt = 0;
            const int nrc = be->nvml.running_procs(g->nvh, &cnt, nullptr);  // count only (INSUFFICIENT_SIZE = 7)
            if ((nrc != 0 && nrc != 7) || cnt <= 1) continue;              // this process holds one context itself
            if (be->cfg.busy_policy == 1) { state[i] = 3; rflags[i] = B2DP_RES_SKIPPED_BUSY; }
            else {
                unsigned long long sv = be->cfg.shrink_bytes / 16;
                res[i]->n_vec = sv < g->n_vec ? (sv ? sv : 1) : g->n_vec;
                res[i]->advance = false;
                rflags[i] = B2DP_RES_SHRUNK;
            }
        }
    }

    if (via_workers) {
        // fully isolated path: each GPU's own thread launches and waits; a wedged driver call can
        // only ever block that worker
        for (size_t i = 0; i < n; ++i) {  // launch everywhere before waiting anywhere
            Gpu* g = be->gpus[i].get();
            auto r = res[i];
            if (state[i] != 0) continue;
            if (g->inflight.load()) { state[i] = 2; continue; }
            g->inflight.store(true);  // until collected: a pass that misses the deadline still owns seed/ring state
            cs[i] = post(g, [g, r, variant] {
                probe_flush(g);
                probe_issue(g, r.get(), variant);
                if (r->ce == cudaSuccess) r->ce = cudaStreamSynchronize(g->stream);
                probe_collect(g, r.get());
                g->inflight.store(false);
            });
        }
        for (size_t i = 0; i < n; ++i)
            if (state[i] == 0) state[i] = cs[i]->wait_until(deadline) ? 1 : 2;
    } else {
        // low-latency path (default): the calling thread enqueues on every GPU's stream, then polls
        // the completion events; no thread hand-offs on the critical path.  A device that misses
        // the deadline is handed to its worker to be collected whenever it finishes.  The caller's
        // current CUDA device is restored before returning.
        int prev_dev = -1;
        cudaGetDevice(&prev_dev);
        if (be->have_caller_cpus) {  // pin=1: keep the enqueue + poll thread on the CPUs next to its GPUs (once per thread)
            static thread_local const CudaBackend* pinned_for = nullptr;
            if (pinned_for != be) { pthread_setaffinity_np(pthread_self(), sizeof be->caller_cpus, &be->caller_cpus); pinned_for = be; }
        }
        Launcher* L = be->launcher.get();
        unsigned long long cmd = 0;
        if (L) {  // hand the other NUMA node's GPUs to the helper, then enqueue our own
            L->res = &res; L->state = &state; L->variant = variant;
            cmd = L->cmd.fetch_add(1) + 1;  // seq_cst: ordered against the `sleeping` load below (store/load pair on both sides)
            if (L->sleeping.load()) { std::lock_guard<std::mutex> l(L->mu); L->cv.notify_one(); }
        }
        // prearm=1: a pass with the default options may be the one that is already enqueued behind its doorbell
        const bool can_arm = be->wait32 && variant == B2DP_PROBE_VARIANT_TMA && !timed && grid == 0 && be->cfg.busy_policy == 0;
        std::vector<char> arm_ok(n, 0);  // decided before any pass is issued (issuing fills in r->n_vec)
        for (size_t i = 0; i < n; ++i) arm_ok[i] = can_arm && res[i]->n_vec == 0 && res[i]->advance;
        auto armable = [&](size_t i) { return arm_ok[i] != 0; };
        std::vector<char> rung(n, 0);
        for (size_t i : be->caller_idx) {  // doorbells first: one host store each, every armed GPU starts within microseconds
            Gpu* g = be->gpus[i].get();
            if (state[i] != 0 || !g->armed || !armable(i) || g->inflight.load()) continue;
            ProbeJobResult* r = res[i].get();
            r->n_vec = g->n_vec; r->seed = g->armed_seed; r->seq = g->armed_seq; r->ce = cudaSuccess;
            probe_ring(g, g->armed_seq);
            g->armed = false;
            rung[i] = rung_any[i] = 1;
        }
        for (size_t i : be->caller_idx) {
            Gpu* g = be->gpus[i].get();
            if (state[i] != 0 || rung[i]) continue;
            if (g->inflight.load()) { state[i] = 2; continue; }
            cudaSetDevice(g->ordinal);
            probe_flush(g);  // an armed pass that does not fit this call's options is discarded
            probe_issue(g, res[i].get(), variant);
        }
        if (L) while (L->done.load(std::memory_order_acquire) != cmd) {
#if defined(__x86_64__)
            __builtin_ia32_pause();
#endif
        }
        // while the passes run: enqueue the NEXT one behind its doorbell (overlapped with ~0.33 ms of GPU work)
        if (can_arm)
            for (size_t i : be->caller_idx) {
                Gpu* g = be->gpus[i].get();
                if (state[i] != 0 || !armable(i) || res[i]->ce != cudaSuccess) continue;
                cudaSetDevice(g->ordinal);
                probe_arm(be, g);
            }
        size_t pending = 0;
        for (size_t i = 0; i < n; ++i) pending += state[i] == 0;
        unsigned spins = 0;
        while (pending) {
            for (size_t i = 0; i < n; ++i) {
                if (state[i] != 0) continue;
                Gpu* g = be->gpus[i].get();
                if (res[i]->ce == cudaSuccess && !probe_published(g, res[i].get())) {
                    // not there yet; now and then ask the driver too, so that a faulted kernel (which
                    // never publishes) is reported at once instead of at the deadline
                    if ((spins & 0x3ff) != 0x3ff) continue;
                    const cudaError_t q = cudaStreamQuery(g->stream);
                    if (q == cudaErrorNotReady) continue;
                    if (q != cudaSuccess) res[i]->ce = q;
                }
                probe_collect(g, res[i].get());  // no driver call unless event-timed or a repair is due
                state[i] = 1;
                --pending;
            }
            if (pending && (++spins & 0x3ff) == 0 && std::chrono::steady_clock::now() > deadline) break;
        }
        for (size_t i = 0; i < n; ++i) {
            if (state[i] != 0) continue;
            state[i] = 2;
            Gpu* g = be->gpus[i].get();
            auto r = res[i];
            g->inflight.store(true);
            post(g, [g, r] {
                // with a pass armed behind this one, "this pass is done" is the event recorded between the two
                if (r->ce == cudaSuccess) r->ce = g->armed ? cudaEventSynchronize(g->done_ev) : cudaStreamSynchronize(g->stream);
                probe_collect(g, r.get());
                probe_flush(g);
                g->inflight.store(false);
            });
        }
        if (prev_dev >= 0) cudaSetDevice(prev_dev);
    }

    out.assign(n, b2dp_probe_result{});
    for (size_t i = 0; i < n; ++i) {
        b2dp_probe_result& o = out[i];
        o.device = (int)i;
        o.bytes = 2ull * be->gpus[i]->n_vec * 16;
        o.first_bad_word = ~0ull;
        o.flags = rflags[i] | (be->gpus[i]->small_ring ? B2DP_RES_SMALL_RING : 0u) | (!via_workers && rung_any[i] ? B2DP_RES_PREARMED : 0u);
        if (state[i] == 2) { o.err = B2DP_E_TIMEOUT; o.healthy = 0; be->gpus[i]->last_healthy = 0; continue; }
        if (state[i] == 3) { o.bytes = 0; o.healthy = be->gpus[i]->last_healthy; continue; }  // skipped: last verdict stands
        if (state[i] == 4) { o.bytes = 0; o.err = B2DP_E_CUDA; o.healthy = 0; err = be->gpus[i]->broken_reason + " on " + be->gpus[i]->dev.id; continue; }
        const ProbeJobResult& r = *res[i];
        o.seed = r.seed;
        if (r.ce != cudaSuccess) {
            o.err = B2DP_E_CUDA; o.healthy = 0;
            be->gpus[i]->last_healthy = 0;
            err = cuda_err("probe", r.ce) + " on " + be->gpus[i]->dev.id;
            continue;
        }
        Gpu* g = be->gpus[i].get();
        o.expected_checksum = expected_checksum_from_counts(
            r.n_vec == g->n_vec ? g->bc : host_bitcounts(be, r.n_vec * 4), r.n_vec * 4, r.seed);  // host closed form
        o.bytes = 2ull * r.n_vec * 16;
        o.checksum = r.out.checksum;
        o.mismatches = r.out.mismatches;
        o.first_bad_word = r.out.first_bad;
        o.ms_event = r.ms;  // 0 unless B2DP_PROBE_EVENT_TIMING
        o.ms_device = (float)((double)(r.out.t_end_ns - r.out.t_start_ns) * 1e-6);
        const float ms_for_rate = r.timed ? r.ms : o.ms_device;
        o.gbs = ms_for_rate > 0 ? (float)((double)o.bytes / (double)ms_for_rate * 1e-6) : 0.f;
        // the verdict's rate: bytes over the in-kernel span, the same clock the ceiling was calibrated with (o.gbs is
        // the event-timed figure when B2DP_PROBE_EVENT_TIMING asks for the roofline's clock)
        const float gbs_span = o.ms_device > 0 ? (float)((double)o.bytes / (double)o.ms_device * 1e-6) : 0.f;
        o.gbs_ref = g->gbs_ref.load();
        o.frac = o.gbs_ref > 0 ? gbs_span / o.gbs_ref : 0.f;
        // verdict (oracle/probe.py probe_healthy).  No GB/s floor for a pass that shares the GPU with a tenant by
        // design (shrunk / small ring); the fractional floor needs a ring that streams from HBM (> the 50 MB L2).
        float floor = 0.f;
        if (!(o.flags & (B2DP_RES_SHRUNK | B2DP_RES_SMALL_RING))) {
            if (abs_floor > 0) floor = abs_floor;
            else if (o.bytes / 2 >= kFloorMinBytes && o.gbs_ref > 0) floor = be->cfg.min_frac * o.gbs_ref;
            else o.flags |= B2DP_RES_NO_FLOOR;
        }
        o.min_gbs_applied = floor;
        bool fast_enough = gbs_span >= floor;
        if (fast_enough) g->slow_streak = 0;
        else {
            o.flags |= B2DP_RES_SLOW;
            // slow_passes=K: only the K-th consecutive slow pass is a verdict (a one-heartbeat dip is flagged, not failed);
            // integrity faults are never debounced
            if (++g->slow_streak < be->cfg.slow_passes) fast_enough = true;
            // Slow path only: a pass that shared HBM bandwidth with another process on the GPU says nothing about the
            // part.  NVML counts the compute processes; this one holds one context itself.
            unsigned cnt = 0;
            if (be->nvml.ok && be->nvml.running_procs && g->nvh) {
                const int nrc = be->nvml.running_procs(g->nvh, &cnt, nullptr);  // count only (INSUFFICIENT_SIZE = 7)
                if ((nrc == 0 || nrc == 7) && cnt > 1) { o.flags |= B2DP_RES_CONTENDED; fast_enough = true; }
            }
        }
        o.healthy = (r.seq_ok && o.mismatches == 0 && o.checksum == o.expected_checksum && fast_enough) ? 1 : 0;
        if (be->cfg.check_ecc && be->gpus[i]->have_ecc) {  // opt-in: an NVML query per device per pass
            unsigned long long now = 0;
            if (be->nvml.ecc_total(be->gpus[i]->nvh, 1, 0, &now) == 0 && now > be->gpus[i]->ecc_base) {
                o.flags |= B2DP_RES_ECC;
                o.healthy = 0;
            }
            // HBM row remapping: a failed remap means the bad row stays in use (the part is due for replacement)
            unsigned corr = 0, unc = 0, pending = 0, failed = 0;
            if (be->nvml.remapped_rows && be->nvml.remapped_rows(be->gpus[i]->nvh, &corr, &unc, &pending, &failed) == 0 && failed) {
                o.flags |= B2DP_RES_ECC;
                o.healthy = 0;
            }
        }
        be->gpus[i]->last_healthy = o.healthy;
    }
    if (be->cfg.check_xid) {  // opt-in: a critical Xid since open fails the device whatever the pass said
        for (size_t i = 0; i < n; ++i)
            if (be->gpus[i]->xid_fault.load()) {
                out[i].flags |= B2DP_RES_XID;
                out[i].healthy = 0;
                be->gpus[i]->last_healthy = 0;
            }
    }
    for (size_t i = 0; i < n; ++i)  // a failed memory test fails the device whatever the pass said, until reset
        if (be->gpus[i]->memtest_fault.load(std::memory_order_relaxed)) {
            out[i].flags |= B2DP_RES_MEMTEST;
            out[i].healthy = 0;
            be->gpus[i]->last_healthy = 0;
        }
    for (size_t i = 0; i < n; ++i)  // and so does a failed compute self-test
        if (be->gpus[i]->compute_fault.load(std::memory_order_relaxed)) {
            out[i].flags |= B2DP_RES_COMPUTE;
            out[i].healthy = 0;
            be->gpus[i]->last_healthy = 0;
        }
    for (size_t i = 0; i < n; ++i)  // and a failed host-link self-test
        if (be->gpus[i]->hostlink_fault.load(std::memory_order_relaxed)) {
            out[i].flags |= B2DP_RES_HOSTLINK;
            out[i].healthy = 0;
            be->gpus[i]->last_healthy = 0;
        }
    return B2DP_OK;
}

static Gpu* gpu_at(CudaBackend* be, int device, std::string& err) {
    if (device < 0 || device >= (int)be->gpus.size()) { err = "device index out of range"; return nullptr; }
    if (be->gpus[device]->broken) { err = "device was not set up: " + be->gpus[device]->broken_reason; return nullptr; }
    return be->gpus[device].get();
}

// helpers mode: forward a single-unit operation to the unit's child
static int units_forward(CudaBackend* be, int device, HelperReq q, std::string& err, std::vector<uint32_t>* payload = nullptr) {
    UnitsBackend* ub = be->units.get();
    if (!ub->helpers) { err = "probe=off: this context enumerates only"; return B2DP_E_UNSUPPORTED; }
    if (device < 0 || device >= (int)ub->units.size()) { err = "device index out of range"; return B2DP_E_INVAL; }
    Unit& u = ub->units[device];
    if (u.broken) { err = "device was not set up: " + u.broken_reason; return B2DP_E_INVAL; }
    HelperRsp r{};
    int rc = units_call(u, q, &r, 30000, payload);
    if (rc == B2DP_OK && r.rc != B2DP_OK) { rc = r.rc; err = r.text; }
    else if (rc != B2DP_OK) {
        // the stream is out of step (a late answer may carry a payload): drop this child, the next heartbeat restarts it
        err = "probe helper did not answer";
        units_kill(u);
        u.broken = true;
        u.broken_reason = "probe helper unresponsive";
    }
    return rc;
}

int cuda_inject_fault(CudaBackend* be, int device, uint64_t word, uint32_t mask, std::string& err) {
    if (be->units && word == ~0ull) {  // synthetic critical Xid, as in the in-process mode below
        if (device < 0 || device >= (int)be->unit_xid.size()) { err = "device index out of range"; return B2DP_E_INVAL; }
        if (be->cfg.check_xid && !xid_is_application_error(mask)) {
            unsigned long long none = 0;
            be->unit_xid[device]->compare_exchange_strong(none, mask ? mask : 999);
            be->fire_health_event();
        }
        return B2DP_OK;
    }
    if (be->units) {
        std::lock_guard<std::mutex> pl(be->probe_mu);
        HelperReq q{};
        q.op = HOP_INJECT; q.a = word; q.b = mask;
        return units_forward(be, device, q, err);
    }
    if (word == ~0ull) {  // synthetic critical-Xid event `mask`, handled like one delivered by NVML (xid=1)
        Gpu* g = gpu_at(be, device, err);
        if (!g) return B2DP_E_INVAL;
        // like xid_listener: no backend lock is held while the context's callback runs (it takes the context lock,
        // and Start()/labels/export take that lock before probe_mu)
        if (be->cfg.check_xid && !xid_is_application_error(mask)) {
            latch_xid(g, mask);
            be->fire_health_event();
        }
        return B2DP_OK;
    }
    std::lock_guard<std::mutex> pl(be->probe_mu);
    Gpu* g = gpu_at(be, device, err);
    if (!g) return B2DP_E_INVAL;
    if (word >= g->n_vec * 4) { err = "word index out of range"; return B2DP_E_INVAL; }
    cudaError_t ce = cudaSuccess;
    run_sync(g, [&] {
        probe_flush(g);
        hbm_poke<<<1, 1, 0, g->stream>>>(reinterpret_cast<uint32_t*>(g->buf[g->cur]), word, mask);
        ce = cudaStreamSynchronize(g->stream);
    });
    if (ce != cudaSuccess) { err = cuda_err("hbm_poke", ce); return B2DP_E_CUDA; }
    return B2DP_OK;
}

int cuda_probe_reset(CudaBackend* be, int device, std::string& err) {
    std::lock_guard<std::mutex> pl(be->probe_mu);
    if (be->units) {
        for (int i = 0; i < (int)be->units->units.size(); ++i) {
            if (device >= 0 && device != i) continue;
            be->unit_xid[i]->store(0);  // operator acknowledgement
            if (be->units->units[i].broken || !be->units->helpers) continue;
            HelperReq q{};
            q.op = HOP_RESET;
            int rc = units_forward(be, i, q, err);
            if (rc != B2DP_OK) return rc;
        }
        return device >= (int)be->units->units.size() ? B2DP_E_INVAL : B2DP_OK;
    }
    for (int i = 0; i < (int)be->gpus.size(); ++i) {
        if (device >= 0 && device != i) continue;
        Gpu* g = be->gpus[i].get();
        if (g->broken) continue;
        g->xid_fault.store(0);  // operator acknowledgement: a latched Xid is cleared together with the buffers
        g->memtest_fault.store(false);  // and so is a failed memory test
        g->compute_fault.store(false);  // and a failed compute self-test
        g->hostlink_fault.store(false);  // and a failed host-link self-test
        cudaError_t ce = cudaSuccess;
        run_sync(g, [&] {
            probe_flush(g);
            hbm_fill<256><<<(int)g->sms * 8, 256, 0, g->stream>>>(g->buf[g->cur], g->n_vec, g->seed);
            ce = cudaStreamSynchronize(g->stream);
        });
        if (ce != cudaSuccess) { err = cuda_err("hbm_fill", ce); return B2DP_E_CUDA; }
    }
    if (device >= (int)be->gpus.size()) { err = "device index out of range"; return B2DP_E_INVAL; }
    return B2DP_OK;
}

int cuda_probe_peek(CudaBackend* be, int device, uint64_t word, uint32_t* out, uint64_t n, std::string& err) {
    std::lock_guard<std::mutex> pl(be->probe_mu);
    if (be->units) {
        for (uint64_t done = 0; done < n;) {  // 1 Mi words per exchange
            const uint64_t chunk = std::min<uint64_t>(n - done, 1u << 20);
            HelperReq q{};
            q.op = HOP_PEEK; q.a = word + done; q.b = chunk;
            std::vector<uint32_t> payload;
            int rc = units_forward(be, device, q, err, &payload);
            if (rc != B2DP_OK) return rc;
            memcpy(out + done, payload.data(), (size_t)chunk * 4);
            done += chunk;
        }
        return B2DP_OK;
    }
    Gpu* g = gpu_at(be, device, err);
    if (!g) return B2DP_E_INVAL;
    if (word + n > g->n_vec * 4) { err = "range out of bounds"; return B2DP_E_INVAL; }
    cudaError_t ce = cudaSuccess;
    run_sync(g, [&] {
        probe_flush(g);
        ce = cudaMemcpyAsync(out, reinterpret_cast<const uint32_t*>(g->buf[g->cur]) + word, n * 4, cudaMemcpyDeviceToHost,
                             g->stream);
        if (ce == cudaSuccess) ce = cudaStreamSynchronize(g->stream);
    });
    if (ce != cudaSuccess) { err = cuda_err("peek", ce); return B2DP_E_CUDA; }
    return B2DP_OK;
}

// What the NVIDIA container runtime / a CDI spec calls the device `id` names: the GPU UUID (default, unambiguous)
// or the NVML index.  NOT the /dev/nvidia minor: minors and NVML indices differ on HGX boards.
std::string cuda_runtime_id(CudaBackend* be, const std::string& id, bool by_index) {
    if (be->units) {
        for (auto& u : be->units->units)
            if (u.dev.id == id) {
                if (!by_index || u.nvml_index < 0) return u.uuid;
                // NVIDIA_VISIBLE_DEVICES index syntax: "<gpu>" or "<gpu>:<mig device index>"
                return u.mig_slot >= 0 ? std::to_string(u.nvml_index) + ":" + std::to_string(u.mig_slot) : std::to_string(u.nvml_index);
            }
        return "";
    }
    for (auto& g : be->gpus)
        if (g->dev.id == id) {
            if (by_index && g->nvml_index >= 0) return std::to_string(g->nvml_index);
            return g->uuid;
        }
    return "";
}

int cuda_set_ref(CudaBackend* be, int device, float gbs_ref, std::string& err) {
    if (be->units) {
        std::lock_guard<std::mutex> pl(be->probe_mu);
        if (device >= (int)be->units->units.size()) { err = "device index out of range"; return B2DP_E_INVAL; }
        for (int i = 0; i < (int)be->units->units.size(); ++i) {
            if ((device >= 0 && device != i) || be->units->units[i].broken) continue;
            Unit& u = be->units->units[i];
            u.gbs_ref = gbs_ref > 0 ? gbs_ref : u.gbs_cal;
            HelperReq q{};
            q.op = HOP_SETREF;
            memcpy(&q.a, &u.gbs_ref, sizeof(float));
            int rc = units_forward(be, i, q, err);
            if (rc != B2DP_OK) return rc;
        }
        return B2DP_OK;
    }
    if (device >= (int)be->gpus.size()) { err = "device index out of range"; return B2DP_E_INVAL; }
    for (int i = 0; i < (int)be->gpus.size(); ++i) {
        if (device >= 0 && device != i) continue;
        Gpu* g = be->gpus[i].get();
        g->gbs_ref.store(gbs_ref > 0 ? gbs_ref : g->gbs_cal);  // <= 0: back to this device's own calibration
    }
    return B2DP_OK;
}

int cuda_describe(CudaBackend* be, int device, b2dp_probe_info* o, std::string& err) {
    if (device < 0 || device >= cuda_device_count(be)) { err = "device index out of range"; return B2DP_E_INVAL; }
    if (be->units) {
        std::lock_guard<std::mutex> pl(be->probe_mu);  // a fan-out may be restarting this unit's helper
        const Unit& u = be->units->units[device];
        o->slot_bytes = u.slot_bytes; o->total_memory = (uint64_t)u.vram; o->sm_count = (int32_t)u.sms; o->slots = be->cfg.slots;
        o->gbs_cal = u.gbs_cal; o->gbs_ref = u.gbs_ref; o->usable = u.broken ? 0 : 1; o->via_helper = be->units->helpers ? 1 : 0;
        copy_str(o->uuid, sizeof o->uuid, u.uuid);
        copy_str(o->name, sizeof o->name, u.name);
        return B2DP_OK;
    }
    const Gpu* g = be->gpus[device].get();
    o->slot_bytes = g->n_vec * 16; o->total_memory = (uint64_t)g->vram; o->sm_count = (int32_t)g->sms; o->slots = (int32_t)g->buf.size();
    o->gbs_cal = g->gbs_cal; o->gbs_ref = g->gbs_ref.load(); o->usable = g->broken ? 0 : 1; o->via_helper = 0;
    copy_str(o->uuid, sizeof o->uuid, g->uuid);
    copy_str(o->name, sizeof o->name, g->name);
    return B2DP_OK;
}

bool cuda_device_paths(CudaBackend* be, const std::string& id, std::vector<std::string>& out) {
    if (be->units) {
        for (auto& u : be->units->units)
            if (u.dev.id == id) {
                out.push_back("/dev/nvidia" + std::to_string(u.parent_minor));
                if (u.mig_slot >= 0) {  // a MIG instance needs its GPU-instance and compute-instance capability nodes too
                    if (u.cap_gi >= 0) out.push_back("/dev/nvidia-caps/nvidia-cap" + std::to_string(u.cap_gi));
                    if (u.cap_ci >= 0) out.push_back("/dev/nvidia-caps/nvidia-cap" + std::to_string(u.cap_ci));
                }
                return true;
            }
        return false;
    }
    for (auto& g : be->gpus)
        if (g->dev.id == id) { out.push_back("/dev/nvidia" + std::to_string(g->dev.card)); return true; }
    return false;
}

// ---- on-demand memory test (b2dp_memtest) ------------------------------------------------------
// The march of hbm_memtest.cuh over the free HBM of one GPU, on that GPU's worker.  Every segment is freed before the
// job ends, whatever happened.
constexpr uint32_t kMemtestTimeoutMs = 60000;

template <int MODE>
static void launch_march(Gpu* g, const MarchSegs& segs, unsigned int tiles_per_seg, unsigned long long n_tiles,
                         uint32_t inv, uint32_t delta, ProbeCtl* ctl, ProbeOut* out, unsigned long long seq) {
    hbm_march_tma<kTmaCW, kTmaTileVec, kTmaStages, MODE>
        <<<(int)g->sms * kTmaCtasPerSm, (kTmaCW + 1) * 32, kTmaSmem, g->stream>>>(segs, tiles_per_seg, n_tiles, inv,
                                                                                  delta, ctl, out, seq);
}

template <int MODE>
static cudaError_t march_attributes() {
    cudaError_t e = cudaFuncSetAttribute(hbm_march_tma<kTmaCW, kTmaTileVec, kTmaStages, MODE>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTmaSmem);
    if (e == cudaSuccess)
        e = cudaFuncSetAttribute(hbm_march_tma<kTmaCW, kTmaTileVec, kTmaStages, MODE>,
                                 cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    return e;
}

static void memtest_one(CudaBackend* be, Gpu* g, const b2dp_memtest_opts& o, uint32_t timeout_ms, b2dp_memtest_result* r,
                        std::string* err) {
    constexpr uint64_t kTileBytes = (uint64_t)kTmaTileVec * 16;
    std::vector<uint64_t> got;       // sizes of the segments obtained
    std::vector<void*> seg;
    ProbeCtl* ctl = nullptr;
    ProbeOut* out_h = nullptr;
    ProbeOut* out_d = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    bool timed_out = false;
    cudaError_t ce = cudaSuccess;
    const char* where = "";
    MemtestEvidence ev;
    auto release = [&] {  // every path ends here: nothing the test allocated outlives it
        if (g->stream) cudaStreamSynchronize(g->stream);
        for (void* p : seg) cudaFree(p);
        if (ctl) cudaFree(ctl);
        if (out_h) cudaFreeHost(out_h);
        if (e0) cudaEventDestroy(e0);
        if (e1) cudaEventDestroy(e1);
    };
#define MT_TRY(x) if ((ce = (x)) != cudaSuccess) { where = #x; goto done; }
    {
        probe_flush(g);  // an armed heartbeat pass must not run underneath
        size_t free_b = 0, total_b = 0;
        MT_TRY(cudaMemGetInfo(&free_b, &total_b));
        r->free_before = free_b;
        r->total_memory = total_b;
        // the small blocks first: they must not be what fails once the segments have taken the memory
        MT_TRY(cudaMalloc(&ctl, kMarchElements * sizeof(ProbeCtl)));
        MT_TRY(cudaHostAlloc(&out_h, kMarchElements * sizeof(ProbeOut), cudaHostAllocMapped));
        memset(out_h, 0, kMarchElements * sizeof(ProbeOut));
        MT_TRY(cudaHostGetDevicePointer(&out_d, out_h, 0));
        {
            ProbeCtl init[kMarchElements] = {};
            for (auto& c : init) { c.first_bad = ~0ull; c.t_start_ns = ~0ull; }
            MT_TRY(cudaMemcpy(ctl, init, sizeof init, cudaMemcpyHostToDevice));
        }
        MT_TRY(cudaEventCreate(&e0));
        MT_TRY(cudaEventCreate(&e1));
        MT_TRY(march_attributes<MARCH_WRITE>());
        MT_TRY(march_attributes<MARCH_READ_WRITE>());
        MT_TRY(march_attributes<MARCH_READ>());
        const std::vector<uint64_t> plan = memtest_plan(free_b, total_b, o.reserve_bytes, o.max_bytes);
        if (plan.empty()) r->flags |= B2DP_MT_EMPTY;
        for (uint64_t bytes : plan) {  // a tenant may allocate meanwhile: test what was obtained
            void* p = nullptr;
            const cudaError_t a = cudaMalloc(&p, bytes);
            if (a != cudaSuccess) {
                cudaGetLastError();
                r->flags |= B2DP_MT_PARTIAL;
                break;
            }
            seg.push_back(p);
            got.push_back(bytes);
        }
        r->n_segments = (int32_t)got.size();
        for (uint64_t b : got) r->bytes_tested += b;
        if (got.empty()) { ev.launch_ok = true; goto done; }  // nothing to test

        MarchSegs segs{};
        for (size_t k = 0; k < got.size(); ++k) {
            segs.base[k] = static_cast<uint4*>(seg[k]);
            segs.seed[k] = memtest_segment_seed(r->seed, (uint32_t)k);
        }
        const unsigned int tiles_per_seg = (unsigned int)(got[0] / kTileBytes);
        const unsigned long long n_tiles = r->bytes_tested / kTileBytes;
        const unsigned long long n_words = r->bytes_tested / 4, seg_words = got[0] / 4;
        unsigned long long corr0 = 0, unc0 = 0;
        const bool ecc = g->nvh && be->nvml.ecc_total && be->nvml.ecc_total(g->nvh, 1, 0, &unc0) == 0 &&
                         be->nvml.ecc_total(g->nvh, 0, 0, &corr0) == 0;
        if (!ecc) r->flags |= B2DP_MT_NO_ECC;

        MT_TRY(cudaEventRecord(e0, g->stream));
        launch_march<MARCH_WRITE>(g, segs, tiles_per_seg, n_tiles, 0u, 0u, ctl + 0, out_d + 0, 1);
        if (o.fault_mask) {
            if (o.fault_word < n_words) {
                const unsigned long long s = o.fault_word / seg_words;
                hbm_poke<<<1, 1, 0, g->stream>>>(static_cast<uint32_t*>(seg[s]), o.fault_word - s * seg_words, o.fault_mask);
            } else {
                r->err = B2DP_E_INVAL;  // not injected; the test runs as it would without the hook
            }
        }
        launch_march<MARCH_READ_WRITE>(g, segs, tiles_per_seg, n_tiles, 0u, ~0u, ctl + 1, out_d + 1, 2);
        launch_march<MARCH_READ_WRITE>(g, segs, tiles_per_seg, n_tiles, ~0u, ~0u, ctl + 2, out_d + 2, 3);
        launch_march<MARCH_READ>(g, segs, tiles_per_seg, n_tiles, 0u, 0u, ctl + 3, out_d + 3, 4);
        MT_TRY(cudaGetLastError());
        MT_TRY(cudaEventRecord(e1, g->stream));
        const auto deadline = std::chrono::steady_clock::now() + std::chrono::milliseconds(timeout_ms);
        for (;;) {
            const cudaError_t q = cudaEventQuery(e1);
            if (q == cudaSuccess) break;
            if (q != cudaErrorNotReady) { ce = q; where = "march"; goto done; }
            if (std::chrono::steady_clock::now() > deadline) { timed_out = true; break; }
            std::this_thread::sleep_for(std::chrono::microseconds(200));
        }
        // past the deadline the verdict is made, but the memory can only be returned once the kernels are done
        MT_TRY(cudaEventSynchronize(e1));
        MT_TRY(cudaEventElapsedTime(&r->ms, e0, e1));
        if (ecc) {
            unsigned long long corr1 = corr0, unc1 = unc0;
            be->nvml.ecc_total(g->nvh, 1, 0, &unc1);
            be->nvml.ecc_total(g->nvh, 0, 0, &corr1);
            r->ecc_uncorrected = unc1 > unc0 ? unc1 - unc0 : 0;
            r->ecc_corrected = corr1 > corr0 ? corr1 - corr0 : 0;
        }
        unsigned rc_corr = 0, rc_unc = 0, pending = 0, failed = 0;
        if (g->nvh && be->nvml.remapped_rows && be->nvml.remapped_rows(g->nvh, &rc_corr, &rc_unc, &pending, &failed) == 0) {
            ev.remap_failed = failed != 0;
            ev.remap_pending = pending != 0;
        }
        ev.ecc_uncorrected = r->ecc_uncorrected;
        if (r->ecc_corrected) r->flags |= B2DP_MT_ECC_CORRECTED;
        if (r->ecc_uncorrected || ev.remap_failed || ev.remap_pending) r->flags |= B2DP_MT_ECC;
        std::atomic_thread_fence(std::memory_order_acquire);
        bool seq_ok = true;
        r->first_bad_word = ~0ull;
        for (int k = 0; k < kMarchElements; ++k) {
            ProbeOut po;
            memcpy(&po, (const void*)&out_h[k], sizeof po);  // published by the element's last CTA; the stream is done
            seq_ok = seq_ok && po.seq == (unsigned long long)(k + 1);
            ev.mismatches[k] = r->mismatches[k] = po.mismatches;
            ev.checksum[k] = po.checksum;
            if (po.mismatches && po.first_bad < r->first_bad_word) r->first_bad_word = po.first_bad;
        }
        ev.expected[1] = ev.expected[3] = memtest_expected_checksum(got, r->seed, 0u);
        ev.expected[2] = memtest_expected_checksum(got, r->seed, ~0u);
        ev.launch_ok = seq_ok && !timed_out;
        if (r->ms > 0) r->gbs = (float)(6.0 * (double)r->bytes_tested / (double)r->ms * 1e-6);
    }
done:
#undef MT_TRY
    release();
    if (ce != cudaSuccess) {
        cudaGetLastError();
        r->err = B2DP_E_CUDA;
        r->healthy = 0;
        *err = cuda_err(where, ce) + " on " + g->dev.id;
    } else if (timed_out) {
        r->err = B2DP_E_TIMEOUT;
        r->healthy = 0;
    } else {
        r->healthy = memtest_healthy(ev) ? 1 : 0;
    }
}

// NVML lists a compute process on the GPU other than this one (which holds a context itself).  Without NVML process
// accounting the GPU counts as idle.
static bool used_by_another_process(CudaBackend* be, Gpu* g) {
    if (!be->nvml.ok || !be->nvml.running_procs || !g->nvh) return false;
    unsigned cnt = 0;
    const int nrc = be->nvml.running_procs(g->nvh, &cnt, nullptr);  // count only (INSUFFICIENT_SIZE = 7)
    return (nrc == 0 || nrc == 7) && cnt > 1;
}

static int cuda_memtest(CudaBackend* be, int device, const b2dp_memtest_opts* opts, std::vector<b2dp_memtest_result>& out,
                        std::string& err) {
    if (be->units) {
        err = "the memory test runs in-process only (not with probe=helpers / probe=off / MIG)";
        return B2DP_E_UNSUPPORTED;
    }
    if (device < -1 || device >= (int)be->gpus.size()) { err = "device index out of range"; return B2DP_E_INVAL; }
    const b2dp_memtest_opts o = opts ? *opts : b2dp_memtest_opts{};
    const uint32_t timeout_ms = o.timeout_ms ? o.timeout_ms : kMemtestTimeoutMs;
    bool latched = false;
    {
        std::lock_guard<std::mutex> pl(be->probe_mu);  // a heartbeat waits for a running memory test
        const uint32_t seed = (uint32_t)std::chrono::steady_clock::now().time_since_epoch().count() * kPatternMul;
        std::vector<size_t> sel;
        for (size_t i = 0; i < be->gpus.size(); ++i) if (device < 0 || (int)i == device) sel.push_back(i);
        out.assign(sel.size(), b2dp_memtest_result{});
        std::vector<std::string> errs(sel.size());
        std::vector<std::shared_ptr<Completion>> cs(sel.size());
        for (size_t k = 0; k < sel.size(); ++k) {
            Gpu* g = be->gpus[sel[k]].get();
            b2dp_memtest_result* r = &out[k];
            r->device = (int32_t)sel[k];
            r->seed = seed ^ ((uint32_t)sel[k] << 16);
            r->first_bad_word = ~0ull;
            r->total_memory = (uint64_t)g->vram;
            if (g->broken) { r->err = B2DP_E_CUDA; errs[k] = g->broken_reason + " on " + g->dev.id; continue; }
            if (!(o.flags & B2DP_MT_EVEN_IF_BUSY) && used_by_another_process(be, g)) {
                r->flags |= B2DP_MT_SKIPPED_BUSY;
                r->healthy = g->last_healthy;
                continue;
            }
            std::string* e = &errs[k];
            cs[k] = post(g, [be, g, o, timeout_ms, r, e] { memtest_one(be, g, o, timeout_ms, r, e); });
        }
        for (size_t k = 0; k < sel.size(); ++k) {
            if (cs[k]) cs[k]->wait();  // no deadline here: the segments must be back before the call returns
            if (!errs[k].empty()) err = errs[k];
            if (!cs[k]) continue;       // skipped (busy) or never set up: nothing ran, nothing is latched
            Gpu* g = be->gpus[sel[k]].get();
            const b2dp_memtest_result& r = out[k];
            if (!r.healthy) { g->memtest_fault.store(true); latched = true; }
            logf(r.healthy ? 0 : 2, "%s memtest: %s, %llu MiB in %d segment(s)%s, mismatches %llu/%llu/%llu, first bad word %lld, "
                 "ECC corrected %llu uncorrected %llu%s, %.1f ms, %.0f GB/s%s", g->dev.id.c_str(),
                 r.healthy ? "Healthy" : "Unhealthy (latched)", (unsigned long long)(r.bytes_tested >> 20), r.n_segments,
                 (r.flags & B2DP_MT_PARTIAL) ? " (partial)" : "", (unsigned long long)r.mismatches[1],
                 (unsigned long long)r.mismatches[2], (unsigned long long)r.mismatches[3], (long long)r.first_bad_word,
                 (unsigned long long)r.ecc_corrected, (unsigned long long)r.ecc_uncorrected,
                 (r.flags & B2DP_MT_NO_ECC) ? " (not available)" : "", r.ms, r.gbs,
                 r.err == B2DP_E_TIMEOUT ? ", timed out" : "");
        }
    }
    // like the Xid latch: running ListAndWatch loops send a heartbeat now (no backend lock is held while they do)
    if (latched) be->fire_health_event();
    return B2DP_OK;
}

// ---- on-demand compute self-tests (b2dp_compute_test, b2dp_fp_test, b2dp_sfu_test, b2dp_smem_test,
// b2dp_regfile_test, b2dp_int_test, b2dp_l2_test, b2dp_half_test, b2dp_sync_test, b2dp_l1_test) ------------------
// One launch per format on one GPU, on that GPU's worker: tc_selftest.cuh (tensor cores: BF16, FP8, INT8),
// fp_selftest.cuh (FP32 FMA, FP64 FMA, FP64 tensor cores), sfu_selftest.cuh (the special-function unit),
// smem_selftest.cuh (shared memory and the SM-to-SM DSMEM path), rf_selftest.cuh (the register file), int_selftest.cuh
// (the integer pipes and the warp-exchange network), l2_selftest.cuh (the L2 and its atomic units) or half_selftest.cuh
// (the 16-bit pipes and the type converters).  The host builds
// every operand table and every comparison value itself (compute_test_math.hpp, fp_test_math.hpp, smem_test_math.hpp,
// rf_test_math.hpp, int_test_math.hpp, half_test_math.hpp): a health test must not ask the device under test for its own reference values.  The SFU test departs from that rule, because no
// bit-level model of MUFU is published: its reference step (sfu_reference) runs one CTA on every SM, takes each result
// word's majority over the SMs, names every SM that disagrees, and bounds the majority against the exact function on
// the host; no SM is ever judged against its own output.  The tests share this driver -- grid sizing, records, tally,
// deadline, busy skip and the release of every allocation before the job ends, whatever happened -- through a
// DiagSuite.
constexpr uint32_t kComputeTestDefaultMs = 1000;
constexpr int kDiagScratchHeaderWords = 64;  // DiagSuite::scratch's header
static_assert(kL2HdrWords == kDiagScratchHeaderWords, "l2_selftest's scratch header is the driver's");

using CtKernel = void (*)(const uint8_t*, const uint32_t*, unsigned long long, int, uint32_t, CtRecord*,
                          unsigned long long, uint32_t*);

// The host's inputs of one launch per format: kCtTiles tables of table_bytes[f] and [kCtTiles][kCtThreads] checks.
struct DiagTables {
    std::vector<uint8_t> tables[kCtFormats];
    std::vector<uint32_t> checks[kCtFormats];
};

// What a reference step found on one GPU.
struct DiagRef {
    bool run = true;    // every reference record arrived and every word has a majority: the timed launches can run
    bool clean = true;  // and no CTA dissents from the majority, and every majority result passes the guard
    int bad_sm[kCtFormats] = {-1, -1, -1};    // per format: the lowest dissenting SM id, and its CTA's first bad tile
    int bad_tile[kCtFormats] = {-1, -1, -1};
};

struct DiagSuite {
    const char* log_name;                      // "compute test" / "FP test"
    const char* kernel_name;                   // for a CUDA error
    const char* format_names;                  // "bf16/fp8/int8" / "fp32/fp64/dmma" in the log line
    const CtKernel* kernels;                   // product instantiation per format
    const uint32_t* smem;                      // dynamic shared memory per format
    const uint32_t* table_bytes;               // bytes of one tile's table per format
    void (*build_tile)(uint32_t seed, int fmt, int tile, uint8_t* table, uint32_t* check);
    double (*macs_per_tile)(int fmt);          // multiply-adds of one comparison (null with `scratch`: it sets them)
    bool per_device_seed;                      // seed ^ (device << 16) per GPU, tables built on each worker; else one
                                               // seed and one set of tables per call
    // Optional step on the worker before the timed launches (the SFU test's reference launch; null for the tensor and
    // FP tests): fills `own` with this GPU's tables and checks, `ref` and r's reference tallies.
    // Its deadline is the call's: the timed launches get what is left of timeout_ms.
    cudaError_t (*reference)(Gpu* g, const b2dp_compute_test_opts& o, std::chrono::steady_clock::time_point deadline,
                             const DiagTables& in, DiagTables& own, DiagRef& ref, b2dp_compute_test_result* r,
                             const char** where, bool* timed_out);
    const char* rate_format;                   // the log's tflops[] text; null: "%.0f/%.0f/%.0f TFLOP/s"
    // Optional grid sizing (the shared-memory test; null: every CTA of cudaOccupancyMaxActiveBlocksPerMultiprocessor
    // on every SM), after the kernel's shared-memory attributes are set.  On an error it names the cause in *where.
    cudaError_t (*size_grid)(Gpu* g, int fmt, int* grid, const char** where);
    bool ecc;                                  // read NVML's volatile ECC totals around the timed launches
    const char* test_name;                     // in the error of a backend without the test; null: by the fields above
    // Optional per-format device scratch buffer (the L2 test's spans and hot block; null: none): its size in bytes
    // for `grid` CTAs, the kDiagScratchHeaderWords header words copied to its start (the rest is zeroed), and the
    // per-CTA multiply-adds of one comparison, which depend on the buffer's size and take macs_per_tile's place.  Its
    // pointer is the kernel's last argument; it is allocated and released with the other buffers.
    cudaError_t (*scratch)(Gpu* g, int fmt, int grid, size_t* bytes, uint32_t* header, double* macs_per_cta,
                           const char** where);
    bool cooperative;                          // launch with cudaLaunchCooperativeKernel (every CTA co-resident)
    // Optional per-format shared-memory carve-out in percent (the L1 test's 0: the largest L1 the hardware allows;
    // null: 100).
    const int* carveout = nullptr;
    // Optional host objects the kernels read (the L1 test's CUDA array, texture objects and constant bank; null: none).
    // bind runs on the worker after the buffers exist and before the timed launches, with the call's seed and every
    // format's scratch buffer; an error is a CUDA error of the call, named in *where, and nothing launches.  unbind runs
    // in the release after the stream is synchronized, on every path, and destroys whatever bind made in *state.
    cudaError_t (*bind)(Gpu* g, uint32_t seed, const DiagTables& tabs, uint32_t* const* scratch, void** state,
                        const char** where) = nullptr;
    void (*unbind)(void* state) = nullptr;
};

static void ct_suite_tile(uint32_t seed, int fmt, int tile, uint8_t* table, uint32_t* check) {
    CtTile t;
    ct_build_tile(seed, fmt, tile, t);
    memcpy(table, t.image.data(), t.image.size());
    memcpy(check, t.check, sizeof t.check);
}
static void ft_suite_tile(uint32_t seed, int fmt, int tile, uint8_t* table, uint32_t* check) {
    FtTile t;
    ft_build_tile(seed, fmt, tile, t);
    memcpy(table, t.table.data(), t.table.size());
    memcpy(check, t.check, sizeof t.check);
}

static const CtKernel kCtKernels[kCtFormats] = {tc_selftest<CT_BF16, false>, tc_selftest<CT_FP8, false>,
                                                tc_selftest<CT_INT8, false>};
static const uint32_t kCtSmem[kCtFormats] = {CtShape<CT_BF16>::SMEM, CtShape<CT_FP8>::SMEM, CtShape<CT_INT8>::SMEM};
static const CtKernel kFtKernels[kFtFormats] = {fp_selftest<FT_FP32, false>, fp_selftest<FT_FP64, false>,
                                                fp_selftest<FT_DMMA, false>};
static const uint32_t kFtSmem[kFtFormats] = {0, 0, 0};
static const uint32_t kFtTableBytes[kFtFormats] = {ft_table_bytes(FT_FP32), ft_table_bytes(FT_FP64),
                                                   ft_table_bytes(FT_DMMA)};
static const DiagSuite kTensorSuite = {"compute test", "tc_selftest", "bf16/fp8/int8", kCtKernels, kCtSmem, kCtSmem,
                                       ct_suite_tile, ct_macs_per_tile, true};
static const DiagSuite kFpSuite = {"FP test", "fp_selftest", "fp32/fp64/dmma", kFtKernels, kFtSmem, kFtTableBytes,
                                   ft_suite_tile, ft_macs_per_tile, false};

// ---- the SFU test's suite and reference step ----
static_assert(kSfNoConsensus == B2DP_CT_NO_CONSENSUS && kSfOutOfBound == B2DP_CT_OUT_OF_BOUND, "sfu_test_math.hpp flags");
constexpr int kSfRefSmem = 120 << 10;  // more than half an SM's shared memory, unused: no SM can hold two reference CTAs
static const CtKernel kSfKernels[kSfFormats] = {sfu_selftest<SF_F32, false>, sfu_selftest<SF_ROOT, false>,
                                                sfu_selftest<SF_F16, false>};
static const CtKernel kSfRefKernels[kSfFormats] = {sfu_selftest<SF_F32, true>, sfu_selftest<SF_ROOT, true>,
                                                   sfu_selftest<SF_F16, true>};
static const uint32_t kSfSmem[kSfFormats] = {0, 0, 0};
static const uint32_t kSfTableBytes[kSfFormats] = {sf_table_bytes(SF_F32), sf_table_bytes(SF_ROOT),
                                                   sf_table_bytes(SF_F16)};
// The operand tables only: the checks come from each GPU's reference launch.
static void sf_suite_tile(uint32_t seed, int fmt, int tile, uint8_t* table, uint32_t* check) {
    sf_build_table(seed, fmt, tile, reinterpret_cast<uint32_t*>(table));
    memset(check, 0, kCtThreads * sizeof(uint32_t));
}
// tflops[] = 2 x this x comparisons / ms, and the SFU test counts one op per MUFU result
static double sf_suite_half_results(int fmt) { return 0.5 * sf_results_per_tile(fmt); }

// The reference launch of every format (kSfRefKernels: g->sms CTAs, one round, one per SM because of their shared
// memory, every result word of round 0, repetition 0 dumped), then sf_consensus on each: this GPU's checks, its
// dissenting SMs (counted in mismatches[] and bad_sm_mask), B2DP_CT_NO_CONSENSUS / B2DP_CT_OUT_OF_BOUND, and
// B2DP_CT_PARTIAL_COVERAGE if the records name fewer SM ids than the device has.  Releases what it allocated.
static cudaError_t sfu_reference(Gpu* g, const b2dp_compute_test_opts& o,
                                 std::chrono::steady_clock::time_point deadline, const DiagTables& in, DiagTables& own,
                                 DiagRef& ref, b2dp_compute_test_result* r, const char** where, bool* timed_out) {
    const auto t0 = std::chrono::steady_clock::now();
    const int n = (int)g->sms;
    uint8_t* tab = nullptr;
    uint32_t* dump = nullptr;
    CtRecord* rec_h = nullptr;
    CtRecord* rec_d = nullptr;
    cudaEvent_t ev = nullptr;
    cudaError_t ce = cudaSuccess;
    std::vector<uint32_t> words((size_t)n * kCtTiles * kCtThreads * kSfMaxWords);
    size_t table_max = 0;
    for (int f = 0; f < kSfFormats; ++f) table_max = std::max(table_max, in.tables[f].size());
#define SF_TRY(x) if ((ce = (x)) != cudaSuccess) { *where = #x; goto out; }
    SF_TRY(cudaMalloc(&tab, table_max));
    SF_TRY(cudaMalloc(&dump, words.size() * sizeof(uint32_t)));
    SF_TRY(cudaHostAlloc(&rec_h, (size_t)kSfFormats * n * sizeof(CtRecord), cudaHostAllocMapped));
    memset(rec_h, 0, (size_t)kSfFormats * n * sizeof(CtRecord));
    SF_TRY(cudaHostGetDevicePointer(&rec_d, rec_h, 0));
    SF_TRY(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    for (int f = 0; f < kSfFormats; ++f) {
        SF_TRY(cudaFuncSetAttribute(kSfRefKernels[f], cudaFuncAttributeMaxDynamicSharedMemorySize, kSfRefSmem));
        SF_TRY(cudaFuncSetAttribute(kSfRefKernels[f], cudaFuncAttributePreferredSharedMemoryCarveout, 100));
        SF_TRY(cudaMemcpy(tab, in.tables[f].data(), in.tables[f].size(), cudaMemcpyHostToDevice));
        const unsigned long long seq = (unsigned long long)(f + 1);
        kSfRefKernels[f]<<<n, kCtThreads, kSfRefSmem, g->stream>>>(tab, nullptr, 0ull, o.fault_sm, o.fault_mask,
                                                                     rec_d + (size_t)f * n, seq, dump);
        SF_TRY(cudaGetLastError());
        SF_TRY(cudaEventRecord(ev, g->stream));
        for (;;) {
            const cudaError_t q = cudaEventQuery(ev);
            if (q == cudaSuccess) break;
            if (q != cudaErrorNotReady) { ce = q; *where = "sfu_selftest (reference launch)"; goto out; }
            if (std::chrono::steady_clock::now() > deadline) { *timed_out = true; break; }
            std::this_thread::sleep_for(std::chrono::milliseconds(1));
        }
        SF_TRY(cudaEventSynchronize(ev));  // the buffers can only be released once the kernel is done
        if (*timed_out) goto out;
        std::atomic_thread_fence(std::memory_order_acquire);
        SF_TRY(cudaMemcpy(words.data(), dump, (size_t)n * kCtTiles * kCtThreads * kSfWords[f] * sizeof(uint32_t),
                          cudaMemcpyDeviceToHost));
        const CtRecord* recs = rec_h + (size_t)f * n;
        SfConsensus cons;
        sf_consensus(f, words.data(), recs, n, seq, reinterpret_cast<const uint32_t*>(in.tables[f].data()), cons);
        own.tables[f] = in.tables[f];
        own.checks[f] = cons.check;
        for (int c = 0; c < n; ++c)
            if (recs[c].seq == seq) r->nsmid = std::max<int32_t>(r->nsmid, (int32_t)recs[c].nsmid);
        r->flags |= cons.flags();
        if (cons.sm_ids < r->sm_count) r->flags |= B2DP_CT_PARTIAL_COVERAGE;
        r->mismatches[f] += cons.dissents;
        for (int i = 0; i < 4; ++i) r->bad_sm_mask[i] |= cons.bad_sm_mask[i];
        ref.bad_sm[f] = cons.first_bad_sm;
        ref.bad_tile[f] = cons.first_bad_tile;
        if (cons.arrived != n || cons.no_consensus) ref.run = false;
        if (!cons.clean()) ref.clean = false;
        logf(cons.clean() ? 0 : 2, "%s SFU test reference %s: %d/%d records, %d SM ids, %llu dissents, %llu words "
             "without a majority, %llu results out of bound", g->dev.id.c_str(), f == SF_F32 ? "f32" : f == SF_ROOT ? "root" : "f16",
             cons.arrived, n, cons.sm_ids, cons.dissents, cons.no_consensus, cons.out_of_bound);
    }
    logf(0, "%s SFU test reference launches and consensus: %.1f ms", g->dev.id.c_str(),
         std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count());
out:
#undef SF_TRY
    if (g->stream) cudaStreamSynchronize(g->stream);
    if (tab) cudaFree(tab);
    if (dump) cudaFree(dump);
    if (rec_h) cudaFreeHost(rec_h);
    if (ev) cudaEventDestroy(ev);
    return ce;
}

static const DiagSuite kSfuSuite = {"SFU test", "sfu_selftest", "f32/root/f16", kSfKernels, kSfSmem, kSfTableBytes,
                                    sf_suite_tile, sf_suite_half_results, false, sfu_reference,
                                    "%.2f/%.2f/%.2f T results/s"};

// ---- the shared-memory test's suite ----
static const CtKernel kShKernels[kShFormats] = {smem_selftest<SH_WORD, false>, smem_selftest<SH_BYTE, false>,
                                                smem_selftest<SH_DSMEM, false>};
static const uint32_t kShSmem[kShFormats] = {kShBytes, kShBytes, kShBytes};
static const uint32_t kShTableBytes[kShFormats] = {kShTableWords * 4, kShTableWords * 4, kShTableWords * 4};
static void sh_suite_tile(uint32_t seed, int fmt, int tile, uint8_t* table, uint32_t* check) {
    sh_build_tile(seed, fmt, tile, reinterpret_cast<uint32_t*>(table), check);
}
// tflops[] = 2 x this x comparisons / ms: TB/s of shared-memory traffic
static double sh_suite_half_bytes(int fmt) { return 0.5 * sh_bytes_per_tile(fmt); }

// One CTA per SM for SH_WORD / SH_BYTE (kShBytes each: no SM holds two); SH_DSMEM: every co-resident cluster of two.
static cudaError_t sh_size_grid(Gpu* g, int fmt, int* grid, const char** where) {
    int dev = 0, optin = 0;
    cudaError_t ce = cudaGetDevice(&dev);
    if (ce == cudaSuccess) ce = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    if (ce != cudaSuccess) { *where = "cudaDeviceGetAttribute(cudaDevAttrMaxSharedMemoryPerBlockOptin)"; return ce; }
    if (optin < (int)kShBytes) {
        *where = "smem_selftest: the device's cudaDevAttrMaxSharedMemoryPerBlockOptin is below the 232448 B the test needs";
        return cudaErrorInvalidConfiguration;
    }
    if (fmt != SH_DSMEM) { *grid = (int)g->sms; return cudaSuccess; }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(2);
    cfg.blockDim = dim3(kCtThreads);
    cfg.dynamicSmemBytes = kShBytes;
    int clusters = 0;
    if ((ce = cudaOccupancyMaxActiveClusters(&clusters, kShKernels[SH_DSMEM], &cfg)) != cudaSuccess) {
        *where = "cudaOccupancyMaxActiveClusters(smem_selftest<SH_DSMEM>)";
        return ce;
    }
    if (clusters < 1) { *where = "smem_selftest<SH_DSMEM>: no cluster of two fits"; return cudaErrorInvalidConfiguration; }
    logf(0, "%s shared-memory test: %d clusters of two CTAs co-resident (%u SMs)", g->dev.id.c_str(), clusters, g->sms);
    *grid = 2 * clusters;
    return cudaSuccess;
}

static const DiagSuite kSmemSuite = {"shared-memory test", "smem_selftest", "word/byte/dsmem", kShKernels, kShSmem,
                                     kShTableBytes, sh_suite_tile, sh_suite_half_bytes, false, nullptr,
                                     "%.2f/%.2f/%.2f TB/s", sh_size_grid, true, "shared-memory self-test"};

// ---- the register-file test's suite ----
// __launch_bounds__(kCtThreads, 2) and kRfSmemBytes each: the default grid sizing gives two CTAs on every SM, which
// between them take the whole register file.
static const CtKernel kRfKernels[kRfFormats] = {rf_selftest<RF_ALU, false>, rf_selftest<RF_LOAD, false>,
                                                rf_selftest<RF_HOLD, false>};
static const uint32_t kRfSmem[kRfFormats] = {kRfSmemBytes, kRfSmemBytes, kRfSmemBytes};
static const uint32_t kRfTableBytes[kRfFormats] = {kRfTableWords * 4, kRfTableWords * 4, kRfTableWords * 4};
static void rf_suite_tile(uint32_t seed, int fmt, int tile, uint8_t* table, uint32_t* check) {
    rf_build_tile(seed, fmt, tile, reinterpret_cast<uint32_t*>(table), check);
}
// tflops[] = 2 x this x comparisons / ms: TB/s of register data the march reads and writes
static double rf_suite_half_bytes(int fmt) { return 0.5 * rf_bytes_per_tile(fmt); }

static const DiagSuite kRfSuite = {"register-file test", "rf_selftest", "alu/load/hold", kRfKernels, kRfSmem,
                                   kRfTableBytes, rf_suite_tile, rf_suite_half_bytes, false, nullptr,
                                   "%.2f/%.2f/%.2f TB/s", nullptr, true, "register-file self-test"};

// ---- the integer and warp-exchange test's suite ----
static const CtKernel kItKernels[kItFormats] = {int_selftest<IT_MAD, false>, int_selftest<IT_BIT, false>,
                                                int_selftest<IT_WARP, false>};
static const uint32_t kItSmem[kItFormats] = {0, 0, 0};
static const uint32_t kItTableBytes[kItFormats] = {it_table_bytes(IT_MAD), it_table_bytes(IT_BIT),
                                                   it_table_bytes(IT_WARP)};
static void it_suite_tile(uint32_t seed, int fmt, int tile, uint8_t* table, uint32_t* check) {
    it_build_tile(seed, fmt, tile, reinterpret_cast<uint32_t*>(table), check);
}
// tflops[] = 2 x this x comparisons / ms: T result words/s
static double it_suite_half_results(int fmt) { return 0.5 * it_ops_per_tile(fmt); }

static const DiagSuite kIntSuite = {"integer test", "int_selftest", "mad/bit/warp", kItKernels, kItSmem, kItTableBytes,
                                    it_suite_tile, it_suite_half_results, false, nullptr,
                                    "%.2f/%.2f/%.2f T results/s", nullptr, false, "integer self-test"};

// ---- the L2 test's suite ----
static const CtKernel kL2Kernels[kL2Formats] = {l2_selftest<L2_WORD, false>, l2_selftest<L2_BYTE, false>,
                                                l2_selftest<L2_ATOM, false>};
static const uint32_t kL2Smem[kL2Formats] = {0, 0, 0};
static const uint32_t kL2TableBytes[kL2Formats] = {l2_table_bytes(L2_WORD), l2_table_bytes(L2_BYTE),
                                                   l2_table_bytes(L2_ATOM)};
static void l2_suite_tile(uint32_t seed, int fmt, int tile, uint8_t* table, uint32_t* check) {
    l2_build_tile(seed, fmt, tile, reinterpret_cast<uint32_t*>(table), check);
}

// Every resident CTA, launched cooperatively: the grid barrier needs them all at once.
static cudaError_t l2_size_grid(Gpu* g, int fmt, int* grid, const char** where) {
    int dev = 0, coop = 0, per_sm = 0;
    cudaError_t ce = cudaGetDevice(&dev);
    if (ce == cudaSuccess) ce = cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev);
    if (ce != cudaSuccess) { *where = "cudaDeviceGetAttribute(cudaDevAttrCooperativeLaunch)"; return ce; }
    if (!coop) {
        *where = "l2_selftest: the device has no cooperative launch (cudaDevAttrCooperativeLaunch = 0), which the "
                 "grid barrier needs";
        return cudaErrorNotSupported;
    }
    if ((ce = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kL2Kernels[fmt], kCtThreads, 0)) != cudaSuccess) {
        *where = "cudaOccupancyMaxActiveBlocksPerMultiprocessor(l2_selftest)";
        return ce;
    }
    *grid = (int)g->sms * (per_sm > 0 ? per_sm : 1);
    if (*grid > kL2MaxCtas) { *where = "l2_selftest: more resident CTAs than its fold slots"; return cudaErrorInvalidConfiguration; }
    return cudaSuccess;
}

// WORD / BYTE: kL2Windows spans of 3/8 of the L2 each; ATOM: the hot block.  The rate's numerator depends on the span:
// *half is half of each CTA's share of one comparison's bytes (ATOM: ops x 1e3), as tflops[] = 2 x it x comparisons / ms.
static cudaError_t l2_scratch(Gpu* g, int fmt, int grid, size_t* bytes, uint32_t* header, double* half,
                              const char** where) {
    int dev = 0, l2 = 0;
    cudaError_t ce = cudaGetDevice(&dev);
    if (ce == cudaSuccess) ce = cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, dev);
    if (ce != cudaSuccess) { *where = "cudaDeviceGetAttribute(cudaDevAttrL2CacheSize)"; return ce; }
    size_t data = kL2AtomHotWords * 4ull;
    if (fmt != L2_ATOM) {
        const uint32_t K = l2_span_blocks(l2_default_span((unsigned long long)l2), grid);
        header[kL2HdrBlocks] = K;
        data = (size_t)kL2Windows * K * grid * kL2BlockBytes;
        // tflops[] = 2 x this x comparisons / ms, and every CTA counts each comparison: TB/s of L2 traffic
        *half = 0.5 * l2_bytes_per_comparison(fmt, (double)K * grid * kL2BlockBytes) / grid;
        logf(0, "%s L2 test: %d CTAs, span %.2f MiB of a %d KiB L2", g->dev.id.c_str(), grid,
             (double)K * grid * kL2BlockBytes / (1 << 20), l2 >> 10);
    } else {
        // G ops/s (x 1e3 against the T of the other two): 20 atomics per thread per comparison, a v4 op counts once
        *half = 0.5 * kCtThreads * 20 * 1e3;
    }
    *bytes = (size_t)kL2DataOff * 4 + data;
    return cudaSuccess;
}

// ---- the L1 test's suite ----
static const CtKernel kL1Kernels[kL1Formats] = {l1_selftest<L1_DATA, false>, l1_selftest<L1_TEX, false>,
                                                l1_selftest<L1_CONST, false>};
static const uint32_t kL1Smem[kL1Formats] = {0, 0, 0};
static const uint32_t kL1TableBytesAll[kL1Formats] = {l1_table_bytes(L1_DATA), l1_table_bytes(L1_TEX),
                                                      l1_table_bytes(L1_CONST)};
static const int kL1Carveout[kL1Formats] = {0, 0, 0};
static void l1_suite_tile(uint32_t seed, int fmt, int tile, uint8_t* table, uint32_t* check) {
    l1_build_tile(seed, fmt, tile, reinterpret_cast<uint32_t*>(table), check);
}

// Every resident CTA (no cooperative launch: no CTA waits for another).
static cudaError_t l1_size_grid(Gpu* g, int fmt, int* grid, const char** where) {
    int per_sm = 0;
    cudaError_t ce = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kL1Kernels[fmt], kCtThreads, 0);
    if (ce != cudaSuccess) { *where = "cudaOccupancyMaxActiveBlocksPerMultiprocessor(l1_selftest)"; return ce; }
    *grid = (int)g->sms * (per_sm > 0 ? per_sm : 1);
    return cudaSuccess;
}

// DATA: the header and every CTA's span of K blocks (kL1DefaultSpan per SM over the CTAs an SM holds); TEX: the header
// and the linear copy of the image; CONST: the header.  *half is half of one CTA's bytes of one comparison, as
// tflops[] = 2 x it x comparisons / ms: TB/s the loads deliver (DATA: and its stores).
static cudaError_t l1_scratch(Gpu* g, int fmt, int grid, size_t* bytes, uint32_t* header, double* half,
                              const char** where) {
    const int per_sm = grid / (int)(g->sms ? g->sms : 1);
    const uint32_t K = l1_span_blocks(kL1DefaultSpan, per_sm);
    size_t data = 0;
    if (fmt == L1_DATA) {
        header[kL1HdrBlocks] = K;
        data = (size_t)grid * K * kL1BlockWords;
        logf(0, "%s L1 test: %d CTAs, span %u KiB per CTA, %.0f KiB per SM", g->dev.id.c_str(), grid,
             K * kL1BlockBytes >> 10, (double)K * kL1BlockBytes * per_sm / 1024);
    } else if (fmt == L1_TEX) {
        data = (size_t)kL1Texels * 4;
    }
    *half = 0.5 * l1_bytes_per_comparison(fmt, K);
    *bytes = ((size_t)kL1DataOff + data) * 4;
    (void)where;
    return cudaSuccess;
}

// The constant bank is one per device in the process, shared by every b2dp_ctx, whose probe locks do not serialize each
// other: a bank lock per CUDA ordinal is held from bind to unbind, so no call reloads the bank under another's kernels.
static std::mutex& l1_bank_mutex(int ordinal) {
    static std::mutex guard;
    static std::map<int, std::mutex> per_device;  // map nodes never move: the references stay valid
    std::lock_guard<std::mutex> lk(guard);
    return per_device[ordinal];
}

struct L1SuiteState {
    std::unique_lock<std::mutex> bank;
    L1Bound bound;
};

// The CUDA array, the texture objects (handles into L1_TEX's scratch header) and the constant bank, from the call's seed.
// Refuses, before anything launches, an uploaded tile table whose indices leave their range (l1_selftest masks them all
// the same).
static cudaError_t l1_bind_suite(Gpu* g, uint32_t seed, const DiagTables& tabs, uint32_t* const* scratch, void** state,
                                 const char** where) {
    for (int f = 0; f < kL1Formats; ++f)
        for (int tile = 0; tile < kCtTiles; ++tile)
            if (tabs.tables[f].size() != (size_t)kCtTiles * l1_table_bytes(f) ||
                !l1_table_ok(f, reinterpret_cast<const uint32_t*>(tabs.tables[f].data()) + tile * kL1TableWords)) {
                *where = "l1_selftest: a tile table indexes outside its range";
                return cudaErrorInvalidValue;
            }
    L1SuiteState* st = new L1SuiteState;
    *state = st;
    st->bank = std::unique_lock<std::mutex>(l1_bank_mutex(g->ordinal));
    return l1_bind(seed, scratch[L1_TEX], g->stream, st->bound, where);
}
// Runs on the worker that ran bind, after the stream is synchronized: the bank is released last.
static void l1_unbind_suite(void* state) {
    L1SuiteState* st = static_cast<L1SuiteState*>(state);
    l1_unbind(st->bound);
    delete st;
}

static const DiagSuite kL1Suite = {"L1 test", "l1_selftest", "data/tex/const", kL1Kernels, kL1Smem, kL1TableBytesAll,
                                   l1_suite_tile, nullptr, false, nullptr, "%.2f/%.2f/%.2f TB/s", l1_size_grid, true,
                                   "L1 self-test", l1_scratch, false, kL1Carveout, l1_bind_suite, l1_unbind_suite};

// ---- the half-precision and conversion test's suite ----
static const CtKernel kHpKernels[kHpFormats] = {half_selftest<HP_F16, false>, half_selftest<HP_BF16, false>,
                                                half_selftest<HP_CVT, false>};
static const uint32_t kHpSmem[kHpFormats] = {0, 0, 0};
static const uint32_t kHpTableBytes[kHpFormats] = {hp_table_bytes(HP_F16), hp_table_bytes(HP_BF16),
                                                   hp_table_bytes(HP_CVT)};
static void hp_suite_tile(uint32_t seed, int fmt, int tile, uint8_t* table, uint32_t* check) {
    hp_build_tile(seed, fmt, tile, reinterpret_cast<uint32_t*>(table), check);
}
// tflops[] = 2 x this x comparisons / ms: T result words/s
static double hp_suite_half_results(int fmt) { return 0.5 * hp_ops_per_tile(fmt); }

static const DiagSuite kHalfSuite = {"half-precision test", "half_selftest", "f16/bf16/cvt", kHpKernels, kHpSmem,
                                     kHpTableBytes, hp_suite_tile, hp_suite_half_results, false, nullptr,
                                     "%.2f/%.2f/%.2f T results/s", nullptr, false, "half-precision self-test"};

// ---- the synchronization test's suite ----
static const CtKernel kSyKernels[kSyFormats] = {sync_selftest<SY_ATOM, false>, sync_selftest<SY_BAR, false>,
                                                sync_selftest<SY_WARP, false>};
static const uint32_t kSySmem[kSyFormats] = {0, 0, 0};
static const uint32_t kSyTableBytes[kSyFormats] = {sy_table_bytes(SY_ATOM), sy_table_bytes(SY_BAR),
                                                   sy_table_bytes(SY_WARP)};
static void sy_suite_tile(uint32_t seed, int fmt, int tile, uint8_t* table, uint32_t* check) {
    sy_build_tile(seed, fmt, tile, reinterpret_cast<uint32_t*>(table), check);
}

static const DiagSuite kSyncSuite = {"sync test", "sync_selftest", "atom/bar/warp", kSyKernels, kSySmem,
                                     kSyTableBytes, sy_suite_tile, sy_rate_half_units, false, nullptr,
                                     "%.2f/%.2f/%.2f G atomic ops/s, G barrier ops/s, T results/s", nullptr, false,
                                     "synchronization self-test"};

static const DiagSuite kL2Suite = {"L2 test", "l2_selftest", "word/byte/atom", kL2Kernels, kL2Smem, kL2TableBytes,
                                   l2_suite_tile, nullptr, false, nullptr, "%.2f/%.2f/%.2f TB/s, TB/s, G ops/s",
                                   l2_size_grid, true, "L2 self-test", l2_scratch, true};

static std::shared_ptr<DiagTables> diag_build_tables(const DiagSuite& su, uint32_t seed) {
    auto t = std::make_shared<DiagTables>();
    for (int f = 0; f < kCtFormats; ++f) {
        t->tables[f].resize((size_t)kCtTiles * su.table_bytes[f]);
        t->checks[f].resize((size_t)kCtTiles * kCtThreads);
        for (int tile = 0; tile < kCtTiles; ++tile)
            su.build_tile(seed, f, tile, t->tables[f].data() + (size_t)tile * su.table_bytes[f],
                          t->checks[f].data() + (size_t)tile * kCtThreads);
    }
    return t;
}

static void compute_test_one(const DiagSuite& su, CudaBackend* be, Gpu* g, const b2dp_compute_test_opts& o,
                             uint32_t duration_ms,
                             uint32_t timeout_ms, std::shared_ptr<const DiagTables> tabs, b2dp_compute_test_result* r,
                             std::string* err) {
    uint8_t* img[kCtFormats] = {};
    uint32_t* chk[kCtFormats] = {};
    uint32_t* scr[kCtFormats] = {};
    CtRecord* rec_h = nullptr;
    CtRecord* rec_d = nullptr;
    cudaEvent_t ev[kCtFormats + 1] = {};
    void* bound = nullptr;
    bool timed_out = false;
    cudaError_t ce = cudaSuccess;
    const char* where = "";
    auto release = [&] {  // every path ends here: nothing the test allocated outlives it
        if (g->stream) cudaStreamSynchronize(g->stream);
        if (bound) su.unbind(bound);
        for (int f = 0; f < kCtFormats; ++f) {
            if (img[f]) cudaFree(img[f]);
            if (chk[f]) cudaFree(chk[f]);
            if (scr[f]) cudaFree(scr[f]);
        }
        if (rec_h) cudaFreeHost(rec_h);
        for (cudaEvent_t e : ev)
            if (e) cudaEventDestroy(e);
    };
#define CT_TRY(x) if ((ce = (x)) != cudaSuccess) { where = #x; goto done; }
    {
        probe_flush(g);  // an armed heartbeat pass must not run underneath
        int grid[kCtFormats], off[kCtFormats + 1] = {0};
        double macs[kCtFormats] = {};  // per comparison: from macs_per_tile, or from scratch() once it is sized
        if (su.macs_per_tile)
            for (int f = 0; f < kCtFormats; ++f) macs[f] = su.macs_per_tile(f);
        for (int f = 0; f < kCtFormats; ++f) {
            CT_TRY(cudaFuncSetAttribute(su.kernels[f], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)su.smem[f]));
            CT_TRY(cudaFuncSetAttribute(su.kernels[f], cudaFuncAttributePreferredSharedMemoryCarveout,
                                        su.carveout ? su.carveout[f] : 100));
            if (su.size_grid) {
                if ((ce = su.size_grid(g, f, &grid[f], &where)) != cudaSuccess) goto done;
            } else {
                int per_sm = 0;
                CT_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, su.kernels[f], kCtThreads, su.smem[f]));
                grid[f] = (int)g->sms * (per_sm > 0 ? per_sm : 1);  // every CTA resident at once
            }
            off[f + 1] = off[f] + grid[f];
        }
        CT_TRY(cudaHostAlloc(&rec_h, (size_t)off[kCtFormats] * sizeof(CtRecord), cudaHostAllocMapped));
        memset(rec_h, 0, (size_t)off[kCtFormats] * sizeof(CtRecord));
        CT_TRY(cudaHostGetDevicePointer(&rec_d, rec_h, 0));
        if (!tabs) tabs = diag_build_tables(su, r->seed);
        DiagRef ref;
        std::chrono::steady_clock::duration ref_spent{0};  // counts against the same timeout_ms as the timed launches
        if (su.reference) {
            auto own = std::make_shared<DiagTables>();
            const auto t_ref = std::chrono::steady_clock::now();
            ce = su.reference(g, o, t_ref + std::chrono::milliseconds(timeout_ms), *tabs, *own, ref, r, &where,
                              &timed_out);
            ref_spent = std::chrono::steady_clock::now() - t_ref;
            if (ce != cudaSuccess || timed_out || !ref.run) goto done;  // Unhealthy; the timed launches do not run
            tabs = own;
        }
        for (int f = 0; f < kCtFormats; ++f) {
            const std::vector<uint8_t>& tables = tabs->tables[f];
            const std::vector<uint32_t>& checks = tabs->checks[f];
            CT_TRY(cudaMalloc(&img[f], tables.size()));
            CT_TRY(cudaMalloc(&chk[f], checks.size() * sizeof(uint32_t)));
            CT_TRY(cudaMemcpy(img[f], tables.data(), tables.size(), cudaMemcpyHostToDevice));
            CT_TRY(cudaMemcpy(chk[f], checks.data(), checks.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
            if (su.scratch) {
                size_t bytes = 0;
                uint32_t header[kDiagScratchHeaderWords] = {};
                if ((ce = su.scratch(g, f, grid[f], &bytes, header, &macs[f], &where)) != cudaSuccess) goto done;
                CT_TRY(cudaMalloc(&scr[f], bytes));
                CT_TRY(cudaMemset(scr[f], 0, bytes));
                CT_TRY(cudaMemcpy(scr[f], header, sizeof header, cudaMemcpyHostToDevice));
            }
        }
        if (su.bind && (ce = su.bind(g, r->seed, *tabs, scr, &bound, &where)) != cudaSuccess) goto done;
        for (cudaEvent_t& e : ev) CT_TRY(cudaEventCreate(&e));
        // Device-wide counters, as the memory test reads them: a single-bit defect ECC corrects never reaches the data
        // check, and only the corrected count shows it.
        unsigned long long corr0 = 0, unc0 = 0;
        const bool ecc = su.ecc && g->nvh && be->nvml.ecc_total && be->nvml.ecc_total(g->nvh, 1, 0, &unc0) == 0 &&
                         be->nvml.ecc_total(g->nvh, 0, 0, &corr0) == 0;
        if (su.ecc && !ecc) r->flags |= B2DP_CT_NO_ECC;

        CT_TRY(cudaEventRecord(ev[0], g->stream));
        for (int f = 0; f < kCtFormats; ++f) {
            if (su.cooperative) {
                const uint8_t* a_img = img[f];
                const uint32_t* a_chk = chk[f];
                unsigned long long a_ns = (unsigned long long)duration_ms * 1000000ull, a_seq = (unsigned long long)(f + 1);
                int a_sm = o.fault_sm;
                uint32_t a_mask = o.fault_mask;
                CtRecord* a_rec = rec_d + off[f];
                uint32_t* a_scr = scr[f];
                void* args[] = {&a_img, &a_chk, &a_ns, &a_sm, &a_mask, &a_rec, &a_seq, &a_scr};
                CT_TRY(cudaLaunchCooperativeKernel((const void*)su.kernels[f], dim3(grid[f]), dim3(kCtThreads), args,
                                                   su.smem[f], g->stream));
            } else {
                su.kernels[f]<<<grid[f], kCtThreads, su.smem[f], g->stream>>>(
                    img[f], chk[f], (unsigned long long)duration_ms * 1000000ull, o.fault_sm, o.fault_mask,
                    rec_d + off[f], (unsigned long long)(f + 1), scr[f]);
            }
            CT_TRY(cudaGetLastError());
            CT_TRY(cudaEventRecord(ev[f + 1], g->stream));
        }
        const auto deadline = std::chrono::steady_clock::now() + std::chrono::milliseconds(timeout_ms) - ref_spent;
        for (;;) {
            const cudaError_t q = cudaEventQuery(ev[kCtFormats]);
            if (q == cudaSuccess) break;
            if (q != cudaErrorNotReady) { ce = q; where = su.kernel_name; goto done; }
            if (std::chrono::steady_clock::now() > deadline) { timed_out = true; break; }
            std::this_thread::sleep_for(std::chrono::milliseconds(1));
        }
        // past the deadline the verdict is made, but the buffers can only be released once the kernels are done
        CT_TRY(cudaEventSynchronize(ev[kCtFormats]));
        std::atomic_thread_fence(std::memory_order_acquire);
        bool ecc_clean = true;
        if (ecc) {
            unsigned long long corr1 = corr0, unc1 = unc0;
            be->nvml.ecc_total(g->nvh, 1, 0, &unc1);
            be->nvml.ecc_total(g->nvh, 0, 0, &corr1);
            if (corr1 > corr0) r->flags |= B2DP_CT_ECC_CORRECTED;
            if (unc1 > unc0) { r->flags |= B2DP_CT_ECC; ecc_clean = false; }
            logf(unc1 > unc0 ? 2 : 0, "%s %s: ECC totals corrected +%llu, uncorrected +%llu", g->dev.id.c_str(),
                 su.log_name, corr1 - corr0, unc1 > unc0 ? unc1 - unc0 : 0ull);
        }

        std::vector<CtRecord> recs[kCtFormats];
        unsigned long long seq[kCtFormats];
        std::vector<uint8_t> seen[kCtFormats];
        for (int f = 0; f < kCtFormats; ++f) {
            CT_TRY(cudaEventElapsedTime(&r->ms[f], ev[f], ev[f + 1]));
            seq[f] = (unsigned long long)(f + 1);
            recs[f].resize(grid[f]);
            memcpy(recs[f].data(), (const void*)(rec_h + off[f]), (size_t)grid[f] * sizeof(CtRecord));
            seen[f].assign(kCtMaxSmId, 0);
            unsigned long long compared = 0;
            int bad_sm = -1, bad_tile = -1;
            for (const CtRecord& c : recs[f]) {
                if (c.seq != seq[f]) continue;  // never arrived: fails the verdict below
                r->nsmid = std::max<int32_t>(r->nsmid, (int32_t)c.nsmid);
                compared += c.comparisons;
                r->mismatches[f] += c.mismatches;
                if (c.smid >= (uint32_t)kCtMaxSmId) continue;
                seen[f][c.smid] = 1;
                if (c.mismatches) {
                    r->bad_sm_mask[c.smid / 64] |= 1ull << (c.smid % 64);
                    if (bad_sm < 0 || (int)c.smid < bad_sm) { bad_sm = (int)c.smid; bad_tile = c.first_bad_tile; }
                }
            }
            if (ref.bad_sm[f] >= 0 && (bad_sm < 0 || ref.bad_sm[f] < bad_sm)) {
                bad_sm = ref.bad_sm[f];
                bad_tile = ref.bad_tile[f];
            }
            if (bad_sm >= 0 && r->first_bad_format < 0) {
                r->first_bad_format = f;
                r->first_bad_sm = bad_sm;
                r->first_bad_tile = bad_tile;
            }
            if (r->ms[f] > 0) r->tflops[f] = (float)(2.0 * macs[f] * (double)compared / r->ms[f] * 1e-9);
        }
        for (int s = 0; s < kCtMaxSmId; ++s) r->sms_covered += seen[0][s] && seen[1][s] && seen[2][s];
        if (r->sms_covered < r->sm_count) r->flags |= B2DP_CT_PARTIAL_COVERAGE;
        r->healthy = compute_test_healthy(!timed_out, recs, seq) && ref.clean && ecc_clean ? 1 : 0;
    }
done:
#undef CT_TRY
    release();
    if (ce != cudaSuccess) {
        cudaGetLastError();
        r->err = B2DP_E_CUDA;
        r->healthy = 0;
        *err = cuda_err(where, ce) + " on " + g->dev.id;
    } else if (timed_out) {
        r->err = B2DP_E_TIMEOUT;
        r->healthy = 0;
    }
}

static int cuda_diag_test(const DiagSuite& su, CudaBackend* be, int device, const b2dp_compute_test_opts* opts,
                          std::vector<b2dp_compute_test_result>& out, std::string& err) {
    if (be->units) {
        err = std::string("the ") +
              (su.test_name         ? su.test_name
               : su.per_device_seed ? "compute self-test"
               : su.reference       ? "SFU self-test"
                                    : "FP self-test") +
              " runs in-process only (not with probe=helpers / probe=off / MIG)";
        return B2DP_E_UNSUPPORTED;
    }
    if (device < -1 || device >= (int)be->gpus.size()) { err = "device index out of range"; return B2DP_E_INVAL; }
    const b2dp_compute_test_opts o = opts ? *opts : b2dp_compute_test_opts{};
    const uint32_t duration_ms = o.duration_ms ? o.duration_ms : kComputeTestDefaultMs;
    const uint32_t timeout_ms = o.timeout_ms ? o.timeout_ms : 10000u + 6u * duration_ms;
    bool latched = false;
    {
        std::lock_guard<std::mutex> pl(be->probe_mu);  // a heartbeat waits for a running self-test
        const uint32_t seed = (uint32_t)std::chrono::steady_clock::now().time_since_epoch().count() * kPatternMul;
        // one seed for every GPU: the tables are built once, here, and shared by the workers
        std::shared_ptr<const DiagTables> shared = su.per_device_seed ? nullptr : diag_build_tables(su, seed);
        std::vector<size_t> sel;
        for (size_t i = 0; i < be->gpus.size(); ++i) if (device < 0 || (int)i == device) sel.push_back(i);
        out.assign(sel.size(), b2dp_compute_test_result{});
        std::vector<std::string> errs(sel.size());
        std::vector<std::shared_ptr<Completion>> cs(sel.size());
        for (size_t k = 0; k < sel.size(); ++k) {
            Gpu* g = be->gpus[sel[k]].get();
            b2dp_compute_test_result* r = &out[k];
            r->device = (int32_t)sel[k];
            r->seed = su.per_device_seed ? seed ^ ((uint32_t)sel[k] << 16) : seed;
            r->sm_count = (int32_t)g->sms;
            r->first_bad_sm = r->first_bad_format = r->first_bad_tile = -1;
            if (g->broken) { r->err = B2DP_E_CUDA; errs[k] = g->broken_reason + " on " + g->dev.id; continue; }
            if (!(o.flags & B2DP_CT_EVEN_IF_BUSY) && used_by_another_process(be, g)) {
                r->flags |= B2DP_CT_SKIPPED_BUSY;
                r->healthy = g->last_healthy;
                continue;
            }
            std::string* e = &errs[k];
            const DiagSuite* sp = &su;
            cs[k] = post(g, [sp, be, g, o, duration_ms, timeout_ms, shared, r, e] {
                compute_test_one(*sp, be, g, o, duration_ms, timeout_ms, shared, r, e);
            });
        }
        for (size_t k = 0; k < sel.size(); ++k) {
            if (cs[k]) cs[k]->wait();  // no deadline here: the buffers must be released before the call returns
            if (!errs[k].empty()) err = errs[k];
            if (!cs[k]) continue;       // skipped (busy) or never set up: nothing ran, nothing is latched
            Gpu* g = be->gpus[sel[k]].get();
            const b2dp_compute_test_result& r = out[k];
            if (!r.healthy) { g->compute_fault.store(true); latched = true; }
            char rate[96];
            snprintf(rate, sizeof rate, su.rate_format ? su.rate_format : "%.0f/%.0f/%.0f TFLOP/s", r.tflops[0],
                     r.tflops[1], r.tflops[2]);
            logf(r.healthy ? 0 : 2, "%s %s: %s, SMs %d/%d, mismatches %s %llu/%llu/%llu, first bad SM %d "
                 "format %d tile %d, %.1f/%.1f/%.1f ms, %s%s", g->dev.id.c_str(), su.log_name,
                 r.healthy ? "Healthy" : "Unhealthy (latched)", r.sms_covered, r.sm_count, su.format_names,
                 (unsigned long long)r.mismatches[0], (unsigned long long)r.mismatches[1],
                 (unsigned long long)r.mismatches[2], r.first_bad_sm, r.first_bad_format, r.first_bad_tile, r.ms[0],
                 r.ms[1], r.ms[2], rate, r.err == B2DP_E_TIMEOUT ? ", timed out" : "");
        }
    }
    // like the Xid latch: running ListAndWatch loops send a heartbeat now (no backend lock is held while they do)
    if (latched) be->fire_health_event();
    return B2DP_OK;
}

static int cuda_compute_test(CudaBackend* be, int device, const b2dp_compute_test_opts* opts,
                             std::vector<b2dp_compute_test_result>& out, std::string& err) {
    return cuda_diag_test(kTensorSuite, be, device, opts, out, err);
}

static int cuda_fp_test(CudaBackend* be, int device, const b2dp_compute_test_opts* opts,
                        std::vector<b2dp_compute_test_result>& out, std::string& err) {
    return cuda_diag_test(kFpSuite, be, device, opts, out, err);
}

static int cuda_sfu_test(CudaBackend* be, int device, const b2dp_compute_test_opts* opts,
                         std::vector<b2dp_compute_test_result>& out, std::string& err) {
    return cuda_diag_test(kSfuSuite, be, device, opts, out, err);
}

static int cuda_smem_test(CudaBackend* be, int device, const b2dp_compute_test_opts* opts,
                          std::vector<b2dp_compute_test_result>& out, std::string& err) {
    return cuda_diag_test(kSmemSuite, be, device, opts, out, err);
}

static int cuda_regfile_test(CudaBackend* be, int device, const b2dp_compute_test_opts* opts,
                             std::vector<b2dp_compute_test_result>& out, std::string& err) {
    return cuda_diag_test(kRfSuite, be, device, opts, out, err);
}

static int cuda_int_test(CudaBackend* be, int device, const b2dp_compute_test_opts* opts,
                         std::vector<b2dp_compute_test_result>& out, std::string& err) {
    return cuda_diag_test(kIntSuite, be, device, opts, out, err);
}

static int cuda_l2_test(CudaBackend* be, int device, const b2dp_compute_test_opts* opts,
                        std::vector<b2dp_compute_test_result>& out, std::string& err) {
    return cuda_diag_test(kL2Suite, be, device, opts, out, err);
}

static int cuda_half_test(CudaBackend* be, int device, const b2dp_compute_test_opts* opts,
                          std::vector<b2dp_compute_test_result>& out, std::string& err) {
    return cuda_diag_test(kHalfSuite, be, device, opts, out, err);
}

static int cuda_sync_test(CudaBackend* be, int device, const b2dp_compute_test_opts* opts,
                          std::vector<b2dp_compute_test_result>& out, std::string& err) {
    return cuda_diag_test(kSyncSuite, be, device, opts, out, err);
}

static int cuda_l1_test(CudaBackend* be, int device, const b2dp_compute_test_opts* opts,
                        std::vector<b2dp_compute_test_result>& out, std::string& err) {
    return cuda_diag_test(kL1Suite, be, device, opts, out, err);
}

// ---- on-demand host-link self-test (b2dp_hostlink_test) ---------------------------------------------------------------
// Host memory -> PCIe -> copy engines / SMs -> HBM and back, on the GPU's worker.  Two host buffers (Hs, the source the
// host writes, and Hd, the destination the host checks) are mmap'd, bound to the GPU's NUMA node before their first
// touch, touched, and registered as mapped pinned memory; two device buffers (A, B) of the same size take the copies.
// Per round, with the probe's seed schedule:
//   H2D, D2H: Hs <- pattern(s); A <- Hs (copy engine); hbm_probe_r128 verifies A and re-keys it into B; Hd <- B (copy
//             engine); the host checks Hd against pattern(next).  The two formats run this loop for duration_ms each
//             and differ in where the fault hook applies and which copy their rate times.
//   SM:       Hs <- pattern(s); hostlink_sm reads Hs and writes Hd over the mapped pointers; the host checks Hd.
// The link generation and width are sampled from NVML while a transfer is in flight (an idle link may train down).
// Everything is released before the job ends, whatever happened.
constexpr uint32_t kHostlinkDefaultMs = 1000;

// Bind [p, p + len) to NUMA node `node` with the raw mbind syscall (MPOL_BIND); false if the kernel refuses.
static bool hl_bind(void* p, size_t len, int node) {
    constexpr int kMaxNodes = 1024, kMpolBind = 2;
    constexpr int kBits = 8 * sizeof(unsigned long);
    if (node < 0 || node >= kMaxNodes) return false;
    unsigned long mask[kMaxNodes / kBits] = {};
    mask[node / kBits] = 1ul << (node % kBits);
    return syscall(SYS_mbind, p, len, kMpolBind, mask, (unsigned long)kMaxNodes + 1, 0u) == 0;
}

static void hostlink_one(CudaBackend* be, Gpu* g, const b2dp_hostlink_opts& o, unsigned long long bytes,
                         uint32_t duration_ms, uint32_t timeout_ms, b2dp_hostlink_result* r, std::string* err) {
    const size_t page = (size_t)sysconf(_SC_PAGESIZE);
    const size_t len = (bytes + page - 1) / page * page;
    const unsigned long long n_vec = bytes / 16, n_words = bytes / 4;
    void* host[2] = {};                  // Hs, Hd (mmap)
    bool registered[2] = {};
    uint4* hdev[2] = {};                 // their device-mapped pointers
    uint4* dbuf[2] = {};                 // A, B
    ProbeCtl* ctl = nullptr;
    ProbeOut* out_h = nullptr;
    ProbeOut* out_d = nullptr;
    HlRecord* rec_h = nullptr;
    HlRecord* rec_d = nullptr;
    cudaEvent_t ev[4] = {};
    bool timed_out = false;
    cudaError_t ce = cudaSuccess;
    const char* where = "";
    HlEvidence ev_;
    auto release = [&] {  // every path ends here: nothing the test allocated outlives it
        if (g->stream) cudaStreamSynchronize(g->stream);
        for (int k = 0; k < 2; ++k) {
            if (registered[k]) cudaHostUnregister(host[k]);
            if (host[k]) munmap(host[k], len);
            if (dbuf[k]) cudaFree(dbuf[k]);
        }
        if (ctl) cudaFree(ctl);
        if (out_h) cudaFreeHost(out_h);
        if (rec_h) cudaFreeHost(rec_h);
        for (cudaEvent_t e : ev)
            if (e) cudaEventDestroy(e);
    };
    // NVML: the link while a transfer is in flight (maximum over the samples), and the replay counter around the call
    unsigned replays0 = 0, v = 0;
    const bool nv = g->nvh != nullptr;
    const bool have_replays = nv && be->nvml.pcie_replays && be->nvml.pcie_replays(g->nvh, &replays0) == 0;
    if (nv && be->nvml.pcie_max_gen && be->nvml.pcie_max_gen(g->nvh, &v) == 0) r->max_link_gen = (int32_t)v;
    if (nv && be->nvml.pcie_max_width && be->nvml.pcie_max_width(g->nvh, &v) == 0) r->max_link_width = (int32_t)v;
    bool sampled = false;
    auto sample = [&] {
        unsigned gen = 0, width = 0;
        if (!nv || !be->nvml.pcie_gen || !be->nvml.pcie_width) return;
        if (be->nvml.pcie_gen(g->nvh, &gen) != 0 || be->nvml.pcie_width(g->nvh, &width) != 0) return;
        sampled = true;
        r->link_gen = std::max<int32_t>(r->link_gen, (int32_t)gen);
        r->link_width = std::max<int32_t>(r->link_width, (int32_t)width);
    };
    const auto t_start = std::chrono::steady_clock::now();
    const auto deadline = t_start + std::chrono::milliseconds(timeout_ms);
    // wait for `e`, sampling the link meanwhile; false on a CUDA error (ce, where) or past the deadline (timed_out)
    auto wait = [&](cudaEvent_t e, const char* what) {
        for (;;) {
            const cudaError_t q = cudaEventQuery(e);
            if (q == cudaSuccess) return true;
            if (q != cudaErrorNotReady) { ce = q; where = what; return false; }
            sample();
            if (std::chrono::steady_clock::now() > deadline) { timed_out = true; return false; }
            std::this_thread::sleep_for(std::chrono::microseconds(100));
        }
    };
    const bool inject = o.fault_mask != 0 && o.fault_word < n_words;
    if (o.fault_mask && !inject) r->err = B2DP_E_INVAL;  // not injected; the test runs as it would without the hook
#define HL_TRY(x) if ((ce = (x)) != cudaSuccess) { where = #x; goto done; }
    {
        probe_flush(g);  // an armed heartbeat pass must not run underneath
        r->host_numa_node = g->dev.numa;
        for (int k = 0; k < 2; ++k) {
            void* p = mmap(nullptr, len, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
            if (p == MAP_FAILED) { ce = cudaErrorMemoryAllocation; where = "mmap (host buffer)"; goto done; }
            host[k] = p;
            if (!hl_bind(p, len, g->dev.numa)) r->host_numa_node = -1;  // before the first touch places the pages
            memset(p, 0, len);
            HL_TRY(cudaHostRegister(p, len, cudaHostRegisterMapped));
            registered[k] = true;
            HL_TRY(cudaHostGetDevicePointer((void**)&hdev[k], p, 0));
            HL_TRY(cudaMalloc(&dbuf[k], bytes));
        }
        if (r->host_numa_node < 0) r->flags |= B2DP_HL_NUMA_UNBOUND;
        HL_TRY(cudaMalloc(&ctl, sizeof(ProbeCtl)));
        {
            ProbeCtl init = {};
            init.first_bad = ~0ull;
            init.t_start_ns = ~0ull;
            HL_TRY(cudaMemcpy(ctl, &init, sizeof init, cudaMemcpyHostToDevice));
        }
        HL_TRY(cudaHostAlloc(&out_h, sizeof(ProbeOut), cudaHostAllocMapped));
        memset(out_h, 0, sizeof(ProbeOut));
        HL_TRY(cudaHostGetDevicePointer(&out_d, out_h, 0));
        int per_sm = 0;
        HL_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, hostlink_sm<kHlThreads, kHlUnroll>, kHlThreads, 0));
        const int grid = (int)g->sms * (per_sm > 0 ? per_sm : 1);  // every CTA resident at once: every SM runs one
        HL_TRY(cudaHostAlloc(&rec_h, (size_t)grid * sizeof(HlRecord), cudaHostAllocMapped));
        memset(rec_h, 0, (size_t)grid * sizeof(HlRecord));
        HL_TRY(cudaHostGetDevicePointer(&rec_d, rec_h, 0));
        for (cudaEvent_t& e : ev) HL_TRY(cudaEventCreate(&e));

        const std::array<unsigned long long, 32>& bc = host_bitcounts(be, n_words);
        uint32_t* hs = static_cast<uint32_t*>(host[0]);
        const uint32_t* hd = static_cast<const uint32_t*>(host[1]);
        std::vector<uint8_t> seen(kCtMaxSmId, 0);
        uint32_t s = r->seed;
        unsigned long long seq = 0;
        for (int f = 0; f < kHlFormats; ++f) {
            const auto t_fmt = std::chrono::steady_clock::now();
            double ms_sum = 0.0;
            r->first_bad_word[f] = ~0ull;
            for (unsigned long long k = 0;; ++k) {
                if (k > 0 && std::chrono::steady_clock::now() - t_fmt >= std::chrono::milliseconds(duration_ms)) break;
                if (std::chrono::steady_clock::now() > deadline) { timed_out = true; goto done; }
                const uint32_t next = hl_next_seed(s);
                const bool poke = inject && k == 0;
                hl_fill(hs, n_words, s);
                ++seq;
                float ms = 0.f;
                if (f != B2DP_HL_SM) {
                    HL_TRY(cudaEventRecord(ev[0], g->stream));
                    HL_TRY(cudaMemcpyAsync(dbuf[0], hs, bytes, cudaMemcpyHostToDevice, g->stream));
                    HL_TRY(cudaEventRecord(ev[1], g->stream));
                    if (poke && f == B2DP_HL_H2D)
                        hbm_poke<<<1, 1, 0, g->stream>>>(reinterpret_cast<uint32_t*>(dbuf[0]), o.fault_word, o.fault_mask);
                    hbm_probe_r128<kRegThreads, kRegUnroll><<<(int)g->sms * kRegCtasPerSm, kRegThreads, 0, g->stream>>>(
                        dbuf[0], dbuf[1], n_vec, s, s ^ next, ctl, out_d, seq);
                    if (poke && f == B2DP_HL_D2H)
                        hbm_poke<<<1, 1, 0, g->stream>>>(reinterpret_cast<uint32_t*>(dbuf[1]), o.fault_word, o.fault_mask);
                    HL_TRY(cudaGetLastError());
                    HL_TRY(cudaEventRecord(ev[2], g->stream));
                    HL_TRY(cudaMemcpyAsync(host[1], dbuf[1], bytes, cudaMemcpyDeviceToHost, g->stream));
                    HL_TRY(cudaEventRecord(ev[3], g->stream));
                    if (!wait(ev[3], "host-link copies")) goto done;
                    HL_TRY(cudaEventElapsedTime(&ms, f == B2DP_HL_H2D ? ev[0] : ev[2], f == B2DP_HL_H2D ? ev[1] : ev[3]));
                } else {
                    HL_TRY(cudaEventRecord(ev[0], g->stream));
                    hostlink_sm<kHlThreads, kHlUnroll><<<grid, kHlThreads, 0, g->stream>>>(
                        hdev[0], hdev[1], n_vec, s, s ^ next, poke ? o.fault_word : 0ull, poke ? o.fault_mask : 0u, ctl,
                        out_d, seq, rec_d);
                    HL_TRY(cudaGetLastError());
                    HL_TRY(cudaEventRecord(ev[1], g->stream));
                    if (!wait(ev[1], "hostlink_sm")) goto done;
                    HL_TRY(cudaEventElapsedTime(&ms, ev[0], ev[1]));
                }
                ms_sum += ms;
                std::atomic_thread_fence(std::memory_order_acquire);
                ProbeOut po;
                memcpy(&po, (const void*)out_h, sizeof po);  // published by the kernel's last CTA; the stream is done
                if (po.seq != seq) ev_.seq_ok = false;
                if (po.checksum != expected_checksum_from_counts(bc, n_words, s)) ev_.checksums_ok = false;
                unsigned long long first = po.mismatches ? po.first_bad : ~0ull;
                unsigned long long bad = po.mismatches + hl_check(hd, n_words, next, &first);
                if (f == B2DP_HL_SM) {
                    for (int c = 0; c < grid; ++c) {
                        const HlRecord& rc = rec_h[c];
                        if (rc.seq != seq) { ev_.seq_ok = false; continue; }
                        if (rc.smid >= (uint32_t)kCtMaxSmId) continue;
                        seen[rc.smid] = 1;
                        if (rc.mismatches) r->bad_sm_mask[rc.smid / 64] |= 1ull << (rc.smid % 64);
                    }
                }
                r->mismatches[f] += bad;
                r->first_bad_word[f] = std::min<uint64_t>(r->first_bad_word[f], first);
                ++r->rounds[f];
                s = next;
            }
            r->ms[f] = (float)ms_sum;
            const double moved = (f == B2DP_HL_SM ? 2.0 : 1.0) * (double)bytes * (double)r->rounds[f];
            if (ms_sum > 0) r->gbs[f] = (float)(moved / ms_sum * 1e-6);
        }
        for (int sm = 0; sm < kCtMaxSmId; ++sm) r->sms_covered += seen[sm];
    }
done:
#undef HL_TRY
    release();
    unsigned replays1 = replays0;
    if (have_replays && be->nvml.pcie_replays(g->nvh, &replays1) == 0 && replays1 > replays0)
        r->replays = replays1 - replays0;
    if (!sampled || !have_replays) r->flags |= B2DP_HL_NO_NVML;
    if (r->replays) r->flags |= B2DP_HL_REPLAYS;
    if (r->link_width > 0 && r->max_link_width > 0 && r->link_width < r->max_link_width) r->flags |= B2DP_HL_LINK_NARROW;
    if (r->link_gen > 0 && r->max_link_gen > 0 && r->link_gen < r->max_link_gen) r->flags |= B2DP_HL_LINK_SLOW;
    r->link_gbs = (float)hl_link_gbs(r->link_gen, r->link_width);
    if (ce != cudaSuccess) {
        cudaGetLastError();
        r->err = B2DP_E_CUDA;
        r->healthy = 0;
        *err = cuda_err(where, ce) + " on " + g->dev.id;
    } else if (timed_out) {
        r->err = B2DP_E_TIMEOUT;
        r->healthy = 0;
    } else {
        for (int f = 0; f < kHlFormats; ++f) {
            ev_.rounds[f] = r->rounds[f];
            ev_.mismatches[f] = r->mismatches[f];
        }
        r->healthy = hl_healthy(ev_) ? 1 : 0;
    }
}

static int cuda_hostlink_test(CudaBackend* be, int device, const b2dp_hostlink_opts* opts,
                              std::vector<b2dp_hostlink_result>& out, std::string& err) {
    if (be->units) {
        err = "the host-link self-test runs in-process only (not with probe=helpers / probe=off / MIG)";
        return B2DP_E_UNSUPPORTED;
    }
    if (device < -1 || device >= (int)be->gpus.size()) { err = "device index out of range"; return B2DP_E_INVAL; }
    const b2dp_hostlink_opts o = opts ? *opts : b2dp_hostlink_opts{};
    const unsigned long long bytes = hl_buffer_bytes(o.bytes);
    if (!bytes) { err = "bytes must be a multiple of 16 and at most 1 GiB"; return B2DP_E_INVAL; }
    const uint32_t duration_ms = o.duration_ms ? o.duration_ms : kHostlinkDefaultMs;
    const uint32_t timeout_ms = o.timeout_ms ? o.timeout_ms : 10000u + 3u * duration_ms;
    bool latched = false;
    {
        std::lock_guard<std::mutex> pl(be->probe_mu);  // a heartbeat waits for a running self-test
        const uint32_t seed = (uint32_t)std::chrono::steady_clock::now().time_since_epoch().count() * kPatternMul;
        std::vector<size_t> sel;
        for (size_t i = 0; i < be->gpus.size(); ++i) if (device < 0 || (int)i == device) sel.push_back(i);
        out.assign(sel.size(), b2dp_hostlink_result{});
        std::vector<std::string> errs(sel.size());
        std::vector<std::shared_ptr<Completion>> cs(sel.size());
        for (size_t k = 0; k < sel.size(); ++k) {
            Gpu* g = be->gpus[sel[k]].get();
            b2dp_hostlink_result* r = &out[k];
            r->device = (int32_t)sel[k];
            r->seed = seed ^ ((uint32_t)sel[k] << 16);
            r->sm_count = (int32_t)g->sms;
            r->host_numa_node = -1;
            for (auto& w : r->first_bad_word) w = ~0ull;
            if (g->broken) { r->err = B2DP_E_CUDA; errs[k] = g->broken_reason + " on " + g->dev.id; continue; }
            if (!(o.flags & B2DP_HL_EVEN_IF_BUSY) && used_by_another_process(be, g)) {
                r->flags |= B2DP_HL_SKIPPED_BUSY;
                r->healthy = g->last_healthy;
                continue;
            }
            std::string* e = &errs[k];
            cs[k] = post(g, [be, g, o, bytes, duration_ms, timeout_ms, r, e] {
                hostlink_one(be, g, o, bytes, duration_ms, timeout_ms, r, e);
            });
        }
        for (size_t k = 0; k < sel.size(); ++k) {
            if (cs[k]) cs[k]->wait();  // no deadline here: the buffers must be released before the call returns
            if (!errs[k].empty()) err = errs[k];
            if (!cs[k]) continue;       // skipped (busy) or never set up: nothing ran, nothing is latched
            Gpu* g = be->gpus[sel[k]].get();
            const b2dp_hostlink_result& r = out[k];
            if (!r.healthy) { g->hostlink_fault.store(true); latched = true; }
            logf(r.healthy ? 0 : 2, "%s host-link test: %s, %llu MiB buffers on NUMA node %d, rounds %llu/%llu/%llu, "
                 "mismatches h2d/d2h/sm %llu/%llu/%llu, %.2f/%.2f/%.2f GB/s, SMs %d/%d, PCIe gen %d/%d x%d/%d "
                 "(%.1f GB/s), replays %llu, flags 0x%x%s", g->dev.id.c_str(),
                 r.healthy ? "Healthy" : "Unhealthy (latched)", bytes >> 20, r.host_numa_node,
                 (unsigned long long)r.rounds[0], (unsigned long long)r.rounds[1], (unsigned long long)r.rounds[2],
                 (unsigned long long)r.mismatches[0], (unsigned long long)r.mismatches[1],
                 (unsigned long long)r.mismatches[2], r.gbs[0], r.gbs[1], r.gbs[2], r.sms_covered, r.sm_count,
                 r.link_gen, r.max_link_gen, r.link_width, r.max_link_width, r.link_gbs,
                 (unsigned long long)r.replays, r.flags, r.err == B2DP_E_TIMEOUT ? ", timed out" : "");
        }
    }
    // like the Xid latch: running ListAndWatch loops send a heartbeat now (no backend lock is held while they do)
    if (latched) be->fire_health_event();
    return B2DP_OK;
}

static bool cuda_diag_latched(CudaBackend* be) {
    for (auto& g : be->gpus)
        if (g->memtest_fault.load() || g->compute_fault.load() || g->hostlink_fault.load()) return true;
    return false;
}

// registered when the library is loaded, before any entry point can run (internal.hpp DiagHooks)
[[maybe_unused]] static const bool kDiagRegistered = [] {
    diag_hooks() = DiagHooks{cuda_memtest, cuda_compute_test, cuda_fp_test, cuda_diag_latched, cuda_sfu_test,
                             cuda_smem_test, cuda_regfile_test, cuda_int_test, cuda_l2_test, cuda_hostlink_test,
                             cuda_half_test, cuda_sync_test, cuda_l1_test};
    return true;
}();

// ---- P2P matrix ------------------------------------------------------------------------------
constexpr float kNvlinkRefGbs = 450.f, kNvlinkClassFraction = 0.25f;  // oracle/probe.py

int cuda_p2p_matrix(CudaBackend* be, const b2dp_p2p_opts* opts, float* gbs, int32_t* link_type, uint64_t* mism, int n,
                    std::string& err) {
    std::lock_guard<std::mutex> pl(be->probe_mu);
    if (be->units) {
        // no CUDA context here and no P2P between MIG instances: the link classes are DECLARED from NVML (gbs = 0)
        if (n != (int)be->units->units.size()) { err = "n must equal the device count"; return B2DP_E_INVAL; }
        for (int i = 0; i < n; ++i)
            for (int j = 0; j < n; ++j) {
                gbs[(size_t)i * n + j] = 0; mism[(size_t)i * n + j] = 0;
                link_type[(size_t)i * n + j] = i == j ? 0 : units_link_type(be->nvml, be->units->units[i], be->units->units[j]);
            }
        return B2DP_OK;
    }
    if (n != (int)be->gpus.size()) { err = "n must equal the device count"; return B2DP_E_INVAL; }
    unsigned long long bytes = opts && opts->bytes ? opts->bytes : be->cfg.p2p_bytes;
    for (auto& g : be->gpus) if (!g->broken) bytes = std::min<unsigned long long>(bytes, g->n_vec * 16);  // the smallest ring slot bounds a pass
    bytes &= ~15ull;
    const unsigned long long n_vec = bytes / 16;
    const int iters = opts && opts->iters ? (int)opts->iters : 2;
    for (int i = 0; i < n * n; ++i) { gbs[i] = 0; link_type[i] = 0; mism[i] = 0; }
    // a probe pass that missed its deadline still owns its GPU's seed/ring state: let the workers drain; an armed
    // pass (prearm=1) is discarded, the matrix uses every stream and the spare buffers
    for (auto& g : be->gpus)
        if (!g->broken && g->th.joinable()) { Gpu* gp = g.get(); run_sync(gp, [gp] { probe_flush(gp); }); }
    const std::array<unsigned long long, 32>& bc = host_bitcounts(be, n_vec * 4);  // host closed form

    // peer capability + enable (on the reader's worker)
    std::vector<char> can((size_t)n * n, 0);
    for (int i = 0; i < n; ++i)
        for (int j = 0; j < n; ++j) {
            if (i == j) continue;
            int c = 0;
            if (be->gpus[i]->broken || be->gpus[j]->broken) continue;
            cudaDeviceCanAccessPeer(&c, be->gpus[i]->ordinal, be->gpus[j]->ordinal);
            can[(size_t)i * n + j] = (char)c;
            if (c && !be->gpus[i]->peer_enabled[j]) {
                Gpu* g = be->gpus[i].get();
                const int peer = be->gpus[j]->ordinal;
                cudaError_t ce = cudaSuccess;
                run_sync(g, [&] {
                    ce = cudaDeviceEnablePeerAccess(peer, 0);
                    if (ce == cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); ce = cudaSuccess; }
                });
                if (ce != cudaSuccess) can[(size_t)i * n + j] = 0;
                else g->peer_enabled[j] = 1;
            }
        }

    struct PairRes { cudaError_t ce = cudaSuccess; float best_ms = 1e30f; ProbeOut out{}; bool ran = false; };
    auto run_pair = [&](int i, int j, PairRes* pr) {
        // GPU i reads GPU j's current pattern buffer into its own spare buffer
        Gpu* g = be->gpus[i].get();
        Gpu* peer = be->gpus[j].get();
        const uint4* src = peer->buf[peer->cur];
        const uint32_t seed = peer->seed;
        return post(g, [g, src, seed, n_vec, iters, pr] {
            pr->ran = true;
            for (int it = 0; it < iters + 1; ++it) {  // first iteration is a warm-up
                const unsigned long long seq = ++g->seq;
                cudaEventRecord(g->e0, g->stream);
                // the former health-probe kernel (smem-staged, tile t -> CTA t mod grid) with a peer-mapped
                // source: the bulk copies cross NVLink, verification happens on the receiving GPU
                hbm_probe_tma<kTmaCW, kTmaTileVec, kTmaStages>
                    <<<(int)g->sms * kTmaCtasPerSm, (kTmaCW + 1) * 32, kTmaSmem, g->stream>>>(
                        src, g->buf[g->next()], n_vec, seed, 0u, g->ctl, g->out_d, seq);
                cudaError_t e = cudaGetLastError();
                cudaEventRecord(g->e1, g->stream);
                if (e == cudaSuccess) e = cudaEventSynchronize(g->e1);
                float ms = 0;
                if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, g->e0, g->e1);
                if (e != cudaSuccess) { pr->ce = e; return; }
                memcpy(&pr->out, (const void*)g->out_h, sizeof(ProbeOut));
                if (it > 0 && ms < pr->best_ms) pr->best_ms = ms;
            }
        });
    };

    // N-1 rounds of disjoint matchings (circle method).  Default: one direction of every pair per
    // half-round (a pull's read requests travel against the other direction's data, so both
    // directions at once measure less per direction than the link carries one way -- tools/p2p_sweep);
    // B2DP_P2P_BIDIR runs both directions together (full-duplex stress).
    const bool bidir = opts && (opts->flags & B2DP_P2P_BIDIR);
    const int m = n % 2 ? n + 1 : n;
    for (int hr = 0; hr < 2 * (m - 1) && n > 1; ++hr) {
        const int r = hr / 2, half = hr % 2;
        if (bidir && half) continue;
        std::vector<std::pair<int, int>> pairs;
        auto add = [&](int a, int b) { if (a < n && b < n) pairs.push_back({a, b}); };  // >= n: bye
        add(m - 1, r);
        for (int k = 1; k < m / 2; ++k) add((r + k) % (m - 1), (r - k + (m - 1)) % (m - 1));
        std::vector<std::unique_ptr<PairRes>> prs;
        std::vector<std::shared_ptr<Completion>> cs;
        std::vector<std::pair<int, int>> dirs;
        for (auto& p : pairs)
            for (int d = 0; d < 2; ++d) {
                if (!bidir && d != half) continue;
                const int i = d ? p.second : p.first, j = d ? p.first : p.second;
                if (!can[(size_t)i * n + j]) continue;
                prs.push_back(std::make_unique<PairRes>());
                dirs.push_back({i, j});
                cs.push_back(run_pair(i, j, prs.back().get()));
            }
        for (auto& c : cs) c->wait();
        for (size_t k = 0; k < dirs.size(); ++k) {
            const int i = dirs[k].first, j = dirs[k].second;
            const PairRes& pr = *prs[k];
            if (pr.ce != cudaSuccess) { err = cuda_err("p2p_probe", pr.ce); return B2DP_E_CUDA; }
            const float g_ = (float)((double)bytes / (double)pr.best_ms * 1e-6);
            gbs[(size_t)i * n + j] = g_;
            uint64_t bad = pr.out.mismatches;
            if (pr.out.checksum != expected_checksum_from_counts(bc, n_vec * 4, be->gpus[j]->seed)) bad = bad ? bad : 1;
            mism[(size_t)i * n + j] = bad;
        }
    }
    for (int i = 0; i < n; ++i)
        for (int j = 0; j < n; ++j) {
            if (i == j) continue;
            // oracle/probe.py classify_link
            link_type[(size_t)i * n + j] = !can[(size_t)i * n + j] ? 0
                : gbs[(size_t)i * n + j] >= kNvlinkClassFraction * kNvlinkRefGbs ? 11 : 2;
        }
    return B2DP_OK;
}

}  // namespace b2dp
