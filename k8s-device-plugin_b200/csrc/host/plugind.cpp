// b200dp_plugind -- the device-plugin daemon as ONE native binary over libb200dp.so: the flags and resource list
// of cmd/k8s-device-plugin/main.go:93-155, one v1beta1.DevicePlugin gRPC server per resource on
// <plugin_dir>/<namespace>_<name>, registration with the kubelet, the `-pulse` heartbeat ticker, and dpm's
// lifecycle (vendor/github.com/kubevirt/device-plugin-manager/pkg/dpm): plugin start retried 3 times 3 s apart
// (manager.go:16-20,205-219), re-serve + re-register when kubelet.sock is created and stop serving when it is removed
// (manager.go:73-84: inotify on the plugin directory, dpm's fsnotify watcher; a once-a-second stat of the socket stays
// as the fallback where inotify is unavailable), clean stop on SIGINT/SIGQUIT/SIGTERM (manager.go:47-48,85-91).
// gRPC comes from host/h2grpc.hpp; every RPC body is one C-ABI call (include/b200dp.h).
//
//   b200dp_plugind -pulse=10 -resource_naming_strategy=single -backend=cuda:xid=1 [-plugin_dir DIR]
//   kill -USR1 <pid>     one heartbeat now
//
// Node-labeller mode (cmd/k8s-node-labeller/main.go:383-479 without the controller-runtime client), so the labeller
// DaemonSet needs no Python:
//   b200dp_plugind -labels=vram,cu-count,product-name [-backend=cuda:]       the label map as JSON
//   b200dp_plugind -labels=all -reconcile < node-labels.json                 controller.go:23-58 on that map
//   b200dp_plugind -labels=all -patch < node-labels.json                     the JSON merge patch for `kubectl patch node`
#include <signal.h>
#include <sys/inotify.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <iostream>
#include <iterator>
#include <map>
#include <string>
#include <vector>

#include "../../../include/b200dp.h"
#include "../pbwire.hpp"
#include "h2grpc.hpp"
#include "pbread.hpp"

namespace {

std::atomic<bool> g_stop{false};

// The SM self-tests' -<flag>=1 (2: also on GPUs another process is using): each runs on every GPU once, after open and
// before the first registration, for -compute_test_ms per format, in this order after the memtest; the host-link test
// runs between the L2 and half-precision tests (kSmTestsBeforeHostlink).  A failed device stays latched Unhealthy,
// reported like a failed memtest.
struct SmTest {
    const char* flag;
    const char* log;   // the log lines' prefix
    const char* rate;  // their tflops[] columns
    int (*run)(b2dp_ctx*, int, const b2dp_compute_test_opts*, b2dp_compute_test_result*, int, int*);
};
const SmTest kSmTests[] = {
    {"compute_test_at_start", "compute test", "%.0f/%.0f/%.0f TFLOP/s", b2dp_compute_test},  // tensor cores
    {"fp_test_at_start", "fp test", "%.1f/%.1f/%.1f TFLOP/s", b2dp_fp_test},                  // FFMA, DFMA, DMMA
    // MUFU transcendentals, checked against the SMs' majority and host error bounds
    {"sfu_test_at_start", "sfu test", "%.2f/%.2f/%.2f T results/s", b2dp_sfu_test},
    // every SM's 227 KiB array and the SM-to-SM DSMEM path, marched against host patterns
    {"smem_test_at_start", "smem test", "%.2f/%.2f/%.2f TB/s", b2dp_smem_test},
    // 204 values per thread held in every SM's registers and marched against host patterns
    {"regfile_test_at_start", "regfile test", "%.2f/%.2f/%.2f TB/s", b2dp_regfile_test},
    // every SM's integer pipes and shuffle network against exact host results
    {"int_test_at_start", "int test", "%.2f/%.2f/%.2f T results/s", b2dp_int_test},
    // a march over an L2-resident span that moves between SMs, and the L2 atomic units, against host values
    {"l2_test_at_start", "L2 test", "%.2f/%.2f/%.2f TB/s, TB/s, G ops/s", b2dp_l2_test},
    // every SM's f16x2 / bf16x2 pipes and type converters against exact host results
    {"half_test_at_start", "half test", "%.2f/%.2f/%.2f T results/s", b2dp_half_test},
    // shared-memory atomics, barriers, mbarriers and warp collectives against the PTX ISA
    {"sync_test_at_start", "sync test", "%.2f/%.2f/%.2f G ops/s, G ops/s, T results/s", b2dp_sync_test},
    // the L1 data cache, the texture and read-only paths and the constant cache against host-built data
    {"l1_test_at_start", "L1 test", "%.2f/%.2f/%.2f TB/s", b2dp_l1_test},
};
constexpr size_t kNumSmTests = sizeof kSmTests / sizeof kSmTests[0];
constexpr size_t kSmTestsBeforeHostlink = 7;  // compute ... L2

struct Flags {
    int pulse = 0;                                   // main.go:109
    std::string strategy = "single";                 // main.go:110
    std::string backend = "cuda:";
    std::string plugin_dir = "/var/lib/kubelet/device-plugins/";  // pluginapi.DevicePluginPath, constants.go:26
    std::string ns = "amd.com";                      // plugin.go:406-408
    double start_retry_wait = 3.0;                   // dpm/manager.go:19
    int link_check = 0;
    std::string exporter_socket;                     // optional: serve metricssvc.MetricsService here (health.go:36)
    int memtest_at_start = 0;                        // 1: test the free HBM of every idle GPU before the first registration;
                                                     // 2: also GPUs another process is using
    unsigned long long memtest_max_bytes = 0;        // cap per GPU for that test (0 = all free memory above the reserve)
    unsigned compute_test_ms = 0;                    // the SM and host-link self-tests' duration per format (0 = 1000 ms)
    int sm_test_at_start[kNumSmTests] = {};          // per kSmTests row: its -<flag> level
    int hostlink_test_at_start = 0;                  // likewise for the host-link self-test (after the L2 test)
    bool version = false;
    bool labels_mode = false, reconcile = false, patch = false;
    std::string labels;                              // csv of generator names, or "all"
};

// Go's flag package: -name=value, -name value, --name...; bools not needed here
bool parse_flags(int argc, char** argv, Flags& f, std::string& err) {
    for (int i = 1; i < argc; ++i) {
        std::string a = argv[i];
        if (a.rfind("--", 0) == 0) a = a.substr(1);
        if (a == "-version") { f.version = true; continue; }
        if (a == "-labels") { f.labels_mode = true; f.labels = "all"; continue; }
        if (a == "-reconcile") { f.reconcile = true; continue; }
        if (a == "-patch") { f.patch = true; continue; }
        if (a.empty() || a[0] != '-') { err = "unexpected argument " + a; return false; }
        std::string name = a.substr(1), val;
        const size_t eq = name.find('=');
        const std::string bare = eq == std::string::npos ? name : name.substr(0, eq);
        // glog's flags (the reference's image runs `-logtostderr=true -stderrthreshold=INFO -v=5`, Dockerfile:33) are
        // accepted and ignored so existing DaemonSet args keep working; this daemon always logs to stderr
        const bool glog_bool = bare == "logtostderr" || bare == "alsologtostderr";
        const bool glog_val = bare == "stderrthreshold" || bare == "v" || bare == "log_dir" || bare == "vmodule" || bare == "log_backtrace_at";
        if (eq != std::string::npos) { val = name.substr(eq + 1); name = bare; }
        else if (glog_bool) val = "true";  // Go bool flags take no separate argument
        else if (i + 1 < argc) val = argv[++i];
        else { err = "flag needs an argument: -" + name; return false; }
        if (glog_bool || glog_val) continue;
        if (name == "pulse") f.pulse = atoi(val.c_str());
        else if (name == "resource_naming_strategy") f.strategy = val;
        else if (name == "backend") f.backend = val;
        else if (name == "plugin_dir") f.plugin_dir = val;
        else if (name == "resource_namespace") f.ns = val;
        else if (name == "start_retry_wait") f.start_retry_wait = atof(val.c_str());
        else if (name == "link_check") f.link_check = atoi(val.c_str());
        else if (name == "exporter_socket") f.exporter_socket = val;
        else if (name == "memtest_at_start") f.memtest_at_start = atoi(val.c_str());
        else if (name == "memtest_max_bytes") f.memtest_max_bytes = strtoull(val.c_str(), nullptr, 0);
        else if (name == "compute_test_ms") f.compute_test_ms = (unsigned)strtoul(val.c_str(), nullptr, 0);
        else if (name == "hostlink_test_at_start") f.hostlink_test_at_start = atoi(val.c_str());
        else if (name == "labels") { f.labels_mode = true; f.labels = val; }
        else {
            size_t t = 0;
            while (t < kNumSmTests && name != kSmTests[t].flag) ++t;
            if (t == kNumSmTests) { err = "flag provided but not defined: -" + name; return false; }
            f.sm_test_at_start[t] = atoi(val.c_str());
        }
    }
    if (!f.plugin_dir.empty() && f.plugin_dir.back() != '/') f.plugin_dir += '/';
    return true;
}

void logf(const char* fmt, ...) __attribute__((format(printf, 1, 2)));
void logf(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vfprintf(stderr, fmt, ap);
    va_end(ap);
    fputc('\n', stderr);
}

// One resource's plugin: plugin.go:41-48 AMDGPUPlugin + dpm/plugin.go devicePlugin
class Plugin {
public:
    Plugin(b2dp_ctx* ctx, const Flags& fl, std::string name) : ctx_(ctx), fl_(fl), name_(std::move(name)) {
        socket_ = fl_.plugin_dir + fl_.ns + "_" + name_;  // dpm/plugin.go:51-59
    }
    ~Plugin() { stop(); }

    bool start(std::string& err) {
        // plugin.go:82-91 Start(): allocator init; failure degrades to the kubelet's default allocation
        const int rc = b2dp_start(ctx_);
        alloc_ok_ = rc == B2DP_OK;
        if (!alloc_ok_) logf("allocator init failed (%s). Falling back to kubelet default allocation", b2dp_strerror(rc));
        server_ = std::make_unique<h2::GrpcServer>();
        server_->add_unary("/v1beta1.DevicePlugin/GetDevicePluginOptions", [this](const std::string&, std::string& out) {
            out = options();
            return h2::Status{};
        });
        server_->add_unary("/v1beta1.DevicePlugin/PreStartContainer", [](const std::string&, std::string& out) {
            out.clear();  // plugin.go:222-224
            return h2::Status{};
        });
        server_->add_unary("/v1beta1.DevicePlugin/GetPreferredAllocation",
                           [this](const std::string& in, std::string& out) { return preferred_allocation(in, out); });
        server_->add_unary("/v1beta1.DevicePlugin/Allocate", [this](const std::string& in, std::string& out) { return allocate(in, out); });
        server_->add_server_streaming("/v1beta1.DevicePlugin/ListAndWatch",
                                      [this](const std::string&, std::shared_ptr<h2::ServerStream> s) { list_and_watch(std::move(s)); });
        if (!server_->listen_unix(socket_, err)) { server_.reset(); return false; }
        return true;
    }

    // dpm/plugin.go:127-162 register()
    bool register_with_kubelet(std::string& err) {
        std::string opts, req;
        if (alloc_ok_) { b2dp::pb::tag(opts, 2, 0); b2dp::pb::varint(opts, 1); }  // get_preferred_allocation_available
        b2dp::pb::string_field(req, 1, "v1beta1");                                   // pluginapi.Version
        b2dp::pb::string_field(req, 2, fl_.ns + "_" + name_);                       // endpoint = socket basename
        b2dp::pb::string_field(req, 3, fl_.ns + "/" + name_);                       // resource name
        b2dp::pb::bytes_field(req, 4, opts);
        std::string resp;
        const h2::Status st = h2::unary_call_unix(fl_.plugin_dir + "kubelet.sock", "/v1beta1.Registration/Register", req, resp);
        if (st.code != h2::GRPC_OK) { err = "Register: grpc status " + std::to_string(st.code) + " " + st.message; return false; }
        return true;
    }

    // main.go:129-137: one tick of the shared heartbeat; like the reference's single unbuffered channel a tick
    // wakes ONE ListAndWatch stream (returns false if this plugin has none, so the caller can offer it elsewhere).
    bool beat() {
        std::lock_guard<std::mutex> l(mu_);
        reap_locked();
        if (watches_.empty()) return false;
        rr_ = (rr_ + 1) % watches_.size();
        b2dp_watch_beat(watches_[rr_]->w);
        return true;
    }

    void stop() {
        std::vector<std::unique_ptr<Watch>> ws;
        { std::lock_guard<std::mutex> l(mu_); ws.swap(watches_); }
        for (auto& w : ws) { b2dp_watch_stop(w->w); w->stream->finish({}); }  // returning from ListAndWatch ends the stream
        if (server_) { server_->stop(); server_.reset(); }
    }
    const std::string& name() const { return name_; }

private:
    struct Watch { b2dp_watch* w = nullptr; std::shared_ptr<h2::ServerStream> stream; std::atomic<bool> failed{false}; };

    std::string options() const {  // plugin.go:210-217
        std::string o;
        if (alloc_ok_) { b2dp::pb::tag(o, 2, 0); b2dp::pb::varint(o, 1); }
        return o;
    }

    // plugin.go:229-330: the library's watch loop produces the initial list and one response per heartbeat; this
    // side only forwards bytes to the stream.
    void list_and_watch(std::shared_ptr<h2::ServerStream> s) {
        auto w = std::make_unique<Watch>();
        w->stream = std::move(s);
        b2dp_cycle_opts o{};
        if (fl_.link_check) o.flags |= B2DP_LW_LINK_CHECK;
        Watch* raw = w.get();
        const int rc = b2dp_watch_start(ctx_, name_.c_str(), 0, &o, &Plugin::on_cycle, raw, &raw->w);
        if (rc != B2DP_OK) { raw->stream->finish({h2::GRPC_UNKNOWN, b2dp_strerror(rc)}); return; }
        std::lock_guard<std::mutex> l(mu_);
        reap_locked();
        watches_.push_back(std::move(w));
    }
    static void on_cycle(void* user, int rc, const uint8_t* buf, size_t len, const b2dp_cycle_stats*) {
        Watch* w = (Watch*)user;
        if (rc != B2DP_OK) { logf("ListAndWatch cycle failed: %s", b2dp_strerror(rc)); return; }
        if (!w->stream->send(std::string((const char*)buf, len))) w->failed = true;
    }
    void reap_locked() {  // streams the kubelet cancelled (restart, re-registration)
        for (size_t i = 0; i < watches_.size();) {
            if (watches_[i]->failed.load() || watches_[i]->stream->cancelled()) {
                std::unique_ptr<Watch> w = std::move(watches_[i]);
                watches_.erase(watches_.begin() + (long)i);
                b2dp_watch_stop(w->w);
            } else ++i;
        }
    }

    static bool read_strings(std::string_view msg, int want_field, std::vector<std::string>& out, int varint_field = 0, int64_t* v = nullptr) {
        pbread::Reader r(msg);
        int field, wire;
        while (!r.done()) {
            if (!r.tag(field, wire)) return false;
            if (wire == 2 && field == want_field) { std::string_view b; if (!r.bytes(b)) return false; out.emplace_back(b); }
            else if (wire == 0 && field == varint_field && v) { uint64_t x; if (!r.varint(x)) return false; *v = (int64_t)x; }
            else if (!r.skip(wire)) return false;
        }
        return true;
    }

    // plugin.go:337-351
    h2::Status preferred_allocation(const std::string& in, std::string& out) {
        pbread::Reader r(in);
        int field, wire;
        while (!r.done()) {
            if (!r.tag(field, wire)) return {h2::GRPC_INTERNAL, "bad PreferredAllocationRequest"};
            if (!(field == 1 && wire == 2)) { if (!r.skip(wire)) return {h2::GRPC_INTERNAL, "bad PreferredAllocationRequest"}; continue; }
            std::string_view creq;
            if (!r.bytes(creq)) return {h2::GRPC_INTERNAL, "bad PreferredAllocationRequest"};
            // ContainerPreferredAllocationRequest{available_deviceIDs=1, must_include_deviceIDs=2, allocation_size=3}
            std::vector<std::string> avail, must;
            int64_t size = 0;
            if (!read_strings(creq, 1, avail, 3, &size) || !read_strings(creq, 2, must)) return {h2::GRPC_INTERNAL, "bad ContainerPreferredAllocationRequest"};
            std::vector<const char*> pa, pm;
            for (auto& s : avail) pa.push_back(s.c_str());
            for (auto& s : must) pm.push_back(s.c_str());
            std::vector<char> ids((avail.size() + 1) * 64);
            int n = 0;
            const int rc = b2dp_preferred_allocation(ctx_, pa.data(), (int)pa.size(), pm.data(), (int)pm.size(), (int)(int32_t)size,
                                                     (char (*)[64])ids.data(), (int)avail.size() + 1, &n);
            if (rc != B2DP_OK)  // plugin.go:341-344: a Go error becomes status Unknown with its text
                return {h2::GRPC_UNKNOWN, std::string("unable to get preferred allocation list. Error:") + b2dp_strerror(rc)};
            std::string cresp;
            for (int i = 0; i < n; ++i) b2dp::pb::bytes_field(cresp, 1, std::string(&ids[(size_t)i * 64]));
            b2dp::pb::bytes_field(out, 1, cresp);
        }
        return {};
    }

    // plugin.go:356-393
    h2::Status allocate(const std::string& in, std::string& out) {
        pbread::Reader r(in);
        int field, wire;
        while (!r.done()) {
            if (!r.tag(field, wire)) return {h2::GRPC_INTERNAL, "bad AllocateRequest"};
            if (!(field == 1 && wire == 2)) { if (!r.skip(wire)) return {h2::GRPC_INTERNAL, "bad AllocateRequest"}; continue; }
            std::string_view creq;
            if (!r.bytes(creq)) return {h2::GRPC_INTERNAL, "bad AllocateRequest"};
            std::vector<std::string> ids;
            if (!read_strings(creq, 1, ids)) return {h2::GRPC_INTERNAL, "bad ContainerAllocateRequest"};
            std::vector<const char*> p;
            for (auto& s : ids) p.push_back(s.c_str());
            std::string buf(4096, '\0');
            size_t len = 0;
            int rc = b2dp_allocate_response(ctx_, p.data(), (int)p.size(), (uint8_t*)&buf[0], buf.size(), &len);
            if (rc == B2DP_E_NOSPC) { buf.assign(len, '\0'); rc = b2dp_allocate_response(ctx_, p.data(), (int)p.size(), (uint8_t*)&buf[0], buf.size(), &len); }
            if (rc != B2DP_OK) return {h2::GRPC_UNKNOWN, b2dp_strerror(rc)};
            b2dp::pb::bytes_field(out, 1, buf.substr(0, len));
        }
        return {};
    }

    b2dp_ctx* ctx_;
    const Flags& fl_;
    std::string name_, socket_;
    bool alloc_ok_ = false;
    std::unique_ptr<h2::GrpcServer> server_;
    std::mutex mu_;
    std::vector<std::unique_ptr<Watch>> watches_;
    size_t rr_ = 0;
};

// metricssvc.MetricsService/{List,GetGPUState} (internal/pkg/exporter/metricssvc/metricssvc.pb.go:95-110,284-291;
// metricssvc_grpc.pb.go:45-46) answered from the HBM probe, so that an UNMODIFIED reference plugin reads H100
// verdicts through its own exporter client (health.go:42-82): GPUState{ID=1, UUID=2, Health=3 "healthy"|"unhealthy"
// (health.go:75), AssociatedWorkload=4, Device=5 = the kubelet device id (health.go:98)}.  cuda: backend only.
class ExporterService {
public:
    ExporterService(b2dp_ctx* ctx, std::string path) : ctx_(ctx), path_(std::move(path)) {}
    bool start(std::string& err) {
        const size_t slash = path_.rfind('/');
        if (slash != std::string::npos && slash > 0) ::mkdir(path_.substr(0, slash).c_str(), 0755);
        server_.add_unary("/metricssvc.MetricsService/List", [this](const std::string&, std::string& out) { return states({}, out); });
        server_.add_unary("/metricssvc.MetricsService/GetGPUState", [this](const std::string& in, std::string& out) {
            std::vector<std::string> want;  // GPUGetRequest{ID=1 repeated string}
            pbread::Reader r(in);
            int field, wire;
            while (!r.done()) {
                if (!r.tag(field, wire)) return h2::Status{h2::GRPC_INTERNAL, "bad GPUGetRequest"};
                std::string_view b;
                if (field == 1 && wire == 2) { if (!r.bytes(b)) return h2::Status{h2::GRPC_INTERNAL, "bad GPUGetRequest"}; want.emplace_back(b); }
                else if (!r.skip(wire)) return h2::Status{h2::GRPC_INTERNAL, "bad GPUGetRequest"};
            }
            return states(want, out);
        });
        return server_.listen_unix(path_, err);
    }
    void stop() { server_.stop(); }

private:
    h2::Status states(const std::vector<std::string>& want, std::string& out) {
        std::vector<b2dp_device> devs(64);
        int n = 0;
        int rc = b2dp_enumerate(ctx_, devs.data(), (int)devs.size(), &n);
        if (rc == B2DP_E_NOSPC) { devs.resize((size_t)n); rc = b2dp_enumerate(ctx_, devs.data(), n, &n); }
        if (rc != B2DP_OK) return {h2::GRPC_UNKNOWN, b2dp_strerror(rc)};
        std::vector<b2dp_probe_result> res((size_t)n + 1);
        int m = 0;
        rc = b2dp_probe_health(ctx_, nullptr, res.data(), (int)res.size(), &m);
        if (rc != B2DP_OK) return {h2::GRPC_UNKNOWN, std::string(b2dp_strerror(rc)) + ": " + b2dp_last_error(ctx_)};
        for (int i = 0; i < m; ++i) {
            const int d = res[(size_t)i].device;
            if (d < 0 || d >= n) continue;
            const std::string id = std::to_string(d);
            if (!want.empty() && std::find(want.begin(), want.end(), id) == want.end()) continue;
            std::string g;
            b2dp::pb::string_field(g, 1, id);
            b2dp::pb::string_field(g, 2, devs[(size_t)d].id);
            b2dp::pb::string_field(g, 3, res[(size_t)i].healthy ? "healthy" : "unhealthy");
            b2dp::pb::string_field(g, 5, devs[(size_t)d].id);
            b2dp::pb::bytes_field(out, 1, g);
        }
        return {};
    }
    b2dp_ctx* ctx_;
    std::string path_;
    h2::GrpcServer server_;
};

bool sock_identity(const std::string& path, ino_t& ino, long long& ctime_ns) {
    struct stat st;
    if (::stat(path.c_str(), &st) != 0) return false;
    ino = st.st_ino;
    ctime_ns = (long long)st.st_ctim.tv_sec * 1000000000LL + st.st_ctim.tv_nsec;
    return true;
}

// Sleeps unless a stop signal arrives (signals are blocked and collected with sigtimedwait).
void sleep_interruptible(double seconds) {
    sigset_t stop;
    sigemptyset(&stop);
    for (int s : {SIGINT, SIGTERM, SIGQUIT}) sigaddset(&stop, s);
    const auto until = std::chrono::steady_clock::now() + std::chrono::duration<double>(seconds);
    while (!g_stop.load() && std::chrono::steady_clock::now() < until) {
        struct timespec ts{0, 20 * 1000 * 1000};
        if (sigtimedwait(&stop, nullptr, &ts) > 0) g_stop = true;
    }
}


// ---- node-labeller mode ---------------------------------------------------------------------------------------------
// A flat JSON object of strings (a node's .metadata.labels): parser and writer.  null values are read as absent.
void json_escape(std::string& o, const std::string& v) {
    o.push_back('"');
    for (unsigned char ch : v) {
        if (ch == '"' || ch == '\\') { o.push_back('\\'); o.push_back((char)ch); }
        else if (ch < 0x20) { char b[8]; snprintf(b, sizeof b, "\\u%04x", ch); o += b; }
        else o.push_back((char)ch);
    }
    o.push_back('"');
}
bool json_string(const std::string& s, size_t& i, std::string& out) {
    if (i >= s.size() || s[i] != '"') return false;
    out.clear();
    for (++i; i < s.size(); ++i) {
        const char ch = s[i];
        if (ch == '"') { ++i; return true; }
        if (ch != '\\') { out.push_back(ch); continue; }
        if (++i >= s.size()) return false;
        switch (s[i]) {
            case 'n': out.push_back('\n'); break; case 't': out.push_back('\t'); break; case 'r': out.push_back('\r'); break;
            case 'b': out.push_back('\b'); break; case 'f': out.push_back('\f'); break;
            case 'u': {
                if (i + 4 >= s.size()) return false;
                const unsigned cp = (unsigned)strtoul(s.substr(i + 1, 4).c_str(), nullptr, 16);
                i += 4;
                if (cp < 0x80) out.push_back((char)cp);
                else if (cp < 0x800) { out.push_back((char)(0xc0 | (cp >> 6))); out.push_back((char)(0x80 | (cp & 0x3f))); }
                else { out.push_back((char)(0xe0 | (cp >> 12))); out.push_back((char)(0x80 | ((cp >> 6) & 0x3f))); out.push_back((char)(0x80 | (cp & 0x3f))); }
                break;
            }
            default: out.push_back(s[i]);
        }
    }
    return false;
}
bool json_flat_object(const std::string& s, std::map<std::string, std::string>& out) {
    size_t i = 0;
    auto ws = [&] { while (i < s.size() && isspace((unsigned char)s[i])) ++i; };
    ws();
    if (s.compare(i, 4, "null") == 0) return true;  // a nil label map (controller.go:33-35)
    if (i >= s.size() || s[i] != '{') return false;
    ++i;
    ws();
    if (i < s.size() && s[i] == '}') return true;
    for (;;) {
        std::string k, v;
        ws();
        if (!json_string(s, i, k)) return false;
        ws();
        if (i >= s.size() || s[i] != ':') return false;
        ++i;
        ws();
        if (s.compare(i, 4, "null") == 0) i += 4;
        else { if (!json_string(s, i, v)) return false; out[k] = v; }
        ws();
        if (i < s.size() && s[i] == ',') { ++i; continue; }
        return i < s.size() && s[i] == '}';
    }
}

int labels_main(const Flags& fl) {
    if (fl.ns != "amd.com" && b2dp_set_vendor_domain(fl.ns.c_str()) != B2DP_OK) { logf("bad -resource_namespace %s", fl.ns.c_str()); return 2; }
    std::string uri = fl.backend;
    // labels need no HBM ring and no CUDA context: NVML answers (probe=off) unless the operator chose a probe mode
    if (uri.compare(0, 5, "cuda:") == 0 && uri.find("probe=") == std::string::npos) uri += (uri.size() > 5 ? "," : "") + std::string("probe=off");
    b2dp_ctx* ctx = nullptr;
    int rc = b2dp_open(uri.c_str(), &ctx);
    if (rc != B2DP_OK && uri != fl.backend) rc = b2dp_open(fl.backend.c_str(), &ctx);  // no NVML: the in-process backend answers from CUDA
    if (rc != B2DP_OK) { logf("open %s: %s (%s)", uri.c_str(), b2dp_strerror(rc), b2dp_last_error(nullptr)); return 1; }
    std::string csv = fl.labels;
    if (csv == "all") {  // main.go:46-53: every generator (+ the p2p-link extension on the cuda backend)
        char names[16][64];
        int n = 0;
        b2dp_label_generator_names(names, 16, &n);
        csv.clear();
        for (int i = 0; i < n; ++i) csv += (i ? "," : "") + std::string(names[i]);
        if (fl.backend.compare(0, 5, "cuda:") == 0) csv += ",p2p-link";
    }
    std::vector<b2dp_label> labels(256);
    int n = 0;
    rc = b2dp_generate_labels(ctx, csv.c_str(), labels.data(), (int)labels.size(), &n);
    if (rc == B2DP_E_NOSPC) { labels.resize((size_t)n); rc = b2dp_generate_labels(ctx, csv.c_str(), labels.data(), n, &n); }
    if (rc != B2DP_OK) { logf("generate labels: %s (%s)", b2dp_strerror(rc), b2dp_last_error(ctx)); b2dp_close(ctx); return 1; }
    b2dp_close(ctx);
    std::map<std::string, std::string> gen, before, after;
    for (int i = 0; i < n; ++i) gen[labels[(size_t)i].key] = labels[(size_t)i].value;
    auto dump = [](const std::map<std::string, std::string>& m) {
        std::string o = "{";
        bool first = true;
        for (auto& kv : m) { if (!first) o += ","; first = false; json_escape(o, kv.first); o += ":"; json_escape(o, kv.second); }
        return o + "}";
    };
    if (!fl.reconcile && !fl.patch) { printf("%s\n", dump(gen).c_str()); return 0; }
    const std::string in((std::istreambuf_iterator<char>(std::cin)), std::istreambuf_iterator<char>());
    if (!json_flat_object(in, before)) { logf("stdin is not a JSON object of strings (the node's label map)"); return 2; }
    // controller.go:23-58: drop this labeller's old labels (main.go:55-74), then set the generated ones
    std::vector<b2dp_label> cur(before.size() + 1);
    size_t k = 0;
    for (auto& kv : before) { snprintf(cur[k].key, sizeof cur[k].key, "%s", kv.first.c_str()); snprintf(cur[k].value, sizeof cur[k].value, "%s", kv.second.c_str()); ++k; }
    int kept = 0;
    b2dp_remove_old_node_labels(cur.data(), (int)before.size(), &kept);
    for (int i = 0; i < kept; ++i) after[cur[(size_t)i].key] = before[cur[(size_t)i].key];  // values verbatim (the ABI field is 96 bytes)
    for (auto& kv : gen) after[kv.first] = kv.second;
    if (fl.reconcile) { printf("%s\n", dump(after).c_str()); return 0; }
    // RFC 7386 merge patch: changed / new labels carry their value, removed ones null
    std::string o = "{\"metadata\":{\"labels\":{";
    bool first = true;
    std::map<std::string, const std::string*> diff;
    for (auto& kv : after) { auto it = before.find(kv.first); if (it == before.end() || it->second != kv.second) diff[kv.first] = &kv.second; }
    for (auto& kv : before) if (!after.count(kv.first)) diff[kv.first] = nullptr;
    for (auto& kv : diff) {
        if (!first) o += ",";
        first = false;
        json_escape(o, kv.first);
        o += ":";
        if (kv.second) json_escape(o, *kv.second); else o += "null";
    }
    printf("%s}}}\n", o.c_str());
    return 0;
}

// -memtest_at_start=1: test the free HBM of every GPU once, after open and before the first registration.  A failed
// device stays latched Unhealthy; the watch loop reports it with a heartbeat right after the initial list.
void run_memtest(b2dp_ctx* ctx, const Flags& fl) {
    b2dp_memtest_opts o{};
    o.max_bytes = fl.memtest_max_bytes;
    if (fl.memtest_at_start >= 2) o.flags |= B2DP_MT_EVEN_IF_BUSY;
    b2dp_memtest_result res[64];
    int n = 0;
    const int rc = b2dp_memtest(ctx, -1, &o, res, 64, &n);
    if (rc != B2DP_OK) {
        logf("memtest at start not run: %s (%s)", b2dp_strerror(rc), b2dp_last_error(ctx));
        return;
    }
    std::vector<b2dp_device> devs(n > 0 ? n : 1);
    int nd = 0;
    if (b2dp_enumerate(ctx, devs.data(), (int)devs.size(), &nd) != B2DP_OK) nd = 0;
    for (int i = 0; i < n; ++i) {
        const b2dp_memtest_result& r = res[i];
        logf("memtest %s: %s, %llu bytes in %d segment(s), flags 0x%x, mismatches %llu/%llu/%llu, ECC corrected %llu "
             "uncorrected %llu, %.1f ms, %.0f GB/s", r.device < nd ? devs[r.device].id : "?",
             r.healthy ? "Healthy" : "Unhealthy", (unsigned long long)r.bytes_tested, r.n_segments, r.flags,
             (unsigned long long)r.mismatches[1], (unsigned long long)r.mismatches[2], (unsigned long long)r.mismatches[3],
             (unsigned long long)r.ecc_corrected, (unsigned long long)r.ecc_uncorrected, r.ms, r.gbs);
    }
}

// -<flag>=1 of kSmTests[t] (see there)
void run_sm_test(b2dp_ctx* ctx, const Flags& fl, size_t t) {
    const SmTest& st = kSmTests[t];
    b2dp_compute_test_opts o{};
    o.duration_ms = fl.compute_test_ms;
    o.fault_sm = -1;
    if (fl.sm_test_at_start[t] >= 2) o.flags |= B2DP_CT_EVEN_IF_BUSY;
    b2dp_compute_test_result res[64];
    int n = 0;
    const int rc = st.run(ctx, -1, &o, res, 64, &n);
    if (rc != B2DP_OK) {
        logf("%s at start not run: %s (%s)", st.log, b2dp_strerror(rc), b2dp_last_error(ctx));
        return;
    }
    std::vector<b2dp_device> devs(n > 0 ? n : 1);
    int nd = 0;
    if (b2dp_enumerate(ctx, devs.data(), (int)devs.size(), &nd) != B2DP_OK) nd = 0;
    for (int i = 0; i < n; ++i) {
        const b2dp_compute_test_result& r = res[i];
        char rate[96];
        snprintf(rate, sizeof rate, st.rate, r.tflops[0], r.tflops[1], r.tflops[2]);
        logf("%s %s: %s, flags 0x%x, SMs %d/%d, mismatches %llu/%llu/%llu, first bad SM %d, %s", st.log,
             r.device < nd ? devs[r.device].id : "?", r.healthy ? "Healthy" : "Unhealthy", r.flags, r.sms_covered,
             r.sm_count, (unsigned long long)r.mismatches[0], (unsigned long long)r.mismatches[1],
             (unsigned long long)r.mismatches[2], r.first_bad_sm, rate);
    }
}

// -hostlink_test_at_start=1: likewise for the host-link self-test (the probe's pattern between host memory and the GPU,
// by copy engine and by the SMs' own loads and stores), after the L2 test, for -compute_test_ms per format.
void run_hostlink_test(b2dp_ctx* ctx, const Flags& fl) {
    b2dp_hostlink_opts o{};
    o.duration_ms = fl.compute_test_ms;
    if (fl.hostlink_test_at_start >= 2) o.flags |= B2DP_HL_EVEN_IF_BUSY;
    b2dp_hostlink_result res[64];
    int n = 0;
    const int rc = b2dp_hostlink_test(ctx, -1, &o, res, 64, &n);
    if (rc != B2DP_OK) {
        logf("host-link test at start not run: %s (%s)", b2dp_strerror(rc), b2dp_last_error(ctx));
        return;
    }
    std::vector<b2dp_device> devs(n > 0 ? n : 1);
    int nd = 0;
    if (b2dp_enumerate(ctx, devs.data(), (int)devs.size(), &nd) != B2DP_OK) nd = 0;
    for (int i = 0; i < n; ++i) {
        const b2dp_hostlink_result& r = res[i];
        logf("host-link test %s: %s, flags 0x%x, mismatches %llu/%llu/%llu, %.2f/%.2f/%.2f GB/s h2d/d2h/sm, "
             "PCIe gen %d x%d, replays %llu", r.device < nd ? devs[r.device].id : "?",
             r.healthy ? "Healthy" : "Unhealthy", r.flags, (unsigned long long)r.mismatches[0],
             (unsigned long long)r.mismatches[1], (unsigned long long)r.mismatches[2], r.gbs[0], r.gbs[1], r.gbs[2],
             r.link_gen, r.link_width, (unsigned long long)r.replays);
    }
}

}  // namespace

int main(int argc, char** argv) {
    Flags fl;
    std::string err;
    if (!parse_flags(argc, argv, fl, err)) { logf("%s", err.c_str()); return 2; }
    if (fl.version) {  // the reference stamps main.gitDescribe at link time (Makefile -X main.gitDescribe)
        printf("b200dp_plugind: libb200dp ABI %d (header %d), built %s\n", b2dp_abi_version(), B2DP_ABI_VERSION, __DATE__);
        return 0;
    }
    if (fl.labels_mode) return labels_main(fl);
    if (fl.strategy != "single" && fl.strategy != "mixed") {  // main.go:42-51,113-117
        logf("invalid resource naming strategy: %s", fl.strategy.c_str());
        return 1;
    }
    if (b2dp_abi_version() != B2DP_ABI_VERSION) { logf("libb200dp ABI %d, built against %d", b2dp_abi_version(), B2DP_ABI_VERSION); return 1; }
    // Signals are taken synchronously by this thread (sigtimedwait below): block them before any other thread
    // exists so every thread inherits the mask.  SIGINT/SIGQUIT/SIGTERM stop the daemon (plugin.go:83-84,
    // dpm/manager.go:47-48); SIGUSR1 is an operator's "heartbeat now".
    sigset_t sigs;
    sigemptyset(&sigs);
    for (int s : {SIGINT, SIGTERM, SIGQUIT, SIGUSR1}) sigaddset(&sigs, s);
    pthread_sigmask(SIG_BLOCK, &sigs, nullptr);
    signal(SIGPIPE, SIG_IGN);

    // the library's diagnostics (why a device flipped Unhealthy, helper restarts, Xids, calibration) go to stderr like glog's
    b2dp_set_log_callback([](void*, int level, const char* msg) { fprintf(stderr, "%c libb200dp: %s\n", level >= 2 ? 'E' : level == 1 ? 'W' : 'I', msg); }, nullptr);
    b2dp_ctx* ctx = nullptr;
    int rc = b2dp_open(fl.backend.c_str(), &ctx);
    if (rc != B2DP_OK) { logf("open %s: %s (%s)", fl.backend.c_str(), b2dp_strerror(rc), b2dp_last_error(nullptr)); return 1; }
    if (fl.memtest_at_start) run_memtest(ctx, fl);
    for (size_t t = 0; t < kNumSmTests; ++t) {
        if (t == kSmTestsBeforeHostlink && fl.hostlink_test_at_start) run_hostlink_test(ctx, fl);
        if (fl.sm_test_at_start[t]) run_sm_test(ctx, fl, t);
    }
    char names[64][64];
    int n_res = 0;
    rc = b2dp_resource_list(ctx, fl.strategy.c_str(), names, 64, &n_res);  // main.go:141-146
    if (rc != B2DP_OK) { logf("Error occured: %s", b2dp_strerror(rc)); b2dp_close(ctx); return 1; }

    std::unique_ptr<ExporterService> exporter;
    if (!fl.exporter_socket.empty()) {
        exporter = std::make_unique<ExporterService>(ctx, fl.exporter_socket);
        if (!exporter->start(err)) { logf("exporter socket: %s", err.c_str()); b2dp_close(ctx); return 1; }
        logf("metricssvc.MetricsService on %s", fl.exporter_socket.c_str());
    }
    std::vector<std::unique_ptr<Plugin>> plugins;
    auto start_all = [&] {  // dpm handleNewPlugins + startPlugin
        plugins.clear();
        for (int i = 0; i < n_res && !g_stop.load(); ++i) {
            std::string last;
            for (int attempt = 0; attempt < 3 && !g_stop.load(); ++attempt) {  // dpm/manager.go:16-20,205-219
                auto p = std::make_unique<Plugin>(ctx, fl, names[i]);
                if (p->start(last) && p->register_with_kubelet(last)) {
                    logf("%s/%s: serving on %s%s_%s, registered", fl.ns.c_str(), names[i], fl.plugin_dir.c_str(), fl.ns.c_str(), names[i]);
                    plugins.push_back(std::move(p));
                    last.clear();
                    break;
                }
                p.reset();
                sleep_interruptible(fl.start_retry_wait);
            }
            if (!last.empty()) logf("Failed to start plugin %s: %s", names[i], last.c_str());
        }
    };
    start_all();

    const std::string kubelet_sock = fl.plugin_dir + "kubelet.sock";
    // dpm/manager.go:52-58,73-84: an fsnotify watcher on the plugin directory; Create of kubelet.sock (re)starts the
    // plugin servers and re-registers, Remove stops them
    const int ino_fd = inotify_init1(IN_NONBLOCK | IN_CLOEXEC);
    const int ino_wd = ino_fd >= 0 ? inotify_add_watch(ino_fd, fl.plugin_dir.c_str(), IN_CREATE | IN_MOVED_TO | IN_DELETE | IN_MOVED_FROM) : -1;
    if (ino_wd < 0) logf("inotify on %s unavailable: falling back to a once-a-second check of kubelet.sock", fl.plugin_dir.c_str());
    ino_t seen_ino = 0;
    long long seen_ctime = 0;
    bool have_seen = sock_identity(kubelet_sock, seen_ino, seen_ctime);
    auto next_beat = std::chrono::steady_clock::now() + std::chrono::seconds(fl.pulse > 0 ? fl.pulse : 0);
    auto next_check = std::chrono::steady_clock::now() + std::chrono::seconds(1);
    size_t beat_rr = 0;
    auto heartbeat = [&] {  // main.go:129-137: `l.Heartbeat <- true` reaches one receiver
        for (size_t k = 0; k < plugins.size(); ++k) {
            beat_rr = (beat_rr + 1) % plugins.size();
            if (plugins[beat_rr]->beat()) break;
        }
    };
    while (!g_stop.load()) {
        struct timespec ts{0, 20 * 1000 * 1000};
        const int sig = sigtimedwait(&sigs, nullptr, &ts);
        if (sig == SIGUSR1) heartbeat();
        else if (sig > 0) { g_stop = true; break; }
        const auto now = std::chrono::steady_clock::now();
        if (fl.pulse > 0 && now >= next_beat) {
            next_beat += std::chrono::seconds(fl.pulse);
            heartbeat();
        }
        if (ino_wd >= 0) {
            alignas(struct inotify_event) char evbuf[4096];
            bool created = false, removed = false;
            for (;;) {
                const ssize_t r = read(ino_fd, evbuf, sizeof evbuf);
                if (r <= 0) break;
                for (char* p = evbuf; p < evbuf + r;) {
                    const struct inotify_event* ev = reinterpret_cast<const struct inotify_event*>(p);
                    if (ev->len && strcmp(ev->name, "kubelet.sock") == 0) {
                        if (ev->mask & (IN_CREATE | IN_MOVED_TO)) { created = true; removed = false; }
                        if (ev->mask & (IN_DELETE | IN_MOVED_FROM)) { removed = true; created = false; }
                    }
                    p += sizeof(struct inotify_event) + ev->len;
                }
            }
            if (removed) { logf("kubelet.sock removed: stopping plugin servers"); plugins.clear(); have_seen = false; }
            if (created) {
                logf("kubelet.sock created: restarting plugins");
                start_all();
                have_seen = sock_identity(kubelet_sock, seen_ino, seen_ctime);
                next_check = now + std::chrono::seconds(1);
            }
        }
        if (now >= next_check) {  // fallback / safety net for the same events (a missed or unavailable inotify)
            next_check = now + std::chrono::seconds(1);
            ino_t ino = 0;
            long long ct = 0;
            if (sock_identity(kubelet_sock, ino, ct)) {
                if (have_seen && (ino != seen_ino || ct != seen_ctime)) { logf("kubelet.sock re-created: restarting plugins"); start_all(); }
                else if (!have_seen && plugins.empty()) start_all();
                seen_ino = ino; seen_ctime = ct; have_seen = true;
            }
        }
    }
    logf("Received signal, exiting");
    if (ino_fd >= 0) close(ino_fd);
    plugins.clear();
    if (exporter) exporter->stop();
    b2dp_close(ctx);
    return 0;
}
