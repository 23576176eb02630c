// compute_test_tables_kernels.cu -- test-only harness that launches the tensor-core self-test kernel of tc_selftest.cuh
// on tables the caller built (tests/test_gpu_compute_test_tables.py).
//
// The library is the harness of compute_test_kernels.cu (ck_open, ck_run, ck_dump, ...), compiled into it as it is,
// plus ck_run_tables: either instantiation on operand images and comparison values from tests/compute_test_tables.py.
// So a test can hand the kernel crafted tiles, or wrong operands or wrong comparison values, and see what the product's
// path from operand bytes through the tensor cores, the fold and the CTA-wide compare to the record makes of them.
#include "compute_test_kernels.cu"

namespace {

int upload_tables(Harness* h, Launch& L, int fmt, const uint8_t* images, const uint32_t* checks, int n_rec) {
    const size_t image_bytes = (size_t)kCtTiles * kSmem[fmt], check_bytes = (size_t)kCtTiles * kCtThreads * 4;
    CK(h, cudaMalloc(&L.img, image_bytes));
    CK(h, cudaMalloc(&L.chk, check_bytes));
    CK(h, cudaMemcpy(L.img, images, image_bytes, cudaMemcpyHostToDevice));
    CK(h, cudaMemcpy(L.chk, checks, check_bytes, cudaMemcpyHostToDevice));
    CK(h, cudaHostAlloc(&L.rec_h, (size_t)n_rec * sizeof(CtRecord), cudaHostAllocMapped));
    memset(L.rec_h, 0, (size_t)n_rec * sizeof(CtRecord));
    CK(h, cudaHostGetDevicePointer(&L.rec_d, L.rec_h, 0));
    return 0;
}

}  // namespace

extern "C" {

// Refusals, returned before anything is allocated or launched (CK_E_FMT and CK_E_NOSPC as in ck_run).
enum { CK_E_SIZE = -3, CK_E_GRID = -4, CK_E_DUMP = -5 };

// The product (dump = 0) or DUMP (dump != 0) instantiation of format `fmt` on tables the caller built: `images` holds
// kCtTiles images of CtShape<fmt>::SMEM bytes (image_bytes in all), `checks` [kCtTiles][kCtThreads] comparison values.
// `grid` CTAs, from 1 up to the resident CTAs of that instantiation, run for duration_ns (no fault hook).  Every CTA's
// record goes to recs (cap records), the count to *n, the CUDA-event time of the launch to *ms, and with DUMP CTA 0's
// raw accumulators (kCtTiles x kCtThreads x kCtAcc words) to dump_out.
int ck_run_tables(void* hp, int fmt, int dump, const uint8_t* images, unsigned long long image_bytes,
                  const uint32_t* checks, int grid, unsigned long long duration_ns, CtRecord* recs, int cap, int* n,
                  float* ms, uint32_t* dump_out) {
    Harness* h = static_cast<Harness*>(hp);
    if (fmt < 0 || fmt >= kCtFormats) return CK_E_FMT;
    if (image_bytes != (unsigned long long)kCtTiles * kSmem[fmt]) return CK_E_SIZE;
    if (dump && !dump_out) return CK_E_DUMP;
    const CtKernel fn = dump ? kDump[fmt] : kProduct[fmt];
    CK(h, cudaSetDevice(h->device));
    int per_sm = 0;
    CK(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, kCtThreads, kSmem[fmt]));
    if (grid < 1 || grid > h->sms * per_sm) return CK_E_GRID;
    *n = grid;
    if (grid > cap) return CK_E_NOSPC;
    Launch L;
    if (upload_tables(h, L, fmt, images, checks, grid)) return CK_E_CUDA;
    const size_t words = (size_t)kCtTiles * kCtThreads * kCtAcc;
    if (dump) {
        CK(h, cudaMalloc(&L.dump, words * 4));
        CK(h, cudaMemsetAsync(L.dump, 0xFF, words * 4, h->stream));
    }
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    CK(h, cudaEventCreate(&e0));
    CK(h, cudaEventCreate(&e1));
    cudaEventRecord(e0, h->stream);
    fn<<<grid, kCtThreads, kSmem[fmt], h->stream>>>(L.img, L.chk, duration_ns, -1, 0u, L.rec_d, 9ull, L.dump);
    cudaError_t e = cudaGetLastError();
    cudaEventRecord(e1, h->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
    if (e == cudaSuccess) e = cudaEventElapsedTime(ms, e0, e1);
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    if (e != cudaSuccess) return fail(h, "tc_selftest", e);
    if (dump) CK(h, cudaMemcpy(dump_out, L.dump, words * 4, cudaMemcpyDeviceToHost));
    memcpy(recs, (const void*)L.rec_h, (size_t)grid * sizeof(CtRecord));
    return CK_OK;
}

}  // extern "C"
