// Host-side helpers shared by the translation units of libragmeup_b200.so.
#pragma once
#include <cuda_runtime.h>
#include <cuda.h>
#include <stdint.h>
#include <atomic>
#include <string>

#include "../../include/ragmeup_b200.h"

namespace rmu {

void set_error(const std::string& msg);
extern std::atomic<uint64_t> g_launches;

// every kernel launch in the library goes through this counter (bench.py gpu_launches)
inline void count_launch(int n = 1) { g_launches.fetch_add(static_cast<uint64_t>(n), std::memory_order_relaxed); }

// ---- optional per-kernel-class timing (bench.py roofline): CUDA events on the launching stream
enum ProfClass { PROF_SCAN = 0, PROF_FINALIZE, PROF_EXACT, PROF_MERGE, PROF_GEMM, PROF_ATTN, PROF_LN, PROF_EMBED,
                 PROF_POOL_HEAD, PROF_MISC, PROF_SCAN_LEAD /* second-pass scan launches */,
                 PROF_DECODE_ATTN /* decode attention and the KV cache writes */, PROF_LM_HEAD, PROF_SAMPLE,
                 PROF_NF4 /* NF4 weights: quantiser, dequantiser, decode GEMV */, PROF_NCLASS };
extern std::atomic<int> g_prof_on;
void prof_begin(int cls, cudaStream_t st);
void prof_end(int cls, cudaStream_t st);
struct ProfScope {
    int cls; cudaStream_t st; bool on;
    ProfScope(int c, cudaStream_t s) : cls(c), st(s), on(g_prof_on.load(std::memory_order_relaxed) != 0) { if (on) prof_begin(cls, st); }
    ~ProfScope() { if (on) prof_end(cls, st); }
};

#define RMU_CUDA(expr)                                                                       \
    do {                                                                                     \
        cudaError_t _e = (expr);                                                             \
        if (_e != cudaSuccess) {                                                             \
            ::rmu::set_error(std::string(#expr) + ": " + cudaGetErrorString(_e));            \
            return RMU_ERR_CUDA;                                                             \
        }                                                                                    \
    } while (0)

#define RMU_CHECK_LAUNCH()                                                                   \
    do {                                                                                     \
        cudaError_t _e = cudaGetLastError();                                                 \
        if (_e != cudaSuccess) {                                                             \
            ::rmu::set_error(std::string("kernel launch: ") + cudaGetErrorString(_e));       \
            return RMU_ERR_CUDA;                                                             \
        }                                                                                    \
    } while (0)

// cuTensorMapEncodeTiled resolved through the runtime (no link-time libcuda dependency, so the
// library loads on a GPU-less build box).  Returns nullptr + sets the error when unavailable.
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
PFN_encodeTiled get_encode_tiled();

// 2-D row-major [rows, cols] tensor of `elem_bytes` elements, box {box_cols, box_rows}, 128-B swizzle.
int make_tmap_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t row_stride_bytes,
                 uint32_t box_cols, uint32_t box_rows, int elem_bytes);   // box 128 B wide (SWIZZLE_128B) or 64 B (SWIZZLE_64B)

// fp32 row-major [rows, 32*kblocks] viewed as (32 floats, rows, kblock) so that ONE box
// {32, box_rows, box_kb} lands in smem as box_kb consecutive K-major 128-B-swizzled slabs.
int make_tmap_rows_kblocks(CUtensorMap* out, const void* base, uint64_t rows, uint32_t kblocks,
                           uint32_t box_rows, uint32_t box_kb);

int device_sm_count();

}  // namespace rmu
