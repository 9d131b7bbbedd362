#include "rmu_gemm.cuh"

namespace rmu {

int make_split_operand(SplitOperand* op, __half* hi, __half* lo, int64_t rows, int cols) {
    if (cols % kGemmBK != 0) { set_error("make_split_operand: K must be a multiple of 64"); return RMU_ERR_ARG; }
    op->hi = hi; op->lo = lo; op->rows = rows; op->cols = cols;
    const uint64_t pitch = static_cast<uint64_t>(cols) * sizeof(__half);
    int rc = make_tmap_2d(&op->map_hi, hi, static_cast<uint64_t>(rows), static_cast<uint64_t>(cols), pitch, kGemmBK, 128, 2);
    if (rc == RMU_OK) rc = make_tmap_2d(&op->map_lo, lo, static_cast<uint64_t>(rows), static_cast<uint64_t>(cols), pitch, kGemmBK, 128, 2);
    return rc;
}

template <int MODE>
static int launch_mode(const SplitOperand& A, const SplitOperand& W, const GemmParams& p, int sms, cudaStream_t st) {
    auto kern = gemm_f16x3_kernel<MODE>;
    // the attribute is per device and the call is cheap: set it on every launch (one process may drive several GPUs)
    RMU_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kGemmSmem)));
    // output maps of exactly M rows (the TMA store clips the tail of the last row block): 128-row x 128-byte boxes
    CUtensorMap tOa{}, tOb{};
    // GeGLU / SwiGLU write N / 2 columns: that is also their default row pitch
    const uint64_t ld = static_cast<uint64_t>(p.out_ld ? p.out_ld : (gemm_gated(MODE) ? p.N / 2 : p.N));
    int rc;
    if (MODE == GEMM_BIAS_F32 || MODE == GEMM_BIAS_RESID_F32 || MODE == GEMM_BIAS_RESF32_F32) {
        rc = make_tmap_2d(&tOa, p.out_f32, static_cast<uint64_t>(p.M), static_cast<uint64_t>(p.N), ld * sizeof(float), 32,
                          kGemmBM, 4);
    } else {
        const uint64_t pitch = ld * sizeof(__half);
        const uint64_t cols = static_cast<uint64_t>(gemm_gated(MODE) ? p.N / 2 : p.N);   // GeGLU / SwiGLU: [M, N / 2]
        rc = make_tmap_2d(&tOa, p.out_hi, static_cast<uint64_t>(p.M), cols, pitch, 64, kGemmBM, 2);
        if (rc == RMU_OK) rc = make_tmap_2d(&tOb, p.out_lo, static_cast<uint64_t>(p.M), cols, pitch, 64, kGemmBM, 2);
    }
    if (rc != RMU_OK) return rc;
    const int tiles = ((p.M + kGemmBM - 1) / kGemmBM) * (p.N / kGemmBN);
    const int grid = tiles < sms ? tiles : sms;
    ProfScope _ps(PROF_GEMM, st);
    kern<<<grid, kGemmThreads, kGemmSmem, st>>>(A.map_hi, A.map_lo, W.map_hi, W.map_lo, tOa, tOb, p);
    count_launch();
    RMU_CHECK_LAUNCH();
    return RMU_OK;
}

int launch_gemm(int mode, const SplitOperand& A, const SplitOperand& W, const GemmParams& p, int sms, cudaStream_t st) {
    if (p.M <= 0) return RMU_OK;
    if (p.N % kGemmBN != 0 || p.K % kGemmBK != 0 || A.cols != p.K || W.cols != p.K || W.rows < p.N || A.rows < p.M ||
        (p.out_ld != 0 && p.out_ld < (gemm_gated(mode) ? p.N / 2 : p.N))) {
        set_error("launch_gemm: shape not supported (N % 128, K % 64)");
        return RMU_ERR_UNSUPPORTED;
    }
    switch (mode) {
        case GEMM_BIAS_F32: return launch_mode<GEMM_BIAS_F32>(A, W, p, sms, st);
        case GEMM_BIAS_GELU_SPLIT: return launch_mode<GEMM_BIAS_GELU_SPLIT>(A, W, p, sms, st);
        case GEMM_BIAS_RESID_F32: return launch_mode<GEMM_BIAS_RESID_F32>(A, W, p, sms, st);
        case GEMM_BIAS_SPLIT_QSCALE: return launch_mode<GEMM_BIAS_SPLIT_QSCALE>(A, W, p, sms, st);
        case GEMM_BIAS_SPLIT_ROPE:
            if (!p.pos || !p.rope_cos || !p.rope_sin || p.rope_rows <= 0 || (p.rope_hd != 32 && p.rope_hd != 64) ||
                p.qcols % 64 != 0 || p.qcols % p.rope_hd != 0) {
                set_error("launch_gemm: the rotary epilogue needs positions, cos / sin tables, head_dim 32 or 64 and qcols a "
                          "multiple of 64");
                return RMU_ERR_ARG;
            }
            return launch_mode<GEMM_BIAS_SPLIT_ROPE>(A, W, p, sms, st);
        case GEMM_BIAS_GEGLU_SPLIT: return launch_mode<GEMM_BIAS_GEGLU_SPLIT>(A, W, p, sms, st);
        case GEMM_BIAS_RESF32_F32:
            if (!p.res_f32) { set_error("launch_gemm: the fp32 residual epilogue needs res_f32"); return RMU_ERR_ARG; }
            return launch_mode<GEMM_BIAS_RESF32_F32>(A, W, p, sms, st);
        case GEMM_BIAS_SWIGLU_SPLIT: return launch_mode<GEMM_BIAS_SWIGLU_SPLIT>(A, W, p, sms, st);
    }
    set_error("launch_gemm: bad mode");
    return RMU_ERR_ARG;
}

static_assert(RMU_GEMM_BIAS_F32 == GEMM_BIAS_F32 && RMU_GEMM_BIAS_GELU_SPLIT == GEMM_BIAS_GELU_SPLIT &&
              RMU_GEMM_BIAS_RESID_F32 == GEMM_BIAS_RESID_F32 && RMU_GEMM_BIAS_SPLIT_QSCALE == GEMM_BIAS_SPLIT_QSCALE &&
              RMU_GEMM_BIAS_SPLIT_ROPE == GEMM_BIAS_SPLIT_ROPE && RMU_GEMM_BIAS_GEGLU_SPLIT == GEMM_BIAS_GEGLU_SPLIT &&
              RMU_GEMM_BIAS_RESF32_F32 == GEMM_BIAS_RESF32_F32 && RMU_GEMM_BIAS_SWIGLU_SPLIT == GEMM_BIAS_SWIGLU_SPLIT,
              "the C ABI mode ids are the kernel's");

}  // namespace rmu

using namespace rmu;

extern "C" int rmu_debug_gemm(int mode, const uint16_t* a_hi, const uint16_t* a_lo, int64_t a_rows, const uint16_t* w_hi,
                              const uint16_t* w_lo, int M, int N, int K, const float* bias, const uint16_t* res_hi,
                              const uint16_t* res_lo, int qcols, float qscale, int max_ctas, float* out_f32,
                              uint16_t* out_hi, uint16_t* out_lo, void* stream) {
    const bool f32_out = mode == GEMM_BIAS_F32 || mode == GEMM_BIAS_RESID_F32;
    if (mode < GEMM_BIAS_F32 || mode > GEMM_BIAS_SPLIT_QSCALE || !a_hi || !a_lo || !w_hi || !w_lo || !bias ||
        (f32_out ? !out_f32 : (!out_hi || !out_lo)) || (mode == GEMM_BIAS_RESID_F32 && (!res_hi || !res_lo)) ||
        M <= 0 || N <= 0 || K <= 0 || max_ctas < 0) {
        set_error("rmu_debug_gemm: bad argument");
        return RMU_ERR_ARG;
    }
    if (N % kGemmBN != 0 || K % kGemmBK != 0 || a_rows < M) {
        set_error("rmu_debug_gemm: shape not supported (N % 128, K % 64, a_rows >= M)");
        return RMU_ERR_UNSUPPORTED;
    }
    SplitOperand A, W;
    int rc = make_split_operand(&A, const_cast<__half*>(reinterpret_cast<const __half*>(a_hi)),
                                const_cast<__half*>(reinterpret_cast<const __half*>(a_lo)), a_rows, K);
    if (rc == RMU_OK)
        rc = make_split_operand(&W, const_cast<__half*>(reinterpret_cast<const __half*>(w_hi)),
                                const_cast<__half*>(reinterpret_cast<const __half*>(w_lo)), N, K);
    if (rc != RMU_OK) return rc;
    GemmParams p{};
    p.M = M; p.N = N; p.K = K; p.bias = bias;
    p.out_f32 = out_f32;
    p.out_hi = reinterpret_cast<__half*>(out_hi); p.out_lo = reinterpret_cast<__half*>(out_lo);
    p.res_hi = reinterpret_cast<const __half*>(res_hi); p.res_lo = reinterpret_cast<const __half*>(res_lo);
    p.qcols = qcols; p.qscale = qscale;
    const int sms = max_ctas > 0 ? max_ctas : device_sm_count();
    if (sms <= 0) { set_error("rmu_debug_gemm: no CUDA device"); return RMU_ERR_CUDA; }
    return launch_gemm(mode, A, W, p, sms, static_cast<cudaStream_t>(stream));
}

extern "C" int rmu_debug_gemm_ex(int mode, const uint16_t* a_hi, const uint16_t* a_lo, int64_t a_rows, const uint16_t* w_hi,
                                 const uint16_t* w_lo, int M, int N, int K, const float* bias, const float* res_f32,
                                 int qcols, float qscale, const int32_t* pos, const float* rope_cos, const float* rope_sin,
                                 int rope_rows, int head_dim, int max_ctas, float* out_f32, uint16_t* out_hi,
                                 uint16_t* out_lo, void* stream) {
    const bool f32_out = mode == GEMM_BIAS_RESF32_F32;
    if (mode < GEMM_BIAS_SPLIT_ROPE || mode > GEMM_BIAS_RESF32_F32 || !a_hi || !a_lo || !w_hi || !w_lo || !bias ||
        (f32_out ? (!out_f32 || !res_f32) : (!out_hi || !out_lo)) ||
        (mode == GEMM_BIAS_SPLIT_ROPE && (!pos || !rope_cos || !rope_sin || rope_rows <= 0)) || M <= 0 || N <= 0 ||
        K <= 0 || max_ctas < 0) {
        set_error("rmu_debug_gemm_ex: bad argument");
        return RMU_ERR_ARG;
    }
    if (N % kGemmBN != 0 || K % kGemmBK != 0 || a_rows < M ||
        (mode == GEMM_BIAS_SPLIT_ROPE && ((head_dim != 32 && head_dim != 64) || qcols % 64 != 0 || qcols % head_dim != 0))) {
        set_error("rmu_debug_gemm_ex: shape not supported (N % 128, K % 64, a_rows >= M; rotary: head_dim 32 or 64, qcols "
                  "a multiple of 64)");
        return RMU_ERR_UNSUPPORTED;
    }
    SplitOperand A, W;
    int rc = make_split_operand(&A, const_cast<__half*>(reinterpret_cast<const __half*>(a_hi)),
                                const_cast<__half*>(reinterpret_cast<const __half*>(a_lo)), a_rows, K);
    if (rc == RMU_OK)
        rc = make_split_operand(&W, const_cast<__half*>(reinterpret_cast<const __half*>(w_hi)),
                                const_cast<__half*>(reinterpret_cast<const __half*>(w_lo)), N, K);
    if (rc != RMU_OK) return rc;
    GemmParams p{};
    p.M = M; p.N = N; p.K = K; p.bias = bias;
    p.out_f32 = out_f32;
    p.out_hi = reinterpret_cast<__half*>(out_hi); p.out_lo = reinterpret_cast<__half*>(out_lo);
    p.res_f32 = res_f32;
    p.qcols = qcols; p.qscale = qscale;
    p.pos = pos; p.rope_cos = rope_cos; p.rope_sin = rope_sin; p.rope_hd = head_dim; p.rope_rows = rope_rows;
    const int sms = max_ctas > 0 ? max_ctas : device_sm_count();
    if (sms <= 0) { set_error("rmu_debug_gemm_ex: no CUDA device"); return RMU_ERR_CUDA; }
    return launch_gemm(mode, A, W, p, sms, static_cast<cudaStream_t>(stream));
}

extern "C" int rmu_debug_gemm_swiglu(const uint16_t* a_hi, const uint16_t* a_lo, int64_t a_rows, const uint16_t* w_hi,
                                     const uint16_t* w_lo, int M, int N, int K, const float* bias, int max_ctas,
                                     uint16_t* out_hi, uint16_t* out_lo, int32_t* range_flag, void* stream) {
    if (!a_hi || !a_lo || !w_hi || !w_lo || !bias || !out_hi || !out_lo || M <= 0 || N <= 0 || K <= 0 || max_ctas < 0) {
        set_error("rmu_debug_gemm_swiglu: bad argument");
        return RMU_ERR_ARG;
    }
    if (N % kGemmBN != 0 || K % kGemmBK != 0 || a_rows < M) {
        set_error("rmu_debug_gemm_swiglu: shape not supported (N % 128, K % 64, a_rows >= M)");
        return RMU_ERR_UNSUPPORTED;
    }
    SplitOperand A, W;
    int rc = make_split_operand(&A, const_cast<__half*>(reinterpret_cast<const __half*>(a_hi)),
                                const_cast<__half*>(reinterpret_cast<const __half*>(a_lo)), a_rows, K);
    if (rc == RMU_OK)
        rc = make_split_operand(&W, const_cast<__half*>(reinterpret_cast<const __half*>(w_hi)),
                                const_cast<__half*>(reinterpret_cast<const __half*>(w_lo)), N, K);
    if (rc != RMU_OK) return rc;
    GemmParams p{};
    p.M = M; p.N = N; p.K = K; p.bias = bias;
    p.out_hi = reinterpret_cast<__half*>(out_hi); p.out_lo = reinterpret_cast<__half*>(out_lo);
    p.range_flag = range_flag;
    const int sms = max_ctas > 0 ? max_ctas : device_sm_count();
    if (sms <= 0) { set_error("rmu_debug_gemm_swiglu: no CUDA device"); return RMU_ERR_CUDA; }
    return launch_gemm(GEMM_BIAS_SWIGLU_SPLIT, A, W, p, sms, static_cast<cudaStream_t>(stream));
}
