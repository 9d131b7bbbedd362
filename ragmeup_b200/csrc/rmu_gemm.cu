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
    int rc;
    if (MODE == GEMM_BIAS_F32 || MODE == GEMM_BIAS_RESID_F32) {
        rc = make_tmap_2d(&tOa, p.out_f32, static_cast<uint64_t>(p.M), static_cast<uint64_t>(p.N),
                          static_cast<uint64_t>(p.N) * sizeof(float), 32, kGemmBM, 4);
    } else {
        const uint64_t pitch = static_cast<uint64_t>(p.N) * sizeof(__half);
        rc = make_tmap_2d(&tOa, p.out_hi, static_cast<uint64_t>(p.M), static_cast<uint64_t>(p.N), pitch, 64, kGemmBM, 2);
        if (rc == RMU_OK) rc = make_tmap_2d(&tOb, p.out_lo, static_cast<uint64_t>(p.M), static_cast<uint64_t>(p.N), pitch, 64, kGemmBM, 2);
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
    if (p.N % kGemmBN != 0 || p.K % kGemmBK != 0 || A.cols != p.K || W.cols != p.K || W.rows < p.N || A.rows < p.M) {
        set_error("launch_gemm: shape not supported (N % 128, K % 64)");
        return RMU_ERR_UNSUPPORTED;
    }
    switch (mode) {
        case GEMM_BIAS_F32: return launch_mode<GEMM_BIAS_F32>(A, W, p, sms, st);
        case GEMM_BIAS_GELU_SPLIT: return launch_mode<GEMM_BIAS_GELU_SPLIT>(A, W, p, sms, st);
        case GEMM_BIAS_RESID_F32: return launch_mode<GEMM_BIAS_RESID_F32>(A, W, p, sms, st);
        case GEMM_BIAS_SPLIT_QSCALE: return launch_mode<GEMM_BIAS_SPLIT_QSCALE>(A, W, p, sms, st);
    }
    set_error("launch_gemm: bad mode");
    return RMU_ERR_ARG;
}

}  // namespace rmu
