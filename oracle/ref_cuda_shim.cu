// ref_cuda_shim.cu -- TEST / BENCH INFRASTRUCTURE ONLY.  Thin entry into the reference's own CUDA GEMV so that it can run on the same
// GPU as a GPU-side baseline and as a second oracle (SURVEY.md 8(c), 8(d) config 2: "the reference gemv_kernel_g128 compiled for
// sm_90a as reference CUDA on the same GPU").  oracle/Makefile compiles /root/reference/kernels/cuda/gemv_cuda.cu where it lies, unchanged,
// next to this file; nothing of the reference is copied.  The only code here fills `matmul_params` exactly like the reference call
// site Linear_half_int4::forward (llm/src/ops/cuda/linear.cu:20-33) and calls MatmulOperator::gemv_forward_cuda.
#include <cuda_runtime.h>

#include "matmul.h"

extern "C" __attribute__((visibility("default"))) int ref_cuda_gemv(void *x_half, void *w_u32, void *zeros_u32, void *scales_half, void *y_half, int M,
                                                                    int IC, int OC) {
    struct matmul_params params;
    params.A.row = M;
    params.A.column = IC;
    params.A.half_data_ptr = reinterpret_cast<float16_t *>(x_half);
    params.B.row = IC / 8;  // k
    params.B.column = OC;   // n
    params.B.int32_data_ptr = reinterpret_cast<int *>(w_u32);
    params.C.row = M;
    params.C.column = OC;
    params.C.half_data_ptr = reinterpret_cast<float16_t *>(y_half);
    params.opt_params.num_thread = 8;
    params.half_scales = reinterpret_cast<float16_t *>(scales_half);
    params.int32_zero_point = reinterpret_cast<int *>(zeros_u32);
    params.block_size = 128;  // QK of the QM_CUDA build (llm/include/common.h)
    matmul::MatmulOperator op = matmul::MatmulOperator();
    op.gemv_forward_cuda(&params);  // launches on the legacy default stream, unchecked, like the reference
    return (int)cudaGetLastError();
}
