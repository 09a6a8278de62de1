// matmul.h -- operator surface of libtce_host.so: the CUDA-backend half of the reference's `matmul::MatmulOperator`, backed by the
// C ABI of libtce_b200.so.
//
// The four parameter structs below are binary-compatible (same fields, same order, same types, QM_CUDA flavour: float16_t = half)
// with the reference's kernels/matmul.h:52-100, so objects filled by the reference's llm/ call sites (Linear_half_int4::forward
// llm/src/ops/cuda/linear.cu:5-40, W8A8B8O8Linear::forward llm/src/ops/W8A8B8O8Linear.cc:38-78, the BMM_S8T_* wrappers, ...) can be
// handed to this library unchanged; tests/test_host_header_abi.py compiles an offsetof/sizeof probe against both headers.
// The class declares every method of the reference's matmul::MatmulOperator (kernels/matmul.h:110-166), so a call site written against
// the reference header also compiles against this one.  matmul_operator.cu DEFINES the ones the reference's kernels/cuda/ directory
// defines (TCE_MATMUL_OPS) plus the gemm_forward_cuda* slot it declares without defining; the rest (TCE_MATMUL_OPS_ELSEWHERE) are the
// backend-independent or other-backend methods: no CUDA call site of the reference reaches them, and a full build keeps taking them
// from the reference's own kernels/*.cc (INTEGRATION.md).  tests/test_gpu_callsites.py goes one step further and compiles the
// reference's call sites against the reference's OWN header (-DTCE_REFERENCE_MATMUL_H=...) and this library.
#ifndef TCE_HOST_MATMUL_H
#define TCE_HOST_MATMUL_H
#include <cuda_fp16.h>
#include <stdint.h>
#include <sys/time.h>

// host-side fp16 type of the reference (half_float::half) when its header is reachable, a storage-only stand-in otherwise
#if defined(__has_include)
#if __has_include("half.hpp")
#include "half.hpp"
typedef half_float::half naive_float16_t;
#define TCE_HAVE_HALF_HPP 1
#endif
#endif
#ifndef TCE_HAVE_HALF_HPP
struct naive_float16_t { uint16_t bits; };
#endif
typedef half float16_t;

// ---- parameter blocks (layout contract; do not reorder) ----
struct quantization_params { float scale; bool per_channel = false; int32_t zero_point; int8_t q_min = -128, q_max = 127; };

struct matrix {
    int row, column;                               // meaning is per call site (DESIGN.md 1, SURVEY.md 8b)
    float *data_ptr; float16_t *half_data_ptr; naive_float16_t *fp16_data_ptr;   // exactly one typed pointer is set per op
    int32_t *int32_data_ptr; int8_t *int8_data_ptr; uint8_t *uint8_data_ptr, *int4_data_ptr;
    struct quantization_params qparams;
    int length() { return row * column; }
};

struct optimization_params { int blk_size; int num_thread = 8; };

struct matmul_params {
    struct matrix A, B, C, bias;
    struct optimization_params opt_params;
    float alpha, beta; float16_t half_alpha;
    float *scales, *offset, *zero_point;           // W4 CPU formats
    float16_t *half_scales;                        // W4 QM_CUDA: half[OC][zeros_w * 8]
    naive_float16_t *fp16_scales;                  // AWQ-GEMM layout of the fp16 host reference
    int *int32_zero_point;                         // W4 QM_CUDA: uint32[OC][zeros_w]
    int block_size;
    float *A_scales; int8_t A_zero_point;          // W4A8 CPU path
};

namespace matmul {

// X(name): takes `const struct matmul_params *`
#define TCE_MATMUL_OPS(X)                                                                                                            \
    /* W4A16 decode GEMV, kernels/cuda/gemv_cuda.cu:213-260 */ X(gemv_forward_cuda)                                                 \
    /* fp16 host reference in the AWQ-GEMM layout, kernels/cuda/matmul_int4.cu:8-48 */ X(naive_mat_mul_fp16_int4)                    \
    /* fp32 C = A * B^T, kernels/cuda/matmul_ref_fp32.cc:11-34 */ X(mat_mul_accelerator_transposed_fastover_column)                  \
    /* empty in the reference CUDA build, gemv_cuda.cu:262-268 */ X(mat_mul_accelerator_int4_fast) X(mat_mul_accelerator_int4_fast_no_offset) \
    /* W8A8 family, kernels/ref/matmul_ref_int8.cc:11-192 */                                                                       \
    X(mat_mul_accelerator_int8_fast_2x2_32unroll) X(mat_mul_accelerator_int8_fast_32unroll_over_column)                              \
    X(mat_mul_accelerator_int8_fast_2x2_32unroll_nobias) X(mat_mul_accelerator_int8_fast_2x2_32unroll_nobias_batch)                  \
    X(mat_mul_accelerator_int8_fast_2x2_32unroll_nobias_ofp32) X(mat_mul_accelerator_int8_fast_2x2_32unroll_nobias_ofp32_batch)      \
    X(mat_mul_accelerator_int8_fast_2x2_32unroll_bfp32_ofp32) X(mat_mul_accelerator_int8_fast_2x2_32unroll_bfp32_ofp32_over_column)

// declared for source compatibility, defined outside this library (X: const params, Y: mutable params -- as in the reference)
#define TCE_MATMUL_OPS_ELSEWHERE(X, Y)                                                                                               \
    X(mat_mul_transposed) X(mat_mul_accelerator_transposed_fastover_column_bias) X(mat_mul_accelerator_untransposed_fastover_column) \
    X(naive_mat_mul_int8) X(naive_mat_mul_int4) X(naive_mat_mul_int4_with_offset) X(mat_mul_cuda)                                    \
    Y(mat_mul_accelerator_int8_int4_fast_no_offset) Y(gemv_accelerator_int8_int4_fast_no_offset)                                     \
    Y(gemm_accelerator_int8_int4_fast_no_offset) Y(gemm_accelerator_int8_int4_fast_no_offset_v2) Y(cblas_gemm_accelerator_no_offset)

struct thread_args {  // kernels/matmul.h:94-101 (CPU worker-thread argument block; unused by the CUDA backend)
    const struct matrix *A, *B, *C;
    const struct matmul_params *params;
    int start_i, end_i, blk_size;
};

class MatmulOperator {  // stateless, constructed per call by the reference's wrappers
   public:
#define TCE_DECLARE_OP(name) void name(const struct matmul_params *params);
#define TCE_DECLARE_OP_MUT(name) void name(struct matmul_params *params);
    TCE_MATMUL_OPS(TCE_DECLARE_OP)
    TCE_MATMUL_OPS_ELSEWHERE(TCE_DECLARE_OP, TCE_DECLARE_OP_MUT)
#undef TCE_DECLARE_OP
#undef TCE_DECLARE_OP_MUT
    // the prefill GEMM slot (kernels/matmul.h:142-145: declared, never defined by the reference): wgmma GEMM for M >= 16
    void gemm_forward_cuda(const struct matmul_params *params, int split_k_iters);
    void gemm_forward_cuda_8splits(const struct matmul_params *params, float16_t *split_8_buffer);
    void gemm_forward_cuda_half(const struct matmul_params *params, int split_k_iters);
    void gemm_forward_cuda_half_test(const struct matmul_params *params, int split_k_iters);

   private:  // kernels/matmul.h:149-153
    float interval_to_us(struct timeval *start, struct timeval *end);
    void CHECK_MATRICES(const struct matrix *A, const struct matrix *B, const struct matrix *C);
    void CHECK_MATRICES_int4weight(const struct matrix *A, const struct matrix *B, const struct matrix *C);
};

}  // namespace matmul

// Library-wide context used by the adapters: device 0, the legacy default stream (the reference launches every kernel on stream 0
// and relies on in-order semantics, SURVEY.md 8(b) Threading).  tce_host_set_stream() moves it.
struct tce_ctx;
extern "C" tce_ctx *tce_host_ctx(void);
extern "C" void tce_host_set_stream(void *cuda_stream);

#endif
