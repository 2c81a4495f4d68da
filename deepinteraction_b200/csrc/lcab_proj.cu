// The five 1x1 Conv(+folded BN)+ReLU projections of LocalContextAttentionBlock
// (reference projects/mmdet3d_plugin/models/utils/encoder_utils.py:92-131: query_project = 2 layers on the target map,
// key_project = 2 layers and value_project = 1 layer on the source map):
//
//     q = relu(W_q2 relu(W_q1 x_t + b_q1) + b_q2)      k = relu(W_k2 relu(W_k1 x_s + b_k1) + b_k2)      v = relu(W_v x_s + b_v)
//
// written directly in the planar bf16 hi|mid operand format of the window kernel (di_lcab_window_tc_f32), as a chain of
// five launches of the bf16-split tensor-core GEMM (gemm_tc.cu).  Each layer is the same launch the unfused chain makes,
// so results equal the unfused path bit for bit.  The first-stage activations q1 / k1 are written into the q / k output
// buffers and the second stage runs IN PLACE over them: with N = 128 there is one column tile, and a CTA has read all
// A rows of a tile (every K chunk) before its epilogue writes that tile's rows, while no other CTA touches those rows.
#include "common.cuh"
#include "di_b200.h"

extern "C" {

// x_t / x_s [M, 128] fp32 rows (leading dimensions ld_t / ld_s; x_s == x_t for self attention).
// W1_hi / W1_mid [384, 128] bf16 = rows (q1 | k1 | v), b1 [384]; W2_hi / W2_mid [256, 128] = rows (q2 | k2), b2 [256]
// (BN folded; hi = bf16(W), mid = bf16(W - hi)).  q, k, v: [M, 128] 32-bit words each (contiguous), planar operands
// of di_lcab_window_tc_f32.  C = 128 only.
int di_lcab_proj_f32(const float* x_t, int ld_t, const float* x_s, int ld_s, const void* W1_hi, const void* W1_mid,
                     const float* b1, const void* W2_hi, const void* W2_mid, const float* b2, float* q, float* k, float* v,
                     int M, cudaStream_t stream) {
  DI_CHECK_ARG(x_t && x_s && W1_hi && W1_mid && b1 && W2_hi && W2_mid && b2 && q && k && v && M > 0, "di_lcab_proj_f32: bad argument");
  DI_CHECK_ARG(ld_t % 4 == 0 && ld_s % 4 == 0 && ld_t >= 128 && ld_s >= 128, "di_lcab_proj_f32: leading dimensions");
  DI_CHECK_ARG((((uintptr_t)x_t | (uintptr_t)x_s | (uintptr_t)W1_hi | (uintptr_t)W1_mid | (uintptr_t)W2_hi | (uintptr_t)W2_mid |
                 (uintptr_t)q | (uintptr_t)k | (uintptr_t)v) & 15) == 0, "di_lcab_proj_f32: pointers must be 16-byte aligned");
  DI_CHECK_ARG(q != k && q != v && k != v, "di_lcab_proj_f32: q, k, v must be distinct buffers");
  constexpr size_t WB = 128 * 128 * 2;               // bytes of one 128 x 128 bf16 weight block
  auto w = [&](const void* p, int blk) { return static_cast<const void*>(static_cast<const char*>(p) + blk * WB); };
  struct Layer {
    const float* a; int lda; const void* wh; const void* wm; const float* b; float* out; int kind;
  };
  const Layer chain[5] = {
      {x_t, ld_t, w(W1_hi, 0), w(W1_mid, 0), b1, q, 0},            // q1 = relu(W_q1 x_t + b_q1)  -> q (fp32)
      {q, 128, w(W2_hi, 0), w(W2_mid, 0), b2, q, 3},               // q  = relu(W_q2 q1 + b_q2)   -> q (planar, in place)
      {x_s, ld_s, w(W1_hi, 1), w(W1_mid, 1), b1 + 128, k, 0},      // k1 = relu(W_k1 x_s + b_k1)  -> k (fp32)
      {k, 128, w(W2_hi, 1), w(W2_mid, 1), b2 + 128, k, 3},         // k  = relu(W_k2 k1 + b_k2)   -> k (planar, in place)
      {x_s, ld_s, w(W1_hi, 2), w(W1_mid, 2), b1 + 256, v, 3},      // v  = relu(W_v x_s + b_v)    -> v (planar)
  };
  for (const Layer& l : chain) {
    const int rc = di_linear_tcb_split_f32(l.a, l.lda, 128, nullptr, 0, 0, nullptr, 0, 0, l.wh, l.wm, l.b, nullptr, 0, 0,
                                           l.out, 128, M, 128, DI_ACT_RELU, 0, l.kind, stream);
    if (rc != DI_OK) return rc;
  }
  return DI_OK;
}

// LocalContextAttentionBlock.forward (models/utils/encoder_utils.py:119-135) for C = 128 as ONE call: the projection chain
// (di_lcab_proj_f32) followed by the window kernel (di_lcab_window_tc_f32) on `stream`.  x_t / x_s [N*H*W, 128]
// fp32 pixel-major rows (x_s == x_t: self attention), folded weights as for di_lcab_proj_f32, qkv: workspace of
// 3 * N*H*W * 128 32-bit words (16-byte aligned), out [N*H*W, ldo] fp32.  This is the entry SURVEY.md 8(b) calls
// `di_lcab_forward`: module-boundary traffic = x_t (+ x_s) read once, out written once; q / k / v pass through `qkv` (L2).
int di_lcab_window_tc_f32(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv, float* out, int ldo, int N,
                          int H, int W, int C, cudaStream_t stream);
int di_lcab_forward_f32(const float* x_t, int ld_t, const float* x_s, int ld_s, const void* W1_hi, const void* W1_mid,
                        const float* b1, const void* W2_hi, const void* W2_mid, const float* b2, float* qkv, float* out, int ldo,
                        int N, int H, int W, cudaStream_t stream) {
  DI_CHECK_ARG(qkv && out && N > 0 && H > 0 && W > 0, "di_lcab_forward_f32: bad argument");
  const size_t M = (size_t)N * H * W;
  float* q = qkv;
  float* k = qkv + M * 128;
  float* v = qkv + 2 * M * 128;
  const int rc = di_lcab_proj_f32(x_t, ld_t, x_s, ld_s, W1_hi, W1_mid, b1, W2_hi, W2_mid, b2, q, k, v, (int)M, stream);
  if (rc != DI_OK) return rc;
  return di_lcab_window_tc_f32(q, 128, k, 128, v, 128, out, ldo, N, H, W, 128, stream);
}

}  // extern "C"
