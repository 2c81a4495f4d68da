/* libdi_b200 -- C ABI of the H100-native (sm_90a) kernels for DeepInteraction's MMRI encoder +
 * MMPI decoder forward path.
 *
 * Conventions (every entry point):
 *   - plain C types only: device pointers, sizes, a cudaStream_t; no torch / C++ types;
 *   - returns int: 0 (or a non-negative count where stated) on success, < 0 on error
 *     (-1 bad argument, -2 launch failure, -3 unsupported configuration); the message is in
 *     di_last_error() (thread-local);
 *   - never allocates, never synchronises, never throws: launches on `stream` and returns;
 *     the caller owns all buffers (inputs are borrowed, outputs/workspaces are caller-provided);
 *   - stateless and re-entrant; distinct streams may be driven from distinct host threads.
 *   - fp32 in / fp32 out / fp32 accumulate.  Feature maps are "pixel-major" (NHWC): the C channels
 *     of one pixel are contiguous; query tensors are row-major [B*P, C].
 *
 * The reference has exactly one native boundary on this path, the pybind module `localattention`
 * (projects/mmdet3d_plugin/models/utils/ops/locatt_ops/localAttention.cpp:61-73; callers
 * models/utils/encoder_utils.py:43,67).  di_lcab_window_f32 replaces its similar_forward +
 * softmax + weighting_forward sequence; the other entry points replace the torch / detectron2 / OpenCV
 * calls of the surrounding Python (cited per function, paths relative to
 * projects/mmdet3d_plugin/).  INTEGRATION.md shows the reference-side binding.
 */
#ifndef DI_B200_H_
#define DI_B200_H_

#include <cuda_runtime_api.h>

#ifdef __cplusplus
extern "C" {
#endif

const char* di_last_error(void);
int di_version(void);
int di_built_arch(void); /* 90 == sm_90a */

/* Activation codes */
#define DI_ACT_NONE 0
#define DI_ACT_RELU 1
#define DI_ACT_GELU 2

/* ---- dense layers (gemm.cu) ------------------------------------------------------------------ */

/* C[M,N] = act([A0|A1|A2][M,K0+K1+K2] * W[N,K0+K1+K2]^T + bias[N] + res[m % res_mod, N]).
 * Replaces every 1x1 Conv(+folded BN)(+ReLU) of the encoder (models/utils/encoder_utils.py:11-34,92-117),
 * the cat + 1x1 Conv+BN pairs (models/necks/deepinteraction_encoder.py:26-27,31-32; the K-concatenated
 * sources make the torch.cat implicit) and every nn.Linear / Conv1d(k=1) of the decoder
 * (models/utils/decoder_utils.py).  splits > 1 = deterministic split-K: partial s goes to
 * C + s*split_stride without bias/act; returns the number of partials written (reduce them with
 * di_rows_finish_f32). */
int di_linear_f32(const float* A0, int lda0, int K0, const float* A1, int lda1, int K1, const float* A2, int lda2,
                  int K2, const float* W, const float* bias, const float* res, int ldres, int res_mod, float* C,
                  int ldc, int M, int N, int act, int splits, long long split_stride, cudaStream_t stream);

/* 3x3 conv, stride 1, pad 1 (models/necks/deepinteraction_encoder.py:47-62,80-81 shared convs;
 * models/dense_heads/deepinteraction_decoder.py:83-101,223-224 heatmap heads).
 * x: NCHW (x_nhwc=0) or NHWC (1); w: [Cout][(ky*3+kx)*Cin + ci]; y: NHWC (y_nchw=0) or NCHW (1). */
int di_conv3x3_f32(const float* x, int x_nhwc, const float* w, const float* bias, float* y, int y_nchw, int N,
                   int Cin, int H, int W, int Cout, int act, cudaStream_t stream);

/* Tensor-core versions (gemm_tc.cu): error-compensated split products on warpgroup MMA (wgmma; A split in registers,
 * fp32 accumulators in registers), operands staged by TMA.  Two operand precisions:
 *   _tc_  : 3xTF32.     W_hi / W_lo  fp32 [N,K]: hi = tf32(W), lo = W - hi.             every K_s % 32 == 0
 *   _tcb_ : bf16 split. W_hi / W_mid bf16 [N,K]: hi = bf16(W), mid = bf16(W - hi).      every K_s % 64 == 0
 *           (16 mantissa bits, ~1e-5 per layer; half the tensor instructions and weight bytes -- the default)
 * Output width N % 4 == 0.  Return -3 (unsupported) when the shape/alignment constraints are not met; the caller then falls back
 * (tcb -> tc -> the FFMA entry point). */
int di_linear_tc_f32(const float* A0, int lda0, int K0, const float* A1, int lda1, int K1, const float* A2, int lda2,
                     int K2, const float* W_hi, const float* W_lo, const float* bias, const float* res, int ldres,
                     int res_mod, float* C, int ldc, int M, int N, int act, cudaStream_t stream);
int di_linear_tcb_f32(const float* A0, int lda0, int K0, const float* A1, int lda1, int K1, const float* A2, int lda2,
                      int K2, const void* W_hi, const void* W_mid, const float* bias, const float* res, int ldres,
                      int res_mod, float* C, int ldc, int M, int N, int act, cudaStream_t stream);
/* di_linear_tcb_f32 whose output columns >= split_col0 (a multiple of 32; N % 32 == 0) are written PRE-SPLIT for
 * di_lcab_window_pre_f32: each value keeps its 4 bytes and its position, but holds packed bf16x2 words
 * (hi = bf16(x), mid = bf16(x - hi)); split_kind 1 = Q/K layout (channel pair 2j,2j+1 -> words 2j = hi, 2j+1 = mid),
 * 2 = V layout (channel group of 8 -> 4 hi words | 4 mid words); split_kind 3 = PLANAR layout for
 * di_lcab_window_tc_f32 (split_col0 % 128 == 0, N % 128 == 0): every group of 128 channels becomes 64 words of bf16
 * hi followed by 64 words of bf16 mid, i.e. two bf16 planes per pixel.
 * Replaces the k/q/v projections of LocalContextAttentionBlock (models/utils/encoder_utils.py:95-131) when their
 * consumer is the window kernel. */
int di_linear_tcb_split_f32(const float* A0, int lda0, int K0, const float* A1, int lda1, int K1, const float* A2,
                            int lda2, int K2, const void* W_hi, const void* W_mid, const float* bias, const float* res,
                            int ldres, int res_mod, float* C, int ldc, int M, int N, int act, int split_col0,
                            int split_kind, cudaStream_t stream);
int di_conv3x3_tc_f32(const float* x, const float* w_hi, const float* w_lo, const float* bias, float* y, int N, int Cin,
                      int H, int W, int Cout, int act, cudaStream_t stream);
int di_conv3x3_tcb_f32(const float* x, const void* w_hi, const void* w_mid, const float* bias, float* y, int N, int Cin,
                       int H, int W, int Cout, int act, cudaStream_t stream);
/* the same two convolutions over an NCHW input x [N,Cin,H,W] (W % 4 == 0), output pixel-major: the encoder's
 * boundary tensors (deepinteraction_encoder.py:47-62) are consumed without a transposition pass */
int di_conv3x3_tc_nchw_f32(const float* x, const float* w_hi, const float* w_lo, const float* bias, float* y, int N,
                           int Cin, int H, int W, int Cout, int act, cudaStream_t stream);
int di_conv3x3_tcb_nchw_f32(const float* x, const void* w_hi, const void* w_mid, const float* bias, float* y, int N,
                            int Cin, int H, int W, int Cout, int act, cudaStream_t stream);

/* diagnostics: clock64 pipeline trace of CTA 0 of the next tensor-core launch (8 x 512 stamps) */
int di_tc_set_debug(int on);
int di_tc_set_mode(int mode); /* 3 = weights resident in shared memory when K <= 128 (default), 4 = always streamed */
int di_tc_set_sm_limit(int n); /* persistent tensor-core grids use at most n CTAs (0 = one per SM) */
int di_tc_debug_read(long long* host_buf);

/* ---- local-window attention (lcab.cu) ---------------------------------------------------------- */

/* out = weighting(v, softmax(similar(q, k) / sqrt(C))) over a ksize x ksize window, fused
 * (models/utils/encoder_utils.py:132-134; locatt_ops/kernels.cuh:4-80).  Out-of-image taps: logit 0
 * (kept in the softmax), value skipped.  q,k,v,out [N,H,W,*] with per-pixel strides ld*. */
int di_lcab_window_f32(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, float* out, int ldo,
                       int N, int H, int W, int C, int ksize, cudaStream_t stream);

/* Same op for q, k (kind 1) and v (kind 2) emitted pre-split by di_linear_tcb_split_f32: no conversion passes. */
int di_lcab_window_pre_f32(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, float* out, int ldo,
                           int N, int H, int W, int C, cudaStream_t stream);

/* The same op for PLANAR pre-split operands (split_kind 3 above; lcab.cu, bf16-split mma.sync tensor-core kernel on a
 * persistent grid of at most di_tc_set_sm_limit CTAs, operands loaded by TMA), bit-identical to di_lcab_window_pre_f32:
 * q, k, v -- [N*H*W] pixels with a stride of ld* 32-bit words, 128 bf16 hi | 128 bf16 mid per pixel;
 * out fp32 [N,H,W,ldo].  C must be 128 (returns -3 otherwise: use di_lcab_window_pre_f32 / di_lcab_window_f32).
 * Replaces similar_forward + softmax + weighting_forward (encoder_utils.py:132-134, localAttention.cpp:7-15,31-39). */
int di_lcab_window_tc_f32(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv, float* out, int ldo,
                          int N, int H, int W, int C, cudaStream_t stream);

/* The five 1x1 Conv(+folded BN)+ReLU projections of LocalContextAttentionBlock (models/utils/encoder_utils.py:92-131:
 * query_project 2 layers on the target map x_t, key_project 2 layers and value_project 1 layer on the source map x_s)
 * writing q, k, v in the planar operand format of di_lcab_window_tc_f32 (lcab_proj.cu).  By default ONE persistent
 * wgmma launch: each CTA has a Q, K or V role with that role's weights resident in shared memory, and the first-stage
 * activations q1 / k1 stay in registers (each x tile read from HBM once, q, k, v written once).  x_t / x_s [M,128] fp32
 * rows (x_s == x_t: self attention; ld >= 128, ld % 4 == 0); W1_hi / W1_mid [384,128] bf16 rows (q1 | k1 | v), b1 [384];
 * W2_hi / W2_mid [256,128] rows (q2 | k2), b2 [256]; q, k, v [M,128] words each (contiguous, distinct); 16-byte aligned
 * pointers.  Results equal the unfused di_linear_tcb_split_f32 chain bit for bit. */
int di_lcab_proj_f32(const float* x_t, int ld_t, const float* x_s, int ld_s, const void* W1_hi, const void* W1_mid,
                     const float* b1, const void* W2_hi, const void* W2_mid, const float* b2, float* q, float* k, float* v,
                     int M, cudaStream_t stream);
/* CTAs per role (Q, K, V) the fused kernel launches for M rows under the current SM budget (di_tc_set_sm_limit) */
int di_lcab_proj_grid(int M, int* nq, int* nk, int* nv);

/* LocalContextAttentionBlock.forward for C = 128 as one call = di_lcab_proj_f32 + di_lcab_window_tc_f32 on `stream`
 * (models/utils/encoder_utils.py:119-135; SURVEY.md 8(b) `di_lcab_forward`).  qkv: workspace of 3 * N*H*W * 128 words. */
int di_lcab_forward_f32(const float* x_t, int ld_t, const float* x_s, int ld_s, const void* W1_hi, const void* W1_mid,
                        const float* b1, const void* W2_hi, const void* W2_mid, const float* b2, float* qkv, float* out, int ldo,
                        int N, int H, int W, cudaStream_t stream);

/* test/diagnostic hook for di_lcab_window_f32: 0 = the bf16-split mma.sync kernel when ksize == 9 and C % 32 == 0,
 * else FFMA (default); 1 = always the FFMA kernel.  Other values are rejected. */
int di_set_window_ffma(int on);

/* The reference extension's own five entry points, unfused and NCHW, for drop-in compatibility
 * (locatt_ops/localAttention.cpp:61-73): similar_forward = cc2k(x_ori, x_loc); weighting_forward =
 * ck2c_ori(x, weight); similar_backward(is_ori) = ck2c_ori / ck2c_loc(x, grad); weighting_backward_ori =
 * ck2c_loc(weight-side); weighting_backward_weight = cc2k(x_ori, grad).  fp32 data, fp64 accumulate. */
int di_locatt_cc2k_f32(const float* x_ori, const float* x_loc, float* y, int N, int C, int H, int W, int kH, int kW,
                       cudaStream_t stream);
int di_locatt_ck2c_ori_f32(const float* x_loc, const float* wgt, float* y, int N, int C, int H, int W, int kH, int kW,
                           cudaStream_t stream);
int di_locatt_ck2c_loc_f32(const float* x_ori, const float* wgt, float* y, int N, int C, int H, int W, int kH, int kW,
                           cudaStream_t stream);

/* ---- geometry-driven gathers (geometry.cu) ------------------------------------------------------ */

/* rows[p,:] = map[coors[p] = (b,z,y,x)]  (models/utils/encoder_utils.py:313) */
/* n_dev (this and the next three entry points; may be NULL): device pointer to the LIVE element count when the arrays
 * are allocated at a capacity P / n -- min(capacity, *n_dev) elements are processed.  Launch configurations and
 * buffer addresses then do not depend on the per-frame pillar / point counts (shape-independent CUDA-graph replay). */
int di_gather_rows_f32(const float* map, const int* coors, float* rows, int P, int Y, int X, int C, const int* n_dev,
                       cudaStream_t stream);
/* map[coors[p]] = cnt[p] > 0 ? rows[p,:] : 0  (models/utils/encoder_utils.py:314-318) */
int di_scatter_rows_f32(const float* rows, const int* cnt, const int* coors, float* map, int P, int Y, int X, int C,
                        const int* n_dev, cudaStream_t stream);
/* Per pillar: project its <=T points to V cameras, strict in-image / z>1e-5 / point<num_points mask,
 * bilinear gather of the image feature, single-head softmax attention with the folded query qk
 * (models/utils/encoder_utils.py:270-316; fold: SURVEY.md section 0).  s_out = sum_j a_j k_j, cnt = #valid keys. */
int di_i2p_attend_f32(const float* qk, const float* pillars, const int* npts, const int* coors, const float* proj,
                      const float* img, float* s_out, int* cnt_out, int P, int T, int pdim, int V, int h, int w, int C,
                      int H_in, int W_in, const int* n_dev, cudaStream_t stream);
/* Sparse depth maps: keys[v,r,c] = max((point index+1)<<32 | depth bits)  (models/utils/encoder_utils.py:155-174) */
int di_depth_scatter(const float* pts, int stride, int n, const float* proj, unsigned long long* keys, int V, int h,
                     int w, int H_in, int W_in, const int* n_dev, cudaStream_t stream);
/* ip_basic fill_in_multiscale(extrapolate=False, blur_type='bilateral') on the GPU
 * (models/utils/ip_basic/depth_map_utils.py:134-287; called at models/utils/encoder_utils.py:175-182).
 * scratch: 3*n_img*h*w floats. */
int di_depth_complete(const unsigned long long* keys, float* scratch, float* dense, float* sparse_out, int n_img, int h,
                      int w, cudaStream_t stream);
/* Lift feature pixels to LiDAR space and record BEV sampling coordinates (models/utils/encoder_utils.py:183-194). */
int di_lift_grid(const float* depth, const float* i2l, float* grid_xy, int n_img, int h, int w, int H_in, int W_in,
                 int Yb, int Xb, const float* pc_range6_host, cudaStream_t stream);
/* warped = grid_sample(bev, grid) with the lift mask folded into the grid (models/utils/encoder_utils.py:195-196). */
int di_bev_sample_f32(const float* bev, const float* grid_xy, float* out, int B, int V, int hw, int Yb, int Xb, int C,
                      cudaStream_t stream);

/* ---- pillar generation (pillar.cu) ------------------------------------------------------------------- */

/* Raw points -> pts_metas {pillars, pillar_coors, pillars_num_points} on the GPU, the live pillar count left in device
 * memory: replaces the spconv 2.1.21 PointToVoxel wrapper of the reference for the 'pillar' voxelisation
 * (models/updated_modules/sparse_voxelize.py:9-60; models/detectors/deepinteraction.py:132-139,151-171).
 * cell = floor((xy - range_min) / cell_size) on a Y x X grid over range[0..1]..range[3..4], z strictly inside
 * (range[2], range[5]); a pillar keeps its T lowest-index points in index order, pillars are emitted sorted by
 * (b, y, x), coors = (b, 0, y, x) -- deterministic where spconv's hash insertion order is not.
 * pts_ptrs / n_caps / range: HOST arrays (B device pointers, B capacities, 6 floats); n_dev: device int32 [B] live point
 * counts or NULL; work: device int32 [4*B*Y*X + 1 + B*max(n_caps) + sum(n_caps)]; outputs at capacity `cap` rows. */
int di_pillarize_f32(const float* const* pts_ptrs, const int* n_caps, const int* n_dev, int B, int stride, int pdim,
                     int Y, int X, int T, const float* range, int* work, float* pillars, int* coors, int* npts,
                     int* n_pillars, int cap, cudaStream_t stream);

/* ---- ++ ("deformable") encoder, DeepInteraction++ (deform.cu) ------------------------------------------ */

/* Core of mmcv 1.3.18 MultiScaleDeformableAttention as the reference uses it (models/necks/fusion_transformerv4.py:
 * 169-177 self attention over the multi-scale maps, :226-238 MMRI_P2I over the warped BEV map): per query and head,
 * softmax over the L*P logits, sampling location = reference point (pixel centre of the Hq x Wq query grid, :129-138)
 * + offset / (W_l, H_l), bilinear zero-padded sampling of the projected value map, weighted sum.
 * value0 / value1 [B, H_l, W_l, 128]: projected value map of level 0 / 1 (shapes[2l], shapes[2l+1] = H_l, W_l);
 * raw [B*NQ, ld_raw]: 8*L*P*2 offsets (head, level, point, xy) then 8*L*P logits (= the outputs of the
 * sampling_offsets / attention_weights Linear layers, one fused GEMM); out [B*NQ, ldo].
 * Supported: 8 heads x 16 channels, P = 4, L in {1, 2} (the ++ config); -3 otherwise.  shapes: HOST array. */
int di_msdeform_f32(const float* value0, const float* value1, const float* raw, int ld_raw, float* out, int ldo, int B,
                    int NQ, int Hq, int Wq, int heads, int dim, int L, int P, const int* shapes, cudaStream_t stream);
/* out = a + scale[0] * b (DeepInteractionLayer's `self_feat + self.scale * query`, fusion_transformerv4.py:217);
 * scale is a device pointer (learned parameter); n % 4 == 0. */
int di_axpy_f32(const float* a, const float* b, const float* scale, float* out, long long n, cudaStream_t stream);
/* map[coors[p]] += rows[p,:] where cnt[p] > 0 (++ MMRI_I2P returns decorated + lidar_feat, fusion_transformerv4.py:364) */
int di_scatter_rows_add_f32(const float* rows, const int* cnt, const int* coors, float* map, int P, int Y, int X, int C,
                            const int* n_dev, cudaStream_t stream);

/* MMRI_I2P_Polar (models/necks/fusion_transformerv4.py:487-640).
 * di_polar_grid_f32: BEV pixel coordinates [BV,R,W,2] (input of di_bev_sample_f32) at which the ray queries are
 *   sampled (:551-577); cam [BV,26] = rows 0-1 of inverse(lidar2img) (8), camera centre xy (2), rows 0-1 of the forward
 *   augmentation affine (8), 8 unused; pc_range: host float[6].
 * di_add_rows_mod_f32: out[m] = x[m] + pos[m % mod] (sine position tables, :537-548,576,579).
 * di_seq_attn_f32: multi-head softmax attention over column sequences -- token t of sequence (g, w) is row
 *   (g*L + t)*Wn + w -- replacing the flash-attn calls of the polar decoder layer (:651-759), in fp32.
 * di_polar_gather_f32: decoded rays [B*V,R,W,128] -> BEV (:579-636): per cell and camera the mean over 10 heights of
 *   (projected pixel x, clamped radius), any-height visibility, bilinear gather, mean over the seeing cameras, + lidar. */
int di_polar_grid_f32(const float* cam, float* grid, int BV, int R, int W, int h_feat, float im_scale, float r0,
                      float r_step, const float* pc_range, int Yb, int Xb, cudaStream_t stream);
int di_add_rows_mod_f32(const float* x, const float* pos, float* out, long long M, int C, long long mod, cudaStream_t stream);
int di_seq_attn_f32(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, float* out, int ldo, int G,
                    int Wn, int Lq, int Lk, int heads, int dim, cudaStream_t stream);
int di_polar_gather_f32(const float* rays, const float* lidar, const float* proj, const float* undo, const float* camc,
                        float* out, int B, int V, int R, int W, int Y, int X, int C, int H_in, int W_in,
                        const float* pc_range, float r0, float r_count, cudaStream_t stream);

/* Backward of the ++ encoder's kernels (deform.cu).
 * di_msdeform_bwd_f32: gradient of di_msdeform_f32 (same inputs and configuration; -3 for the same unsupported ones):
 *   dout [B*NQ, ldo] -> d_raw [B*NQ, ld_draw] in raw's layout (written without atomics: the same bits on every call),
 *   d_value0 / d_value1 [B, H_l, W_l, 128] += value-map gradients (zero them first).
 * di_seq_attn_bwd_f32: gradient of di_seq_attn_f32 from its saved output out: dq, dk, dv written into row views
 *   (strides as the forward's); Lq <= 128 (-3 otherwise), any Lk; no atomics.
 * di_polar_gather_bwd_f32: d_rays [B*V, R, W, 128] += adjoint of di_polar_gather_f32 applied to d_out [B, Y, X, 128]
 *   (zero d_rays first; the residual's gradient is d_out).
 * di_axpy_bwd_f32: gradient of di_axpy_f32 w.r.t. b and scale: db = scale[0] dout, ds[0] = sum dout . b (device scalar);
 *   work: di_axpy_bwd_workspace() doubles; block partials in double, summed in a fixed order. */
int di_msdeform_bwd_f32(const float* value0, const float* value1, const float* raw, int ld_raw, const float* dout, int ldo,
                        float* d_raw, int ld_draw, float* d_value0, float* d_value1, int B, int NQ, int Hq, int Wq,
                        int heads, int dim, int L, int P, const int* shapes, cudaStream_t stream);
int di_seq_attn_bwd_f32(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, const float* out, int ldo,
                        const float* dout, int ldd, float* dq, int lddq, float* dk, int lddk, float* dv, int lddv, int G,
                        int Wn, int Lq, int Lk, int heads, int dim, cudaStream_t stream);
int di_polar_gather_bwd_f32(const float* d_out, const float* proj, const float* undo, const float* camc, float* d_rays, int B,
                            int V, int R, int W, int Y, int X, int C, int H_in, int W_in, const float* pc_range, float r0,
                            float r_count, cudaStream_t stream);
int di_axpy_bwd_workspace(void);
int di_axpy_bwd_f32(const float* dout, const float* b, const float* scale, float* db, float* ds, double* work, long long n,
                    cudaStream_t stream);

/* ---- decoder (decoder.cu) ------------------------------------------------------------------------ */

/* models/dense_heads/deepinteraction_decoder.py:225-239 */
int di_heatmap_nms_f32(const float* a, const float* b, int ld, float* out, float* dense_b, int B, int K, int H, int W,
                       int ks, int no_nms_class_mask, cudaStream_t stream);
/* :242 (argsort descending, first k).  scores [B,n] >= 0 -> idx [B,k], 0 < k <= min(n, 1024): descending score, ties
 * by ascending index however many tie at the cut, deterministic; every index is in [0, n).  work: float [2*B*slices*k]
 * (NULL / slices <= 1: one level; slices are at least k long, so their number may come out smaller). */
int di_topk_f32(const float* scores, int* idx, int B, int n, int k, void* work, int slices, cudaStream_t stream);
/* :243-253, :299 */
int di_query_init_f32(const float* feat, const int* top, const float* heat, const float* wce_t, const float* bce,
                      float* qfeat, float* qpos, int* labels, float* qscore, int B, int HW, int W, int C, int K, int P,
                      cudaStream_t stream);
/* its backward (:245-251, q0 = feat[b, pix] + class_encoding(one_hot(label))): dq [B*P, C] -> d_feat [B, HW, C] += the dq
 * rows at the selected pixels (proposals sharing a pixel summed in proposal order; other rows untouched), d_wce [C, K]
 * (class_encoding.weight [C, K, 1]) and d_bce [C] written, rows summed in order.  No atomics; P <= 8192. */
int di_query_init_bwd_f32(const float* dq, const int* top, const int* labels, float* d_feat, float* d_wce, float* d_bce, int B,
                          int HW, int C, int K, int P, cudaStream_t stream);
/* self-attention among the queries of a sample (models/utils/decoder_utils.py:95-99, :745, :826) */
int di_mha_small_f32(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, float* out, int ldo,
                     const int* onbits, const int* win, int B, int P, int heads, int head_dim, cudaStream_t stream);
/* its backward: dout -> dq, dk, dv rows [B*P, ldg]; work: float [2 * B * heads * P * P]; deterministic.  onbits / win: the
 * forward's optional group mask (both or neither): key j is visible to query i iff win[i] >= 0 and bit win[i] of onbits[j]
 * is set; a query with win < 0 gets dq = 0, a key no query sees dk = dv = 0, and the rows of masked pairs are not read. */
int di_mha_small_bwd_f32(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, const float* dout, int ldd,
                         float* dq, float* dk, float* dv, int ldg, float* work, const int* onbits, const int* win, int B, int P,
                         int heads, int head_dim, cudaStream_t stream);
/* query x BEV cross attention (models/utils/decoder_utils.py:101-103, 466-488) */
int di_cross_attn_f32(const float* q, const float* kv, float* part, float* out, int B, int P, int HW, int C, int heads,
                      int nsplit, cudaStream_t stream);
/* x = sum_s part[s] + bias + res; y = act(LayerNorm(x)); residual + LayerNorm steps of decoder_utils.py */
int di_rows_finish_f32(const float* part, int nsplit, long long split_stride, int ldp, const float* bias,
                       const float* res, int ldres, const float* gamma, const float* beta, float* out, int ldo,
                       const int* zero_if_neg, int M, int C, int act, float eps, cudaStream_t stream);
/* models/dense_heads/deepinteraction_decoder.py:265, :290-295 */
int di_pred_finish_f32(float* pred, float* qpos, const float* first, const int* win, int M, int NP,
                       cudaStream_t stream);
/* ++ decoder (models/dense_heads/deepinteractionplusplus_decoder.py:285-302): look-forward centre update, cumulative
 * on-image mask `keep` (int32 [M]), first-layer fallback at every layer */
int di_pred_finish_pp_f32(float* pred, float* qpos, float* look, const float* first, const int* win, int* keep,
                          int first_layer, int M, int NP, cudaStream_t stream);
/* V2 RCNN blocks (models/utils/decoder_utils.py:844-1089).  di_rcnn_leaders: first query of every (sample, view) group;
 * di_mha_small_rows_f32: the group self-attention for a list of (query row, group) pairs; di_take_rows_f32: row
 * gather; di_branch_mix_f32: out = main * scale + leader_self * self_scale (:987, :1085) */
int di_rcnn_leaders(const int* onbits, int* lead_row, int* lead_win, int B, int P, int V, cudaStream_t stream);
int di_mha_small_rows_f32(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, float* out, int ldo,
                          const int* onbits, const int* rows, const int* rwin, int R, int rows_per_b, int B, int P,
                          int heads, int head_dim, cudaStream_t stream);
int di_take_rows_f32(const float* src, int ld, const int* idx, float* out, int R, int C, cudaStream_t stream);
int di_branch_mix_f32(const float* a, const float* lead, const int* win, const float* scale, const float* self_scale,
                      float* out, int M, int C, int P, int V, int zero_off, cudaStream_t stream);
/* their backward.  di_mha_small_rows_bwd_f32: dout [R, ldd] -> dq [R, lddq] (rows[r] = -1: zero row), the key and value
 * gradients ADDED to dk / dv [B*P, ldg] (after di_mha_small_bwd_f32 has written the main attention's); work: float
 * [2 * B * heads * P * rows_per_b].  di_rows_scatter_add_f32: dst[idx[r]] += src[r], r ascending, idx[r] = -1 skipped (the
 * adjoint of di_take_rows_f32).  di_branch_mix_bwd_f32: da = scale * dout (0 on zeroed rows), dlead [M / P * V, C] =
 * self_scale * the sum of dout over each group's rows, d_scale / d_self_scale [1] in fixed-order two-level sums; work:
 * float [2 * M].  di_pred_finish_pp_bwd_f32: dpred [L, M, NP] and the per-layer keep [L, M] of di_pred_finish_pp_f32 ->
 * d_delta [L, M, NP] (each prediction head's output gradient), d_first [M, NP].  Deterministic, no atomics. */
int di_mha_small_rows_bwd_f32(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, const float* dout,
                              int ldd, float* dq, int lddq, float* dk, float* dv, int ldg, float* work, const int* onbits,
                              const int* rows, const int* rwin, int R, int rows_per_b, int B, int P, int heads, int head_dim,
                              cudaStream_t stream);
int di_rows_scatter_add_f32(const float* src, int lds, const int* idx, float* dst, int ldd, int R, int C, cudaStream_t stream);
int di_branch_mix_bwd_f32(const float* dout, const float* a, const float* lead, const int* win, const float* scale,
                          const float* self_scale, float* da, float* dlead, float* d_scale, float* d_self_scale, float* work,
                          int M, int C, int P, int V, int zero_off, cudaStream_t stream);
int di_pred_finish_pp_bwd_f32(const float* dpred, const int* keep, float* d_delta, float* d_first, int L, int M, int NP,
                              cudaStream_t stream);
/* box decode + RoI rectangles: image mode 0 (models/utils/decoder_utils.py:660-741), BEV mode 1 (:788-819);
 * core/bbox/coders/transfusion_bbox_coder.py:59-76 */
int di_rcnn_rois_f32(const float* pred, int NP, const float* proj, const float* aux, float* rois, int* win, int* onbits,
                     int B, int P, int V, int mode, const float* params10, cudaStream_t stream);
/* detectron2 ROIAlignV2 7x7, sampling_ratio 2 (models/utils/decoder_utils.py:641-646, 739-741, 769-774, 822-823) */
int di_roi_align_f32(const float* maps, const float* rois, float* out, int n, int H, int W, int C, float scale,
                     cudaStream_t stream);
/* DynamicConv bmm + LayerNorm + ReLU x2 (models/utils/decoder_utils.py:610-624) */
int di_dynconv_f32(const float* roi, const float* params, const float* g1, const float* b1, const float* g2,
                   const float* b2, float* out, int n, float eps, cudaStream_t stream);
/* layout converters for the NCHW drop-in boundary */
int di_nchw_to_nhwc_f32(const float* in, float* out, int N, int C, int HW, cudaStream_t stream);
int di_nhwc_to_nchw_f32(const float* in, float* out, int N, int C, int HW, cudaStream_t stream);

/* Query-row MLP: up to two chained dense layers, residual, LayerNorm and activation on M <= a few hundred rows in ONE
 * launch (4 rows per CTA, fp32 FFMA): Y = act_out(LN(act1([X0|X1] W1t + b1) [W2t + b2] + res)); rows with
 * zero_if_neg[m] < 0 are written as 0.  Replaces the nn.Linear / Conv1d(k=1) chains of models/utils/decoder_utils.py
 * (pos-embed MLPs :16-32, attention projections + norms :73-113, FFNs :104-109,754-757, prediction heads :498-581).
 * W1t [K0+K1, N1], W2t [N1, N2]: TRANSPOSED weights; W2t / b1 / b2 / res / gamma+beta / zero_if_neg may be NULL. */
int di_rows_mlp_f32(const float* X0, int ld0, int K0, const float* X1, int ld1, int K1, const float* W1t, const float* b1,
                    int N1, int act1, const float* W2t, const float* b2, int N2, const float* res, int ldres,
                    const float* gamma, const float* beta, float eps, int act_out, const int* zero_if_neg, float* Y, int ldy,
                    int M, cudaStream_t stream);

/* ---- box coder and get_bboxes post-processing (decoder.cu) ------------------------------------- */

/* TransFusionBBoxCoder.decode (core/bbox/coders/transfusion_bbox_coder.py:40-126): class = first arg-max of the
 * score over K, box = (x, y, z_bottom, dx, dy, dz, yaw[, vx, vy]); keep = centre inside range6 (host pointer to
 * post_center_range, or NULL) and, when use_thr, score > score_thr.  With qscore/qlabel the score is composed as in
 * DeepInteractionDecoder.get_bboxes (models/dense_heads/deepinteraction_decoder.py:561-563):
 * sigmoid(heat) * query_heatmap_score * one_hot(query_label).  Inputs contiguous [B,k,P]. */
int di_bbox_decode_f32(const float* heat, const float* qscore, const int* qlabel, const float* rot, const float* dim,
                       const float* center, const float* height, const float* vel, int B, int K, int P, float sx, float sy,
                       float ox, float oy, const float* range6, float score_thr, int use_thr, float* boxes, float* scores,
                       int* labels, unsigned char* keep, cudaStream_t stream);
/* TransFusionBBoxCoder.encode (transfusion_bbox_coder.py:24-38): boxes [n,7|9] -> targets [n,8|10]. */
int di_bbox_encode_f32(const float* boxes, int nb, float* targets, int code, int n, float sx, float sy, float ox, float oy,
                       cudaStream_t stream);
/* Per-task circle NMS of get_bboxes (deepinteraction_decoder.py:594-625; mmdet3d circle_nms semantics: greedy in
 * descending score, squared centre distance <= thresh suppresses, at most post_max kept).  keep_io [B,P] in place. */
int di_circle_nms_f32(const float* boxes, int nb, const float* scores, const int* labels, unsigned char* keep_io, int B,
                      int P, unsigned class_mask, float thresh, int post_max, cudaStream_t stream);

/* ---- MMPI loss path (SURVEY.md 8(f) rank 3) ------------------------------------------------------------------------
 * replaces core/bbox/assigners/hungarian_assigner.py:14-47 (match costs) + mmdet FocalLossCost + mmdet3d BboxOverlaps3D */
int di_match_cost_f32(const float* boxes, int nb, const float* score, int K, const float* gt, const int* gt_labels,
                      const int* n_gt, int B, int LP, int Gmax, const float* params11, float* cost, float* iou,
                      cudaStream_t stream);
/* hungarian_assigner.py:132-149 (scipy linear_sum_assignment on the CPU in the reference): one warp per (sample, layer) */
int di_hungarian_f32(const float* cost, const float* iou, const int* n_gt, int B, int L, int P, int Gmax, long long* gt_inds,
                     float* max_overlaps, cudaStream_t stream);
/* HeuristicAssigner3D.assign (hungarian_assigner.py:60-91); work: int32 [G] + float [G] */
int di_heuristic_assign_f32(const float* boxes, int nb, int P, const float* gt, const int* gt_labels, int G,
                            const int* query_labels, float dist_thre, long long* gt_inds, float* max_overlaps, float* labels,
                            void* work, cudaStream_t stream);
/* models/dense_heads/deepinteraction_decoder.py:400-441 (+ the on-image mask products of :501-509) */
int di_loss_targets_f32(const long long* gt_inds, const float* max_overlaps, const float* gt, const int* gt_labels, int Gmax,
                        const unsigned char* mask, int mask_mode, int B, int L, int P, int nb, int code, int num_classes,
                        float pos_weight, const float* coder4, long long* labels, long long* label_w, float* bbox_t,
                        float* bbox_w, float* ious, float* num_pos, float* iou_sum, int* pos_cnt, cudaStream_t stream);
/* deepinteraction_decoder.py:443-476 (gaussian_radius + draw_heatmap_gaussian per ground-truth box) */
int di_gaussian_heatmap_f32(const float* gt, int nb, const int* gt_labels, const int* n_gt, int B, int Gmax, int K, int Y, int X,
                            const float* params7, float* heat, cudaStream_t stream);
/* deepinteraction_decoder.py:511-545: GaussianFocalLoss(clip_sigmoid(dense_heatmap)), per layer FocalLoss + weighted L1 */
int di_mmpi_losses_f32(const float* dense_logit, const float* heat_target, long long n_heat, const float* score,
                       const float* center, const float* height, const float* dim, const float* rot, const float* vel,
                       const long long* labels, const long long* label_w, const float* bbox_t, const float* bbox_w,
                       const float* num_pos, const float* iou_sum, const int* pos_cnt, int B, int K, int L, int P, int code,
                       const float* code_w, const float* focal2, const float* gfl2, const float* weights3, double* work,
                       float* out, cudaStream_t stream);
/* its gradient for upstream grad [2 + 2 L] (device) on the outputs: d_heat [B, HW, 32] d loss / d dense logit, pixel-major,
 * channels K..31 zero (clip_sigmoid's clamp passes the gradient on [1e-4, 1 - 1e-4]); d_pred [L, B*P, code + K] d loss /
 * d prediction rows in head order (L1: sign, 0 at equality; focal: mmcv's closed form; rows of zero weight written 0).
 * Avg factors from the device; one thread per output element, no atomics.  work: double [2 * 256 + L * 2 * 64]. */
int di_mmpi_losses_bwd_f32(const float* dense_logit, const float* heat_target, long long n_heat, int HW, const float* score,
                           const float* center, const float* height, const float* dim, const float* rot, const float* vel,
                           const long long* labels, const long long* label_w, const float* bbox_t, const float* bbox_w,
                           const float* num_pos, int B, int K, int L, int P, int code, const float* code_w, const float* focal2,
                           const float* gfl2, const float* weights3, const float* grad, double* work, float* d_heat,
                           float* d_pred, cudaStream_t stream);

/* ---- backward of the window attention (SURVEY.md 8(b) `di_lcab_backward`; host composition: deepinteraction_b200/backward.py)
 * Pixel-major maps [N*H*W, ld]; tap j = (dy + r) * ks + (dx + r) (locatt_ops/similar.cu:15-17).
 * di_win_dot_f32     out[p, j] = a[p] . b[nbr(p, j)]          similar_forward / weighting_backward_weight (kernels.cuh:4-41, weighting.cu:83-121)
 * di_win_gather_f32  out[p]  = sum_j w[p, j] b[nbr(p, j)]       weighting_forward / similar_backward(is_ori)   (kernels.cuh:44-80)
 * di_win_scatter_f32 out[p'] = sum_{nbr(p,j)=p'} w[p, j] b[p]   similar_backward(!is_ori) / weighting_backward_ori (kernels.cuh:82-119) */
int di_win_dot_f32(const float* a, int lda, const float* b, int ldb, float* out, int N, int H, int W, int C, int ks,
                   cudaStream_t stream);
int di_win_gather_f32(const float* w, const float* b, int ldb, float* out, int ldo, int N, int H, int W, int C, int ks,
                      cudaStream_t stream);
int di_win_scatter_f32(const float* w, const float* b, int ldb, float* out, int ldo, int N, int H, int W, int C, int ks,
                       cudaStream_t stream);
/* softmax over the ks*ks taps (encoder_utils.py:133) and its backward */
int di_win_softmax_f32(const float* S, float* A, long long P, int KK, float scale, cudaStream_t stream);
int di_win_softmax_bwd_f32(const float* A, const float* dA, float* dS, long long P, int KK, float scale, cudaStream_t stream);
/* ReLU backward from the saved output; column sums of a [M, C] matrix (bias gradients; work: float [256 * C]) */
int di_relu_bwd_f32(const float* dy, const float* y, float* dx, long long n, cudaStream_t stream);
int di_col_sum_f32(const float* x, int ld, long long M, int C, float* work, float* out, cudaStream_t stream);
/* backward of y = LayerNorm(z) over [M, C] rows (z = the saved pre-norm sum): dz, dgamma, dbeta (fixed-order column sums);
 * work: float [M * C + 256 * C] */
int di_ln_bwd_f32(const float* dy, int ldy, const float* z, int ldz, const float* gamma, float* dz, int lddz, float* dgamma,
                  float* dbeta, float* work, int M, int C, float eps, cudaStream_t stream);
/* zero-filled shift of a pixel-major map (weight gradient of the 3x3 shared convolutions) */
int di_shift_map_f32(const float* in, float* out, int N, int H, int W, int C, int dy, int dx, cudaStream_t stream);

/* ---- train-mode BatchNorm over pixel-major rows (csrc/bn_train.cu) -------------------------------------------------------
 * models/utils/encoder_utils.py:11-34 (ConvBNReLU with nn.BatchNorm2d in training mode; every norm of the encoder follows a
 * 1x1 convolution, so its input is a [M = N*H*W, C] row matrix).  di_bn_stats_f32: batch mean / biased variance, optional
 * in-place update of the running statistics (momentum, unbiased variance); work: float [592 * C * 3].
 * di_bn_apply_f32: z = act((y - mean) / sqrt(var + eps) * gamma + beta), gamma / beta NULL = affine=False.
 * di_bn_bwd_f32: dz, saved z (NULL = no ReLU), saved y -> dy, dgamma, dbeta incl. the gradient through the batch
 * statistics; work: float [592 * C * 2]. */
int di_bn_stats_f32(const float* y, long long M, int C, float* work, float* mean, float* var, float* run_mean, float* run_var,
                    float momentum, cudaStream_t stream);
int di_bn_apply_f32(const float* y, long long M, int C, const float* mean, const float* var, const float* gamma, const float* beta,
                    float eps, int relu, float* z, cudaStream_t stream);
int di_bn_bwd_f32(const float* dz, const float* z, const float* y, long long M, int C, const float* mean, const float* var,
                  const float* gamma, float eps, float* work, float* dy, float* dgamma, float* dbeta, cudaStream_t stream);

/* ---- I2P backward (SURVEY.md 8(b) `di_i2p_backward`; host composition: deepinteraction_b200/backward.py i2p_backward)
 * gradient of di_i2p_attend_f32 (models/utils/encoder_utils.py:281-311): ds [P,C] -> dqk [P,C], d_img += (atomic) */
int di_i2p_attend_bwd_f32(const float* qk, const float* ds, const float* pillars, const int* npts, const int* coors,
                          const float* proj, const float* img, float* d_img, float* dqk, int P, int T, int pdim, int V, int h,
                          int w, int C, int H_in, int W_in, const int* n_dev, cudaStream_t stream);
/* Training-mode variants with the attention dropout of nn.MultiheadAttention (encoder_utils.py:223; the softmax weights times
 * keep / (1 - pdrop), keep = counter-based hash of (seed, pillar, key index), regenerated in the backward);
 * s_out / ds are [P, C + 4]: column C carries rho = sum_j a_j m_j (the weights no longer sum to 1 and the value bias of the
 * attention is weighted by that sum) resp. its gradient.  di_i2p_dropout_mask_f32 writes the factors [P, S = T*V] (tests). */
int di_i2p_attend_dropout_f32(const float* qk, const float* pillars, const int* npts, const int* coors, const float* proj,
                              const float* img, float* s_out, int* cnt_out, int P, int T, int pdim, int V, int h, int w, int C,
                              int H_in, int W_in, const int* n_dev, float pdrop, unsigned int seed, cudaStream_t stream);
int di_i2p_attend_bwd_dropout_f32(const float* qk, const float* ds, const float* pillars, const int* npts, const int* coors,
                                  const float* proj, const float* img, float* d_img, float* dqk, int P, int T, int pdim, int V,
                                  int h, int w, int C, int H_in, int W_in, const int* n_dev, float pdrop, unsigned int seed,
                                  cudaStream_t stream);
int di_i2p_dropout_mask_f32(float* mask, int P, int S, float pdrop, unsigned int seed, cudaStream_t stream);
/* backward of di_bev_sample_f32 w.r.t. the BEV map (encoder_utils.py:193-195 grid_sample): d_bev += bilinear scatter */
int di_bev_sample_bwd_f32(const float* d_out, const float* grid_xy, float* d_bev, int B, int V, int hw, int Yb, int Xb, int C,
                          cudaStream_t stream);
int di_gather_rows_masked_f32(const float* map, const int* cnt, const int* coors, float* rows, int P, int Y, int X, int C,
                              cudaStream_t stream);

/* ---- query x BEV cross attention on the tensor cores, mma.sync bf16 split (models/utils/decoder_utils.py:101-103, 466-493; xattn_tc.cu)
 * di_attn_planes_f32: fp32 rows -> bf16 operand planes (queries, pre-scaled by head_dim^-0.5, and keys: hi | mid | lo = 192
 * words per row; values: hi | mid = 128 words); either input may be NULL.  di_xattn_tc_f32: part = float workspace of
 * B * heads * di_xattn_tc_splits(B, HW) * 18 * P; out [B*P, 128] fp32.  8 heads x 16 channels, P <= 256 (returns -3
 * otherwise: use di_cross_attn_f32). */
int di_attn_planes_f32(const float* q, int ld_q, void* qplanes, int M, const float* kv, int ld_kv, void* kplanes,
                       void* vplanes, long long Mk, cudaStream_t stream);
int di_xattn_tc_splits(int B, int HW);
int di_xattn_tc_f32(const void* q, const void* k, const void* v, float* part, float* out, int B, int P, int HW, int heads,
                    cudaStream_t stream);
/* di_xattn_tc_lse_f32: the same kernels, plus lse [B, heads, P] = the row log-sum-exp of the logits (from the split merge);
 * out is bit-identical to di_xattn_tc_f32's. */
int di_xattn_tc_lse_f32(const void* q, const void* k, const void* v, float* part, float* out, float* lse, int B, int P,
                        int HW, int heads, cudaStream_t stream);
/* ---- backward of the query x BEV cross attention (xattn_bwd.cu): mma.sync bf16 split on the operand planes, key splits with
 * dK / dV written once per key and per-split dQ partials merged in a fixed order (no atomics; deterministic).
 * q / k / v: planes of di_attn_planes_f32; out, lse: outputs of di_xattn_tc_lse_f32; dout [B*P, ld_dout] -> dq [B*P, 128]
 * (w.r.t. the pre-scaled queries), dk / dv rows [B*HW, ld_dkv]; work: di_xattn_bwd_workspace(B, P, HW) floats.  8 heads x 16
 * channels, P <= 256. */
int di_xattn_bwd_workspace(int B, int P, int HW);
int di_xattn_bwd_f32(const void* q, const void* k, const void* v, const float* out, const float* dout, int ld_dout,
                     const float* lse, float* work, float* dq, float* dk, float* dv, int ld_dkv, int B, int P, int HW,
                     int heads, cudaStream_t stream);

/* ---- backward of the RCNN blocks' kernels (decoder.cu; host composition: backward.py point_rcnn_backward)
 * di_roi_align_bwd_f32: gradient of di_roi_align_f32 w.r.t. the maps.  rois [n, 5] and scale as in the forward (map index < 0
 * or >= n_maps: no contribution), d_out [n, 49, C] -> d_maps [n_maps, H, W, C], every pixel written (exactly 0 where no
 * sample reaches: no memset needed).  Same skip, clamp and last-pixel rules as the forward.  A gather over pixel tiles,
 * RoIs summed in ascending index: deterministic, no atomics, no workspace.  n >= 0, C % 4 == 0, C <= 512, d_out and d_maps
 * 16-byte aligned.
 * di_dynconv_bwd_f32: gradient of di_dynconv_f32.  roi [n, 49, 128], params [n, 2*128*128], g1, b1, g2, b2 [128], d_out
 * [n, 49*128] -> d_roi [n, 49, 128], d_params [n, 2*128*128] (P1 then P2, [c][d], as params), d_norm [n, 4*128] = per-query
 * partials of dgamma1 | dbeta1 | dgamma2 | dbeta2 (reduce over n with di_col_sum_f32).  One CTA per query recomputes the
 * forward in shared memory (231 424 B of dynamic shared memory); no workspace, deterministic, no atomics.  roi, params,
 * d_out, d_params and the norm vectors 16-byte aligned.
 * di_gelu_bwd_f32: dx = dy (Phi(h) + h phi(h)), the derivative of the exact (erf) GELU at the pre-activation h; n elements. */
int di_roi_align_bwd_f32(const float* rois, const float* d_out, float* d_maps, int n, int n_maps, int H, int W, int C,
                         float scale, cudaStream_t stream);
int di_dynconv_bwd_f32(const float* roi, const float* params, const float* g1, const float* b1, const float* g2, const float* b2,
                       const float* d_out, float* d_roi, float* d_params, float* d_norm, int n, float eps, cudaStream_t stream);
int di_gelu_bwd_f32(const float* dy, const float* h, float* dx, long long n, cudaStream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* DI_B200_H_ */
