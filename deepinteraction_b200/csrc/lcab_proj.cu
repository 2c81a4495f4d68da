// The five 1x1 Conv(+folded BN)+ReLU projections of LocalContextAttentionBlock
// (reference projects/mmdet3d_plugin/models/utils/encoder_utils.py:92-131: query_project = 2 layers on the target map,
// key_project = 2 layers and value_project = 1 layer on the source map):
//
//     q = relu(W_q2 relu(W_q1 x_t + b_q1) + b_q2)      k = relu(W_k2 relu(W_k1 x_s + b_k1) + b_k2)      v = relu(W_v x_s + b_v)
//
// written directly in the planar bf16 hi|mid operand format of the window kernel (di_lcab_window_tc_f32).
//
// Fused kernel (default): one persistent launch.  Each CTA has one role for its lifetime -- Q (x_t -> q1 -> q),
// K (x_s -> k1 -> k) or V (x_s -> v) -- and keeps that role's weights (bf16 hi + mid, 128 KB for Q / K, 64 KB for V)
// resident in shared memory; the grid is split between the roles by the time a work item of each takes (role_split).
// All roles walk the 64-row work items in the same order, so the K and V (and, for self attention, Q) reads of an x
// tile after the first are mostly L2 hits.  The chained layer never leaves registers: the m64n128 accumulator fragment
// a warp holds after layer 1 (bias, ReLU) is split into bf16 hi / mid and is exactly the A fragment of layer 2, so
// q1 / k1 are never stored.  Warpgroup 0 is the TMA producer (one thread); warpgroups 1 and 2 each own whole 64-row
// items (alternating) and take turns on the tensor cores, so one warpgroup's epilogue runs under the other's MMA.  The
// epilogue writes the output words into the item's own x stage (128-byte swizzle) and one thread stores the tile by
// TMA.  Every layer issues the same k-steps with the same three split products in the same order as the bf16-split
// GEMM (gemm_tc.cu), and the stored words are the same, so the results equal the five layers run as separate
// di_linear_tcb_split_f32 launches bit for bit (tests/lcab_chain.py).
#include "tc_common.cuh"
#include "di_b200.h"

namespace {

using namespace tc;

constexpr int PJ_ROWS = 64;                          // rows per work item (one consumer warpgroup)
constexpr int PJ_BOX = PJ_ROWS * 32 * 4;             // 8 KB: 64 rows x 32 words (one 128-byte swizzle row each)
constexpr int PJ_STAGE = 4 * PJ_BOX;                 // 32 KB: the 64 x 128 fp32 x tile of one item, then its output
constexpr int PJ_WBOX = 128 * 64 * 2;                // 16 KB: 128 rows x 64 bf16 of a weight
constexpr int PJ_W_BYTES = 8 * PJ_WBOX;              // W1 hi | W1 mid | W2 hi | W2 mid of one role (2 boxes each)
constexpr int PJ_POOL = PJ_W_BYTES + 3 * PJ_STAGE;   // weights + ring: Q / K hold 3 stages, V (half the weights) 5
constexpr int PJ_MAX_S = 5;
constexpr int PJ_BAR_BYTES = 128;
constexpr int PJ_SMEM_BYTES = PJ_POOL + 1024 /*alignment*/ + PJ_BAR_BYTES;
constexpr int PJ_THREADS = 384;
static_assert(PJ_SMEM_BYTES <= 232448, "lcab_proj exceeds the 227 KB shared-memory limit");
static_assert(PJ_W_BYTES / 2 + PJ_MAX_S * PJ_STAGE <= PJ_POOL, "V ring overflow");
static_assert(8 * (2 * PJ_MAX_S + 1) <= PJ_BAR_BYTES, "barrier block overflow");

struct ProjParams {
  const float* b1;          // [384] = b_q1 | b_k1 | b_v
  const float* b2;          // [256] = b_q2 | b_k2
  int M, items;             // rows, 64-row work items
  int nq, nk, nv;           // CTAs per role (blocks [0, nq) = Q, [nq, nq + nk) = K, the rest = V)
};

// 24 wgmma (8 k-steps x 3 split products) of one 64 x 128 x 128 layer, in the order of gemm_tc_kernel_v3<.., BF = true>
__device__ __forceinline__ void layer_mma(float (&acc)[64], const uint32_t (&ahi)[8][4], const uint32_t (&amid)[8][4],
                                          uint32_t whi, uint32_t wmid) {
  fence_regs(acc);
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < 8; ++ks) {
    const uint32_t off = (ks >> 2) * PJ_WBOX + (ks & 3) * 32;
    const uint64_t w_hi = wgmma_desc(whi + off), w_mid = wgmma_desc(wmid + off);
    wgmma_bf16_rs(acc, amid[ks], w_hi, ks != 0);     // A_mid * W_hi
    wgmma_bf16_rs(acc, ahi[ks], w_mid, 1);           // A_hi * W_mid
    wgmma_bf16_rs(acc, ahi[ks], w_hi, 1);            // A_hi * W_hi
  }
  wgmma_commit();
  wgmma_wait_all();
  fence_regs(acc);
}

__device__ __forceinline__ void split_pair(float x0, float x1, uint32_t& hi, uint32_t& mid) {
  hi = pack_bf16x2(x0, x1);
  mid = pack_bf16x2(x0 - __uint_as_float(hi << 16), x1 - __uint_as_float(hi & 0xFFFF0000u));
}

// acc = relu(acc + bias); acc[4j + 2h + e] is (row r0 + 8h, column 8j + 2t + e) of the warp's 16 rows
__device__ __forceinline__ void bias_relu(float (&acc)[64], const float* bias, int t) {
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const float2 b = *reinterpret_cast<const float2*>(bias + 8 * j + 2 * t);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      acc[4 * j + 2 * h] += b.x;
      acc[4 * j + 2 * h + 1] += b.y;
    }
  }
#pragma unroll
  for (int j = 0; j < 64; ++j) acc[j] = fmaxf(acc[j], 0.f);
}

__global__ void __launch_bounds__(PJ_THREADS, 1)
lcab_proj_kernel(const __grid_constant__ CUtensorMap mapXt, const __grid_constant__ CUtensorMap mapXs,
                 const __grid_constant__ CUtensorMap mapW1h, const __grid_constant__ CUtensorMap mapW1m,
                 const __grid_constant__ CUtensorMap mapW2h, const __grid_constant__ CUtensorMap mapW2m,
                 const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                 const __grid_constant__ CUtensorMap mapV, const ProjParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* const base_ptr = smem_raw + (base - smem_u32(smem_raw));
  const uint32_t bars = base + PJ_POOL;
  auto full = [&](int s) { return bars + 8u * s; };
  auto empty = [&](int s) { return bars + 8u * (PJ_MAX_S + s); };
  const uint32_t w_full = bars + 8u * (2 * PJ_MAX_S);

  const int bid = blockIdx.x;
  const int role = bid < p.nq ? 0 : (bid < p.nq + p.nk ? 1 : 2);        // 0 = Q, 1 = K, 2 = V
  const int first = role == 0 ? bid : (role == 1 ? bid - p.nq : bid - p.nq - p.nk);
  const int stride = role == 0 ? p.nq : (role == 1 ? p.nk : p.nv);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // the x ring follows this role's weights: 3 stages for Q / K, 5 for V
  const uint32_t ring_off = role == 2 ? PJ_W_BYTES / 2 : PJ_W_BYTES;
  const int S = (PJ_POOL - (int)ring_off) / PJ_STAGE;

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(full(s), 1);
      mbar_init(empty(s), 1);                        // the consuming warpgroup's storing thread
    }
    mbar_init(w_full, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    // ---------------- TMA producer (one thread) ----------------
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      const int wrow = role * 128;                   // this role's 128 output channels in W1 / W2
      mbar_expect_tx(w_full, (role == 2 ? 4 : 8) * PJ_WBOX);
      for (int kc = 0; kc < 2; ++kc) {
        tma_load_2d(base + kc * PJ_WBOX, &mapW1h, w_full, kc * 64, wrow);
        tma_load_2d(base + (2 + kc) * PJ_WBOX, &mapW1m, w_full, kc * 64, wrow);
        if (role != 2) {
          tma_load_2d(base + (4 + kc) * PJ_WBOX, &mapW2h, w_full, kc * 64, wrow);
          tma_load_2d(base + (6 + kc) * PJ_WBOX, &mapW2m, w_full, kc * 64, wrow);
        }
      }
      const CUtensorMap* mx = role == 0 ? &mapXt : &mapXs;
      int n = 0;
      for (int item = first; item < p.items; item += stride, ++n) {
        const int s = n % S;
        if (n >= S) mbar_wait(empty(s), ((n / S) - 1) & 1);
        const uint32_t st = base + ring_off + s * PJ_STAGE;
        mbar_expect_tx(full(s), PJ_STAGE);
        for (int b = 0; b < 4; ++b) tma_load_2d(st + b * PJ_BOX, mx, full(s), 32 * b, item * PJ_ROWS);
        const int ahead = item + S * stride;         // the item this stage is loaded with next: L2 prefetch
        if (ahead < p.items)
          for (int b = 0; b < 4; ++b) tma_prefetch_2d(mx, 32 * b, ahead * PJ_ROWS);
      }
    }
  } else {
    // ---------------- consumers: warpgroup 1 takes the CTA's even items, warpgroup 2 the odd ones ----------------
    // The CTA's items take turns in order: a warpgroup waits for its stage, converts it and runs its MMA only after
    // the other warpgroup has done so for the previous item (named barrier 1 + wg), so one warpgroup's epilogue and
    // stores run under the other's MMA.  The turn order also keeps every wait on a stage's `full` barrier at most one
    // phase ahead of it, which a parity wait needs when two warpgroups share one ring.
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int wg = (warp >> 2) - 1, wl = warp & 3;
    const int g = lane >> 2, t = lane & 3;
    const int r0 = wl * 16 + g, r1 = r0 + 8;         // item rows of this thread's fragments (row & 7 == g)
    const bool storer = (threadIdx.x & 127) == 0;
    const uint32_t w1h = base, w1m = base + 2 * PJ_WBOX, w2h = base + 4 * PJ_WBOX, w2m = base + 6 * PJ_WBOX;
    const float* b1 = p.b1 + role * 128;
    const float* b2 = p.b2 + role * 128;
    const CUtensorMap* mo = role == 0 ? &mapQ : (role == 1 ? &mapK : &mapV);
    const int n_items = first < p.items ? (p.items - 1 - first) / stride + 1 : 0;   // items of this CTA
    mbar_wait(w_full, 0);
    float acc[64];
    uint32_t ahi[8][4], amid[8][4];
    int n = wg;
    for (int item = first + wg * stride; item < p.items; item += 2 * stride, n += 2) {
      const int s = n % S;
      if (n > 0) bar_sync(1 + wg, 256);              // item n - 1 has been converted and multiplied
      mbar_wait(full(s), (n / S) & 1);
      // landed x tile -> bf16 hi / mid A fragments of all 8 k-steps
      uint32_t* const tile = reinterpret_cast<uint32_t*>(base_ptr + ring_off + s * PJ_STAGE);
      const float* xt = reinterpret_cast<const float*>(tile);
#pragma unroll
      for (int ks = 0; ks < 8; ++ks)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int row = (e & 1) ? r1 : r0, c = 16 * ks + 2 * t + 8 * (e >> 1);
          const int b = c >> 5, kk = c & 31;
          const float2 x = *reinterpret_cast<const float2*>(xt + b * (PJ_BOX / 4) + row * 32 +
                                                            (((kk >> 2) ^ (row & 7)) << 2) + (kk & 3));
          split_pair(x.x, x.y, ahi[ks][e], amid[ks][e]);
        }
      layer_mma(acc, ahi, amid, w1h, w1m);
      bias_relu(acc, b1, t);
      if (role != 2) {
        // q1 / k1 fragment -> A fragment of layer 2: k-step ks = columns 16 ks .. 16 ks + 15 = accumulator pairs j = 2 ks, 2 ks + 1
#pragma unroll
        for (int ks = 0; ks < 8; ++ks)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int a = 4 * (2 * ks + (e >> 1)) + 2 * (e & 1);
            split_pair(acc[a], acc[a + 1], ahi[ks][e], amid[ks][e]);
          }
        layer_mma(acc, ahi, amid, w2h, w2m);
        bias_relu(acc, b2, t);
      }
      if (n + 1 < n_items) bar_arrive(2 - wg, 256);  // the other warpgroup's turn
      // planar epilogue into the stage, in place: a warp overwrites only its own 16 rows, which it has already read.
      // Per row 64 words of bf16 hi pairs (boxes 0, 1), then 64 words of bf16 mid pairs (boxes 2, 3), in the
      // 128-byte swizzle of the x tile: word 4j + t of a box row r lies in 16-byte chunk j ^ (r & 7), so the 8 rows x
      // 4 words of one warp store fill all 32 banks.
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = h ? r1 : r0;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          uint32_t hi, mid;
          split_pair(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], hi, mid);
          const int w = (j >> 3) * (PJ_BOX / 4) + row * 32 + (((j & 7) ^ g) << 2) + t;
          tile[w] = hi;
          tile[w + 2 * (PJ_BOX / 4)] = mid;
        }
      }
      fence_proxy_async();
      bar_sync(3 + wg, 128);
      if (storer) {
        // four 32-word x 64-row boxes; TMA does not write rows >= M
        const uint32_t st = base + ring_off + s * PJ_STAGE;
        for (int b = 0; b < 4; ++b) tma_store_2d(mo, st + b * PJ_BOX, 32 * b, item * PJ_ROWS);
        bulk_commit();
        bulk_wait_read_all();
        mbar_arrive(empty(s));
      }
    }
    if (storer) bulk_wait_all();
  }
}

bool make_map(CUtensorMap* m, CUtensorMapDataType dt, const void* ptr, long long rows, long long cols, long long ld_bytes,
              int box_cols, int box_rows) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return false;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld_bytes};
  cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  return enc(m, dt, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// CTAs per role for a grid of G >= 3: in proportion to the time one 64-row work item of that role takes, at least one
// each.  The stores, not the MMA, set that time (DESIGN 4.2), so a V item costs nearly as much as a Q / K item
// although it has half the MMA.  PJ_COST_QK : PJ_COST_V = 4 : 3 gives 48 : 48 : 36 CTAs at 132 SMs; a sweep of the V
// count on an H100 (tools/bench_lcab.py shapes, L2 flushed) was fastest at 32 V CTAs for self attention and 38 for
// cross attention, and 26 (the earlier 2 : 2 : 1 FLOP split) was 1.2-1.3x slower than either.
constexpr int PJ_COST_QK = 4, PJ_COST_V = 3;
void role_split(int sms, int items, int* nq, int* nk, int* nv) {
  constexpr int total = 2 * PJ_COST_QK + PJ_COST_V;
  const int G = sms > 3 ? sms : 3;
  int v = (G * PJ_COST_V + total / 2) / total;
  v = v < 1 ? 1 : (v > G - 2 ? G - 2 : v);
  const int q = (G - v + 1) / 2, k = G - v - q;
  *nq = q < items ? q : items;                       // none without an item
  *nk = k < items ? k : items;
  *nv = v < items ? v : items;
}

constexpr int MAX_DEV = 64;
bool g_attr_set[MAX_DEV];

int proj_fused(const float* x_t, int ld_t, const float* x_s, int ld_s, const void* W1_hi, const void* W1_mid,
               const float* b1, const void* W2_hi, const void* W2_mid, const float* b2, float* q, float* k, float* v,
               int M, cudaStream_t stream) {
  const char* name = "di_lcab_proj_f32";
  int sms = 0;
  int rc = sm_budget(name, &sms);
  if (rc != DI_OK) return rc;
  int devid = 0;
  cudaGetDevice(&devid);
  if (!g_attr_set[devid]) {
    if (cudaFuncSetAttribute(lcab_proj_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PJ_SMEM_BYTES) != cudaSuccess) {
      di_set_error("%s: cannot reserve %d bytes of shared memory", name, PJ_SMEM_BYTES);
      return DI_ERR_LAUNCH;
    }
    g_attr_set[devid] = true;
  }
  CUtensorMap maps[9];
  const auto bf16 = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, f32 = CU_TENSOR_MAP_DATA_TYPE_FLOAT32, u32 = CU_TENSOR_MAP_DATA_TYPE_UINT32;
  if (!(make_map(&maps[0], f32, x_t, M, 128, 4ll * ld_t, 32, PJ_ROWS) && make_map(&maps[1], f32, x_s, M, 128, 4ll * ld_s, 32, PJ_ROWS) &&
        make_map(&maps[2], bf16, W1_hi, 384, 128, 256, 64, 128) && make_map(&maps[3], bf16, W1_mid, 384, 128, 256, 64, 128) &&
        make_map(&maps[4], bf16, W2_hi, 256, 128, 256, 64, 128) && make_map(&maps[5], bf16, W2_mid, 256, 128, 256, 64, 128) &&
        make_map(&maps[6], u32, q, M, 128, 512, 32, PJ_ROWS) && make_map(&maps[7], u32, k, M, 128, 512, 32, PJ_ROWS) &&
        make_map(&maps[8], u32, v, M, 128, 512, 32, PJ_ROWS))) {
    di_set_error("%s: cuTensorMapEncodeTiled failed", name);
    return DI_ERR_LAUNCH;
  }
  ProjParams p{};
  p.b1 = b1;
  p.b2 = b2;
  p.M = M;
  p.items = di_cdiv(M, PJ_ROWS);
  role_split(sms, p.items, &p.nq, &p.nk, &p.nv);
  lcab_proj_kernel<<<p.nq + p.nk + p.nv, PJ_THREADS, PJ_SMEM_BYTES, stream>>>(maps[0], maps[1], maps[2], maps[3], maps[4],
                                                                                maps[5], maps[6], maps[7], maps[8], p);
  DI_CHECK_LAUNCH(name);
  return DI_OK;
}

}  // namespace

extern "C" {

int di_lcab_proj_grid(int M, int* nq, int* nk, int* nv) {
  DI_CHECK_ARG(M > 0 && nq && nk && nv, "di_lcab_proj_grid: bad argument");
  int sms = 0;
  const int rc = sm_budget("di_lcab_proj_grid", &sms);
  if (rc != DI_OK) return rc;
  role_split(sms, di_cdiv(M, PJ_ROWS), nq, nk, nv);
  return DI_OK;
}

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
  return proj_fused(x_t, ld_t, x_s, ld_s, W1_hi, W1_mid, b1, W2_hi, W2_mid, b2, q, k, v, M, stream);
}

// LocalContextAttentionBlock.forward (models/utils/encoder_utils.py:119-135) for C = 128 as ONE call: the projections
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
