// MMPI decoder kernels (forward).  Reference (projects/mmdet3d_plugin/):
//   models/dense_heads/deepinteraction_decoder.py:223-253  heatmap fusion, 3x3 max-pool NMS, top-k, query init
//   models/utils/decoder_utils.py:35-113,246-495         transformer decoder layer (self + cross attention)
//   models/utils/decoder_utils.py:632-841                 Image/Point RCNN blocks (box decode, projection,
//                                                         RoIAlign 7x7, masked self-attention, DynamicConv)
//   core/bbox/coders/transfusion_bbox_coder.py:39-76      box decode
// Queries are stored row-major [B*P, C] ("one query = one row"); feature maps are pixel-major (NHWC).
#include "common.cuh"
#include "tc_common.cuh"
#include <math.h>


namespace {

// ------------------------------------------------------------------------------------------------
// Heatmap fusion + NMS  (decoder.py:225-239)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

// a, b: raw logits, pixel-major [B, HW, ld] (first K columns valid).  out [B,K,HW] = NMS-masked mean of
// sigmoids; dense_b [B,K,H,W] = head-b logits in the NCHW layout the reference returns as `dense_heatmap`.
__global__ void heatmap_nms_kernel(const float* __restrict__ a, const float* __restrict__ b, int ld,
                                   float* __restrict__ out, float* __restrict__ dense_b, int K, int H, int W, int ks,
                                   unsigned no_nms_mask, int total) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  int x = i % W, y = (i / W) % H, c = (i / (W * H)) % K, n = i / (W * H * K);
  const float* pa = a + (size_t)n * H * W * ld + c;
  const float* pb = b + (size_t)n * H * W * ld + c;
  const float lb = pb[(size_t)(y * W + x) * ld];
  float hc = (sigmoidf_(pa[(size_t)(y * W + x) * ld]) + sigmoidf_(lb)) * 0.5f;
  float res;
  if ((no_nms_mask >> c) & 1u) {
    res = hc;
  } else {
    int r = ks / 2;
    if (y < r || y >= H - r || x < r || x >= W - r) {
      res = 0.f;  // local_max stays 0 on the border ring => never equal to a positive score
    } else {
      float m = hc;
      for (int dy = -r; dy <= r; ++dy)
        for (int dx = -r; dx <= r; ++dx) {
          size_t o = (size_t)((y + dy) * W + x + dx) * ld;
          m = fmaxf(m, (sigmoidf_(pa[o]) + sigmoidf_(pb[o])) * 0.5f);
        }
      res = hc == m ? hc : 0.f;
    }
  }
  out[i] = res;
  if (dense_b) dense_b[i] = lb;
}

// ------------------------------------------------------------------------------------------------
// Top-k of non-negative scores (descending, ties -> smaller index first).  One CTA per batch row.
// Radix select on the float bit pattern (12 + 12 + 8 bits), then a bitonic sort of the k winners.
// ------------------------------------------------------------------------------------------------
constexpr int TOPK_MAX = 1024;

// Two levels: level 1 = one CTA per (slice, batch row) keeps the slice's top-k as (value, global index)
// candidates; level 2 = one CTA per batch row selects the final top-k among the G*k candidates.
__global__ void __launch_bounds__(1024)
topk_kernel(const float* __restrict__ scores_all, const int* __restrict__ src_idx_all, int n_row, int n_slice, int k,
            float* __restrict__ val_out, int* __restrict__ idx_out) {
  __shared__ unsigned hist[4096];
  __shared__ unsigned s_prefix, s_need, s_cnt_gt, s_cnt_eq;
  __shared__ unsigned long long cand[TOPK_MAX];  // (value bits << 32) | (0xffffffff - index): sort descending
  __shared__ unsigned eq_idx[TOPK_MAX];
  // blockIdx.y = batch row, blockIdx.x = slice; this CTA looks at elements [off, off + n) of its row
  const int off = blockIdx.x * n_slice;
  const int n = min(n_slice, n_row - off);
  const float* s = scores_all + (size_t)blockIdx.y * n_row + off;
  const int* sidx = src_idx_all ? src_idx_all + (size_t)blockIdx.y * n_row + off : nullptr;
  const int t = threadIdx.x;
  const int k_host = k;
  if (n < k) k = max(n, 0);
  unsigned prefix = 0, need = (unsigned)k;
  // pass p examines bits [hi, lo)
  const int shifts[3] = {20, 8, 0};
  const int widths[3] = {12, 12, 8};
  unsigned known_mask = 0;
  for (int pass = 0; pass < 3; ++pass) {
    for (int i = t; i < 4096; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    const int sh = shifts[pass];
    const unsigned wmask = (1u << widths[pass]) - 1u;
    for (int i = t; i < n; i += blockDim.x) {
      unsigned u = __float_as_uint(s[i]);
      if ((u & known_mask) == prefix) atomicAdd(&hist[(u >> sh) & wmask], 1u);
    }
    __syncthreads();
    if (t < 32) {
      // warp-parallel search of the bin where the count from the top reaches `need`
      const int nb = (int)wmask + 1, per = (nb + 31) / 32;
      const int hi_bin = min(nb, (t + 1) * per) - 1, lo_bin = t * per;
      unsigned mine = 0;
      for (int bnum = lo_bin; bnum <= hi_bin; ++bnum) mine += hist[bnum];
      // above[t] = elements in bins owned by lanes > t
      unsigned above = 0;
      for (int l = 31; l >= 0; --l) {
        unsigned v = __shfl_sync(0xffffffffu, mine, l);
        if (l > t) above += v;
      }
      const bool owner = above < need && above + mine >= need;
      unsigned vote = __ballot_sync(0xffffffffu, owner);
      if (vote == 0) {            // cannot happen (the matching count is always >= need); keep the prefix
        if (t == 0) {
          s_prefix = prefix;
          s_need = 0;
        }
      } else if (owner) {
        unsigned acc = above;
        int bin = hi_bin;
        for (; bin > lo_bin; --bin) {
          if (acc + hist[bin] >= need) break;
          acc += hist[bin];
        }
        s_prefix = prefix | ((unsigned)bin << sh);
        s_need = need - acc;
      }
    }
    __syncthreads();
    prefix = s_prefix;
    need = s_need;
    known_mask |= wmask << sh;
    __syncthreads();
  }
  // prefix == bit pattern of the k-th largest value; `need` of the elements equal to it are taken
  if (t == 0) {
    s_cnt_gt = 0;
    s_cnt_eq = 0;
  }
  for (int i = t; i < TOPK_MAX; i += blockDim.x) cand[i] = 0ull;
  __syncthreads();
  for (int i = t; i < n; i += blockDim.x) {
    unsigned u = __float_as_uint(s[i]);
    if (u > prefix) {
      unsigned pos = atomicAdd(&s_cnt_gt, 1u);
      cand[pos] = ((unsigned long long)u << 32) | (unsigned long long)(0xffffffffu - (unsigned)i);
    } else if (u == prefix && k > 0) {
      unsigned pos = atomicAdd(&s_cnt_eq, 1u);
      if (pos < TOPK_MAX) eq_idx[pos] = (unsigned)i;
    }
  }
  __syncthreads();
  if (s_cnt_eq > TOPK_MAX) {
    // more ties than eq_idx holds (e.g. a row of zeros): block-wide pass over the slice in ascending index order, chunks of
    // blockDim indices, each tie ranked by a ballot and a prefix count over the warps, until `need` of them are taken
    __shared__ unsigned warp_cnt[32];
    const int lane = t & 31, w = t >> 5, nw = blockDim.x >> 5;
    for (unsigned taken = 0, base = 0; taken < need && base < (unsigned)n; base += blockDim.x) {
      const unsigned i = base + t;
      const bool hit = i < (unsigned)n && __float_as_uint(s[i]) == prefix;
      const unsigned bal = __ballot_sync(0xffffffffu, hit);
      if (lane == 0) warp_cnt[w] = __popc(bal);
      __syncthreads();
      unsigned rank = taken + __popc(bal & ((1u << lane) - 1u)), total = 0;
      for (int j = 0; j < nw; ++j) {
        if (j < w) rank += warp_cnt[j];
        total += warp_cnt[j];
      }
      if (hit && rank < need)
        cand[s_cnt_gt + rank] = ((unsigned long long)prefix << 32) | (unsigned long long)(0xffffffffu - i);
      __syncthreads();
      taken += total;
    }
  } else if (t == 0) {
    // ties at the threshold: take the `need` smallest indices (a single thread; ties are measure-zero)
    unsigned ne = s_cnt_eq;
    for (unsigned a = 0; a < need; ++a) {
      unsigned best = a;
      for (unsigned b2 = a + 1; b2 < ne; ++b2)
        if (eq_idx[b2] < eq_idx[best]) best = b2;
      unsigned tmp = eq_idx[a];
      eq_idx[a] = eq_idx[best];
      eq_idx[best] = tmp;
      cand[s_cnt_gt + a] = ((unsigned long long)prefix << 32) | (unsigned long long)(0xffffffffu - eq_idx[a]);
    }
  }
  __syncthreads();
  // bitonic sort, descending, over TOPK_MAX slots (empty slots are 0 and sink to the end)
  for (int size = 2; size <= TOPK_MAX; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = t; i < TOPK_MAX / 2; i += blockDim.x) {
        int lo = (i / stride) * stride * 2 + (i % stride);
        int hi = lo + stride;
        bool desc = ((lo / size) & 1) == 0;
        unsigned long long a = cand[lo], b2 = cand[hi];
        if ((a < b2) == desc) {
          cand[lo] = b2;
          cand[hi] = a;
        }
      }
      __syncthreads();
    }
  }
  // output slot of this CTA: [row][slice][k_out] where k_out = the k passed by the host (before clamping)
  const size_t obase = ((size_t)blockIdx.y * gridDim.x + blockIdx.x) * (size_t)k_host;
  for (int i = t; i < k_host; i += blockDim.x) {
    int gi = -1;
    float gv = 0.f;
    if (i < k) {
      int local = (int)(0xffffffffu - (unsigned)(cand[i] & 0xffffffffull));
      gi = sidx ? sidx[local] : off + local;
      gv = __uint_as_float((unsigned)(cand[i] >> 32));
    }
    idx_out[obase + i] = gi;
    if (val_out) val_out[obase + i] = gv;
  }
}

// query_feat[b,q,:] = feat[b, pix, :] + Wce[cls, :] + bce ; query_pos = (x+.5, y+.5) ; score gather
__global__ void query_init_kernel(const float* __restrict__ feat, const int* __restrict__ top,
                                  const float* __restrict__ heat, const float* __restrict__ wce_t,
                                  const float* __restrict__ bce, float* __restrict__ qfeat, float* __restrict__ qpos,
                                  int* __restrict__ labels, float* __restrict__ qscore, int HW, int W, int C, int K,
                                  int P) {
  int bq = blockIdx.x;  // b*P + q
  int b = bq / P, qi = bq - b * P;
  int flat = top[bq];
  int cls = flat / HW, pix = flat - cls * HW;
  const float* src = feat + ((size_t)b * HW + pix) * C;
  for (int c = threadIdx.x; c < C; c += blockDim.x)
    qfeat[(size_t)bq * C + c] = src[c] + wce_t[(size_t)cls * C + c] + bce[c];
  if (threadIdx.x == 0) {
    qpos[bq * 2 + 0] = (float)(pix % W) + 0.5f;
    qpos[bq * 2 + 1] = (float)(pix / W) + 0.5f;
    labels[bq] = cls;
  }
  for (int c = threadIdx.x; c < K; c += blockDim.x)
    qscore[((size_t)b * K + c) * P + qi] = heat[((size_t)b * K + c) * HW + pix];
}

// Backward of the feature gather: d_feat[b, pix, :] += the d qfeat rows of the proposals at pix, in proposal order.  One
// CTA per proposal; the first proposal at a pixel owns it and sums all of them, the others return (no atomics).
__global__ void __launch_bounds__(128)
query_init_bwd_feat_kernel(const float* __restrict__ dq, const int* __restrict__ top, float* __restrict__ d_feat, int HW,
                           int C, int P) {
  extern __shared__ int s_pix[];
  const int b = blockIdx.y, qi = blockIdx.x;
  for (int j = threadIdx.x; j < P; j += blockDim.x) s_pix[j] = top[b * P + j] % HW;
  __syncthreads();
  const int pix = s_pix[qi];
  int shared_earlier = 0;
  for (int j = threadIdx.x; j < qi; j += blockDim.x) shared_earlier |= s_pix[j] == pix;
  if (__syncthreads_or(shared_earlier)) return;
  float* dst = d_feat + ((size_t)b * HW + pix) * C;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float s = dst[c];
    for (int j = qi; j < P; ++j)
      if (s_pix[j] == pix) s += dq[((size_t)b * P + j) * C + c];
    dst[c] = s;
  }
}

// Backward of the class encoding (Conv1d(K, C, 1) on the one-hot labels): block k < K -> d_w[c, k] = sum of the d qfeat
// rows with label k; block K -> d_b[c] = sum of all rows.  Rows in order, one thread per output.
__global__ void __launch_bounds__(128)
query_init_bwd_class_kernel(const float* __restrict__ dq, const int* __restrict__ labels, float* __restrict__ d_w,
                            float* __restrict__ d_b, int M, int C, int K) {
  const int k = blockIdx.x;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float s = 0.f;
    for (int r = 0; r < M; ++r)
      if (k == K || labels[r] == k) s += dq[(size_t)r * C + c];
    if (k == K) d_b[c] = s;
    else d_w[(size_t)c * K + k] = s;
  }
}

// ------------------------------------------------------------------------------------------------
// Small multi-head attention among the P queries of one sample (self-attention of the transformer
// layer and of the RCNN blocks).  One warp per (query, head).  Optional group mask: key j is visible to
// query q iff (onbits[j] >> win[q]) & 1 (queries that project into the same camera view).
// ------------------------------------------------------------------------------------------------
template <int D>
__global__ void __launch_bounds__(256)
mha_small_kernel(const float* __restrict__ q, int ldq, const float* __restrict__ k, int ldk, const float* __restrict__ v,
                 int ldv, float* __restrict__ out, int ldo, const int* __restrict__ onbits, const int* __restrict__ win,
                 int B, int P, int Hh, const int* __restrict__ rows, int R, int rows_per_b) {
  int wid = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  int lane = threadIdx.x & 31;
  if (wid >= (rows ? R : B * P) * Hh) return;
  int head = wid % Hh, bq = wid / Hh;
  int b = bq / P;
  int wq = win ? win[bq] : 0;
  float* o = out + (size_t)bq * ldo + head * D;
  if (rows) {
    // row-map form (V2 blocks): output row r = query rows[r] seen from group win[r] (= the r-th (sample, view) pair)
    b = bq / rows_per_b;
    const int r = bq;
    bq = rows[r];
    if (bq < 0) wq = -1;
  }
  if (wq < 0) {
    if (lane < D) o[lane] = 0.f;
    return;
  }
  float qr[D];
#pragma unroll
  for (int d = 0; d < D; d += 4) {
    float4 t4 = ldg4(q + (size_t)bq * ldq + head * D + d);
    qr[d] = t4.x; qr[d + 1] = t4.y; qr[d + 2] = t4.z; qr[d + 3] = t4.w;
  }
  // pass 1: scores of this lane's keys
  constexpr int MAXK = 16;  // P <= 512
  float sc[MAXK];
  float m = -INFINITY;
#pragma unroll
  for (int i = 0; i < MAXK; ++i) {
    int j = i * 32 + lane;
    sc[i] = -INFINITY;
    if (j < P) {
      int bj = b * P + j;
      bool vis = onbits ? ((onbits[bj] >> wq) & 1) : true;
      if (vis) {
        const float* kr = k + (size_t)bj * ldk + head * D;
        float s = 0.f;
#pragma unroll
        for (int d = 0; d < D; d += 4) {
          float4 t4 = ldg4(kr + d);
          s += qr[d] * t4.x + qr[d + 1] * t4.y + qr[d + 2] * t4.z + qr[d + 3] * t4.w;
        }
        sc[i] = s;
        m = fmaxf(m, s);
      }
    }
  }
  m = warp_max(m);
  float acc[D];
#pragma unroll
  for (int d = 0; d < D; ++d) acc[d] = 0.f;
  float l = 0.f;
#pragma unroll
  for (int i = 0; i < MAXK; ++i) {
    int j = i * 32 + lane;
    if (j < P && sc[i] > -INFINITY) {
      float p = expf(sc[i] - m);
      l += p;
      const float* vr = v + (size_t)(b * P + j) * ldv + head * D;
#pragma unroll
      for (int d = 0; d < D; d += 4) {
        float4 t4 = ldg4(vr + d);
        acc[d] += p * t4.x; acc[d + 1] += p * t4.y; acc[d + 2] += p * t4.z; acc[d + 3] += p * t4.w;
      }
    }
  }
  l = warp_sum(l);
  float inv = l > 0.f ? 1.f / l : 0.f;
#pragma unroll
  for (int d = 0; d < D; ++d) {
    float a = warp_sum(acc[d]);
    if (lane == d) o[d] = a * inv;
  }
}

// Backward of mha_small_kernel (the self-attention of the transformer layer, decoder_utils.py:95-99, and of the RCNN
// blocks, with the same optional group mask: key j is visible to query i iff win[i] >= 0 and (onbits[j] >> win[i]) & 1).
// Pass 1, one warp per (query i, head): recompute A_i = softmax(q_i K^T) over the visible keys, dA_ij = dO_i . v_j,
// D_i = sum_j A_ij dA_ij, dS_ij = A_ij (dA_ij - D_i), dq_i = sum_j dS_ij k_j; A and dS are stored key-major
// ([b, head, j, i]) for pass 2, for the visible pairs only.  A query with win < 0 gets a zero dq row and writes nothing.
// Pass 2, one warp per (key j, head): dk_j = sum_i dS_ij q_i, dv_j = sum_i A_ij dO_i over the queries that see key j,
// tested here again (pass 1 leaves the invisible pairs of the workspace unwritten).  Neither pass reads the rows of a
// masked pair.  Fixed summation orders (lanes over a strided index range, then the warp butterfly): deterministic, no
// atomics; without a mask every pair is visible and the arithmetic is that of the unmasked form.
// ROWS: pass 1 of the row-map form (di_mha_small_rows_bwd_f32): warp (r, head) takes query rows[r] (-1: zero dq row) of
// sample r / NI seen from group win[r]; dout and dq are indexed by r, and the workspace holds NI = rows_per_b columns.
template <int D, bool ROWS>
__global__ void __launch_bounds__(256)
mha_small_bwd_q_kernel(const float* __restrict__ q, int ldq, const float* __restrict__ k, int ldk, const float* __restrict__ v,
                       int ldv, const float* __restrict__ dout, int ldd, float* __restrict__ dq, int ldg, float* __restrict__ aw,
                       float* __restrict__ sw, const int* __restrict__ onbits, const int* __restrict__ win, int B, int P, int Hh,
                       const int* __restrict__ rows, int NI) {
  const int wid = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (wid >= B * NI * Hh) return;
  const int head = wid % Hh, r = wid / Hh, b = r / NI, i = r % NI;
  const int bq = ROWS ? rows[r] : r;
  const int wq = ROWS ? (bq < 0 ? -1 : win[r]) : (win ? win[bq] : 0);
  if (wq < 0) {
    if (lane < D) dq[(size_t)r * ldg + head * D + lane] = 0.f;
    return;
  }
  float qr[D], gr[D];
#pragma unroll
  for (int d = 0; d < D; d += 4) {
    const float4 a = ldg4(q + (size_t)bq * ldq + head * D + d), c = ldg4(dout + (size_t)r * ldd + head * D + d);
    qr[d] = a.x; qr[d + 1] = a.y; qr[d + 2] = a.z; qr[d + 3] = a.w;
    gr[d] = c.x; gr[d + 1] = c.y; gr[d + 2] = c.z; gr[d + 3] = c.w;
  }
  constexpr int MAXK = 16;  // P <= 512
  float sc[MAXK], dav[MAXK];
  unsigned vis = 0;         // bit n: key n * 32 + lane exists and is visible
  float m = -INFINITY;
#pragma unroll
  for (int n = 0; n < MAXK; ++n) {
    const int j = n * 32 + lane;
    sc[n] = -INFINITY;
    dav[n] = 0.f;
    if (j < P && (!onbits || ((onbits[b * P + j] >> wq) & 1))) {
      vis |= 1u << n;
      const float* kr = k + (size_t)(b * P + j) * ldk + head * D;
      const float* vr = v + (size_t)(b * P + j) * ldv + head * D;
      float s = 0.f, da = 0.f;
#pragma unroll
      for (int d = 0; d < D; d += 4) {
        const float4 a = ldg4(kr + d), c = ldg4(vr + d);
        s += qr[d] * a.x + qr[d + 1] * a.y + qr[d + 2] * a.z + qr[d + 3] * a.w;
        da += gr[d] * c.x + gr[d + 1] * c.y + gr[d + 2] * c.z + gr[d + 3] * c.w;
      }
      sc[n] = s;
      dav[n] = da;
      m = fmaxf(m, s);
    }
  }
  m = warp_max(m);
  float l = 0.f;
#pragma unroll
  for (int n = 0; n < MAXK; ++n) {
    sc[n] = (vis >> n) & 1 ? expf(sc[n] - m) : 0.f;
    l += sc[n];
  }
  l = warp_sum(l);
  // a group that hides every key: zero weights and gradients, as the forward writes a zero row
  const float inv = onbits && !(l > 0.f) ? 0.f : 1.f / l;
  float dsum = 0.f;
#pragma unroll
  for (int n = 0; n < MAXK; ++n) {
    sc[n] *= inv;
    dsum += sc[n] * dav[n];
  }
  dsum = warp_sum(dsum);
  float acc[D];
#pragma unroll
  for (int d = 0; d < D; ++d) acc[d] = 0.f;
  const size_t col = ((size_t)(b * Hh + head) * P) * NI + i;     // [b, head, j, i]
#pragma unroll
  for (int n = 0; n < MAXK; ++n) {
    const int j = n * 32 + lane;
    if ((vis >> n) & 1) {
      const float ds = sc[n] * (dav[n] - dsum);
      aw[col + (size_t)j * NI] = sc[n];
      sw[col + (size_t)j * NI] = ds;
      const float* kr = k + (size_t)(b * P + j) * ldk + head * D;
#pragma unroll
      for (int d = 0; d < D; d += 4) {
        const float4 a = ldg4(kr + d);
        acc[d] += ds * a.x; acc[d + 1] += ds * a.y; acc[d + 2] += ds * a.z; acc[d + 3] += ds * a.w;
      }
    }
  }
#pragma unroll
  for (int d = 0; d < D; ++d) {
    const float a = warp_sum(acc[d]);
    if (lane == d) dq[(size_t)r * ldg + head * D + d] = a;
  }
}

template <int D>
__global__ void __launch_bounds__(256)
mha_small_bwd_kv_kernel(const float* __restrict__ q, int ldq, const float* __restrict__ dout, int ldd,
                        const float* __restrict__ aw, const float* __restrict__ sw, float* __restrict__ dk,
                        float* __restrict__ dv, int ldg, const int* __restrict__ onbits, const int* __restrict__ win,
                        int B, int P, int Hh) {
  const int wid = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (wid >= B * P * Hh) return;
  const int head = wid % Hh, bj = wid / Hh, b = bj / P, j = bj % P;
  const int bits = onbits ? onbits[bj] : 0;
  const float* ar = aw + ((size_t)(b * Hh + head) * P + j) * P;
  const float* sr = sw + ((size_t)(b * Hh + head) * P + j) * P;
  float ak[D], av[D];
#pragma unroll
  for (int d = 0; d < D; ++d) ak[d] = av[d] = 0.f;
  for (int i = lane; i < P; i += 32) {
    if (onbits) {
      const int wi = win[b * P + i];
      if (wi < 0 || !((bits >> wi) & 1)) continue;
    }
    const float a = ar[i], ds = sr[i];
    const float* qr = q + (size_t)(b * P + i) * ldq + head * D;
    const float* gr = dout + (size_t)(b * P + i) * ldd + head * D;
#pragma unroll
    for (int d = 0; d < D; d += 4) {
      const float4 x = ldg4(qr + d), y = ldg4(gr + d);
      ak[d] += ds * x.x; ak[d + 1] += ds * x.y; ak[d + 2] += ds * x.z; ak[d + 3] += ds * x.w;
      av[d] += a * y.x; av[d + 1] += a * y.y; av[d + 2] += a * y.z; av[d + 3] += a * y.w;
    }
  }
#pragma unroll
  for (int d = 0; d < D; ++d) {
    const float x = warp_sum(ak[d]), y = warp_sum(av[d]);
    if (lane == d) {
      dk[(size_t)bj * ldg + head * D + d] = x;
      dv[(size_t)bj * ldg + head * D + d] = y;
    }
  }
}

// Pass 2 of the row-map form, one warp per (key j, head): lanes 0-15 hold dk_j's channels, lanes 16-31 dv_j's.  The warp
// walks the NI leader rows of key j's sample in ascending r, skipping rows[r] = -1 and the rows whose group bit
// rwin[r] key j lacks (as pass 1 does), and ADDS dk_j += sum_r dS_rj q_rows[r], dv_j += sum_r A_rj dO_r to the gradient
// already there (the main attention's).
template <int D>
__global__ void __launch_bounds__(256)
mha_small_rows_bwd_kv_kernel(const float* __restrict__ q, int ldq, const float* __restrict__ dout, int ldd,
                             const float* __restrict__ aw, const float* __restrict__ sw, float* __restrict__ dk,
                             float* __restrict__ dv, int ldg, const int* __restrict__ onbits, const int* __restrict__ rows,
                             const int* __restrict__ rwin, int B, int P, int Hh, int NI) {
  static_assert(2 * D == 32, "one lane per dk and per dv channel");
  const int wid = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (wid >= B * P * Hh) return;
  const int head = wid % Hh, bj = wid / Hh, b = bj / P, j = bj % P;
  const int bits = onbits[bj], d = lane & (D - 1);
  const bool val = lane >= D;
  const size_t col = ((size_t)(b * Hh + head) * P + j) * NI;
  float acc = 0.f;
  for (int i = 0; i < NI; ++i) {
    const int r = b * NI + i, row = rows[r];
    if (row < 0 || !((bits >> rwin[r]) & 1)) continue;
    acc += val ? aw[col + i] * dout[(size_t)r * ldd + head * D + d] : sw[col + i] * q[(size_t)row * ldq + head * D + d];
  }
  float* g = (val ? dv : dk) + (size_t)bj * ldg + head * D + d;
  *g += acc;
}

// ------------------------------------------------------------------------------------------------
// Query x BEV cross attention (decoder_utils.py:101-103,466-488): P queries x HW keys, Hh heads of D=16.
// kv [B*HW, 2*C]: projected keys (cols [0,C)) and values (cols [C,2C)).  Split over key chunks
// (flash-decoding): each CTA = (key chunk, head, batch, query tile of 256) keeps a running
// (max, sum, acc[D]) per query; a second kernel merges the chunks.
// ------------------------------------------------------------------------------------------------
template <int D>
__global__ void __launch_bounds__(256)
cross_attn_kernel(const float* __restrict__ q, const float* __restrict__ kv, float* __restrict__ part, int P, int HW,
                  int C, int Hh, int chunk, int nsplit) {
  constexpr int TK = 128;                        // keys per shared-memory tile
  __shared__ __align__(16) float ks[TK][D];
  __shared__ __align__(16) float vs[TK][D];
  const int split = blockIdx.x % nsplit, qt = blockIdx.x / nsplit;
  const int head = blockIdx.y, b = blockIdx.z;
  const int qi = qt * 256 + threadIdx.x;
  const bool active = qi < P;
  float qr[D];
#pragma unroll
  for (int d = 0; d < D; ++d) qr[d] = 0.f;
  if (active) {
#pragma unroll
    for (int d = 0; d < D; d += 4) {
      float4 t4 = ldg4(q + (size_t)(b * P + qi) * C + head * D + d);
      qr[d] = t4.x; qr[d + 1] = t4.y; qr[d + 2] = t4.z; qr[d + 3] = t4.w;
    }
  }
  float m = -INFINITY, l = 0.f, acc[D];
#pragma unroll
  for (int d = 0; d < D; ++d) acc[d] = 0.f;
  const int k_begin = split * chunk, k_end = min(HW, k_begin + chunk);
  for (int k0 = k_begin; k0 < k_end; k0 += TK) {
    int nk = min(TK, k_end - k0);
    __syncthreads();
    for (int i = threadIdx.x; i < TK * (D / 4); i += blockDim.x) {
      int kk = i / (D / 4), d4 = i % (D / 4);
      float4 kx = make_float4(0, 0, 0, 0), vx = kx;
      if (kk < nk) {
        const float* row = kv + (size_t)(b * HW + k0 + kk) * (2 * C) + head * D + d4 * 4;
        kx = ldg4(row);
        vx = ldg4(row + C);
      }
      *reinterpret_cast<float4*>(&ks[kk][d4 * 4]) = kx;
      *reinterpret_cast<float4*>(&vs[kk][d4 * 4]) = vx;
    }
    __syncthreads();
    if (active) {
      for (int kk = 0; kk < nk; kk += 4) {   // 4 keys per rescale
        float s[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          float a = 0.f;
#pragma unroll
          for (int d = 0; d < D; d += 4) {
            float4 t4 = *reinterpret_cast<const float4*>(&ks[kk + u][d]);
            a += qr[d] * t4.x + qr[d + 1] * t4.y + qr[d + 2] * t4.z + qr[d + 3] * t4.w;
          }
          s[u] = (kk + u < nk) ? a : -INFINITY;
        }
        const float mn = fmaxf(fmaxf(m, fmaxf(s[0], s[1])), fmaxf(s[2], s[3]));
        if (mn > m) {                              // the running maximum rarely moves after the first keys
          const float corr = expf(m - mn);
          l *= corr;
#pragma unroll
          for (int d = 0; d < D; ++d) acc[d] *= corr;
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          float p = expf(s[u] - mn);
          l += p;
#pragma unroll
          for (int d = 0; d < D; d += 4) {
            float4 t4 = *reinterpret_cast<const float4*>(&vs[kk + u][d]);
            acc[d] += p * t4.x; acc[d + 1] += p * t4.y; acc[d + 2] += p * t4.z; acc[d + 3] += p * t4.w;
          }
        }
        m = mn;
      }
    }
  }
  if (active) {
    // partials as [b, head, split, field, q]: the threads of a warp (consecutive q) write / read consecutive floats
    float* o = part + ((((size_t)b * Hh + head) * nsplit + split) * (D + 2)) * P + qi;
    o[0] = m;
    o[P] = l;
#pragma unroll
    for (int d = 0; d < D; ++d) o[(size_t)(2 + d) * P] = acc[d];
  }
}

template <int D>
__global__ void cross_attn_combine_kernel(const float* __restrict__ part, float* __restrict__ out, int B, int P, int C,
                                          int Hh, int nsplit) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;  // (b, head, q)
  if (i >= B * Hh * P) return;
  int qi = i % P, head = (i / P) % Hh, b = i / (P * Hh);
  const float* pp = part + (size_t)(b * Hh + head) * nsplit * (D + 2) * P + qi;   // [split][field][q]
  const size_t ss = (size_t)(D + 2) * P;
  float M = -INFINITY;
  for (int s = 0; s < nsplit; ++s) M = fmaxf(M, pp[s * ss]);
  float L = 0.f, acc[D];
#pragma unroll
  for (int d = 0; d < D; ++d) acc[d] = 0.f;
  for (int s = 0; s < nsplit; ++s) {
    float w = expf(pp[s * ss] - M);
    L += w * pp[s * ss + P];
#pragma unroll
    for (int d = 0; d < D; ++d) acc[d] += w * pp[s * ss + (size_t)(2 + d) * P];
  }
  float inv = 1.f / L;
  float* o = out + (size_t)(b * P + qi) * C + head * D;
#pragma unroll
  for (int d = 0; d < D; ++d) o[d] = acc[d] * inv;
}

// ------------------------------------------------------------------------------------------------
// Row-wise finish: x = sum_s part[s][m,:] + bias + res[m,:];  y = act(LayerNorm(x) * gamma + beta)
// (no LayerNorm when gamma == nullptr); rows with zero_if_neg[m] < 0 are written as 0.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
rows_finish_kernel(const float* __restrict__ part, int nsplit, size_t split_stride, int ldp,
                   const float* __restrict__ bias, const float* __restrict__ res, int ldres,
                   const float* __restrict__ gamma, const float* __restrict__ beta, float* __restrict__ out, int ldo,
                   const int* __restrict__ zero_if_neg, int M, int C, int act, float eps) {
  int m = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  int lane = threadIdx.x & 31;
  if (m >= M) return;
  constexpr int MAXV = 16;  // C <= 512
  float x[MAXV];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    int c = i * 32 + lane;
    float a = 0.f;
    if (c < C) {
      for (int s = 0; s < nsplit; ++s) a += part[s * split_stride + (size_t)m * ldp + c];
      if (bias) a += bias[c];
      if (res) a += res[(size_t)m * ldres + c];
      sum += a;
    }
    x[i] = a;
  }
  bool zero = zero_if_neg && zero_if_neg[m] < 0;
  if (gamma) {
    float mean = warp_sum(sum) / (float)C;
    float var = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      int c = i * 32 + lane;
      if (c < C) {
        float d = x[i] - mean;
        var += d * d;
      }
    }
    var = warp_sum(var) / (float)C;
    float rstd = 1.f / sqrtf(var + eps);
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      int c = i * 32 + lane;
      if (c < C) x[i] = (x[i] - mean) * rstd * gamma[c] + beta[c];
    }
  }
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    int c = i * 32 + lane;
    if (c < C) out[(size_t)m * ldo + c] = zero ? 0.f : di_act(x[i], act);
  }
}

// Fast path of rows_finish for the map-sized calls of the ++ encoder (C == 128, one partial, 16-byte aligned rows):
// one warp per row, one float4 per lane -- 512 contiguous bytes in and out per row.
__global__ void __launch_bounds__(256)
rows_finish_c128_kernel(const float* __restrict__ x, int ldx, const float* __restrict__ bias, const float* __restrict__ res,
                        int ldres, const float* __restrict__ gamma, const float* __restrict__ beta, float* __restrict__ out,
                        int ldo, const int* __restrict__ zero_if_neg, int M, int act, float eps) {
  const int m = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (m >= M) return;
  float4 a = ldg4(x + (size_t)m * ldx + lane * 4);
  if (bias) {
    const float4 b = ldg4(bias + lane * 4);
    a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
  }
  if (res) {
    const float4 r = ldg4(res + (size_t)m * ldres + lane * 4);
    a.x += r.x; a.y += r.y; a.z += r.z; a.w += r.w;
  }
  if (gamma) {
    const float mean = warp_sum(a.x + a.y + a.z + a.w) * (1.f / 128.f);
    const float dx = a.x - mean, dy = a.y - mean, dz = a.z - mean, dw = a.w - mean;
    const float var = warp_sum(dx * dx + dy * dy + dz * dz + dw * dw) * (1.f / 128.f);
    const float rstd = 1.f / sqrtf(var + eps);
    const float4 g = ldg4(gamma + lane * 4), b = ldg4(beta + lane * 4);
    a = make_float4(dx * rstd * g.x + b.x, dy * rstd * g.y + b.y, dz * rstd * g.z + b.z, dw * rstd * g.w + b.w);
  }
  if (zero_if_neg && zero_if_neg[m] < 0) a = make_float4(0.f, 0.f, 0.f, 0.f);
  else a = make_float4(di_act(a.x, act), di_act(a.y, act), di_act(a.z, act), di_act(a.w, act));
  *reinterpret_cast<float4*>(out + (size_t)m * ldo + lane * 4) = a;
}


// ------------------------------------------------------------------------------------------------
// Query-row MLP: the decoder runs dozens of dense layers on B*P = 200..600 query rows.  On the tensor-core GEMM each is a
// launch dominated by start-up (tensor maps, barrier set-up); here one CTA takes 4 rows through
// up to TWO chained dense layers, a residual, a LayerNorm and an activation without leaving shared memory:
//     H = act1([X0 | X1] W1^T + b1)            Y = H W2^T + b2   (or Y = H)
//     Y = act_out(LN(Y + res))                 rows with zero_if_neg[m] < 0 are written as 0
// -> nn.Linear / Conv1d(k=1) chains of decoder_utils.py: pos-embed MLPs :16-32, attention in/out projections + norm
// :73-113, FFNs :104-109,754-757, prediction heads :498-581.  fp32 FFMA, sequential accumulation over k.
// Weights are passed TRANSPOSED ([K, N], so that lanes read consecutive output columns).
// ------------------------------------------------------------------------------------------------
constexpr int MLP_R = 4;        // rows per CTA: small, so that 200 query rows already spread over 50 SMs
constexpr int MLP_NT = 512;     // threads: k-groups of column threads (16 warps hide the shared-memory / FMA latencies)
constexpr int MLP_NS = 5;       // weight stages in shared memory (160 KB in flight: the copies are latency-bound)
constexpr int MLP_CHUNK = 8192; // floats per stage (32 KB): KC = 8192 / N consecutive rows of the transposed weight

// Weight streaming: the [K, N] transposed weights are contiguous, so KC rows are one 32 KB block; every thread copies
// 16-byte pieces of it with cp.async into a 5-stage ring (128 KB in flight per CTA; layer 2's first chunks are under way
// while layer 1 still computes), instead of dependent batches of __ldg (K / 16 round trips per layer).
__device__ __forceinline__ void mlp_copy_chunk(float* dst, const float* src, int floats, int tid) {
  const uint32_t d = tc::smem_u32(dst);
  for (int i = tid * 4; i < floats; i += MLP_NT * 4)
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d + i * 4), "l"(src + i) : "memory");
}

__global__ void __launch_bounds__(MLP_NT)
rows_mlp_kernel(const float* __restrict__ X0, int ld0, int K0, const float* __restrict__ X1, int ld1, int K1,
                const float* __restrict__ W1t, const float* __restrict__ b1, int N1, int act1,
                const float* __restrict__ W2t, const float* __restrict__ b2, int N2, const float* __restrict__ res, int ldres,
                const float* __restrict__ gamma, const float* __restrict__ beta, float eps, int act_out,
                const int* __restrict__ zero_if_neg, float* __restrict__ Y, int ldy, int M) {
  extern __shared__ __align__(128) float sm[];
  const int K = K0 + K1;
  float* wbuf = sm;                               // [MLP_NS][MLP_CHUNK]
  float* xs = wbuf + MLP_NS * MLP_CHUNK;          // [R][K]
  float* hs = xs + MLP_R * K;                     // [R][N1]
  float* ys = hs + MLP_R * N1;                    // [R][N2] (only with a second layer)
  const int m0 = blockIdx.x * MLP_R, tid = threadIdx.x;
  float* red = ys + MLP_R * (W2t ? N2 : 0);       // [groups][R][N] partial sums of the narrow layers (N <= 128)
  // job list: chunks of layer 1, then chunks of layer 2.  Chunk rows are a multiple of 4 (float4 activations).
  auto rows_per_chunk = [](int N) { const int kc = MLP_CHUNK / N; return kc >= 4 ? (kc & ~3) : max(1, kc); };
  const int kc1 = rows_per_chunk(N1), n1 = (K + kc1 - 1) / kc1;
  const int kc2 = W2t ? rows_per_chunk(N2) : 1, n2 = W2t ? (N1 + kc2 - 1) / kc2 : 0;
  const int njobs = n1 + n2;
  auto issue = [&](int j) {                       // all threads; always commits a group (possibly an empty one)
    if (j < njobs) {
      float* dst = wbuf + (size_t)(j % MLP_NS) * MLP_CHUNK;
      if (j < n1) {
        const int k0 = j * kc1, kc = min(kc1, K - k0);
        mlp_copy_chunk(dst, W1t + (size_t)k0 * N1, kc * N1, tid);
      } else {
        const int k0 = (j - n1) * kc2, kc = min(kc2, N1 - k0);
        mlp_copy_chunk(dst, W2t + (size_t)k0 * N2, kc * N2, tid);
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  for (int j = 0; j < MLP_NS - 1; ++j) issue(j);
  for (int i = tid; i < MLP_R * K; i += MLP_NT) {
    const int r = i / K, k = i - r * K, m = m0 + r;
    float v = 0.f;
    if (m < M) v = k < K0 ? X0[(size_t)m * ld0 + k] : X1[(size_t)m * ld1 + (k - K0)];
    xs[i] = v;
  }
  __syncthreads();
  // A layer of N columns uses groups of tpg = N / 4 threads, each thread a 4-row x 4-column register tile (float4
  // weight and activation reads: 8 shared-memory loads per 64 FMAs); the `ng` groups take disjoint k-slices of every
  // weight chunk and their partial sums are added in group order when the layer ends.
  float acc[MLP_R][4];
  for (int j = 0; j < njobs; ++j) {
    const bool l1 = j < n1;
    const int N = l1 ? N1 : N2, Kin = l1 ? K : N1;
    const int kc_full = l1 ? kc1 : kc2, k0 = (l1 ? j : j - n1) * kc_full, kc = min(kc_full, Kin - k0);
    const float* in = l1 ? xs : hs;
    const float* bias = l1 ? b1 : b2;
    const int tpg = N >> 2, ng = min(16, MLP_NT / tpg);
    const int grp = tid / tpg, col = (tid - grp * tpg) * 4;
    const bool live = grp < ng;
    if (k0 == 0) {
      float4 bb = make_float4(0.f, 0.f, 0.f, 0.f);
      if (bias && live && grp == 0) bb = *reinterpret_cast<const float4*>(bias + col);
#pragma unroll
      for (int r = 0; r < MLP_R; ++r) { acc[r][0] = bb.x; acc[r][1] = bb.y; acc[r][2] = bb.z; acc[r][3] = bb.w; }
    }
    // chunk j has landed for this thread; after the barrier for all threads, and the stage consumed in iteration j - 1
    // is free for chunk j + NS - 1 (the barrier also publishes hs when layer 2 starts)
    asm volatile("cp.async.wait_group %0;" ::"n"(MLP_NS - 2) : "memory");
    __syncthreads();
    issue(j + MLP_NS - 1);
    const float* w = wbuf + (size_t)(j % MLP_NS) * MLP_CHUNK;
    const int slice = ((kc + 4 * ng - 1) / (4 * ng)) * 4;
    const int ka = min(kc, grp * slice), kb = min(kc, ka + slice);
    if (live) {
      const bool vec = (Kin & 3) == 0 && ((k0 + ka) & 3) == 0;
      int kk = ka;
      if (vec) {
#pragma unroll 2
        for (; kk + 4 <= kb; kk += 4) {
          float4 xv[MLP_R], wv[4];
#pragma unroll
          for (int r = 0; r < MLP_R; ++r) xv[r] = *reinterpret_cast<const float4*>(in + r * Kin + k0 + kk);
#pragma unroll
          for (int q = 0; q < 4; ++q) wv[q] = *reinterpret_cast<const float4*>(w + (kk + q) * N + col);
#pragma unroll
          for (int r = 0; r < MLP_R; ++r) {
            const float xq[4] = {xv[r].x, xv[r].y, xv[r].z, xv[r].w};
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              acc[r][0] = fmaf(xq[q], wv[q].x, acc[r][0]);
              acc[r][1] = fmaf(xq[q], wv[q].y, acc[r][1]);
              acc[r][2] = fmaf(xq[q], wv[q].z, acc[r][2]);
              acc[r][3] = fmaf(xq[q], wv[q].w, acc[r][3]);
            }
          }
        }
      }
      for (; kk < kb; ++kk) {
        const float4 wv = *reinterpret_cast<const float4*>(w + kk * N + col);
#pragma unroll
        for (int r = 0; r < MLP_R; ++r) {
          const float x = in[r * Kin + k0 + kk];
          acc[r][0] = fmaf(x, wv.x, acc[r][0]);
          acc[r][1] = fmaf(x, wv.y, acc[r][1]);
          acc[r][2] = fmaf(x, wv.z, acc[r][2]);
          acc[r][3] = fmaf(x, wv.w, acc[r][3]);
        }
      }
    }
    if (k0 + kc == Kin) {                            // layer finished: group sum, activation, results to shared memory
      float* dstbuf = l1 ? hs : ys;
      if (live) {
#pragma unroll
        for (int r = 0; r < MLP_R; ++r)
          *reinterpret_cast<float4*>(red + (grp * MLP_R + r) * N + col) = make_float4(acc[r][0], acc[r][1], acc[r][2], acc[r][3]);
      }
      __syncthreads();
      for (int i = tid; i < MLP_R * N; i += MLP_NT) {
        const int r = i / N, n = i - r * N;
        float v = red[r * N + n];
        for (int g = 1; g < ng; ++g) v += red[(g * MLP_R + r) * N + n];
        dstbuf[r * N + n] = l1 ? di_act(v, act1) : v;
      }
    }
  }
  __syncthreads();                                   // results of the last layer visible
  const float* outs = W2t ? ys : hs;
  const int N = W2t ? N2 : N1;
  // finish: warp r owns row r (N <= 512 -> up to 16 values per lane)
  const int r = tid >> 5, lane = tid & 31, m = m0 + r;
  if (r >= MLP_R || m >= M) return;
  float x[16];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const int c = i * 32 + lane;
    float a = 0.f;
    if (c < N) {
      a = outs[r * N + c];
      if (res) a += res[(size_t)m * ldres + c];
      sum += a;
    }
    x[i] = a;
  }
  if (gamma) {
    const float mean = warp_sum(sum) / (float)N;
    float var = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int c = i * 32 + lane;
      if (c < N) {
        const float d = x[i] - mean;
        var += d * d;
      }
    }
    var = warp_sum(var) / (float)N;
    const float rstd = 1.f / sqrtf(var + eps);
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int c = i * 32 + lane;
      if (c < N) x[i] = (x[i] - mean) * rstd * gamma[c] + beta[c];
    }
  }
  const bool zero = zero_if_neg && zero_if_neg[m] < 0;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const int c = i * 32 + lane;
    if (c < N) Y[(size_t)m * ldy + c] = zero ? 0.f : di_act(x[i], act_out);
  }
}

// pred [M, NP]: center(0,1) height(2) dim(3..5) rot(6,7) vel(8,9) heatmap(10..).  center += query_pos;
// rows whose query fell on no image (win < 0) take the first layer's prediction (decoder.py:290-295).
__global__ void pred_finish_kernel(float* __restrict__ pred, float* __restrict__ qpos, const float* __restrict__ first,
                                   const int* __restrict__ win, int M, int NP) {
  int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  float* p = pred + (size_t)m * NP;
  p[0] += qpos[m * 2];
  p[1] += qpos[m * 2 + 1];
  if (win && first && win[m] < 0)
    for (int c = 0; c < NP; ++c) p[c] = first[(size_t)m * NP + c];
  qpos[m * 2] = p[0];
  qpos[m * 2 + 1] = p[1];
}

__global__ void pred_finish_pp_kernel(float* __restrict__ pred, float* __restrict__ qpos, float* __restrict__ look,
                                      const float* __restrict__ first, const int* __restrict__ win,
                                      int* __restrict__ keep, int first_layer, int M, int NP) {
  int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  float* p = pred + (size_t)m * NP;
  const float d0 = p[0], d1 = p[1];
  p[0] = d0 + look[m * 2];
  p[1] = d1 + look[m * 2 + 1];
  look[m * 2] = d0 + qpos[m * 2];
  look[m * 2 + 1] = d1 + qpos[m * 2 + 1];
  int k = first_layer ? 1 : keep[m];
  if (win) k = k && (win[m] >= 0);
  keep[m] = k;
  if (!k)
    for (int c = 0; c < NP; ++c) p[c] = first[(size_t)m * NP + c];
  qpos[m * 2] = p[0];
  qpos[m * 2 + 1] = p[1];
}

__global__ void rcnn_leaders_kernel(const int* __restrict__ onbits, int* __restrict__ lead_row, int* __restrict__ lead_win,
                                    int P, int V) {
  const int b = blockIdx.x / V, v = blockIdx.x % V, lane = threadIdx.x;
  int best = 0x7fffffff;
  for (int i = lane; i < P; i += 32)
    if ((onbits[b * P + i] >> v) & 1) best = min(best, i);
  for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
  if (lane == 0) {
    lead_row[blockIdx.x] = best < P ? b * P + best : -1;
    lead_win[blockIdx.x] = best < P ? v : -1;
  }
}

__global__ void take_rows_kernel(const float* __restrict__ src, int ld, const int* __restrict__ idx, float* __restrict__ out,
                                 int C) {
  const int r = blockIdx.x, i = idx[r];
  for (int c = threadIdx.x; c < C; c += blockDim.x) out[(size_t)r * C + c] = i >= 0 ? src[(size_t)i * ld + c] : 0.f;
}

__global__ void branch_mix_kernel(const float* __restrict__ a, const float* __restrict__ lead, const int* __restrict__ win,
                                  const float* __restrict__ scale, const float* __restrict__ self_scale,
                                  float* __restrict__ out, int C, int P, int V, int zero_off) {
  const int m = blockIdx.x, w = win[m];
  const float s = scale[0], t = self_scale[0];
  const float* l = lead + (size_t)((m / P) * V + (w < 0 ? 0 : w)) * C;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float y = __fadd_rn(__fmul_rn(a[(size_t)m * C + c], s), __fmul_rn(l[c], t));
    out[(size_t)m * C + c] = (w < 0 && zero_off) ? 0.f : y;
  }
}

// dst[idx[r], :C] += src[r, :C] for r = 0..R-1 in order, rows with idx[r] < 0 skipped: one thread per column walks every
// r, so equal indices are added in ascending r without atomics (R = B * V leader rows).
__global__ void rows_scatter_add_kernel(const float* __restrict__ src, int lds, const int* __restrict__ idx, float* __restrict__ dst,
                                        int ldd, int R, int C) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  for (int r = 0; r < R; ++r) {
    const int i = idx[r];
    if (i >= 0) dst[(size_t)i * ldd + c] += src[(size_t)r * lds + c];
  }
}

// sum of v over a CTA of 128 threads in a fixed order (warp butterfly, then the 4 warps in order); valid in thread 0
__device__ __forceinline__ float block128_sum(float v, float* red) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  return ((red[0] + red[1]) + red[2]) + red[3];
}

// The (sample, view) group row m feeds in branch_mix_kernel: its win, or view 0 for win < 0 without zero_off; -1 when the
// row is written as 0.
__device__ __forceinline__ int branch_group(int w, int zero_off) { return w >= 0 ? w : (zero_off ? -1 : 0); }

// Backward of branch_mix_kernel, one CTA of 128 per row m: da = dout * scale (0 on the zeroed rows) and the row's partial
// sums of dout * a and dout * lead (the d scale and d self_scale terms) into part[2m], part[2m + 1].
__global__ void __launch_bounds__(128)
branch_mix_bwd_rows_kernel(const float* __restrict__ dout, const float* __restrict__ a, const float* __restrict__ lead,
                           const int* __restrict__ win, const float* __restrict__ scale, float* __restrict__ da,
                           float* __restrict__ part, int C, int P, int V, int zero_off) {
  __shared__ float red[2][4];
  const int m = blockIdx.x, g = branch_group(win[m], zero_off);
  const float s = scale[0];
  const float* l = lead + (size_t)((m / P) * V + (g < 0 ? 0 : g)) * C;
  float ps = 0.f, pt = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float y = dout[(size_t)m * C + c];
    da[(size_t)m * C + c] = g < 0 ? 0.f : y * s;
    if (g >= 0) {
      ps += y * a[(size_t)m * C + c];
      pt += y * l[c];
    }
  }
  ps = block128_sum(ps, red[0]);
  pt = block128_sum(pt, red[1]);
  if (threadIdx.x == 0) {
    part[2 * m] = ps;
    part[2 * m + 1] = pt;
  }
}

// dlead[g = b * V + v] = self_scale * (sum of dout over the rows of sample b in group v, ascending row order): one CTA per
// group, one thread per channel; 0 for a group no row belongs to.
__global__ void branch_mix_bwd_lead_kernel(const float* __restrict__ dout, const int* __restrict__ win,
                                           const float* __restrict__ self_scale, float* __restrict__ dlead, int C, int P,
                                           int V, int zero_off) {
  const int b = blockIdx.x / V, v = blockIdx.x % V;
  const float t = self_scale[0];
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float acc = 0.f;
    for (int i = 0; i < P; ++i)
      if (branch_group(win[b * P + i], zero_off) == v) acc += dout[(size_t)(b * P + i) * C + c];
    dlead[(size_t)blockIdx.x * C + c] = t * acc;
  }
}

// d scale = sum_m part[2m], d self_scale = sum_m part[2m + 1]: one CTA of 128, each thread over m = t, t + 128, ...
__global__ void __launch_bounds__(128)
branch_mix_bwd_scales_kernel(const float* __restrict__ part, float* __restrict__ d_scale, float* __restrict__ d_self_scale,
                             int M) {
  __shared__ float red[2][4];
  float ps = 0.f, pt = 0.f;
  for (int m = threadIdx.x; m < M; m += blockDim.x) {
    ps += part[2 * m];
    pt += part[2 * m + 1];
  }
  ps = block128_sum(ps, red[0]);
  pt = block128_sum(pt, red[1]);
  if (threadIdx.x == 0) {
    d_scale[0] = ps;
    d_self_scale[0] = pt;
  }
}

// Backward of the ++ prediction finish over all L layers, one thread per (row m, column c): pred_l = keep_l ? delta_l (+ look_l
// on the centre) : first, look_{l+1} = delta_l[:, 0:2] + qpos_l (qpos and the first look detached), so
// d delta_l = keep_l dpred_l (+ keep_{l+1} dpred_{l+1} on columns 0, 1) and d first = sum_l !keep_l dpred_l, l ascending.
__global__ void pred_finish_pp_bwd_kernel(const float* __restrict__ dpred, const int* __restrict__ keep,
                                          float* __restrict__ d_delta, float* __restrict__ d_first, int L, int M, int NP) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= M * NP) return;
  const int m = e / NP, c = e % NP;
  const size_t LS = (size_t)M * NP;
  float f = 0.f;
  for (int l = 0; l < L; ++l) {
    const float g = dpred[l * LS + e];
    const bool k = keep[(size_t)l * M + m] != 0;
    float d = k ? g : 0.f;
    if (c < 2 && l + 1 < L && keep[(size_t)(l + 1) * M + m]) d += dpred[(l + 1) * LS + e];
    d_delta[l * LS + e] = d;
    if (!k) f += g;
  }
  d_first[e] = f;
}

// ------------------------------------------------------------------------------------------------
// RoI generation.  mode 0 (image, decoder_utils.py:660-741): box centre + 8 corners -> every view,
// on-image test on the centre, views with <= 1 query skipped, later views win.
// mode 1 (BEV, :788-819): footprint of the box with doubled dims in BEV cells.
// ------------------------------------------------------------------------------------------------
struct RoiParams {
  float sx, sy, ox, oy;        // bbox_coder: out_size_factor*voxel_size[0|1], pc_range[0|1]
  float csx, cox;              // test_cfg: out_size_factor*voxel_size[0], pc_range[0] (centre path uses index 0 twice)
  float h_pad, w_pad;          // input_shape
  float bev_scale, bev_off;    // bbox_coder.voxel_size[0]*out_size_factor, bbox_coder.pc_range[0]
};

__device__ __forceinline__ void box_corners_xy(float cx, float cy, float dx, float dy, float yaw, float* xs, float* ys) {
  // mmdet3d 0.17.1 LiDARInstance3DBoxes.corners: (dims * ({0,1}^3 - (.5,.5,0))) @ [[c,-s],[s,c]] + centre
  float c = cosf(yaw), s = sinf(yaw);
  int n = 0;
  for (int ix = 0; ix < 2; ++ix)
    for (int iy = 0; iy < 2; ++iy) {
      float lx = dx * ((float)ix - 0.5f), ly = dy * ((float)iy - 0.5f);
      xs[n] = lx * c + ly * s + cx;
      ys[n] = -lx * s + ly * c + cy;
      ++n;
    }
}

constexpr int MAXV = 8;

__global__ void __launch_bounds__(1024)
rcnn_rois_kernel(const float* __restrict__ pred, int NP, const float* __restrict__ proj, const float* __restrict__ aux,
                 float* __restrict__ rois, int* __restrict__ win, int* __restrict__ onbits, int P, int V, int mode,
                 RoiParams rp) {
  __shared__ int cnt[MAXV];
  const int b = blockIdx.x, qi = threadIdx.x;
  if (qi < MAXV) cnt[qi] = 0;
  __syncthreads();
  const bool act = qi < P;
  const int bq = b * P + qi;
  float rect[MAXV][4];
  int bits = 0;
  float cxr = 0, cyr = 0, dx = 0, dy = 0, dz = 0, yaw = 0, zc = 0, zb = 0;
  if (act) {
    const float* p = pred + (size_t)bq * NP;
    cxr = p[0] * rp.sx + rp.ox;
    cyr = p[1] * rp.sy + rp.oy;
    dx = expf(p[3]); dy = expf(p[4]); dz = expf(p[5]);
    zc = p[2];
    zb = zc - dz * 0.5f;
    yaw = atan2f(p[6], p[7]);
  }
  if (mode == 1) {
    if (act) {
      float xs[4], ys[4];
      box_corners_xy(cxr, cyr, dx * 2.f, dy * 2.f, yaw, xs, ys);
      float x0 = INFINITY, y0 = INFINITY, x1 = -INFINITY, y1 = -INFINITY;
      for (int i = 0; i < 4; ++i) {
        float u = (xs[i] - rp.bev_off) / rp.bev_scale, v = (ys[i] - rp.bev_off) / rp.bev_scale;
        x0 = fminf(x0, u); x1 = fmaxf(x1, u); y0 = fminf(y0, v); y1 = fmaxf(y1, v);
      }
      float* r = rois + (size_t)bq * 5;
      r[0] = (float)b; r[1] = x0; r[2] = y0; r[3] = x1; r[4] = y1;
      win[bq] = 0;
      onbits[bq] = 1;
    }
    return;
  }
  if (act) {
    // centre used for the on-image test: (centre_real via test_cfg, raw height)
    float ccx = pred[(size_t)bq * NP] * rp.csx + rp.cox, ccy = pred[(size_t)bq * NP + 1] * rp.csx + rp.cox;
    float xs[4], ys[4];
    box_corners_xy(cxr, cyr, dx, dy, yaw, xs, ys);
    const float* ax = aux + b * 4;  // crop_x, crop_y, flip (0/1), orig_w
    for (int v = 0; v < V; ++v) {
      const float* M = proj + ((size_t)b * V + v) * 12;
      auto prj = [&](float X, float Y, float Z, float& u, float& w) {
        float a = M[0] * X + M[1] * Y + M[2] * Z + M[3];
        float bb = M[4] * X + M[5] * Y + M[6] * Z + M[7];
        float c = fmaxf(M[8] * X + M[9] * Y + M[10] * Z + M[11], 1e-5f);
        u = a / c - ax[0];
        w = bb / c - ax[1];
        if (ax[2] != 0.f) u = ax[3] - u;
      };
      float u, w;
      prj(ccx, ccy, zc, u, w);
      bool on = (u > 0.f) && (u < rp.w_pad) && (w > 0.f) && (w < rp.h_pad);
      float x0 = INFINITY, y0 = INFINITY, x1 = -INFINITY, y1 = -INFINITY;
      for (int i = 0; i < 4; ++i)
        for (int iz = 0; iz < 2; ++iz) {
          prj(xs[i], ys[i], zb + (iz ? dz : 0.f), u, w);
          x0 = fminf(x0, u); x1 = fmaxf(x1, u); y0 = fminf(y0, w); y1 = fmaxf(y1, w);
        }
      rect[v][0] = x0; rect[v][1] = y0; rect[v][2] = x1; rect[v][3] = y1;
      if (on) {
        bits |= 1 << v;
        atomicAdd(&cnt[v], 1);
      }
    }
  }
  __syncthreads();
  if (act) {
    int w = -1;
    for (int v = 0; v < V; ++v)
      if (((bits >> v) & 1) && cnt[v] > 1) w = v;
    int live = 0;  // views that were actually processed (count > 1)
    for (int v = 0; v < V; ++v)
      if (cnt[v] > 1) live |= 1 << v;
    float* r = rois + (size_t)bq * 5;
    r[0] = w >= 0 ? (float)(b * V + w) : -1.f;
    for (int i = 0; i < 4; ++i) r[1 + i] = w >= 0 ? rect[w][i] : 0.f;
    win[bq] = w;
    onbits[bq] = bits & live;
  }
}

// ------------------------------------------------------------------------------------------------
// RoIAlign (detectron2 ROIAlignV2 == aligned=True), 7x7 bins, 2x2 samples per bin, pixel-major map.
// One warp per (roi, bin).  out [n, 49, C].
// ------------------------------------------------------------------------------------------------
template <int NJ>
__global__ void __launch_bounds__(256)
roi_align_kernel(const float* __restrict__ maps, const float* __restrict__ rois, float* __restrict__ out, int n, int H,
                 int W, int C, float scale) {
  constexpr int R = 7, G = 2;
  int wid = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  int lane = threadIdx.x & 31;
  if (wid >= n * R * R) return;
  int bin = wid % (R * R), ri = wid / (R * R);
  int ph = bin / R, pw = bin % R;
  const float* r = rois + (size_t)ri * 5;
  int mi = (int)r[0];
  float4 acc[NJ];
#pragma unroll
  for (int j = 0; j < NJ; ++j) acc[j] = make_float4(0, 0, 0, 0);
  if (mi >= 0) {
    const float* map = maps + (size_t)mi * H * W * C;
    float x0 = r[1] * scale - 0.5f, y0 = r[2] * scale - 0.5f;
    float x1 = r[3] * scale - 0.5f, y1 = r[4] * scale - 0.5f;
    float bw = (x1 - x0) / (float)R, bh = (y1 - y0) / (float)R;
    for (int iy = 0; iy < G; ++iy)
      for (int ix = 0; ix < G; ++ix) {
        float y = y0 + (float)ph * bh + ((float)iy + 0.5f) * bh / (float)G;
        float x = x0 + (float)pw * bw + ((float)ix + 0.5f) * bw / (float)G;
        if (y < -1.f || y > (float)H || x < -1.f || x > (float)W) continue;
        if (!(y == y) || !(x == x)) continue;
        y = fmaxf(y, 0.f);
        x = fmaxf(x, 0.f);
        int yl = (int)y, xl = (int)x, yh, xh;
        if (yl >= H - 1) { yh = yl = H - 1; y = (float)yl; } else yh = yl + 1;
        if (xl >= W - 1) { xh = xl = W - 1; x = (float)xl; } else xh = xl + 1;
        float ly = y - (float)yl, lx = x - (float)xl, hy = 1.f - ly, hx = 1.f - lx;
        float wg[4] = {hy * hx, hy * lx, ly * hx, ly * lx};
        const float* rows[4] = {map + ((size_t)yl * W + xl) * C, map + ((size_t)yl * W + xh) * C,
                                map + ((size_t)yh * W + xl) * C, map + ((size_t)yh * W + xh) * C};
#pragma unroll
        for (int cnr = 0; cnr < 4; ++cnr)
#pragma unroll
          for (int j = 0; j < NJ; ++j) {
            int c = 4 * lane + 128 * j;
            if (c < C) {
              float4 t4 = ldg4(rows[cnr] + c);
              acc[j].x += wg[cnr] * t4.x; acc[j].y += wg[cnr] * t4.y;
              acc[j].z += wg[cnr] * t4.z; acc[j].w += wg[cnr] * t4.w;
            }
          }
      }
  }
  const float inv = 1.f / (float)(G * G);
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    int c = 4 * lane + 128 * j;
    if (c < C)
      *reinterpret_cast<float4*>(out + ((size_t)ri * R * R + bin) * C + c) =
          make_float4(acc[j].x * inv, acc[j].y * inv, acc[j].z * inv, acc[j].w * inv);
  }
}

// ------------------------------------------------------------------------------------------------
// RoIAlign backward: d_maps [n_maps, H, W, C] from d_out [n, 49, C], as a gather (no atomics, deterministic).
// The forward's bilinear weight is separable: pixel (py, px) receives from bin (ph, pw) the weight
// Ay[ph](py) Ax[pw](px) / 4, where Ay[ph](py) sums over the bin's two y-samples that sample's row weight on py (0 for a
// skipped sample) and Ax is the same along x.  A sample is skipped when y or x is out of [-1, L] or NaN, so the skip
// factor of a sample is the product of a y and an x factor.  A CTA owns a 4 x 8 pixel tile of one map; it culls the RoI
// list against the tile, 256 RoIs at a time, into an ascending list in shared memory; each warp owns 4 pixels of one tile
// row (lanes over channels, the sums in registers) and adds the surviving RoIs in ascending RoI index, bins in ascending
// order.  Pixels no sample reaches get exactly 0.
// ------------------------------------------------------------------------------------------------
constexpr int RB_TY = 4, RB_TX = 8, RB_PPW = 4, RB_T = 256;

// One axis sample of roi_align_kernel (bin p, sub-sample i of 2; start a0, bin size bsz, L pixels): false when skipped,
// else the two taps lo, hi (equal at the last pixel) and their weights.  The expressions are the forward's.
__device__ __forceinline__ bool roi_axis_sample(float a0, float bsz, int p, int i, int L, int& lo, int& hi, float& wlo,
                                                float& whi) {
  float y = a0 + (float)p * bsz + ((float)i + 0.5f) * bsz / (float)2;
  if (y < -1.f || y > (float)L) return false;
  if (!(y == y)) return false;
  y = fmaxf(y, 0.f);
  lo = (int)y;
  if (lo >= L - 1) { hi = lo = L - 1; y = (float)lo; } else hi = lo + 1;
  const float l = y - (float)lo;
  wlo = 1.f - l;
  whi = l;
  return true;
}

// weights a[p] of pixel q on the 7 bins of one axis
__device__ __forceinline__ bool roi_axis_weights(float a0, float bsz, int L, int q, float (&a)[7]) {
  bool any = false;
#pragma unroll
  for (int p = 0; p < 7; ++p) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      int lo, hi;
      float wl, wh;
      if (roi_axis_sample(a0, bsz, p, i, L, lo, hi, wl, wh)) {
        if (lo == q) s += wl;
        if (hi == q) s += wh;
      }
    }
    a[p] = s;
    any |= s != 0.f;
  }
  return any;
}

// [first, last] pixel an axis' samples touch (last < 0: none)
__device__ __forceinline__ void roi_axis_span(float a0, float bsz, int L, int& first, int& last) {
  first = L;
  last = -1;
  for (int p = 0; p < 7; ++p)
    for (int i = 0; i < 2; ++i) {
      int lo, hi;
      float wl, wh;
      if (roi_axis_sample(a0, bsz, p, i, L, lo, hi, wl, wh)) {
        first = min(first, lo);
        last = max(last, hi);
      }
    }
}

template <int NJ>
__global__ void __launch_bounds__(RB_T)
roi_align_bwd_kernel(const float* __restrict__ rois, const float* __restrict__ dout, float* __restrict__ dmaps, int n, int H,
                     int W, int C, float scale, int tiles_x) {
  constexpr int R = 7;
  __shared__ int list[RB_T];
  __shared__ int wcount[RB_T / 32];
  const int map = blockIdx.y;
  const int ty0 = (blockIdx.x / tiles_x) * RB_TY, tx0 = (blockIdx.x % tiles_x) * RB_TX;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int py = ty0 + (warp >> 1), px0 = tx0 + (warp & 1) * RB_PPW;
  float4 acc[RB_PPW][NJ];
#pragma unroll
  for (int q = 0; q < RB_PPW; ++q)
#pragma unroll
    for (int j = 0; j < NJ; ++j) acc[q][j] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int c0 = 0; c0 < n; c0 += RB_T) {
    const int ri = c0 + t;
    bool hit = false;
    if (ri < n) {
      const float* r = rois + (size_t)ri * 5;
      if ((int)r[0] == map) {
        const float x0 = r[1] * scale - 0.5f, y0 = r[2] * scale - 0.5f;
        const float x1 = r[3] * scale - 0.5f, y1 = r[4] * scale - 0.5f;
        const float bw = (x1 - x0) / (float)R, bh = (y1 - y0) / (float)R;
        int yf, yl, xf, xl;
        roi_axis_span(y0, bh, H, yf, yl);
        roi_axis_span(x0, bw, W, xf, xl);
        hit = yl >= 0 && xl >= 0 && yf < ty0 + RB_TY && yl >= ty0 && xf < tx0 + RB_TX && xl >= tx0;
      }
    }
    const unsigned b = __ballot_sync(0xffffffffu, hit);
    if (lane == 0) wcount[warp] = __popc(b);
    __syncthreads();
    int base = 0, total = 0;
#pragma unroll
    for (int w = 0; w < RB_T / 32; ++w) {
      base += w < warp ? wcount[w] : 0;
      total += wcount[w];
    }
    if (hit) list[base + __popc(b & ((1u << lane) - 1u))] = ri;
    __syncthreads();
    for (int s = 0; s < total; ++s) {
      const int ri2 = list[s];
      const float* r = rois + (size_t)ri2 * 5;
      const float x0 = r[1] * scale - 0.5f, y0 = r[2] * scale - 0.5f;
      const float x1 = r[3] * scale - 0.5f, y1 = r[4] * scale - 0.5f;
      const float bw = (x1 - x0) / (float)R, bh = (y1 - y0) / (float)R;
      float ay[7];
      if (!roi_axis_weights(y0, bh, H, py, ay)) continue;        // warp-uniform
      const float* g = dout + (size_t)ri2 * R * R * C;
#pragma unroll
      for (int q = 0; q < RB_PPW; ++q) {
        float ax[7];
        if (!roi_axis_weights(x0, bw, W, px0 + q, ax)) continue;
        for (int ph = 0; ph < R; ++ph) {
          if (ay[ph] == 0.f) continue;
          for (int pw = 0; pw < R; ++pw) {
            const float wgt = ay[ph] * ax[pw];
            if (wgt == 0.f) continue;
#pragma unroll
            for (int j = 0; j < NJ; ++j) {
              const int c = 4 * lane + 128 * j;
              if (c < C) {
                const float4 v = ldg4(g + (size_t)(ph * R + pw) * C + c);
                acc[q][j].x = fmaf(wgt, v.x, acc[q][j].x); acc[q][j].y = fmaf(wgt, v.y, acc[q][j].y);
                acc[q][j].z = fmaf(wgt, v.z, acc[q][j].z); acc[q][j].w = fmaf(wgt, v.w, acc[q][j].w);
              }
            }
          }
        }
      }
    }
    __syncthreads();                                     // the list is rewritten by the next chunk
  }
  const float inv = 1.f / (float)(2 * 2);
#pragma unroll
  for (int q = 0; q < RB_PPW; ++q) {
    const int px = px0 + q;
    if (py >= H || px >= W) continue;
    float* dst = dmaps + (((size_t)map * H + py) * W + px) * C;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int c = 4 * lane + 128 * j;
      if (c < C)
        *reinterpret_cast<float4*>(dst + c) = make_float4(acc[q][j].x * inv, acc[q][j].y * inv, acc[q][j].z * inv, acc[q][j].w * inv);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// DynamicConv core (decoder_utils.py:610-624), hidden = dim_dynamic = 128, 49 RoI bins:
//   f1 = relu(LN1(F @ P1)); f2 = relu(LN2(f1 @ P2)); out = f2 flattened [49*128].  One CTA per query.
// ------------------------------------------------------------------------------------------------
constexpr int DC = 128, DR = 49;

constexpr int DYN_T = 512;       // 16 warps: rows ty, ty + 16, ... per thread (the product loop is latency-bound at 8 warps)
constexpr int DYN_NW = DYN_T / 32;
constexpr int DYN_NR = (DR + DYN_NW - 1) / DYN_NW;      // 4

// acc[i] = X[ty + 16 i][:] . Pm[:][4 tx .. 4 tx + 3] (Pm [c][d] in shared memory), the product loop of dynconv_kernel and of
// the recompute in dynconv_bwd_kernel: one accumulation order over c, so both see the same LayerNorm inputs.
// register tile: thread = 4 output columns (4 tx .. 4 tx + 3) x the rows ty, ty + 16, ... (4 rows); per 4 input channels
// 4 parameter loads (float4) and 4 broadcast activation loads feed 64 FMAs (the one-column mapping spent one
// 16-byte shared-memory load per 4 FMAs and was bound by the shared-memory pipe).
__device__ __forceinline__ void dyn_rows_times(const float (*X)[DC], const float* Pm, float4 (&acc)[DYN_NR], int tx, int ty) {
#pragma unroll
  for (int i = 0; i < DYN_NR; ++i) acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 2
  for (int c = 0; c < DC; c += 4) {
    const float4 p0 = *reinterpret_cast<const float4*>(Pm + (c + 0) * DC + 4 * tx), p1 = *reinterpret_cast<const float4*>(Pm + (c + 1) * DC + 4 * tx);
    const float4 p2 = *reinterpret_cast<const float4*>(Pm + (c + 2) * DC + 4 * tx), p3 = *reinterpret_cast<const float4*>(Pm + (c + 3) * DC + 4 * tx);
#pragma unroll
    for (int i = 0; i < DYN_NR; ++i) {
      const int r = ty + DYN_NW * i;
      if (r < DR) {
        const float4 x = *reinterpret_cast<const float4*>(&X[r][c]);
        acc[i].x = fmaf(x.x, p0.x, acc[i].x); acc[i].y = fmaf(x.x, p0.y, acc[i].y);
        acc[i].z = fmaf(x.x, p0.z, acc[i].z); acc[i].w = fmaf(x.x, p0.w, acc[i].w);
        acc[i].x = fmaf(x.y, p1.x, acc[i].x); acc[i].y = fmaf(x.y, p1.y, acc[i].y);
        acc[i].z = fmaf(x.y, p1.z, acc[i].z); acc[i].w = fmaf(x.y, p1.w, acc[i].w);
        acc[i].x = fmaf(x.z, p2.x, acc[i].x); acc[i].y = fmaf(x.z, p2.y, acc[i].y);
        acc[i].z = fmaf(x.z, p2.z, acc[i].z); acc[i].w = fmaf(x.z, p2.w, acc[i].w);
        acc[i].x = fmaf(x.w, p3.x, acc[i].x); acc[i].y = fmaf(x.w, p3.y, acc[i].y);
        acc[i].z = fmaf(x.w, p3.z, acc[i].z); acc[i].w = fmaf(x.w, p3.w, acc[i].w);
      }
    }
  }
}

__global__ void __launch_bounds__(DYN_T)
dynconv_kernel(const float* __restrict__ roi, const float* __restrict__ params, const float* __restrict__ g1,
               const float* __restrict__ b1, const float* __restrict__ g2, const float* __restrict__ b2,
               float* __restrict__ out, float eps) {
  extern __shared__ __align__(16) float dyn_smem[];
  float(*F)[DC] = reinterpret_cast<float(*)[DC]>(dyn_smem);
  float(*T)[DC] = reinterpret_cast<float(*)[DC]>(dyn_smem + DR * DC);
  const int qn = blockIdx.x, t = threadIdx.x;
  // the query's two 128 x 128 parameter matrices (128 KB, written by the generator GEMM just before) are pulled into
  // shared memory with cp.async while the RoI tile loads: reading them with dependent __ldg batches inside the product
  // loop leaves the kernel latency-bound
  float* PS = dyn_smem + 2 * DR * DC;                    // [2][DC][DC]
  {
    const float* psrc = params + (size_t)qn * 2 * DC * DC;
    for (int l = 0; l < 2; ++l) {
      for (int i = t * 4; i < DC * DC; i += DYN_T * 4)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(tc::smem_u32(PS + l * DC * DC + i)), "l"(psrc + l * DC * DC + i)
                     : "memory");
      asm volatile("cp.async.commit_group;" ::: "memory");
    }
  }
  const float* src = roi + (size_t)qn * DR * DC;
  for (int i = t; i < DR * DC / 4; i += blockDim.x)
    reinterpret_cast<float4*>(&F[0][0])[i] = ldg4(src + i * 4);
  asm volatile("cp.async.wait_group 1;" ::: "memory");
  __syncthreads();
  const int tx = t & 31, ty = t >> 5;
  for (int layer = 0; layer < 2; ++layer) {
    if (layer == 1) {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
      __syncthreads();
    }
    const float* Pm = PS + layer * DC * DC;               // [c][d] in shared memory
    float(*X)[DC] = layer == 0 ? F : T;
    float4 acc[DYN_NR];
    dyn_rows_times(X, Pm, acc, tx, ty);
    __syncthreads();  // everyone finished reading X before it may be overwritten
    float(*Y)[DC] = layer == 0 ? T : F;
#pragma unroll
    for (int i = 0; i < DYN_NR; ++i) {
      const int r = ty + DYN_NW * i;
      if (r < DR) *reinterpret_cast<float4*>(&Y[r][4 * tx]) = acc[i];
    }
    __syncthreads();
    // LayerNorm over d + ReLU, one warp per row
    const float* g = layer == 0 ? g1 : g2;
    const float* bb = layer == 0 ? b1 : b2;
    for (int r = t >> 5; r < DR; r += (blockDim.x >> 5)) {
      int lane = t & 31;
      float4 x = *reinterpret_cast<const float4*>(&Y[r][lane * 4]);
      float mean = warp_sum(x.x + x.y + x.z + x.w) / (float)DC;
      float dx0 = x.x - mean, dx1 = x.y - mean, dx2 = x.z - mean, dx3 = x.w - mean;
      float var = warp_sum(dx0 * dx0 + dx1 * dx1 + dx2 * dx2 + dx3 * dx3) / (float)DC;
      float rstd = 1.f / sqrtf(var + eps);
      float4 gg = ldg4(g + lane * 4), be = ldg4(bb + lane * 4);
      float4 y;
      y.x = fmaxf(dx0 * rstd * gg.x + be.x, 0.f);
      y.y = fmaxf(dx1 * rstd * gg.y + be.y, 0.f);
      y.z = fmaxf(dx2 * rstd * gg.z + be.z, 0.f);
      y.w = fmaxf(dx3 * rstd * gg.w + be.w, 0.f);
      *reinterpret_cast<float4*>(&Y[r][lane * 4]) = y;
    }
    __syncthreads();
  }
  // after layer 1 the result is in F
  float* dst = out + (size_t)qn * DR * DC;
  for (int i = t; i < DR * DC / 4; i += blockDim.x)
    *reinterpret_cast<float4*>(dst + i * 4) = reinterpret_cast<const float4*>(&F[0][0])[i];
}

// ------------------------------------------------------------------------------------------------
// DynamicConv backward.  One CTA per query; the forward is recomputed in shared memory with dyn_rows_times and the
// forward's LayerNorm statistics code, so Z1, Z2 and the statistics equal the forward's bit for bit.  Per query:
//   dA2 = dY2 * [Y2 > 0]; LN2 backward -> dZ2 (in place of x^2); dP2 = Y1^T dZ2; dY1 = dZ2 P2^T;
//   dA1 = dY1 * [Y1 > 0]; LN1 backward -> dZ1 (in place of dY1); dP1 = F^T dZ1; dF = dZ1 P1^T.
// Shared memory: P1, P2 (128 KB) and four 49 x 128 tiles F, x^1, Y1 (then dY1, dZ1), x^2 (then dZ2): 231 424 B.
// LayerNorm parameter gradients: per query partials (one thread per column, rows in ascending order), reduced by the
// caller in a fixed order.  Every output element is written once: no atomics, deterministic.
// ------------------------------------------------------------------------------------------------
// out[c][d] = sum_r A[r][c] B[r][d] (128 x 128, to global memory): thread = columns 4 tx .. 4 tx + 3 of the rows
// c = ty + 16 i (B loads are float4 rows, A loads warp broadcasts)
__device__ __forceinline__ void dyn_at_b(const float (*A)[DC], const float (*Bm)[DC], float* __restrict__ out, int tx, int ty) {
  constexpr int NC = DC / DYN_NW;      // 8
  float4 acc[NC];
#pragma unroll
  for (int i = 0; i < NC; ++i) acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int r = 0; r < DR; ++r) {
    const float4 bv = *reinterpret_cast<const float4*>(&Bm[r][4 * tx]);
#pragma unroll
    for (int i = 0; i < NC; ++i) {
      const float a = A[r][ty + DYN_NW * i];
      acc[i].x = fmaf(a, bv.x, acc[i].x); acc[i].y = fmaf(a, bv.y, acc[i].y);
      acc[i].z = fmaf(a, bv.z, acc[i].z); acc[i].w = fmaf(a, bv.w, acc[i].w);
    }
  }
#pragma unroll
  for (int i = 0; i < NC; ++i) *reinterpret_cast<float4*>(out + (size_t)(ty + DYN_NW * i) * DC + 4 * tx) = acc[i];
}

// acc[i][j] = X[ty + 16 i][:] . Pm[tx + 32 j][:] (rows times Pm transposed).  Lane tx starts its walk over d at 4 tx, so the
// 16-byte loads of one quarter-warp cover all 32 banks (rows of X and of Pm are 128 floats apart).
__device__ __forceinline__ void dyn_rows_times_t(const float (*X)[DC], const float* Pm, float (&acc)[DYN_NR][4], int tx, int ty) {
#pragma unroll
  for (int i = 0; i < DYN_NR; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k = 0; k < DC / 4; ++k) {
    const int d = ((k + tx) & (DC / 4 - 1)) * 4;
    float4 p[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) p[j] = *reinterpret_cast<const float4*>(Pm + (tx + 32 * j) * DC + d);
#pragma unroll
    for (int i = 0; i < DYN_NR; ++i) {
      const int r = ty + DYN_NW * i;
      if (r < DR) {
        const float4 x = *reinterpret_cast<const float4*>(&X[r][d]);
#pragma unroll
        for (int j = 0; j < 4; ++j)
          acc[i][j] = fmaf(x.w, p[j].w, fmaf(x.z, p[j].z, fmaf(x.y, p[j].y, fmaf(x.x, p[j].x, acc[i][j]))));
      }
    }
  }
}

// Z (in place) -> x^ = (Z - mean) rstd with the forward's statistics code; Y = relu(x^ g + b) (Y may be null)
__device__ __forceinline__ void dyn_ln_fwd_rows(float (*Z)[DC], float (*Y)[DC], const float* __restrict__ g,
                                                const float* __restrict__ b, float* rstd_out, float eps, int t) {
  for (int r = t >> 5; r < DR; r += DYN_NW) {
    const int lane = t & 31;
    float4 x = *reinterpret_cast<const float4*>(&Z[r][lane * 4]);
    float mean = warp_sum(x.x + x.y + x.z + x.w) / (float)DC;
    float dx0 = x.x - mean, dx1 = x.y - mean, dx2 = x.z - mean, dx3 = x.w - mean;
    float var = warp_sum(dx0 * dx0 + dx1 * dx1 + dx2 * dx2 + dx3 * dx3) / (float)DC;
    float rstd = 1.f / sqrtf(var + eps);
    const float4 xh = make_float4(dx0 * rstd, dx1 * rstd, dx2 * rstd, dx3 * rstd);
    *reinterpret_cast<float4*>(&Z[r][lane * 4]) = xh;
    if (Y) {
      const float4 gg = ldg4(g + lane * 4), be = ldg4(b + lane * 4);
      *reinterpret_cast<float4*>(&Y[r][lane * 4]) = make_float4(fmaxf(xh.x * gg.x + be.x, 0.f), fmaxf(xh.y * gg.y + be.y, 0.f),
                                                                fmaxf(xh.z * gg.z + be.z, 0.f), fmaxf(xh.w * gg.w + be.w, 0.f));
    }
    if (lane == 0) rstd_out[r] = rstd;
  }
}

// per-query dgamma / dbeta of relu(LN(.)): thread c < 128 sums dA x^ and dA over the rows in ascending order
__device__ __forceinline__ void dyn_ln_col(const float* dy, const float (*Xh)[DC], const float* __restrict__ g,
                                           const float* __restrict__ b, float* out_g, float* out_b, int t) {
  if (t >= DC) return;
  const float gc = __ldg(g + t), bc = __ldg(b + t);
  float sg = 0.f, sb = 0.f;
  for (int r = 0; r < DR; ++r) {
    const float xh = Xh[r][t];
    const float da = xh * gc + bc > 0.f ? dy[r * DC + t] : 0.f;
    sg = fmaf(da, xh, sg);
    sb += da;
  }
  out_g[t] = sg;
  out_b[t] = sb;
}

// dZ = rstd (dx^ - mean(dx^) - x^ mean(dx^ x^)), dx^ = dA g, dA = dY [x^ g + b > 0]; one warp per row, dZ may alias dY
__device__ __forceinline__ void dyn_ln_bwd_rows(const float* dy, const float (*Xh)[DC], float (*Dz)[DC], const float* __restrict__ g,
                                                const float* __restrict__ b, const float* rstd, int t) {
  const int lane = t & 31;
  const float4 gg = ldg4(g + lane * 4), be = ldg4(b + lane * 4);
  for (int r = t >> 5; r < DR; r += DYN_NW) {
    const float4 d = *reinterpret_cast<const float4*>(dy + r * DC + lane * 4);
    const float4 x = *reinterpret_cast<const float4*>(&Xh[r][lane * 4]);
    const float h0 = (x.x * gg.x + be.x > 0.f ? d.x : 0.f) * gg.x, h1 = (x.y * gg.y + be.y > 0.f ? d.y : 0.f) * gg.y;
    const float h2 = (x.z * gg.z + be.z > 0.f ? d.z : 0.f) * gg.z, h3 = (x.w * gg.w + be.w > 0.f ? d.w : 0.f) * gg.w;
    const float s1 = warp_sum(h0 + h1 + h2 + h3) / (float)DC;
    const float s2 = warp_sum(h0 * x.x + h1 * x.y + h2 * x.z + h3 * x.w) / (float)DC;
    const float rs = rstd[r];
    *reinterpret_cast<float4*>(&Dz[r][lane * 4]) = make_float4((h0 - s1 - x.x * s2) * rs, (h1 - s1 - x.y * s2) * rs,
                                                               (h2 - s1 - x.z * s2) * rs, (h3 - s1 - x.w * s2) * rs);
  }
}

constexpr int DYN_BWD_SMEM = (2 * DC * DC + 4 * DR * DC) * (int)sizeof(float);    // 231 424 B

__global__ void __launch_bounds__(DYN_T)
dynconv_bwd_kernel(const float* __restrict__ roi, const float* __restrict__ params, const float* __restrict__ g1,
                   const float* __restrict__ b1, const float* __restrict__ g2, const float* __restrict__ b2,
                   const float* __restrict__ dout, float* __restrict__ droi, float* __restrict__ dparams,
                   float* __restrict__ dnorm, float eps) {
  extern __shared__ __align__(16) float dyn_smem[];
  __shared__ float rstd[2][DR];
  float* PS = dyn_smem;                                                          // P1 | P2, [c][d]
  float(*F)[DC] = reinterpret_cast<float(*)[DC]>(dyn_smem + 2 * DC * DC);
  float(*X1)[DC] = F + DR;              // x^1
  float(*Y1)[DC] = F + 2 * DR;          // relu(LN1), then dY1, then dZ1
  float(*X2)[DC] = F + 3 * DR;          // x^2, then dZ2
  const int qn = blockIdx.x, t = threadIdx.x, tx = t & 31, ty = t >> 5;
  {
    const float* psrc = params + (size_t)qn * 2 * DC * DC;
    for (int l = 0; l < 2; ++l) {
      for (int i = t * 4; i < DC * DC; i += DYN_T * 4)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(tc::smem_u32(PS + l * DC * DC + i)), "l"(psrc + l * DC * DC + i)
                     : "memory");
      asm volatile("cp.async.commit_group;" ::: "memory");
    }
  }
  const float* src = roi + (size_t)qn * DR * DC;
  for (int i = t; i < DR * DC / 4; i += DYN_T) reinterpret_cast<float4*>(&F[0][0])[i] = ldg4(src + i * 4);
  asm volatile("cp.async.wait_group 1;" ::: "memory");
  __syncthreads();
  // forward recompute
  float4 acc[DYN_NR];
  dyn_rows_times(F, PS, acc, tx, ty);
#pragma unroll
  for (int i = 0; i < DYN_NR; ++i)
    if (ty + DYN_NW * i < DR) *reinterpret_cast<float4*>(&X1[ty + DYN_NW * i][4 * tx]) = acc[i];
  __syncthreads();
  dyn_ln_fwd_rows(X1, Y1, g1, b1, rstd[0], eps, t);
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  __syncthreads();
  dyn_rows_times(Y1, PS + DC * DC, acc, tx, ty);
#pragma unroll
  for (int i = 0; i < DYN_NR; ++i)
    if (ty + DYN_NW * i < DR) *reinterpret_cast<float4*>(&X2[ty + DYN_NW * i][4 * tx]) = acc[i];
  __syncthreads();
  dyn_ln_fwd_rows(X2, nullptr, g2, b2, rstd[1], eps, t);
  __syncthreads();
  // second layer
  const float* dy2 = dout + (size_t)qn * DR * DC;
  float* dn = dnorm + (size_t)qn * 4 * DC;                 // dgamma1 | dbeta1 | dgamma2 | dbeta2
  dyn_ln_col(dy2, X2, g2, b2, dn + 2 * DC, dn + 3 * DC, t);
  __syncthreads();
  dyn_ln_bwd_rows(dy2, X2, X2, g2, b2, rstd[1], t);
  __syncthreads();
  float* dp = dparams + (size_t)qn * 2 * DC * DC;
  dyn_at_b(Y1, X2, dp + DC * DC, tx, ty);                  // dP2 = Y1^T dZ2
  float acc2[DYN_NR][4];
  dyn_rows_times_t(X2, PS + DC * DC, acc2, tx, ty);        // dY1 = dZ2 P2^T
  __syncthreads();
#pragma unroll
  for (int i = 0; i < DYN_NR; ++i)
    if (ty + DYN_NW * i < DR)
#pragma unroll
      for (int j = 0; j < 4; ++j) Y1[ty + DYN_NW * i][tx + 32 * j] = acc2[i][j];
  __syncthreads();
  // first layer
  dyn_ln_col(&Y1[0][0], X1, g1, b1, dn, dn + DC, t);
  __syncthreads();
  dyn_ln_bwd_rows(&Y1[0][0], X1, Y1, g1, b1, rstd[0], t);
  __syncthreads();
  dyn_at_b(F, Y1, dp, tx, ty);                              // dP1 = F^T dZ1
  dyn_rows_times_t(Y1, PS, acc2, tx, ty);                   // dF = dZ1 P1^T
  float* dst = droi + (size_t)qn * DR * DC;
#pragma unroll
  for (int i = 0; i < DYN_NR; ++i)
    if (ty + DYN_NW * i < DR)
#pragma unroll
      for (int j = 0; j < 4; ++j) dst[(ty + DYN_NW * i) * DC + tx + 32 * j] = acc2[i][j];
}

// dx = dy (Phi(h) + h phi(h)): the derivative of the exact (erf) GELU of di_gelu
__global__ void gelu_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ h, float* __restrict__ dx, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = h[i];
  const float cdf = 0.5f * (1.f + erff(v * 0.70710678118654752440f));
  const float pdf = 0.39894228040143267794f * expf(-0.5f * v * v);
  dx[i] = dy[i] * fmaf(v, pdf, cdf);
}

// layout converters (drop-in boundary: the reference hands NCHW tensors around)
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ in, float* __restrict__ out, int C, int HW) {
  __shared__ float tile[32][33];
  int n = blockIdx.z, c0 = blockIdx.y * 32, p0 = blockIdx.x * 32;
  int tx = threadIdx.x, ty = threadIdx.y;
  for (int i = ty; i < 32; i += blockDim.y) {
    int c = c0 + i, p = p0 + tx;
    tile[i][tx] = (c < C && p < HW) ? in[((size_t)n * C + c) * HW + p] : 0.f;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += blockDim.y) {
    int p = p0 + i, c = c0 + tx;
    if (p < HW && c < C) out[((size_t)n * HW + p) * C + c] = tile[tx][i];
  }
}
__global__ void nhwc_to_nchw_kernel(const float* __restrict__ in, float* __restrict__ out, int C, int HW) {
  __shared__ float tile[32][33];
  int n = blockIdx.z, c0 = blockIdx.y * 32, p0 = blockIdx.x * 32;
  int tx = threadIdx.x, ty = threadIdx.y;
  for (int i = ty; i < 32; i += blockDim.y) {
    int p = p0 + i, c = c0 + tx;
    tile[i][tx] = (c < C && p < HW) ? in[((size_t)n * HW + p) * C + c] : 0.f;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += blockDim.y) {
    int c = c0 + i, p = p0 + tx;
    if (p < HW && c < C) out[((size_t)n * C + c) * HW + p] = tile[tx][i];
  }
}


// ------------------------------------------------------------------------------------------------
// Box coder (core/bbox/coders/transfusion_bbox_coder.py) and the post-processing of get_bboxes
// (models/dense_heads/deepinteraction_decoder.py:549-638).
// ------------------------------------------------------------------------------------------------
struct CoderParams {
  float sx, sy, ox, oy;          // centre: feature cell -> metres (out_size_factor * voxel_size, pc_range)
  float rng[6];                  // post_center_range
  int use_range, use_thr;
  float thr;
};

// One thread per (sample, proposal).  score_c = heat_c, or sigmoid(heat_c) * qscore_c * [c == qlabel] when qscore
// is given (decoder.py:561-563); class = first arg-max over c (torch.max).  Box = transfusion_bbox_coder.py:61-75.
__global__ void bbox_decode_kernel(const float* __restrict__ heat, const float* __restrict__ qscore,
                                   const int* __restrict__ qlabel, const float* __restrict__ rot,
                                   const float* __restrict__ dim, const float* __restrict__ center,
                                   const float* __restrict__ height, const float* __restrict__ vel, int B, int K, int P,
                                   CoderParams cp, float* __restrict__ boxes, float* __restrict__ scores,
                                   int* __restrict__ labels, unsigned char* __restrict__ keep) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * P) return;
  const int b = i / P, p = i - b * P;
  float best = -INFINITY;
  int arg = 0;
  for (int c = 0; c < K; ++c) {
    float v = heat[((size_t)b * K + c) * P + p];
    if (qscore) {
      v = 1.f / (1.f + expf(-v));
      v = v * qscore[((size_t)b * K + c) * P + p] * (qlabel[i] == c ? 1.f : 0.f);
    }
    if (v > best) { best = v; arg = c; }
  }
  const int nb = vel ? 9 : 7;
  float* o = boxes + (size_t)i * nb;
  const float cx = center[((size_t)b * 2 + 0) * P + p] * cp.sx + cp.ox;
  const float cy = center[((size_t)b * 2 + 1) * P + p] * cp.sy + cp.oy;
  const float dx = expf(dim[((size_t)b * 3 + 0) * P + p]);
  const float dy = expf(dim[((size_t)b * 3 + 1) * P + p]);
  const float dz = expf(dim[((size_t)b * 3 + 2) * P + p]);
  const float z = height[(size_t)b * P + p] - dz * 0.5f;                 // gravity centre -> bottom centre
  o[0] = cx; o[1] = cy; o[2] = z; o[3] = dx; o[4] = dy; o[5] = dz;
  o[6] = atan2f(rot[((size_t)b * 2 + 0) * P + p], rot[((size_t)b * 2 + 1) * P + p]);
  if (vel) {
    o[7] = vel[((size_t)b * 2 + 0) * P + p];
    o[8] = vel[((size_t)b * 2 + 1) * P + p];
  }
  scores[i] = best;
  labels[i] = arg;
  bool k = true;
  if (cp.use_range)
    k = cx >= cp.rng[0] && cy >= cp.rng[1] && z >= cp.rng[2] && cx <= cp.rng[3] && cy <= cp.rng[4] && z <= cp.rng[5];
  if (cp.use_thr) k = k && best > cp.thr;
  keep[i] = k ? 1 : 0;
}

// transfusion_bbox_coder.py:24-38
__global__ void bbox_encode_kernel(const float* __restrict__ boxes, int nb, float* __restrict__ t, int code, int n,
                                   CoderParams cp) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* s = boxes + (size_t)i * nb;
  float* o = t + (size_t)i * code;
  for (int c = 0; c < code; ++c) o[c] = 0.f;
  o[0] = (s[0] - cp.ox) / cp.sx;
  o[1] = (s[1] - cp.oy) / cp.sy;
  o[3] = logf(s[3]); o[4] = logf(s[4]); o[5] = logf(s[5]);
  o[2] = s[2] + s[5] * 0.5f;
  o[6] = sinf(s[6]);
  o[7] = cosf(s[6]);
  if (code == 10) { o[8] = s[7]; o[9] = s[8]; }
}

// Circle NMS of one task (a set of classes, squared-distance threshold) for one sample per CTA, greedy in descending
// score order (ties: lower index first), at most post_max kept (mmdet3d circle_nms as called at decoder.py:603-609).
// keep_io: in = candidates that survived the coder's filter, out = survivors of this task are left set, the
// suppressed candidates of this task are cleared; other classes are untouched.
constexpr int NMS_MAX = 1024;
__global__ void __launch_bounds__(256)
circle_nms_kernel(const float* __restrict__ boxes, int nb, const float* __restrict__ scores, const int* __restrict__ labels,
                  unsigned char* __restrict__ keep_io, int P, unsigned class_mask, float thresh, int post_max) {
  __shared__ float sk[NMS_MAX];        // sort key: score (descending)
  __shared__ int si[NMS_MAX];          // proposal index, -1 = padding
  __shared__ unsigned char sup[NMS_MAX];
  __shared__ int kept;
  const int b = blockIdx.x, tid = threadIdx.x;
  const float* bx = boxes + (size_t)b * P * nb;
  for (int i = tid; i < NMS_MAX; i += 256) {
    bool cand = i < P && keep_io[(size_t)b * P + i] && ((class_mask >> labels[(size_t)b * P + i]) & 1u);
    sk[i] = cand ? scores[(size_t)b * P + i] : -INFINITY;
    si[i] = cand ? i : -1;
    sup[i] = 0;
  }
  if (tid == 0) kept = 0;
  __syncthreads();
  // bitonic sort, descending score, ascending index among equal scores, padding last
  for (int k = 2; k <= NMS_MAX; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < NMS_MAX; i += 256) {
        const int l = i ^ j;
        if (l > i) {
          const bool up = (i & k) == 0;
          const bool a_first = (si[i] >= 0) && (si[l] < 0 || sk[i] > sk[l] || (sk[i] == sk[l] && si[i] < si[l]));
          if (up ? !a_first : a_first) {
            const float tk = sk[i]; sk[i] = sk[l]; sk[l] = tk;
            const int ti = si[i]; si[i] = si[l]; si[l] = ti;
          }
        }
      }
      __syncthreads();
    }
  for (int a = 0; a < NMS_MAX; ++a) {
    const int ia = si[a];
    if (ia < 0) break;                                   // uniform: shared value
    if (!sup[a]) {
      const bool over = kept >= post_max;
      __syncthreads();
      if (over) {
        if (tid == 0) sup[a] = 1;                        // beyond post_max_size: dropped
      } else {
        if (tid == 0) ++kept;
        const float xa = bx[(size_t)ia * nb], ya = bx[(size_t)ia * nb + 1];
        for (int c = a + 1 + tid; c < NMS_MAX; c += 256) {
          const int ic = si[c];
          if (ic >= 0 && !sup[c]) {
            const float dx = xa - bx[(size_t)ic * nb], dy = ya - bx[(size_t)ic * nb + 1];
            if (dx * dx + dy * dy <= thresh) sup[c] = 1;
          }
        }
      }
    }
    __syncthreads();
  }
  for (int a = tid; a < NMS_MAX; a += 256)
    if (si[a] >= 0 && sup[a]) keep_io[(size_t)b * P + si[a]] = 0;
}

}  // namespace

extern "C" {

// a, b: raw heatmap logits, pixel-major [B,H*W,ld]; out [B,K,H*W] = nms-masked mean of sigmoids;
// dense_b (optional) [B,K,H,W] = logits of b in NCHW.
int di_heatmap_nms_f32(const float* a, const float* b, int ld, float* out, float* dense_b, int B, int K, int H, int W,
                       int ks, int no_nms_class_mask, cudaStream_t stream) {
  DI_CHECK_ARG(a && b && out && B > 0 && K > 0 && K <= 32 && ld >= K && ks % 2 == 1, "di_heatmap_nms_f32: bad argument");
  int total = B * K * H * W;
  heatmap_nms_kernel<<<di_cdiv(total, 256), 256, 0, stream>>>(a, b, ld, out, dense_b, K, H, W, ks,
                                                              (unsigned)no_nms_class_mask, total);
  DI_CHECK_LAUNCH("di_heatmap_nms_f32");
  return DI_OK;
}

// scores [B,n] >= 0 -> idx [B,k] (descending score, ties by ascending index, however many tie); k <= 1024.
// work: B * slices * k * 2 ints/floats of scratch (pass nullptr/0 slices for the single-level path).
int di_topk_f32(const float* scores, int* idx, int B, int n, int k, void* work, int slices, cudaStream_t stream) {
  DI_CHECK_ARG(scores && idx && B > 0 && n >= k && k > 0 && k <= TOPK_MAX, "di_topk_f32: bad argument (k=%d n=%d)", k, n);
  if (!work || slices <= 1 || slices * k > (1 << 20)) {
    topk_kernel<<<dim3(1, B), 1024, 0, stream>>>(scores, nullptr, n, n, k, nullptr, idx);
    DI_CHECK_LAUNCH("di_topk_f32");
    return DI_OK;
  }
  float* cval = reinterpret_cast<float*>(work);
  int* cidx = reinterpret_cast<int*>(cval + (size_t)B * slices * k);
  // no slice but the last is shorter than k: the index -1 pads of a short slice then trail every real candidate, and
  // level 2 (ties by ascending candidate position) reaches them only after all real indices
  int n_slice = max(di_cdiv(n, slices), k);
  slices = di_cdiv(n, n_slice);
  topk_kernel<<<dim3(slices, B), 1024, 0, stream>>>(scores, nullptr, n, n_slice, k, cval, cidx);
  DI_CHECK_LAUNCH("di_topk_f32(level 1)");
  // level 2: candidates of empty tail slots carry value 0 / index -1; they sit after every real candidate, of which there
  // are at least k, so they are never selected
  topk_kernel<<<dim3(1, B), 1024, 0, stream>>>(cval, cidx, slices * k, slices * k, k, nullptr, idx);
  DI_CHECK_LAUNCH("di_topk_f32(level 2)");
  return DI_OK;
}

int di_query_init_f32(const float* feat, const int* top, const float* heat, const float* wce_t, const float* bce,
                      float* qfeat, float* qpos, int* labels, float* qscore, int B, int HW, int W, int C, int K, int P,
                      cudaStream_t stream) {
  DI_CHECK_ARG(feat && top && heat && wce_t && bce && qfeat && qpos && labels && qscore, "di_query_init_f32: null pointer");
  query_init_kernel<<<B * P, 128, 0, stream>>>(feat, top, heat, wce_t, bce, qfeat, qpos, labels, qscore, HW, W, C, K, P);
  DI_CHECK_LAUNCH("di_query_init_f32");
  return DI_OK;
}

int di_query_init_bwd_f32(const float* dq, const int* top, const int* labels, float* d_feat, float* d_wce, float* d_bce, int B,
                          int HW, int C, int K, int P, cudaStream_t stream) {
  DI_CHECK_ARG(dq && top && labels && d_feat && d_wce && d_bce && B > 0 && HW > 0 && C > 0 && K > 0 && P > 0 && P <= 8192,
               "di_query_init_bwd_f32: bad argument");
  query_init_bwd_feat_kernel<<<dim3(P, B), 128, P * sizeof(int), stream>>>(dq, top, d_feat, HW, C, P);
  query_init_bwd_class_kernel<<<K + 1, 128, 0, stream>>>(dq, labels, d_wce, d_bce, B * P, C, K);
  DI_CHECK_LAUNCH("di_query_init_bwd_f32");
  return DI_OK;
}

// q/k/v/out: [B*P, ld*] rows, heads of 16 channels; onbits/win optional (see kernel comment)
int di_mha_small_f32(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, float* out, int ldo,
                     const int* onbits, const int* win, int B, int P, int heads, int head_dim, cudaStream_t stream) {
  DI_CHECK_ARG(q && k && v && out && head_dim == 16 && P <= 512, "di_mha_small_f32: unsupported shape (head_dim=%d P=%d)", head_dim, P);
  DI_CHECK_ARG(ldq % 4 == 0 && ldk % 4 == 0 && ldv % 4 == 0, "di_mha_small_f32: strides must be multiples of 4");
  DI_CHECK_ARG((onbits == nullptr) == (win == nullptr), "di_mha_small_f32: onbits and win go together");
  int warps = B * P * heads;
  mha_small_kernel<16><<<di_cdiv(warps, 8), 256, 0, stream>>>(q, ldq, k, ldk, v, ldv, out, ldo, onbits, win, B, P, heads,
                                                              nullptr, 0, 1);
  DI_CHECK_LAUNCH("di_mha_small_f32");
  return DI_OK;
}

// Backward of di_mha_small_f32 with the same optional group mask (onbits, win): dout [B*P, ldd] -> dq / dk / dv rows
// [B*P, ldg] (e.g. the three column blocks of one [B*P, 3C] gradient); work: float [2 * B * heads * P * P].
int di_mha_small_bwd_f32(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, const float* dout, int ldd,
                         float* dq, float* dk, float* dv, int ldg, float* work, const int* onbits, const int* win, int B, int P,
                         int heads, int head_dim, cudaStream_t stream) {
  DI_CHECK_ARG(q && k && v && dout && dq && dk && dv && work && B > 0 && P > 0 && heads > 0 && head_dim == 16 && P <= 512,
               "di_mha_small_bwd_f32: unsupported shape (head_dim=%d P=%d)", head_dim, P);
  DI_CHECK_ARG(ldq % 4 == 0 && ldk % 4 == 0 && ldv % 4 == 0 && ldd % 4 == 0, "di_mha_small_bwd_f32: strides must be multiples of 4");
  DI_CHECK_ARG((onbits == nullptr) == (win == nullptr), "di_mha_small_bwd_f32: onbits and win go together");
  const int warps = B * P * heads;
  float* aw = work;
  float* sw = work + (size_t)B * heads * P * P;
  mha_small_bwd_q_kernel<16, false><<<di_cdiv(warps, 8), 256, 0, stream>>>(q, ldq, k, ldk, v, ldv, dout, ldd, dq, ldg, aw, sw,
                                                                           onbits, win, B, P, heads, nullptr, P);
  DI_CHECK_LAUNCH("di_mha_small_bwd_f32");
  mha_small_bwd_kv_kernel<16><<<di_cdiv(warps, 8), 256, 0, stream>>>(q, ldq, dout, ldd, aw, sw, dk, dv, ldg, onbits, win, B, P,
                                                                     heads);
  DI_CHECK_LAUNCH("di_mha_small_bwd_f32 (keys)");
  return DI_OK;
}

// Row-map form: out row r (of R = B * rows_per_b) = attention of query rows[r] (a global row b*P+i, or -1 -> zero row)
// over the keys of its sample whose onbits have bit rwin[r].  Used for the "view leader" rows of the V2 RCNN blocks.
int di_mha_small_rows_f32(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, float* out, int ldo,
                          const int* onbits, const int* rows, const int* rwin, int R, int rows_per_b, int B, int P,
                          int heads, int head_dim, cudaStream_t stream) {
  DI_CHECK_ARG(q && k && v && out && onbits && rows && rwin && head_dim == 16 && P <= 512 && R == B * rows_per_b,
               "di_mha_small_rows_f32: unsupported shape (head_dim=%d P=%d R=%d)", head_dim, P, R);
  DI_CHECK_ARG(ldq % 4 == 0 && ldk % 4 == 0 && ldv % 4 == 0, "di_mha_small_rows_f32: strides must be multiples of 4");
  mha_small_kernel<16><<<di_cdiv(R * heads, 8), 256, 0, stream>>>(q, ldq, k, ldk, v, ldv, out, ldo, onbits, rwin, B, P, heads,
                                                                  rows, R, rows_per_b);
  DI_CHECK_LAUNCH("di_mha_small_rows_f32");
  return DI_OK;
}

// lead_row [B*V]: global row (b*P + i) of the FIRST query of sample b whose onbits have bit v, or -1; lead_win [B*V] = v
// or -1.  (decoder_utils.py:987 / :1085: the self-branch feature every query of a view receives is the one of the
// view's first query -- see oracle/mmpi_pp.py.)
int di_rcnn_leaders(const int* onbits, int* lead_row, int* lead_win, int B, int P, int V, cudaStream_t stream) {
  DI_CHECK_ARG(onbits && lead_row && lead_win && B > 0 && P > 0 && V > 0 && V <= MAXV, "di_rcnn_leaders: bad argument");
  rcnn_leaders_kernel<<<B * V, 32, 0, stream>>>(onbits, lead_row, lead_win, P, V);
  DI_CHECK_LAUNCH("di_rcnn_leaders");
  return DI_OK;
}

// out[r, :C] = idx[r] >= 0 ? src[idx[r], :C] : 0
int di_take_rows_f32(const float* src, int ld, const int* idx, float* out, int R, int C, cudaStream_t stream) {
  DI_CHECK_ARG(src && idx && out && R > 0 && C > 0, "di_take_rows_f32: bad argument");
  take_rows_kernel<<<R, 128, 0, stream>>>(src, ld, idx, out, C);
  DI_CHECK_LAUNCH("di_take_rows_f32");
  return DI_OK;
}

// out[m] = a[m] * scale[0] + lead[(m / P) * V + win[m]] * self_scale[0]  (two rounded products, one rounded sum, as
// torch evaluates decoder_utils.py:987); rows with win[m] < 0 are zero when zero_off != 0 (queries on no image).
int di_branch_mix_f32(const float* a, const float* lead, const int* win, const float* scale, const float* self_scale,
                      float* out, int M, int C, int P, int V, int zero_off, cudaStream_t stream) {
  DI_CHECK_ARG(a && lead && win && scale && self_scale && out && M > 0 && C > 0 && P > 0 && V > 0, "di_branch_mix_f32: bad argument");
  branch_mix_kernel<<<M, 128, 0, stream>>>(a, lead, win, scale, self_scale, out, C, P, V, zero_off);
  DI_CHECK_LAUNCH("di_branch_mix_f32");
  return DI_OK;
}

// ++ decoder, deepinteractionplusplus_decoder.py:285-302: pred[:, 0:2] = delta + look; look' = delta + qpos;
// keep' = image layer ? (win >= 0 [&& keep]) : keep;  rows with !keep' take `first`;  qpos' = pred[:, 0:2].
// keep: int32 [M] cumulative mask (read unless first_layer, always written); win: this layer's winning view or NULL.
int di_pred_finish_pp_f32(float* pred, float* qpos, float* look, const float* first, const int* win, int* keep,
                          int first_layer, int M, int NP, cudaStream_t stream) {
  DI_CHECK_ARG(pred && qpos && look && first && keep && M > 0 && NP >= 2 && (win || !first_layer),
               "di_pred_finish_pp_f32: bad argument");
  pred_finish_pp_kernel<<<di_cdiv(M, 128), 128, 0, stream>>>(pred, qpos, look, first, win, keep, first_layer, M, NP);
  DI_CHECK_LAUNCH("di_pred_finish_pp_f32");
  return DI_OK;
}

// Backward of di_mha_small_rows_f32: dout [R, ldd] -> dq [R, lddq] (rows[r] = -1: zero row); dk / dv [B*P, ldg] are ADDED
// to.  work: float [2 * B * heads * P * rows_per_b].
int di_mha_small_rows_bwd_f32(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, const float* dout,
                              int ldd, float* dq, int lddq, float* dk, float* dv, int ldg, float* work, const int* onbits,
                              const int* rows, const int* rwin, int R, int rows_per_b, int B, int P, int heads, int head_dim,
                              cudaStream_t stream) {
  DI_CHECK_ARG(q && k && v && dout && dq && dk && dv && work && onbits && rows && rwin && B > 0 && rows_per_b > 0 &&
               R == B * rows_per_b && P > 0 && P <= 512 && heads > 0 && head_dim == 16,
               "di_mha_small_rows_bwd_f32: unsupported shape (head_dim=%d P=%d R=%d)", head_dim, P, R);
  DI_CHECK_ARG(ldq % 4 == 0 && ldk % 4 == 0 && ldv % 4 == 0 && ldd % 4 == 0, "di_mha_small_rows_bwd_f32: strides must be multiples of 4");
  float* aw = work;
  float* sw = work + (size_t)B * heads * P * rows_per_b;
  mha_small_bwd_q_kernel<16, true><<<di_cdiv(R * heads, 8), 256, 0, stream>>>(q, ldq, k, ldk, v, ldv, dout, ldd, dq, lddq, aw,
                                                                              sw, onbits, rwin, B, P, heads, rows, rows_per_b);
  DI_CHECK_LAUNCH("di_mha_small_rows_bwd_f32");
  mha_small_rows_bwd_kv_kernel<16><<<di_cdiv(B * P * heads, 8), 256, 0, stream>>>(q, ldq, dout, ldd, aw, sw, dk, dv, ldg, onbits,
                                                                                 rows, rwin, B, P, heads, rows_per_b);
  DI_CHECK_LAUNCH("di_mha_small_rows_bwd_f32 (keys)");
  return DI_OK;
}

// dst[idx[r], :C] += src[r, :C], r ascending, idx[r] < 0 skipped (the adjoint of di_take_rows_f32)
int di_rows_scatter_add_f32(const float* src, int lds, const int* idx, float* dst, int ldd, int R, int C, cudaStream_t stream) {
  DI_CHECK_ARG(src && idx && dst && R > 0 && C > 0, "di_rows_scatter_add_f32: bad argument");
  rows_scatter_add_kernel<<<di_cdiv(C, 128), 128, 0, stream>>>(src, lds, idx, dst, ldd, R, C);
  DI_CHECK_LAUNCH("di_rows_scatter_add_f32");
  return DI_OK;
}

// Backward of di_branch_mix_f32: dout [M, C] -> da [M, C], dlead [M / P * V, C], d_scale [1], d_self_scale [1].
// work: float [2 * M].
int di_branch_mix_bwd_f32(const float* dout, const float* a, const float* lead, const int* win, const float* scale,
                          const float* self_scale, float* da, float* dlead, float* d_scale, float* d_self_scale, float* work,
                          int M, int C, int P, int V, int zero_off, cudaStream_t stream) {
  DI_CHECK_ARG(dout && a && lead && win && scale && self_scale && da && dlead && d_scale && d_self_scale && work && M > 0 &&
               C > 0 && P > 0 && V > 0 && M % P == 0, "di_branch_mix_bwd_f32: bad argument");
  branch_mix_bwd_rows_kernel<<<M, 128, 0, stream>>>(dout, a, lead, win, scale, da, work, C, P, V, zero_off);
  DI_CHECK_LAUNCH("di_branch_mix_bwd_f32");
  branch_mix_bwd_lead_kernel<<<M / P * V, 128, 0, stream>>>(dout, win, self_scale, dlead, C, P, V, zero_off);
  DI_CHECK_LAUNCH("di_branch_mix_bwd_f32 (leaders)");
  branch_mix_bwd_scales_kernel<<<1, 128, 0, stream>>>(work, d_scale, d_self_scale, M);
  DI_CHECK_LAUNCH("di_branch_mix_bwd_f32 (scales)");
  return DI_OK;
}

// Backward of di_pred_finish_pp_f32 over the L layers: dpred [L, M, NP], keep [L, M] (each layer's cumulative mask) ->
// d_delta [L, M, NP] (the gradient of each prediction head's output rows), d_first [M, NP].
int di_pred_finish_pp_bwd_f32(const float* dpred, const int* keep, float* d_delta, float* d_first, int L, int M, int NP,
                              cudaStream_t stream) {
  DI_CHECK_ARG(dpred && keep && d_delta && d_first && L > 0 && M > 0 && NP >= 2, "di_pred_finish_pp_bwd_f32: bad argument");
  pred_finish_pp_bwd_kernel<<<di_cdiv(M * NP, 128), 128, 0, stream>>>(dpred, keep, d_delta, d_first, L, M, NP);
  DI_CHECK_LAUNCH("di_pred_finish_pp_bwd_f32");
  return DI_OK;
}

// part: workspace [B, heads, P, nsplit, 18]; out [B*P, C]
int di_cross_attn_f32(const float* q, const float* kv, float* part, float* out, int B, int P, int HW, int C, int heads,
                      int nsplit, cudaStream_t stream) {
  DI_CHECK_ARG(q && kv && part && out && C == heads * 16 && nsplit > 0, "di_cross_attn_f32: bad argument");
  int chunk = di_cdiv(HW, nsplit);
  chunk = (chunk + 3) / 4 * 4;
  int qtiles = di_cdiv(P, 256);
  dim3 grid(nsplit * qtiles, heads, B);
  cross_attn_kernel<16><<<grid, 256, 0, stream>>>(q, kv, part, P, HW, C, heads, chunk, nsplit);
  DI_CHECK_LAUNCH("di_cross_attn_f32");
  cross_attn_combine_kernel<16><<<di_cdiv(B * heads * P, 128), 128, 0, stream>>>(part, out, B, P, C, heads, nsplit);
  DI_CHECK_LAUNCH("di_cross_attn_combine");
  return DI_OK;
}

int di_rows_finish_f32(const float* part, int nsplit, long long split_stride, int ldp, const float* bias,
                       const float* res, int ldres, const float* gamma, const float* beta, float* out, int ldo,
                       const int* zero_if_neg, int M, int C, int act, float eps, cudaStream_t stream) {
  DI_CHECK_ARG(part && out && M > 0 && C > 0 && C <= 512 && nsplit >= 1, "di_rows_finish_f32: bad argument");
  DI_CHECK_ARG((gamma == nullptr) == (beta == nullptr), "di_rows_finish_f32: gamma and beta go together");
  const bool al = (((uintptr_t)part | (uintptr_t)out | (uintptr_t)bias | (uintptr_t)res | (uintptr_t)gamma | (uintptr_t)beta) & 15) == 0;
  if (C == 128 && nsplit == 1 && M >= 4096 && al && ldp % 4 == 0 && ldo % 4 == 0 && (!res || ldres % 4 == 0))
    rows_finish_c128_kernel<<<di_cdiv(M, 8), 256, 0, stream>>>(part, ldp, bias, res, ldres, gamma, beta, out, ldo, zero_if_neg,
                                                              M, act, eps);
  else
    rows_finish_kernel<<<di_cdiv(M, 8), 256, 0, stream>>>(part, nsplit, (size_t)split_stride, ldp, bias, res, ldres, gamma,
                                                         beta, out, ldo, zero_if_neg, M, C, act, eps);
  DI_CHECK_LAUNCH("di_rows_finish_f32");
  return DI_OK;
}

// Query-row MLP (see rows_mlp_kernel): Y[M, N] = act_out(LN(act1([X0|X1] W1t + b1) [W2t + b2] + res)).
// W1t [K0+K1, N1] and W2t [N1, N2] are TRANSPOSED weights (row = input channel); W2t / b1 / b2 / res / gamma may be NULL.
// K0 + K1 <= 1024, N1, N2 <= 512, K0 + K1 + N1 + N2 <= 1800.
int di_rows_mlp_f32(const float* X0, int ld0, int K0, const float* X1, int ld1, int K1, const float* W1t, const float* b1,
                    int N1, int act1, const float* W2t, const float* b2, int N2, const float* res, int ldres,
                    const float* gamma, const float* beta, float eps, int act_out, const int* zero_if_neg, float* Y, int ldy,
                    int M, cudaStream_t stream) {
  DI_CHECK_ARG(X0 && W1t && Y && M > 0 && K0 > 0 && K1 >= 0 && (K1 == 0 || X1) && N1 > 0, "di_rows_mlp_f32: bad argument");
  DI_CHECK_ARG(K0 + K1 <= 1024 && N1 <= 512 && (!W2t || (N2 > 0 && N2 <= 512)), "di_rows_mlp_f32: K <= 1024, N <= 512");
  DI_CHECK_ARG((gamma == nullptr) == (beta == nullptr), "di_rows_mlp_f32: gamma and beta go together");
  DI_CHECK_ARG(N1 % 4 == 0 && (!W2t || N2 % 4 == 0) && ((uintptr_t)W1t & 15) == 0 && ((uintptr_t)W2t & 15) == 0,
               "di_rows_mlp_f32: N1, N2 must be multiples of 4 and the weights 16-byte aligned (bulk copies)");
  const size_t smem = sizeof(float) * ((size_t)MLP_NS * MLP_CHUNK + MLP_R * (size_t)(K0 + K1 + N1 + (W2t ? N2 : 0) + 2048));
  DI_CHECK_ARG(smem <= 226 * 1024, "di_rows_mlp_f32: K + N1 + N2 too large for shared memory (%d)", K0 + K1 + N1 + N2);
  static DiSmemOnce once{};
  if (!di_smem_once(once, rows_mlp_kernel, 226 * 1024)) {
    di_set_error("di_rows_mlp_f32: cannot reserve shared memory");
    return DI_ERR_LAUNCH;
  }
  rows_mlp_kernel<<<di_cdiv(M, MLP_R), MLP_NT, smem, stream>>>(X0, ld0, K0, X1, ld1, K1, W1t, b1, N1, act1, W2t, b2, N2, res,
                                                           ldres, gamma, beta, eps, act_out, zero_if_neg, Y, ldy, M);
  DI_CHECK_LAUNCH("di_rows_mlp_f32");
  return DI_OK;
}

int di_pred_finish_f32(float* pred, float* qpos, const float* first, const int* win, int M, int NP, cudaStream_t stream) {
  DI_CHECK_ARG(pred && qpos && M > 0 && NP >= 2, "di_pred_finish_f32: bad argument");
  pred_finish_kernel<<<di_cdiv(M, 128), 128, 0, stream>>>(pred, qpos, first, win, M, NP);
  DI_CHECK_LAUNCH("di_pred_finish_f32");
  return DI_OK;
}

// params10 (host): sx, sy, ox, oy, csx, cox, h_pad, w_pad, bev_scale, bev_off.  proj [B,V,12] and aux [B,4]
// (crop_x, crop_y, flip, orig_w) are device pointers used by mode 0 only.
int di_rcnn_rois_f32(const float* pred, int NP, const float* proj, const float* aux, float* rois, int* win, int* onbits,
                     int B, int P, int V, int mode, const float* params10, cudaStream_t stream) {
  DI_CHECK_ARG(pred && rois && win && onbits && params10 && P <= 1024 && V <= MAXV && NP >= 8, "di_rcnn_rois_f32: bad argument");
  DI_CHECK_ARG(mode == 1 || (proj && aux), "di_rcnn_rois_f32: image mode needs proj and aux");
  RoiParams rp;
  rp.sx = params10[0]; rp.sy = params10[1]; rp.ox = params10[2]; rp.oy = params10[3];
  rp.csx = params10[4]; rp.cox = params10[5]; rp.h_pad = params10[6]; rp.w_pad = params10[7];
  rp.bev_scale = params10[8]; rp.bev_off = params10[9];
  int threads = ((P + 31) / 32) * 32;
  if (threads < 32) threads = 32;
  rcnn_rois_kernel<<<B, threads, 0, stream>>>(pred, NP, proj, aux, rois, win, onbits, P, V, mode, rp);
  DI_CHECK_LAUNCH("di_rcnn_rois_f32");
  return DI_OK;
}

// maps [n_maps,H,W,C] pixel-major; rois [n,5] = (map index or -1, x0,y0,x1,y1); out [n,49,C]
int di_roi_align_f32(const float* maps, const float* rois, float* out, int n, int H, int W, int C, float scale,
                     cudaStream_t stream) {
  DI_CHECK_ARG(maps && rois && out && n > 0 && C % 4 == 0 && C <= 512, "di_roi_align_f32: bad argument");
  dim3 grid(di_cdiv(n * 49, 8));
  if (C <= 128) roi_align_kernel<1><<<grid, 256, 0, stream>>>(maps, rois, out, n, H, W, C, scale);
  else if (C <= 256) roi_align_kernel<2><<<grid, 256, 0, stream>>>(maps, rois, out, n, H, W, C, scale);
  else roi_align_kernel<4><<<grid, 256, 0, stream>>>(maps, rois, out, n, H, W, C, scale);
  DI_CHECK_LAUNCH("di_roi_align_f32");
  return DI_OK;
}

// roi [n,49,128]; params [n, 2*128*128]; out [n, 49*128]
int di_dynconv_f32(const float* roi, const float* params, const float* g1, const float* b1, const float* g2,
                   const float* b2, float* out, int n, float eps, cudaStream_t stream) {
  DI_CHECK_ARG(roi && params && g1 && b1 && g2 && b2 && out && n > 0 && (((uintptr_t)params | (uintptr_t)roi) & 15) == 0,
               "di_dynconv_f32: bad argument");
  const int smem = (2 * DR * DC + 2 * DC * DC) * (int)sizeof(float);
  static DiSmemOnce once{};
  if (!di_smem_once(once, dynconv_kernel, smem)) {
    di_set_error("di_dynconv_f32: cannot reserve shared memory");
    return DI_ERR_LAUNCH;
  }
  dynconv_kernel<<<n, DYN_T, smem, stream>>>(roi, params, g1, b1, g2, b2, out, eps);
  DI_CHECK_LAUNCH("di_dynconv_f32");
  return DI_OK;
}

// Backward of di_roi_align_f32 w.r.t. the maps: d_out [n, 49, C] -> d_maps [n_maps, H, W, C], every pixel written (0 where
// no sample reaches); RoIs with a map index outside [0, n_maps) contribute nothing.  Deterministic (a gather, no atomics).
int di_roi_align_bwd_f32(const float* rois, const float* d_out, float* d_maps, int n, int n_maps, int H, int W, int C,
                         float scale, cudaStream_t stream) {
  DI_CHECK_ARG(d_maps && (n == 0 || (rois && d_out)) && n >= 0 && n_maps > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0 &&
                   C <= 512 && (((uintptr_t)d_out | (uintptr_t)d_maps) & 15) == 0,
               "di_roi_align_bwd_f32: bad argument (n=%d n_maps=%d H=%d W=%d C=%d)", n, n_maps, H, W, C);
  DI_CHECK_ARG(n_maps <= 65535, "di_roi_align_bwd_f32: n_maps <= 65535");
  const int tiles_x = di_cdiv(W, RB_TX);
  dim3 grid(tiles_x * di_cdiv(H, RB_TY), n_maps);
  if (C <= 128) roi_align_bwd_kernel<1><<<grid, RB_T, 0, stream>>>(rois, d_out, d_maps, n, H, W, C, scale, tiles_x);
  else if (C <= 256) roi_align_bwd_kernel<2><<<grid, RB_T, 0, stream>>>(rois, d_out, d_maps, n, H, W, C, scale, tiles_x);
  else roi_align_bwd_kernel<4><<<grid, RB_T, 0, stream>>>(rois, d_out, d_maps, n, H, W, C, scale, tiles_x);
  DI_CHECK_LAUNCH("di_roi_align_bwd_f32");
  return DI_OK;
}

// Backward of di_dynconv_f32: d_out [n, 49*128] -> d_roi [n, 49, 128], d_params [n, 2*128*128] (layout of params),
// d_norm [n, 4*128] = per-query partials of dgamma1 | dbeta1 | dgamma2 | dbeta2 (sum over n with di_col_sum_f32).
int di_dynconv_bwd_f32(const float* roi, const float* params, const float* g1, const float* b1, const float* g2, const float* b2,
                       const float* d_out, float* d_roi, float* d_params, float* d_norm, int n, float eps, cudaStream_t stream) {
  DI_CHECK_ARG(roi && params && g1 && b1 && g2 && b2 && d_out && d_roi && d_params && d_norm && n > 0 &&
                   (((uintptr_t)params | (uintptr_t)roi | (uintptr_t)d_out | (uintptr_t)d_params | (uintptr_t)g1 |
                     (uintptr_t)b1 | (uintptr_t)g2 | (uintptr_t)b2) & 15) == 0,
               "di_dynconv_bwd_f32: bad argument");
  static DiSmemOnce once{};
  if (!di_smem_once(once, dynconv_bwd_kernel, DYN_BWD_SMEM)) {
    di_set_error("di_dynconv_bwd_f32: cannot reserve shared memory");
    return DI_ERR_LAUNCH;
  }
  dynconv_bwd_kernel<<<n, DYN_T, DYN_BWD_SMEM, stream>>>(roi, params, g1, b1, g2, b2, d_out, d_roi, d_params, d_norm, eps);
  DI_CHECK_LAUNCH("di_dynconv_bwd_f32");
  return DI_OK;
}

int di_gelu_bwd_f32(const float* dy, const float* h, float* dx, long long n, cudaStream_t stream) {
  DI_CHECK_ARG(dy && h && dx && n > 0, "di_gelu_bwd_f32: bad argument");
  gelu_bwd_kernel<<<di_cdiv(n, 256), 256, 0, stream>>>(dy, h, dx, n);
  DI_CHECK_LAUNCH("di_gelu_bwd_f32");
  return DI_OK;
}

int di_nchw_to_nhwc_f32(const float* in, float* out, int N, int C, int HW, cudaStream_t stream) {
  DI_CHECK_ARG(in && out && N > 0 && C > 0 && HW > 0, "di_nchw_to_nhwc_f32: bad argument");
  dim3 grid(di_cdiv(HW, 32), di_cdiv(C, 32), N), block(32, 8);
  nchw_to_nhwc_kernel<<<grid, block, 0, stream>>>(in, out, C, HW);
  DI_CHECK_LAUNCH("di_nchw_to_nhwc_f32");
  return DI_OK;
}

int di_nhwc_to_nchw_f32(const float* in, float* out, int N, int C, int HW, cudaStream_t stream) {
  DI_CHECK_ARG(in && out && N > 0 && C > 0 && HW > 0, "di_nhwc_to_nchw_f32: bad argument");
  dim3 grid(di_cdiv(HW, 32), di_cdiv(C, 32), N), block(32, 8);
  nhwc_to_nchw_kernel<<<grid, block, 0, stream>>>(in, out, C, HW);
  DI_CHECK_LAUNCH("di_nhwc_to_nchw_f32");
  return DI_OK;
}

// TransFusionBBoxCoder.decode (+ the score composition of get_bboxes when qscore/qlabel are given).  All inputs
// contiguous [B, k, P]; range6 = post_center_range or NULL; boxes [B,P,7|9] (9 iff vel), scores [B,P], labels [B,P]
// (int32), keep [B,P] (uint8: centre inside range and score > thr when use_thr).
int di_bbox_decode_f32(const float* heat, const float* qscore, const int* qlabel, const float* rot, const float* dim,
                       const float* center, const float* height, const float* vel, int B, int K, int P, float sx, float sy,
                       float ox, float oy, const float* range6, float score_thr, int use_thr, float* boxes, float* scores,
                       int* labels, unsigned char* keep, cudaStream_t stream) {
  DI_CHECK_ARG(heat && rot && dim && center && height && boxes && scores && labels && keep && B > 0 && K > 0 && P > 0,
               "di_bbox_decode_f32: bad argument");
  DI_CHECK_ARG((qscore == nullptr) == (qlabel == nullptr), "di_bbox_decode_f32: qscore and qlabel go together");
  CoderParams cp{};
  cp.sx = sx; cp.sy = sy; cp.ox = ox; cp.oy = oy; cp.use_range = range6 != nullptr; cp.use_thr = use_thr; cp.thr = score_thr;
  if (range6) memcpy(cp.rng, range6, sizeof(cp.rng));               // host pointer
  bbox_decode_kernel<<<di_cdiv((long long)B * P, 128), 128, 0, stream>>>(heat, qscore, qlabel, rot, dim, center, height, vel,
                                                                        B, K, P, cp, boxes, scores, labels, keep);
  DI_CHECK_LAUNCH("di_bbox_decode_f32");
  return DI_OK;
}

// TransFusionBBoxCoder.encode: boxes [n, nb = 7|9] -> targets [n, code = 8|10]
int di_bbox_encode_f32(const float* boxes, int nb, float* targets, int code, int n, float sx, float sy, float ox, float oy,
                       cudaStream_t stream) {
  DI_CHECK_ARG(boxes && targets && n > 0 && (nb == 7 || nb == 9) && (code == 8 || code == 10) && (code != 10 || nb == 9),
               "di_bbox_encode_f32: bad argument");
  CoderParams cp{};
  cp.sx = sx; cp.sy = sy; cp.ox = ox; cp.oy = oy;
  bbox_encode_kernel<<<di_cdiv(n, 128), 128, 0, stream>>>(boxes, nb, targets, code, n, cp);
  DI_CHECK_LAUNCH("di_bbox_encode_f32");
  return DI_OK;
}

// Circle NMS of one task over B samples (get_bboxes, nms_type == 'circle'): classes in class_mask, squared-distance
// threshold `thresh`, at most post_max survivors; keep_io [B,P] is updated in place.  P <= 1024.
int di_circle_nms_f32(const float* boxes, int nb, const float* scores, const int* labels, unsigned char* keep_io, int B,
                      int P, unsigned class_mask, float thresh, int post_max, cudaStream_t stream) {
  DI_CHECK_ARG(boxes && scores && labels && keep_io && B > 0 && P > 0 && P <= NMS_MAX && nb >= 2,
               "di_circle_nms_f32: bad argument (P must be <= 1024)");
  circle_nms_kernel<<<B, 256, 0, stream>>>(boxes, nb, scores, labels, keep_io, P, class_mask, thresh, post_max);
  DI_CHECK_LAUNCH("di_circle_nms_f32");
  return DI_OK;
}

}  // extern "C"
