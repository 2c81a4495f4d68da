// Geometry-driven gathers of the MMRI encoder:
//   * I2P  (image -> pillar)  per-pillar projected bilinear gather + single-head attention
//          reference models/utils/encoder_utils.py:257-320 (MMRI_I2P.forward, group_attn :226-255)
//   * BEVWarp (pillar/BEV -> image): point projection + sparse depth maps (:152-174), classical
//          depth completion (models/utils/ip_basic/depth_map_utils.py:134-287, run on the CPU with
//          OpenCV by the reference), pixel lifting (:183-194) and BEV bilinear sampling (:195-196)
//
// All feature maps are pixel-major (NHWC) fp32: one pixel's C channels are one contiguous row, so
// every bilinear corner is a coalesced 4*C-byte read (a warp reads it with one float4 per lane).
#include "common.cuh"
#include <math.h>

namespace {

// 3x4 projection rows: cam = P * (x,y,z,1)
struct Proj {
  float m[12];
};

__device__ __forceinline__ void project(const float* __restrict__ P, float x, float y, float z, float& cx, float& cy,
                                        float& cz) {
  cx = P[0] * x + P[1] * y + P[2] * z + P[3];
  cy = P[4] * x + P[5] * y + P[6] * z + P[7];
  cz = P[8] * x + P[9] * y + P[10] * z + P[11];
}

// torch grid_sample(bilinear, zeros, align_corners=False) of a pixel-major map at pixel-space
// coordinates (ix, iy); lane handles channels 4*lane + 128*j.
template <int NJ>
__device__ __forceinline__ void bilinear_row(const float* __restrict__ map, int H, int W, int C, float ix, float iy,
                                             int lane, float4 (&out)[NJ]) {
  float fx = floorf(ix), fy = floorf(iy);
  int x0 = (int)fx, y0 = (int)fy;
  float wx1 = ix - fx, wx0 = (fx + 1.f) - ix;
  float wy1 = iy - fy, wy0 = (fy + 1.f) - iy;
  float wgt[4] = {wx0 * wy0, wx1 * wy0, wx0 * wy1, wx1 * wy1};  // nw, ne, sw, se
#pragma unroll
  for (int j = 0; j < NJ; ++j) out[j] = make_float4(0, 0, 0, 0);
  // guard against huge / NaN coordinates before the int conversion is trusted
  if (!(ix > -2.f && ix < (float)W + 1.f && iy > -2.f && iy < (float)H + 1.f)) return;
#pragma unroll
  for (int cnr = 0; cnr < 4; ++cnr) {
    int xx = x0 + (cnr & 1), yy = y0 + (cnr >> 1);
    if (xx < 0 || xx >= W || yy < 0 || yy >= H) continue;
    const float* row = map + ((size_t)yy * W + xx) * C;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      int c = 4 * lane + 128 * j;
      if (c < C) {
        float4 v = ldg4(row + c);
        out[j].x = fmaf(v.x, wgt[cnr], out[j].x);
        out[j].y = fmaf(v.y, wgt[cnr], out[j].y);
        out[j].z = fmaf(v.z, wgt[cnr], out[j].z);
        out[j].w = fmaf(v.w, wgt[cnr], out[j].w);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// I2P: one warp per pillar.
// ------------------------------------------------------------------------------------------------
// Attention dropout of nn.MultiheadAttention in training mode (encoder_utils.py:223, dropout = 0.1 in the reference config):
// the softmax weights are multiplied by keep / (1 - p) AFTER normalisation.  keep is a counter-based hash of (seed, pillar,
// key index), so the backward regenerates the same mask without storing it.  Returns 0 or 1 / (1 - p).
__device__ __forceinline__ float i2p_keep_scale(unsigned seed, int p, int key, float pdrop) {
  unsigned x = seed ^ (0x9E3779B9u * (unsigned)(p + 1));
  x ^= (unsigned)key * 0x85EBCA6Bu + 0xC2B2AE35u;
  x ^= x >> 16; x *= 0x7FEB352Du; x ^= x >> 15; x *= 0x846CA68Bu; x ^= x >> 16;
  return (float)(x >> 8) * (1.f / 16777216.f) >= pdrop ? 1.f / (1.f - pdrop) : 0.f;
}

template <int NJ, bool DROP>
__device__ __forceinline__ void
i2p_attend_body(const float* __restrict__ qk, const float* __restrict__ pillars, const int* __restrict__ npts,
                const int* __restrict__ coors, const float* __restrict__ proj, const float* __restrict__ img,
                float* __restrict__ s_out, int* __restrict__ cnt_out, int P, int T, int pdim, int V, int h, int w,
                int C, float H_in, float W_in, const int* __restrict__ n_dev, float pdrop, unsigned seed) {
  const int lane = threadIdx.x & 31;
  const int p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n_dev) P = min(P, __ldg(n_dev));          // capacity-sized arrays: the live count sits in device memory
  if (p >= P) return;
  const int b = coors[p * 4];
  const int np = min(npts[p], T);
  const int S = T * V;
  constexpr int NS = 8;  // up to 256 samples per pillar
  float sx[NS], sy[NS];
  bool ok[NS];
#pragma unroll
  for (int s = 0; s < NS; ++s) {
    int i = s * 32 + lane;
    ok[s] = false;
    sx[s] = sy[s] = 0.f;
    if (i < S) {
      int t = i / V, v = i - t * V;  // key index = point*V + cam (reference :298,:309)
      if (t < np) {
        const float* pt = pillars + ((size_t)p * T + t) * pdim;
        float cx, cy, cz;
        project(proj + ((size_t)b * V + v) * 12, pt[0], pt[1], pt[2], cx, cy, cz);
        const float eps = 1e-5f;
        float zz = fmaxf(cz, eps);
        float u = cx / zz, vv = cy / zz;
        float nx = (u / W_in - 0.5f) * 2.f, ny = (vv / H_in - 0.5f) * 2.f;
        ok[s] = (cz > eps) && (nx > -1.f) && (nx < 1.f) && (ny > -1.f) && (ny < 1.f);
        sx[s] = ((nx + 1.f) * (float)w - 1.f) * 0.5f;  // grid_sample un-normalisation, align_corners=False
        sy[s] = ((ny + 1.f) * (float)h - 1.f) * 0.5f;
      }
    }
  }
  float4 q[NJ], acc[NJ];
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    int c = 4 * lane + 128 * j;
    q[j] = c < C ? ldg4(qk + (size_t)p * C + c) : make_float4(0, 0, 0, 0);
    acc[j] = make_float4(0, 0, 0, 0);
  }
  float mrun = -INFINITY, lrun = 0.f, rrun = 0.f;
  int count = 0;
#pragma unroll
  for (int s = 0; s < NS; ++s) {
    unsigned mask = __ballot_sync(0xffffffffu, ok[s]);
    while (mask) {
      int src = __ffs(mask) - 1;
      mask &= mask - 1;
      float ix = __shfl_sync(0xffffffffu, sx[s], src);
      float iy = __shfl_sync(0xffffffffu, sy[s], src);
      int v = (s * 32 + src) % V;
      float4 kv[NJ];
      bilinear_row<NJ>(img + (size_t)(b * V + v) * h * w * C, h, w, C, ix, iy, lane, kv);
      float part = 0.f;
#pragma unroll
      for (int j = 0; j < NJ; ++j)
        part += q[j].x * kv[j].x + q[j].y * kv[j].y + q[j].z * kv[j].z + q[j].w * kv[j].w;
      float logit = warp_sum(part);
      float mnew = fmaxf(mrun, logit);
      float corr = expf(mrun - mnew);
      float pw = expf(logit - mnew);
      lrun = lrun * corr + pw;
      if (DROP) {
        pw *= i2p_keep_scale(seed, p, s * 32 + src, pdrop);               // the normaliser keeps the dropped keys
        rrun = rrun * corr + pw;
      }
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        acc[j].x = acc[j].x * corr + pw * kv[j].x;
        acc[j].y = acc[j].y * corr + pw * kv[j].y;
        acc[j].z = acc[j].z * corr + pw * kv[j].z;
        acc[j].w = acc[j].w * corr + pw * kv[j].w;
      }
      mrun = mnew;
      ++count;
    }
  }
  float inv = count > 0 ? 1.f / lrun : 0.f;
  // DROP: rows of C + 4 floats; column C carries rho = sum_j a_j m_j (the weights no longer sum to 1, and the value bias of
  // nn.MultiheadAttention is weighted by that sum: out = W_o W_v s + rho W_o b_v + b_o), columns C+1..C+3 are 0
  const int ld = DROP ? C + 4 : C;
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    int c = 4 * lane + 128 * j;
    if (c < C)
      *reinterpret_cast<float4*>(s_out + (size_t)p * ld + c) =
          make_float4(acc[j].x * inv, acc[j].y * inv, acc[j].z * inv, acc[j].w * inv);
  }
  if (DROP && lane == 0) *reinterpret_cast<float4*>(s_out + (size_t)p * ld + C) = make_float4(rrun * inv, 0.f, 0.f, 0.f);
  if (lane == 0) cnt_out[p] = count;
}

template <int NJ>
__global__ void __launch_bounds__(256)
i2p_attend_kernel(const float* __restrict__ qk, const float* __restrict__ pillars, const int* __restrict__ npts,
                  const int* __restrict__ coors, const float* __restrict__ proj, const float* __restrict__ img,
                  float* __restrict__ s_out, int* __restrict__ cnt_out, int P, int T, int pdim, int V, int h, int w,
                  int C, float H_in, float W_in, const int* __restrict__ n_dev) {
  i2p_attend_body<NJ, false>(qk, pillars, npts, coors, proj, img, s_out, cnt_out, P, T, pdim, V, h, w, C, H_in, W_in, n_dev, 0.f, 0u);
}
template <int NJ>
__global__ void __launch_bounds__(256)
i2p_attend_drop_kernel(const float* __restrict__ qk, const float* __restrict__ pillars, const int* __restrict__ npts,
                       const int* __restrict__ coors, const float* __restrict__ proj, const float* __restrict__ img,
                       float* __restrict__ s_out, int* __restrict__ cnt_out, int P, int T, int pdim, int V, int h, int w,
                       int C, float H_in, float W_in, const int* __restrict__ n_dev, float pdrop, unsigned seed) {
  i2p_attend_body<NJ, true>(qk, pillars, npts, coors, proj, img, s_out, cnt_out, P, T, pdim, V, h, w, C, H_in, W_in, n_dev, pdrop, seed);
}

// mask[p, key] = 0 or 1 / (1 - p): the factors the two kernels above / below apply (tests, debugging)
__global__ void i2p_dropout_mask_kernel(float* __restrict__ mask, int P, int S, float pdrop, unsigned seed) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < P * S) mask[i] = i2p_keep_scale(seed, i / S, i % S, pdrop);
}

// ------------------------------------------------------------------------------------------------
// I2P backward (SURVEY.md 8(b) `di_i2p_backward`): gradient of s[p] = sum_j softmax_j(qk[p] . k_j) k_j, k_j = bilinear
// sample of the image map at the projection of point j (encoder_utils.py:281-311; forward: i2p_attend_kernel).
// One warp per pillar; pass A recomputes the logits l_j and t_j = ds . k_j, then a = softmax(l), D = sum a t,
// dl_j = a_j (t_j - D); pass B re-samples k_j and emits
//     dqk[p]  = sum_j dl_j k_j
//     dk_j    = a_j ds[p] + dl_j qk[p]   -> scattered into d_img with the bilinear weights (atomicAdd; the sums over
//                                           pillars are order-dependent in the last bit, as in torch's grid_sample backward)
// ------------------------------------------------------------------------------------------------
template <int NJ>
__device__ __forceinline__ void bilinear_scatter(float* __restrict__ dmap, int H, int W, int C, float ix, float iy, int lane,
                                                 const float4 (&g)[NJ]) {
  float fx = floorf(ix), fy = floorf(iy);
  int x0 = (int)fx, y0 = (int)fy;
  float wx1 = ix - fx, wx0 = (fx + 1.f) - ix;
  float wy1 = iy - fy, wy0 = (fy + 1.f) - iy;
  float wgt[4] = {wx0 * wy0, wx1 * wy0, wx0 * wy1, wx1 * wy1};
  if (!(ix > -2.f && ix < (float)W + 1.f && iy > -2.f && iy < (float)H + 1.f)) return;
#pragma unroll
  for (int cnr = 0; cnr < 4; ++cnr) {
    int xx = x0 + (cnr & 1), yy = y0 + (cnr >> 1);
    if (xx < 0 || xx >= W || yy < 0 || yy >= H) continue;
    float* row = dmap + ((size_t)yy * W + xx) * C;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      int c = 4 * lane + 128 * j;
      if (c < C) {
        // one 16-byte vector reduction per lane (red.global.add.v4.f32, sm_90+) instead of four scalar atomics
        atomicAdd(reinterpret_cast<float4*>(row + c),
                  make_float4(g[j].x * wgt[cnr], g[j].y * wgt[cnr], g[j].z * wgt[cnr], g[j].w * wgt[cnr]));
      }
    }
  }
}

template <int NJ, bool DROP>
__device__ __forceinline__ void
i2p_attend_bwd_body(const float* __restrict__ qk, const float* __restrict__ ds, const float* __restrict__ pillars,
                    const int* __restrict__ npts, const int* __restrict__ coors, const float* __restrict__ proj,
                    const float* __restrict__ img, float* __restrict__ d_img, float* __restrict__ dqk, int P, int T, int pdim,
                    int V, int h, int w, int C, float H_in, float W_in, const int* __restrict__ n_dev, float pdrop, unsigned seed) {
  const int lane = threadIdx.x & 31;
  const int p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n_dev) P = min(P, __ldg(n_dev));
  if (p >= P) return;
  const int b = coors[p * 4];
  const int np = min(npts[p], T);
  const int S = T * V;
  constexpr int NS = 8;
  float sx[NS], sy[NS], lg[NS], tv[NS];
  bool ok[NS];
#pragma unroll
  for (int s = 0; s < NS; ++s) {
    int i = s * 32 + lane;
    ok[s] = false;
    sx[s] = sy[s] = 0.f;
    lg[s] = -INFINITY;
    tv[s] = 0.f;
    if (i < S) {
      int t = i / V, v = i - t * V;
      if (t < np) {
        const float* pt = pillars + ((size_t)p * T + t) * pdim;
        float cx, cy, cz;
        project(proj + ((size_t)b * V + v) * 12, pt[0], pt[1], pt[2], cx, cy, cz);
        const float eps = 1e-5f;
        float zz = fmaxf(cz, eps);
        float u = cx / zz, vv = cy / zz;
        float nx = (u / W_in - 0.5f) * 2.f, ny = (vv / H_in - 0.5f) * 2.f;
        ok[s] = (cz > eps) && (nx > -1.f) && (nx < 1.f) && (ny > -1.f) && (ny < 1.f);
        sx[s] = ((nx + 1.f) * (float)w - 1.f) * 0.5f;
        sy[s] = ((ny + 1.f) * (float)h - 1.f) * 0.5f;
      }
    }
  }
  float4 q[NJ], g[NJ], acc[NJ];
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    int c = 4 * lane + 128 * j;
    q[j] = c < C ? ldg4(qk + (size_t)p * C + c) : make_float4(0, 0, 0, 0);
    g[j] = c < C ? ldg4(ds + (size_t)p * (DROP ? C + 4 : C) + c) : make_float4(0, 0, 0, 0);
    acc[j] = make_float4(0, 0, 0, 0);
  }
  const float drho = DROP ? __ldg(ds + (size_t)p * (C + 4) + C) : 0.f;     // gradient of rho (column C of the forward's rows)
  // pass A: logits and t_j
  int count = 0;
#pragma unroll
  for (int s = 0; s < NS; ++s) {
    unsigned mask = __ballot_sync(0xffffffffu, ok[s]);
    while (mask) {
      int src = __ffs(mask) - 1;
      mask &= mask - 1;
      float ix = __shfl_sync(0xffffffffu, sx[s], src), iy = __shfl_sync(0xffffffffu, sy[s], src);
      int v = (s * 32 + src) % V;
      float4 kv[NJ];
      bilinear_row<NJ>(img + (size_t)(b * V + v) * h * w * C, h, w, C, ix, iy, lane, kv);
      float pl = 0.f, pt = 0.f;
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        pl += q[j].x * kv[j].x + q[j].y * kv[j].y + q[j].z * kv[j].z + q[j].w * kv[j].w;
        pt += g[j].x * kv[j].x + g[j].y * kv[j].y + g[j].z * kv[j].z + g[j].w * kv[j].w;
      }
      pl = warp_sum(pl);
      pt = warp_sum(pt);
      if (lane == src) { lg[s] = pl; tv[s] = pt; }
      ++count;
    }
  }
  if (count > 0) {
    float m = -INFINITY;
#pragma unroll
    for (int s = 0; s < NS; ++s) m = fmaxf(m, lg[s]);
    m = warp_max(m);
    float L = 0.f;
#pragma unroll
    for (int s = 0; s < NS; ++s) {
      lg[s] = ok[s] ? expf(lg[s] - m) : 0.f;          // now the un-normalised weights
      L += lg[s];
    }
    L = warp_sum(L);
    const float inv = 1.f / L;
    float D = 0.f;
#pragma unroll
    for (int s = 0; s < NS; ++s) {
      lg[s] *= inv;                                    // a_j
      if (DROP) tv[s] = (tv[s] + drho) * i2p_keep_scale(seed, p, s * 32 + lane, pdrop);   // [s, rho] = sum a_j m_j [k_j, 1]
      D += lg[s] * tv[s];
    }
    D = warp_sum(D);
#pragma unroll
    for (int s = 0; s < NS; ++s) tv[s] = lg[s] * (tv[s] - D);   // dl_j
    // pass B
#pragma unroll
    for (int s = 0; s < NS; ++s) {
      unsigned mask = __ballot_sync(0xffffffffu, ok[s]);
      while (mask) {
        int src = __ffs(mask) - 1;
        mask &= mask - 1;
        float ix = __shfl_sync(0xffffffffu, sx[s], src), iy = __shfl_sync(0xffffffffu, sy[s], src);
        float a = __shfl_sync(0xffffffffu, lg[s], src), dl = __shfl_sync(0xffffffffu, tv[s], src);
        if (DROP) a *= i2p_keep_scale(seed, p, s * 32 + src, pdrop);       // the direct path carries a_j m_j
        int v = (s * 32 + src) % V;
        float4 kv[NJ], dk[NJ];
        bilinear_row<NJ>(img + (size_t)(b * V + v) * h * w * C, h, w, C, ix, iy, lane, kv);
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          acc[j].x = fmaf(dl, kv[j].x, acc[j].x);
          acc[j].y = fmaf(dl, kv[j].y, acc[j].y);
          acc[j].z = fmaf(dl, kv[j].z, acc[j].z);
          acc[j].w = fmaf(dl, kv[j].w, acc[j].w);
          dk[j] = make_float4(a * g[j].x + dl * q[j].x, a * g[j].y + dl * q[j].y, a * g[j].z + dl * q[j].z,
                              a * g[j].w + dl * q[j].w);
        }
        bilinear_scatter<NJ>(d_img + (size_t)(b * V + v) * h * w * C, h, w, C, ix, iy, lane, dk);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    int c = 4 * lane + 128 * j;
    if (c < C) *reinterpret_cast<float4*>(dqk + (size_t)p * C + c) = acc[j];
  }
}

template <int NJ>
__global__ void __launch_bounds__(256)
i2p_attend_bwd_kernel(const float* __restrict__ qk, const float* __restrict__ ds, const float* __restrict__ pillars,
                      const int* __restrict__ npts, const int* __restrict__ coors, const float* __restrict__ proj,
                      const float* __restrict__ img, float* __restrict__ d_img, float* __restrict__ dqk, int P, int T, int pdim,
                      int V, int h, int w, int C, float H_in, float W_in, const int* __restrict__ n_dev) {
  i2p_attend_bwd_body<NJ, false>(qk, ds, pillars, npts, coors, proj, img, d_img, dqk, P, T, pdim, V, h, w, C, H_in, W_in, n_dev, 0.f, 0u);
}
template <int NJ>
__global__ void __launch_bounds__(256)
i2p_attend_bwd_drop_kernel(const float* __restrict__ qk, const float* __restrict__ ds, const float* __restrict__ pillars,
                           const int* __restrict__ npts, const int* __restrict__ coors, const float* __restrict__ proj,
                           const float* __restrict__ img, float* __restrict__ d_img, float* __restrict__ dqk, int P, int T,
                           int pdim, int V, int h, int w, int C, float H_in, float W_in, const int* __restrict__ n_dev, float pdrop,
                           unsigned seed) {
  i2p_attend_bwd_body<NJ, true>(qk, ds, pillars, npts, coors, proj, img, d_img, dqk, P, T, pdim, V, h, w, C, H_in, W_in, n_dev, pdrop, seed);
}

// rows[p,:] = cnt[p] > 0 ? map[b, y, x, :] : 0   (transpose of scatter_rows_kernel)
__global__ void gather_rows_masked_kernel(const float* __restrict__ map, const int* __restrict__ cnt,
                                          const int* __restrict__ coors, float* __restrict__ rows, int P, int Y, int X, int C) {
  int p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  int lane = threadIdx.x & 31;
  if (p >= P) return;
  const int* c4 = coors + p * 4;
  const float* src = map + (((size_t)c4[0] * Y + c4[2]) * X + c4[3]) * C;
  const bool on = cnt[p] > 0;
  for (int c = lane * 4; c < C; c += 128)
    *reinterpret_cast<float4*>(rows + (size_t)p * C + c) = on ? ldg4(src + c) : make_float4(0, 0, 0, 0);
}

// rows[p,:] = map[b, y, x, :]   (coors = [b, z, y, x])
__global__ void gather_rows_kernel(const float* __restrict__ map, const int* __restrict__ coors, float* __restrict__ rows,
                                   int P, int Y, int X, int C, const int* __restrict__ n_dev) {
  int p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  int lane = threadIdx.x & 31;
  if (n_dev) P = min(P, __ldg(n_dev));
  if (p >= P) return;
  const int* c4 = coors + p * 4;
  const float* src = map + (((size_t)c4[0] * Y + c4[2]) * X + c4[3]) * C;
  for (int c = lane * 4; c < C; c += 128) *reinterpret_cast<float4*>(rows + (size_t)p * C + c) = ldg4(src + c);
}

// map[b, y, x, :] = cnt[p] > 0 ? rows[p,:] : 0
__global__ void scatter_rows_kernel(const float* __restrict__ rows, const int* __restrict__ cnt,
                                    const int* __restrict__ coors, float* __restrict__ map, int P, int Y, int X, int C,
                                    const int* __restrict__ n_dev) {
  int p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  int lane = threadIdx.x & 31;
  if (n_dev) P = min(P, __ldg(n_dev));
  if (p >= P) return;
  const int* c4 = coors + p * 4;
  float* dst = map + (((size_t)c4[0] * Y + c4[2]) * X + c4[3]) * C;
  bool on = cnt[p] > 0;
  for (int c = lane * 4; c < C; c += 128)
    *reinterpret_cast<float4*>(dst + c) = on ? ldg4(rows + (size_t)p * C + c) : make_float4(0, 0, 0, 0);
}

// ------------------------------------------------------------------------------------------------
// BEVWarp stage 1: sparse depth maps.  key = (point index + 1) << 32 | depth bits; atomicMax keeps the
// LAST point in order for duplicate pixels (the CPU index_put_ rule the oracle follows).
// ------------------------------------------------------------------------------------------------
__global__ void depth_scatter_kernel(const float* __restrict__ pts, int stride, int n, const float* __restrict__ proj,
                                     unsigned long long* __restrict__ keys, int V, int h, int w, float H_in, float W_in,
                                     const int* __restrict__ n_dev) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (n_dev) n = min(n, __ldg(n_dev));
  if (i >= n) return;
  float x = pts[(size_t)i * stride], y = pts[(size_t)i * stride + 1], z = pts[(size_t)i * stride + 2];
  for (int v = 0; v < V; ++v) {
    float cx, cy, cz;
    project(proj + v * 12, x, y, z, cx, cy, cz);
    const float eps = 1e-5f;
    float zz = fmaxf(cz, eps);
    float u = cx / zz, vv = cy / zz;
    float nx = (u / W_in - 0.5f) * 2.f, ny = (vv / H_in - 0.5f) * 2.f;
    bool ok = (cz > eps) && (nx > -1.f) && (nx < 1.f) && (ny > -1.f) && (ny < 1.f);
    if (!ok) continue;
    int r = (int)(vv / H_in * (float)h), c = (int)(u / W_in * (float)w);   // .long() truncation (:174)
    if (r < 0 || r >= h || c < 0 || c >= w) continue;
    unsigned long long key = ((unsigned long long)(unsigned)(i + 1) << 32) | __float_as_uint(cz);
    atomicMax(keys + ((size_t)v * h + r) * w + c, key);
  }
}

// ------------------------------------------------------------------------------------------------
// BEVWarp stage 2: depth completion (ip_basic fill_in_multiscale, extrapolate=False, bilateral).
// One thread-block CLUSTER of DC_CL CTAs per camera image (the ~18 dependent stencil stages are bound by the per-SM
// L2 load rate, so the pixels of an image are dealt over DC_CL SMs); planes live in global scratch (L2) and are
// read with ld.cg, so every stage sees the previous stage's stores after the cluster barrier (release / acquire at
// cluster scope).  Column scans and the min/max reduction are done redundantly by every CTA of the cluster.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float ldcg(const float* p) { return __ldcg(p); }

constexpr int DC_CL = 8;

__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ unsigned cluster_cta_rank() {
  unsigned r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}

template <class F>
__device__ __forceinline__ void for_pixels(int n, F f) {
  for (int i = cluster_cta_rank() * blockDim.x + threadIdx.x; i < n; i += DC_CL * blockDim.x) f(i);
}

// max over a full (2r+1)^2 window, out-of-image ignored
__device__ __forceinline__ float dil_full(const float* src, int h, int w, int y, int x, int r) {
  float m = -INFINITY;
  int y0 = max(0, y - r), y1 = min(h - 1, y + r), x0 = max(0, x - r), x1 = min(w - 1, x + r);
  for (int yy = y0; yy <= y1; ++yy)
    for (int xx = x0; xx <= x1; ++xx) m = fmaxf(m, ldcg(src + yy * w + xx));
  return m;
}
__device__ __forceinline__ float ero_full(const float* src, int h, int w, int y, int x, int r) {
  float m = INFINITY;
  int y0 = max(0, y - r), y1 = min(h - 1, y + r), x0 = max(0, x - r), x1 = min(w - 1, x + r);
  for (int yy = y0; yy <= y1; ++yy)
    for (int xx = x0; xx <= x1; ++xx) m = fminf(m, ldcg(src + yy * w + xx));
  return m;
}
// exact median of the 5x5 neighbourhood, replicate border (cv2.medianBlur float32)
__device__ float median5(const float* src, int h, int w, int y, int x) {
  float v[25];
#pragma unroll
  for (int dy = -2; dy <= 2; ++dy)
#pragma unroll
    for (int dx = -2; dx <= 2; ++dx) {
      int yy = min(max(y + dy, 0), h - 1), xx = min(max(x + dx, 0), w - 1);
      v[(dy + 2) * 5 + dx + 2] = ldcg(src + yy * w + xx);
    }
  // partial selection: after 13 passes v[12] is the 13th smallest
#pragma unroll
  for (int i = 0; i <= 12; ++i) {
#pragma unroll
    for (int j = i + 1; j < 25; ++j) {
      float a = v[i], b = v[j];
      v[i] = fminf(a, b);
      v[j] = fmaxf(a, b);
    }
  }
  return v[12];
}

__device__ __forceinline__ float invert_depth(float d) { return d > 0.1f ? 100.0f - d : d; }

__global__ void __cluster_dims__(DC_CL, 1, 1) __launch_bounds__(1024)
depth_complete_kernel(const unsigned long long* __restrict__ keys, float* __restrict__ scratch, float* __restrict__ out,
                      float* __restrict__ sparse_out, int h, int w) {
  const int n = h * w;
  const size_t img = blockIdx.x / DC_CL;
  const unsigned long long* key = keys + img * n;
  float* A = scratch + img * 3 * n;
  float* Bp = A + n;
  float* Cp = Bp + n;
  extern __shared__ int first_row[];  // [w]
  __shared__ float red_min[32], red_max[32];
  __shared__ float s_min, s_max;

  // S0: raw sparse depth -> A (kept as d0)
  for_pixels(n, [&](int i) {
    unsigned long long kk = key[i];
    float d = kk ? __uint_as_float((unsigned)(kk & 0xffffffffu)) : 0.f;
    A[i] = d;
    if (sparse_out) sparse_out[img * n + i] = d;
  });
  cluster_sync_all();
  // S1: per-bin cross dilations (3: far, 5: medium, 7: near), merged far -> near; B = s2
  for_pixels(n, [&](int i) {
    int y = i / w, x = i - y * w;
    float d0 = ldcg(A + i);
    float far_m = -INFINITY, med_m = -INFINITY, near_m = -INFINITY;
    auto visit = [&](int yy, int xx, int dist) {
      if (yy < 0 || yy >= h || xx < 0 || xx >= w) return;
      float d = ldcg(A + yy * w + xx);
      float s1 = invert_depth(d);
      float vf = d > 30.0f ? s1 : 0.f * s1;
      float vm = (d > 15.0f && d <= 30.0f) ? s1 : 0.f * s1;
      float vn = (d > 0.1f && d <= 15.0f) ? s1 : 0.f * s1;
      if (dist <= 1) far_m = fmaxf(far_m, vf);
      if (dist <= 2) med_m = fmaxf(med_m, vm);
      near_m = fmaxf(near_m, vn);
    };
    visit(y, x, 0);
    for (int k = 1; k <= 3; ++k) {
      visit(y - k, x, k);
      visit(y + k, x, k);
      visit(y, x - k, k);
      visit(y, x + k, k);
    }
    float s2 = invert_depth(d0);
    if (far_m > 0.1f) s2 = far_m;
    if (med_m > 0.1f) s2 = med_m;
    if (near_m > 0.1f) s2 = near_m;
    Bp[i] = s2;
  });
  cluster_sync_all();
  // S2: 5x5 closing: C = dilate(B); A = erode(C) = s3
  for_pixels(n, [&](int i) { Cp[i] = dil_full(Bp, h, w, i / w, i % w, 2); });
  cluster_sync_all();
  for_pixels(n, [&](int i) { A[i] = ero_full(Cp, h, w, i / w, i % w, 2); });
  cluster_sync_all();
  // S3: median where valid; B = s4
  for_pixels(n, [&](int i) {
    float s3 = ldcg(A + i);
    Bp[i] = s3 > 0.1f ? median5(A, h, w, i / w, i % w) : s3;
  });
  cluster_sync_all();
  // S4: top mask of s4
  // first row with a valid value per column (argmax of an all-false column is 0); every CTA builds its own copy
  auto top_mask = [&](const float* src) {
    for (int x = threadIdx.x; x < w; x += blockDim.x) first_row[x] = h;
    __syncthreads();
    // thread t scans column t % w over the rows t / w, t / w + groups, ...  (w <= blockDim.x: checked by the host)
    const int groups = blockDim.x / w, g = threadIdx.x / w, x = threadIdx.x - g * w;
    if (g < groups) {
      int f = h;
#pragma unroll 4
      for (int y = g; y < h; y += groups)
        if (ldcg(src + y * w + x) > 0.1f) f = min(f, y);
      if (f < h) atomicMin(&first_row[x], f);
    }
    __syncthreads();
    for (int x1 = threadIdx.x; x1 < w; x1 += blockDim.x)
      if (first_row[x1] == h) first_row[x1] = 0;
    __syncthreads();
  };
  top_mask(Bp);
  // S5: fill empties under the top mask with a 9x9 dilation; A = s5
  for_pixels(n, [&](int i) {
    int y = i / w, x = i - y * w;
    float s4 = ldcg(Bp + i);
    bool empty = !(s4 > 0.1f) && y >= first_row[x];
    A[i] = empty ? dil_full(Bp, h, w, y, x, 4) : s4;
  });
  cluster_sync_all();
  // S6: top mask of s5
  top_mask(A);
  // S7: six masked 5x5 dilations, ping-pong A -> B -> A ... (ends in A)
  float* src = A;
  float* dst = Bp;
  for (int it = 0; it < 6; ++it) {
    for_pixels(n, [&](int i) {
      int y = i / w, x = i - y * w;
      float s = ldcg(src + i);
      bool empty = (s < 0.1f) && y >= first_row[x];
      dst[i] = empty ? dil_full(src, h, w, y, x, 2) : s;
    });
    cluster_sync_all();
    float* tmp = src;
    src = dst;
    dst = tmp;
  }
  // src == A holds s7 (pre-median).  S8: median where valid (mask from pre-median values); B = s7m
  for_pixels(n, [&](int i) {
    int y = i / w, x = i - y * w;
    float s = ldcg(A + i);
    bool valid = (s > 0.1f) && y >= first_row[x];
    Bp[i] = valid ? median5(A, h, w, y, x) : s;
  });
  cluster_sync_all();
  // S9: bilateral (d=5, sigmaColor=0.5, sigmaSpace=2) of s7m, written at the pre-median mask; re-invert
  {
    float mn = INFINITY, mx = -INFINITY;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      float s = ldcg(Bp + i);
      mn = fminf(mn, s);
      mx = fmaxf(mx, s);
    }
    mn = -warp_max(-mn);
    mx = warp_max(mx);
    if ((threadIdx.x & 31) == 0) {
      red_min[threadIdx.x >> 5] = mn;
      red_max[threadIdx.x >> 5] = mx;
    }
    __syncthreads();
    if (threadIdx.x < 32) {
      int nw = blockDim.x >> 5;
      float a = threadIdx.x < nw ? red_min[threadIdx.x] : INFINITY;
      float b = threadIdx.x < nw ? red_max[threadIdx.x] : -INFINITY;
      a = -warp_max(-a);
      b = warp_max(b);
      if (threadIdx.x == 0) {
        s_min = a;
        s_max = b;
      }
    }
    __syncthreads();
  }
  const float len = s_max - s_min;
  const bool flat = fabsf(len) < 1.1920929e-07f;
  const float scale_index = 4096.0f / len;
  const float sw1 = (float)exp(-0.125), sw2 = (float)exp(-0.25), sw4 = (float)exp(-0.5);  // r^2 * (-0.5/2^2)
  for_pixels(n, [&](int i) {
    int y = i / w, x = i - y * w;
    float s7 = ldcg(A + i);
    float val0 = ldcg(Bp + i);
    bool valid = (s7 > 0.1f) && y >= first_row[x];
    float res = val0;
    if (valid && !flat) {
      float sum = 0.f, wsum = 0.f;
#pragma unroll
      for (int dy = -2; dy <= 2; ++dy)
#pragma unroll
        for (int dx = -2; dx <= 2; ++dx) {
          int r2 = dy * dy + dx * dx;
          if (r2 > 4) continue;
          int yy = y + dy, xx = x + dx;
          yy = yy < 0 ? -yy : (yy >= h ? 2 * h - 2 - yy : yy);   // reflect-101
          xx = xx < 0 ? -xx : (xx >= w ? 2 * w - 2 - xx : xx);
          float val = ldcg(Bp + yy * w + xx);
          float swt = r2 == 0 ? 1.f : (r2 == 1 ? sw1 : (r2 == 2 ? sw2 : sw4));
          float alpha = fabsf(val - val0) * scale_index;
          float fl = floorf(alpha);
          int idx = (int)fl;
          alpha -= fl;
          double v0 = (double)((float)idx / scale_index), v1 = (double)((float)(idx + 1) / scale_index);
          float l0 = (float)exp(v0 * v0 * -2.0), l1 = (float)exp(v1 * v1 * -2.0);
          float wgt = swt * (l0 + alpha * (l1 - l0));
          sum += val * wgt;
          wsum += wgt;
        }
      res = sum / wsum;
    }
    out[img * n + i] = res > 0.1f ? 100.0f - res : res;
  });
}

// ------------------------------------------------------------------------------------------------
// BEVWarp stage 3: lift every feature pixel to LiDAR space and record where it samples the BEV map.
// grid[bv, y, x] = (ix, iy) in BEV pixel space (align_corners=False); outside pc_range -> (-1e30,-1e30)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float linspace_at(int i, int steps, float end) {
  // torch.linspace(0, end, steps): start + step*i for the first half, end - step*(steps-1-i) after
  if (steps == 1) return 0.f;
  float step = end / (float)(steps - 1);
  return i < steps / 2 ? step * (float)i : end - step * (float)(steps - 1 - i);
}

__global__ void lift_kernel(const float* __restrict__ depth, const float* __restrict__ i2l, float2* __restrict__ grid,
                            int h, int w, float H_in, float W_in, int Yb, int Xb, float lo_x, float lo_y, float lo_z,
                            float hi_x, float hi_y, float hi_z, int total) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  int bv = i / (h * w);
  int r = i - bv * h * w;
  int y = r / w, x = r - y * w;
  float d = depth[i];
  float xs = linspace_at(x, w, W_in - 1.f), ys = linspace_at(y, h, H_in - 1.f);
  float X = xs * d, Y = ys * d;
  const float* M = i2l + (size_t)bv * 12;
  float px = M[0] * X + M[1] * Y + M[2] * d + M[3];
  float py = M[4] * X + M[5] * Y + M[6] * d + M[7];
  float pz = M[8] * X + M[9] * Y + M[10] * d + M[11];
  bool ok = px > lo_x && py > lo_y && pz > lo_z && px < hi_x && py < hi_y && pz < hi_z;
  float gx = ((px - lo_x) / (hi_x - lo_x) - 0.5f) * 2.f;
  float gy = ((py - lo_y) / (hi_y - lo_y) - 0.5f) * 2.f;
  float ix = ((gx + 1.f) * (float)Xb - 1.f) * 0.5f;
  float iy = ((gy + 1.f) * (float)Yb - 1.f) * 0.5f;
  grid[i] = ok ? make_float2(ix, iy) : make_float2(-1e30f, -1e30f);
}

// BEVWarp stage 4: warped[bv, y, x, :] = bilinear(bev[b], grid[bv, y, x]); one warp per pixel.
template <int NJ>
__global__ void __launch_bounds__(256)
bev_sample_kernel(const float* __restrict__ bev, const float2* __restrict__ grid, float* __restrict__ out, int V,
                  int hw, int Yb, int Xb, int C, int total) {
  int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  int lane = threadIdx.x & 31;
  if (i >= total) return;
  int b = i / (V * hw);
  float2 g = grid[i];
  float4 v[NJ];
  bilinear_row<NJ>(bev + (size_t)b * Yb * Xb * C, Yb, Xb, C, g.x, g.y, lane, v);
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    int c = 4 * lane + 128 * j;
    if (c < C) *reinterpret_cast<float4*>(out + (size_t)i * C + c) = v[j];
  }
}

// transpose of bev_sample_kernel: d_bev[b] += bilinear scatter of d_out[bv, y, x, :] at grid[bv, y, x]
template <int NJ>
__global__ void __launch_bounds__(256)
bev_sample_bwd_kernel(const float* __restrict__ d_out, const float2* __restrict__ grid, float* __restrict__ d_bev, int V, int hw,
                      int Yb, int Xb, int C, int total) {
  int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  int lane = threadIdx.x & 31;
  if (i >= total) return;
  int b = i / (V * hw);
  float2 g = grid[i];
  float4 v[NJ];
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    int c = 4 * lane + 128 * j;
    v[j] = c < C ? ldg4(d_out + (size_t)i * C + c) : make_float4(0, 0, 0, 0);
  }
  bilinear_scatter<NJ>(d_bev + (size_t)b * Yb * Xb * C, Yb, Xb, C, g.x, g.y, lane, v);
}

}  // namespace

extern "C" {

// n_dev (all four entry points below; may be NULL): device pointer to the LIVE element count when the arrays are
// allocated at capacity P / n -- the kernels then process min(capacity, *n_dev) elements.  This keeps launch
// configurations and buffer addresses independent of the per-frame pillar / point counts (CUDA-graph replay).
int di_gather_rows_f32(const float* map, const int* coors, float* rows, int P, int Y, int X, int C, const int* n_dev,
                       cudaStream_t stream) {
  DI_CHECK_ARG(P >= 0 && C % 4 == 0, "di_gather_rows_f32: bad argument");
  if (P == 0) return DI_OK;                     // empty tensors may have null data pointers
  DI_CHECK_ARG(map && coors && rows, "di_gather_rows_f32: null pointer");
  gather_rows_kernel<<<di_cdiv(P, 8), 256, 0, stream>>>(map, coors, rows, P, Y, X, C, n_dev);
  DI_CHECK_LAUNCH("di_gather_rows_f32");
  return DI_OK;
}

int di_scatter_rows_f32(const float* rows, const int* cnt, const int* coors, float* map, int P, int Y, int X, int C,
                        const int* n_dev, cudaStream_t stream) {
  DI_CHECK_ARG(P >= 0 && C % 4 == 0, "di_scatter_rows_f32: bad argument");
  if (P == 0) return DI_OK;
  DI_CHECK_ARG(map && coors && rows && cnt, "di_scatter_rows_f32: null pointer");
  scatter_rows_kernel<<<di_cdiv(P, 8), 256, 0, stream>>>(rows, cnt, coors, map, P, Y, X, C, n_dev);
  DI_CHECK_LAUNCH("di_scatter_rows_f32");
  return DI_OK;
}

// qk [P,C]: folded queries (W_k^T (W_q q + b_q) / sqrt(C)); s_out [P,C] = sum_j softmax_j(qk.k_j) k_j over the
// valid projected samples of each pillar; cnt_out [P] = number of valid samples (0 => s_out row is 0).
// proj [B,V,12]: rows 0..2 of lidar2img[b,v] @ undo-augmentation; img [B*V,h,w,C] pixel-major.
int di_i2p_attend_f32(const float* qk, const float* pillars, const int* npts, const int* coors, const float* proj,
                      const float* img, float* s_out, int* cnt_out, int P, int T, int pdim, int V, int h, int w, int C,
                      int H_in, int W_in, const int* n_dev, cudaStream_t stream) {
  DI_CHECK_ARG(qk && pillars && npts && coors && proj && img && s_out && cnt_out, "di_i2p_attend_f32: null pointer");
  DI_CHECK_ARG(C % 4 == 0 && C <= 512 && pdim >= 3 && T * V <= 256, "di_i2p_attend_f32: unsupported shape (C=%d T=%d V=%d)", C, T, V);
  if (P == 0) return DI_OK;
  dim3 grid(di_cdiv(P, 8));
  if (C <= 128)
    i2p_attend_kernel<1><<<grid, 256, 0, stream>>>(qk, pillars, npts, coors, proj, img, s_out, cnt_out, P, T, pdim, V, h, w, C, (float)H_in, (float)W_in, n_dev);
  else if (C <= 256)
    i2p_attend_kernel<2><<<grid, 256, 0, stream>>>(qk, pillars, npts, coors, proj, img, s_out, cnt_out, P, T, pdim, V, h, w, C, (float)H_in, (float)W_in, n_dev);
  else
    i2p_attend_kernel<4><<<grid, 256, 0, stream>>>(qk, pillars, npts, coors, proj, img, s_out, cnt_out, P, T, pdim, V, h, w, C, (float)H_in, (float)W_in, n_dev);
  DI_CHECK_LAUNCH("di_i2p_attend_f32");
  return DI_OK;
}

// Backward of di_i2p_attend_f32: ds [P,C] = gradient of s_out; d_img [B*V,h,w,C] is ACCUMULATED into (zero it first);
// dqk [P,C] written.  Same geometry arguments as the forward.
int di_i2p_attend_bwd_f32(const float* qk, const float* ds, const float* pillars, const int* npts, const int* coors,
                          const float* proj, const float* img, float* d_img, float* dqk, int P, int T, int pdim, int V, int h,
                          int w, int C, int H_in, int W_in, const int* n_dev, cudaStream_t stream) {
  DI_CHECK_ARG(qk && ds && pillars && npts && coors && proj && img && d_img && dqk, "di_i2p_attend_bwd_f32: null pointer");
  DI_CHECK_ARG(C % 4 == 0 && C <= 512 && pdim >= 3 && T * V <= 256, "di_i2p_attend_bwd_f32: unsupported shape (C=%d T=%d V=%d)", C, T, V);
  if (P == 0) return DI_OK;
  dim3 grid(di_cdiv(P, 8));
  if (C <= 128)
    i2p_attend_bwd_kernel<1><<<grid, 256, 0, stream>>>(qk, ds, pillars, npts, coors, proj, img, d_img, dqk, P, T, pdim, V, h, w, C, (float)H_in, (float)W_in, n_dev);
  else if (C <= 256)
    i2p_attend_bwd_kernel<2><<<grid, 256, 0, stream>>>(qk, ds, pillars, npts, coors, proj, img, d_img, dqk, P, T, pdim, V, h, w, C, (float)H_in, (float)W_in, n_dev);
  else
    i2p_attend_bwd_kernel<4><<<grid, 256, 0, stream>>>(qk, ds, pillars, npts, coors, proj, img, d_img, dqk, P, T, pdim, V, h, w, C, (float)H_in, (float)W_in, n_dev);
  DI_CHECK_LAUNCH("di_i2p_attend_bwd_f32");
  return DI_OK;
}

// Training-mode variants with attention dropout (pdrop in [0, 1), mask = hash(seed, pillar, key); see i2p_keep_scale).
// s_out (forward) and ds (backward) are [P, C + 4] here: column C = rho = sum_j a_j m_j resp. its gradient, C+1..C+3 = 0.
int di_i2p_attend_dropout_f32(const float* qk, const float* pillars, const int* npts, const int* coors, const float* proj,
                              const float* img, float* s_out, int* cnt_out, int P, int T, int pdim, int V, int h, int w, int C,
                              int H_in, int W_in, const int* n_dev, float pdrop, unsigned int seed, cudaStream_t stream) {
  DI_CHECK_ARG(qk && pillars && npts && coors && proj && img && s_out && cnt_out, "di_i2p_attend_dropout_f32: null pointer");
  DI_CHECK_ARG(C % 4 == 0 && C <= 512 && pdim >= 3 && T * V <= 256 && pdrop >= 0.f && pdrop < 1.f,
               "di_i2p_attend_dropout_f32: unsupported shape or rate (C=%d T=%d V=%d)", C, T, V);
  if (P == 0) return DI_OK;
  dim3 grid(di_cdiv(P, 8));
  if (C <= 128)
    i2p_attend_drop_kernel<1><<<grid, 256, 0, stream>>>(qk, pillars, npts, coors, proj, img, s_out, cnt_out, P, T, pdim, V, h, w, C, (float)H_in, (float)W_in, n_dev, pdrop, seed);
  else if (C <= 256)
    i2p_attend_drop_kernel<2><<<grid, 256, 0, stream>>>(qk, pillars, npts, coors, proj, img, s_out, cnt_out, P, T, pdim, V, h, w, C, (float)H_in, (float)W_in, n_dev, pdrop, seed);
  else
    i2p_attend_drop_kernel<4><<<grid, 256, 0, stream>>>(qk, pillars, npts, coors, proj, img, s_out, cnt_out, P, T, pdim, V, h, w, C, (float)H_in, (float)W_in, n_dev, pdrop, seed);
  DI_CHECK_LAUNCH("di_i2p_attend_dropout_f32");
  return DI_OK;
}

int di_i2p_attend_bwd_dropout_f32(const float* qk, const float* ds, const float* pillars, const int* npts, const int* coors,
                                  const float* proj, const float* img, float* d_img, float* dqk, int P, int T, int pdim, int V,
                                  int h, int w, int C, int H_in, int W_in, const int* n_dev, float pdrop, unsigned int seed,
                                  cudaStream_t stream) {
  DI_CHECK_ARG(qk && ds && pillars && npts && coors && proj && img && d_img && dqk, "di_i2p_attend_bwd_dropout_f32: null pointer");
  DI_CHECK_ARG(C % 4 == 0 && C <= 512 && pdim >= 3 && T * V <= 256 && pdrop >= 0.f && pdrop < 1.f,
               "di_i2p_attend_bwd_dropout_f32: unsupported shape or rate (C=%d T=%d V=%d)", C, T, V);
  if (P == 0) return DI_OK;
  dim3 grid(di_cdiv(P, 8));
  if (C <= 128)
    i2p_attend_bwd_drop_kernel<1><<<grid, 256, 0, stream>>>(qk, ds, pillars, npts, coors, proj, img, d_img, dqk, P, T, pdim, V, h, w, C, (float)H_in, (float)W_in, n_dev, pdrop, seed);
  else if (C <= 256)
    i2p_attend_bwd_drop_kernel<2><<<grid, 256, 0, stream>>>(qk, ds, pillars, npts, coors, proj, img, d_img, dqk, P, T, pdim, V, h, w, C, (float)H_in, (float)W_in, n_dev, pdrop, seed);
  else
    i2p_attend_bwd_drop_kernel<4><<<grid, 256, 0, stream>>>(qk, ds, pillars, npts, coors, proj, img, d_img, dqk, P, T, pdim, V, h, w, C, (float)H_in, (float)W_in, n_dev, pdrop, seed);
  DI_CHECK_LAUNCH("di_i2p_attend_bwd_dropout_f32");
  return DI_OK;
}

// mask [P, S = T*V]: the factor (0 or 1 / (1 - pdrop)) the two entry points above apply to key `key` of pillar p
int di_i2p_dropout_mask_f32(float* mask, int P, int S, float pdrop, unsigned int seed, cudaStream_t stream) {
  DI_CHECK_ARG(mask && P >= 0 && S > 0 && pdrop >= 0.f && pdrop < 1.f, "di_i2p_dropout_mask_f32: bad argument");
  if (P == 0) return DI_OK;
  i2p_dropout_mask_kernel<<<di_cdiv((long long)P * S, 256), 256, 0, stream>>>(mask, P, S, pdrop, seed);
  DI_CHECK_LAUNCH("di_i2p_dropout_mask_f32");
  return DI_OK;
}

// rows[p] = cnt[p] > 0 ? map[coors[p]] : 0 : the gradient that reaches the attention output of pillar p
int di_gather_rows_masked_f32(const float* map, const int* cnt, const int* coors, float* rows, int P, int Y, int X, int C,
                              cudaStream_t stream) {
  DI_CHECK_ARG(P >= 0 && C % 4 == 0, "di_gather_rows_masked_f32: bad argument");
  if (P == 0) return DI_OK;
  DI_CHECK_ARG(map && cnt && coors && rows, "di_gather_rows_masked_f32: null pointer");
  gather_rows_masked_kernel<<<di_cdiv(P, 8), 256, 0, stream>>>(map, cnt, coors, rows, P, Y, X, C);
  DI_CHECK_LAUNCH("di_gather_rows_masked_f32");
  return DI_OK;
}

// keys [V,h,w] uint64 must be zeroed by the caller; one call per sample (its points + its V projections).
int di_depth_scatter(const float* pts, int stride, int n, const float* proj, unsigned long long* keys, int V, int h,
                     int w, int H_in, int W_in, const int* n_dev, cudaStream_t stream) {
  DI_CHECK_ARG(pts && proj && keys && stride >= 3 && n >= 0, "di_depth_scatter: bad argument");
  if (n == 0) return DI_OK;
  depth_scatter_kernel<<<di_cdiv(n, 256), 256, 0, stream>>>(pts, stride, n, proj, keys, V, h, w, (float)H_in, (float)W_in, n_dev);
  DI_CHECK_LAUNCH("di_depth_scatter");
  return DI_OK;
}

// keys [n_img,h,w] -> dense [n_img,h,w]; scratch: 3*n_img*h*w floats; sparse_out optional (debug/tests).
int di_depth_complete(const unsigned long long* keys, float* scratch, float* dense, float* sparse_out, int n_img, int h,
                      int w, cudaStream_t stream) {
  DI_CHECK_ARG(keys && scratch && dense && n_img > 0 && h > 4 && w > 4, "di_depth_complete: bad argument");
  DI_CHECK_ARG(w <= 1024, "di_depth_complete: image too wide");
  depth_complete_kernel<<<n_img * DC_CL, 1024, w * sizeof(int), stream>>>(keys, scratch, dense, sparse_out, h, w);
  DI_CHECK_LAUNCH("di_depth_complete");
  return DI_OK;
}

// i2l [n_img,12]: rows 0..2 of (re-apply-augmentation @ inverse(lidar2img)); pc_range = lo xyz, hi xyz.
int di_lift_grid(const float* depth, const float* i2l, float* grid_xy, int n_img, int h, int w, int H_in, int W_in,
                 int Yb, int Xb, const float* pc_range6_host, cudaStream_t stream) {
  DI_CHECK_ARG(depth && i2l && grid_xy && pc_range6_host && n_img > 0, "di_lift_grid: bad argument");
  int total = n_img * h * w;
  const float* r = pc_range6_host;
  lift_kernel<<<di_cdiv(total, 256), 256, 0, stream>>>(depth, i2l, reinterpret_cast<float2*>(grid_xy), h, w, (float)H_in,
                                                        (float)W_in, Yb, Xb, r[0], r[1], r[2], r[3], r[4], r[5], total);
  DI_CHECK_LAUNCH("di_lift_grid");
  return DI_OK;
}

// bev [B,Yb,Xb,C], grid [B*V,h*w] (ix,iy) -> out [B*V,h*w,C]
int di_bev_sample_f32(const float* bev, const float* grid_xy, float* out, int B, int V, int hw, int Yb, int Xb, int C,
                      cudaStream_t stream) {
  DI_CHECK_ARG(bev && grid_xy && out && C % 4 == 0 && C <= 512, "di_bev_sample_f32: bad argument");
  int total = B * V * hw;
  dim3 grid(di_cdiv(total, 8));
  const float2* g = reinterpret_cast<const float2*>(grid_xy);
  if (C <= 128)
    bev_sample_kernel<1><<<grid, 256, 0, stream>>>(bev, g, out, V, hw, Yb, Xb, C, total);
  else if (C <= 256)
    bev_sample_kernel<2><<<grid, 256, 0, stream>>>(bev, g, out, V, hw, Yb, Xb, C, total);
  else
    bev_sample_kernel<4><<<grid, 256, 0, stream>>>(bev, g, out, V, hw, Yb, Xb, C, total);
  DI_CHECK_LAUNCH("di_bev_sample_f32");
  return DI_OK;
}

// Backward of di_bev_sample_f32 w.r.t. the BEV map: d_bev [B,Yb,Xb,C] += scatter of d_out [B*V,hw,C] (atomicAdd; zero it first)
int di_bev_sample_bwd_f32(const float* d_out, const float* grid_xy, float* d_bev, int B, int V, int hw, int Yb, int Xb, int C,
                          cudaStream_t stream) {
  DI_CHECK_ARG(d_out && grid_xy && d_bev && C % 4 == 0 && C <= 512, "di_bev_sample_bwd_f32: bad argument");
  int total = B * V * hw;
  dim3 grid(di_cdiv(total, 8));
  const float2* g = reinterpret_cast<const float2*>(grid_xy);
  if (C <= 128)
    bev_sample_bwd_kernel<1><<<grid, 256, 0, stream>>>(d_out, g, d_bev, V, hw, Yb, Xb, C, total);
  else if (C <= 256)
    bev_sample_bwd_kernel<2><<<grid, 256, 0, stream>>>(d_out, g, d_bev, V, hw, Yb, Xb, C, total);
  else
    bev_sample_bwd_kernel<4><<<grid, 256, 0, stream>>>(d_out, g, d_bev, V, hw, Yb, Xb, C, total);
  DI_CHECK_LAUNCH("di_bev_sample_bwd_f32");
  return DI_OK;
}

}  // extern "C"
