// Kernels of the ++ ("deformable") MMRI encoder, DeepInteraction++ (reference
// projects/mmdet3d_plugin/models/necks/fusion_transformerv4.py; BASELINE.json config 4).
//
// di_msdeform_f32 replaces mmcv 1.3.18 MultiScaleDeformableAttention's core (ms_deform_attn CUDA op + the softmax and
// sampling-location arithmetic around it; call sites fusion_transformerv4.py:169-177 self attention over 2 levels,
// :226-238 MMRI_P2I over the warped BEV map): for every query and head, softmax over the L x P attention logits,
// sampling locations = reference point + offset / (W_l, H_l), bilinear zero-padded sampling (grid_sample,
// align_corners=False) of the projected value map, weighted sum.  One warp per query: lane = (head, 4-channel group),
// so every tap of a head is one contiguous 64-byte read of the pixel-major value map; nothing but the output row is
// written (mmcv materialises sampling locations and attention weights, 2 x N x 8 x L x P x 3 floats).
#include <algorithm>

#include "common.cuh"

namespace {

constexpr int MAX_LEVELS = 4;
struct DeformLevels {
  int H[MAX_LEVELS], W[MAX_LEVELS];
};

// value_l [B, H_l, W_l, C] per level (C = heads * d, d == 16, heads == 8 -> 128 channels = 32 lanes x float4);
// raw [B*NQ, ld_raw]: sampling offsets (heads, L, P, 2) then attention logits (heads, L, P) of each query;
// the query grid is Hq x Wq (reference points = pixel centres / (Wq, Hq), fusion_transformerv4.py:129-138)
template <int L, int P>
__global__ void __launch_bounds__(256)
msdeform_kernel(const float* __restrict__ value0, const float* __restrict__ value1, const float* __restrict__ raw,
                int ld_raw, float* __restrict__ out, int ldo, long long total_q, int NQ, int Wq, float inv_wq,
                float inv_hq, DeformLevels lv) {
  const long long q = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (q >= total_q) return;
  const int lane = threadIdx.x & 31;
  const int head = lane >> 2, sub = lane & 3;
  const int b = (int)(q / NQ), qi = (int)(q - (long long)b * NQ);
  const float refx = ((float)(qi % Wq) + 0.5f) * inv_wq, refy = ((float)(qi / Wq) + 0.5f) * inv_hq;
  const float* r = raw + q * ld_raw;
  constexpr int LP = L * P;
  const float* off = r + head * LP * 2;
  const float* lg = r + 8 * LP * 2 + head * LP;
  float w[LP];
  float m = -INFINITY;
#pragma unroll
  for (int i = 0; i < LP; ++i) {
    w[i] = __ldg(lg + i);
    m = fmaxf(m, w[i]);
  }
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < LP; ++i) {
    w[i] = expf(w[i] - m);
    s += w[i];
  }
  const float inv = 1.f / s;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int l = 0; l < L; ++l) {
    const int H = lv.H[l], W = lv.W[l];
    const float* vl = (l == 0 ? value0 : value1) + (size_t)b * H * W * 128 + head * 16 + sub * 4;
#pragma unroll
    for (int p = 0; p < P; ++p) {
      const float ox = __ldg(off + (l * P + p) * 2), oy = __ldg(off + (l * P + p) * 2 + 1);
      // location in [0,1] -> grid_sample(align_corners=False) pixel coordinate: x * W - 0.5
      const float x = (refx + ox / (float)W) * (float)W - 0.5f, y = (refy + oy / (float)H) * (float)H - 0.5f;
      const float x0f = floorf(x), y0f = floorf(y);
      const int x0 = (int)x0f, y0 = (int)y0f;
      const float fx = x - x0f, fy = y - y0f;
      const float wgt = w[l * P + p] * inv;
      const float w00 = (1.f - fx) * (1.f - fy) * wgt, w01 = fx * (1.f - fy) * wgt, w10 = (1.f - fx) * fy * wgt,
                  w11 = fx * fy * wgt;
      const bool xa = x0 >= 0 && x0 < W, xb = x0 + 1 >= 0 && x0 + 1 < W, ya = y0 >= 0 && y0 < H, yb = y0 + 1 >= 0 && y0 + 1 < H;
      if (ya && xa) {
        const float4 t = ldg4(vl + ((size_t)y0 * W + x0) * 128);
        acc.x += w00 * t.x; acc.y += w00 * t.y; acc.z += w00 * t.z; acc.w += w00 * t.w;
      }
      if (ya && xb) {
        const float4 t = ldg4(vl + ((size_t)y0 * W + x0 + 1) * 128);
        acc.x += w01 * t.x; acc.y += w01 * t.y; acc.z += w01 * t.z; acc.w += w01 * t.w;
      }
      if (yb && xa) {
        const float4 t = ldg4(vl + ((size_t)(y0 + 1) * W + x0) * 128);
        acc.x += w10 * t.x; acc.y += w10 * t.y; acc.z += w10 * t.z; acc.w += w10 * t.w;
      }
      if (yb && xb) {
        const float4 t = ldg4(vl + ((size_t)(y0 + 1) * W + x0 + 1) * 128);
        acc.x += w11 * t.x; acc.y += w11 * t.y; acc.z += w11 * t.z; acc.w += w11 * t.w;
      }
    }
  }
  *reinterpret_cast<float4*>(out + q * ldo + head * 16 + sub * 4) = acc;
}

// out = a + s[0] * b   (DeepInteractionLayer: self_feat + scale * query, fusion_transformerv4.py:217)
__global__ void axpy_kernel(const float4* __restrict__ a, const float4* __restrict__ b, const float* __restrict__ s,
                            float4* __restrict__ out, long long n4) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const float sc = __ldg(s);
  const float4 x = a[i], y = b[i];
  out[i] = make_float4(x.x + sc * y.x, x.y + sc * y.y, x.z + sc * y.z, x.w + sc * y.w);
}

// map[b, y, x, :] += cnt[p] > 0 ? rows[p, :] : 0   (++ MMRI_I2P: decorated + lidar_feat, fusion_transformerv4.py:364)
__global__ void scatter_rows_add_kernel(const float* __restrict__ rows, const int* __restrict__ cnt,
                                        const int* __restrict__ coors, float* __restrict__ map, int P, int Y, int X, int C,
                                        const int* __restrict__ n_dev) {
  int p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  int lane = threadIdx.x & 31;
  if (n_dev) P = min(P, __ldg(n_dev));
  if (p >= P || cnt[p] <= 0) return;
  const int* c4 = coors + p * 4;
  float* dst = map + (((size_t)c4[0] * Y + c4[2]) * X + c4[3]) * C;
  for (int c = lane * 4; c < C; c += 128) {
    float4 d = *reinterpret_cast<float4*>(dst + c);
    const float4 r = ldg4(rows + (size_t)p * C + c);
    d.x += r.x; d.y += r.y; d.z += r.z; d.w += r.w;
    *reinterpret_cast<float4*>(dst + c) = d;
  }
}

// ------------------------------------------------------------------------------------------------
// MMRI_I2P_Polar (fusion_transformerv4.py:487-640)
// ------------------------------------------------------------------------------------------------
// Sampling grid of the polar ray queries (:551-577): for camera bv, image column w and radius bin r the BEV pixel
// coordinate (align_corners=False) of  aug( depth_r * normalize( (img2lidar [u, v, 1, 1])_xy - cam_centre ) , z = 0 ).
// cam [BV, 26] per camera: rows 0-1 of inverse(lidar2img) (8 floats), camera centre xy (2), forward augmentation
// affine rows 0-1 (8: x' = a0 x + a1 y + a2 z + a3 ...), then 8 unused.
__global__ void polar_grid_kernel(const float* __restrict__ cam, float2* __restrict__ grid, int BV, int R, int W,
                                  float u_scale, float v_pix, float r0, float r_step, float x_min, float x_rng, float y_min,
                                  float y_rng, int Xb, int Yb) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= BV * R * W) return;
  const int w = i % W, r = (i / W) % R, bv = i / (W * R);
  const float* c = cam + bv * 26;
  const float u = ((float)w + 0.5f) * u_scale, v = v_pix;
  const float lx = c[0] * u + c[1] * v + c[2] + c[3], ly = c[4] * u + c[5] * v + c[6] + c[7];
  float dx = lx - c[8], dy = ly - c[9];
  const float nrm = sqrtf(dx * dx + dy * dy);
  dx /= nrm;
  dy /= nrm;
  const float depth = r0 + ((float)r + 0.5f) * r_step;
  const float px = depth * dx, py = depth * dy;                       // z = 0
  const float ax = c[10] * px + c[11] * py + c[13], ay = c[14] * px + c[15] * py + c[17];
  const float nx = (ax - x_min) / x_rng, ny = (ay - y_min) / y_rng;   // [0, 1]
  grid[i] = make_float2(nx * (float)Xb - 0.5f, ny * (float)Yb - 0.5f);
}

// out[m, :] = x[m, :] + pos[m % mod, :]   (positional encodings are constant tables, broadcast over the cameras)
__global__ void add_rows_mod_kernel(const float4* __restrict__ x, const float4* __restrict__ pos, float4* __restrict__ out,
                                    long long n4, long long mod4) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const float4 a = x[i], b = __ldg(pos + i % mod4);
  out[i] = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
}

// Multi-head attention over short sequences laid out as image columns: sequence (g, w) has its token t at row
// (g * L + t) * Wn + w of a [G, L, Wn, *] row tensor (no transposition of the maps).  One warp per (sequence, head);
// lane = query token (two rounds cover Lq <= 64), keys / values broadcast through L1.  d = 16 channels per head.
__global__ void __launch_bounds__(256)
seq_attn_kernel(const float* __restrict__ q, int ldq, const float* __restrict__ k, int ldk, const float* __restrict__ v,
                int ldv, float* __restrict__ out, int ldo, int G, int Wn, int Lq, int Lk, int heads, float scale) {
  const int wid = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (wid >= G * Wn * heads) return;
  const int head = wid % heads, seq = wid / heads;
  const int w = seq % Wn, g = seq / Wn;
  for (int t0 = 0; t0 < Lq; t0 += 32) {
    const int t = t0 + lane;
    const bool on = t < Lq;
    float qv[16], acc[16];
    const float* qp = q + ((size_t)(g * Lq + (on ? t : 0)) * Wn + w) * ldq + head * 16;
#pragma unroll
    for (int c = 0; c < 16; c += 4) {
      const float4 x = ldg4(qp + c);
      qv[c] = x.x * scale; qv[c + 1] = x.y * scale; qv[c + 2] = x.z * scale; qv[c + 3] = x.w * scale;
      acc[c] = acc[c + 1] = acc[c + 2] = acc[c + 3] = 0.f;
    }
    float m = -INFINITY, l = 0.f;
    for (int j = 0; j < Lk; ++j) {
      const size_t row = (size_t)(g * Lk + j) * Wn + w;
      const float* kp = k + row * ldk + head * 16;
      const float* vp = v + row * ldv + head * 16;
      float s = 0.f;
#pragma unroll
      for (int c = 0; c < 16; c += 4) {
        const float4 x = ldg4(kp + c);
        s += qv[c] * x.x + qv[c + 1] * x.y + qv[c + 2] * x.z + qv[c + 3] * x.w;
      }
      const float mn = fmaxf(m, s);
      const float corr = expf(m - mn), pw = expf(s - mn);
      l = l * corr + pw;
#pragma unroll
      for (int c = 0; c < 16; c += 4) {
        const float4 x = ldg4(vp + c);
        acc[c] = acc[c] * corr + pw * x.x;
        acc[c + 1] = acc[c + 1] * corr + pw * x.y;
        acc[c + 2] = acc[c + 2] * corr + pw * x.z;
        acc[c + 3] = acc[c + 3] * corr + pw * x.w;
      }
      m = mn;
    }
    if (on) {
      const float inv = 1.f / l;
      float* op = out + ((size_t)(g * Lq + t) * Wn + w) * ldo + head * 16;
#pragma unroll
      for (int c = 0; c < 16; c += 4)
        *reinterpret_cast<float4*>(op + c) = make_float4(acc[c] * inv, acc[c + 1] * inv, acc[c + 2] * inv, acc[c + 3] * inv);
    }
  }
}

struct PolarParams {
  int B, V, R, W, Y, X, Z;
  float H_in, W_in, x_min, x_rng, y_min, y_rng, z_min, z_rng, r0, r_cnt;
};

// Rays -> BEV (:579-636): one warp per BEV cell.  Per camera, lanes 0..Z-1 project the cell's Z height samples
// (undo the augmentation, lidar2img), the warp averages (pixel x, clamped radius) over ALL samples and ORs the strict
// in-image / depth masks (the reference's .mean(dim=3) / .sum(dim=3) > 0), then every lane gathers its 4 channels of the
// decoded rays bilinearly (zeros outside, align_corners=False); cameras that see the cell are averaged; + residual.
// proj [B,V,12]: rows 0-2 of lidar2img @ undo-aug; undo [B,12]: rows 0-2 of the undo-aug affine; camc [B*V,2].
//
// polar_cell / polar_cell_loc hold the per-(cell, camera) arithmetic, so that the gather and its adjoint use the same
// positions, masks and camera count.
struct PolarCell {
  int b;
  float px, py, pz, rx, ry;
};

__device__ __forceinline__ PolarCell polar_cell(const float* __restrict__ undo, const PolarParams& p, int cell, int lane) {
  PolarCell c;
  const int ix = cell % p.X, iy = (cell / p.X) % p.Y;
  c.b = cell / (p.X * p.Y);
  c.px = ((float)ix + 0.5f) / (float)p.X * p.x_rng + p.x_min;
  c.py = ((float)iy + 0.5f) / (float)p.Y * p.y_rng + p.y_min;
  c.pz = ((float)(lane < p.Z ? lane : 0) + 0.5f) / (float)p.Z * p.z_rng + p.z_min;
  const float* ua = undo + c.b * 12;
  c.rx = ua[0] * c.px + ua[1] * c.py + ua[2] * c.pz + ua[3];
  c.ry = ua[4] * c.px + ua[5] * c.py + ua[6] * c.pz + ua[7];
  return c;
}

// Whether camera `cam` sees the cell (warp-uniform; every lane of the warp must call it), and the ray-map position
// (gx, gy) of the mean pixel x and mean clamped radius over the Z height samples.
__device__ __forceinline__ bool polar_cell_loc(const float* __restrict__ proj, const float* __restrict__ camc,
                                               const PolarParams& p, const PolarCell& c, int cam, int lane, float& gx,
                                               float& gy) {
  const float px = c.px, py = c.py, pz = c.pz;
  const float* m = proj + (c.b * p.V + cam) * 12;
  const float cx = m[0] * px + m[1] * py + m[2] * pz + m[3], cy = m[4] * px + m[5] * py + m[6] * pz + m[7],
              cz = m[8] * px + m[9] * py + m[10] * pz + m[11];
  const float eps = 1e-5f;
  const float zz = fmaxf(cz, eps);
  const float nx = 2.f * (cx / zz / p.W_in) - 1.f, ny = 2.f * (cy / zz / p.H_in) - 1.f;
  bool ok = lane < p.Z && cz > eps && nx > -1.f && nx < 1.f && ny > -1.f && ny < 1.f;
  const float ddx = c.rx - camc[(c.b * p.V + cam) * 2], ddy = c.ry - camc[(c.b * p.V + cam) * 2 + 1];
  float nr = 2.f * (sqrtf(ddx * ddx + ddy * ddy) - p.r0) / p.r_cnt - 1.f;
  nr = fminf(fmaxf(nr, -1.f), 1.f);
  float sx = lane < p.Z ? nx : 0.f, sr = lane < p.Z ? nr : 0.f;
  sx = warp_sum(sx) / (float)p.Z;
  sr = warp_sum(sr) / (float)p.Z;
  gx = (sx + 1.f) * 0.5f * (float)p.W - 0.5f;
  gy = (sr + 1.f) * 0.5f * (float)p.R - 0.5f;
  return __any_sync(0xffffffffu, ok);
}

__device__ __forceinline__ bool polar_loc_near(const PolarParams& p, float gx, float gy) {
  return gx > -2.f && gx < (float)p.W + 1.f && gy > -2.f && gy < (float)p.R + 1.f;
}

__global__ void __launch_bounds__(256)
polar_gather_kernel(const float* __restrict__ rays, const float* __restrict__ lidar, const float* __restrict__ proj,
                    const float* __restrict__ undo, const float* __restrict__ camc, float* __restrict__ out, PolarParams p) {
  const int cell = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (cell >= p.B * p.Y * p.X) return;
  const PolarCell c = polar_cell(undo, p, cell, lane);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  float vis = 0.f;
  for (int cam = 0; cam < p.V; ++cam) {
    float gx, gy;
    if (!polar_cell_loc(proj, camc, p, c, cam, lane, gx, gy)) continue;
    vis += 1.f;
    if (!polar_loc_near(p, gx, gy)) continue;
    const float fx = floorf(gx), fy = floorf(gy);
    const int x0 = (int)fx, y0 = (int)fy;
    const float wx1 = gx - fx, wx0 = 1.f - wx1, wy1 = gy - fy, wy0 = 1.f - wy1;
    const float* base = rays + (size_t)(c.b * p.V + cam) * p.R * p.W * 128 + lane * 4;
#pragma unroll
    for (int cnr = 0; cnr < 4; ++cnr) {
      const int xx = x0 + (cnr & 1), yy = y0 + (cnr >> 1);
      if (xx < 0 || xx >= p.W || yy < 0 || yy >= p.R) continue;
      const float wgt = ((cnr & 1) ? wx1 : wx0) * ((cnr >> 1) ? wy1 : wy0);
      const float4 t = ldg4(base + ((size_t)yy * p.W + xx) * 128);
      acc.x += wgt * t.x; acc.y += wgt * t.y; acc.z += wgt * t.z; acc.w += wgt * t.w;
    }
  }
  const float inv = 1.f / (vis > 0.f ? vis : 1.f);
  const float4 res = ldg4(lidar + (size_t)cell * 128 + lane * 4);
  *reinterpret_cast<float4*>(out + (size_t)cell * 128 + lane * 4) =
      make_float4(acc.x * inv + res.x, acc.y * inv + res.y, acc.z * inv + res.z, acc.w * inv + res.w);
}

// Adjoint of polar_gather_kernel with respect to the rays: d_rays[bv, yy, xx, :] += (w_corner / count) d_out[cell, :]
// over the cameras that see the cell and the in-map corners of its sample.  One warp per cell: a first pass counts the
// seeing cameras, a second scatters with one 16-byte vector reduction per lane and corner (d_rays zeroed by the caller).
__global__ void __launch_bounds__(256)
polar_gather_bwd_kernel(const float* __restrict__ d_out, const float* __restrict__ proj, const float* __restrict__ undo,
                        const float* __restrict__ camc, float* __restrict__ d_rays, PolarParams p) {
  const int cell = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (cell >= p.B * p.Y * p.X) return;
  const PolarCell c = polar_cell(undo, p, cell, lane);
  float vis = 0.f;
  for (int cam = 0; cam < p.V; ++cam) {
    float gx, gy;
    if (polar_cell_loc(proj, camc, p, c, cam, lane, gx, gy)) vis += 1.f;
  }
  if (vis == 0.f) return;
  const float inv = 1.f / vis;
  const float4 g = ldg4(d_out + (size_t)cell * 128 + lane * 4);
  for (int cam = 0; cam < p.V; ++cam) {
    float gx, gy;
    if (!polar_cell_loc(proj, camc, p, c, cam, lane, gx, gy) || !polar_loc_near(p, gx, gy)) continue;
    const float fx = floorf(gx), fy = floorf(gy);
    const int x0 = (int)fx, y0 = (int)fy;
    const float wx1 = gx - fx, wx0 = 1.f - wx1, wy1 = gy - fy, wy0 = 1.f - wy1;
    float* base = d_rays + (size_t)(c.b * p.V + cam) * p.R * p.W * 128 + lane * 4;
#pragma unroll
    for (int cnr = 0; cnr < 4; ++cnr) {
      const int xx = x0 + (cnr & 1), yy = y0 + (cnr >> 1);
      if (xx < 0 || xx >= p.W || yy < 0 || yy >= p.R) continue;
      const float wgt = ((cnr & 1) ? wx1 : wx0) * ((cnr >> 1) ? wy1 : wy0) * inv;
      atomicAdd(reinterpret_cast<float4*>(base + ((size_t)yy * p.W + xx) * 128),
                make_float4(wgt * g.x, wgt * g.y, wgt * g.z, wgt * g.w));
    }
  }
}

// Gradient of msdeform_kernel (same warp layout: lane = (head, 4-channel group)).  For sample i = (l, p) of a head with
// softmax weight a_i and bilinear sample s_i:  d logit_i = a_i (dw_i - sum_j a_j dw_j), dw_i = dout . s_i;
// d offset_x = a_i dout . ds_i/dx (the pixel coordinate x = (ref + off / W) W - 0.5 moves one-for-one with the offset),
// from the in-map corners only (grid_sample's zero padding); d value += a_i w_corner dout at every in-map corner (16-byte
// vector reductions; d_value zeroed by the caller).  The four lanes of a head reduce their partial dot products in a
// fixed order and its first lane writes the head's row of d_raw, so d_raw is the same bit for bit on every call.
template <int L, int P>
__global__ void __launch_bounds__(256)
msdeform_bwd_kernel(const float* __restrict__ value0, const float* __restrict__ value1, const float* __restrict__ raw,
                    int ld_raw, const float* __restrict__ dout, int ldo, float* __restrict__ d_raw, int ld_draw,
                    float* __restrict__ dvalue0, float* __restrict__ dvalue1, long long total_q, int NQ, int Wq,
                    float inv_wq, float inv_hq, DeformLevels lv) {
  const long long q = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (q >= total_q) return;
  const int lane = threadIdx.x & 31;
  const int head = lane >> 2, sub = lane & 3;
  const int b = (int)(q / NQ), qi = (int)(q - (long long)b * NQ);
  const float refx = ((float)(qi % Wq) + 0.5f) * inv_wq, refy = ((float)(qi / Wq) + 0.5f) * inv_hq;
  const float* r = raw + q * ld_raw;
  constexpr int LP = L * P;
  const float* off = r + head * LP * 2;
  const float* lg = r + 8 * LP * 2 + head * LP;
  float w[LP];
  float m = -INFINITY;
#pragma unroll
  for (int i = 0; i < LP; ++i) {
    w[i] = __ldg(lg + i);
    m = fmaxf(m, w[i]);
  }
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < LP; ++i) {
    w[i] = expf(w[i] - m);
    s += w[i];
  }
  const float inv = 1.f / s;
  const float4 go = ldg4(dout + q * ldo + head * 16 + sub * 4);
  auto dot4 = [](float4 a, float4 c) { return a.x * c.x + a.y * c.y + a.z * c.z + a.w * c.w; };
  float dw[LP], gx[LP], gy[LP];
#pragma unroll
  for (int l = 0; l < L; ++l) {
    const int H = lv.H[l], W = lv.W[l];
    const size_t lane_off = (size_t)b * H * W * 128 + head * 16 + sub * 4;
    const float* vl = (l == 0 ? value0 : value1) + lane_off;
    float* dl = (l == 0 ? dvalue0 : dvalue1) + lane_off;
#pragma unroll
    for (int p = 0; p < P; ++p) {
      const int i = l * P + p;
      const float ox = __ldg(off + i * 2), oy = __ldg(off + i * 2 + 1);
      const float x = (refx + ox / (float)W) * (float)W - 0.5f, y = (refy + oy / (float)H) * (float)H - 0.5f;
      const float x0f = floorf(x), y0f = floorf(y);
      const int x0 = (int)x0f, y0 = (int)y0f;
      const float fx = x - x0f, fy = y - y0f;
      const bool xa = x0 >= 0 && x0 < W, xb = x0 + 1 >= 0 && x0 + 1 < W, ya = y0 >= 0 && y0 < H, yb = y0 + 1 >= 0 && y0 + 1 < H;
      const size_t r00 = ((size_t)y0 * W + x0) * 128;
      const float d00 = (ya && xa) ? dot4(go, ldg4(vl + r00)) : 0.f;
      const float d01 = (ya && xb) ? dot4(go, ldg4(vl + r00 + 128)) : 0.f;
      const float d10 = (yb && xa) ? dot4(go, ldg4(vl + r00 + (size_t)W * 128)) : 0.f;
      const float d11 = (yb && xb) ? dot4(go, ldg4(vl + r00 + (size_t)W * 128 + 128)) : 0.f;
      dw[i] = (1.f - fx) * (1.f - fy) * d00 + fx * (1.f - fy) * d01 + (1.f - fx) * fy * d10 + fx * fy * d11;
      gx[i] = (1.f - fy) * (d01 - d00) + fy * (d11 - d10);
      gy[i] = (1.f - fx) * (d10 - d00) + fx * (d11 - d01);
      const float a = w[i] * inv;
      const float c00 = (1.f - fx) * (1.f - fy) * a, c01 = fx * (1.f - fy) * a, c10 = (1.f - fx) * fy * a, c11 = fx * fy * a;
      auto scale4 = [&](float c) { return make_float4(c * go.x, c * go.y, c * go.z, c * go.w); };
      if (ya && xa) atomicAdd(reinterpret_cast<float4*>(dl + r00), scale4(c00));
      if (ya && xb) atomicAdd(reinterpret_cast<float4*>(dl + r00 + 128), scale4(c01));
      if (yb && xa) atomicAdd(reinterpret_cast<float4*>(dl + r00 + (size_t)W * 128), scale4(c10));
      if (yb && xb) atomicAdd(reinterpret_cast<float4*>(dl + r00 + (size_t)W * 128 + 128), scale4(c11));
    }
  }
#pragma unroll
  for (int i = 0; i < LP; ++i) {
#pragma unroll
    for (int o = 1; o < 4; o <<= 1) {
      dw[i] += __shfl_xor_sync(0xffffffffu, dw[i], o);
      gx[i] += __shfl_xor_sync(0xffffffffu, gx[i], o);
      gy[i] += __shfl_xor_sync(0xffffffffu, gy[i], o);
    }
  }
  if (sub != 0) return;
  float sdw = 0.f;
#pragma unroll
  for (int i = 0; i < LP; ++i) sdw += w[i] * inv * dw[i];
  float* dr = d_raw + q * ld_draw;
#pragma unroll
  for (int i = 0; i < LP; ++i) {
    const float a = w[i] * inv;
    dr[head * LP * 2 + i * 2] = a * gx[i];
    dr[head * LP * 2 + i * 2 + 1] = a * gy[i];
    dr[8 * LP * 2 + head * LP + i] = a * (dw[i] - sdw);
  }
}

// Gradient of seq_attn_kernel, one warp per (sequence, head) as the forward.  Pass A, lane = query token t: the row
// statistics (m_t, l_t) by the forward's own online loop over the keys, D_t = dout_t . out_t from the saved output, and
// dq_t = scale sum_j P_tj (dout_t . v_j - D_t) k_j.  Pass B, lane = key token j: dk_j = sum_t dS_tj scale q_t and
// dv_j = sum_t P_tj dout_t, the queries summed in order t = 0 .. Lq-1 (no atomics: the same bits on every call).  The
// per-query statistics pass between the two through shared memory (Lq <= SEQ_BWD_MAX_LQ).
constexpr int SEQ_BWD_MAX_LQ = 128;

__global__ void __launch_bounds__(256)
seq_attn_bwd_kernel(const float* __restrict__ q, int ldq, const float* __restrict__ k, int ldk, const float* __restrict__ v,
                    int ldv, const float* __restrict__ out, int ldo, const float* __restrict__ dout, int ldd,
                    float* __restrict__ dq, int lddq, float* __restrict__ dk, int lddk, float* __restrict__ dv, int lddv,
                    int G, int Wn, int Lq, int Lk, int heads, float scale) {
  __shared__ float s_m[8][SEQ_BWD_MAX_LQ], s_il[8][SEQ_BWD_MAX_LQ], s_D[8][SEQ_BWD_MAX_LQ];
  const int wid = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31, wl = threadIdx.x >> 5;
  if (wid >= G * Wn * heads) return;
  const int head = wid % heads, seq = wid / heads;
  const int w = seq % Wn, g = seq / Wn;
  auto qrow = [&](int t) { return (size_t)(g * Lq + t) * Wn + w; };
  auto krow = [&](int j) { return (size_t)(g * Lk + j) * Wn + w; };
  for (int t0 = 0; t0 < Lq; t0 += 32) {
    const int t = t0 + lane;
    const bool on = t < Lq;
    float qv[16], go[16], acc[16];
    const size_t rq = qrow(on ? t : 0);
    const float* qp = q + rq * ldq + head * 16;
    float D = 0.f;
#pragma unroll
    for (int c = 0; c < 16; c += 4) {
      const float4 x = ldg4(qp + c);
      qv[c] = x.x * scale; qv[c + 1] = x.y * scale; qv[c + 2] = x.z * scale; qv[c + 3] = x.w * scale;
      const float4 d = ldg4(dout + rq * ldd + head * 16 + c), o = ldg4(out + rq * ldo + head * 16 + c);
      go[c] = d.x; go[c + 1] = d.y; go[c + 2] = d.z; go[c + 3] = d.w;
      D += d.x * o.x + d.y * o.y + d.z * o.z + d.w * o.w;
      acc[c] = acc[c + 1] = acc[c + 2] = acc[c + 3] = 0.f;
    }
    float m = -INFINITY, l = 0.f;
    for (int j = 0; j < Lk; ++j) {
      const float* kp = k + krow(j) * ldk + head * 16;
      float s = 0.f;
#pragma unroll
      for (int c = 0; c < 16; c += 4) {
        const float4 x = ldg4(kp + c);
        s += qv[c] * x.x + qv[c + 1] * x.y + qv[c + 2] * x.z + qv[c + 3] * x.w;
      }
      const float mn = fmaxf(m, s);
      const float corr = expf(m - mn), pw = expf(s - mn);
      l = l * corr + pw;
      m = mn;
    }
    const float il = 1.f / l;
    for (int j = 0; j < Lk; ++j) {
      const size_t row = krow(j);
      const float* kp = k + row * ldk + head * 16;
      const float* vp = v + row * ldv + head * 16;
      float s = 0.f, dp = 0.f;
#pragma unroll
      for (int c = 0; c < 16; c += 4) {
        const float4 x = ldg4(kp + c), y = ldg4(vp + c);
        s += qv[c] * x.x + qv[c + 1] * x.y + qv[c + 2] * x.z + qv[c + 3] * x.w;
        dp += go[c] * y.x + go[c + 1] * y.y + go[c + 2] * y.z + go[c + 3] * y.w;
      }
      const float ds = expf(s - m) * il * (dp - D);
#pragma unroll
      for (int c = 0; c < 16; c += 4) {
        const float4 x = ldg4(kp + c);
        acc[c] += ds * x.x; acc[c + 1] += ds * x.y; acc[c + 2] += ds * x.z; acc[c + 3] += ds * x.w;
      }
    }
    if (on) {
      float* op = dq + (size_t)qrow(t) * lddq + head * 16;
#pragma unroll
      for (int c = 0; c < 16; c += 4)
        *reinterpret_cast<float4*>(op + c) = make_float4(acc[c] * scale, acc[c + 1] * scale, acc[c + 2] * scale, acc[c + 3] * scale);
      s_m[wl][t] = m;
      s_il[wl][t] = il;
      s_D[wl][t] = D;
    }
  }
  __syncwarp();
  for (int j0 = 0; j0 < Lk; j0 += 32) {
    const int j = j0 + lane;
    const bool on = j < Lk;
    const size_t row = krow(on ? j : 0);
    float kv[16], vv[16], ak[16], av[16];
#pragma unroll
    for (int c = 0; c < 16; c += 4) {
      const float4 x = ldg4(k + row * ldk + head * 16 + c), y = ldg4(v + row * ldv + head * 16 + c);
      kv[c] = x.x; kv[c + 1] = x.y; kv[c + 2] = x.z; kv[c + 3] = x.w;
      vv[c] = y.x; vv[c + 1] = y.y; vv[c + 2] = y.z; vv[c + 3] = y.w;
      ak[c] = ak[c + 1] = ak[c + 2] = ak[c + 3] = 0.f;
      av[c] = av[c + 1] = av[c + 2] = av[c + 3] = 0.f;
    }
    for (int t = 0; t < Lq; ++t) {
      const size_t rq = qrow(t);
      const float* qp = q + rq * ldq + head * 16;
      const float* dp_ = dout + rq * ldd + head * 16;
      float qs[16], gd[16];
      float s = 0.f, dp = 0.f;
#pragma unroll
      for (int c = 0; c < 16; c += 4) {
        const float4 x = ldg4(qp + c), y = ldg4(dp_ + c);
        qs[c] = x.x * scale; qs[c + 1] = x.y * scale; qs[c + 2] = x.z * scale; qs[c + 3] = x.w * scale;
        gd[c] = y.x; gd[c + 1] = y.y; gd[c + 2] = y.z; gd[c + 3] = y.w;
        s += qs[c] * kv[c] + qs[c + 1] * kv[c + 1] + qs[c + 2] * kv[c + 2] + qs[c + 3] * kv[c + 3];
        dp += gd[c] * vv[c] + gd[c + 1] * vv[c + 1] + gd[c + 2] * vv[c + 2] + gd[c + 3] * vv[c + 3];
      }
      const float pr = expf(s - s_m[wl][t]) * s_il[wl][t];
      const float ds = pr * (dp - s_D[wl][t]);
#pragma unroll
      for (int c = 0; c < 16; ++c) {
        ak[c] += ds * qs[c];
        av[c] += pr * gd[c];
      }
    }
    if (on) {
      float* kp = dk + row * lddk + head * 16;
      float* vp = dv + row * lddv + head * 16;
#pragma unroll
      for (int c = 0; c < 16; c += 4) {
        *reinterpret_cast<float4*>(kp + c) = make_float4(ak[c], ak[c + 1], ak[c + 2], ak[c + 3]);
        *reinterpret_cast<float4*>(vp + c) = make_float4(av[c], av[c + 1], av[c + 2], av[c + 3]);
      }
    }
  }
}

// Gradient of axpy_kernel: db = s dout, and per block the partial sum of dout . b in double (a fixed grid-stride
// assignment and a fixed reduction tree); axpy_bwd_sum_kernel adds the partials in order into d s.
constexpr int AXPY_BWD_BLOCKS = 512;

__device__ __forceinline__ double block_sum_double(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int wl = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) red[wl] = v;
  __syncthreads();
  double t = 0.0;
  if (threadIdx.x == 0)
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += red[i];
  return t;
}

__global__ void __launch_bounds__(256)
axpy_bwd_kernel(const float4* __restrict__ dout, const float4* __restrict__ b, const float* __restrict__ s,
                float4* __restrict__ db, double* __restrict__ part, long long n4) {
  __shared__ double red[8];
  const float sc = __ldg(s);
  double acc = 0.0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 g = dout[i], y = b[i];
    db[i] = make_float4(sc * g.x, sc * g.y, sc * g.z, sc * g.w);
    acc += (double)g.x * y.x + (double)g.y * y.y + (double)g.z * y.z + (double)g.w * y.w;
  }
  const double t = block_sum_double(acc, red);
  if (threadIdx.x == 0) part[blockIdx.x] = t;
}

__global__ void __launch_bounds__(256) axpy_bwd_sum_kernel(const double* __restrict__ part, int n, float* __restrict__ ds) {
  __shared__ double red[8];
  double acc = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) acc += part[i];
  const double t = block_sum_double(acc, red);
  if (threadIdx.x == 0) *ds = (float)t;
}

}  // namespace

extern "C" {

// grid [BV, R, W, 2] (BEV pixel coordinates for di_bev_sample_f32) of the polar ray queries; cam [BV, 26] (see kernel).
int di_polar_grid_f32(const float* cam, float* grid, int BV, int R, int W, int h_feat, float im_scale, float r0,
                      float r_step, const float* pc_range, int Yb, int Xb, cudaStream_t stream) {
  DI_CHECK_ARG(cam && grid && pc_range && BV > 0 && R > 0 && W > 0, "di_polar_grid_f32: bad argument");
  const int n = BV * R * W;
  polar_grid_kernel<<<di_cdiv(n, 256), 256, 0, stream>>>(cam, reinterpret_cast<float2*>(grid), BV, R, W, im_scale,
                                                        (float)(h_feat / 2) * im_scale, r0, r_step, pc_range[0],
                                                        pc_range[3] - pc_range[0], pc_range[1], pc_range[4] - pc_range[1], Xb, Yb);
  DI_CHECK_LAUNCH("di_polar_grid_f32");
  return DI_OK;
}

// out[m,:] = x[m,:] + pos[m % mod,:]; x, out [M, C] contiguous, pos [mod, C]; C % 4 == 0
int di_add_rows_mod_f32(const float* x, const float* pos, float* out, long long M, int C, long long mod, cudaStream_t stream) {
  DI_CHECK_ARG(x && pos && out && M > 0 && C > 0 && C % 4 == 0 && mod > 0, "di_add_rows_mod_f32: bad argument");
  const long long n4 = M * C / 4;
  add_rows_mod_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const float4*>(x),
                                                                        reinterpret_cast<const float4*>(pos),
                                                                        reinterpret_cast<float4*>(out), n4, mod * C / 4);
  DI_CHECK_LAUNCH("di_add_rows_mod_f32");
  return DI_OK;
}

// softmax(q k^T / sqrt(16)) v per head over column sequences (token t of sequence (g, w) = row (g*L + t)*Wn + w);
// q [G*Lq*Wn, ldq], k / v [G*Lk*Wn, ld*], out [G*Lq*Wn, ldo]; heads x 16 channels.  Replaces the two
// FlashMultiheadAttention cores of the polar decoder layer (fusion_transformerv4.py:651-759), evaluated in fp32.
int di_seq_attn_f32(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, float* out, int ldo, int G,
                    int Wn, int Lq, int Lk, int heads, int dim, cudaStream_t stream) {
  DI_CHECK_ARG(q && k && v && out && G > 0 && Wn > 0 && Lq > 0 && Lk > 0 && heads > 0, "di_seq_attn_f32: bad argument");
  if (dim != 16) {
    di_set_error("di_seq_attn_f32: head dimension must be 16 (got %d)", dim);
    return DI_ERR_UNSUPPORTED;
  }
  DI_CHECK_ARG(ldq % 4 == 0 && ldk % 4 == 0 && ldv % 4 == 0 && ldo % 4 == 0 &&
                   ((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)out) % 16 == 0,
               "di_seq_attn_f32: strides / alignment");
  const long long warps = (long long)G * Wn * heads;
  seq_attn_kernel<<<(unsigned)((warps + 7) / 8), 256, 0, stream>>>(q, ldq, k, ldk, v, ldv, out, ldo, G, Wn, Lq, Lk, heads, 0.25f);
  DI_CHECK_LAUNCH("di_seq_attn_f32");
  return DI_OK;
}

// rays [B*V, R, W, 128] decoded polar rays; lidar / out [B, Y, X, 128]; proj [B,V,12]; undo [B,12]; camc [B*V,2];
// geom (host): H_in, W_in, pc_range[6], r0, r_count.  Z = 10 height samples per cell (fusion_transformerv4.py:587).
int di_polar_gather_f32(const float* rays, const float* lidar, const float* proj, const float* undo, const float* camc,
                        float* out, int B, int V, int R, int W, int Y, int X, int C, int H_in, int W_in,
                        const float* pc_range, float r0, float r_count, cudaStream_t stream) {
  DI_CHECK_ARG(rays && lidar && proj && undo && camc && out && pc_range && B > 0 && V > 0, "di_polar_gather_f32: bad argument");
  if (C != 128) {
    di_set_error("di_polar_gather_f32: C must be 128 (got %d)", C);
    return DI_ERR_UNSUPPORTED;
  }
  PolarParams p;
  p.B = B; p.V = V; p.R = R; p.W = W; p.Y = Y; p.X = X; p.Z = 10;
  p.H_in = (float)H_in; p.W_in = (float)W_in;
  p.x_min = pc_range[0]; p.x_rng = pc_range[3] - pc_range[0];
  p.y_min = pc_range[1]; p.y_rng = pc_range[4] - pc_range[1];
  p.z_min = pc_range[2]; p.z_rng = pc_range[5] - pc_range[2];
  p.r0 = r0; p.r_cnt = r_count;
  polar_gather_kernel<<<di_cdiv((long long)B * Y * X, 8), 256, 0, stream>>>(rays, lidar, proj, undo, camc, out, p);
  DI_CHECK_LAUNCH("di_polar_gather_f32");
  return DI_OK;
}

// value0 / value1 [B, H_l, W_l, 128]: pixel-major projected value maps of level 0 / 1 (value1 may be NULL when L == 1),
// shapes[2l], shapes[2l+1] = H_l, W_l; raw [B*NQ, ld_raw]: per query 8*L*P*2 sampling offsets then 8*L*P logits;
// out [B*NQ, ldo] (128 channels written).  8 heads x 16 channels, P = 4 points, L = 1 or 2 levels.
int di_msdeform_f32(const float* value0, const float* value1, const float* raw, int ld_raw, float* out, int ldo, int B,
                    int NQ, int Hq, int Wq, int heads, int dim, int L, int P, const int* shapes, cudaStream_t stream) {
  const float* value = value0;
  DI_CHECK_ARG(value0 && raw && out && shapes && B > 0 && NQ > 0 && Hq * Wq == NQ && (L == 1 || value1),
               "di_msdeform_f32: bad argument");
  if (!(heads == 8 && dim == 16 && P == 4 && (L == 1 || L == 2))) {
    di_set_error("di_msdeform_f32: supported configuration is 8 heads x 16 channels, 4 points, 1 or 2 levels");
    return DI_ERR_UNSUPPORTED;
  }
  DI_CHECK_ARG(ld_raw >= heads * L * P * 3 && ldo >= 128 && ldo % 4 == 0 && ((uintptr_t)value | (uintptr_t)out) % 16 == 0,
               "di_msdeform_f32: strides / alignment");
  DeformLevels lv{};
  for (int l = 0; l < L; ++l) {
    lv.H[l] = shapes[2 * l];
    lv.W[l] = shapes[2 * l + 1];
  }
  const long long total = (long long)B * NQ;
  const unsigned grid = (unsigned)((total + 7) / 8);
  if (L == 1)
    msdeform_kernel<1, 4><<<grid, 256, 0, stream>>>(value0, value1, raw, ld_raw, out, ldo, total, NQ, Wq, 1.f / Wq, 1.f / Hq, lv);
  else
    msdeform_kernel<2, 4><<<grid, 256, 0, stream>>>(value0, value1, raw, ld_raw, out, ldo, total, NQ, Wq, 1.f / Wq, 1.f / Hq, lv);
  DI_CHECK_LAUNCH("di_msdeform_f32");
  return DI_OK;
}

// out[i] = a[i] + scale[0] * b[i], n % 4 == 0; scale is a DEVICE pointer (a learned parameter: no host sync)
int di_axpy_f32(const float* a, const float* b, const float* scale, float* out, long long n, cudaStream_t stream) {
  DI_CHECK_ARG(a && b && scale && out && n > 0 && n % 4 == 0, "di_axpy_f32: bad argument");
  DI_CHECK_ARG(((uintptr_t)a | (uintptr_t)b | (uintptr_t)out) % 16 == 0, "di_axpy_f32: pointers must be 16-byte aligned");
  const long long n4 = n / 4;
  axpy_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const float4*>(a),
                                                                 reinterpret_cast<const float4*>(b), scale,
                                                                 reinterpret_cast<float4*>(out), n4);
  DI_CHECK_LAUNCH("di_axpy_f32");
  return DI_OK;
}

// Gradient of di_msdeform_f32 (same value maps, raw and configuration): dout [B*NQ, ldo] ->
// d_raw [B*NQ, ld_draw] in raw's layout (8*L*P*2 offset gradients then 8*L*P logit gradients; other columns untouched;
// written without atomics), d_value0 / d_value1 [B, H_l, W_l, 128] += the value-map gradients (zero them first).
int di_msdeform_bwd_f32(const float* value0, const float* value1, const float* raw, int ld_raw, const float* dout, int ldo,
                        float* d_raw, int ld_draw, float* d_value0, float* d_value1, int B, int NQ, int Hq, int Wq,
                        int heads, int dim, int L, int P, const int* shapes, cudaStream_t stream) {
  DI_CHECK_ARG(value0 && raw && dout && d_raw && d_value0 && shapes && B > 0 && NQ > 0 && Hq * Wq == NQ &&
                   (L == 1 || (value1 && d_value1)),
               "di_msdeform_bwd_f32: bad argument");
  if (!(heads == 8 && dim == 16 && P == 4 && (L == 1 || L == 2))) {
    di_set_error("di_msdeform_bwd_f32: supported configuration is 8 heads x 16 channels, 4 points, 1 or 2 levels");
    return DI_ERR_UNSUPPORTED;
  }
  DI_CHECK_ARG(ld_raw >= heads * L * P * 3 && ld_draw >= heads * L * P * 3 && ldo >= 128 && ldo % 4 == 0 &&
                   ((uintptr_t)value0 | (uintptr_t)dout | (uintptr_t)d_value0 | (uintptr_t)(L == 2 ? value1 : value0) |
                    (uintptr_t)(L == 2 ? d_value1 : d_value0)) % 16 == 0,
               "di_msdeform_bwd_f32: strides / alignment");
  DeformLevels lv{};
  for (int l = 0; l < L; ++l) {
    lv.H[l] = shapes[2 * l];
    lv.W[l] = shapes[2 * l + 1];
  }
  const long long total = (long long)B * NQ;
  const unsigned grid = (unsigned)((total + 7) / 8);
  if (L == 1)
    msdeform_bwd_kernel<1, 4><<<grid, 256, 0, stream>>>(value0, value1, raw, ld_raw, dout, ldo, d_raw, ld_draw, d_value0,
                                                        d_value1, total, NQ, Wq, 1.f / Wq, 1.f / Hq, lv);
  else
    msdeform_bwd_kernel<2, 4><<<grid, 256, 0, stream>>>(value0, value1, raw, ld_raw, dout, ldo, d_raw, ld_draw, d_value0,
                                                        d_value1, total, NQ, Wq, 1.f / Wq, 1.f / Hq, lv);
  DI_CHECK_LAUNCH("di_msdeform_bwd_f32");
  return DI_OK;
}

// Gradient of di_seq_attn_f32: q / k / v / out as the forward (out = its saved output), dout [G*Lq*Wn, ldd] ->
// dq [G*Lq*Wn, lddq], dk / dv [G*Lk*Wn, ld*] (row views; written, not accumulated).  Lq <= 128, any Lk.
int di_seq_attn_bwd_f32(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, const float* out, int ldo,
                        const float* dout, int ldd, float* dq, int lddq, float* dk, int lddk, float* dv, int lddv, int G,
                        int Wn, int Lq, int Lk, int heads, int dim, cudaStream_t stream) {
  DI_CHECK_ARG(q && k && v && out && dout && dq && dk && dv && G > 0 && Wn > 0 && Lq > 0 && Lk > 0 && heads > 0,
               "di_seq_attn_bwd_f32: bad argument");
  if (dim != 16 || Lq > SEQ_BWD_MAX_LQ) {
    di_set_error("di_seq_attn_bwd_f32: head dimension 16 and at most %d queries per sequence (got %d, %d)", SEQ_BWD_MAX_LQ,
                 dim, Lq);
    return DI_ERR_UNSUPPORTED;
  }
  DI_CHECK_ARG(ldq % 4 == 0 && ldk % 4 == 0 && ldv % 4 == 0 && ldo % 4 == 0 && ldd % 4 == 0 && lddq % 4 == 0 &&
                   lddk % 4 == 0 && lddv % 4 == 0 &&
                   ((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)out | (uintptr_t)dout | (uintptr_t)dq |
                    (uintptr_t)dk | (uintptr_t)dv) % 16 == 0,
               "di_seq_attn_bwd_f32: strides / alignment");
  const long long warps = (long long)G * Wn * heads;
  seq_attn_bwd_kernel<<<(unsigned)((warps + 7) / 8), 256, 0, stream>>>(q, ldq, k, ldk, v, ldv, out, ldo, dout, ldd, dq, lddq,
                                                                      dk, lddk, dv, lddv, G, Wn, Lq, Lk, heads, 0.25f);
  DI_CHECK_LAUNCH("di_seq_attn_bwd_f32");
  return DI_OK;
}

// Adjoint of di_polar_gather_f32 with respect to the rays: d_rays [B*V, R, W, 128] += gather^T(d_out [B, Y, X, 128])
// (zero d_rays first); the residual's gradient is d_out itself.  Other arguments as the forward.
int di_polar_gather_bwd_f32(const float* d_out, const float* proj, const float* undo, const float* camc, float* d_rays, int B,
                            int V, int R, int W, int Y, int X, int C, int H_in, int W_in, const float* pc_range, float r0,
                            float r_count, cudaStream_t stream) {
  DI_CHECK_ARG(d_out && proj && undo && camc && d_rays && pc_range && B > 0 && V > 0, "di_polar_gather_bwd_f32: bad argument");
  if (C != 128) {
    di_set_error("di_polar_gather_bwd_f32: C must be 128 (got %d)", C);
    return DI_ERR_UNSUPPORTED;
  }
  PolarParams p;
  p.B = B; p.V = V; p.R = R; p.W = W; p.Y = Y; p.X = X; p.Z = 10;
  p.H_in = (float)H_in; p.W_in = (float)W_in;
  p.x_min = pc_range[0]; p.x_rng = pc_range[3] - pc_range[0];
  p.y_min = pc_range[1]; p.y_rng = pc_range[4] - pc_range[1];
  p.z_min = pc_range[2]; p.z_rng = pc_range[5] - pc_range[2];
  p.r0 = r0; p.r_cnt = r_count;
  polar_gather_bwd_kernel<<<di_cdiv((long long)B * Y * X, 8), 256, 0, stream>>>(d_out, proj, undo, camc, d_rays, p);
  DI_CHECK_LAUNCH("di_polar_gather_bwd_f32");
  return DI_OK;
}

// Gradient of di_axpy_f32 (out = a + s b) with respect to b and s: db = s dout, ds[0] = sum dout . b (device scalar);
// work: >= di_axpy_bwd_workspace() doubles.  Two launches, no host synchronisation, the same bits on every call.
int di_axpy_bwd_workspace(void) { return AXPY_BWD_BLOCKS; }

int di_axpy_bwd_f32(const float* dout, const float* b, const float* scale, float* db, float* ds, double* work, long long n,
                    cudaStream_t stream) {
  DI_CHECK_ARG(dout && b && scale && db && ds && work && n > 0 && n % 4 == 0, "di_axpy_bwd_f32: bad argument");
  DI_CHECK_ARG(((uintptr_t)dout | (uintptr_t)b | (uintptr_t)db) % 16 == 0, "di_axpy_bwd_f32: pointers must be 16-byte aligned");
  const long long n4 = n / 4;
  const int blocks = (int)std::min<long long>((n4 + 255) / 256, AXPY_BWD_BLOCKS);
  axpy_bwd_kernel<<<blocks, 256, 0, stream>>>(reinterpret_cast<const float4*>(dout), reinterpret_cast<const float4*>(b), scale,
                                              reinterpret_cast<float4*>(db), work, n4);
  axpy_bwd_sum_kernel<<<1, 256, 0, stream>>>(work, blocks, ds);
  DI_CHECK_LAUNCH("di_axpy_bwd_f32");
  return DI_OK;
}

// map[coors[p]] += rows[p, :] where cnt[p] > 0 (n_dev as in di_scatter_rows_f32)
int di_scatter_rows_add_f32(const float* rows, const int* cnt, const int* coors, float* map, int P, int Y, int X, int C,
                            const int* n_dev, cudaStream_t stream) {
  DI_CHECK_ARG(P >= 0 && C % 4 == 0, "di_scatter_rows_add_f32: bad argument");
  if (P == 0) return DI_OK;                     // empty tensors may have null data pointers
  DI_CHECK_ARG(map && coors && rows && cnt, "di_scatter_rows_add_f32: null pointer");
  scatter_rows_add_kernel<<<di_cdiv(P, 8), 256, 0, stream>>>(rows, cnt, coors, map, P, Y, X, C, n_dev);
  DI_CHECK_LAUNCH("di_scatter_rows_add_f32");
  return DI_OK;
}

}  // extern "C"
