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
__global__ void __launch_bounds__(256)
polar_gather_kernel(const float* __restrict__ rays, const float* __restrict__ lidar, const float* __restrict__ proj,
                    const float* __restrict__ undo, const float* __restrict__ camc, float* __restrict__ out, PolarParams p) {
  const int cell = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (cell >= p.B * p.Y * p.X) return;
  const int ix = cell % p.X, iy = (cell / p.X) % p.Y, b = cell / (p.X * p.Y);
  const float px = ((float)ix + 0.5f) / (float)p.X * p.x_rng + p.x_min, py = ((float)iy + 0.5f) / (float)p.Y * p.y_rng + p.y_min;
  const float pz = ((float)(lane < p.Z ? lane : 0) + 0.5f) / (float)p.Z * p.z_rng + p.z_min;
  const float* ua = undo + b * 12;
  const float rx = ua[0] * px + ua[1] * py + ua[2] * pz + ua[3], ry = ua[4] * px + ua[5] * py + ua[6] * pz + ua[7];
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  float vis = 0.f;
  for (int cam = 0; cam < p.V; ++cam) {
    const float* m = proj + (b * p.V + cam) * 12;
    const float cx = m[0] * px + m[1] * py + m[2] * pz + m[3], cy = m[4] * px + m[5] * py + m[6] * pz + m[7],
                cz = m[8] * px + m[9] * py + m[10] * pz + m[11];
    const float eps = 1e-5f;
    const float zz = fmaxf(cz, eps);
    const float nx = 2.f * (cx / zz / p.W_in) - 1.f, ny = 2.f * (cy / zz / p.H_in) - 1.f;
    bool ok = lane < p.Z && cz > eps && nx > -1.f && nx < 1.f && ny > -1.f && ny < 1.f;
    const float ddx = rx - camc[(b * p.V + cam) * 2], ddy = ry - camc[(b * p.V + cam) * 2 + 1];
    float nr = 2.f * (sqrtf(ddx * ddx + ddy * ddy) - p.r0) / p.r_cnt - 1.f;
    nr = fminf(fmaxf(nr, -1.f), 1.f);
    float sx = lane < p.Z ? nx : 0.f, sr = lane < p.Z ? nr : 0.f;
    sx = warp_sum(sx) / (float)p.Z;
    sr = warp_sum(sr) / (float)p.Z;
    const bool any = __any_sync(0xffffffffu, ok);
    if (!any) continue;
    vis += 1.f;
    const float gx = (sx + 1.f) * 0.5f * (float)p.W - 0.5f, gy = (sr + 1.f) * 0.5f * (float)p.R - 0.5f;
    if (!(gx > -2.f && gx < (float)p.W + 1.f && gy > -2.f && gy < (float)p.R + 1.f)) continue;
    const float fx = floorf(gx), fy = floorf(gy);
    const int x0 = (int)fx, y0 = (int)fy;
    const float wx1 = gx - fx, wx0 = 1.f - wx1, wy1 = gy - fy, wy0 = 1.f - wy1;
    const float* base = rays + (size_t)(b * p.V + cam) * p.R * p.W * 128 + lane * 4;
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
