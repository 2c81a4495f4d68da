// Backward of the 9x9 window attention of LocalContextAttentionBlock on pixel-major maps (SURVEY.md 8(b) `di_lcab_backward`).
//
// Forward (models/utils/encoder_utils.py:132-134 with the window ops of locatt_ops/kernels.cuh:4-80):
//     S[p, j] = q[p] . k[nbr(p, j)]   (0 for a tap outside the map -- it still takes softmax mass)
//     A       = softmax_j(S * scale)
//     out[p]  = sum_j A[p, j] v[nbr(p, j)]   (taps outside the map skipped)
// Backward for a given dOut, in the same order the reference's autograd runs its kernels (weighting_backward_weight /
// weighting_backward_ori, softmax backward, similar_backward x 2; kernels.cuh:44-119, similar.cu:43-92, weighting.cu:44-121):
//     dA[p, j] = dOut[p] . v[nbr(p, j)]                         di_win_dot_f32(dOut, v)
//     dv[p']   = sum_{nbr(p, j) = p'} A[p, j] dOut[p]           di_win_scatter_f32(A, dOut)
//     dS       = A * (dA - sum_j A dA) * scale                  di_win_softmax_bwd_f32
//     dq[p]    = sum_j dS[p, j] k[nbr(p, j)]                    di_win_gather_f32(dS, k)
//     dk[p']   = sum_{nbr(p, j) = p'} dS[p, j] q[p]             di_win_scatter_f32(dS, q)
// One warp per 4 x-adjacent pixels, lanes over channels (float4), the kH*kW taps in a loop; tap j = (dy + r) * kW + (dx + r), the
// reference's order (similar.cu:15-17).  fp32 throughout.  These are the training-side counterparts of the fused
// forward kernels; they are not fused (the [P, 81] tensors go through memory) -- first correct, measured version.
#include "common.cuh"

namespace {

// A warp owns WPX pixels adjacent in x: their windows overlap in (ks - 1) of ks columns, so every neighbour row is loaded once
// per warp and used for up to WPX taps (3x fewer L2 -> SM bytes than one pixel per warp at ks = 9).  The per-pixel
// arithmetic and its order are those of the one-pixel form.
constexpr int WPX = 4;

// out[p, j] = a[p] . b[nbr(p, j)]
template <int VEC>
__global__ void __launch_bounds__(256)
win_dot_kernel(const float* __restrict__ a, int lda, const float* __restrict__ b, int ldb, float* __restrict__ out, int N, int H,
               int W, int C, int ks) {
  const int gpr = (W + WPX - 1) / WPX;
  const int gid = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (gid >= N * H * gpr) return;
  const int row = gid / gpr, x0 = (gid - row * gpr) * WPX, n = row / H, y = row - n * H, r = ks >> 1, KK = ks * ks;
  const int npx = min(WPX, W - x0);
  float4 av[WPX][VEC];
#pragma unroll
  for (int i = 0; i < WPX; ++i)
#pragma unroll
    for (int v = 0; v < VEC; ++v) {
      const int c = (v * 32 + lane) * 4;
      av[i][v] = (i < npx && c < C) ? ldg4(a + ((size_t)row * W + x0 + i) * lda + c) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  float* o = out + ((size_t)row * W + x0) * KK;
  for (int dy = -r; dy <= r; ++dy) {
    const int yy = y + dy;
    const bool rowok = yy >= 0 && yy < H;
    for (int cx = -r; cx <= r + WPX - 1; ++cx) {
      const int xx = x0 + cx;
      const bool ok = rowok && xx >= 0 && xx < W;                 // warp-uniform
      float4 bv[VEC];
#pragma unroll
      for (int v = 0; v < VEC; ++v) {
        const int c = (v * 32 + lane) * 4;
        bv[v] = (ok && c < C) ? ldg4(b + ((size_t)(n * H + yy) * W + xx) * ldb + c) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
      // the WPX dot products of this neighbour row, reduced together: two exchange steps fold 4 values per lane into 1
      // (lanes with bits 4:3 = i keep pixel i), three more finish the sum -- 6 shuffles instead of 4 x 5
      float s[WPX];
#pragma unroll
      for (int i = 0; i < WPX; ++i) {
        s[i] = 0.f;
#pragma unroll
        for (int v = 0; v < VEC; ++v) s[i] += av[i][v].x * bv[v].x + av[i][v].y * bv[v].y + av[i][v].z * bv[v].z + av[i][v].w * bv[v].w;
      }
      const bool up16 = lane & 16, up8 = lane & 8;
      const float k0 = up16 ? s[2] : s[0], k1 = up16 ? s[3] : s[1];          // kept pair
      const float g0 = up16 ? s[0] : s[2], g1 = up16 ? s[1] : s[3];          // given to the partner half
      const float t0 = k0 + __shfl_xor_sync(0xffffffffu, g0, 16), t1 = k1 + __shfl_xor_sync(0xffffffffu, g1, 16);
      float t = (up8 ? t1 : t0) + __shfl_xor_sync(0xffffffffu, up8 ? t0 : t1, 8);
      t += __shfl_xor_sync(0xffffffffu, t, 4);
      t += __shfl_xor_sync(0xffffffffu, t, 2);
      t += __shfl_xor_sync(0xffffffffu, t, 1);
      const int i = lane >> 3, dx = cx - i;                                  // lanes 0, 8, 16, 24 write pixels 0..3
      if ((lane & 7) == 0 && i < npx && dx >= -r && dx <= r) o[(size_t)i * KK + (dy + r) * ks + dx + r] = ok ? t : 0.f;
    }
  }
}

// gather: out[p] = sum_j w[p, j] b[nbr(p, j)];   scatter (transposed): out[p] = sum_j w[p - off_j, j] b[p - off_j]
template <int VEC, bool SCATTER>
__global__ void __launch_bounds__(256)
win_apply_kernel(const float* __restrict__ w, const float* __restrict__ b, int ldb, float* __restrict__ out, int ldo, int N,
                 int H, int W, int C, int ks) {
  const int gpr = (W + WPX - 1) / WPX;
  const int gid = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (gid >= N * H * gpr) return;
  const int row = gid / gpr, x0 = (gid - row * gpr) * WPX, n = row / H, y = row - n * H, r = ks >> 1, KK = ks * ks;
  const int npx = min(WPX, W - x0);
  float4 acc[WPX][VEC];
#pragma unroll
  for (int i = 0; i < WPX; ++i)
#pragma unroll
    for (int v = 0; v < VEC; ++v) acc[i][v] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int dy = -r; dy <= r; ++dy) {                              // tap row, in the reference's order
    const int yy = SCATTER ? y - dy : y + dy;
    if (yy < 0 || yy >= H) continue;
    for (int u = 0; u < ks + WPX - 1; ++u) {
      const int cx = SCATTER ? r + WPX - 1 - u : u - r;            // source column relative to x0; tap dx ascends with u
      const int xx = x0 + cx;
      if (xx < 0 || xx >= W) continue;
      const size_t src = (size_t)(n * H + yy) * W + xx;
      float4 bv[VEC];
#pragma unroll
      for (int v = 0; v < VEC; ++v) {
        const int c = (v * 32 + lane) * 4;
        bv[v] = c < C ? ldg4(b + src * ldb + c) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int i = 0; i < WPX; ++i) {
        const int dx = SCATTER ? i - cx : cx - i;
        if (dx < -r || dx > r || i >= npx) continue;
        const int j = (dy + r) * ks + dx + r;
        const float wt = SCATTER ? __ldg(w + src * KK + j) : __ldg(w + ((size_t)row * W + x0 + i) * KK + j);
#pragma unroll
        for (int v = 0; v < VEC; ++v) {
          acc[i][v].x = fmaf(wt, bv[v].x, acc[i][v].x);
          acc[i][v].y = fmaf(wt, bv[v].y, acc[i][v].y);
          acc[i][v].z = fmaf(wt, bv[v].z, acc[i][v].z);
          acc[i][v].w = fmaf(wt, bv[v].w, acc[i][v].w);
        }
      }
    }
  }
#pragma unroll
  for (int i = 0; i < WPX; ++i)
#pragma unroll
    for (int v = 0; v < VEC; ++v) {
      const int c = (v * 32 + lane) * 4;
      if (i < npx && c < C) *reinterpret_cast<float4*>(out + ((size_t)row * W + x0 + i) * ldo + c) = acc[i][v];
    }
}

// rows of KK <= 128 values: A = softmax(S * scale) (forward, in place allowed)
__global__ void __launch_bounds__(256)
win_softmax_kernel(const float* __restrict__ S, float* __restrict__ A, long long P, int KK, float scale) {
  const long long wid = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (wid >= P) return;
  float v[4];
  float m = -INFINITY;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int j = i * 32 + lane;
    v[i] = j < KK ? S[wid * KK + j] * scale : -INFINITY;
    m = fmaxf(m, v[i]);
  }
  m = warp_max(m);
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    v[i] = (i * 32 + lane) < KK ? expf(v[i] - m) : 0.f;
    sum += v[i];
  }
  sum = warp_sum(sum);
  const float inv = 1.f / sum;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int j = i * 32 + lane;
    if (j < KK) A[wid * KK + j] = v[i] * inv;
  }
}

// dS = A * (dA - sum_j A dA) * scale   (dS may alias dA)
__global__ void __launch_bounds__(256)
win_softmax_bwd_kernel(const float* __restrict__ A, const float* __restrict__ dA, float* __restrict__ dS, long long P, int KK,
                       float scale) {
  const long long wid = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (wid >= P) return;
  float a[4], g[4];
  float dot = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int j = i * 32 + lane;
    a[i] = j < KK ? A[wid * KK + j] : 0.f;
    g[i] = j < KK ? dA[wid * KK + j] : 0.f;
    dot += a[i] * g[i];
  }
  dot = warp_sum(dot);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int j = i * 32 + lane;
    if (j < KK) dS[wid * KK + j] = a[i] * (g[i] - dot) * scale;
  }
}

// dx = dy * [y > 0]  (ReLU backward from the saved OUTPUT), in place allowed
__global__ void relu_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y, float* __restrict__ dx, long long n) {
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (i + 3 < n) {
    const float4 g = ldg4(dy + i), v = ldg4(y + i);
    *reinterpret_cast<float4*>(dx + i) = make_float4(v.x > 0.f ? g.x : 0.f, v.y > 0.f ? g.y : 0.f, v.z > 0.f ? g.z : 0.f,
                                                     v.w > 0.f ? g.w : 0.f);
  } else {
    for (long long k = i; k < n; ++k) dx[k] = y[k] > 0.f ? dy[k] : 0.f;
  }
}

// column sums of a [M, C] matrix (bias gradients): part[blk, c] then a fixed-order final pass -> deterministic
__global__ void __launch_bounds__(256)
col_sum_part_kernel(const float* __restrict__ x, int ld, long long M, int C, float* __restrict__ part) {
  const int c = blockIdx.y * 256 + threadIdx.x;
  if (c >= C) return;
  const long long rows = (M + gridDim.x - 1) / gridDim.x, m0 = blockIdx.x * rows, m1 = min(M, m0 + rows);
  float s = 0.f;
  for (long long m = m0; m < m1; ++m) s += x[m * ld + c];
  part[(size_t)blockIdx.x * C + c] = s;
}
__global__ void col_sum_final_kernel(const float* __restrict__ part, int nblk, int C, float* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double s = 0.0;
  for (int b = 0; b < nblk; ++b) s += (double)part[(size_t)b * C + c];
  out[c] = (float)s;
}

// LayerNorm backward over [M, C] rows, one warp per row (C <= 512): y = (z - mean) rstd gamma + beta ->
// dz = rstd (gamma dy - mean(gamma dy) - xhat mean(gamma dy xhat)); prod = dy xhat (its column sums are d gamma)
__global__ void __launch_bounds__(256)
ln_bwd_kernel(const float* __restrict__ dy, int ldy, const float* __restrict__ z, int ldz, const float* __restrict__ gamma,
              float* __restrict__ dz, int lddz, float* __restrict__ prod, int M, int C, float eps) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= M) return;
  constexpr int NV = 16;
  float zv[NV], gv[NV];
  float s = 0.f;
#pragma unroll
  for (int n = 0; n < NV; ++n) {
    const int c = n * 32 + lane;
    zv[n] = c < C ? z[(size_t)row * ldz + c] : 0.f;
    s += zv[n];
  }
  const float mean = warp_sum(s) / (float)C;
  float var = 0.f;
#pragma unroll
  for (int n = 0; n < NV; ++n) {
    const int c = n * 32 + lane;
    const float d = c < C ? zv[n] - mean : 0.f;
    var += d * d;
  }
  const float rstd = 1.f / sqrtf(warp_sum(var) / (float)C + eps);
  float s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int n = 0; n < NV; ++n) {
    const int c = n * 32 + lane;
    gv[n] = 0.f;
    if (c < C) {
      const float g = dy[(size_t)row * ldy + c];
      zv[n] = (zv[n] - mean) * rstd;                   // xhat
      prod[(size_t)row * C + c] = g * zv[n];
      gv[n] = g * gamma[c];
      s1 += gv[n];
      s2 += gv[n] * zv[n];
    }
  }
  s1 = warp_sum(s1) / (float)C;
  s2 = warp_sum(s2) / (float)C;
#pragma unroll
  for (int n = 0; n < NV; ++n) {
    const int c = n * 32 + lane;
    if (c < C) dz[(size_t)row * lddz + c] = (gv[n] - s1 - zv[n] * s2) * rstd;
  }
}

// out[n, y, x, :] = in[n, y + dy, x + dx, :] (zero outside the map): the shifted copies behind the weight gradient of a
// 3x3 convolution (dW[co, tap, ci] = sum_p dY[p, co] X[p + tap, ci])
__global__ void shift_map_kernel(const float4* __restrict__ in, float4* __restrict__ out, int N, int H, int W, int C4, int dy,
                                 int dx) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)N * H * W * C4) return;
  const int c = (int)(i % C4);
  const long long p = i / C4;
  const int x = (int)(p % W), y = (int)((p / W) % H), n = (int)(p / ((long long)W * H));
  const int yy = y + dy, xx = x + dx;
  out[i] = (yy >= 0 && yy < H && xx >= 0 && xx < W) ? in[(((long long)n * H + yy) * W + xx) * C4 + c] : make_float4(0.f, 0.f, 0.f, 0.f);
}

template <int VEC>
int launch_dot(const float* a, int lda, const float* b, int ldb, float* out, int N, int H, int W, int C, int ks, cudaStream_t st) {
  win_dot_kernel<VEC><<<di_cdiv((long long)N * H * di_cdiv(W, WPX), 8), 256, 0, st>>>(a, lda, b, ldb, out, N, H, W, C, ks);
  return 0;
}
template <int VEC, bool SC>
int launch_apply(const float* w, const float* b, int ldb, float* out, int ldo, int N, int H, int W, int C, int ks, cudaStream_t st) {
  win_apply_kernel<VEC, SC><<<di_cdiv((long long)N * H * di_cdiv(W, WPX), 8), 256, 0, st>>>(w, b, ldb, out, ldo, N, H, W, C, ks);
  return 0;
}

}  // namespace

extern "C" {

#define DI_WIN_CHECK(name)                                                                                              \
  DI_CHECK_ARG(N > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0 && C <= 512 && ks >= 1 && (ks & 1) && ks * ks <= 128,      \
               name ": unsupported shape (C=%d ks=%d)", C, ks)

// out [N*H*W, ks*ks] = a[p] . b[nbr(p, j)]  (0 outside the map): similar_forward (a = q, b = k) and
// weighting_backward_weight (a = dOut, b = v).  a, b pixel-major rows with leading dimensions lda, ldb.
int di_win_dot_f32(const float* a, int lda, const float* b, int ldb, float* out, int N, int H, int W, int C, int ks,
                   cudaStream_t stream) {
  DI_CHECK_ARG(a && b && out && lda % 4 == 0 && ldb % 4 == 0, "di_win_dot_f32: bad argument");
  DI_WIN_CHECK("di_win_dot_f32");
  if (C <= 128) launch_dot<1>(a, lda, b, ldb, out, N, H, W, C, ks, stream);
  else if (C <= 256) launch_dot<2>(a, lda, b, ldb, out, N, H, W, C, ks, stream);
  else launch_dot<4>(a, lda, b, ldb, out, N, H, W, C, ks, stream);
  DI_CHECK_LAUNCH("di_win_dot_f32");
  return DI_OK;
}

// out[p] = sum_j w[p, j] b[nbr(p, j)]: weighting_forward (w = A, b = v) and similar_backward(is_ori) (w = dS, b = k)
int di_win_gather_f32(const float* w, const float* b, int ldb, float* out, int ldo, int N, int H, int W, int C, int ks,
                      cudaStream_t stream) {
  DI_CHECK_ARG(w && b && out && ldb % 4 == 0 && ldo % 4 == 0, "di_win_gather_f32: bad argument");
  DI_WIN_CHECK("di_win_gather_f32");
  if (C <= 128) launch_apply<1, false>(w, b, ldb, out, ldo, N, H, W, C, ks, stream);
  else if (C <= 256) launch_apply<2, false>(w, b, ldb, out, ldo, N, H, W, C, ks, stream);
  else launch_apply<4, false>(w, b, ldb, out, ldo, N, H, W, C, ks, stream);
  DI_CHECK_LAUNCH("di_win_gather_f32");
  return DI_OK;
}

// out[p'] = sum over (p, j) with nbr(p, j) = p' of w[p, j] b[p]: similar_backward(!is_ori) (w = dS, b = q) and
// weighting_backward_ori (w = A, b = dOut)
int di_win_scatter_f32(const float* w, const float* b, int ldb, float* out, int ldo, int N, int H, int W, int C, int ks,
                       cudaStream_t stream) {
  DI_CHECK_ARG(w && b && out && ldb % 4 == 0 && ldo % 4 == 0, "di_win_scatter_f32: bad argument");
  DI_WIN_CHECK("di_win_scatter_f32");
  if (C <= 128) launch_apply<1, true>(w, b, ldb, out, ldo, N, H, W, C, ks, stream);
  else if (C <= 256) launch_apply<2, true>(w, b, ldb, out, ldo, N, H, W, C, ks, stream);
  else launch_apply<4, true>(w, b, ldb, out, ldo, N, H, W, C, ks, stream);
  DI_CHECK_LAUNCH("di_win_scatter_f32");
  return DI_OK;
}

int di_win_softmax_f32(const float* S, float* A, long long P, int KK, float scale, cudaStream_t stream) {
  DI_CHECK_ARG(S && A && P > 0 && KK > 0 && KK <= 128, "di_win_softmax_f32: bad argument");
  win_softmax_kernel<<<di_cdiv(P, 8), 256, 0, stream>>>(S, A, P, KK, scale);
  DI_CHECK_LAUNCH("di_win_softmax_f32");
  return DI_OK;
}

int di_win_softmax_bwd_f32(const float* A, const float* dA, float* dS, long long P, int KK, float scale, cudaStream_t stream) {
  DI_CHECK_ARG(A && dA && dS && P > 0 && KK > 0 && KK <= 128, "di_win_softmax_bwd_f32: bad argument");
  win_softmax_bwd_kernel<<<di_cdiv(P, 8), 256, 0, stream>>>(A, dA, dS, P, KK, scale);
  DI_CHECK_LAUNCH("di_win_softmax_bwd_f32");
  return DI_OK;
}

int di_relu_bwd_f32(const float* dy, const float* y, float* dx, long long n, cudaStream_t stream) {
  DI_CHECK_ARG(dy && y && dx && n > 0 && ((((uintptr_t)dy | (uintptr_t)y | (uintptr_t)dx) & 15) == 0), "di_relu_bwd_f32: bad argument");
  relu_bwd_kernel<<<di_cdiv(di_cdiv(n, 4), 256), 256, 0, stream>>>(dy, y, dx, n);
  DI_CHECK_LAUNCH("di_relu_bwd_f32");
  return DI_OK;
}

// out [N, H, W, C] = in shifted by (dy, dx) with zero fill (pixel-major maps, C % 4 == 0)
int di_shift_map_f32(const float* in, float* out, int N, int H, int W, int C, int dy, int dx, cudaStream_t stream) {
  DI_CHECK_ARG(in && out && N > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0 && ((((uintptr_t)in | (uintptr_t)out) & 15) == 0),
               "di_shift_map_f32: bad argument");
  const long long n4 = (long long)N * H * W * (C / 4);
  shift_map_kernel<<<di_cdiv(n4, 256), 256, 0, stream>>>(reinterpret_cast<const float4*>(in), reinterpret_cast<float4*>(out), N,
                                                        H, W, C / 4, dy, dx);
  DI_CHECK_LAUNCH("di_shift_map_f32");
  return DI_OK;
}

// out[c] = sum_m x[m, c]; work: float [256 * C]
int di_col_sum_f32(const float* x, int ld, long long M, int C, float* work, float* out, cudaStream_t stream) {
  DI_CHECK_ARG(x && work && out && M > 0 && C > 0, "di_col_sum_f32: bad argument");
  const int nblk = (int)(M < 256 ? M : 256);
  col_sum_part_kernel<<<dim3(nblk, di_cdiv(C, 256)), 256, 0, stream>>>(x, ld, M, C, work);
  col_sum_final_kernel<<<di_cdiv(C, 128), 128, 0, stream>>>(work, nblk, C, out);
  DI_CHECK_LAUNCH("di_col_sum_f32");
  return DI_OK;
}

// Backward of y = LayerNorm(z) (gamma, beta) over [M, C] rows, C <= 512: dy -> dz, dgamma, dbeta (fixed-order column sums,
// as di_col_sum_f32); work: float [M * C + 256 * C].
int di_ln_bwd_f32(const float* dy, int ldy, const float* z, int ldz, const float* gamma, float* dz, int lddz, float* dgamma,
                  float* dbeta, float* work, int M, int C, float eps, cudaStream_t stream) {
  DI_CHECK_ARG(dy && z && gamma && dz && dgamma && dbeta && work && M > 0 && C > 0 && C <= 512, "di_ln_bwd_f32: bad argument");
  float* prod = work;
  float* part = work + (size_t)M * C;
  ln_bwd_kernel<<<di_cdiv(M, 8), 256, 0, stream>>>(dy, ldy, z, ldz, gamma, dz, lddz, prod, M, C, eps);
  DI_CHECK_LAUNCH("di_ln_bwd_f32");
  const int nblk = M < 256 ? M : 256;
  col_sum_part_kernel<<<dim3(nblk, di_cdiv(C, 256)), 256, 0, stream>>>(prod, C, M, C, part);
  col_sum_final_kernel<<<di_cdiv(C, 128), 128, 0, stream>>>(part, nblk, C, dgamma);
  col_sum_part_kernel<<<dim3(nblk, di_cdiv(C, 256)), 256, 0, stream>>>(dy, ldy, M, C, part);
  col_sum_final_kernel<<<di_cdiv(C, 128), 128, 0, stream>>>(part, nblk, C, dbeta);
  DI_CHECK_LAUNCH("di_ln_bwd_f32 (column sums)");
  return DI_OK;
}

}  // extern "C"
