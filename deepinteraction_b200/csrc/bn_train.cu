// Train-mode BatchNorm over pixel-major rows: batch statistics, normalise (+ReLU), and the backward with the statistics'
// own gradient.  Reference: models/utils/encoder_utils.py:11-34 (ConvBNReLU: conv -> nn.BatchNorm2d -> ReLU, the norm
// in training mode whenever the module is; momentum set in deepinteraction_encoder.py:52-57).  Every BatchNorm of the
// encoder follows a 1x1 convolution, so its input is a [M = N*H*W, C] row matrix here and the statistics are column
// moments.  HBM-bound element-wise / reduction work: float4 channel vectors, fixed-order partials -> deterministic.
#include "common.cuh"

namespace {

constexpr int BN_BLOCKS = 528;   // 4 x 132 row blocks (H100 SXM)

__device__ __forceinline__ float4 ld4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
inline int bn_blocks(long long M) { return (int)(M < BN_BLOCKS ? M : BN_BLOCKS); }
inline bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// Thread layout of the two column-reduction kernels: 256 threads = 32 float4 channel lanes (a 128-channel tile, blockIdx.y)
// x 8 row lanes; a block owns a contiguous row chunk (blockIdx.x), every load is an independent 16-byte one.
constexpr int BN_RL = 8;

__device__ __forceinline__ float4 f4_add(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }

// per row block and channel: pivot, mean - pivot and M2 (sum of squared deviations from the block mean); the final kernel
// recomputes the block's row count from M.  Two passes over the block's rows: the first estimates the mean from the
// deviations from the block's first row; that estimate becomes the pivot, and the second pass sums the deviations d from
// it: M2 = sum d^2 - (sum d)^2 / n.  One pass shifted by the first row loses M2 to cancellation when that row is an
// outlier.  The mean stays split because pivot + offset rounded to fp32 costs half an ulp of |mean|, which the merge turns
// into spurious variance between blocks when |mean| >> spread.
__global__ void __launch_bounds__(256)
bn_stats_part_kernel(const float* __restrict__ y, long long M, int C, float* __restrict__ part) {
  __shared__ float4 sh1[BN_RL][32], sh2[BN_RL][32];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c = blockIdx.y * 128 + tx * 4;
  const long long rows = (M + gridDim.x - 1) / gridDim.x, m0 = blockIdx.x * rows, m1 = min(M, m0 + rows);
  const bool on = c < C && m0 < m1;
  const float n = (float)max(0LL, m1 - m0), inv = n > 0.f ? 1.f / n : 0.f;
  float4 s1 = make_float4(0.f, 0.f, 0.f, 0.f), s2 = s1, p = s1;
  if (on) {
    p = ld4(y + m0 * C + c);
#pragma unroll 4
    for (long long m = m0 + ty; m < m1; m += BN_RL) {
      const float4 v = ld4(y + m * C + c);
      s1.x += v.x - p.x; s1.y += v.y - p.y; s1.z += v.z - p.z; s1.w += v.w - p.w;
    }
  }
  sh1[ty][tx] = s1;
  __syncthreads();
  s1 = sh1[0][tx];
  for (int r = 1; r < BN_RL; ++r) s1 = f4_add(s1, sh1[r][tx]);
  p = make_float4(p.x + s1.x * inv, p.y + s1.y * inv, p.z + s1.z * inv, p.w + s1.w * inv);
  s1 = make_float4(0.f, 0.f, 0.f, 0.f);
  if (on) {
#pragma unroll 4
    for (long long m = m0 + ty; m < m1; m += BN_RL) {
      const float4 v = ld4(y + m * C + c);
      const float dx = v.x - p.x, dy = v.y - p.y, dz = v.z - p.z, dw = v.w - p.w;
      s1.x += dx; s1.y += dy; s1.z += dz; s1.w += dw;
      s2.x = fmaf(dx, dx, s2.x); s2.y = fmaf(dy, dy, s2.y); s2.z = fmaf(dz, dz, s2.z); s2.w = fmaf(dw, dw, s2.w);
    }
  }
  __syncthreads();
  sh1[ty][tx] = s1;
  sh2[ty][tx] = s2;
  __syncthreads();
  if (ty != 0 || c >= C) return;
  for (int r = 1; r < BN_RL; ++r) { s1 = f4_add(s1, sh1[r][tx]); s2 = f4_add(s2, sh2[r][tx]); }
  const float a1[4] = {s1.x, s1.y, s1.z, s1.w}, a2[4] = {s2.x, s2.y, s2.z, s2.w}, pv[4] = {p.x, p.y, p.z, p.w};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    float* o = part + ((size_t)blockIdx.x * C + c + k) * 3;
    o[0] = pv[k]; o[1] = a1[k] * inv; o[2] = fmaxf(a2[k] - a1[k] * a1[k] * inv, 0.f);
  }
}

// Chan's pairwise combination in double, one warp per channel: lane l folds blocks l, l + 32, ... in order, then a fixed
// shuffle tree merges the 32 partial (n, mean, M2) triples -> deterministic.  Optional running-statistics update (unbiased
// variance, momentum).
__device__ __forceinline__ void chan_merge(double& n, double& mu, double& m2, double nb, double mub, double m2b) {
  if (nb <= 0.0) return;
  const double nn = n + nb, d = mub - mu;
  mu += d * nb / nn;
  m2 += m2b + d * d * n * nb / nn;
  n = nn;
}
__global__ void __launch_bounds__(256)
bn_stats_final_kernel(const float* __restrict__ part, int nblk, int C, long long M, float* __restrict__ mean,
                      float* __restrict__ var, float* __restrict__ run_mean, float* __restrict__ run_var, float momentum) {
  const int c = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (c >= C) return;
  const long long rows = (M + nblk - 1) / nblk;      // the row split of bn_stats_part_kernel
  double n = 0.0, mu = 0.0, m2 = 0.0;
  for (int b = lane; b < nblk; b += 32) {
    const float* p = part + ((size_t)b * C + c) * 3;
    chan_merge(n, mu, m2, (double)max(0LL, min(rows, M - b * rows)), (double)p[0] + (double)p[1], (double)p[2]);
  }
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const double nb = __shfl_xor_sync(0xffffffffu, n, o), mub = __shfl_xor_sync(0xffffffffu, mu, o),
                 m2b = __shfl_xor_sync(0xffffffffu, m2, o);
    // both partners must compute the same merged triple: order the pair by lane so the arithmetic is identical
    if (lane & o) {
      double n2 = nb, mu2 = mub, m22 = m2b;
      chan_merge(n2, mu2, m22, n, mu, m2);
      n = n2; mu = mu2; m2 = m22;
    } else {
      chan_merge(n, mu, m2, nb, mub, m2b);
    }
  }
  if (lane != 0) return;
  mean[c] = (float)mu;
  var[c] = (float)(m2 / (double)M);
  if (run_mean) {
    run_mean[c] = (1.f - momentum) * run_mean[c] + momentum * (float)mu;
    run_var[c] = (1.f - momentum) * run_var[c] + momentum * (float)(M > 1 ? m2 / (double)(M - 1) : m2);
  }
}

// z = act((y - mean) * rstd * gamma + beta)
__global__ void __launch_bounds__(256)
bn_apply_kernel(const float* __restrict__ y, long long n4, int C4, const float* __restrict__ mean, const float* __restrict__ var,
                const float* __restrict__ gamma, const float* __restrict__ beta, float eps, int relu, float* __restrict__ z) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const int c = (int)(i % C4) * 4;
  const float4 v = ld4(y + i * 4), mu = ld4(mean + c), va = ld4(var + c);
  const float4 g = gamma ? ld4(gamma + c) : make_float4(1.f, 1.f, 1.f, 1.f), b = beta ? ld4(beta + c) : make_float4(0.f, 0.f, 0.f, 0.f);
  float4 o;
  o.x = (v.x - mu.x) * (1.f / sqrtf(va.x + eps)) * g.x + b.x;
  o.y = (v.y - mu.y) * (1.f / sqrtf(va.y + eps)) * g.y + b.y;
  o.z = (v.z - mu.z) * (1.f / sqrtf(va.z + eps)) * g.z + b.z;
  o.w = (v.w - mu.w) * (1.f / sqrtf(va.w + eps)) * g.w + b.w;
  if (relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
  *reinterpret_cast<float4*>(z + i * 4) = o;
}

// per row block and channel: sum g, sum g * xhat with g = dz * [z > 0] (z == NULL: no activation), xhat = (y - mean) * rstd
__global__ void __launch_bounds__(256)
bn_bwd_part_kernel(const float* __restrict__ dz, const float* __restrict__ z, const float* __restrict__ y, long long M, int C,
                   const float* __restrict__ mean, const float* __restrict__ var, float eps, float* __restrict__ part) {
  __shared__ float4 sh1[BN_RL][32], sh2[BN_RL][32];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c = blockIdx.y * 128 + tx * 4;
  const long long rows = (M + gridDim.x - 1) / gridDim.x, m0 = blockIdx.x * rows, m1 = min(M, m0 + rows);
  float4 s1 = make_float4(0.f, 0.f, 0.f, 0.f), s2 = s1;
  if (c < C) {
    const float4 mu = ld4(mean + c), va = ld4(var + c);
    const float4 rs = make_float4(1.f / sqrtf(va.x + eps), 1.f / sqrtf(va.y + eps), 1.f / sqrtf(va.z + eps), 1.f / sqrtf(va.w + eps));
#pragma unroll 4
    for (long long m = m0 + ty; m < m1; m += BN_RL) {
      float4 g = ld4(dz + m * C + c);
      const float4 v = ld4(y + m * C + c);
      if (z) {
        const float4 zz = ld4(z + m * C + c);
        g.x = zz.x > 0.f ? g.x : 0.f; g.y = zz.y > 0.f ? g.y : 0.f; g.z = zz.z > 0.f ? g.z : 0.f; g.w = zz.w > 0.f ? g.w : 0.f;
      }
      s1.x += g.x; s1.y += g.y; s1.z += g.z; s1.w += g.w;
      s2.x = fmaf(g.x, (v.x - mu.x) * rs.x, s2.x); s2.y = fmaf(g.y, (v.y - mu.y) * rs.y, s2.y);
      s2.z = fmaf(g.z, (v.z - mu.z) * rs.z, s2.z); s2.w = fmaf(g.w, (v.w - mu.w) * rs.w, s2.w);
    }
  }
  sh1[ty][tx] = s1;
  sh2[ty][tx] = s2;
  __syncthreads();
  if (ty != 0 || c >= C) return;
  for (int r = 1; r < BN_RL; ++r) { s1 = f4_add(s1, sh1[r][tx]); s2 = f4_add(s2, sh2[r][tx]); }
  const float a1[4] = {s1.x, s1.y, s1.z, s1.w}, a2[4] = {s2.x, s2.y, s2.z, s2.w};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    part[((size_t)blockIdx.x * C + c + k) * 2] = a1[k];
    part[((size_t)blockIdx.x * C + c + k) * 2 + 1] = a2[k];
  }
}
__global__ void __launch_bounds__(256)
bn_bwd_final_kernel(const float* __restrict__ part, int nblk, int C, float* __restrict__ s1, float* __restrict__ s2) {
  const int c = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;     // one warp per channel, fixed order
  if (c >= C) return;
  double a = 0.0, b = 0.0;
  for (int k = lane; k < nblk; k += 32) {
    a += (double)part[((size_t)k * C + c) * 2];
    b += (double)part[((size_t)k * C + c) * 2 + 1];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_down_sync(0xffffffffu, a, o);
    b += __shfl_down_sync(0xffffffffu, b, o);
  }
  if (lane != 0) return;
  s1[c] = (float)a;     // = d beta
  s2[c] = (float)b;     // = d gamma
}

// dy = gamma * rstd * (g - s1 / M - xhat * s2 / M)
__global__ void __launch_bounds__(256)
bn_bwd_apply_kernel(const float* __restrict__ dz, const float* __restrict__ z, const float* __restrict__ y, long long n4, int C4,
                    const float* __restrict__ mean, const float* __restrict__ var, const float* __restrict__ gamma, float eps,
                    const float* __restrict__ s1, const float* __restrict__ s2, float inv_m, float* __restrict__ dy) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const int c = (int)(i % C4) * 4;
  float4 g = ld4(dz + i * 4);
  if (z) {
    const float4 zz = ld4(z + i * 4);
    g.x = zz.x > 0.f ? g.x : 0.f; g.y = zz.y > 0.f ? g.y : 0.f; g.z = zz.z > 0.f ? g.z : 0.f; g.w = zz.w > 0.f ? g.w : 0.f;
  }
  const float4 v = ld4(y + i * 4), mu = ld4(mean + c), va = ld4(var + c), a = ld4(s1 + c), b = ld4(s2 + c);
  const float4 ga = gamma ? ld4(gamma + c) : make_float4(1.f, 1.f, 1.f, 1.f);
  float4 o;
  float r;
  r = 1.f / sqrtf(va.x + eps); o.x = ga.x * r * (g.x - a.x * inv_m - (v.x - mu.x) * r * b.x * inv_m);
  r = 1.f / sqrtf(va.y + eps); o.y = ga.y * r * (g.y - a.y * inv_m - (v.y - mu.y) * r * b.y * inv_m);
  r = 1.f / sqrtf(va.z + eps); o.z = ga.z * r * (g.z - a.z * inv_m - (v.z - mu.z) * r * b.z * inv_m);
  r = 1.f / sqrtf(va.w + eps); o.w = ga.w * r * (g.w - a.w * inv_m - (v.w - mu.w) * r * b.w * inv_m);
  *reinterpret_cast<float4*>(dy + i * 4) = o;
}

}  // namespace

extern "C" {

// y [M, C] contiguous rows -> mean [C], var [C] (biased, as the normalisation uses); run_mean / run_var (optional) updated
// in place with `momentum` and the unbiased variance (torch.nn.BatchNorm2d training semantics).  C % 4 == 0.
// work: float [592 * C * 3]
int di_bn_stats_f32(const float* y, long long M, int C, float* work, float* mean, float* var, float* run_mean, float* run_var,
                    float momentum, cudaStream_t stream) {
  DI_CHECK_ARG(y && work && mean && var && M > 0 && C > 0 && C % 4 == 0 && al16(y) && (!run_mean == !run_var),
               "di_bn_stats_f32: bad argument");
  const int nblk = bn_blocks(M);
  bn_stats_part_kernel<<<dim3(nblk, di_cdiv(C, 128)), 256, 0, stream>>>(y, M, C, work);
  bn_stats_final_kernel<<<di_cdiv(C, 8), 256, 0, stream>>>(work, nblk, C, M, mean, var, run_mean, run_var, momentum);
  DI_CHECK_LAUNCH("di_bn_stats_f32");
  return DI_OK;
}

// z = act((y - mean) / sqrt(var + eps) * gamma + beta); gamma / beta NULL = affine=False; z may alias y
int di_bn_apply_f32(const float* y, long long M, int C, const float* mean, const float* var, const float* gamma, const float* beta,
                    float eps, int relu, float* z, cudaStream_t stream) {
  DI_CHECK_ARG(y && mean && var && z && M > 0 && C > 0 && C % 4 == 0 && al16(y) && al16(z) && al16(mean) && al16(var) &&
                   al16(gamma) && al16(beta), "di_bn_apply_f32: bad argument");
  const long long n4 = M * (C / 4);
  bn_apply_kernel<<<(unsigned)di_cdiv(n4, 256), 256, 0, stream>>>(y, n4, C / 4, mean, var, gamma, beta, eps, relu, z);
  DI_CHECK_LAUNCH("di_bn_apply_f32");
  return DI_OK;
}

// Backward of z = act(BN_train(y)): dz [M, C], z (the saved output; NULL when there is no ReLU), y (the saved input) ->
// dy [M, C] (may alias dz), dgamma [C], dbeta [C].  work: float [592 * C * 2]
int di_bn_bwd_f32(const float* dz, const float* z, const float* y, long long M, int C, const float* mean, const float* var,
                  const float* gamma, float eps, float* work, float* dy, float* dgamma, float* dbeta, cudaStream_t stream) {
  DI_CHECK_ARG(dz && y && mean && var && work && dy && dgamma && dbeta && M > 0 && C > 0 && C % 4 == 0 && al16(dz) && al16(z) &&
                   al16(y) && al16(dy) && al16(mean) && al16(var) && al16(gamma) && al16(dgamma) && al16(dbeta),
               "di_bn_bwd_f32: bad argument");
  const int nblk = bn_blocks(M);
  bn_bwd_part_kernel<<<dim3(nblk, di_cdiv(C, 128)), 256, 0, stream>>>(dz, z, y, M, C, mean, var, eps, work);
  bn_bwd_final_kernel<<<di_cdiv(C, 8), 256, 0, stream>>>(work, nblk, C, dbeta, dgamma);
  const long long n4 = M * (C / 4);
  bn_bwd_apply_kernel<<<(unsigned)di_cdiv(n4, 256), 256, 0, stream>>>(dz, z, y, n4, C / 4, mean, var, gamma, eps, dbeta, dgamma,
                                                                     1.f / (float)M, dy);
  DI_CHECK_LAUNCH("di_bn_bwd_f32");
  return DI_OK;
}

}  // extern "C"
