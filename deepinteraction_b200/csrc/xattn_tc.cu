// Query x BEV cross attention of the MMPI decoder on the tensor cores (mma.sync bf16, cp.async-staged operands).
//
// Reference: TransformerDecoderLayer / multi_head_attention_forward, models/utils/decoder_utils.py:101-103, 466-493:
// P = 200 object queries x HW = 32 400 BEV keys, 8 heads of 16 channels, softmax over all keys.  The K / V projection
// (with the folded key positional term) stays a 3xTF32 GEMM; di_attn_planes_f32 then writes the operands as bf16 PLANES:
// K and the pre-scaled queries as hi | mid | lo (x = hi + mid + lo to 24 mantissa bits: the logits go through exp, and a
// two-plane product -- 3 * 2^-18 relative -- moved the decoder outputs by up to 3e-3), V as hi | mid.  The 16 channels
// of a head are one k16 step of the MMA.
//
// CTA = (key split, query tile of 64, batch); 8 warps: warp w owns queries 16 (w & 3) .. + 15 and heads 4 (w >> 2) .. + 3.
// Key tiles of 64 keys stream through a double-buffered cp.async ring (K planes | V planes, padded rows: conflict-free
// fragment loads).  Per key tile and head:
//   S_h[16 q x 64 keys] = Q_h K_h^T   six-term split product (lo hi, hi lo, mid mid, mid hi, hi mid, hi hi: error ~2^-26)
//   P_h = exp(S_h - m)                online softmax, running maximum m and sum l per query row in registers; the S
//                                     accumulator fragments ARE the A fragments of the next product (bf16 hi | mid)
//   O_h = O_h * corr + P_h V_h        three-term split product; V fragments through ldmatrix.trans
// At the end every warp writes (m, l, acc[16]) per (query, head) -- flash-decoding partials -- and
// xattn_combine_kernel merges the key splits (one warp per (batch, head, query), lanes over the splits).
#include "tc_common.cuh"

namespace {
using namespace tc;

constexpr int XT_KEYS = 64;                          // keys per tile
constexpr int XT_QT = 64;                            // queries per CTA
constexpr int KSTR = 196, VSTR = 132;                // padded row strides (words) of the K (hi|mid|lo) and V (hi|mid) planes
constexpr int XT_STAGE_WORDS = XT_KEYS * (KSTR + VSTR);
constexpr int XT_Q_WORDS = XT_QT * KSTR;
constexpr int XT_SMEM = (XT_Q_WORDS + 2 * XT_STAGE_WORDS) * 4;
constexpr int XT_THREADS = 256;
static_assert(XT_SMEM <= 232448, "xattn kernel exceeds the shared-memory limit");

__device__ __forceinline__ void x_mma(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void x_cp16(uint32_t dst, const void* src, bool ok) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(ok ? 16 : 0) : "memory");
}

struct XtParams {
  int P, HW, heads, nsplit, chunk;       // chunk: keys per split (multiple of 64)
  float* part;                           // [B, heads, nsplit, 18, P]
};

__global__ void __launch_bounds__(XT_THREADS, 1)
xattn_tc_kernel(const uint32_t* __restrict__ qp, const uint32_t* __restrict__ kp, const uint32_t* __restrict__ vp,
                const XtParams p) {
  extern __shared__ __align__(16) uint32_t xs[];     // Q tile [64][KSTR] | 2 stages of K [64][KSTR], V [64][VSTR]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int sp = blockIdx.x, mt = blockIdx.y, b = blockIdx.z;
  const int k_begin = sp * p.chunk, k_end = min(p.HW, k_begin + p.chunk);
  const int ntiles = (k_end - k_begin + XT_KEYS - 1) / XT_KEYS;          // >= 1 (the host sizes the splits)
  const uint32_t sbase = smem_u32(xs);

  // Q tile (rows past P are zero)
  for (int i = tid; i < XT_QT * 48; i += XT_THREADS) {
    const int r = i / 48, c4 = i % 48;
    const int qi = mt * XT_QT + r;
    const bool ok = qi < p.P;
    x_cp16(sbase + (uint32_t)(r * KSTR + c4 * 4) * 4u, ok ? qp + ((size_t)b * p.P + qi) * 192 + c4 * 4 : qp, ok);
  }
  auto issue = [&](int i) {
    const uint32_t st = sbase + (uint32_t)(XT_Q_WORDS + (i & 1) * XT_STAGE_WORDS) * 4u;
    const int row0 = k_begin + i * XT_KEYS;
    for (int j = tid; j < XT_KEYS * 80; j += XT_THREADS) {
      const int r = j / 80, c4 = j % 80;
      const int key = row0 + r;
      const bool ok = key < k_end;
      const size_t grow = (size_t)b * p.HW + key;
      if (c4 < 48) x_cp16(st + (uint32_t)(r * KSTR + c4 * 4) * 4u, ok ? kp + grow * 192 + c4 * 4 : kp, ok);
      else x_cp16(st + (uint32_t)(XT_KEYS * KSTR + r * VSTR + (c4 - 48) * 4) * 4u, ok ? vp + grow * 128 + (c4 - 48) * 4 : vp, ok);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };

  const int q0 = 16 * (warp & 3), h0 = 4 * (warp >> 2);
  constexpr float L2E = 1.4426950408889634f;
  float m[4][2], l[4][2], acc[4][2][4];
#pragma unroll
  for (int h = 0; h < 4; ++h) {
    m[h][0] = m[h][1] = -INFINITY;
    l[h][0] = l[h][1] = 0.f;
#pragma unroll
    for (int cb = 0; cb < 2; ++cb) acc[h][cb][0] = acc[h][cb][1] = acc[h][cb][2] = acc[h][cb][3] = 0.f;
  }

  issue(0);
  for (int i = 0; i < ntiles; ++i) {
    if (i + 1 < ntiles) {
      issue(i + 1);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    const int nvalid = min(XT_KEYS, k_end - (k_begin + i * XT_KEYS));
    const uint32_t* ks = xs + XT_Q_WORDS + (i & 1) * XT_STAGE_WORDS;
    const uint32_t vs_addr = sbase + (uint32_t)(XT_Q_WORDS + (i & 1) * XT_STAGE_WORDS + XT_KEYS * KSTR) * 4u;
#pragma unroll
    for (int hh = 0; hh < 4; ++hh) {                  // unrolled: the per-head state stays in registers
      const int h = h0 + hh;
      // Q fragments of this head: planes hi (0), mid (64), lo (128); channel pair words 8h + t (+4)
      uint32_t qa[3][4];
#pragma unroll
      for (int pl = 0; pl < 3; ++pl) {
        const uint32_t* qr0 = xs + (q0 + g) * KSTR + 64 * pl + 8 * h + t;
        const uint32_t* qr1 = qr0 + 8 * KSTR;
        qa[pl][0] = qr0[0]; qa[pl][1] = qr1[0]; qa[pl][2] = qr0[4]; qa[pl][3] = qr1[4];
      }
      float S[8][4];
#pragma unroll
      for (int nb = 0; nb < 8; ++nb) {
        S[nb][0] = S[nb][1] = S[nb][2] = S[nb][3] = 0.f;
        const uint32_t* kr = ks + (nb * 8 + g) * KSTR + 8 * h + t;
        const uint32_t khi0 = kr[0], khi1 = kr[4], kmid0 = kr[64], kmid1 = kr[68], klo0 = kr[128], klo1 = kr[132];
        x_mma(S[nb], qa[2], khi0, khi1);            // smallest terms first
        x_mma(S[nb], qa[0], klo0, klo1);
        x_mma(S[nb], qa[1], kmid0, kmid1);
        x_mma(S[nb], qa[1], khi0, khi1);
        x_mma(S[nb], qa[0], kmid0, kmid1);
        x_mma(S[nb], qa[0], khi0, khi1);
      }
      // online softmax: rows g (j = 0, 1) and g + 8 (j = 2, 3); key of element j = nb * 8 + 2t + (j & 1)
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int nb = 0; nb < 8; ++nb)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (nb * 8 + 2 * t + (j & 1) >= nvalid) S[nb][j] = -INFINITY;
          mx[j >> 1] = fmaxf(mx[j >> 1], S[nb][j]);
        }
      float corr[2], mc[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
        const float mn = fmaxf(m[hh][r], mx[r]);
        corr[r] = exp2f((m[hh][r] - mn) * L2E);     // 0 on the first tile (m = -inf)
        mc[r] = mn * L2E;
        m[hh][r] = mn;
      }
      float sum[2] = {0.f, 0.f};
#pragma unroll
      for (int nb = 0; nb < 8; ++nb)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          S[nb][j] = exp2f(fmaf(S[nb][j], L2E, -mc[j >> 1]));   // exp2(-inf) = 0 for keys past the end
          sum[j >> 1] += S[nb][j];
        }
#pragma unroll
      for (int r = 0; r < 2; ++r) l[hh][r] = l[hh][r] * corr[r] + sum[r];
#pragma unroll
      for (int cb = 0; cb < 2; ++cb)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[hh][cb][j] *= corr[j >> 1];
      // O += P V: k-step kt = keys 16 kt .. + 15 (S blocks 2 kt, 2 kt + 1)
#pragma unroll
      for (int kt = 0; kt < 4; ++kt) {
        uint32_t ph[4], pm[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float* sv = S[2 * kt + (e >> 1)] + 2 * (e & 1);
          const uint32_t hw = pack_bf16x2(sv[0], sv[1]);
          ph[e] = hw;
          pm[e] = pack_bf16x2(sv[0] - __uint_as_float(hw << 16), sv[1] - __uint_as_float(hw & 0xFFFF0000u));
        }
#pragma unroll
        for (int cb = 0; cb < 2; ++cb) {
          // matrices: keys 0-7 hi, keys 8-15 hi, keys 0-7 mid, keys 8-15 mid of channels 16 h + 8 cb .. + 7
          const int key = 16 * kt + (lane & 7) + ((lane >> 3) & 1) * 8;
          const uint32_t addr = vs_addr + (uint32_t)(key * VSTR + (lane >> 4) * 64 + 8 * h + 4 * cb) * 4u;
          uint32_t vh0, vh1, vm0, vm1;
          asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
                       : "=r"(vh0), "=r"(vh1), "=r"(vm0), "=r"(vm1)
                       : "r"(addr));
          x_mma(acc[hh][cb], pm, vh0, vh1);
          x_mma(acc[hh][cb], ph, vm0, vm1);
          x_mma(acc[hh][cb], ph, vh0, vh1);
        }
      }
    }
    __syncthreads();                                   // stage (i & 1) is refilled by the next issue
  }
  // partials of rows g, g + 8: (m, l, 16 channels)
#pragma unroll
  for (int hh = 0; hh < 4; ++hh) {
    const int head = h0 + hh;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float lr = l[hh][r];
      lr += __shfl_xor_sync(0xffffffffu, lr, 1);
      lr += __shfl_xor_sync(0xffffffffu, lr, 2);
      const int qi = mt * XT_QT + q0 + g + 8 * r;
      if (qi < p.P) {
        float* pp = p.part + (((size_t)(b * p.heads + head) * p.nsplit + sp) * 18) * p.P + qi;
        if (t == 0) {
          pp[0] = m[hh][r];
          pp[p.P] = lr;
        }
#pragma unroll
        for (int cb = 0; cb < 2; ++cb) {
          const int c = 8 * cb + 2 * t;
          pp[(size_t)(2 + c) * p.P] = acc[hh][cb][2 * r];
          pp[(size_t)(3 + c) * p.P] = acc[hh][cb][2 * r + 1];
        }
      }
    }
  }
}

// merge of the key splits: one warp per (batch, head, query); lanes over the splits.  lse (optional, [B, Hh, P]): the
// row log-sum-exp M + log L of the logits, which the backward (xattn_bwd.cu) needs to recompute the probabilities
__global__ void __launch_bounds__(256)
xattn_combine_kernel(const float* __restrict__ part, float* __restrict__ out, float* __restrict__ lse, int B, int P, int C,
                     int Hh, int nsplit) {
  const int wid = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (wid >= B * Hh * P) return;
  const int qi = wid % P, head = (wid / P) % Hh, b = wid / (P * Hh);
  const float* pp = part + (size_t)(b * Hh + head) * nsplit * 18 * P + qi;
  const size_t ss = (size_t)18 * P;
  float M = -INFINITY;
  for (int s = lane; s < nsplit; s += 32) M = fmaxf(M, pp[s * ss]);
  M = warp_max(M);
  float L = 0.f, acc[16];
#pragma unroll
  for (int d = 0; d < 16; ++d) acc[d] = 0.f;
  for (int s = lane; s < nsplit; s += 32) {
    const float w = expf(pp[s * ss] - M);
    L += w * pp[s * ss + P];
#pragma unroll
    for (int d = 0; d < 16; ++d) acc[d] += w * pp[s * ss + (size_t)(2 + d) * P];
  }
  L = warp_sum(L);
  const float inv = 1.f / L;
  float mine = 0.f;
#pragma unroll
  for (int d = 0; d < 16; ++d) {
    const float a = warp_sum(acc[d]);
    if (lane == d) mine = a * inv;
  }
  if (lane < 16) out[(size_t)(b * P + qi) * C + head * 16 + lane] = mine;
  if (lse && lane == 0) lse[(size_t)(b * Hh + head) * P + qi] = M + logf(L);
}

// bf16 planes of fp32 rows: hi = bf16(x), mid = bf16(x - hi), lo = bf16(x - hi - mid); a plane holds 128 channels as 64
// words of packed pairs (lower channel in the low half)
__device__ __forceinline__ void split3(float a, float b, uint32_t& hi, uint32_t& mid, uint32_t& lo) {
  hi = pack_bf16x2(a, b);
  const float ra = a - __uint_as_float(hi << 16), rb = b - __uint_as_float(hi & 0xFFFF0000u);
  mid = pack_bf16x2(ra, rb);
  lo = pack_bf16x2(ra - __uint_as_float(mid << 16), rb - __uint_as_float(mid & 0xFFFF0000u));
}
// q rows [M, ld] -> [M, 192 words]: hi | mid | lo
__global__ void planes3_kernel(const float* __restrict__ x, int ld, uint32_t* __restrict__ out, int M) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;       // (row, word)
  if (i >= M * 64) return;
  const int r = i >> 6, wd = i & 63;
  uint32_t hi, mid, lo;
  split3(x[(size_t)r * ld + 2 * wd], x[(size_t)r * ld + 2 * wd + 1], hi, mid, lo);
  uint32_t* o = out + (size_t)r * 192;
  o[wd] = hi; o[64 + wd] = mid; o[128 + wd] = lo;
}
// kv rows [M, ld >= 256] (K = columns 0..127, V = 128..255) -> kplanes [M, 192 words] hi | mid | lo, vplanes [M, 128 words] hi | mid
__global__ void kv_planes_kernel(const float* __restrict__ kv, int ld, uint32_t* __restrict__ kp, uint32_t* __restrict__ vp,
                                 long long M) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // (row, word of 128)
  if (i >= M * 128) return;
  const long long r = i >> 7;
  const int wd = (int)(i & 127);
  const float2 v = *reinterpret_cast<const float2*>(kv + (size_t)r * ld + 2 * wd);
  uint32_t hi, mid, lo;
  split3(v.x, v.y, hi, mid, lo);
  if (wd < 64) {
    uint32_t* o = kp + (size_t)r * 192;
    o[wd] = hi; o[64 + wd] = mid; o[128 + wd] = lo;
  } else {
    uint32_t* o = vp + (size_t)r * 128;
    o[wd - 64] = hi; o[wd] = mid;
  }
}

bool g_xt_attr[64];

}  // namespace

extern "C" {

// Operand planes of the tensor-core cross attention.  q [M, ld] fp32 (128 channels, pre-scaled) -> qplanes [M, 192 words]
// (bf16 hi | mid | lo); kv [Mk, ld_kv >= 256] fp32 (K | V) -> kplanes [Mk, 192 words], vplanes [Mk, 128 words] (hi | mid).
int di_attn_planes_f32(const float* q, int ld_q, void* qplanes, int M, const float* kv, int ld_kv, void* kplanes,
                       void* vplanes, long long Mk, cudaStream_t stream) {
  DI_CHECK_ARG((q == nullptr || (qplanes && M > 0 && ld_q >= 128)) && (kv == nullptr || (kplanes && vplanes && Mk > 0 && ld_kv >= 256 &&
               ld_kv % 2 == 0 && ((uintptr_t)kv & 7) == 0)), "di_attn_planes_f32: bad argument");
  if (q) planes3_kernel<<<di_cdiv((long long)M * 64, 256), 256, 0, stream>>>(q, ld_q, reinterpret_cast<uint32_t*>(qplanes), M);
  if (kv)
    kv_planes_kernel<<<di_cdiv(Mk * 128, 256), 256, 0, stream>>>(kv, ld_kv, reinterpret_cast<uint32_t*>(kplanes),
                                                                 reinterpret_cast<uint32_t*>(vplanes), Mk);
  DI_CHECK_LAUNCH("di_attn_planes_f32");
  return DI_OK;
}

// Number of key splits di_xattn_tc_f32 uses for (B, HW): the caller sizes `part` as B * heads * nsplit * 18 * P floats.
int di_xattn_tc_splits(int B, int HW) {
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
      sms <= 0) {
    di_set_error("di_xattn_tc_splits: cannot query the SM count");
    return DI_ERR_LAUNCH;
  }
  int n = sms / (2 * (B > 0 ? B : 1));              // with the 4 query tiles of P = 200: two CTAs' worth of work per SM
  if (n < 1) n = 1;
  const int tiles = (HW + XT_KEYS - 1) / XT_KEYS;
  if (n > tiles) n = tiles;
  // every split must own at least one key tile
  while (n > 1 && (long long)(n - 1) * (((tiles + n - 1) / n) * XT_KEYS) >= HW) --n;
  return n;
}

}  // extern "C"

namespace {
int xattn_tc_run(const char* name, const void* q, const void* k, const void* v, float* part, float* out, float* lse, int B,
                 int P, int HW, int heads, cudaStream_t stream) {
  DI_CHECK_ARG(q && k && v && part && out && B > 0 && P > 0 && HW > 0, "%s: bad argument", name);
  if (heads != 8 || P > 256) {
    di_set_error("%s: supported configuration is 8 heads x 16 channels, P <= 256 (got heads=%d P=%d)", name, heads, P);
    return DI_ERR_UNSUPPORTED;
  }
  DI_CHECK_ARG((((uintptr_t)q | (uintptr_t)k | (uintptr_t)v) & 15) == 0, "%s: operands must be 16-byte aligned", name);
  int devid = 0;
  cudaGetDevice(&devid);
  if (devid < 0 || devid >= 64) {
    di_set_error("%s: device ordinal %d not supported", name, devid);
    return DI_ERR_UNSUPPORTED;
  }
  if (!g_xt_attr[devid]) {
    if (cudaFuncSetAttribute(xattn_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, XT_SMEM) != cudaSuccess) {
      di_set_error("%s: cannot reserve %d bytes of shared memory", name, XT_SMEM);
      return DI_ERR_LAUNCH;
    }
    g_xt_attr[devid] = true;
  }
  XtParams p{};
  p.P = P; p.HW = HW; p.heads = heads;
  p.nsplit = di_xattn_tc_splits(B, HW);
  if (p.nsplit < 0) return p.nsplit;
  const int tiles = (HW + XT_KEYS - 1) / XT_KEYS;
  p.chunk = ((tiles + p.nsplit - 1) / p.nsplit) * XT_KEYS;
  p.part = part;
  const int mtiles = (P + XT_QT - 1) / XT_QT;
  xattn_tc_kernel<<<dim3(p.nsplit, mtiles, B), XT_THREADS, XT_SMEM, stream>>>(static_cast<const uint32_t*>(q),
                                                                            static_cast<const uint32_t*>(k),
                                                                            static_cast<const uint32_t*>(v), p);
  DI_CHECK_LAUNCH(name);
  xattn_combine_kernel<<<di_cdiv((long long)B * heads * P, 8), 256, 0, stream>>>(part, out, lse, B, P, heads * 16, heads,
                                                                                 p.nsplit);
  DI_CHECK_LAUNCH(name);
  return DI_OK;
}
}  // namespace

extern "C" {

// q [B*P, 192 words], k [B*HW, 192 words], v [B*HW, 128 words]: the planes of di_attn_planes_f32; part: workspace
// (di_xattn_tc_splits), out [B*P, 128] fp32.  8 heads x 16 channels.
int di_xattn_tc_f32(const void* q, const void* k, const void* v, float* part, float* out, int B, int P, int HW, int heads,
                    cudaStream_t stream) {
  return xattn_tc_run("di_xattn_tc_f32", q, k, v, part, out, nullptr, B, P, HW, heads, stream);
}

// The same kernels, plus the row log-sum-exp of the logits: lse [B, heads, P] fp32.  out is bit-identical to
// di_xattn_tc_f32's.
int di_xattn_tc_lse_f32(const void* q, const void* k, const void* v, float* part, float* out, float* lse, int B, int P,
                        int HW, int heads, cudaStream_t stream) {
  DI_CHECK_ARG(lse, "di_xattn_tc_lse_f32: bad argument");
  return xattn_tc_run("di_xattn_tc_lse_f32", q, k, v, part, out, lse, B, P, HW, heads, stream);
}

}  // extern "C"
