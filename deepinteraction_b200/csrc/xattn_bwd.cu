// Backward of the query x BEV cross attention (xattn_tc.cu) on the tensor cores (mma.sync bf16 split, cp.async staging).
//
// Reference: TransformerDecoderLayer / multi_head_attention_forward, models/utils/decoder_utils.py:101-103, 466-493.
// Per batch element and head (P <= 256 queries, HW keys, d = 16), with A = softmax(Q K^T) (Q pre-scaled) and O = A V:
//   dV = A^T dO      dA = dO V^T      dS = A o (dA - D), D_i = sum_c dO_ic O_ic      dK = dS^T Q      dQ = dS K
// A is recomputed as exp(S - lse) from the row log-sum-exp the forward's split merge writes (di_xattn_tc_lse_f32).
//
// Operands: the bf16 planes of di_attn_planes_f32 (Q, K: hi | mid | lo; V: hi | mid) and dO split here into hi | mid.
// Split terms per product (smallest first; x = hi + mid (+ lo)):
//   S^T = K Q^T   six terms, the forward's logits product with the roles of the operands swapped
//   dA^T = V dO^T three terms (vh dOm, vm dOh, vh dOh)
//   dV += A^T dO  three terms (Am dOh, Ah dOm, Ah dOh)
//   dK += dS^T Q  three terms (dSm Qh, dSh Qm, dSh Qh)
//   dQ += dS K    three terms (dSm Kh, dSh Km, dSh Kh)
// i.e. 18 one-term products of the five 2 P HW d contractions.
//
// CTA = (key split, head, batch element); 8 warps.  The CTA keeps the Q and dO rows of its head for all P queries in
// shared memory and streams its contiguous key range in tiles of 64 keys through a double-buffered cp.async ring.  Warp w
// owns the query blocks w and w + 8 (16 queries each).  Per key tile and query block, the warp computes S^T, dA^T and dS^T
// as [16 keys x 16 queries] accumulator fragments, which are directly the A fragments of dV and dK (keys = rows).  For
// dQ the dS^T fragments are transposed in registers (movmatrix) into the A fragments of dS (queries = rows).  The warps'
// dK / dV partials of a tile are summed through shared memory in warp order and written once; dQ stays in registers
// across the key range and is written as a per-split partial, which xb_merge_kernel adds in split order.
// No floating-point atomics: two calls on the same inputs are bit-identical.
#include "tc_common.cuh"

namespace {
using namespace tc;

constexpr int XB_KEYS = 64;                       // keys per tile
constexpr int XB_THREADS = 256;
constexpr int XB_MAXP = 256;
constexpr int QSTR = 28;                          // words per query row of the Q tile (hi | mid | lo, 8 words each) and
constexpr int KSTR = 28;                          // of the K tile: conflict-free fragment loads and ldmatrix rows
constexpr int DSTR = 20, VSTR = 20;               // dO and V rows (hi | mid)
constexpr int RSTR = 40;                          // floats per key row of the dK | dV reduction buffer (32 used)
constexpr int XB_STAGE_WORDS = XB_KEYS * (KSTR + VSTR);
constexpr int XB_RED_FLOATS = 8 * XB_KEYS * RSTR;
constexpr float L2E = 1.4426950408889634f;

__host__ __device__ constexpr int xb_smem_bytes(int Pp) {
  return (Pp * (QSTR + DSTR) + 2 * Pp + 2 * XB_STAGE_WORDS + XB_RED_FLOATS) * 4;
}
static_assert(xb_smem_bytes(XB_MAXP) <= 232448, "xattn backward kernel exceeds the shared-memory limit");

__device__ __forceinline__ void b_mma(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void b_cp16(uint32_t dst, const void* src, bool ok) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(ok ? 16 : 0) : "memory");
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ uint32_t movm_t(uint32_t x) {
  uint32_t y;
  asm volatile("movmatrix.sync.aligned.m8n8.trans.b16 %0, %1;" : "=r"(y) : "r"(x));
  return y;
}
// fp32 pair -> (hi, mid) bf16x2 words
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& mid) {
  hi = pack_bf16x2(a, b);
  mid = pack_bf16x2(a - __uint_as_float(hi << 16), b - __uint_as_float(hi & 0xFFFF0000u));
}

struct XbParams {
  int B, P, HW, nsplit, chunk;
  const float* lse;      // [B, 8, P]
  const float* dterm;    // [B, 8, P]: D = sum_c dO O
  float* dk;             // dK rows [B*HW, ld_dkv] (head h: columns 16 h .. + 15)
  float* dv;
  int ld_dkv;
  float* dq_part;        // [nsplit, B*P, 128]
};

__global__ void __launch_bounds__(XB_THREADS, 1)
xattn_bwd_kernel(const uint32_t* __restrict__ qp, const uint32_t* __restrict__ kp, const uint32_t* __restrict__ vp,
                 const uint32_t* __restrict__ dop, const XbParams p) {
  extern __shared__ __align__(16) uint32_t xs[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int sp = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int P = p.P;
  const int Pp = (P + 15) & ~15, nqb = Pp >> 4;
  const int k_begin = sp * p.chunk, k_end = min(p.HW, k_begin + p.chunk);
  const int ntiles = (k_end - k_begin + XB_KEYS - 1) / XB_KEYS;      // >= 1 (the host sizes the splits)
  uint32_t* qs = xs;                                                  // [Pp][QSTR]
  uint32_t* ds = qs + Pp * QSTR;                                      // [Pp][DSTR]
  float* lse2 = reinterpret_cast<float*>(ds + Pp * DSTR);             // lse * log2(e); +inf past P
  float* dd = lse2 + Pp;                                              // D; 0 past P
  uint32_t* stages = reinterpret_cast<uint32_t*>(dd + Pp);            // 2 x (K [64][KSTR] | V [64][VSTR])
  float* red = reinterpret_cast<float*>(stages + 2 * XB_STAGE_WORDS); // [8 warps][64 keys][RSTR]
  const uint32_t qs_addr = smem_u32(qs), ds_addr = smem_u32(ds), st_addr = smem_u32(stages);

  // Q (hi | mid | lo) and dO (hi | mid) words 8h .. 8h + 7 of every plane; rows past P are zero
  for (int i = tid; i < Pp * 10; i += XB_THREADS) {
    const int r = i / 10, c = i % 10;
    const bool ok = r < P;
    const size_t row = (size_t)b * P + r;
    if (c < 6) {
      const int pl = c >> 1, half = c & 1;
      b_cp16(qs_addr + (uint32_t)(r * QSTR + 8 * pl + 4 * half) * 4u, ok ? qp + row * 192 + 64 * pl + 8 * h + 4 * half : qp, ok);
    } else {
      const int pl = (c - 6) >> 1, half = c & 1;
      b_cp16(ds_addr + (uint32_t)(r * DSTR + 8 * pl + 4 * half) * 4u, ok ? dop + row * 128 + 64 * pl + 8 * h + 4 * half : dop, ok);
    }
  }
  for (int i = tid; i < Pp; i += XB_THREADS) {
    const bool ok = i < P;
    const size_t o = ((size_t)b * 8 + h) * P + i;
    lse2[i] = ok ? p.lse[o] * L2E : INFINITY;
    dd[i] = ok ? p.dterm[o] : 0.f;
  }
  auto issue = [&](int i) {
    const uint32_t st = st_addr + (uint32_t)((i & 1) * XB_STAGE_WORDS) * 4u;
    const int row0 = k_begin + i * XB_KEYS;
    for (int j = tid; j < XB_KEYS * 10; j += XB_THREADS) {
      const int r = j / 10, c = j % 10;
      const int key = row0 + r;
      const bool ok = key < k_end;                    // keys at or past the split's end (and HW) are never read
      const size_t grow = (size_t)b * p.HW + key;
      if (c < 6) {
        const int pl = c >> 1, half = c & 1;
        b_cp16(st + (uint32_t)(r * KSTR + 8 * pl + 4 * half) * 4u, ok ? kp + grow * 192 + 64 * pl + 8 * h + 4 * half : kp, ok);
      } else {
        const int pl = (c - 6) >> 1, half = c & 1;
        b_cp16(st + (uint32_t)(XB_KEYS * KSTR + r * VSTR + 8 * pl + 4 * half) * 4u,
               ok ? vp + grow * 128 + 64 * pl + 8 * h + 4 * half : vp, ok);
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };

  float dq[2][2][4];
#pragma unroll
  for (int j = 0; j < 2; ++j)
#pragma unroll
    for (int cb = 0; cb < 2; ++cb) dq[j][cb][0] = dq[j][cb][1] = dq[j][cb][2] = dq[j][cb][3] = 0.f;

  issue(0);
  for (int i = 0; i < ntiles; ++i) {
    if (i + 1 < ntiles) {
      issue(i + 1);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    const int nvalid = min(XB_KEYS, k_end - (k_begin + i * XB_KEYS));
    const uint32_t* ks = stages + (i & 1) * XB_STAGE_WORDS;
    const uint32_t* vs = ks + XB_KEYS * KSTR;
    const uint32_t ks_addr = st_addr + (uint32_t)((i & 1) * XB_STAGE_WORDS) * 4u;
    float dk[4][2][4], dv[4][2][4];
#pragma unroll
    for (int kt = 0; kt < 4; ++kt)
#pragma unroll
      for (int cb = 0; cb < 2; ++cb)
#pragma unroll
        for (int e = 0; e < 4; ++e) dk[kt][cb][e] = dv[kt][cb][e] = 0.f;

#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int qb = warp + 8 * j;
      if (qb < nqb) {
        const int q0 = 16 * qb;
        // B fragments (n = query q0 + 8 nb + g, k = channel pairs t, t + 4): Q planes hi, mid, lo; dO planes hi, mid
        uint32_t qf[2][3][2], of[2][2][2];
        float l2[2][2], dn[2][2];
#pragma unroll
        for (int nb = 0; nb < 2; ++nb) {
          const uint32_t* qr = qs + (q0 + 8 * nb + g) * QSTR + t;
          const uint32_t* orow = ds + (q0 + 8 * nb + g) * DSTR + t;
#pragma unroll
          for (int pl = 0; pl < 3; ++pl) { qf[nb][pl][0] = qr[8 * pl]; qf[nb][pl][1] = qr[8 * pl + 4]; }
#pragma unroll
          for (int pl = 0; pl < 2; ++pl) { of[nb][pl][0] = orow[8 * pl]; of[nb][pl][1] = orow[8 * pl + 4]; }
#pragma unroll
          for (int e = 0; e < 2; ++e) {          // the accumulator columns of this lane: queries q0 + 8 nb + 2t + e
            l2[nb][e] = lse2[q0 + 8 * nb + 2 * t + e];
            dn[nb][e] = dd[q0 + 8 * nb + 2 * t + e];
          }
        }
#pragma unroll
        for (int kt = 0; kt < 4; ++kt) {
          const int k0 = 16 * kt;
          // A fragments (rows = keys k0 + g, k0 + g + 8; k = channel pairs t, t + 4): K hi, mid, lo; V hi, mid
          uint32_t ka[3][4], va[2][4];
          {
            const uint32_t* kr0 = ks + (k0 + g) * KSTR + t;
            const uint32_t* kr1 = kr0 + 8 * KSTR;
#pragma unroll
            for (int pl = 0; pl < 3; ++pl) {
              ka[pl][0] = kr0[8 * pl]; ka[pl][1] = kr1[8 * pl]; ka[pl][2] = kr0[8 * pl + 4]; ka[pl][3] = kr1[8 * pl + 4];
            }
            const uint32_t* vr0 = vs + (k0 + g) * VSTR + t;
            const uint32_t* vr1 = vr0 + 8 * VSTR;
#pragma unroll
            for (int pl = 0; pl < 2; ++pl) {
              va[pl][0] = vr0[8 * pl]; va[pl][1] = vr1[8 * pl]; va[pl][2] = vr0[8 * pl + 4]; va[pl][3] = vr1[8 * pl + 4];
            }
          }
          // S^T and dA^T [16 keys x 8 queries] per nb; element e: key k0 + g + 8 (e >> 1), query q0 + 8 nb + 2t + (e & 1)
          float s[2][4], da[2][4];
#pragma unroll
          for (int nb = 0; nb < 2; ++nb) {
            s[nb][0] = s[nb][1] = s[nb][2] = s[nb][3] = 0.f;
            b_mma(s[nb], ka[0], qf[nb][2][0], qf[nb][2][1]);      // smallest terms first, as the forward
            b_mma(s[nb], ka[2], qf[nb][0][0], qf[nb][0][1]);
            b_mma(s[nb], ka[1], qf[nb][1][0], qf[nb][1][1]);
            b_mma(s[nb], ka[0], qf[nb][1][0], qf[nb][1][1]);
            b_mma(s[nb], ka[1], qf[nb][0][0], qf[nb][0][1]);
            b_mma(s[nb], ka[0], qf[nb][0][0], qf[nb][0][1]);
            da[nb][0] = da[nb][1] = da[nb][2] = da[nb][3] = 0.f;
            b_mma(da[nb], va[0], of[nb][1][0], of[nb][1][1]);
            b_mma(da[nb], va[1], of[nb][0][0], of[nb][0][1]);
            b_mma(da[nb], va[0], of[nb][0][0], of[nb][0][1]);
          }
          // A = exp(S - lse) (0 for keys past the tile's end), dS = A (dA - D)
#pragma unroll
          for (int nb = 0; nb < 2; ++nb)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const int key = k0 + g + 8 * (e >> 1);
              const float a = key < nvalid ? exp2f(fmaf(s[nb][e], L2E, -l2[nb][e & 1])) : 0.f;
              s[nb][e] = a;
              da[nb][e] = a * (da[nb][e] - dn[nb][e & 1]);
            }
          // A fragments (rows = keys, k = queries) of A^T and dS^T, split hi | mid
          uint32_t ah[4], am[4], gh[4], gm[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float* sv = s[e >> 1] + 2 * (e & 1);
            const float* dv_ = da[e >> 1] + 2 * (e & 1);
            split2(sv[0], sv[1], ah[e], am[e]);
            split2(dv_[0], dv_[1], gh[e], gm[e]);
          }
#pragma unroll
          for (int cb = 0; cb < 2; ++cb) {
            // B fragments (k = queries, n = channels 8 cb .. + 7) by ldmatrix.trans: queries q0 .. + 7 hi, q0 + 8 .. + 15
            // hi, q0 .. + 7 mid, q0 + 8 .. + 15 mid
            const int row = q0 + (lane & 7) + ((lane >> 3) & 1) * 8;
            uint32_t oh0, oh1, om0, om1, qh0, qh1, qm0, qm1;
            ldsm_x4_t(ds_addr + (uint32_t)(row * DSTR + (lane >> 4) * 8 + 4 * cb) * 4u, oh0, oh1, om0, om1);
            ldsm_x4_t(qs_addr + (uint32_t)(row * QSTR + (lane >> 4) * 8 + 4 * cb) * 4u, qh0, qh1, qm0, qm1);
            b_mma(dv[kt][cb], am, oh0, oh1);
            b_mma(dv[kt][cb], ah, om0, om1);
            b_mma(dv[kt][cb], ah, oh0, oh1);
            b_mma(dk[kt][cb], gm, qh0, qh1);
            b_mma(dk[kt][cb], gh, qm0, qm1);
            b_mma(dk[kt][cb], gh, qh0, qh1);
          }
          // dQ += dS K.  The 8 x 8 blocks of the dS^T fragment (keys 0-7 | 8-15) x (queries 0-7 | 8-15) transposed give the
          // A fragment of dS (rows = queries, k = keys): a0 = T(keys 0-7, q 0-7), a1 = T(keys 0-7, q 8-15), a2 = T(keys
          // 8-15, q 0-7), a3 = T(keys 8-15, q 8-15)
          uint32_t th[4], tm[4];
          th[0] = movm_t(gh[0]); th[1] = movm_t(gh[2]); th[2] = movm_t(gh[1]); th[3] = movm_t(gh[3]);
          tm[0] = movm_t(gm[0]); tm[1] = movm_t(gm[2]); tm[2] = movm_t(gm[1]); tm[3] = movm_t(gm[3]);
#pragma unroll
          for (int cb = 0; cb < 2; ++cb) {
            const int row = k0 + (lane & 7) + ((lane >> 3) & 1) * 8;
            uint32_t kh0, kh1, km0, km1;
            ldsm_x4_t(ks_addr + (uint32_t)(row * KSTR + (lane >> 4) * 8 + 4 * cb) * 4u, kh0, kh1, km0, km1);
            b_mma(dq[j][cb], tm, kh0, kh1);
            b_mma(dq[j][cb], th, km0, km1);
            b_mma(dq[j][cb], th, kh0, kh1);
          }
        }
      }
    }
    // dK | dV of the tile: the eight warps' partials summed in warp order, written once
    float* rw = red + warp * XB_KEYS * RSTR;
#pragma unroll
    for (int kt = 0; kt < 4; ++kt)
#pragma unroll
      for (int cb = 0; cb < 2; ++cb)
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          float* o = rw + (16 * kt + g + 8 * r) * RSTR + 8 * cb + 2 * t;
          *reinterpret_cast<float2*>(o) = make_float2(dk[kt][cb][2 * r], dk[kt][cb][2 * r + 1]);
          *reinterpret_cast<float2*>(o + 16) = make_float2(dv[kt][cb][2 * r], dv[kt][cb][2 * r + 1]);
        }
    __syncthreads();
    for (int idx = tid; idx < XB_KEYS * 8; idx += XB_THREADS) {
      const int r = idx >> 3, c4 = idx & 7;
      if (r < nvalid) {
        float4 acc = *reinterpret_cast<const float4*>(red + r * RSTR + 4 * c4);
#pragma unroll
        for (int w = 1; w < 8; ++w) {
          const float4 x = *reinterpret_cast<const float4*>(red + (w * XB_KEYS + r) * RSTR + 4 * c4);
          acc.x += x.x; acc.y += x.y; acc.z += x.z; acc.w += x.w;
        }
        const size_t key = (size_t)b * p.HW + k_begin + i * XB_KEYS + r;
        float* dst = (c4 < 4 ? p.dk : p.dv) + key * p.ld_dkv + 16 * h + 4 * (c4 & 3);
        *reinterpret_cast<float4*>(dst) = acc;
      }
    }
    __syncthreads();                                   // stage (i & 1) and the reduction buffer are reused
  }
  // dQ partial of this split: rows q0 + g (+ 8), channels 16 h + 8 cb + 2t
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int qb = warp + 8 * j;
    if (qb < nqb) {
#pragma unroll
      for (int cb = 0; cb < 2; ++cb)
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int q = 16 * qb + g + 8 * r;
          if (q < P) {
            float* o = p.dq_part + (((size_t)sp * p.B + b) * P + q) * 128 + 16 * h + 8 * cb + 2 * t;
            *reinterpret_cast<float2*>(o) = make_float2(dq[j][cb][2 * r], dq[j][cb][2 * r + 1]);
          }
        }
    }
  }
}

// dO rows [B*P, ld] -> planes [B*P, 128 words] (hi | mid) and D [B, 8, P] = per head sum_c dO O; one thread per (row, head)
__global__ void xb_prep_kernel(const float* __restrict__ out, const float* __restrict__ dout, int ld_dout,
                               uint32_t* __restrict__ dop, float* __restrict__ dterm, int M, int P) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * 8) return;
  const int r = i >> 3, h = i & 7;
  const float* o = out + (size_t)r * 128 + 16 * h;
  const float* d = dout + (size_t)r * ld_dout + 16 * h;
  float acc = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) {
    const float a = d[2 * w], b = d[2 * w + 1];
    acc = fmaf(a, o[2 * w], acc);
    acc = fmaf(b, o[2 * w + 1], acc);
    uint32_t hi, mid;
    split2(a, b, hi, mid);
    dop[(size_t)r * 128 + 8 * h + w] = hi;
    dop[(size_t)r * 128 + 64 + 8 * h + w] = mid;
  }
  dterm[((size_t)(r / P) * 8 + h) * P + r % P] = acc;
}

// dQ = sum of the per-split partials, in split order
__global__ void xb_merge_kernel(const float4* __restrict__ part, float4* __restrict__ dq, long long n4, int nsplit) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  float4 acc = part[i];
  for (int s = 1; s < nsplit; ++s) {
    const float4 x = part[(size_t)s * n4 + i];
    acc.x += x.x; acc.y += x.y; acc.z += x.z; acc.w += x.w;
  }
  dq[i] = acc;
}

bool g_xb_attr[64];

int xb_splits(int B, int HW) {
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
      sms <= 0) {
    di_set_error("di_xattn_bwd: cannot query the SM count");
    return DI_ERR_LAUNCH;
  }
  int n = (2 * sms) / (8 * (B > 0 ? B : 1));       // 8 head CTAs per split: about two CTAs per SM
  if (n < 1) n = 1;
  const int tiles = (HW + XB_KEYS - 1) / XB_KEYS;
  if (n > tiles) n = tiles;
  while (n > 1 && (long long)(n - 1) * (((tiles + n - 1) / n) * XB_KEYS) >= HW) --n;   // every split owns >= 1 tile
  return n;
}

}  // namespace

extern "C" {

// Size in floats of the workspace of di_xattn_bwd_f32 for (B, P, HW): dO planes, D and the per-split dQ partials.
int di_xattn_bwd_workspace(int B, int P, int HW) {
  DI_CHECK_ARG(B > 0 && P > 0 && HW > 0, "di_xattn_bwd_workspace: bad argument");
  const int n = xb_splits(B, HW);
  if (n < 0) return n;
  const long long floats = (long long)B * P * 128 + (long long)B * 8 * P + (long long)n * B * P * 128;
  DI_CHECK_ARG(floats < (1ll << 31), "di_xattn_bwd_workspace: shape too large");
  return (int)floats;
}

// Gradient of di_xattn_tc_lse_f32.  q / k / v: the planes of di_attn_planes_f32; out [B*P, 128] and lse [B, 8, P]: the
// forward's outputs; dout [B*P, ld_dout]: gradient of out.  -> dq [B*P, 128] (w.r.t. the pre-scaled queries), dk / dv:
// rows [B*HW, ld_dkv] (only the rows below HW of each batch element are written).  work: di_xattn_bwd_workspace floats.
int di_xattn_bwd_f32(const void* q, const void* k, const void* v, const float* out, const float* dout, int ld_dout,
                     const float* lse, float* work, float* dq, float* dk, float* dv, int ld_dkv, int B, int P, int HW,
                     int heads, cudaStream_t stream) {
  DI_CHECK_ARG(q && k && v && out && dout && lse && work && dq && dk && dv && B > 0 && P > 0 && HW > 0 && ld_dout >= 128 &&
                   ld_dkv >= 128 && ld_dkv % 4 == 0,
               "di_xattn_bwd_f32: bad argument");
  if (heads != 8 || P > XB_MAXP) {
    di_set_error("di_xattn_bwd_f32: supported configuration is 8 heads x 16 channels, P <= 256 (got heads=%d P=%d)", heads, P);
    return DI_ERR_UNSUPPORTED;
  }
  DI_CHECK_ARG((((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)dq | (uintptr_t)dk | (uintptr_t)dv | (uintptr_t)work) &
                15) == 0,
               "di_xattn_bwd_f32: operands must be 16-byte aligned");
  int devid = 0;
  cudaGetDevice(&devid);
  if (devid < 0 || devid >= 64) {
    di_set_error("di_xattn_bwd_f32: device ordinal %d not supported", devid);
    return DI_ERR_UNSUPPORTED;
  }
  if (!g_xb_attr[devid]) {
    if (cudaFuncSetAttribute(xattn_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, xb_smem_bytes(XB_MAXP)) !=
        cudaSuccess) {
      di_set_error("di_xattn_bwd_f32: cannot reserve %d bytes of shared memory", xb_smem_bytes(XB_MAXP));
      return DI_ERR_LAUNCH;
    }
    g_xb_attr[devid] = true;
  }
  const int nsplit = xb_splits(B, HW);
  if (nsplit < 0) return nsplit;
  const int tiles = (HW + XB_KEYS - 1) / XB_KEYS;
  const int M = B * P;
  uint32_t* dop = reinterpret_cast<uint32_t*>(work);
  float* dterm = work + (size_t)M * 128;
  float* part = dterm + (size_t)M * 8;                 // M * 8 floats: keeps 16-byte alignment
  xb_prep_kernel<<<di_cdiv((long long)M * 8, 256), 256, 0, stream>>>(out, dout, ld_dout, dop, dterm, M, P);
  DI_CHECK_LAUNCH("di_xattn_bwd_f32 (prep)");
  XbParams p{};
  p.B = B; p.P = P; p.HW = HW; p.nsplit = nsplit;
  p.chunk = ((tiles + nsplit - 1) / nsplit) * XB_KEYS;
  p.lse = lse; p.dterm = dterm; p.dk = dk; p.dv = dv; p.ld_dkv = ld_dkv; p.dq_part = part;
  const int Pp = (P + 15) & ~15;
  xattn_bwd_kernel<<<dim3(nsplit, 8, B), XB_THREADS, xb_smem_bytes(Pp), stream>>>(
      static_cast<const uint32_t*>(q), static_cast<const uint32_t*>(k), static_cast<const uint32_t*>(v), dop, p);
  DI_CHECK_LAUNCH("di_xattn_bwd_f32");
  const long long n4 = (long long)M * 32;
  xb_merge_kernel<<<di_cdiv(n4, 256), 256, 0, stream>>>(reinterpret_cast<const float4*>(part), reinterpret_cast<float4*>(dq),
                                                         n4, nsplit);
  DI_CHECK_LAUNCH("di_xattn_bwd_f32 (merge)");
  return DI_OK;
}

}  // extern "C"
