// 9x9 (k x k) local-window attention: logits = q . k over the window, softmax(logits/sqrt(C)),
// out = sum_t w_t v_t -- the fused equivalent of the reference's
//   similarFunction -> softmax -> weightingFunction
// (projects/mmdet3d_plugin/models/utils/encoder_utils.py:132-134; kernels
//  models/utils/ops/locatt_ops/kernels.cuh:4-42 `cc2k`, :44-80 `ck2c_ori`).
//
// Semantics kept from the reference kernels: out-of-image taps have logit 0 and STILL take
// softmax mass; their values are skipped.  Both fall out of zero-filling the halo.
//
// Which kernel serves which path (q / k / v / out are pixel-major NHWC rows with a per-pixel stride):
//   lcab_window_tc_kernel    planar bf16 hi | mid operands (di_lcab_window_tc_f32), C = 128: the product path, fed by
//                            the fused projections of lcab_proj.cu (di_lcab_forward_f32).
//   lcab_window_pre_kernel   interleaved pre-split operands (di_lcab_window_pre_f32) for the other C % 64 == 0, e.g.
//                            C = 64, or C = 256 / 512 in config 5: the dense layers' epilogue writes them.
//   lcab_window_bf16_kernel  fp32 operands split in shared memory (di_lcab_window_f32): the other C % 32 == 0, or when
//                            the projections do not pre-split.
//   lcab_window_kernel<KS>   FFMA (di_lcab_window_f32): ks = 3, or C % 32 != 0.
// The three bf16-split kernels run one per-warp core (window_core below) and differ only in how the operands reach
// shared memory and where a fragment lives there, so they are bit-identical on the same hi / mid words.
#include "tc_common.cuh"

namespace {

constexpr int TQ = 16;        // query tile edge
constexpr int CC = 16;        // channels per chunk
constexpr int PSTR = CC + 4;  // padded pixel stride in smem (floats): conflict-free LDS.128

__device__ __forceinline__ void cp_async16(float* smem_dst, const float* gsrc, bool valid) {
  unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  int sz = valid ? 16 : 0;  // src-size 0 => 16 bytes of zero fill
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(d), "l"(gsrc), "r"(sz));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

// ------------------------------------------------------------------------------------------------
// FFMA kernel.  One CTA = 16x16 queries; the (16+2r)^2 halo tile of k (then v) streams through shared memory in
// 16-channel chunks with cp.async double buffering; each thread keeps the k*k logits of its query in registers, so
// logits/probabilities never touch HBM (the reference writes and re-reads 2*N*81*4 bytes per call).
// ------------------------------------------------------------------------------------------------
template <int KS>
__global__ void __launch_bounds__(TQ * TQ, 1)
lcab_window_kernel(const float* __restrict__ q, int ldq, const float* __restrict__ k, int ldk,
                   const float* __restrict__ v, int ldv, float* __restrict__ out, int ldo, int H, int W, int C,
                   float scale) {
  constexpr int R = KS / 2;
  constexpr int TH = TQ + 2 * R;  // halo tile edge
  constexpr int NPIX = TH * TH;
  extern __shared__ __align__(16) float smem[];  // [2][NPIX][PSTR]
  const int t = threadIdx.x;
  const int tx = t % TQ, ty = t / TQ;
  const int x0 = blockIdx.x * TQ, y0 = blockIdx.y * TQ, n = blockIdx.z;
  const int qx = x0 + tx, qy = y0 + ty;
  const bool qin = qx < W && qy < H;
  const size_t img_off = (size_t)n * H * W;
  const int nchunk = C / CC;
  const int nstage = 2 * nchunk;  // k chunks then v chunks

  auto issue = [&](int stage) {
    const float* src = stage < nchunk ? k : v;
    const int ld = stage < nchunk ? ldk : ldv;
    const int c0 = (stage < nchunk ? stage : stage - nchunk) * CC;
    float* dst = smem + (stage & 1) * (NPIX * PSTR);
    for (int i = t; i < NPIX * (CC / 4); i += TQ * TQ) {
      int px = i / (CC / 4), c4 = i % (CC / 4);
      int gy = y0 - R + px / TH, gx = x0 - R + px % TH;
      bool ok = gy >= 0 && gy < H && gx >= 0 && gx < W;
      const float* g = ok ? src + (img_off + (size_t)gy * W + gx) * ld + c0 + c4 * 4 : src;
      cp_async16(dst + px * PSTR + c4 * 4, g, ok);
    }
    cp_async_commit();
  };

  float lg[KS * KS];
#pragma unroll
  for (int i = 0; i < KS * KS; ++i) lg[i] = 0.f;

  issue(0);
  for (int stage = 0; stage < nstage; ++stage) {
    if (stage + 1 < nstage) {
      issue(stage + 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const float* tile = smem + (stage & 1) * (NPIX * PSTR);
    if (stage < nchunk) {
      // ---- logits += q[chunk] . k[chunk] over the window
      float4 qv[CC / 4];
#pragma unroll
      for (int j = 0; j < CC / 4; ++j)
        qv[j] = qin ? ldg4(q + (img_off + (size_t)qy * W + qx) * ldq + stage * CC + j * 4) : make_float4(0, 0, 0, 0);
#pragma unroll
      for (int dy = 0; dy < KS; ++dy)
#pragma unroll
        for (int dx = 0; dx < KS; ++dx) {
          const float* kp = tile + ((ty + dy) * TH + tx + dx) * PSTR;
          float s = lg[dy * KS + dx];
#pragma unroll
          for (int j = 0; j < CC / 4; ++j) {
            float4 kv = *reinterpret_cast<const float4*>(kp + j * 4);
            s = fmaf(qv[j].x, kv.x, s);
            s = fmaf(qv[j].y, kv.y, s);
            s = fmaf(qv[j].z, kv.z, s);
            s = fmaf(qv[j].w, kv.w, s);
          }
          lg[dy * KS + dx] = s;
        }
      if (stage == nchunk - 1) {
        // ---- softmax over the k*k taps (out-of-image taps carry logit 0)
        float m = -INFINITY;
#pragma unroll
        for (int i = 0; i < KS * KS; ++i) {
          lg[i] *= scale;
          m = fmaxf(m, lg[i]);
        }
        float sum = 0.f;
#pragma unroll
        for (int i = 0; i < KS * KS; ++i) {
          lg[i] = expf(lg[i] - m);
          sum += lg[i];
        }
        float inv = 1.f / sum;
#pragma unroll
        for (int i = 0; i < KS * KS; ++i) lg[i] *= inv;
      }
    } else {
      // ---- out[chunk] = sum_t w_t v_t[chunk]
      float4 acc[CC / 4];
#pragma unroll
      for (int j = 0; j < CC / 4; ++j) acc[j] = make_float4(0, 0, 0, 0);
#pragma unroll
      for (int dy = 0; dy < KS; ++dy)
#pragma unroll
        for (int dx = 0; dx < KS; ++dx) {
          const float* vp = tile + ((ty + dy) * TH + tx + dx) * PSTR;
          float w = lg[dy * KS + dx];
#pragma unroll
          for (int j = 0; j < CC / 4; ++j) {
            float4 vv = *reinterpret_cast<const float4*>(vp + j * 4);
            acc[j].x = fmaf(w, vv.x, acc[j].x);
            acc[j].y = fmaf(w, vv.y, acc[j].y);
            acc[j].z = fmaf(w, vv.z, acc[j].z);
            acc[j].w = fmaf(w, vv.w, acc[j].w);
          }
        }
      if (qin) {
        float* o = out + (img_off + (size_t)qy * W + qx) * ldo + (stage - nchunk) * CC;
#pragma unroll
        for (int j = 0; j < CC / 4; ++j) *reinterpret_cast<float4*>(o + j * 4) = acc[j];
      }
    }
    __syncthreads();  // the buffer just consumed is refilled by the next iteration's issue()
  }
}

// ------------------------------------------------------------------------------------------------
// window_core: the per-warp math of the three bf16-split tensor-core kernels.
// One CTA = 8 query rows x 16 query columns; a warp owns a 2 x 8 patch of queries (M = 16) at (wy, wx) of the tile.
// Every operand x is split into hi = bf16(x), mid = bf16(x - hi) (16 mantissa bits kept, product error ~1e-5), and each
// contraction runs on mma.sync.m16n8k16 bf16 as the three products mid.hi, hi.mid, hi.hi:
//   S[16 x (10 rows x 16 cols)] = Q K^T  -> 20 key blocks of 8 (block b = halo row b / 2, column block b % 2),
//                                           accumulated over 32-channel chunks in k16 steps
//   softmax over the 81 in-window keys of each query, entirely in registers (quad shuffles)
//   O[16 x C] = P V                       -> the S accumulator fragments are re-used as the A operand: for halo row r,
//                                            k16 = the 16 halo columns wx .. wx+15
// Band structure: a query uses 9 of the 16 key columns and 9 of the 10 key rows of its patch (1.98x padding).
// The issue order of the mma.sync below is part of the result: per accumulator it fixes the summation order (so the
// bits), and product-major order across accumulators keeps consecutive mma.sync off one accumulator (the legacy
// tensor path has a long issue-to-result latency; 3 back-to-back products into one fragment serialise on it).
// ------------------------------------------------------------------------------------------------
constexpr int MQ_ROWS = 8, MQ_COLS = 16, MCH = 32;                  // query tile, channels per chunk
constexpr int MT_ROWS = MQ_ROWS + 8, MT_COLS = MQ_COLS + 8;          // key / value halo tile
constexpr int BSTR = 40;                                             // words per pixel of the interleaved K / Q rows
constexpr int BKV_WORDS = MT_ROWS * MT_COLS * BSTR;                  // 15360
constexpr int BQ_WORDS = MQ_ROWS * MQ_COLS * BSTR;                   // 5120
constexpr int BSTAGE_WORDS = BKV_WORDS + BQ_WORDS;                   // 20480 (80 KB)
constexpr int VPSTR = 72;                                            // words per key pair of the packed V chunk
constexpr int VPK_WORDS = MT_ROWS * (MT_COLS / 2) * VPSTR;           // 13824 (54 KB)
constexpr int VSTR2 = 36;                                            // pre-split V pixel stride: 8 ldmatrix rows -> 32 banks

__device__ __forceinline__ uint32_t pack_bf16x2(float lo_elem, float hi_elem) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi_elem), "f"(lo_elem));
  return r;
}
// (x0, x1) -> hi = bf16x2(x0, x1), mid = bf16x2(x0 - hi0, x1 - hi1)
__device__ __forceinline__ uint2 split_bf16x2(float x0, float x1) {
  const uint32_t h = pack_bf16x2(x0, x1);
  return make_uint2(h, pack_bf16x2(x0 - __uint_as_float(h << 16), x1 - __uint_as_float(h & 0xFFFF0000u)));
}
__device__ __forceinline__ void mma_bf16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

template <int N>
__device__ __forceinline__ void zero_acc(float (&acc)[N][4]) {
#pragma unroll
  for (int b = 0; b < N; ++b) acc[b][0] = acc[b][1] = acc[b][2] = acc[b][3] = 0.f;
}

// S += Q K^T for one k16 step.  ah / am: the Q A fragment (hi, mid).  kfrag(b, b0, b1) loads the B fragment of key
// block b: b0 = its first k half (k = t, hi in .x, mid in .y), b1 = its second (k = t + 4).
template <class KFrag>
__device__ __forceinline__ void qk_step(float (&S)[20][4], const uint32_t (&ah)[4], const uint32_t (&am)[4], KFrag kfrag) {
  // 4 key blocks at a time, product-major
#pragma unroll
  for (int r2 = 0; r2 < 5; ++r2) {
    uint2 b0[4], b1[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) kfrag(r2 * 4 + u, b0[u], b1[u]);
#pragma unroll
    for (int u = 0; u < 4; ++u) mma_bf16(S[r2 * 4 + u], am, b0[u].x, b1[u].x);
#pragma unroll
    for (int u = 0; u < 4; ++u) mma_bf16(S[r2 * 4 + u], ah, b0[u].y, b1[u].y);
#pragma unroll
    for (int u = 0; u < 4; ++u) mma_bf16(S[r2 * 4 + u], ah, b0[u].x, b1[u].x);
  }
}

// Masked softmax over the 81 in-window keys of the warp's two query rows (fragment rows g: query row wy, g + 8: row
// wy + 1), then P = softmax(S) packed as the bf16 hi / mid A fragments of P V: for halo row r, k = the 16 halo columns
// wx .. wx+15 (block cb = 0 -> k 0..7, cb = 1 -> 8..15).
__device__ __forceinline__ void window_softmax(float (&S)[20][4], float scale, int g, int t, uint32_t (&Ph)[10][4],
                                               uint32_t (&Pm)[10][4]) {
  float m0 = -INFINITY, m1 = -INFINITY;
#pragma unroll
  for (int b = 0; b < 20; ++b) {
    const int r = b >> 1, cb = b & 1;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int d = cb * 8 + 2 * t + j - g;               // key column - query column + 4
      const bool colok = d >= 0 && d <= 8;
      S[b][j] = (colok && r <= 8) ? S[b][j] * scale : -INFINITY;
      S[b][2 + j] = (colok && r >= 1) ? S[b][2 + j] * scale : -INFINITY;
      m0 = fmaxf(m0, S[b][j]);
      m1 = fmaxf(m1, S[b][2 + j]);
    }
  }
  m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1));
  m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
  m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1));
  m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
  float s0 = 0.f, s1 = 0.f;
#pragma unroll
  for (int b = 0; b < 20; ++b)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      S[b][j] = expf(S[b][j] - m0);            // exp(-inf) = 0 for out-of-window entries
      S[b][2 + j] = expf(S[b][2 + j] - m1);
      s0 += S[b][j];
      s1 += S[b][2 + j];
    }
  s0 += __shfl_xor_sync(0xffffffffu, s0, 1);
  s0 += __shfl_xor_sync(0xffffffffu, s0, 2);
  s1 += __shfl_xor_sync(0xffffffffu, s1, 1);
  s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
  const float i0 = 1.f / s0, i1 = 1.f / s1;
#pragma unroll
  for (int r = 0; r < 10; ++r)
#pragma unroll
    for (int cb = 0; cb < 2; ++cb) {
      const uint2 lo = split_bf16x2(S[r * 2 + cb][0] * i0, S[r * 2 + cb][1] * i0);   // row g
      const uint2 hi = split_bf16x2(S[r * 2 + cb][2] * i1, S[r * 2 + cb][3] * i1);   // row g + 8
      Ph[r][cb * 2] = lo.x; Pm[r][cb * 2] = lo.y;
      Ph[r][cb * 2 + 1] = hi.x; Pm[r][cb * 2 + 1] = hi.y;
    }
}

// O += P V for one halo row (k16 = its 16 keys).  b0[nb] / b1[nb]: the B fragment of channel block nb for keys 0-7 /
// 8-15, hi in .x, mid in .y.
__device__ __forceinline__ void pv_row(float (&O)[MCH / 8][4], const uint32_t (&Ph)[4], const uint32_t (&Pm)[4],
                                       const uint2 (&b0)[MCH / 8], const uint2 (&b1)[MCH / 8]) {
#pragma unroll
  for (int nb = 0; nb < MCH / 8; ++nb) mma_bf16(O[nb], Pm, b0[nb].x, b1[nb].x);
#pragma unroll
  for (int nb = 0; nb < MCH / 8; ++nb) mma_bf16(O[nb], Ph, b0[nb].y, b1[nb].y);
#pragma unroll
  for (int nb = 0; nb < MCH / 8; ++nb) mma_bf16(O[nb], Ph, b0[nb].x, b1[nb].x);
}

// V B fragments of one halo row by ldmatrix.x4.trans: the lane's row address picks keys 0-7 / 8-15 (matrices 0 / 1,
// hi) and their mid parts (matrices 2 / 3), so the [key][channel] rows arrive as (k = key pair, n = channel) fragments.
__device__ __forceinline__ void ldsm_v(uint32_t addr, uint2& b0, uint2& b1) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(b0.x), "=r"(b1.x), "=r"(b0.y), "=r"(b1.y)
               : "r"(addr));
}

// out = the warp's 2 x 8 patch of one 32-channel chunk: query (qy0 + half, qx) of image n, channels c + nb * 8 + 2t
__device__ __forceinline__ void store_patch(const float (&O)[MCH / 8][4], float* __restrict__ out, int ldo,
                                            int n, int H, int W, int qy0, int qx, int c, int t) {
  if (qx < W) {
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int qy = qy0 + half;
      if (qy < H) {
        float* o = out + ((size_t)(n * H + qy) * W + qx) * ldo + c + 2 * t;
#pragma unroll
        for (int nb = 0; nb < MCH / 8; ++nb)
          *reinterpret_cast<float2*>(o + nb * 8) = make_float2(O[nb][half * 2], O[nb][half * 2 + 1]);
      }
    }
  }
}

// S += Q K^T over one 32-channel chunk held as interleaved (hi, mid) words, pixel stride BSTR: kw = the 16 x 24 K halo,
// qw = the warp's first query pixel in the 8 x 16 Q tile
__device__ __forceinline__ void qk_chunk_interleaved(float (&S)[20][4], const uint32_t* kw, const uint32_t* qw, int wy,
                                                     int wx, int g, int t) {
#pragma unroll
  for (int ks = 0; ks < MCH / 16; ++ks) {
    uint32_t ah[4], am[4];
    {
      const uint2 a0 = *reinterpret_cast<const uint2*>(qw + g * BSTR + (ks * 8 + t) * 2);
      const uint2 a1 = *reinterpret_cast<const uint2*>(qw + (MQ_COLS + g) * BSTR + (ks * 8 + t) * 2);
      const uint2 a2 = *reinterpret_cast<const uint2*>(qw + g * BSTR + (ks * 8 + t + 4) * 2);
      const uint2 a3 = *reinterpret_cast<const uint2*>(qw + (MQ_COLS + g) * BSTR + (ks * 8 + t + 4) * 2);
      ah[0] = a0.x; am[0] = a0.y; ah[1] = a1.x; am[1] = a1.y;
      ah[2] = a2.x; am[2] = a2.y; ah[3] = a3.x; am[3] = a3.y;
    }
    qk_step(S, ah, am, [&](int b, uint2& b0, uint2& b1) {
      const uint32_t* kp = kw + ((wy + (b >> 1)) * MT_COLS + wx + (b & 1) * 8 + g) * BSTR + (ks * 8 + t) * 2;
      b0 = *reinterpret_cast<const uint2*>(kp);
      b1 = *reinterpret_cast<const uint2*>(kp + 8);
    });
  }
}

// cp.async of one 32-channel chunk of src (K or V) over the 16 x 24 halo tile (pixel stride pstr words, zero fill
// outside the image) and, with a q, of the 8 x 16 Q tile (pixel stride BSTR), into dst; commits one group
__device__ __forceinline__ void stage_chunk(float* dst, const float* __restrict__ src, int ld, int pstr,
                                            const float* __restrict__ q, int ldq, int c0, size_t img_off, int x0, int y0,
                                            int H, int W, int tid) {
  for (int i = tid; i < MT_ROWS * MT_COLS * (MCH / 4); i += 256) {
    int px = i / (MCH / 4), c4 = i % (MCH / 4);
    int gy = y0 - 4 + px / MT_COLS, gx = x0 - 4 + px % MT_COLS;
    bool ok = gy >= 0 && gy < H && gx >= 0 && gx < W;
    const float* gp = ok ? src + (img_off + (size_t)gy * W + gx) * ld + c0 + c4 * 4 : src;
    cp_async16(dst + px * pstr + c4 * 4, gp, ok);
  }
  if (q) {
    float* qd = dst + BKV_WORDS;
    for (int i = tid; i < MQ_ROWS * MQ_COLS * (MCH / 4); i += 256) {
      int px = i / (MCH / 4), c4 = i % (MCH / 4);
      int gy = y0 + px / MQ_COLS, gx = x0 + px % MQ_COLS;
      bool ok = gy < H && gx < W;
      const float* gp = ok ? q + (img_off + (size_t)gy * W + gx) * ldq + c0 + c4 * 4 : q;
      cp_async16(qd + px * BSTR + c4 * 4, gp, ok);
    }
  }
  cp_async_commit();
}

// ------------------------------------------------------------------------------------------------
// fp32 operands (di_lcab_window_f32).  cp.async lands each chunk as fp32 and the CTA splits it in shared memory, once
// per stage rather than per fragment load:
//   K / Q chunk: [pixel][32 ch] rewritten IN PLACE, channel pair (2j, 2j+1) -> the 64-bit word (hi bf16x2, mid
//                bf16x2), the interleaved layout the dense layers' split epilogue writes (kind 1)
//   V chunk:     the k index of P V is the key, so V is re-laid as [key pair along x][channel] -> (hi, mid) words in
//                a separate buffer (pair stride 72 words)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256, 1)
lcab_window_bf16_kernel(const float* __restrict__ q, int ldq, const float* __restrict__ k, int ldk,
                        const float* __restrict__ v, int ldv, float* __restrict__ out, int ldo, int H, int W, int C,
                        float scale) {
  extern __shared__ __align__(16) float smem[];   // [2][BSTAGE_WORDS] landing / converted K,Q | [VPK_WORDS] packed V
  uint32_t* vpk = reinterpret_cast<uint32_t*>(smem + 2 * BSTAGE_WORDS);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int x0 = blockIdx.x * MQ_COLS, y0 = blockIdx.y * MQ_ROWS, n = blockIdx.z;
  const size_t img_off = (size_t)n * H * W;
  const int nchunk = C / MCH;
  const int nstage = 2 * nchunk;
  auto issue = [&](int stage) {
    const bool is_k = stage < nchunk;
    stage_chunk(smem + (stage & 1) * BSTAGE_WORDS, is_k ? k : v, is_k ? ldk : ldv, BSTR, is_k ? q : nullptr, ldq,
                (is_k ? stage : stage - nchunk) * MCH, img_off, x0, y0, H, W, tid);
  };

  const int wy = 2 * (warp >> 1), wx = 8 * (warp & 1);
  float S[20][4];
  zero_acc(S);
  uint32_t Ph[10][4], Pm[10][4];                     // P = softmax(S) as packed bf16 hi / mid A fragments

  issue(0);
  for (int stage = 0; stage < nstage; ++stage) {
    if (stage + 1 < nstage) {
      issue(stage + 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    float* buf = smem + (stage & 1) * BSTAGE_WORDS;
    if (stage < nchunk) {
      // ---- split K and Q in place: channel pair (2j, 2j+1) of a pixel -> (hi, mid) ----
      for (int i = tid; i < (MT_ROWS * MT_COLS + MQ_ROWS * MQ_COLS) * (MCH / 2); i += 256) {
        float* pp = buf + (i >> 4) * BSTR + (i & 15) * 2;
        const float2 x = *reinterpret_cast<const float2*>(pp);
        *reinterpret_cast<uint2*>(pp) = split_bf16x2(x.x, x.y);
      }
      __syncthreads();
      const uint32_t* kw = reinterpret_cast<const uint32_t*>(buf);
      qk_chunk_interleaved(S, kw, kw + BKV_WORDS + (wy * MQ_COLS + wx) * BSTR, wy, wx, g, t);
      if (stage == nchunk - 1) window_softmax(S, scale, g, t, Ph, Pm);
    } else {
      // ---- re-lay the V chunk: (key 2i, key 2i+1 of a halo row) x channel -> (hi, mid) ----
      for (int i = tid; i < MT_ROWS * (MT_COLS / 2) * MCH; i += 256) {
        const int c = i & (MCH - 1), pr = i >> 5;               // pr = row * 12 + pair
        const int px = (pr / (MT_COLS / 2)) * MT_COLS + (pr % (MT_COLS / 2)) * 2;
        const float v0 = buf[px * BSTR + c], v1 = buf[(px + 1) * BSTR + c];
        *reinterpret_cast<uint2*>(vpk + pr * VPSTR + 2 * c) = split_bf16x2(v0, v1);
      }
      __syncthreads();
      float O[MCH / 8][4];
      zero_acc(O);
#pragma unroll
      for (int r = 0; r < 10; ++r) {
        const uint32_t* vp = vpk + ((wy + r) * (MT_COLS / 2) + wx / 2 + t) * VPSTR + 2 * g;
        uint2 b0[MCH / 8], b1[MCH / 8];
#pragma unroll
        for (int nb = 0; nb < MCH / 8; ++nb) {
          b0[nb] = *reinterpret_cast<const uint2*>(vp + nb * 16);
          b1[nb] = *reinterpret_cast<const uint2*>(vp + 4 * VPSTR + nb * 16);
        }
        pv_row(O, Ph[r], Pm[r], b0, b1);
      }
      store_patch(O, out, ldo, n, H, W, y0 + wy, x0 + wx + g, (stage - nchunk) * MCH, t);
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------
// Interleaved PRE-SPLIT operands (di_lcab_window_pre_f32): q, k (kind 1) and v (kind 2) were written by the producing
// dense layer's epilogue already as bf16 (hi, mid) words (gemm_tc.cu), 4 bytes per value at the value's own position.
// No conversion pass, no packed-V buffer and one barrier less per stage: stages go straight from cp.async to fragments
// (LDS.64 for Q/K; for V, which arrives in 8-channel groups [4 hi words | 4 mid words], ldmatrix.x4.trans).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256, 1)
lcab_window_pre_kernel(const float* __restrict__ q, int ldq, const float* __restrict__ k, int ldk,
                       const float* __restrict__ v, int ldv, float* __restrict__ out, int ldo, int H, int W, int C,
                       float scale) {
  extern __shared__ __align__(16) float smem[];   // [2][BSTAGE_WORDS]: K,Q chunk (pixel stride 40 words) or V chunk (36)
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int x0 = blockIdx.x * MQ_COLS, y0 = blockIdx.y * MQ_ROWS, n = blockIdx.z;
  const size_t img_off = (size_t)n * H * W;
  const int nchunk = C / MCH;
  const int nstage = 2 * nchunk;
  auto issue = [&](int stage) {
    const bool is_k = stage < nchunk;
    stage_chunk(smem + (stage & 1) * BSTAGE_WORDS, is_k ? k : v, is_k ? ldk : ldv, is_k ? BSTR : VSTR2,
                is_k ? q : nullptr, ldq, (is_k ? stage : stage - nchunk) * MCH, img_off, x0, y0, H, W, tid);
  };

  const int wy = 2 * (warp >> 1), wx = 8 * (warp & 1);
  float S[20][4];
  zero_acc(S);
  uint32_t Ph[10][4], Pm[10][4];                     // P = softmax(S) as packed bf16 hi / mid A fragments

  issue(0);
  for (int stage = 0; stage < nstage; ++stage) {
    if (stage + 1 < nstage) {
      issue(stage + 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    float* buf = smem + (stage & 1) * BSTAGE_WORDS;
    if (stage < nchunk) {
      const uint32_t* kw = reinterpret_cast<const uint32_t*>(buf);
      qk_chunk_interleaved(S, kw, kw + BKV_WORDS + (wy * MQ_COLS + wx) * BSTR, wy, wx, g, t);
      if (stage == nchunk - 1) window_softmax(S, scale, g, t, Ph, Pm);
    } else {
      float O[MCH / 8][4];
      zero_acc(O);
      const uint32_t vbase = (uint32_t)__cvta_generic_to_shared(buf) +
                             (uint32_t)(((wy * MT_COLS + wx + (lane & 7) + ((lane >> 3) & 1) * 8) * VSTR2 + (lane >> 4) * 4) * 4);
#pragma unroll
      for (int r = 0; r < 10; ++r) {
        uint2 b0[MCH / 8], b1[MCH / 8];
#pragma unroll
        for (int nb = 0; nb < MCH / 8; ++nb) ldsm_v(vbase + (uint32_t)((r * MT_COLS * VSTR2 + nb * 8) * 4), b0[nb], b1[nb]);
        pv_row(O, Ph[r], Pm[r], b0, b1);
      }
      store_patch(O, out, ldo, n, H, W, y0 + wy, x0 + wx + g, (stage - nchunk) * MCH, t);
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------
// PLANAR operands (split kind 3, C = 128: per pixel 64 hi words | 64 mid words; lcab_proj.cu writes them), the product
// path.  window_core as in the kernels above; what differs is how the operands arrive:
//   persistent grid: min(tiles, SMs) CTAs walk the 8 x 16 query tiles with a static stride in (image, band, column)
//     order (no atomic tile counter: graphs on concurrent streams must not share scheduler state);
//   TMA: per stage one elected thread loads the hi and the mid plane of the 32-channel chunk -- K (16 x 24 halo) and Q
//     (8 x 16), or V -- as boxes of a 4-D tensor map {word, x, y, image}; out-of-image pixels (negative or too large
//     coordinates) arrive zero-filled, which gives the reference's out-of-image rule as the padded kernels' halo does;
//   a 3-slot full / empty mbarrier ring over the 8 stages of a tile (4 K+Q, 4 V) and across tiles, so the next
//     tile's first stages load while the current one runs its softmax, P V and stores.  The producer is thread 0, which
//     refills a slot once all 8 warps have released it; no block-wide barrier is left in the loop;
//   64-byte swizzle: a plane is rows of 64 bytes (16 words of one pixel); TMA stores 16-byte chunk c of row R at chunk
//     c ^ ((R >> 1) & 3).  Every fragment load reads 8 consecutive pixels of a row block starting at a multiple of 8,
//     so the XOR is a per-lane constant, and the 8 pixels cover all 32 banks (R & 1 picks the bank half, the XOR the
//     quarter): Q / K loads and the V ldmatrix rows are conflict-free.
// ------------------------------------------------------------------------------------------------
constexpr int TC_KV_PLANE = MT_ROWS * MT_COLS * 64;                  // 24576 B: one half (hi or mid) of a 16 x 24 halo chunk
constexpr int TC_Q_PLANE = MQ_ROWS * MQ_COLS * 64;                   // 8192 B
constexpr int TC_SLOT = 2 * TC_KV_PLANE + 2 * TC_Q_PLANE;            // 64 KB: K hi | K mid | Q hi | Q mid, or V hi | V mid
constexpr int TC_S = 3;                                              // ring slots
constexpr int TC_SMEM_BYTES = TC_S * TC_SLOT + 1024 /*alignment*/ + 64 /*barriers*/;
static_assert(TC_SMEM_BYTES <= 232448, "lcab_window_tc exceeds the 227 KB shared-memory limit");

__global__ void __launch_bounds__(256, 1)
lcab_window_tc_kernel(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                      const __grid_constant__ CUtensorMap mapV, float* __restrict__ out, int ldo, int H, int W, int bands,
                      int cols, int tiles, float scale) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (tc::smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint8_t* base_ptr = smem_raw + (base - tc::smem_u32(smem_raw));
  const uint32_t bars = base + TC_S * TC_SLOT;
  auto full = [&](int s) { return bars + 8u * s; };
  auto empty = [&](int s) { return bars + 8u * (TC_S + s); };
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int per_image = bands * cols;

  if (tid == 0) {
    for (int s = 0; s < TC_S; ++s) {
      tc::mbar_init(full(s), 1);
      tc::mbar_init(empty(s), 8);                    // one arrival per warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // ---- producer (thread 0): the next stage to load is stage pj of tile ptile, the pit-th stage of this CTA
  int ptile = blockIdx.x, pj = 0, pit = 0;
  auto produce = [&]() {
    if (ptile >= tiles) return;
    const int s = pit % TC_S;
    if (pit >= TC_S) tc::mbar_wait(empty(s), (pit / TC_S - 1) & 1);
    const int n = ptile / per_image, rem = ptile - n * per_image;
    const int y0 = (rem / cols) * MQ_ROWS, x0 = (rem % cols) * MQ_COLS;
    const uint32_t dst = base + s * TC_SLOT;
    const int c = (pj & 3) * 16;                     // hi words of the chunk; its mid words are at 64 + c
    if (pj < 4) {
      tc::mbar_expect_tx(full(s), TC_SLOT);
      tc::tma_load_4d(dst, &mapK, full(s), c, x0 - 4, y0 - 4, n);
      tc::tma_load_4d(dst + TC_KV_PLANE, &mapK, full(s), 64 + c, x0 - 4, y0 - 4, n);
      tc::tma_load_4d(dst + 2 * TC_KV_PLANE, &mapQ, full(s), c, x0, y0, n);
      tc::tma_load_4d(dst + 2 * TC_KV_PLANE + TC_Q_PLANE, &mapQ, full(s), 64 + c, x0, y0, n);
    } else {
      tc::mbar_expect_tx(full(s), 2 * TC_KV_PLANE);
      tc::tma_load_4d(dst, &mapV, full(s), c, x0 - 4, y0 - 4, n);
      tc::tma_load_4d(dst + TC_KV_PLANE, &mapV, full(s), 64 + c, x0 - 4, y0 - 4, n);
    }
    ++pit;
    if (++pj == 8) {
      pj = 0;
      ptile += gridDim.x;
    }
  };
  if (tid == 0) {
    produce();
    produce();
  }

  // ---- consumers: all 8 warps
  int slot = 0;
  uint32_t phase = 0;
  auto release = [&]() {                             // this warp is done reading the slot
    __syncwarp();
    if (lane == 0) tc::mbar_arrive(empty(slot));
    if (++slot == TC_S) {
      slot = 0;
      phase ^= 1u;
    }
  };
  const int wy = 2 * (warp >> 1), wx = 8 * (warp & 1);
  // byte offset of word t of 16-byte chunk c in pixel g of an 8-aligned row block: fl ^ (c << 4)
  const uint32_t fl = g * 64 + (((g >> 1) & 3) << 4) + t * 4;
  // ldmatrix row of lane l: pixel l & 15 of the block (keys 0-7 / 8-15), hi plane for l < 16, mid plane above
  const uint32_t vl = (lane >> 4) * TC_KV_PLANE + (lane & 15) * 64 + (((lane >> 1) & 3) << 4);
  auto ld32 = [&](uint32_t off) { return *reinterpret_cast<const uint32_t*>(base_ptr + off); };

  for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int n = tile / per_image, rem = tile - n * per_image;
    const int y0 = (rem / cols) * MQ_ROWS, x0 = (rem % cols) * MQ_COLS;
    float S[20][4];
    zero_acc(S);
    uint32_t Ph[10][4], Pm[10][4];

#pragma unroll 1
    for (int j = 0; j < 4; ++j) {
      // ---------------- S += Q[chunk] K[chunk]^T ----------------
      if (tid == 0) produce();
      tc::mbar_wait(full(slot), phase);
      const uint32_t kb = slot * TC_SLOT + (wy * MT_COLS + wx) * 64;
      const uint32_t qb = slot * TC_SLOT + 2 * TC_KV_PLANE + (wy * MQ_COLS + wx) * 64;
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) {
        const uint32_t f0 = fl ^ ((2 * ks) << 4), f1 = fl ^ ((2 * ks + 1) << 4);   // words ks*8 + t, ks*8 + t + 4
        uint32_t ah[4], am[4];
        ah[0] = ld32(qb + f0);                       am[0] = ld32(qb + TC_Q_PLANE + f0);
        ah[1] = ld32(qb + MQ_COLS * 64 + f0);        am[1] = ld32(qb + TC_Q_PLANE + MQ_COLS * 64 + f0);
        ah[2] = ld32(qb + f1);                       am[2] = ld32(qb + TC_Q_PLANE + f1);
        ah[3] = ld32(qb + MQ_COLS * 64 + f1);        am[3] = ld32(qb + TC_Q_PLANE + MQ_COLS * 64 + f1);
        qk_step(S, ah, am, [&](int b, uint2& b0, uint2& b1) {
          const uint32_t kp = kb + ((b >> 1) * MT_COLS + (b & 1) * 8) * 64;
          b0 = make_uint2(ld32(kp + f0), ld32(kp + TC_KV_PLANE + f0));
          b1 = make_uint2(ld32(kp + f1), ld32(kp + TC_KV_PLANE + f1));
        });
      }
      release();
      if (j == 3) window_softmax(S, scale, g, t, Ph, Pm);
    }

#pragma unroll 1
    for (int j = 0; j < 4; ++j) {
      // ---------------- O[chunk] = P V[chunk] ----------------
      if (tid == 0) produce();
      tc::mbar_wait(full(slot), phase);
      float O[MCH / 8][4];
      zero_acc(O);
      const uint32_t vb = base + slot * TC_SLOT + (wy * MT_COLS + wx) * 64;
#pragma unroll
      for (int r = 0; r < 10; ++r) {
        uint2 b0[MCH / 8], b1[MCH / 8];
#pragma unroll
        for (int nb = 0; nb < MCH / 8; ++nb) ldsm_v(vb + r * MT_COLS * 64 + (vl ^ (nb << 4)), b0[nb], b1[nb]);
        pv_row(O, Ph[r], Pm[r], b0, b1);
      }
      release();
      store_patch(O, out, ldo, n, H, W, y0 + wy, x0 + wx + g, j * MCH, t);
    }
  }
}

// 4-D tensor map {word, x, y, image} over the first 128 words of each pixel (row stride ld words), box of 16 words x
// box_w x box_h pixels of one image, 64-byte swizzle, out-of-range pixels zero-filled
bool window_map(CUtensorMap* m, const void* ptr, int ld, int N, int H, int W, int box_w, int box_h) {
  tc::EncodeTiledFn enc = tc::get_encode();
  if (!enc) return false;
  const cuuint64_t row = 4ull * ld;
  cuuint64_t dims[4] = {128, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t strides[3] = {row, row * W, row * W * H};
  cuuint32_t box[4] = {16, (cuuint32_t)box_w, (cuuint32_t)box_h, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_UINT32, 4, const_cast<void*>(ptr), dims, strides, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// ------------------------------------------------------------------------------------------------
// Unfused NCHW window ops with the exact contract of the reference extension `localattention`
// (locatt_ops/kernels.cuh: cc2k :4-42, ck2c_ori :44-80, ck2c_loc :82-119; fp32 data, fp64 accumulate
// as in f_cc2k<float,double>).  They exist for drop-in compatibility (autograd of the unfused path);
// the product forward uses the fused window kernels above.
// ------------------------------------------------------------------------------------------------
__global__ void locatt_cc2k_kernel(const float* __restrict__ x_ori, const float* __restrict__ x_loc,
                                   float* __restrict__ y, int C, int H, int W, int kH, int kW, long long total) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;     // over N*H*W*patch, w fastest then tap
  if (i >= total) return;
  const int patch = kH * kW, hw = H * W;
  int w = (int)(i % W);
  int t = (int)((i / W) % patch);
  int h = (int)((i / ((long long)W * patch)) % H);
  int n = (int)(i / ((long long)W * patch * H));
  int hh = h - kH / 2 + t / kW, ww = w - kW / 2 + t % kW;
  double acc = 0.0;
  if (hh >= 0 && hh < H && ww >= 0 && ww < W) {
    const float* a = x_ori + (size_t)n * C * hw + h * W + w;
    const float* b = x_loc + (size_t)n * C * hw + hh * W + ww;
    for (int c = 0; c < C; ++c) acc += (double)(__ldg(a + (size_t)c * hw) * __ldg(b + (size_t)c * hw));
  }
  y[((size_t)n * hw + h * W + w) * patch + t] = (float)acc;
}

// y[n,c,h,w] = sum_t x_loc[n,c,h+dy,w+dx] * wgt[n,h,w,t]
__global__ void locatt_ck2c_ori_kernel(const float* __restrict__ x_loc, const float* __restrict__ wgt,
                                       float* __restrict__ y, int C, int H, int W, int kH, int kW, long long total) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;     // over N*C*H*W
  if (i >= total) return;
  const int patch = kH * kW, hw = H * W;
  int w = (int)(i % W), h = (int)((i / W) % H);
  long long nc = i / hw;
  int n = (int)(nc / C);
  const float* src = x_loc + nc * hw;
  const float* pw = wgt + ((size_t)n * hw + h * W + w) * patch;
  double acc = 0.0;
  for (int t = 0; t < patch; ++t) {
    int hh = h - kH / 2 + t / kW, ww = w - kW / 2 + t % kW;
    if (hh >= 0 && hh < H && ww >= 0 && ww < W) acc += (double)(__ldg(src + hh * W + ww) * __ldg(pw + t));
  }
  y[i] = (float)acc;
}

// y[n,c,h,w] = sum_t x_ori[n,c,h-dy,w-dx] * wgt[n,h-dy,w-dx,t]
__global__ void locatt_ck2c_loc_kernel(const float* __restrict__ x_ori, const float* __restrict__ wgt,
                                       float* __restrict__ y, int C, int H, int W, int kH, int kW, long long total) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int patch = kH * kW, hw = H * W;
  int w = (int)(i % W), h = (int)((i / W) % H);
  long long nc = i / hw;
  int n = (int)(nc / C);
  const float* src = x_ori + nc * hw;
  const float* pw = wgt + (size_t)n * hw * patch;
  double acc = 0.0;
  for (int t = 0; t < patch; ++t) {
    int hh = h + kH / 2 - t / kW, ww = w + kW / 2 - t % kW;
    if (hh >= 0 && hh < H && ww >= 0 && ww < W)
      acc += (double)(__ldg(src + hh * W + ww) * __ldg(pw + ((size_t)hh * W + ww) * patch + t));
  }
  y[i] = (float)acc;
}

}  // namespace

static int g_force_ffma_window = 0;   // 1: di_lcab_window_f32 always runs the FFMA kernel

extern "C" {

// test hook: 0 = di_lcab_window_f32 picks its kernel (default), 1 = always the FFMA kernel
int di_set_window_ffma(int on) {
  DI_CHECK_ARG(on == 0 || on == 1, "di_set_window_ffma: expected 0 or 1 (got %d)", on);
  g_force_ffma_window = on;
  return DI_OK;
}

// di_lcab_window_f32 for operands that the producing layers emitted pre-split (di_linear_tcb_split_f32: q, k kind 1,
// v kind 2).  9x9 window, C % 32 == 0.
int di_lcab_window_pre_f32(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, float* out, int ldo,
                           int N, int H, int W, int C, cudaStream_t stream) {
  DI_CHECK_ARG(q && k && v && out && N > 0 && H > 0 && W > 0, "di_lcab_window_pre_f32: bad argument");
  DI_CHECK_ARG(C > 0 && C % MCH == 0, "di_lcab_window_pre_f32: C must be a multiple of 32 (got %d)", C);
  DI_CHECK_ARG(ldq % 4 == 0 && ldk % 4 == 0 && ldv % 4 == 0 && ldo % 4 == 0, "di_lcab_window_pre_f32: strides must be multiples of 4");
  DI_CHECK_ARG(((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)out) % 16 == 0, "di_lcab_window_pre_f32: pointers must be 16-byte aligned");
  dim3 mgrid(di_cdiv(W, MQ_COLS), di_cdiv(H, MQ_ROWS), N);
  size_t smem = 2ull * BSTAGE_WORDS * sizeof(float);
  static DiSmemOnce once{};
  if (!di_smem_once(once, lcab_window_pre_kernel, (int)smem)) {
    di_set_error("di_lcab_window_pre_f32: cannot reserve shared memory");
    return DI_ERR_LAUNCH;
  }
  lcab_window_pre_kernel<<<mgrid, 256, smem, stream>>>(q, ldq, k, ldk, v, ldv, out, ldo, H, W, C, 1.0f / sqrtf((float)C));
  DI_CHECK_LAUNCH("di_lcab_window_pre_f32");
  return DI_OK;
}

// 9x9 window attention for PLANAR pre-split operands (di_linear_tcb_split_f32 split_kind 3): q, k, v point at [N*H*W]
// pixels with a per-pixel stride of ld* 32-bit words, each pixel holding 128 bf16 hi values followed by 128 bf16 mid
// values (x = hi + mid to 16 mantissa bits).  out: fp32 [N, H, W, ldo], C = 128 channels written.
int di_lcab_window_tc_f32(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv, float* out, int ldo,
                          int N, int H, int W, int C, cudaStream_t stream) {
  DI_CHECK_ARG(q && k && v && out && N > 0 && H > 0 && W > 0, "di_lcab_window_tc_f32: bad argument");
  if (C != 128) {
    di_set_error("di_lcab_window_tc_f32: C must be 128 (got %d)", C);
    return DI_ERR_UNSUPPORTED;
  }
  DI_CHECK_ARG(ldq % 4 == 0 && ldk % 4 == 0 && ldv % 4 == 0 && ldo % 4 == 0 && ldq >= 128 && ldk >= 128 && ldv >= 128 && ldo >= 128,
               "di_lcab_window_tc_f32: strides must be multiples of 4 words and >= 128");
  DI_CHECK_ARG(((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)out) % 16 == 0,
               "di_lcab_window_tc_f32: pointers must be 16-byte aligned");
  const char* name = "di_lcab_window_tc_f32";
  const long long tiles = (long long)N * di_cdiv(H, MQ_ROWS) * di_cdiv(W, MQ_COLS);
  DI_CHECK_ARG(tiles < (1ll << 31), "%s: too many tiles", name);
  int sms = 0;
  const int rc = tc::sm_budget(name, &sms);
  if (rc != DI_OK) return rc;
  static DiSmemOnce once{};
  if (!di_smem_once(once, lcab_window_tc_kernel, TC_SMEM_BYTES)) {
    di_set_error("%s: cannot reserve %d bytes of shared memory", name, TC_SMEM_BYTES);
    return DI_ERR_LAUNCH;
  }
  CUtensorMap maps[3];
  if (!(window_map(&maps[0], q, ldq, N, H, W, MQ_COLS, MQ_ROWS) && window_map(&maps[1], k, ldk, N, H, W, MT_COLS, MT_ROWS) &&
        window_map(&maps[2], v, ldv, N, H, W, MT_COLS, MT_ROWS))) {
    di_set_error("%s: cuTensorMapEncodeTiled failed", name);
    return DI_ERR_LAUNCH;
  }
  const int grid = tiles < sms ? (int)tiles : sms;
  lcab_window_tc_kernel<<<grid, 256, TC_SMEM_BYTES, stream>>>(maps[0], maps[1], maps[2], out, ldo, H, W, di_cdiv(H, MQ_ROWS),
                                                               di_cdiv(W, MQ_COLS), (int)tiles, 1.0f / sqrtf((float)C));
  DI_CHECK_LAUNCH("di_lcab_window_tc_f32");
  return DI_OK;
}

// q,k,v,out: [N,H,W,*] pixel-major fp32 with per-pixel strides ldq/ldk/ldv/ldo (>= C, multiples of 4).
// ksize must be 9 (the only window the reference configs use) or 3 (tests).  C % 16 == 0.
int di_lcab_window_f32(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, float* out, int ldo,
                       int N, int H, int W, int C, int ksize, cudaStream_t stream) {
  DI_CHECK_ARG(q && k && v && out && N > 0 && H > 0 && W > 0, "di_lcab_window_f32: bad argument");
  DI_CHECK_ARG(C > 0 && C % CC == 0, "di_lcab_window_f32: C must be a multiple of 16 (got %d)", C);
  DI_CHECK_ARG(ldq % 4 == 0 && ldk % 4 == 0 && ldv % 4 == 0 && ldo % 4 == 0, "di_lcab_window_f32: strides must be multiples of 4");
  DI_CHECK_ARG(((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)out) % 16 == 0, "di_lcab_window_f32: pointers must be 16-byte aligned");
  dim3 grid(di_cdiv(W, TQ), di_cdiv(H, TQ), N);
  float scale = 1.0f / sqrtf((float)C);
  if (ksize == 9 && C % MCH == 0 && g_force_ffma_window == 0) {
    dim3 mgrid(di_cdiv(W, MQ_COLS), di_cdiv(H, MQ_ROWS), N);
    size_t smem = (2ull * BSTAGE_WORDS + VPK_WORDS) * sizeof(float);
    static DiSmemOnce once_bf{};
    if (!di_smem_once(once_bf, lcab_window_bf16_kernel, (int)smem)) {
      di_set_error("di_lcab_window_f32: cannot reserve shared memory");
      return DI_ERR_LAUNCH;
    }
    lcab_window_bf16_kernel<<<mgrid, 256, smem, stream>>>(q, ldq, k, ldk, v, ldv, out, ldo, H, W, C, scale);
  } else if (ksize == 9) {
    size_t smem = 2ull * (TQ + 8) * (TQ + 8) * PSTR * sizeof(float);
    static DiSmemOnce once9{};
    if (!di_smem_once(once9, lcab_window_kernel<9>, (int)smem)) {
      di_set_error("di_lcab_window_f32: cannot reserve shared memory");
      return DI_ERR_LAUNCH;
    }
    lcab_window_kernel<9><<<grid, TQ * TQ, smem, stream>>>(q, ldq, k, ldk, v, ldv, out, ldo, H, W, C, scale);
  } else if (ksize == 3) {
    size_t smem = 2ull * (TQ + 2) * (TQ + 2) * PSTR * sizeof(float);
    static DiSmemOnce once3{};
    if (!di_smem_once(once3, lcab_window_kernel<3>, (int)smem)) {
      di_set_error("di_lcab_window_f32: cannot reserve shared memory");
      return DI_ERR_LAUNCH;
    }
    lcab_window_kernel<3><<<grid, TQ * TQ, smem, stream>>>(q, ldq, k, ldk, v, ldv, out, ldo, H, W, C, scale);
  } else {
    di_set_error("di_lcab_window_f32: unsupported window %d", ksize);
    return DI_ERR_UNSUPPORTED;
  }
  DI_CHECK_LAUNCH("di_lcab_window_f32");
  return DI_OK;
}

// localattention.similar_forward / weighting_backward_weight  (localAttention.cpp:7-15, 51-59):
// x_ori, x_loc [N,C,H,W] -> y [N,H,W,kH*kW]
int di_locatt_cc2k_f32(const float* x_ori, const float* x_loc, float* y, int N, int C, int H, int W, int kH, int kW,
                       cudaStream_t stream) {
  DI_CHECK_ARG(x_ori && x_loc && y && N > 0 && C > 0 && H > 0 && W > 0 && kH > 0 && kW > 0, "di_locatt_cc2k_f32: bad argument");
  long long total = (long long)N * H * W * kH * kW;
  locatt_cc2k_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(x_ori, x_loc, y, C, H, W, kH, kW, total);
  DI_CHECK_LAUNCH("di_locatt_cc2k_f32");
  return DI_OK;
}
// localattention.weighting_forward / similar_backward(is_ori=True)  (localAttention.cpp:31-39, 17-28)
int di_locatt_ck2c_ori_f32(const float* x_loc, const float* wgt, float* y, int N, int C, int H, int W, int kH, int kW,
                           cudaStream_t stream) {
  DI_CHECK_ARG(x_loc && wgt && y && N > 0 && C > 0 && H > 0 && W > 0, "di_locatt_ck2c_ori_f32: bad argument");
  long long total = (long long)N * C * H * W;
  locatt_ck2c_ori_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(x_loc, wgt, y, C, H, W, kH, kW, total);
  DI_CHECK_LAUNCH("di_locatt_ck2c_ori_f32");
  return DI_OK;
}
// localattention.similar_backward(is_ori=False) / weighting_backward_ori  (localAttention.cpp:17-28, 41-49)
int di_locatt_ck2c_loc_f32(const float* x_ori, const float* wgt, float* y, int N, int C, int H, int W, int kH, int kW,
                           cudaStream_t stream) {
  DI_CHECK_ARG(x_ori && wgt && y && N > 0 && C > 0 && H > 0 && W > 0, "di_locatt_ck2c_loc_f32: bad argument");
  long long total = (long long)N * C * H * W;
  locatt_ck2c_loc_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(x_ori, wgt, y, C, H, W, kH, kW, total);
  DI_CHECK_LAUNCH("di_locatt_ck2c_loc_f32");
  return DI_OK;
}

}  // extern "C"
