// Hopper tensor-core path of the dense layers: C[M,N] = act(A[M,K] * W[N,K]^T + bias (+res)), fp32 in/out,
// computed as an error-compensated SPLIT product on warpgroup MMA (wgmma) with fp32 accumulators in registers:
//
//     A = A_hi + A_lo,  W = W_hi + W_lo,    A*W ~= A_hi*W_hi + A_lo*W_hi + A_hi*W_lo
//
// with either hi = tf32(x) ("3xTF32", dropped term ~2^-22) or hi = bf16(x), lo = bf16(x - hi) ("bf16 split", 16
// mantissa bits kept, error ~1e-5) -- see the BF template flag below.  A plain TF32/BF16 product is not admissible:
// the parity bar of this path is 1e-3 end to end over ~40 chained layers and includes exact top-k indices.
// Same layers as gemm.cu: every 1x1 Conv(+BN)(+ReLU) / cat+conv pair (reference models/utils/encoder_utils.py:11-34,
// models/necks/deepinteraction_encoder.py:26-32) and the 3x3 convs over channel-major (NCHW) inputs as implicit GEMM
// (variant ANCHW below); the 3x3 convs over pixel-major (NHWC) maps have their own kernel in conv_tc.cu.
//
// Persistent CTAs (at most one per SM) walk the 128 x 128 output tiles with a static stride; 384 threads in three
// warpgroups, all hand-offs through mbarriers:
//   warpgroup 0   TMA producer (one thread): per K chunk, box loads of fp32 A (2-D [rows,K] map) and of W_hi / W_lo
//                 into a ring of 128B-swizzled K-major tiles (cp.async.bulk.tensor + mbarrier tx-count); L2 prefetch of
//                 the next tile's A rows.  For K <= 128 the weight slice is loaded once and stays resident.
//   warpgroups 1-2  consumers, 64 output rows each: landed A chunk -> registers (the wgmma A fragment, read through
//                 the swizzle) -> hi / lo split in registers -> wgmma with W_hi / W_lo straight from shared memory;
//                 then the epilogue from the accumulator registers: bias / residual / activation -> global stores.
#include "tc_common.cuh"

namespace {

constexpr int TM = 128, TN = 128, TK = 32;          // tile; TK fp32 = 128 bytes = one swizzle row
constexpr int A_BYTES = TM * TK * 4;                // 16 KB: one 128-row x 128-byte operand box
constexpr int NTHREADS = 384;
constexpr int RING_BYTES = 192 * 1024;
constexpr int BAR_BYTES = 256;
constexpr int V3_SMEM_BYTES = RING_BYTES + 1024 /*alignment*/ + BAR_BYTES;
static_assert(V3_SMEM_BYTES <= 232448, "gemm_tc exceeds the 227 KB shared-memory limit");

using namespace tc;

// optional pipeline trace (CTA 0 only): clock64 stamps per role and chunk, read back with di_tc_debug_read
constexpr int DBG_SLOTS = 8, DBG_N = 512;
__device__ long long g_dbg[DBG_SLOTS * DBG_N];
#define DBG_STAMP(slot, i)                                                            \
  do {                                                                               \
    if (p.dbg && blockIdx.x == 0 && (i) < DBG_N) g_dbg[(slot) * DBG_N + (i)] = clock64(); \
  } while (0)

struct TcParams {
  int M, N;                 // logical output size (rows, columns)
  int nsrc;                 // linear: number of A sources (1..3)
  int k0, k1, k2;           // linear: K_s / KE per source; conv: k0 = Cin / KE.  (Scalars, not an array: a dynamically
                            // indexed kernel parameter makes ptxas copy the whole struct to LOCAL memory.)
  int conv;                 // 1: 3x3 conv over an NCHW map (variant ANCHW, A map is 4-D)
  int H, W, tiles_x, tiles_y;  // conv geometry: tile = 8 rows x 16 cols of pixels
  int m_tiles, n_tiles;     // tile grid (m_tiles = images * tiles_y * tiles_x for conv)
  float* C;
  int ldc;
  const float* bias;
  const float* res;
  int ldres, res_mod, act;
  int dbg;
  int split_col0, split_kind;  // output columns >= split_col0 are emitted as bf16 (hi, mid) words (0 = off), see below
  int a_nchw;               // conv: the input map is NCHW (kernel variant ANCHW)
};
__host__ __device__ __forceinline__ int tc_kch(const TcParams& p, int s) { return s == 0 ? p.k0 : (s == 1 ? p.k1 : p.k2); }

// Two operand precisions share this kernel (template flag BF):
//   BF = false  "3xTF32" (the PRECISE mode): x = hi + lo with hi = tf32(x); products A_hi W_hi into the main
//               accumulator, A_lo W_hi + A_hi W_lo into a second one that is added in the epilogue (the tensor core
//               truncates at every accumulate, so the main product's error grows with the number of instructions that
//               hit its accumulator); wgmma k8, 32 k-values per pipeline chunk.  Error ~2^-21 per product.
//   BF = true   "bf16 split": x = hi + mid with hi = bf16(x), mid = bf16(x - hi) (16 mantissa bits kept);
//               products A_mid W_hi + A_hi W_mid + A_hi W_hi into one accumulator; wgmma k16, 64 k-values per chunk.
//               Error ~3 * 2^-18 per product (1e-5), far inside the 1e-3 budget of the path.
// Both variants use the same weight tiles: a weight chunk is 128 rows x 128 B (32 tf32 or 64 bf16), 4 wgmma k-steps
// of 32 bytes.
//
// Pre-split outputs for the window-attention kernels (lcab.cu), same 4 bytes per value: the consumer then needs no
// conversion pass.  hi = bf16(x), mid = bf16(x - hi), packed bf16x2 with the lower channel in the low half.
//   kind 1 (Q, K): channel pair (2j, 2j+1) -> words 2j = hi pair, 2j+1 = mid pair
//   kind 2 (V):    channel group of 8      -> words 8g..8g+3 = hi pairs, 8g+4..8g+7 = mid pairs
//   kind 3 (planar): group of 128 channels -> 64 hi words | 64 mid words
// Every thread holds channel pairs (2j, 2j+1) of the accumulator, so each kind is a per-pair address computation.
//
// WRES: the whole [128, K<=128] weight slice (hi + lo, 128 KB) of this CTA's column tile stays resident in shared
// memory (the grid is a multiple of n_tiles, so the column tile of a CTA never changes); only A streams.
// ANCHW (convolution only): the input map is NCHW.  A TMA box must start on a 16-byte boundary in the innermost
// dimension, so single-pixel tap shifts along x cannot be expressed as box coordinates of a channel-major map.
// Instead ONE box [KE channels][8 rows][24 pixels] starting at x0 - 4 is loaded per (tap row, channel chunk) into a
// 2-deep ring and serves the three taps of that row: the consumers read channel k of pixel (y, x + 3 + dx) straight
// into their fragments.  Weights stream through their own ring (one 32 KB hi|lo stage per tap and channel chunk).
template <bool WRES, bool BF, bool ANCHW>
__global__ void __launch_bounds__(NTHREADS, 1)
gemm_tc_kernel_v3(const __grid_constant__ CUtensorMap mapA0, const __grid_constant__ CUtensorMap mapA1,
                  const __grid_constant__ CUtensorMap mapA2, const __grid_constant__ CUtensorMap mapWhi,
                  const __grid_constant__ CUtensorMap mapWlo, const TcParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint8_t* base_ptr = smem_raw + (base - smem_u32(smem_raw));
  constexpr int KE = BF ? 64 : 32;                                // k-values per chunk
  constexpr int AL = TM * KE * 4;                                 // fp32 A landing bytes per chunk (BF: two 16 KB boxes)
  static_assert(!(ANCHW && WRES), "the NCHW conv variant streams its weights");
  constexpr int AB = 24 * 8 * KE * 4;                             // ANCHW: bytes of one [KE][8][24] A box
  constexpr int S = WRES ? (BF ? 2 : 4) : (BF ? 3 : 4);           // pipeline stages
  constexpr int STG = ANCHW ? 2 * A_BYTES : (WRES ? AL : AL + 2 * A_BYTES);   // stage: [A landing |] W_hi | W_lo
  constexpr int NKW = BF ? 2 : 4;                                 // resident chunks (K <= 128)
  constexpr int WRES_BYTES = WRES ? 2 * NKW * A_BYTES : 0;        // resident W: hi chunks | lo chunks
  constexpr int RING_OFF = ANCHW ? 2 * AB : WRES_BYTES;           // stage ring starts after the resident weights / A ring
  static_assert(RING_OFF + S * STG <= RING_BYTES, "operand ring exceeds its 192 KB");
  constexpr int NCONS_WARPS = 8;
  const uint32_t bars = base + RING_BYTES;
  auto full = [&](int s) { return bars + 8u * s; };
  auto empty = [&](int s) { return bars + 8u * (S + s); };
  const uint32_t w_full = bars + 8u * (2 * S);
  auto a2_full = [&](int i) { return bars + 8u * (2 * S + 1 + i); };       // ANCHW A-box ring
  auto a2_empty = [&](int i) { return bars + 8u * (2 * S + 3 + i); };
  static_assert(8 * (2 * S + 5) <= BAR_BYTES, "barrier block overflow");

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) DBG_STAMP(7, 100);            // kernel entry
  if (warp == 1 && lane < 5) {                         // pull the TMA descriptors into the descriptor cache early
    const CUtensorMap* mp = lane == 0 ? &mapA0 : lane == 1 ? &mapA1 : lane == 2 ? &mapA2 : lane == 3 ? &mapWhi : &mapWlo;
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(mp)) : "memory");
  }
  int nk = 0;
  if (p.conv) nk = 9 * p.k0;
  else
    for (int s = 0; s < p.nsrc; ++s) nk += tc_kch(p, s);
  const int num_tiles = p.m_tiles * p.n_tiles;

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(full(s), 1);
      mbar_init(empty(s), NCONS_WARPS);
    }
    mbar_init(w_full, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(a2_full(i), 1);
      mbar_init(a2_empty(i), NCONS_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  auto tile_coords = [&](int tile, int& m0, int& n0, int& img, int& y0, int& x0) {
    const int mt = tile / p.n_tiles, nt = tile - mt * p.n_tiles;
    n0 = nt * TN;
    m0 = mt * TM;
    img = 0; y0 = 0; x0 = 0;
    if (p.conv) {
      int t = mt;
      img = t / (p.tiles_x * p.tiles_y);
      t -= img * p.tiles_x * p.tiles_y;
      y0 = (t / p.tiles_x) * 8;
      x0 = (t % p.tiles_x) * 16;
    }
  };

  if (warp < 4) {
    // ---------------- TMA producer ----------------
    // one thread issues all loads: the warpgroup hands most of its registers to the consumers (128 x 40 + 256 x 232)
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      int it = 0, t3 = 0;
      if (WRES && (int)blockIdx.x < num_tiles) {
        // resident weights: gridDim.x % n_tiles == 0, so the column tile of this CTA is fixed
        const int n0w = (int)(blockIdx.x % p.n_tiles) * TN;
        mbar_expect_tx(w_full, 2 * nk * A_BYTES);
        for (int kc = 0; kc < nk; ++kc) {
          tma_load_2d(base + kc * A_BYTES, &mapWhi, w_full, kc * KE, n0w);
          tma_load_2d(base + (NKW + kc) * A_BYTES, &mapWlo, w_full, kc * KE, n0w);
        }
      }
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int m0, n0, img, y0, x0;
        tile_coords(tile, m0, n0, img, y0, x0);
        if (ANCHW) {
          for (int dy = 0; dy < 3; ++dy)
            for (int kc = 0; kc < p.k0; ++kc, ++t3) {
              const int ab = t3 & 1;
              if (t3 >= 2) mbar_wait(a2_empty(ab), ((t3 >> 1) - 1) & 1);
              mbar_expect_tx(a2_full(ab), AB);
              tma_load_4d(base + ab * AB, &mapA0, a2_full(ab), x0 - 4, y0 + dy - 1, kc * KE, img);
              for (int dx = 0; dx < 3; ++dx, ++it) {
                const int s = it % S;
                if (it >= S) mbar_wait(empty(s), ((it / S) - 1) & 1);
                DBG_STAMP(0, it);
                const uint32_t st = base + RING_OFF + s * STG;
                const int kw = ((dy * 3 + dx) * p.k0 + kc) * KE;
                mbar_expect_tx(full(s), STG);
                tma_load_2d(st, &mapWhi, full(s), kw, n0);
                tma_load_2d(st + A_BYTES, &mapWlo, full(s), kw, n0);
              }
            }
        } else {
          for (int kc_all = 0; kc_all < nk; ++kc_all, ++it) {
            const int s = it % S;
            if (it >= S) mbar_wait(empty(s), ((it / S) - 1) & 1);
            DBG_STAMP(0, it);
            const uint32_t st = base + RING_OFF + s * STG;
            mbar_expect_tx(full(s), STG);
            int src = 0, kc = kc_all;
            while (kc >= tc_kch(p, src)) {
              kc -= tc_kch(p, src);
              ++src;
            }
            const CUtensorMap* mp = src == 0 ? &mapA0 : (src == 1 ? &mapA1 : &mapA2);
            tma_load_2d(st, mp, full(s), kc * KE, m0);
            if (BF) tma_load_2d(st + A_BYTES, mp, full(s), kc * KE + 32, m0);
            if (!WRES) {
              tma_load_2d(st + AL, &mapWhi, full(s), kc_all * KE, n0);
              tma_load_2d(st + AL + A_BYTES, &mapWlo, full(s), kc_all * KE, n0);
            }
          }
          const int nxt = tile + (int)gridDim.x;       // L2 prefetch of the next tile's A rows
          if (nxt < num_tiles) {
            const int mt = nxt / p.n_tiles;
            for (int src = 0; src < p.nsrc; ++src)
              for (int kc = 0; kc < tc_kch(p, src); ++kc) {
                const CUtensorMap* mp = src == 0 ? &mapA0 : (src == 1 ? &mapA1 : &mapA2);
                tma_prefetch_2d(mp, kc * KE, mt * TM);
                if (BF) tma_prefetch_2d(mp, kc * KE + 32, mt * TM);
              }
          }
        }
      }
    }
  } else {
    // ---------------- consumers (warpgroups 1, 2): 64 rows each ----------------
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int wg = (warp >> 2) - 1, wl = warp & 3;
    const int g = lane >> 2, t = lane & 3;
    const int r0 = wg * 64 + wl * 16 + g, r1 = r0 + 8;   // tile rows of this thread's fragments
    constexpr int NX = BF ? 1 : 64;
    float acc[64], accx[NX];
    int it = 0;
    bool w_ready = !WRES;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int m0, n0, img, y0, x0;
      tile_coords(tile, m0, n0, img, y0, x0);
      if (!w_ready) {
        mbar_wait(w_full, 0);
        w_ready = true;
      }
      for (int kc_all = 0; kc_all < nk; ++kc_all, ++it) {
        const int s = it % S;
        const uint32_t st = base + RING_OFF + s * STG;
        mbar_wait(full(s), (it / S) & 1);
        if (threadIdx.x == 128) DBG_STAMP(1, it);
        // A element (row, k) of this chunk -> shared-memory address
        int t3 = 0, dx = 0, ab = 0;
        if (ANCHW) {
          t3 = it / 3; dx = it - 3 * t3; ab = t3 & 1;
          if (dx == 0) mbar_wait(a2_full(ab), (t3 >> 1) & 1);
        }
        const float* abox = reinterpret_cast<const float*>(base_ptr + (ANCHW ? ab * AB : RING_OFF + s * STG));
        auto a_at = [&](int row, int k) -> float {      // k < KE
          if (ANCHW) return abox[k * 192 + (row >> 4) * 24 + (row & 15) + 3 + dx];
          const int h = k >> 5, kk = k & 31;           // BF: two 32-column boxes
          return abox[h * (A_BYTES / 4) + row * 32 + ((((kk >> 2) ^ (row & 7))) << 2) + (kk & 3)];
        };
        auto a_pair = [&](int row, int k) -> float2 {   // (k, k + 1), k even
          if (ANCHW) return make_float2(a_at(row, k), a_at(row, k + 1));
          const int h = k >> 5, kk = k & 31;
          return *reinterpret_cast<const float2*>(abox + h * (A_BYTES / 4) + row * 32 + ((((kk >> 2) ^ (row & 7))) << 2) +
                                                  (kk & 3));
        };
        const uint32_t whi = WRES ? base + kc_all * A_BYTES : st + (ANCHW ? 0 : AL);
        const uint32_t wlo = WRES ? base + (NKW + kc_all) * A_BYTES : st + (ANCHW ? 0 : AL) + A_BYTES;
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {                // two k-steps per wgmma group
          uint32_t ahi[2][4], alo[2][4];
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const int ks = 2 * hf + u;
            if (BF) {
              const int kb = 16 * ks + 2 * t;
              const float2 x[4] = {a_pair(r0, kb), a_pair(r1, kb), a_pair(r0, kb + 8), a_pair(r1, kb + 8)};
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const uint32_t h = pack_bf16x2(x[e].x, x[e].y);
                ahi[u][e] = h;
                alo[u][e] = pack_bf16x2(x[e].x - __uint_as_float(h << 16), x[e].y - __uint_as_float(h & 0xFFFF0000u));
              }
            } else {
              const int kb = 8 * ks + t;
              const float x[4] = {a_at(r0, kb), a_at(r1, kb), a_at(r0, kb + 4), a_at(r1, kb + 4)};
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                ahi[u][e] = (__float_as_uint(x[e]) + 0x1000u) & 0xFFFFE000u;        // round to nearest tf32
                alo[u][e] = __float_as_uint(x[e] - __uint_as_float(ahi[u][e]));     // exact remainder
              }
            }
          }
          fence_regs(acc);
          if (!BF) fence_regs(accx);
          wgmma_fence();
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const int ks = 2 * hf + u;
            const uint32_t first = (kc_all | ks) != 0;
            const uint64_t w_hi = wgmma_desc(whi + ks * 32), w_lo = wgmma_desc(wlo + ks * 32);
            if constexpr (BF) {
              wgmma_bf16_rs(acc, alo[u], w_hi, first);   // A_mid * W_hi
              wgmma_bf16_rs(acc, ahi[u], w_lo, 1);       // A_hi * W_mid
              wgmma_bf16_rs(acc, ahi[u], w_hi, 1);       // A_hi * W_hi
            } else {
              wgmma_tf32_rs(accx, alo[u], w_hi, first);  // A_lo * W_hi
              wgmma_tf32_rs(accx, ahi[u], w_lo, 1);      // A_hi * W_lo
              wgmma_tf32_rs(acc, ahi[u], w_hi, first);   // A_hi * W_hi
            }
          }
          wgmma_commit();
          wgmma_wait_all();
          fence_regs(acc);
          if (!BF) fence_regs(accx);
        }
        if (threadIdx.x == 128) DBG_STAMP(4, it);
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(empty(s));                        // stage (A landing and / or weights) read by this warp
          if (ANCHW && dx == 2) mbar_arrive(a2_empty(ab));
        }
      }
      if constexpr (!BF) {
#pragma unroll
        for (int j = 0; j < 64; ++j) acc[j] += accx[j];
      }
      // ---------------- epilogue: bias / residual / activation, stores ----------------
      long long grow[2];
      bool rok[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = h ? r1 : r0;
        if (p.conv) {
          const int yy = y0 + row / 16, xx = x0 + row % 16;
          rok[h] = yy < p.H && xx < p.W;
          grow[h] = ((long long)img * p.H + min(yy, p.H - 1)) * p.W + min(xx, p.W - 1);
        } else {
          rok[h] = m0 + row < p.M;
          grow[h] = min((long long)(m0 + row), (long long)p.M - 1);
        }
      }
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int col = n0 + 8 * j + 2 * t;
        if (col < p.N) {                                // N % 4 == 0: the pair is valid as a whole
          float2 b2 = make_float2(0.f, 0.f);
          if (p.bias) b2 = *reinterpret_cast<const float2*>(p.bias + col);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            acc[4 * j + 2 * h] += b2.x;
            acc[4 * j + 2 * h + 1] += b2.y;
            if (p.res) {
              const float2 r2 = *reinterpret_cast<const float2*>(p.res + (size_t)(grow[h] % p.res_mod) * p.ldres + col);
              acc[4 * j + 2 * h] += r2.x;
              acc[4 * j + 2 * h + 1] += r2.y;
            }
          }
        }
      }
      if (p.act == DI_ACT_RELU) {                       // one warp-uniform branch per activation (no per-element
#pragma unroll                                          // if-conversion of the GELU polynomial)
        for (int j = 0; j < 64; ++j) acc[j] = fmaxf(acc[j], 0.f);
      } else if (p.act == DI_ACT_GELU) {
#pragma unroll
        for (int j = 0; j < 64; ++j) acc[j] = 0.5f * acc[j] * (1.f + erff(acc[j] * 0.70710678118654752440f));
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (!rok[h]) continue;
        float* crow = p.C + (size_t)grow[h] * p.ldc;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int col = n0 + 8 * j + 2 * t;
          if (col >= p.N) continue;
          const float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
          if (p.split_kind && col >= p.split_col0) {
            const uint32_t hi = pack_bf16x2(v0, v1);
            const uint32_t mid = pack_bf16x2(v0 - __uint_as_float(hi << 16), v1 - __uint_as_float(hi & 0xFFFF0000u));
            uint32_t* cw = reinterpret_cast<uint32_t*>(crow);
            if (p.split_kind == 1) {
              *reinterpret_cast<uint2*>(cw + col) = make_uint2(hi, mid);
            } else if (p.split_kind == 2) {
              const int g8 = col & ~7, q = (col & 7) >> 1;
              cw[g8 + q] = hi;
              cw[g8 + 4 + q] = mid;
            } else {
              const int rel = col - p.split_col0;
              const int w0 = p.split_col0 + (rel & ~127) + ((rel & 127) >> 1);
              cw[w0] = hi;
              cw[w0 + 64] = mid;
            }
          } else {
            *reinterpret_cast<float2*>(crow + col) = make_float2(v0, v1);
          }
        }
      }
      if (threadIdx.x == 128) DBG_STAMP(6, (tile - (int)blockIdx.x) / (int)gridDim.x);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) DBG_STAMP(7, 102);            // all roles done
}

// ---- host side ----------------------------------------------------------------------------------

// 2-D fp32 map over a row-major [rows, cols] matrix with row stride ld (elements); box = 32 cols x 128 rows
bool make_map_2d(CUtensorMap* m, const float* ptr, long long rows, long long cols, long long ld) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return false;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 4};
  cuuint32_t box[2] = {TK, TM};
  cuuint32_t estr[2] = {1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(ptr), dims, strides, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
// 2-D bf16 map over a row-major [rows, cols] weight (cols contiguous); box = 64 cols (128 B) x 128 rows
bool make_map_2d_bf16(CUtensorMap* m, const void* ptr, long long rows, long long cols) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return false;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)cols * 2};
  cuuint32_t box[2] = {64, TM};
  cuuint32_t estr[2] = {1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// 4-D fp32 map over an NCHW tensor (dims W, H, C, N); box = 24 x-pixels x 8 y-pixels x ke channels, no swizzle.
// Boxes must start on 16-byte boundaries in x: the kernel loads from x0 - 4 (x0 % 16 == 0).
bool make_map_nchw(CUtensorMap* m, const float* ptr, int N, int H, int W, int C, int ke) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return false;
  cuuint64_t dims[4] = {(cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)C, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)W * 4, (cuuint64_t)H * W * 4, (cuuint64_t)C * H * W * 4};
  cuuint32_t box[4] = {24, 8, (cuuint32_t)ke, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(ptr), dims, strides, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// Per-device launch state (one process may drive several GPUs): SM count and the one-time shared-memory attribute.
constexpr int MAX_DEV = 64;
struct DevState {
  int num_sms = 0;
  bool attr_set = false;
};
DevState g_dev[MAX_DEV];
int g_tc_debug = 0;
int g_tc_wres = 1;    // keep the weight slice resident in shared memory when K <= 128
int g_tc_sm_limit = 0; // > 0: persistent grids use at most this many CTAs (leaves SMs to kernels of other streams)

template <bool WRES, bool BF, bool ANCHW = false>
void launch_v3(dim3 grid, const CUtensorMap maps[5], const TcParams& p, cudaStream_t stream) {
  gemm_tc_kernel_v3<WRES, BF, ANCHW><<<grid, NTHREADS, V3_SMEM_BYTES, stream>>>(maps[0], maps[1], maps[2], maps[3], maps[4], p);
}

}  // namespace

int tc::sm_budget(const char* name, int* sms) {
  int devid = 0;
  cudaGetDevice(&devid);
  if (devid < 0 || devid >= MAX_DEV) {
    di_set_error("%s: device ordinal %d not supported", name, devid);
    return DI_ERR_UNSUPPORTED;
  }
  DevState& ds = g_dev[devid];
  if (ds.num_sms == 0) {
    if (cudaDeviceGetAttribute(&ds.num_sms, cudaDevAttrMultiProcessorCount, devid) != cudaSuccess || ds.num_sms <= 0) {
      ds.num_sms = 0;
      di_set_error("%s: cannot query the SM count of device %d", name, devid);
      return DI_ERR_LAUNCH;
    }
  }
  *sms = (g_tc_sm_limit > 0 && g_tc_sm_limit < ds.num_sms) ? g_tc_sm_limit : ds.num_sms;
  return DI_OK;
}

namespace {

// bf = 1: bf16-split operands (chunks of 64 k-values), 0: 3xTF32 (chunks of 32)
int launch_tc(const CUtensorMap maps[5], const TcParams& p, int bf, cudaStream_t stream, const char* name) {
  int sms = 0;
  const int rc = sm_budget(name, &sms);
  if (rc != DI_OK) return rc;
  int devid = 0;
  cudaGetDevice(&devid);
  DevState& ds = g_dev[devid];
  if (!ds.attr_set) {
    if (cudaFuncSetAttribute(gemm_tc_kernel_v3<false, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, V3_SMEM_BYTES) != cudaSuccess ||
        cudaFuncSetAttribute(gemm_tc_kernel_v3<true, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, V3_SMEM_BYTES) != cudaSuccess ||
        cudaFuncSetAttribute(gemm_tc_kernel_v3<false, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, V3_SMEM_BYTES) != cudaSuccess ||
        cudaFuncSetAttribute(gemm_tc_kernel_v3<true, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, V3_SMEM_BYTES) != cudaSuccess ||
        cudaFuncSetAttribute(gemm_tc_kernel_v3<false, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, V3_SMEM_BYTES) != cudaSuccess ||
        cudaFuncSetAttribute(gemm_tc_kernel_v3<false, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, V3_SMEM_BYTES) != cudaSuccess) {
      di_set_error("%s: cannot reserve %d bytes of shared memory", name, V3_SMEM_BYTES);
      return DI_ERR_LAUNCH;
    }
    ds.attr_set = true;
  }
  const int tiles = p.m_tiles * p.n_tiles;
  int nk = p.k0 + p.k1 + p.k2;
  const bool wres = !p.conv && nk <= (bf ? 2 : 4) && g_tc_wres && p.n_tiles <= 14;
  int g = tiles < sms ? tiles : sms;
  if (wres) {
    // every CTA keeps one column tile's weights resident: the grid must be a multiple of n_tiles
    if (tiles >= sms) g = (sms / p.n_tiles) * p.n_tiles;
    if (g < p.n_tiles) g = p.n_tiles;
  }
  if (p.a_nchw && bf) launch_v3<false, true, true>(dim3(g), maps, p, stream);
  else if (p.a_nchw) launch_v3<false, false, true>(dim3(g), maps, p, stream);
  else if (wres && bf) launch_v3<true, true>(dim3(g), maps, p, stream);
  else if (wres) launch_v3<true, false>(dim3(g), maps, p, stream);
  else if (bf) launch_v3<false, true>(dim3(g), maps, p, stream);
  else launch_v3<false, false>(dim3(g), maps, p, stream);
  DI_CHECK_LAUNCH(name);
  return DI_OK;
}

inline bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// shared body of di_linear_tc_f32 (bf = 0) and di_linear_tcb_f32 (bf = 1)
int linear_tc_impl(const char* name, int bf, const float* A0, int lda0, int K0, const float* A1, int lda1, int K1,
                   const float* A2, int lda2, int K2, const void* W_hi, const void* W_lo, const float* bias,
                   const float* res, int ldres, int res_mod, float* C, int ldc, int M, int N, int act,
                   int split_col0, int split_kind, cudaStream_t stream) {
  if (!(A0 && W_hi && W_lo && C && M > 0 && N > 0 && K0 > 0)) {
    di_set_error("%s: null pointer or empty shape", name);
    return DI_ERR_ARG;
  }
  const int KE = bf ? 64 : 32;
  const float* As[3] = {A0, A1, A2};
  const int lds[3] = {lda0, lda1, lda2}, Ks[3] = {K0, K1, K2};
  int nsrc = 1 + (K1 > 0) + (K2 > 0);
  int K = K0 + K1 + K2;
  bool ok = al16(W_hi) && al16(W_lo) && al16(C) && ldc % 4 == 0 && N % 4 == 0 && (K2 == 0 || K1 > 0) && (!bias || al16(bias)) &&
            (!res || (al16(res) && ldres % 4 == 0));
  for (int s = 0; s < nsrc; ++s) ok = ok && As[s] && Ks[s] % KE == 0 && lds[s] % 4 == 0 && al16(As[s]);
  if (!ok) {
    di_set_error("%s: shape/alignment not supported by the tensor-core path", name);
    return DI_ERR_UNSUPPORTED;
  }
  CUtensorMap maps[5];
  bool made = true;
  for (int s = 0; s < 3 && made; ++s) {
    int u = s < nsrc ? s : 0;
    made = make_map_2d(&maps[s], As[u], M, Ks[u], lds[u]);
  }
  if (made) {
    if (bf) made = make_map_2d_bf16(&maps[3], W_hi, N, K) && make_map_2d_bf16(&maps[4], W_lo, N, K);
    else made = make_map_2d(&maps[3], (const float*)W_hi, N, K, K) && make_map_2d(&maps[4], (const float*)W_lo, N, K, K);
  }
  if (!made) {
    di_set_error("%s: cuTensorMapEncodeTiled failed", name);
    return DI_ERR_LAUNCH;
  }
  TcParams p{};
  p.M = M; p.N = N; p.nsrc = nsrc;
  p.k0 = Ks[0] / KE; p.k1 = Ks[1] / KE; p.k2 = Ks[2] / KE;
  p.conv = 0; p.C = C; p.ldc = ldc; p.bias = bias; p.res = res; p.ldres = ldres;
  p.res_mod = res_mod > 0 ? res_mod : M; p.act = act; p.dbg = g_tc_debug;
  p.m_tiles = di_cdiv(M, TM);
  p.n_tiles = di_cdiv(N, TN);
  if (split_kind) {
    const bool ok12 = (split_kind == 1 || split_kind == 2) && split_col0 >= 0 && split_col0 % 32 == 0 && N % 32 == 0;
    const bool ok3 = split_kind == 3 && split_col0 >= 0 && split_col0 % 128 == 0 && N % 128 == 0;
    if (!(ok12 || ok3)) {
      di_set_error("%s: split output needs kind 1|2 (split_col0 %% 32 == 0, N %% 32 == 0) or kind 3 (both %% 128 == 0)", name);
      return DI_ERR_ARG;
    }
    p.split_col0 = split_col0;
    p.split_kind = split_kind;
  }
  return launch_tc(maps, p, bf, stream, name);
}

int conv3x3_tc_impl(const char* name, int bf, int x_nchw, const float* x, const void* w_hi, const void* w_lo,
                    const float* bias, float* y, int N, int Cin, int H, int W, int Cout, int act, cudaStream_t stream) {
  if (!(x && w_hi && w_lo && y && N > 0 && H > 0 && W > 0)) {
    di_set_error("%s: bad argument", name);
    return DI_ERR_ARG;
  }
  const int KE = bf ? 64 : 32;
  if (!(Cin % KE == 0 && Cout % 4 == 0 && al16(x) && al16(y) && al16(w_hi) && al16(w_lo) && (!bias || al16(bias)) &&
        (!x_nchw || W % 4 == 0))) {
    di_set_error("%s: shape/alignment not supported by the tensor-core path", name);
    return DI_ERR_UNSUPPORTED;
  }
  if (!x_nchw) return conv3x3_nhwc(name, bf, x, w_hi, w_lo, bias, y, N, Cin, H, W, Cout, act, stream);
  CUtensorMap maps[5];
  long long K = 9ll * Cin;
  bool made = make_map_nchw(&maps[0], x, N, H, W, Cin, KE);
  if (made) {
    if (bf) made = make_map_2d_bf16(&maps[3], w_hi, Cout, K) && make_map_2d_bf16(&maps[4], w_lo, Cout, K);
    else made = make_map_2d(&maps[3], (const float*)w_hi, Cout, K, K) && make_map_2d(&maps[4], (const float*)w_lo, Cout, K, K);
  }
  if (!made) {
    di_set_error("%s: cuTensorMapEncodeTiled failed", name);
    return DI_ERR_LAUNCH;
  }
  maps[1] = maps[0];
  maps[2] = maps[0];
  TcParams p{};
  p.M = N * H * W; p.N = Cout; p.nsrc = 1; p.k0 = Cin / KE; p.conv = 1; p.a_nchw = x_nchw; p.H = H; p.W = W;
  p.tiles_x = di_cdiv(W, 16); p.tiles_y = di_cdiv(H, 8);
  p.C = y; p.ldc = Cout; p.bias = bias; p.res = nullptr; p.ldres = 0; p.res_mod = 1; p.act = act; p.dbg = g_tc_debug;
  p.m_tiles = N * p.tiles_x * p.tiles_y;
  p.n_tiles = di_cdiv(Cout, TN);
  return launch_tc(maps, p, bf, stream, name);
}

}  // namespace

extern "C" {

// Pipeline trace of CTA 0 (diagnostics): enable, run ONE tensor-core launch, then read 8 x 512 clock64 stamps
// (rows: 0 producer issue, 1 bytes landed, 2 split done, 3 mma ready, 4 mma issued, 5 acc ready, 6 tile stored,
// 7 epilogue phases / kernel entry-exit).
int di_tc_set_debug(int on) {
  g_tc_debug = on;
  return DI_OK;
}
// 3 (default): weights resident in shared memory when K <= 128; 4: always streamed (A/B tests)
int di_tc_set_mode(int mode) {
  DI_CHECK_ARG(mode == 3 || mode == 4, "di_tc_set_mode: mode must be 3 or 4");
  g_tc_wres = mode != 4;
  return DI_OK;
}
// Persistent tensor-core grids use at most n CTAs (0 = all SMs): with several frames in flight the other streams'
// small kernels then always find a free SM.  The tiles are strided over the grid, so any grid size is correct.
int di_tc_set_sm_limit(int n) {
  DI_CHECK_ARG(n >= 0, "di_tc_set_sm_limit: n must be >= 0");
  g_tc_sm_limit = n;
  return DI_OK;
}
int di_tc_debug_read(long long* host_buf) {
  DI_CHECK_ARG(host_buf, "di_tc_debug_read: null buffer");
  if (cudaMemcpyFromSymbol(host_buf, g_dbg, sizeof(long long) * DBG_SLOTS * DBG_N) != cudaSuccess) {
    di_set_error("di_tc_debug_read: copy failed");
    return DI_ERR_LAUNCH;
  }
  return DI_OK;
}

// Tensor-core (wgmma + TMA) versions of di_linear_f32: C = act([A0|A1|A2] W^T + bias + res).
//   di_linear_tc_f32 : 3xTF32.  W_hi / W_lo fp32 [N, K]: hi = tf32(W), lo = W - hi.        every K_s % 32 == 0
//   di_linear_tcb_f32: bf16 split.  W_hi / W_mid bf16 [N, K]: hi = bf16(W), mid = bf16(W - hi).  every K_s % 64 == 0
// Common constraints: lda % 4 == 0, ldc % 4 == 0, 16-byte aligned pointers.  Return DI_ERR_UNSUPPORTED (-3) when a
// constraint is not met so that the caller can fall back (tcb -> tc -> di_linear_f32).
int di_linear_tc_f32(const float* A0, int lda0, int K0, const float* A1, int lda1, int K1, const float* A2, int lda2,
                     int K2, const float* W_hi, const float* W_lo, const float* bias, const float* res, int ldres,
                     int res_mod, float* C, int ldc, int M, int N, int act, cudaStream_t stream) {
  return linear_tc_impl("di_linear_tc_f32", 0, A0, lda0, K0, A1, lda1, K1, A2, lda2, K2, W_hi, W_lo, bias, res, ldres,
                        res_mod, C, ldc, M, N, act, 0, 0, stream);
}
int di_linear_tcb_f32(const float* A0, int lda0, int K0, const float* A1, int lda1, int K1, const float* A2, int lda2,
                      int K2, const void* W_hi, const void* W_mid, const float* bias, const float* res, int ldres,
                      int res_mod, float* C, int ldc, int M, int N, int act, cudaStream_t stream) {
  return linear_tc_impl("di_linear_tcb_f32", 1, A0, lda0, K0, A1, lda1, K1, A2, lda2, K2, W_hi, W_mid, bias, res, ldres,
                        res_mod, C, ldc, M, N, act, 0, 0, stream);
}
// di_linear_tcb_f32 whose output columns >= split_col0 are written pre-split for di_lcab_window_pre_f32
// (split_kind 1 = Q / K layout, 2 = V layout; see split_block above; split_col0 % 32 == 0, N % 32 == 0) or for
// di_lcab_window_tc_f32 (split_kind 3 = planar: per 128 channels 64 words of bf16 hi, then 64 words of bf16 mid;
// split_col0 % 128 == 0, N % 128 == 0).
int di_linear_tcb_split_f32(const float* A0, int lda0, int K0, const float* A1, int lda1, int K1, const float* A2,
                            int lda2, int K2, const void* W_hi, const void* W_mid, const float* bias, const float* res,
                            int ldres, int res_mod, float* C, int ldc, int M, int N, int act, int split_col0,
                            int split_kind, cudaStream_t stream) {
  return linear_tc_impl("di_linear_tcb_split_f32", 1, A0, lda0, K0, A1, lda1, K1, A2, lda2, K2, W_hi, W_mid, bias, res,
                        ldres, res_mod, C, ldc, M, N, act, split_col0, split_kind, stream);
}

// Tensor-core 3x3 convolution (stride 1, zero pad 1) over a pixel-major map: x [N,H,W,Cin] -> y [N,H,W,Cout],
// w_hi / w_lo [Cout][(ky*3+kx)*Cin + ci] (fp32 tf32-split, Cin % 32 == 0) or bf16 hi / mid (Cin % 64 == 0).
int di_conv3x3_tc_f32(const float* x, const float* w_hi, const float* w_lo, const float* bias, float* y, int N, int Cin,
                      int H, int W, int Cout, int act, cudaStream_t stream) {
  return conv3x3_tc_impl("di_conv3x3_tc_f32", 0, 0, x, w_hi, w_lo, bias, y, N, Cin, H, W, Cout, act, stream);
}
int di_conv3x3_tcb_f32(const float* x, const void* w_hi, const void* w_mid, const float* bias, float* y, int N, int Cin,
                       int H, int W, int Cout, int act, cudaStream_t stream) {
  return conv3x3_tc_impl("di_conv3x3_tcb_f32", 1, 0, x, w_hi, w_mid, bias, y, N, Cin, H, W, Cout, act, stream);
}
// Same convolutions reading an NCHW input x [N,Cin,H,W] directly (W % 4 == 0); y stays pixel-major [N,H,W,Cout].
// The boundary tensors of the path are NCHW (deepinteraction_encoder.py:47-62): no transposition pass is needed.
int di_conv3x3_tc_nchw_f32(const float* x, const float* w_hi, const float* w_lo, const float* bias, float* y, int N,
                           int Cin, int H, int W, int Cout, int act, cudaStream_t stream) {
  return conv3x3_tc_impl("di_conv3x3_tc_nchw_f32", 0, 1, x, w_hi, w_lo, bias, y, N, Cin, H, W, Cout, act, stream);
}
int di_conv3x3_tcb_nchw_f32(const float* x, const void* w_hi, const void* w_mid, const float* bias, float* y, int N,
                            int Cin, int H, int W, int Cout, int act, cudaStream_t stream) {
  return conv3x3_tc_impl("di_conv3x3_tcb_nchw_f32", 1, 1, x, w_hi, w_mid, bias, y, N, Cin, H, W, Cout, act, stream);
}

}  // extern "C"
