// Tensor-core 3x3 convolution (stride 1, zero pad 1) over a pixel-major map, as an implicit GEMM with the split
// products of gemm_tc.cu:  y[pixel, co] = act(sum_{tap, ci} x[pixel + tap - (1, 1), ci] * w[co, tap * Cin + ci] + b[co]).
// Reference layers: models/necks/deepinteraction_encoder.py:47-62, models/dense_heads/deepinteraction_decoder.py:83-101.
//
// A CTA tile is ty x tx output pixels (at most 128 GEMM rows; 8 x 16 unless another shape needs fewer rounds over the
// grid, see conv3x3_nhwc) by NT output channels (NT = 128, or 16 when Cout <= 16).
//   3xTF32 (KE = 32 channels per chunk): per chunk ONE TMA box loads the tile plus its one-pixel halo, (ty + 2) x
//     (tx + 2) pixels (zero-filled outside the image), into a 2-stage ring, and all nine taps read their A fragments
//     from it at a shifted pixel.  A warp's 8 fragment rows are 8 consecutive pixels; within one tile row they are 8
//     consecutive halo rows, whose 128-byte swizzle puts them in distinct bank groups.  Steps run chunk-major.
//   bf16 split (KE = 64): per (tap, chunk) a box of the tile shifted by the tap lands in the weight stage, and the
//     steps run tap-major.  That is the summation order of the encoder's shared convolutions before this kernel, so
//     their outputs keep their bits; at Cin = 256 / 512 the halo of every chunk would not fit in shared memory.
// The weights stream per (tap, chunk) through a ring of [A |] W_hi | W_lo stages.
//
// Persistent CTAs (at most one per SM, capped by di_tc_set_sm_limit) walk the tiles with a static stride: graphs replay
// on concurrent streams, so no tile counter lives in global memory.  384 threads: warpgroup 0 is the one-thread TMA
// producer; warpgroups 1-2 consume 64 rows each.  The products and their order inside a (tap, chunk) step are those of
// gemm_tc.cu (bf16 split: A_mid W_hi, A_hi W_mid, A_hi W_hi into one accumulator; 3xTF32: A_lo W_hi + A_hi W_lo into a
// second accumulator added in the epilogue).  A consumer keeps one wgmma group
// (two k-steps) in flight while it splits the next group's A fragments into a second register buffer, and releases a
// weight stage (and, after a chunk's last tap, the halo) once wgmma.wait_group has retired the groups that read it.
#include "tc_common.cuh"

namespace {

using namespace tc;

constexpr int TM = 128;                              // GEMM rows per tile: ty x tx <= TM output pixels
constexpr int HBOX = 23 * 1024;                      // slot of one 32-channel halo box, (ty + 2) (tx + 2) <= 184 pixels
constexpr int NTHREADS = 384;
constexpr int RING_BYTES = 220 * 1024;
constexpr int BAR_BYTES = 256;
constexpr int SMEM_BYTES = RING_BYTES + 1024 /*alignment*/ + BAR_BYTES;
static_assert(SMEM_BYTES <= 232448, "conv_tc exceeds the 227 KB shared-memory limit");

struct ConvParams {
  int H, W, ty, tx, tiles_x, tiles_y;
  int m_tiles, n_tiles, nch;   // pixel tiles, column tiles, channel chunks
  int Cin, Cout;
  float* y;
  const float* bias;
  int act;
};

template <bool BF, int NT>
__global__ void __launch_bounds__(NTHREADS, 1)
conv3x3_tc_kernel(const __grid_constant__ CUtensorMap mapX, const __grid_constant__ CUtensorMap mapWhi,
                  const __grid_constant__ CUtensorMap mapWlo, const ConvParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint8_t* base_ptr = smem_raw + (base - smem_u32(smem_raw));
  constexpr int KE = BF ? 64 : 32;                   // channels per chunk
  constexpr int NB = KE / 32;                        // 32-channel A boxes per chunk
  constexpr bool HALO = !BF;                         // else one shifted tile box per (tap, chunk), in the stage
  constexpr int HSTG = HALO ? NB * HBOX : 0;         // halo stage (double-buffered)
  constexpr int ABOX = HALO ? HBOX : TM * 128;       // bytes between the 32-channel boxes of a chunk
  constexpr int AL = HALO ? 0 : NB * ABOX;           // A landing bytes per weight stage
  constexpr int WT = NT * 128;                       // one weight tile: NT rows x 128 B
  constexpr int WSTG = AL + 2 * WT;                  // [A |] W_hi | W_lo
  constexpr int S = (RING_BYTES - 2 * HSTG) / WSTG < 8 ? (RING_BYTES - 2 * HSTG) / WSTG : 8;
  static_assert(S >= 3, "weight ring too short");
  constexpr int W_OFF = 2 * HSTG;
  constexpr int NCONS_WARPS = 8;
  const uint32_t bars = base + RING_BYTES;
  auto w_full = [&](int s) { return bars + 8u * s; };
  auto w_empty = [&](int s) { return bars + 8u * (S + s); };
  auto h_full = [&](int i) { return bars + 8u * (2 * S + i); };
  auto h_empty = [&](int i) { return bars + 8u * (2 * S + 2 + i); };
  static_assert(8 * (2 * S + 4) <= BAR_BYTES, "barrier block overflow");

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 1 && lane < 3) {
    const CUtensorMap* mp = lane == 0 ? &mapX : lane == 1 ? &mapWhi : &mapWlo;
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(mp)) : "memory");
  }
  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(w_full(s), 1);
      mbar_init(w_empty(s), NCONS_WARPS);
    }
    for (int i = 0; i < 2; ++i) {
      mbar_init(h_full(i), 1);
      mbar_init(h_empty(i), NCONS_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int num_tiles = p.m_tiles * p.n_tiles;
  // halo: chunk-major, tap-minor (a chunk's nine taps share its halo); per-tap boxes: tap-major, the order of the
  // one-box-per-tap GEMM, so those results keep their bits
  auto step_order = [&](int step, int& tap, int& kc) {
    if (HALO) {
      kc = step / 9;
      tap = step - 9 * kc;
    } else {
      tap = step / p.nch;
      kc = step - tap * p.nch;
    }
  };
  auto tile_coords = [&](int tile, int& n0, int& img, int& y0, int& x0) {
    const int mt = tile / p.n_tiles;
    n0 = (tile - mt * p.n_tiles) * NT;
    img = mt / (p.tiles_x * p.tiles_y);
    const int t = mt - img * p.tiles_x * p.tiles_y;
    y0 = (t / p.tiles_x) * p.ty;
    x0 = (t % p.tiles_x) * p.tx;
  };

  if (warp < 4) {
    // ---------------- TMA producer ----------------
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      int it = 0, hc = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int n0, img, y0, x0;
        tile_coords(tile, n0, img, y0, x0);
        for (int step = 0; step < 9 * p.nch; ++step, ++it) {
          int tap, kc;
          step_order(step, tap, kc);
          if (HALO && tap == 0) {
            const int hb = hc & 1;
            if (hc >= 2) mbar_wait(h_empty(hb), ((hc >> 1) - 1) & 1);
            mbar_expect_tx(h_full(hb), NB * (p.ty + 2) * (p.tx + 2) * 128);
            for (int b = 0; b < NB; ++b)
              tma_load_4d(base + hb * HSTG + b * HBOX, &mapX, h_full(hb), kc * KE + 32 * b, x0 - 1, y0 - 1, img);
            ++hc;
          }
          const int s = it % S;
          if (it >= S) mbar_wait(w_empty(s), ((it / S) - 1) & 1);
          const uint32_t st = base + W_OFF + s * WSTG;
          const int kw = tap * p.Cin + kc * KE;
          mbar_expect_tx(w_full(s), (HALO ? 0 : NB * p.ty * p.tx * 128) + 2 * WT);
          if (!HALO)
            for (int b = 0; b < NB; ++b)
              tma_load_4d(st + b * ABOX, &mapX, w_full(s), kc * KE + 32 * b, x0 + tap % 3 - 1, y0 + tap / 3 - 1, img);
          tma_load_2d(st + AL, &mapWhi, w_full(s), kw, n0);
          tma_load_2d(st + AL + WT, &mapWlo, w_full(s), kw, n0);
        }
      }
    }
  } else {
    // ---------------- consumers (warpgroups 1, 2): 64 rows each ----------------
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int wg = (warp >> 2) - 1, wl = warp & 3;
    const int g = lane >> 2, t = lane & 3;
    const int r0 = wg * 64 + wl * 16 + g, r1 = r0 + 8;   // tile rows of this thread's fragments
    // box row of tile row r: in the tap's own box r itself; in the halo the pixel at tap (0, 0), to which tap (dy, dx)
    // adds dy * (tx + 2) + dx.  Rows past the tile's ty * tx pixels read its last pixel and are not stored.
    const int npx = p.ty * p.tx;
    auto box_row = [&](int r) {
      r = min(r, npx - 1);
      return HALO ? (r / p.tx) * (p.tx + 2) + r % p.tx : r;
    };
    const int brow0 = box_row(r0), brow1 = box_row(r1);
    constexpr int NACC = NT / 2;
    constexpr int NX = BF ? 1 : NACC;
    float acc[NACC], accx[NX];
    // A fragments of the two k-step groups of a step: group hf is split into buffer hf while the other group's wgmma
    // run, so a buffer is rewritten only after wgmma.wait_group 1 has retired the group that read it
    uint32_t ahi[2][2][4] = {}, alo[2][2][4] = {};
    int it = 0, hc = 0;
    int rel_s = -1, rel_h = -1;                      // stage (and halo, after a chunk's last tap) still being read
    auto release = [&]() {
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(w_empty(rel_s));
        if (rel_h >= 0) mbar_arrive(h_empty(rel_h));
      }
    };
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int n0, img, y0, x0;
      tile_coords(tile, n0, img, y0, x0);
      for (int step = 0; step < 9 * p.nch; ++step, ++it) {
        int tap, kc;
        step_order(step, tap, kc);
        const int hb = hc & 1;
        if (HALO && tap == 0) mbar_wait(h_full(hb), (hc >> 1) & 1);
        const int s = it % S;
        const uint32_t st = base + W_OFF + s * WSTG;
        mbar_wait(w_full(s), (it / S) & 1);
        const float* abox = reinterpret_cast<const float*>(base_ptr + (HALO ? hb * HSTG : W_OFF + s * WSTG));
        // box rows of r0, r1: the halo row shifted by the tap, or the tile row in the tap's own box
        const int tap_off = HALO ? (tap / 3) * (p.tx + 2) + tap % 3 : 0;
        const int hr0 = brow0 + tap_off, hr1 = brow1 + tap_off;
        {
          // A element pair (k, k + 1) of box row hr, k even: 128B swizzle, 16-byte chunk (k / 4) ^ (hr & 7)
          auto a_pair = [&](int hr, int k) -> float2 {
            const int b = k >> 5, kk = k & 31;
            return *reinterpret_cast<const float2*>(abox + b * (ABOX / 4) + hr * 32 + (((kk >> 2) ^ (hr & 7)) << 2) +
                                                    (kk & 3));
          };
          auto a_at = [&](int hr, int k) -> float {
            return abox[hr * 32 + (((k >> 2) ^ (hr & 7)) << 2) + (k & 3)];
          };
#pragma unroll
          for (int hf = 0; hf < 2; ++hf) {              // two k-steps per wgmma group
#pragma unroll
            for (int u = 0; u < 2; ++u) {
              const int ks = 2 * hf + u;
              if (BF) {
                const int kb = 16 * ks + 2 * t;
                const float2 x[4] = {a_pair(hr0, kb), a_pair(hr1, kb), a_pair(hr0, kb + 8), a_pair(hr1, kb + 8)};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                  const uint32_t h = pack_bf16x2(x[e].x, x[e].y);
                  ahi[hf][u][e] = h;
                  alo[hf][u][e] = pack_bf16x2(x[e].x - __uint_as_float(h << 16), x[e].y - __uint_as_float(h & 0xFFFF0000u));
                }
              } else {
                const int kb = 8 * ks + t;
                const float x[4] = {a_at(hr0, kb), a_at(hr1, kb), a_at(hr0, kb + 4), a_at(hr1, kb + 4)};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                  ahi[hf][u][e] = (__float_as_uint(x[e]) + 0x1000u) & 0xFFFFE000u;    // round to nearest tf32
                  alo[hf][u][e] = __float_as_uint(x[e] - __uint_as_float(ahi[hf][u][e]));   // exact remainder
                }
              }
            }
            fence_regs(acc);
            if (!BF) fence_regs(accx);
            wgmma_fence();
#pragma unroll
            for (int u = 0; u < 2; ++u) {
              const int ks = 2 * hf + u;
              const uint32_t first = (kc | tap | ks) != 0;
              const uint64_t w_hi = wgmma_desc(st + AL + ks * 32), w_lo = wgmma_desc(st + AL + WT + ks * 32);
              if constexpr (BF) {
                wgmma_bf16_rs(acc, alo[hf][u], w_hi, first);   // A_mid * W_hi
                wgmma_bf16_rs(acc, ahi[hf][u], w_lo, 1);       // A_hi * W_mid
                wgmma_bf16_rs(acc, ahi[hf][u], w_hi, 1);       // A_hi * W_hi
              } else {
                wgmma_tf32_rs(accx, alo[hf][u], w_hi, first);  // A_lo * W_hi
                wgmma_tf32_rs(accx, ahi[hf][u], w_lo, 1);      // A_hi * W_lo
                wgmma_tf32_rs(acc, ahi[hf][u], w_hi, first);   // A_hi * W_hi
              }
            }
            wgmma_commit();
            wgmma_wait_one();                            // the previous group has retired: its A buffer is free
#pragma unroll
            for (int u = 0; u < 2; ++u) {
              fence_regs(ahi[hf ^ 1][u]);
              fence_regs(alo[hf ^ 1][u]);
            }
            if (hf == 0 && rel_s >= 0) release();        // ... and with it the previous step's stage
          }
        }
        rel_s = s;
        rel_h = HALO && tap == 8 ? hb : -1;
        if (HALO && tap == 8) ++hc;
      }
      wgmma_wait_all();
      fence_regs(acc);
      if (!BF) fence_regs(accx);
      release();
      rel_s = -1;
      if constexpr (!BF) {
#pragma unroll
        for (int j = 0; j < NACC; ++j) acc[j] += accx[j];
      }
      // ---------------- epilogue: bias, activation, stores ----------------
      long long grow[2];
      bool rok[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = h ? r1 : r0;
        const int yy = y0 + row / p.tx, xx = x0 + row % p.tx;
        rok[h] = row < npx && yy < p.H && xx < p.W;
        grow[h] = ((long long)img * p.H + min(yy, p.H - 1)) * p.W + min(xx, p.W - 1);
      }
#pragma unroll
      for (int j = 0; j < NT / 8; ++j) {
        const int col = n0 + 8 * j + 2 * t;
        if (col < p.Cout && p.bias) {                   // Cout % 4 == 0: the pair is valid as a whole
          const float2 b2 = *reinterpret_cast<const float2*>(p.bias + col);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            acc[4 * j + 2 * h] += b2.x;
            acc[4 * j + 2 * h + 1] += b2.y;
          }
        }
      }
      if (p.act == DI_ACT_RELU) {
#pragma unroll
        for (int j = 0; j < NACC; ++j) acc[j] = fmaxf(acc[j], 0.f);
      } else if (p.act == DI_ACT_GELU) {
#pragma unroll
        for (int j = 0; j < NACC; ++j) acc[j] = 0.5f * acc[j] * (1.f + erff(acc[j] * 0.70710678118654752440f));
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (!rok[h]) continue;
        float* yrow = p.y + (size_t)grow[h] * p.Cout;
#pragma unroll
        for (int j = 0; j < NT / 8; ++j) {
          const int col = n0 + 8 * j + 2 * t;
          if (col < p.Cout) *reinterpret_cast<float2*>(yrow + col) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        }
      }
    }
  }
  __syncthreads();
}

// 4-D fp32 map over an NHWC tensor; box = 32 channels x bx x-pixels x by y-pixels x 1 image (a tile, or its halo)
bool make_map_x(CUtensorMap* m, const float* ptr, int N, int H, int W, int C, int bx, int by) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return false;
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)C * 4, (cuuint64_t)W * C * 4, (cuuint64_t)H * W * C * 4};
  cuuint32_t box[4] = {32, (cuuint32_t)bx, (cuuint32_t)by, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(ptr), dims, strides, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// 2-D map over a row-major weight [rows, cols] (bf16 or fp32); box = 128 bytes of columns x `box_rows` rows
bool make_map_w(CUtensorMap* m, const void* ptr, bool bf16, long long rows, long long cols, int box_rows) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return false;
  const int eb = bf16 ? 2 : 4;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)cols * eb};
  cuuint32_t box[2] = {(cuuint32_t)(128 / eb), (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  return enc(m, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(ptr), dims,
             strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
             CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

template <bool BF, int NT>
int launch(const char* name, const CUtensorMap maps[3], const ConvParams& p, int grid, cudaStream_t stream) {
  static DiSmemOnce once{};
  if (!di_smem_once(once, conv3x3_tc_kernel<BF, NT>, SMEM_BYTES)) {
    di_set_error("%s: cannot reserve %d bytes of shared memory", name, SMEM_BYTES);
    return DI_ERR_LAUNCH;
  }
  conv3x3_tc_kernel<BF, NT><<<grid, NTHREADS, SMEM_BYTES, stream>>>(maps[0], maps[1], maps[2], p);
  DI_CHECK_LAUNCH(name);
  return DI_OK;
}

}  // namespace

int tc::conv3x3_nhwc(const char* name, int bf, const float* x, const void* w_hi, const void* w_lo, const float* bias,
                     float* y, int N, int Cin, int H, int W, int Cout, int act, cudaStream_t stream) {
  const int NT = Cout <= 16 ? 16 : 128;
  int sms = 0;
  const int rc = sm_budget(name, &sms);
  if (rc != DI_OK) return rc;
  // Tile shape from the shape and the grid: every tile costs the same 128-row MMA steps, so the time is the largest
  // number of tiles a CTA walks.  8 x 16 unless another shape of 112..128 pixels needs fewer rounds over the grid
  // (at 180 x 180 on 132 SMs: 9 x 14 = 260 tiles in two rounds where 8 x 16 = 276 tiles need three).  A pixel's sum
  // runs through the same steps in any tile shape.
  const int n_tiles = di_cdiv(Cout, NT);
  int ty = 8, tx = 16;
  auto rounds = [&](int a, int b) { return di_cdiv((long long)N * di_cdiv(H, a) * di_cdiv(W, b) * n_tiles, sms); };
  for (int a = 4; a <= 16; ++a)
    for (int b = 8; b <= 32; ++b)
      if (a * b <= TM && a * b >= 112 && (a + 2) * (b + 2) * 128 <= HBOX && rounds(a, b) < rounds(ty, tx)) {
        ty = a;
        tx = b;
      }
  CUtensorMap maps[3];
  const long long K = 9ll * Cin;
  if (!(make_map_x(&maps[0], x, N, H, W, Cin, bf ? tx : tx + 2, bf ? ty : ty + 2) &&
        make_map_w(&maps[1], w_hi, bf, Cout, K, NT) &&
        make_map_w(&maps[2], w_lo, bf, Cout, K, NT))) {
    di_set_error("%s: cuTensorMapEncodeTiled failed", name);
    return DI_ERR_LAUNCH;
  }
  ConvParams p{};
  p.H = H; p.W = W; p.ty = ty; p.tx = tx; p.tiles_x = di_cdiv(W, tx); p.tiles_y = di_cdiv(H, ty);
  p.m_tiles = N * p.tiles_x * p.tiles_y; p.n_tiles = n_tiles; p.nch = Cin / (bf ? 64 : 32);
  p.Cin = Cin; p.Cout = Cout; p.y = y; p.bias = bias; p.act = act;
  const int tiles = p.m_tiles * p.n_tiles, grid = tiles < sms ? tiles : sms;
  if (bf) return NT == 16 ? launch<true, 16>(name, maps, p, grid, stream) : launch<true, 128>(name, maps, p, grid, stream);
  return NT == 16 ? launch<false, 16>(name, maps, p, grid, stream) : launch<false, 128>(name, maps, p, grid, stream);
}
