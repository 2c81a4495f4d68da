// MMPI loss path on the GPU (SURVEY.md 8(f) rank 3): matching costs, Hungarian assignment, targets, gaussian heat-map
// targets and the three losses, without a host round trip (the reference copies every cost matrix to the CPU and runs
// scipy's linear_sum_assignment per layer and sample, hungarian_assigner.py:132-138).
//
// Reference: projects/mmdet3d_plugin/core/bbox/assigners/hungarian_assigner.py:14-47 (costs), :94-153 (assignment),
// models/dense_heads/deepinteraction_decoder.py:355-482 (targets), :484-547 (losses).  Third-party semantics restated
// from their published behaviour (mmdet 2.14 FocalLossCost / FocalLoss / L1Loss / GaussianFocalLoss, mmdet3d 0.17.1
// BboxOverlaps3D, gaussian_radius, draw_heatmap_gaussian): see oracle/loss.py part 2.
//
// Layouts: predictions are the forward's [B, k, L*P] tensors (L layers of P proposals on the last axis); ground truth
// is padded to Gmax boxes per sample with a count per sample.
#include "common.cuh"

namespace {

// ---------------------------------------------------------------------------------------------------------------------
// rotated rectangle intersection (BEV), mmdet3d 0.17 yaw convention: x' = x cos + y sin, y' = -x sin + y cos
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void rect_corners(float x, float y, float dx, float dy, float r, float (&cx)[4], float (&cy)[4]) {
  const float c = cosf(r), s = sinf(r);
  const float sx[4] = {-1.f, 1.f, 1.f, -1.f}, sy[4] = {-1.f, -1.f, 1.f, 1.f};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float lx = sx[k] * dx * 0.5f, ly = sy[k] * dy * 0.5f;
    cx[k] = lx * c + ly * s + x;
    cy[k] = -lx * s + ly * c + y;
  }
}

// Sutherland-Hodgman: rectangle A clipped by the four half planes of rectangle B -> area of the intersection
__device__ float rect_intersection(const float* a, const float* b) {
  const float ra = 0.5f * sqrtf(a[2] * a[2] + a[3] * a[3]), rb = 0.5f * sqrtf(b[2] * b[2] + b[3] * b[3]);
  const float ddx = a[0] - b[0], ddy = a[1] - b[1];
  if (ddx * ddx + ddy * ddy > (ra + rb) * (ra + rb)) return 0.f;
  // coordinates relative to B's centre: the shoelace products then involve metres, not the +-54 m scene offsets
  // (fp32 cancellation would otherwise cost ~1e-4 of absolute area)
  float px[8], py[8], qx[4], qy[4];
  {
    float ax[4], ay[4];
    rect_corners(ddx, ddy, a[2], a[3], a[4], ax, ay);
#pragma unroll
    for (int k = 0; k < 4; ++k) { px[k] = ax[k]; py[k] = ay[k]; }
  }
  rect_corners(0.f, 0.f, b[2], b[3], b[4], qx, qy);
  const float orient = (qx[1] - qx[0]) * (qy[2] - qy[1]) - (qy[1] - qy[0]) * (qx[2] - qx[1]);
  const float sgn = orient < 0.f ? -1.f : 1.f;
  int n = 4;
  for (int e = 0; e < 4 && n > 0; ++e) {
    const float p0x = qx[e], p0y = qy[e], ex = qx[(e + 1) & 3] - p0x, ey = qy[(e + 1) & 3] - p0y;
    float nx[8], ny[8];
    int m = 0;
    for (int k = 0; k < n; ++k) {
      const int k1 = k + 1 == n ? 0 : k + 1;
      const float sa = sgn * (ex * (py[k] - p0y) - ey * (px[k] - p0x));
      const float sb = sgn * (ex * (py[k1] - p0y) - ey * (px[k1] - p0x));
      if (sa >= 0.f && m < 8) { nx[m] = px[k]; ny[m] = py[k]; ++m; }
      if (((sa > 0.f && sb < 0.f) || (sa < 0.f && sb > 0.f)) && m < 8) {
        const float t = sa / (sa - sb);
        nx[m] = px[k] + t * (px[k1] - px[k]);
        ny[m] = py[k] + t * (py[k1] - py[k]);
        ++m;
      }
    }
    n = m;
    for (int k = 0; k < n; ++k) { px[k] = nx[k]; py[k] = ny[k]; }
  }
  if (n < 3) return 0.f;
  float area = 0.f;
  for (int k = 0; k < n; ++k) {
    const int k1 = k + 1 == n ? 0 : k + 1;
    area += px[k] * py[k1] - py[k] * px[k1];
  }
  return 0.5f * fabsf(area);
}

// boxes (x, y, z_bottom, dx, dy, dz, yaw): BboxOverlaps3D(coordinate='lidar', mode='iou')
__device__ float iou3d(const float* p, const float* g) {
  const float oh = fmaxf(fminf(p[2] + p[5], g[2] + g[5]) - fmaxf(p[2], g[2]), 0.f);
  const float a5[5] = {p[0], p[1], p[3], p[4], p[6]}, b5[5] = {g[0], g[1], g[3], g[4], g[6]};
  const float o3 = rect_intersection(a5, b5) * oh;
  const float v1 = p[3] * p[4] * p[5], v2 = g[3] * g[4] * g[5];
  return o3 / fmaxf(v1 + v2 - o3, 1e-8f);
}

struct CostParams {
  float cls_w, alpha, gamma, eps;       // FocalLossCost
  float reg_w;                          // BBoxBEVL1Cost (reg_kind 0) / BBox3DL1Cost (reg_kind 1)
  int reg_kind;
  float iou_w;                          // IoU3DCost
  float x0, y0, xr, yr;                 // point_cloud_range start and extent (BEV)
};

// cost[b, l, i, j] and iou[b, l, i, j] for i < P, j < n_gt[b];  score [B, K, LP] logits; boxes [B, LP, nb]
__global__ void match_cost_kernel(const float* __restrict__ boxes, int nb, const float* __restrict__ score, int K,
                                  const float* __restrict__ gt, const int* __restrict__ gt_labels, const int* __restrict__ n_gt,
                                  int Gmax, int LP, CostParams cp, float* __restrict__ cost, float* __restrict__ iou) {
  const int b = blockIdx.z;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;       // proposal over all layers
  const int j = blockIdx.y;
  if (i >= LP || j >= n_gt[b]) return;
  const float* p = boxes + ((size_t)b * LP + i) * nb;
  const float* g = gt + ((size_t)b * Gmax + j) * nb;
  const int lab = gt_labels[b * Gmax + j];
  const float x = score[((size_t)b * K + lab) * LP + i];
  const float pr = 1.f / (1.f + expf(-x));
  const float neg = -logf(1.f - pr + cp.eps) * (1.f - cp.alpha) * powf(pr, cp.gamma);
  const float pos = -logf(pr + cp.eps) * cp.alpha * powf(1.f - pr, cp.gamma);
  const float c_cls = (pos - neg) * cp.cls_w;
  float c_reg;
  if (cp.reg_kind == 0) {
    c_reg = fabsf((p[0] - cp.x0) / cp.xr - (g[0] - cp.x0) / cp.xr) + fabsf((p[1] - cp.y0) / cp.yr - (g[1] - cp.y0) / cp.yr);
  } else {
    c_reg = 0.f;
    for (int d = 0; d < nb; ++d) c_reg += fabsf(p[d] - g[d]);
  }
  c_reg *= cp.reg_w;
  const float u = iou3d(p, g);
  const size_t o = ((size_t)b * LP + i) * Gmax + j;
  cost[o] = (c_cls + c_reg) + (-u) * cp.iou_w;
  iou[o] = u;
}

// ---------------------------------------------------------------------------------------------------------------------
// Rectangular linear sum assignment (shortest augmenting paths with dual variables; the formulation of D. F. Crouse,
// "On implementing 2D rectangular assignment algorithms", 2016, which scipy.optimize.linear_sum_assignment implements).
// One warp per (sample, layer) problem, float64 like scipy.  Ties are broken as scipy breaks them, because the reference's
// matching is scipy's: the [P, G] cost matrix is transposed only when G < P (so the outer loop runs over the smaller
// side), and each step scans the unvisited columns in scipy's `remaining` order (reversed at the start of each row,
// shrunk by swap-removal), taking the first column of least cost unless a later one of that cost is unassigned, in which
// case the last such one.  gt_inds [B, LP]: 0 = background, j + 1 = matched to box j.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32)
hungarian_kernel(const float* __restrict__ cost, const float* __restrict__ iou, const int* __restrict__ n_gt, int P, int L,
                 int Gmax, long long* __restrict__ gt_inds, float* __restrict__ max_overlaps) {
  extern __shared__ double sm[];
  const int b = blockIdx.x / L, l = blockIdx.x % L, lane = threadIdx.x;
  const int G = n_gt[b];
  const int LP = L * P;
  long long* gi = gt_inds + (size_t)b * LP + (size_t)l * P;
  float* mo = max_overlaps + (size_t)b * LP + (size_t)l * P;
  for (int i = lane; i < P; i += 32) { gi[i] = 0; mo[i] = 0.f; }
  if (G == 0) return;
  const float* C = cost + ((size_t)b * LP + (size_t)l * P) * Gmax;       // C[i * Gmax + j]
  const bool tr = G < P;                   // rows of the solver = ground-truth boxes when there are fewer of them
  const int nr = tr ? G : P, nc = tr ? P : G;
  auto cst = [&](int r, int c) -> double { return tr ? (double)C[(size_t)c * Gmax + r] : (double)C[(size_t)r * Gmax + c]; };
  const int NMAX = max(P, Gmax);
  double* u = sm;                          // [NMAX] row duals
  double* v = u + NMAX;                    // [NMAX] column duals
  double* spc = v + NMAX;                  // [NMAX] shortest path costs
  int* path = reinterpret_cast<int*>(spc + NMAX);
  int* col4row = path + NMAX;
  int* row4col = col4row + NMAX;
  int* SR = row4col + NMAX;
  int* SC = SR + NMAX;
  int* rem = SC + NMAX;                    // scipy's `remaining`: the unvisited columns, in its scan order
  for (int k = lane; k < NMAX; k += 32) { u[k] = 0.0; v[k] = 0.0; col4row[k] = -1; row4col[k] = -1; }
  __syncwarp();
  const double INF = 1e300;
  // scan position `it` of cost s (free: unassigned column) beats the best so far: the least cost; among equal costs an
  // unassigned column, the last one in scan order; else the first one (scipy's sequential `<`, `== && free` rule)
  auto better = [](double s, int fr, int it, double best, int bfree, int bit) {
    return s < best || (s == best && (fr > bfree || (fr == bfree && (fr ? it > bit : it < bit))));
  };
  for (int cur = 0; cur < nr; ++cur) {
    for (int k = lane; k < NMAX; k += 32) { spc[k] = INF; SR[k] = 0; SC[k] = 0; }
    for (int k = lane; k < nc; k += 32) rem[k] = nc - 1 - k;
    __syncwarp();
    double minVal = 0.0;
    int i = cur, sink = -1, nrem = nc;
    while (sink < 0) {
      if (lane == 0) SR[i] = 1;
      double best = INF;
      int bit = -1, bfree = 0;
      const double ui = u[i];
      for (int it = lane; it < nrem; it += 32) {
        const int j = rem[it];
        const double r = minVal + cst(i, j) - ui - v[j];
        if (r < spc[j]) { spc[j] = r; path[j] = i; }
        const double s = spc[j];
        const int fr = row4col[j] < 0;
        if (better(s, fr, it, best, bfree, bit)) { best = s; bit = it; bfree = fr; }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const double ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bit, o), of = __shfl_xor_sync(0xffffffffu, bfree, o);
        if (better(ob, of, oi, best, bfree, bit)) { best = ob; bit = oi; bfree = of; }
      }
      minVal = best;
      if (bit < 0) { sink = -2; break; }                      // infeasible (cannot happen with finite costs)
      const int j = rem[bit];
      if (row4col[j] < 0) sink = j; else i = row4col[j];
      __syncwarp();
      if (lane == 0) { SC[j] = 1; rem[bit] = rem[nrem - 1]; }
      --nrem;
      __syncwarp();
    }
    if (sink == -2) break;
    // dual update
    for (int r = lane; r < nr; r += 32)
      if (SR[r]) u[r] += (r == cur) ? minVal : minVal - spc[col4row[r]];
    for (int c = lane; c < nc; c += 32)
      if (SC[c]) v[c] -= minVal - spc[c];
    __syncwarp();
    // augment along the alternating path
    if (lane == 0) {
      int j = sink;
      while (true) {
        const int r = path[j];
        row4col[j] = r;
        const int t = col4row[r];
        col4row[r] = j;
        j = t;
        if (r == cur) break;
      }
    }
    __syncwarp();
  }
  for (int r = lane; r < nr; r += 32) {
    const int c = col4row[r];
    if (c < 0) continue;
    const int q = tr ? c : r, g = tr ? r : c;                  // proposal, ground-truth box
    gi[q] = g + 1;
    mo[q] = iou[((size_t)b * LP + (size_t)l * P + q) * Gmax + g];
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// targets of deepinteraction_decoder.py:400-441 (+ the on-image mask products of :501-509) and the per-layer positive counts
// ---------------------------------------------------------------------------------------------------------------------
struct TargetParams {
  float sx, sy, ox, oy;        // TransFusionBBoxCoder.encode
  int code, nb, num_classes;
  float pos_weight;
};

__global__ void loss_targets_kernel(const long long* __restrict__ gt_inds, const float* __restrict__ max_overlaps,
                                    const float* __restrict__ gt, const int* __restrict__ gt_labels, int Gmax,
                                    const unsigned char* __restrict__ mask, int mask_stride_l, int P, int L, int B,
                                    TargetParams tp, long long* __restrict__ labels, long long* __restrict__ label_w,
                                    float* __restrict__ bbox_t, float* __restrict__ bbox_w, float* __restrict__ ious,
                                    float* __restrict__ num_pos, float* __restrict__ iou_sum, int* __restrict__ pos_cnt) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int LP = L * P;
  if (t >= B * LP) return;
  const int b = t / LP, q = t - b * LP, l = q / P, i = q - l * P;
  const long long gi = gt_inds[t];
  const float ov = fminf(fmaxf(max_overlaps[t], 0.f), 1.f);
  ious[t] = ov;
  // mask[l'][b][i]: mask_stride_l == 0 -> no mask for this layer is encoded by the caller passing mask == nullptr
  float mk = 1.f;
  if (mask && mask_stride_l >= 0) {
    // base decoder: layers 0, 2 use mask l / 2 (mask_stride_l = 1 flags "even layers only"); ++: every layer its own
    if (mask_stride_l == 1) { if ((l & 1) == 0) mk = mask[((size_t)(l >> 1) * B + b) * P + i] ? 1.f : 0.f; }
    else mk = mask[((size_t)l * B + b) * P + i] ? 1.f : 0.f;
  }
  float* bt = bbox_t + (size_t)t * tp.code;
  float* bw = bbox_w + (size_t)t * tp.code;
  if (gi > 0) {
    const float* g = gt + ((size_t)b * Gmax + (gi - 1)) * tp.nb;
    bt[0] = (g[0] - tp.ox) / tp.sx;
    bt[1] = (g[1] - tp.oy) / tp.sy;
    bt[2] = g[2] + g[5] * 0.5f;
    bt[3] = logf(g[3]); bt[4] = logf(g[4]); bt[5] = logf(g[5]);
    bt[6] = sinf(g[6]); bt[7] = cosf(g[6]);
    if (tp.code == 10) { bt[8] = g[7]; bt[9] = g[8]; }
    for (int c = 0; c < tp.code; ++c) bw[c] = mk;
    labels[t] = gt_labels[b * Gmax + (gi - 1)];
    label_w[t] = (long long)((tp.pos_weight <= 0.f ? 1.f : tp.pos_weight) * mk);
    atomicAdd(num_pos + l, mk);
    atomicAdd(iou_sum + b, ov);
    atomicAdd(pos_cnt + b, 1);
  } else {
    for (int c = 0; c < tp.code; ++c) { bt[c] = 0.f; bw[c] = 0.f; }
    labels[t] = tp.num_classes;
    label_w[t] = (long long)mk;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// gaussian heat-map targets (deepinteraction_decoder.py:443-476): one CTA per ground-truth box
// ---------------------------------------------------------------------------------------------------------------------
struct HeatParams {
  float vx, vy, x0, y0;      // voxel_size[0|1], point_cloud_range[0|1]
  int osf, min_radius;
  float min_overlap;
  int X, Y, K;
};

__device__ __forceinline__ float gaussian_radius_f(float height, float width, float mo) {
  const float b1 = height + width, c1 = width * height * (1.f - mo) / (1.f + mo);
  const float r1 = (b1 + sqrtf(b1 * b1 - 4.f * c1)) / 2.f;
  const float b2 = 2.f * (height + width), c2 = (1.f - mo) * width * height;
  const float r2 = (b2 + sqrtf(b2 * b2 - 16.f * c2)) / 2.f;
  const float a3 = 4.f * mo, b3 = -2.f * mo * (height + width), c3 = (mo - 1.f) * width * height;
  const float r3 = (b3 + sqrtf(b3 * b3 - 4.f * a3 * c3)) / 2.f;
  return fminf(r1, fminf(r2, r3));
}

__global__ void gaussian_heatmap_kernel(const float* __restrict__ gt, int nb, const int* __restrict__ gt_labels,
                                        const int* __restrict__ n_gt, int Gmax, HeatParams hp, float* __restrict__ heat) {
  const int b = blockIdx.y, j = blockIdx.x;
  if (j >= n_gt[b]) return;
  const float* g = gt + ((size_t)b * Gmax + j) * nb;
  const float width = g[3] / hp.vx / (float)hp.osf, length = g[4] / hp.vy / (float)hp.osf;
  if (!(width > 0.f && length > 0.f)) return;
  const int radius = max(hp.min_radius, (int)gaussian_radius_f(length, width, hp.min_overlap));
  const int x = (int)((g[0] - hp.x0) / hp.vx / (float)hp.osf), y = (int)((g[1] - hp.y0) / hp.vy / (float)hp.osf);
  const int left = min(x, radius), right = min(hp.X - x, radius + 1), top = min(y, radius), bottom = min(hp.Y - y, radius + 1);
  const int w = right + left, h = bottom + top;
  if (w <= 0 || h <= 0) return;
  // python slices heatmap[y - top : y + bottom, x - left : x + right] (negative starts cannot occur: top <= y when y >= 0;
  // for y < 0 the start y - top is 0 and the extent y + bottom): same index arithmetic below, clipped to the map
  const double sigma = (double)(2 * radius + 1) / 6.0;
  float* plane = heat + ((size_t)b * hp.K + gt_labels[b * Gmax + j]) * hp.Y * hp.X;
  for (int t = threadIdx.x; t < w * h; t += blockDim.x) {
    const int dy = t / w - top, dx = t - (t / w) * w - left;
    const int yy = y + dy, xx = x + dx;
    if (yy < 0 || yy >= hp.Y || xx < 0 || xx >= hp.X) continue;
    const float val = (float)exp(-(double)(dx * dx + dy * dy) / (2.0 * sigma * sigma));
    atomicMax(reinterpret_cast<int*>(plane + (size_t)yy * hp.X + xx), __float_as_int(val));   // values >= 0
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// losses: per-block partial sums in double, fixed-order final sum (deterministic)
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double block_sum(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
    for (int k = 0; k < (int)(blockDim.x >> 5); ++k) s += red[k];
  __syncthreads();
  return s;
}

// GaussianFocalLoss(alpha 2, gamma 4) on clip_sigmoid(logits): part[blk] = sum, cnt[blk] = #(target == 1)
__global__ void __launch_bounds__(256)
heatmap_loss_kernel(const float* __restrict__ logit, const float* __restrict__ target, long long n, float alpha, float gamma,
                    double* __restrict__ part, double* __restrict__ cnt) {
  __shared__ double red[8];
  double s = 0.0, c = 0.0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float p = 1.f / (1.f + expf(-logit[i]));
    p = fminf(fmaxf(p, 1e-4f), 1.f - 1e-4f);
    const float t = target[i];
    const float posw = t == 1.f ? 1.f : 0.f, negw = powf(1.f - t, gamma);
    const float lp = -logf(p + 1e-12f) * powf(1.f - p, alpha) * posw;
    const float ln = -logf(1.f - p + 1e-12f) * powf(p, alpha) * negw;
    s += (double)(lp + ln);
    c += posw;
  }
  s = block_sum(s, red);
  c = block_sum(c, red);
  if (threadIdx.x == 0) { part[blockIdx.x] = s; cnt[blockIdx.x] = c; }
}

// per layer: sigmoid focal loss (background label == K) weighted per row, and weighted L1 of the box code
// score [B, K, LP]; preds: the five head tensors [B, k, LP]; out part [L, 2, nblk]
struct LayerLossParams {
  const float* center; const float* height; const float* dim; const float* rot; const float* vel;
  float code_w[10];
  float alpha, gamma;
  int K, P, L, B, code;
};

__global__ void __launch_bounds__(256)
layer_loss_kernel(const float* __restrict__ score, LayerLossParams lp, const long long* __restrict__ labels,
                  const long long* __restrict__ label_w, const float* __restrict__ bbox_t, const float* __restrict__ bbox_w,
                  double* __restrict__ part) {
  __shared__ double red[8];
  const int l = blockIdx.y, LP = lp.L * lp.P;
  double s_cls = 0.0, s_box = 0.0;
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < lp.B * lp.P; r += gridDim.x * blockDim.x) {
    const int b = r / lp.P, i = r - b * lp.P, q = l * lp.P + i;
    const size_t t = (size_t)b * LP + q;
    const float w = (float)label_w[t];
    const long long lab = labels[t];
    for (int c = 0; c < lp.K; ++c) {
      const float x = score[((size_t)b * lp.K + c) * LP + q];
      const float p = 1.f / (1.f + expf(-x));
      const float v = lab == c ? -lp.alpha * powf(1.f - p, lp.gamma) * logf(fmaxf(p, 1.17549435e-38f))
                               : -(1.f - lp.alpha) * powf(p, lp.gamma) * logf(fmaxf(1.f - p, 1.17549435e-38f));
      s_cls += (double)(v * w);
    }
    const float* bt = bbox_t + t * lp.code;
    const float* bw = bbox_w + t * lp.code;
    float pr[10];
    pr[0] = lp.center[((size_t)b * 2 + 0) * LP + q]; pr[1] = lp.center[((size_t)b * 2 + 1) * LP + q];
    pr[2] = lp.height[(size_t)b * LP + q];
    pr[3] = lp.dim[((size_t)b * 3 + 0) * LP + q]; pr[4] = lp.dim[((size_t)b * 3 + 1) * LP + q]; pr[5] = lp.dim[((size_t)b * 3 + 2) * LP + q];
    pr[6] = lp.rot[((size_t)b * 2 + 0) * LP + q]; pr[7] = lp.rot[((size_t)b * 2 + 1) * LP + q];
    if (lp.code == 10) { pr[8] = lp.vel[((size_t)b * 2 + 0) * LP + q]; pr[9] = lp.vel[((size_t)b * 2 + 1) * LP + q]; }
    for (int c = 0; c < lp.code; ++c) s_box += (double)(fabsf(pr[c] - bt[c]) * (bw[c] * lp.code_w[c]));
  }
  s_cls = block_sum(s_cls, red);
  s_box = block_sum(s_box, red);
  if (threadIdx.x == 0) {
    part[((size_t)l * 2 + 0) * gridDim.x + blockIdx.x] = s_cls;
    part[((size_t)l * 2 + 1) * gridDim.x + blockIdx.x] = s_box;
  }
}

// out[0] = heat-map loss, out[1 + 2 l] = cls loss of layer l, out[2 + 2 l] = bbox loss of layer l, out[1 + 2 L] = mean over
// samples of (sum of matched ious / max(#pos, 1))
__global__ void loss_finish_kernel(const double* __restrict__ hpart, const double* __restrict__ hcnt, int nh,
                                   const double* __restrict__ lpart, int nl, const float* __restrict__ num_pos,
                                   const float* __restrict__ iou_sum, const int* __restrict__ pos_cnt, int L, int B,
                                   float w_heat, float w_cls, float w_box, float* __restrict__ out) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  double s = 0.0, c = 0.0;
  for (int k = 0; k < nh; ++k) { s += hpart[k]; c += hcnt[k]; }
  out[0] = (float)(s / fmax(c, 1.0)) * w_heat;
  for (int l = 0; l < L; ++l) {
    double a = 0.0, bsum = 0.0;
    for (int k = 0; k < nl; ++k) { a += lpart[((size_t)l * 2 + 0) * nl + k]; bsum += lpart[((size_t)l * 2 + 1) * nl + k]; }
    const double af = fmax((double)num_pos[l], 1.0);
    out[1 + 2 * l] = (float)(a / af) * w_cls;
    out[2 + 2 * l] = (float)(bsum / af) * w_box;
  }
  double m = 0.0;
  for (int b = 0; b < B; ++b) m += (double)iou_sum[b] / (double)max(pos_cnt[b], 1);
  out[1 + 2 * L] = (float)(m / (double)B);
}

// ---------------------------------------------------------------------------------------------------------------------
// loss gradients: the avg factors come from the device (no .item()), one thread per output element, no atomics
// ---------------------------------------------------------------------------------------------------------------------
// cnt[blk] = #(target == 1) of the block's grid-stride share, as heatmap_loss_kernel counts it
__global__ void __launch_bounds__(256)
heat_count_kernel(const float* __restrict__ target, long long n, double* __restrict__ cnt) {
  __shared__ double red[8];
  double c = 0.0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    c += target[i] == 1.f ? 1.0 : 0.0;
  c = block_sum(c, red);
  if (threadIdx.x == 0) cnt[blockIdx.x] = c;
}

// scale[0] = g[0] w_heat / max(#ones, 1); scale[1 + 2 l] = g[1 + 2 l] w_cls / max(num_pos_l, 1); scale[2 + 2 l] likewise
// with w_box: d loss / d (one weighted term) of every loss, as loss_finish_kernel divides
__global__ void loss_bwd_scale_kernel(const double* __restrict__ hcnt, int nh, const float* __restrict__ num_pos, int L,
                                      const float* __restrict__ grad, float w_heat, float w_cls, float w_box,
                                      float* __restrict__ scale) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  double c = 0.0;
  for (int k = 0; k < nh; ++k) c += hcnt[k];
  scale[0] = (float)((double)grad[0] * (double)w_heat / fmax(c, 1.0));
  for (int l = 0; l < L; ++l) {
    const double af = fmax((double)num_pos[l], 1.0);
    scale[1 + 2 * l] = (float)((double)grad[1 + 2 * l] * (double)w_cls / af);
    scale[2 + 2 * l] = (float)((double)grad[2 + 2 * l] * (double)w_box / af);
  }
}

// d GaussianFocalLoss(clip_sigmoid(logit)) / d logit, written pixel-major [B, HW, 32] (channels K..31 = 0): the input
// layout of the transposed 3x3 convolution.  clip_sigmoid's clamp passes the gradient by torch's rule (zero strictly
// outside [1e-4, 1 - 1e-4]); the sigmoid's derivative is taken at the unclamped p.  One thread per 4 channels of a pixel.
__global__ void __launch_bounds__(256)
heatmap_loss_bwd_kernel(const float* __restrict__ logit, const float* __restrict__ target, int B, int K, int HW, float alpha,
                        float gamma, const float* __restrict__ scale, float* __restrict__ d_out) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)B * HW * 8) return;
  const int c4 = (int)(t & 7);
  const long long bp = t >> 3;
  const int b = (int)(bp / HW), pix = (int)(bp - (long long)b * HW);
  const float s = scale[0];
  float d[4];
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int c = c4 * 4 + u;
    d[u] = 0.f;
    if (c >= K) continue;
    const size_t i = ((size_t)b * K + c) * HW + pix;
    const float p = 1.f / (1.f + expf(-logit[i]));
    if (!(p >= 1e-4f && p <= 1.f - 1e-4f)) continue;
    const float tg = target[i];
    float g = 0.f;
    if (tg == 1.f)
      g = -powf(1.f - p, alpha) / (p + 1e-12f) + alpha * logf(p + 1e-12f) * powf(1.f - p, alpha - 1.f);
    else
      g = (powf(p, alpha) / (1.f - p + 1e-12f) - alpha * logf(1.f - p + 1e-12f) * powf(p, alpha - 1.f)) * powf(1.f - tg, gamma);
    d[u] = g * (p * (1.f - p)) * s;
  }
  reinterpret_cast<float4*>(d_out)[t] = make_float4(d[0], d[1], d[2], d[3]);
}

// d layer losses / d prediction rows [L, B*P, NP] in head order (centre, height, dim, rot[, vel], heatmap): the box-code
// columns take sign(pred - target) x bbox weight x code weight (0 at equality, as torch's abs), the K class columns
// mmcv's closed-form sigmoid focal gradient (FLT_MIN inside the logs only) x label weight.  A zero weight writes 0.
__global__ void __launch_bounds__(256)
layer_loss_bwd_kernel(const float* __restrict__ score, LayerLossParams lp, const long long* __restrict__ labels,
                      const long long* __restrict__ label_w, const float* __restrict__ bbox_t, const float* __restrict__ bbox_w,
                      const float* __restrict__ scale, float* __restrict__ d_pred) {
  const int NP = lp.code + lp.K, LP = lp.L * lp.P;
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)lp.L * lp.B * lp.P * NP) return;
  const int j = (int)(e % NP);
  const int r = (int)(e / NP);                                  // l * B*P + b * P + i
  const int l = r / (lp.B * lp.P), bi = r - l * (lp.B * lp.P), b = bi / lp.P, i = bi - b * lp.P, q = l * lp.P + i;
  const size_t t = (size_t)b * LP + q;
  float d = 0.f;
  if (j < lp.code) {
    const float w = bbox_w[t * lp.code + j] * lp.code_w[j];
    if (w != 0.f) {
      const float* src = j < 2 ? lp.center + ((size_t)b * 2 + j) * LP : j == 2 ? lp.height + (size_t)b * LP
                       : j < 6 ? lp.dim + ((size_t)b * 3 + (j - 3)) * LP : j < 8 ? lp.rot + ((size_t)b * 2 + (j - 6)) * LP
                       : lp.vel + ((size_t)b * 2 + (j - 8)) * LP;
      const float v = src[q] - bbox_t[t * lp.code + j];
      d = (v > 0.f ? 1.f : v < 0.f ? -1.f : 0.f) * w * scale[2 + 2 * l];
    }
  } else {
    const float w = (float)label_w[t];
    if (w != 0.f) {
      const int c = j - lp.code;
      const float p = 1.f / (1.f + expf(-score[((size_t)b * lp.K + c) * LP + q]));
      const float g = labels[t] == c
          ? -lp.alpha * powf(1.f - p, lp.gamma) * (1.f - p - lp.gamma * p * logf(fmaxf(p, 1.17549435e-38f)))
          : -(1.f - lp.alpha) * powf(p, lp.gamma) * (lp.gamma * (1.f - p) * logf(fmaxf(1.f - p, 1.17549435e-38f)) - p);
      d = g * w * scale[1 + 2 * l];
    }
  }
  d_pred[e] = d;
}

// HeuristicAssigner3D.assign (hungarian_assigner.py:60-91): every ground-truth box claims its nearest prediction (BEV centre
// distance, + dist_thre when the query's class differs); a prediction claimed twice keeps the nearer box (ties: the earlier
// box, the reference's strict `<`).  As in the reference, a claim must also be nearer than 10000, the distance an
// unclaimed prediction starts with.  One CTA; P, G small.
__global__ void __launch_bounds__(256)
heuristic_assign_kernel(const float* __restrict__ boxes, int nb, int P, const float* __restrict__ gt, const int* __restrict__ gt_labels,
                        int G, const int* __restrict__ query_labels, float dist_thre, long long* __restrict__ gt_inds,
                        float* __restrict__ overlaps, float* __restrict__ labels, int* __restrict__ nearest, float* __restrict__ ndist) {
  for (int i = threadIdx.x; i < P; i += blockDim.x) { gt_inds[i] = 0; overlaps[i] = 0.f; labels[i] = -1.f; }
  for (int g = threadIdx.x; g < G; g += blockDim.x) {
    const float gx = gt[(size_t)g * nb], gy = gt[(size_t)g * nb + 1];
    float best = INFINITY;
    int arg = 0;
    for (int i = 0; i < P; ++i) {
      const float dx = boxes[(size_t)i * nb] - gx, dy = boxes[(size_t)i * nb + 1] - gy;
      float d = sqrtf(dx * dx + dy * dy);
      if (query_labels && query_labels[i] != gt_labels[g]) d += dist_thre;
      if (d < best) { best = d; arg = i; }           // torch.min: first minimum
    }
    nearest[g] = arg;
    ndist[g] = best;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int g = 0; g < G; ++g) {
      const int i = nearest[g];
      const float d = ndist[g];
      if (d <= dist_thre && d < (gt_inds[i] == 0 ? 10000.f : overlaps[i])) {   // overlaps[] holds the claimed distance for now
        overlaps[i] = d;
        gt_inds[i] = g + 1;
        labels[i] = (float)gt_labels[g];
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < P; i += blockDim.x) {
    const long long gi = gt_inds[i];
    overlaps[i] = gi > 0 ? iou3d(gt + (size_t)(gi - 1) * nb, boxes + (size_t)i * nb) : 0.f;
  }
}

}  // namespace

extern "C" {

// boxes [B, LP, nb] decoded predictions (di_bbox_decode_f32), score [B, K, LP] class logits, gt [B, Gmax, nb] padded
// ground truth, gt_labels [B, Gmax] int32, n_gt [B] int32 (device).  params11 (host): cls_w, alpha, gamma, eps, reg_w,
// reg_kind (0 BBoxBEVL1Cost / 1 BBox3DL1Cost), iou_w, pc x0, y0, x extent, y extent.  cost / iou [B, LP, Gmax].
int di_match_cost_f32(const float* boxes, int nb, const float* score, int K, const float* gt, const int* gt_labels,
                      const int* n_gt, int B, int LP, int Gmax, const float* params11, float* cost, float* iou,
                      cudaStream_t stream) {
  DI_CHECK_ARG(boxes && score && gt && gt_labels && n_gt && params11 && cost && iou && B > 0 && LP > 0 && Gmax > 0 && nb >= 7 && nb <= 16,
               "di_match_cost_f32: bad argument");
  CostParams cp;
  cp.cls_w = params11[0]; cp.alpha = params11[1]; cp.gamma = params11[2]; cp.eps = params11[3]; cp.reg_w = params11[4];
  cp.reg_kind = (int)params11[5]; cp.iou_w = params11[6]; cp.x0 = params11[7]; cp.y0 = params11[8]; cp.xr = params11[9]; cp.yr = params11[10];
  dim3 grid(di_cdiv(LP, 128), Gmax, B);
  match_cost_kernel<<<grid, 128, 0, stream>>>(boxes, nb, score, K, gt, gt_labels, n_gt, Gmax, LP, cp, cost, iou);
  DI_CHECK_LAUNCH("di_match_cost_f32");
  return DI_OK;
}

// boxes [P, nb] predictions, gt [G, nb], gt_labels [G] int32, query_labels [P] int32 or NULL; work: int32 [G] + float [G];
// -> gt_inds [P] int64 (0 = unassigned, g + 1), max_overlaps [P] (3-D IoU of the matched pairs), labels [P] float (-1 unassigned)
int di_heuristic_assign_f32(const float* boxes, int nb, int P, const float* gt, const int* gt_labels, int G,
                            const int* query_labels, float dist_thre, long long* gt_inds, float* max_overlaps, float* labels,
                            void* work, cudaStream_t stream) {
  DI_CHECK_ARG(boxes && gt && gt_labels && gt_inds && max_overlaps && labels && work && P > 0 && G > 0 && nb >= 7,
               "di_heuristic_assign_f32: bad argument");
  heuristic_assign_kernel<<<1, 256, 0, stream>>>(boxes, nb, P, gt, gt_labels, G, query_labels, dist_thre, gt_inds, max_overlaps,
                                               labels, reinterpret_cast<int*>(work), reinterpret_cast<float*>(work) + G);
  DI_CHECK_LAUNCH("di_heuristic_assign_f32");
  return DI_OK;
}

// cost / iou [B, L*P, Gmax] -> gt_inds [B, L*P] int64 (0 background, j + 1 matched), max_overlaps [B, L*P]
int di_hungarian_f32(const float* cost, const float* iou, const int* n_gt, int B, int L, int P, int Gmax, long long* gt_inds,
                     float* max_overlaps, cudaStream_t stream) {
  DI_CHECK_ARG(cost && iou && n_gt && gt_inds && max_overlaps && B > 0 && L > 0 && P > 0 && Gmax > 0, "di_hungarian_f32: bad argument");
  const int nmax = P > Gmax ? P : Gmax;
  const int smem = nmax * (3 * (int)sizeof(double) + 6 * (int)sizeof(int));
  DI_CHECK_ARG(smem <= 200 * 1024, "di_hungarian_f32: problem too large (P=%d, G=%d)", P, Gmax);
  static DiSmemOnce once{};
  if (!di_smem_once(once, hungarian_kernel, 200 * 1024)) {
    di_set_error("di_hungarian_f32: cannot reserve shared memory");
    return DI_ERR_LAUNCH;
  }
  hungarian_kernel<<<B * L, 32, smem, stream>>>(cost, iou, n_gt, P, L, Gmax, gt_inds, max_overlaps);
  DI_CHECK_LAUNCH("di_hungarian_f32");
  return DI_OK;
}

// mask: uint8 [n_masks, B, P] or NULL; mask_mode 0 = none, 1 = base decoder (even layers use mask l/2), 2 = ++ (mask l).
// coder4 (host) = out_size_factor*voxel (x, y), pc_range (x, y).  num_pos [L], iou_sum [B], pos_cnt [B] must be zeroed.
int di_loss_targets_f32(const long long* gt_inds, const float* max_overlaps, const float* gt, const int* gt_labels, int Gmax,
                        const unsigned char* mask, int mask_mode, int B, int L, int P, int nb, int code, int num_classes,
                        float pos_weight, const float* coder4, long long* labels, long long* label_w, float* bbox_t,
                        float* bbox_w, float* ious, float* num_pos, float* iou_sum, int* pos_cnt, cudaStream_t stream) {
  DI_CHECK_ARG(gt_inds && max_overlaps && gt && gt_labels && coder4 && labels && label_w && bbox_t && bbox_w && ious && num_pos &&
               iou_sum && pos_cnt && (code == 8 || code == 10) && (code != 10 || nb == 9), "di_loss_targets_f32: bad argument");
  TargetParams tp;
  tp.sx = coder4[0]; tp.sy = coder4[1]; tp.ox = coder4[2]; tp.oy = coder4[3];
  tp.code = code; tp.nb = nb; tp.num_classes = num_classes; tp.pos_weight = pos_weight;
  loss_targets_kernel<<<di_cdiv((long long)B * L * P, 128), 128, 0, stream>>>(
      gt_inds, max_overlaps, gt, gt_labels, Gmax, mask_mode ? mask : nullptr, mask_mode == 1 ? 1 : 2, P, L, B, tp, labels,
      label_w, bbox_t, bbox_w, ious, num_pos, iou_sum, pos_cnt);
  DI_CHECK_LAUNCH("di_loss_targets_f32");
  return DI_OK;
}

// heat [B, K, Y, X] must be zeroed.  params7 (host): voxel x, y, range x0, y0, out_size_factor, min_radius, gaussian_overlap
int di_gaussian_heatmap_f32(const float* gt, int nb, const int* gt_labels, const int* n_gt, int B, int Gmax, int K, int Y, int X,
                            const float* params7, float* heat, cudaStream_t stream) {
  DI_CHECK_ARG(gt && gt_labels && n_gt && params7 && heat && B > 0 && Gmax > 0, "di_gaussian_heatmap_f32: bad argument");
  HeatParams hp;
  hp.vx = params7[0]; hp.vy = params7[1]; hp.x0 = params7[2]; hp.y0 = params7[3]; hp.osf = (int)params7[4];
  hp.min_radius = (int)params7[5]; hp.min_overlap = params7[6]; hp.X = X; hp.Y = Y; hp.K = K;
  gaussian_heatmap_kernel<<<dim3(Gmax, B), 128, 0, stream>>>(gt, nb, gt_labels, n_gt, Gmax, hp, heat);
  DI_CHECK_LAUNCH("di_gaussian_heatmap_f32");
  return DI_OK;
}

// work: double [2 * 256 + L * 2 * 64]; out: float [2 + 2 L] (see loss_finish_kernel).  weights3 / focal2 / gfl2 / code_w host.
int di_mmpi_losses_f32(const float* dense_logit, const float* heat_target, long long n_heat, const float* score,
                       const float* center, const float* height, const float* dim, const float* rot, const float* vel,
                       const long long* labels, const long long* label_w, const float* bbox_t, const float* bbox_w,
                       const float* num_pos, const float* iou_sum, const int* pos_cnt, int B, int K, int L, int P, int code,
                       const float* code_w, const float* focal2, const float* gfl2, const float* weights3, double* work,
                       float* out, cudaStream_t stream) {
  DI_CHECK_ARG(dense_logit && heat_target && score && center && height && dim && rot && labels && label_w && bbox_t && bbox_w &&
               num_pos && iou_sum && pos_cnt && code_w && focal2 && gfl2 && weights3 && work && out && (code == 8 || (code == 10 && vel)),
               "di_mmpi_losses_f32: bad argument");
  const int NH = 256, NL = 64;
  double* hpart = work;
  double* hcnt = work + NH;
  double* lpart = work + 2 * NH;
  heatmap_loss_kernel<<<NH, 256, 0, stream>>>(dense_logit, heat_target, n_heat, gfl2[0], gfl2[1], hpart, hcnt);
  LayerLossParams lp;
  lp.center = center; lp.height = height; lp.dim = dim; lp.rot = rot; lp.vel = vel;
  for (int c = 0; c < 10; ++c) lp.code_w[c] = c < code ? code_w[c] : 0.f;
  lp.gamma = focal2[0]; lp.alpha = focal2[1];
  lp.K = K; lp.P = P; lp.L = L; lp.B = B; lp.code = code;
  layer_loss_kernel<<<dim3(NL, L), 256, 0, stream>>>(score, lp, labels, label_w, bbox_t, bbox_w, lpart);
  loss_finish_kernel<<<1, 32, 0, stream>>>(hpart, hcnt, NH, lpart, NL, num_pos, iou_sum, pos_cnt, L, B, weights3[0], weights3[1],
                                          weights3[2], out);
  DI_CHECK_LAUNCH("di_mmpi_losses_f32");
  return DI_OK;
}

// The inputs of di_mmpi_losses_f32 (dense logits / targets [B, K, Y, X] with HW = Y * X), grad [2 + 2 L] (device): the
// upstream gradient of each output (the last, matched_ious, takes none).  -> d_heat [B, HW, 32] (pixel-major, channels
// K..31 written as 0), d_pred [L, B*P, code + K] (head order).  work: double [2 * 256 + L * 2 * 64], as the forward's.
int di_mmpi_losses_bwd_f32(const float* dense_logit, const float* heat_target, long long n_heat, int HW, const float* score,
                           const float* center, const float* height, const float* dim, const float* rot, const float* vel,
                           const long long* labels, const long long* label_w, const float* bbox_t, const float* bbox_w,
                           const float* num_pos, int B, int K, int L, int P, int code, const float* code_w, const float* focal2,
                           const float* gfl2, const float* weights3, const float* grad, double* work, float* d_heat,
                           float* d_pred, cudaStream_t stream) {
  DI_CHECK_ARG(dense_logit && heat_target && score && center && height && dim && rot && labels && label_w && bbox_t && bbox_w &&
               num_pos && code_w && focal2 && gfl2 && weights3 && grad && work && d_heat && d_pred && B > 0 && L > 0 && P > 0 &&
               HW > 0 && K > 0 && K <= 32 && n_heat == (long long)B * K * HW && (code == 8 || (code == 10 && vel)),
               "di_mmpi_losses_bwd_f32: bad argument");
  const int NH = 256;
  double* hcnt = work;
  float* scale = reinterpret_cast<float*>(work + NH);
  heat_count_kernel<<<NH, 256, 0, stream>>>(heat_target, n_heat, hcnt);
  loss_bwd_scale_kernel<<<1, 32, 0, stream>>>(hcnt, NH, num_pos, L, grad, weights3[0], weights3[1], weights3[2], scale);
  const long long nq = (long long)B * HW * 8;
  heatmap_loss_bwd_kernel<<<(unsigned)((nq + 255) / 256), 256, 0, stream>>>(dense_logit, heat_target, B, K, HW, gfl2[0], gfl2[1],
                                                                           scale, d_heat);
  LayerLossParams lp;
  lp.center = center; lp.height = height; lp.dim = dim; lp.rot = rot; lp.vel = vel;
  for (int c = 0; c < 10; ++c) lp.code_w[c] = c < code ? code_w[c] : 0.f;
  lp.gamma = focal2[0]; lp.alpha = focal2[1];
  lp.K = K; lp.P = P; lp.L = L; lp.B = B; lp.code = code;
  const long long ne = (long long)L * B * P * (code + K);
  layer_loss_bwd_kernel<<<(unsigned)((ne + 255) / 256), 256, 0, stream>>>(score, lp, labels, label_w, bbox_t, bbox_w, scale, d_pred);
  DI_CHECK_LAUNCH("di_mmpi_losses_bwd_f32");
  return DI_OK;
}

}  // extern "C"
