// Bilateral-grid colour correction (DESIGN 3.20; the fp64 model is oracle/bilagrid_oracle.py).
// grids[M, 12, L, Y, X]: channel c = 4 r + k is entry A[r][k] of a 3 x 4 affine colour matrix.  A
// pixel (px, py) of rgb[3, H, W] reads A by trilinear interpolation at
//   gx = (px + 1/2) / W (X - 1),  gy = (py + 1/2) / H (Y - 1),  gz = clamp(g, 0, 1) (L - 1),
//   g = 0.299 r + 0.587 g + 0.114 b  (the luminance of the input),
// and writes out = A[:, :3] rgb + A[:, 3].
//
//  k_bilagrid_slice      one CTA per (band of rows of one grid cell, batch item).  Every pixel of
//                        the CTA reads the same 2 x 2 spatial corners, so their L levels x 12
//                        channels are staged in shared memory once; the pixel loop reads 3 planes and
//                        writes 3 (HBM-bound).
//  k_bilagrid_slice_bwd  the same CTAs.  Each lane computes dL/drgb of its pixel and stages the
//                        pixel's terms (dL/dout, [rgb, 1], tx, ty, tz, z0) in shared memory; then the
//                        warp walks its 32 staged pixels one at a time, every lane owning one
//                        accumulator column (spatial corner j, column k of [rgb, 1], z corner m) for
//                        the three rows r.  A run of pixels with the same z0 (warp-uniform) is summed
//                        in registers and added to the warp's private [L][3][16] shared array only
//                        when z0 changes: no atomics, no bank conflicts (the two z corners sit 48
//                        words apart).  At the end the CTA sums its warps in warp order and issues one
//                        global atomicAdd per non-zero window element (4 L 12 per CTA, not 96 per
//                        pixel).
//  k_bilagrid_tv         total variation over the grids, its gradient, and per-CTA partial sums
//                        (double) that k_bilagrid_tv_sum adds in a fixed order: bit-reproducible.
#include <algorithm>

#include "common.cuh"
#include "kernels.h"

namespace gsb {

namespace {

constexpr int BG_THREADS = 256, BG_WARPS = BG_THREADS / 32;
constexpr int BG_BAND_PIXELS = 1024;  // pixels of one cell a CTA covers, about (whole rows)
constexpr int TV_THREADS = 256, TV_MAX_BLOCKS = 1056;

struct BgIds {
  int32_t id[BILAGRID_MAX_BATCH];
};
struct BgGeom {
  int L, Y, X, H, W;
  int ncx, ncy;      // cells per axis: max(X - 1, 1), max(Y - 1, 1)
  int rows, nbands;  // rows per band, bands per cell
};

// ((p + 1/2) / n) (G - 1), in this order and in fp32: the cell ranges and the per-pixel weights
// come from the same function, so every pixel lies in the cell of the CTA that owns it
__device__ __forceinline__ float grid_coord(int p, int n, int G) {
  return __fmul_rn(__fdiv_rn(__fadd_rn((float)p, 0.5f), (float)n), (float)(G - 1));
}
__device__ __forceinline__ int cell_of(float g, int G) { return G == 1 ? 0 : min((int)g, G - 2); }

// the first pixel of [0, n] whose cell is >= c (cell_of is monotone in p)
__device__ int cell_start(int c, int n, int G) {
  if (c <= 0) return 0;
  if (c >= max(G - 1, 1)) return n;
  int p = min(max((int)((float)c * ((float)n / (float)(G - 1))), 0), n);
  while (p > 0 && cell_of(grid_coord(p - 1, n, G), G) >= c) p--;
  while (p < n && cell_of(grid_coord(p, n, G), G) < c) p++;
  return p;
}

// the pixel rectangle [x0, x1) x [y0, y1) of CTA `blk`, in cell (cx, cy); false: empty
struct Band {
  int x0, x1, y0, y1, cx, cy;
};
__device__ __forceinline__ bool band_of(const BgGeom &g, int blk, Band &b) {
  const int cell = blk / g.nbands, band = blk - cell * g.nbands;
  b.cx = cell % g.ncx;
  b.cy = cell / g.ncx;
  b.x0 = cell_start(b.cx, g.W, g.X);
  b.x1 = cell_start(b.cx + 1, g.W, g.X);
  const int ys = cell_start(b.cy, g.H, g.Y), ye = cell_start(b.cy + 1, g.H, g.Y);
  b.y0 = ys + band * g.rows;
  b.y1 = min(ye, b.y0 + g.rows);
  return b.x0 < b.x1 && b.y0 < b.y1;
}

// win[(j Ls + s) 12 + c] = grid entry c at spatial corner j = (cx + (j & 1), cy + (j >> 1)) and level
// min(s, L - 1), s < Ls = max(L, 2); corners past a size-1 axis repeat the last entry
__device__ __forceinline__ void load_window(const float *__restrict__ grid, const BgGeom &g, int cx, int cy,
                                            float *win) {
  const int Ls = max(g.L, 2);
  const size_t plane = (size_t)g.L * g.Y * g.X;
  for (int q = threadIdx.x; q < 4 * Ls * 12; q += BG_THREADS) {
    const int c = q % 12, t = q / 12, s = t % Ls, j = t / Ls;
    const int x = min(cx + (j & 1), g.X - 1), y = min(cy + (j >> 1), g.Y - 1), z = min(s, g.L - 1);
    win[q] = __ldg(grid + c * plane + ((size_t)z * g.Y + y) * g.X + x);
  }
}

__device__ __forceinline__ float lerp_rn(float a, float b, float t) { return __fmaf_rn(t, __fsub_rn(b, a), a); }
__device__ __forceinline__ float4 lerp4(float4 a, float4 b, float t) {
  return make_float4(lerp_rn(a.x, b.x, t), lerp_rn(a.y, b.y, t), lerp_rn(a.z, b.z, t), lerp_rn(a.w, b.w, t));
}
// the 12 channels (3 rows of 4) at level slot s, bilinear in (tx, ty); a constant grid gives the
// constant exactly
__device__ __forceinline__ void bilerp(const float4 *win4, int Ls, int s, float tx, float ty, float4 a[3]) {
#pragma unroll
  for (int r = 0; r < 3; r++) {
    const float4 f00 = win4[(0 * Ls + s) * 3 + r], f10 = win4[(1 * Ls + s) * 3 + r];
    const float4 f01 = win4[(2 * Ls + s) * 3 + r], f11 = win4[(3 * Ls + s) * 3 + r];
    a[r] = lerp4(lerp4(f00, f10, tx), lerp4(f01, f11, tx), ty);
  }
}
__device__ __forceinline__ float affine_row(float4 a, float r, float g, float b) {
  return __fmaf_rn(a.x, r, __fmaf_rn(a.y, g, __fmaf_rn(a.z, b, a.w)));
}

// what a pixel needs besides the grid: its luminance, level slot z0 and the three fractions
struct PixelAt {
  float g, tx, ty, tz;
  int z0;
};
__device__ __forceinline__ PixelAt pixel_at(const BgGeom &gm, const Band &b, int px, int py, float r, float gg,
                                            float bb) {
  PixelAt p;
  p.g = __fmaf_rn(0.114f, bb, __fmaf_rn(0.587f, gg, __fmul_rn(0.299f, r)));
  const float gz = __fmul_rn(fminf(fmaxf(p.g, 0.f), 1.f), (float)(gm.L - 1));  // NaN -> 0
  p.z0 = cell_of(gz, gm.L);
  p.tz = __fsub_rn(gz, (float)p.z0);
  p.tx = __fsub_rn(grid_coord(px, gm.W, gm.X), (float)b.cx);
  p.ty = __fsub_rn(grid_coord(py, gm.H, gm.Y), (float)b.cy);
  return p;
}

__global__ void __launch_bounds__(BG_THREADS) k_bilagrid_slice(BgGeom gm, BgIds ids, const float *__restrict__ grids,
                                                               const float *__restrict__ rgb,
                                                               float *__restrict__ out) {
  extern __shared__ float4 win4[];
  Band b;
  if (!band_of(gm, blockIdx.x, b)) return;
  const int item = blockIdx.y, Ls = max(gm.L, 2);
  load_window(grids + (size_t)ids.id[item] * 12 * gm.L * gm.Y * gm.X, gm, b.cx, b.cy,
              reinterpret_cast<float *>(win4));
  __syncthreads();
  const size_t HW = (size_t)gm.H * gm.W;
  const float *src = rgb + (size_t)item * 3 * HW;
  float *dst = out + (size_t)item * 3 * HW;
  const int bw = b.x1 - b.x0, n = bw * (b.y1 - b.y0);
  for (int i = threadIdx.x; i < n; i += BG_THREADS) {
    const int ry = i / bw, px = b.x0 + i - ry * bw, py = b.y0 + ry;
    const size_t o = (size_t)py * gm.W + px;
    const float r = __ldg(src + o), gg = __ldg(src + HW + o), bb = __ldg(src + 2 * HW + o);
    const PixelAt p = pixel_at(gm, b, px, py, r, gg, bb);
    float4 a0[3], a1[3];
    bilerp(win4, Ls, p.z0, p.tx, p.ty, a0);
    bilerp(win4, Ls, p.z0 + 1, p.tx, p.ty, a1);
#pragma unroll
    for (int k = 0; k < 3; k++) dst[k * HW + o] = affine_row(lerp4(a0[k], a1[k], p.tz), r, gg, bb);
  }
}

// the warp's running sums for one z0 go to its shared accumulators: lane (m, col) owns
// wacc[((z0 + m) 3 + r) 16 + col], r = 0..2
__device__ __forceinline__ void flush_run(float *wacc, int z0, int m, int col, float run[3]) {
#pragma unroll
  for (int r = 0; r < 3; r++) {
    float *a = wacc + ((z0 + m) * 3 + r) * 16 + col;
    *a = __fadd_rn(*a, run[r]);
    run[r] = 0.f;
  }
}

__global__ void __launch_bounds__(BG_THREADS) k_bilagrid_slice_bwd(BgGeom gm, BgIds ids,
                                                                   const float *__restrict__ grids,
                                                                   const float *__restrict__ rgb,
                                                                   const float *__restrict__ dout,
                                                                   float *__restrict__ drgb,
                                                                   float *__restrict__ dgrids) {
  extern __shared__ float4 smem4[];
  Band b;
  if (!band_of(gm, blockIdx.x, b)) return;
  const int item = blockIdx.y, Ls = max(gm.L, 2);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float4 *win4 = smem4;                                          // [4 Ls][3] float4
  float *acc = reinterpret_cast<float *>(smem4 + 4 * Ls * 3);    // [warp][Ls][3][16]
  float4 *stage = reinterpret_cast<float4 *>(acc + BG_WARPS * Ls * 48);  // [warp][32 pixels][3] float4
  const size_t plane = (size_t)gm.L * gm.Y * gm.X, gsize = 12 * plane;
  load_window(grids + (size_t)ids.id[item] * gsize, gm, b.cx, b.cy, reinterpret_cast<float *>(win4));
  for (int q = threadIdx.x; q < BG_WARPS * Ls * 48; q += BG_THREADS) acc[q] = 0.f;
  __syncthreads();

  const size_t HW = (size_t)gm.H * gm.W, off = (size_t)item * 3 * HW;
  const float *src = rgb + off, *dsrc = dout + off;
  float *ddst = drgb + off;
  float *wacc = acc + warp * Ls * 48;
  float4 *wst = stage + warp * 96;
  const float gscale = (float)(gm.L - 1);
  // this lane's accumulator column: column k of [rgb, 1], spatial corner (jx, jy), z corner m
  const int col = lane & 15, k = lane & 3, jx = (lane >> 2) & 1, jy = (lane >> 3) & 1, m = lane >> 4;
  float run[3] = {0.f, 0.f, 0.f};
  int run_z = -1;
  const int bw = b.x1 - b.x0, n = bw * (b.y1 - b.y0);
  for (int base = warp * 32; base < n; base += BG_THREADS) {
    const int i = base + lane;
    if (i < n) {
      const int ry = i / bw, px = b.x0 + i - ry * bw, py = b.y0 + ry;
      const size_t o = (size_t)py * gm.W + px;
      const float r = __ldg(src + o), gg = __ldg(src + HW + o), bb = __ldg(src + 2 * HW + o);
      const float d0 = __ldg(dsrc + o), d1 = __ldg(dsrc + HW + o), d2 = __ldg(dsrc + 2 * HW + o);
      const PixelAt p = pixel_at(gm, b, px, py, r, gg, bb);
      float4 a0[3], a1[3];
      bilerp(win4, Ls, p.z0, p.tx, p.ty, a0);
      bilerp(win4, Ls, p.z0 + 1, p.tx, p.ty, a1);
      float4 a[3];
#pragma unroll
      for (int q = 0; q < 3; q++) a[q] = lerp4(a0[q], a1[q], p.tz);
      // dL/drgb = A[:, :3]^T dL/dout, plus the guidance term through g where it is not clamped
      float dr = __fmaf_rn(a[2].x, d2, __fmaf_rn(a[1].x, d1, __fmul_rn(a[0].x, d0)));
      float dg = __fmaf_rn(a[2].y, d2, __fmaf_rn(a[1].y, d1, __fmul_rn(a[0].y, d0)));
      float db = __fmaf_rn(a[2].z, d2, __fmaf_rn(a[1].z, d1, __fmul_rn(a[0].z, d0)));
      if (gm.L > 1 && p.g > 0.f && p.g < 1.f) {
        float s = 0.f;
        const float dq[3] = {d0, d1, d2};
#pragma unroll
        for (int q = 0; q < 3; q++) {
          const float4 da = make_float4(__fsub_rn(a1[q].x, a0[q].x), __fsub_rn(a1[q].y, a0[q].y),
                                        __fsub_rn(a1[q].z, a0[q].z), __fsub_rn(a1[q].w, a0[q].w));
          s = __fmaf_rn(dq[q], affine_row(da, r, gg, bb), s);
        }
        s = __fmul_rn(s, gscale);
        dr = __fmaf_rn(s, 0.299f, dr);
        dg = __fmaf_rn(s, 0.587f, dg);
        db = __fmaf_rn(s, 0.114f, db);
      }
      ddst[o] = dr;
      ddst[HW + o] = dg;
      ddst[2 * HW + o] = db;
      wst[lane * 3 + 0] = make_float4(d0, d1, d2, p.tz);
      wst[lane * 3 + 1] = make_float4(r, gg, bb, 1.f);
      wst[lane * 3 + 2] = make_float4(p.tx, p.ty, __int_as_float(p.z0), 0.f);
    }
    __syncwarp();
    const int cnt = min(32, n - base);
    for (int q = 0; q < cnt; q++) {
      const float4 dz = wst[q * 3], xy = wst[q * 3 + 2];
      const float v = reinterpret_cast<const float *>(wst + q * 3 + 1)[k];
      const int z0 = __float_as_int(xy.z);
      if (z0 != run_z) {  // warp-uniform: every lane reads the same pixel
        if (run_z >= 0) flush_run(wacc, run_z, m, col, run);
        run_z = z0;
      }
      const float wx = jx ? xy.x : __fsub_rn(1.f, xy.x), wy = jy ? xy.y : __fsub_rn(1.f, xy.y);
      const float wz = m ? dz.w : __fsub_rn(1.f, dz.w);
      const float w = __fmul_rn(__fmul_rn(__fmul_rn(wx, wy), wz), v);
      run[0] = __fmaf_rn(w, dz.x, run[0]);
      run[1] = __fmaf_rn(w, dz.y, run[1]);
      run[2] = __fmaf_rn(w, dz.z, run[2]);
    }
    __syncwarp();
  }
  if (run_z >= 0) flush_run(wacc, run_z, m, col, run);
  __syncthreads();
  float *dgrid = dgrids + (size_t)ids.id[item] * gsize;
  for (int q = threadIdx.x; q < Ls * 48; q += BG_THREADS) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < BG_WARPS; w++) s = __fadd_rn(s, acc[w * Ls * 48 + q]);
    if (s != 0.f) {
      const int c16 = q & 15, r = (q >> 4) % 3, slot = q / 48;
      const int x = min(b.cx + ((c16 >> 2) & 1), gm.X - 1), y = min(b.cy + (c16 >> 3), gm.Y - 1);
      const int z = min(slot, gm.L - 1);
      atomicAdd(dgrid + (4 * r + (c16 & 3)) * plane + ((size_t)z * gm.Y + y) * gm.X + x, s);
    }
  }
}

// TV = sum over the axes a of sum (grid shifted by one along a - grid)^2 / n_a, n_a the number of
// such differences; grad = dTV/dgrid.  Each element adds the differences to its successors.
__global__ void __launch_bounds__(TV_THREADS) k_bilagrid_tv(int64_t n, int L, int Y, int X, double ix, double iy,
                                                            double iz, const float *__restrict__ g,
                                                            float *__restrict__ grad, double *__restrict__ part) {
  __shared__ double red[TV_THREADS / 32];
  const float fx = (float)(2.0 * ix), fy = (float)(2.0 * iy), fz = (float)(2.0 * iz);
  const int64_t sy = X, sz = (int64_t)X * Y;
  double sx2 = 0.0, sy2 = 0.0, sz2 = 0.0;
  for (int64_t e = (int64_t)blockIdx.x * TV_THREADS + threadIdx.x; e < n; e += (int64_t)gridDim.x * TV_THREADS) {
    const int x = (int)(e % X);
    const int64_t t = e / X;
    const int y = (int)(t % Y), z = (int)((t / Y) % L);
    const float v = g[e];
    float gr = 0.f;
    if (x + 1 < X) {
      const float d = __fsub_rn(g[e + 1], v);
      sx2 += (double)d * d;
      gr = __fmaf_rn(-fx, d, gr);
    }
    if (x > 0) gr = __fmaf_rn(fx, __fsub_rn(v, g[e - 1]), gr);
    if (y + 1 < Y) {
      const float d = __fsub_rn(g[e + sy], v);
      sy2 += (double)d * d;
      gr = __fmaf_rn(-fy, d, gr);
    }
    if (y > 0) gr = __fmaf_rn(fy, __fsub_rn(v, g[e - sy]), gr);
    if (z + 1 < L) {
      const float d = __fsub_rn(g[e + sz], v);
      sz2 += (double)d * d;
      gr = __fmaf_rn(-fz, d, gr);
    }
    if (z > 0) gr = __fmaf_rn(fz, __fsub_rn(v, g[e - sz]), gr);
    if (grad) grad[e] = gr;
  }
  double s = sx2 * ix + sy2 * iy + sz2 * iz;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < TV_THREADS / 32; w++) t += red[w];
    part[blockIdx.x] = t;
  }
}

// one CTA: the partial sums in a fixed order
__global__ void __launch_bounds__(TV_THREADS) k_bilagrid_tv_sum(int parts, const double *__restrict__ part,
                                                                float *__restrict__ tv) {
  __shared__ double red[TV_THREADS];
  double s = 0.0;
  for (int i = threadIdx.x; i < parts; i += TV_THREADS) s += part[i];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int h = TV_THREADS / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) tv[0] = (float)red[0];
}

int tv_blocks(const BilagridShape &s) {
  const int64_t n = (int64_t)s.M * 12 * s.L * s.Y * s.X;
  return (int)std::min<int64_t>((n + TV_THREADS - 1) / TV_THREADS, TV_MAX_BLOCKS);
}

// the CTA grid: cells x bands per cell, bands of whole rows of about BG_BAND_PIXELS pixels
BgGeom geom(const BilagridShape &s, int H, int W) {
  BgGeom g;
  g.L = s.L, g.Y = s.Y, g.X = s.X, g.H = H, g.W = W;
  g.ncx = std::max(s.X - 1, 1), g.ncy = std::max(s.Y - 1, 1);
  // a cell spans at most ceil(n / cells) pixels along an axis; +2 covers fp32 rounding at its ends
  const int cw = std::min(W, W / g.ncx + 3), ch = std::min(H, H / g.ncy + 3);
  g.rows = std::max(1, BG_BAND_PIXELS / cw);
  g.nbands = (ch + g.rows - 1) / g.rows;
  return g;
}

BgIds ids_of(int B, const int32_t *ids) {
  BgIds r = {};
  for (int i = 0; i < B; i++) r.id[i] = ids[i];
  return r;
}

size_t slice_bwd_smem(int L) {
  const int Ls = std::max(L, 2);
  return (size_t)4 * Ls * 12 * sizeof(float) + (size_t)BG_WARPS * Ls * 48 * sizeof(float) +
         (size_t)BG_WARPS * 32 * 12 * sizeof(float);
}

}  // namespace

size_t bilagrid_tv_workspace_bytes(const BilagridShape &s) { return (size_t)tv_blocks(s) * sizeof(double); }

int launch_bilagrid_slice(const BilagridShape &s, const float *grids, int B, const int32_t *ids, int H, int W,
                          const float *rgb, float *out, cudaStream_t st) {
  const BgGeom g = geom(s, H, W);
  const dim3 grid((unsigned)(g.ncx * g.ncy * g.nbands), (unsigned)B);
  const size_t smem = (size_t)4 * std::max(s.L, 2) * 12 * sizeof(float);
  ProfScope ps(K_BILAGRID_SLICE, st);
  k_bilagrid_slice<<<grid, BG_THREADS, smem, st>>>(g, ids_of(B, ids), grids, rgb, out);
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_bilagrid_slice_bwd(const BilagridShape &s, const float *grids, int B, const int32_t *ids, int H, int W,
                              const float *rgb, const float *dout, float *drgb, float *dgrids, cudaStream_t st) {
  const BgGeom g = geom(s, H, W);
  const dim3 grid((unsigned)(g.ncx * g.ncy * g.nbands), (unsigned)B);
  const size_t smem = slice_bwd_smem(s.L);
  if (smem > 48 * 1024)
    GSB_CUDA_TRY(cudaFuncSetAttribute(k_bilagrid_slice_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  ProfScope ps(K_BILAGRID_SLICE_BWD, st);
  k_bilagrid_slice_bwd<<<grid, BG_THREADS, smem, st>>>(g, ids_of(B, ids), grids, rgb, dout, drgb, dgrids);
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_bilagrid_tv(const BilagridShape &s, const float *grids, float *tv, float *dgrids, void *ws,
                       cudaStream_t st) {
  const int64_t n = (int64_t)s.M * 12 * s.L * s.Y * s.X;
  // n_a: the differences along each axis; an axis of size 1 has none and adds nothing
  const int64_t per = n / ((int64_t)s.L * s.Y * s.X);
  const int64_t nx = per * s.L * s.Y * (s.X - 1), ny = per * s.L * (s.Y - 1) * s.X, nz = per * (s.L - 1) * s.Y * s.X;
  const double ix = nx ? 1.0 / (double)nx : 0.0, iy = ny ? 1.0 / (double)ny : 0.0, iz = nz ? 1.0 / (double)nz : 0.0;
  const int blocks = tv_blocks(s);
  double *part = static_cast<double *>(ws);
  ProfScope ps(K_BILAGRID_TV, st);
  k_bilagrid_tv<<<blocks, TV_THREADS, 0, st>>>(n, s.L, s.Y, s.X, ix, iy, iz, grids, dgrids, part);
  GSB_CUDA_TRY(cudaGetLastError());
  k_bilagrid_tv_sum<<<1, TV_THREADS, 0, st>>>(blocks, part, tv);
  GSB_CUDA_TRY(cudaGetLastError());
  return 0;
}

}  // namespace gsb
