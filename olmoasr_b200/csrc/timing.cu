// Word-level timestamps: the cross-attention alignment matrix and its dynamic time warping (whisper/timing.py
// find_alignment and dtw, restated in the header next to oasr_align_cost / oasr_dtw).
//
// Each kernel reads its window from a descriptor (oasr_align_window / oasr_dtw_window): one CTA grid dimension walks the
// windows of a batched call, and a single-window call is the one-window case with the descriptor passed by value.
//
// Everything is fp32 after the 16-bit q / k are read.  Every sum has one fixed order (a thread's own loop, then
// xor-butterfly shuffles, then a fixed block merge), there are no float atomics, so results are bit-identical from run
// to run.
#include "common.cuh"

#include <math.h>

namespace oasr {
namespace {

constexpr int HD = 64;              // head dim of every OLMoASR variant
constexpr int ALIGN_MAX_TOK = 448;  // n_text_ctx
constexpr int MAX_MEDFILT = 7;

// ---- row statistics: softmax max / sum over frames -------------------------------------------------------------
constexpr int RS_ROWS = 32;   // query rows per CTA
constexpr int RS_FR = 64;     // frames per smem tile
constexpr int KPAD = HD + 1;  // padded k / q rows (no bank conflicts on column walks)

template <typename T>
__device__ __forceinline__ float ld16(const T* p) { return Act16<T>::to_f(*p); }

// The windows of a call: a device table, or (table == nullptr) the one window of a single-window entry point.
template <typename W>
struct Windows {
  const W* table;
  W one;
  __device__ __forceinline__ W get(int i) const { return table ? table[i] : one; }
};

// QK value of one (row, frame): the dot product in d order, then the exact 1/8 = hd^-1/2 scale (qk_scale = 1).  Both
// passes use this loop, so the row maxima of pass 1 are values pass 2 recomputes bit for bit.
__device__ __forceinline__ float qk_dot(const float* q, const float* k) {
  float acc = 0.f;
#pragma unroll 16
  for (int d = 0; d < HD; ++d) acc = __fmaf_rn(q[d], k[d], acc);
  return acc * 0.125f;
}

// grid (ceil(max n_tok / RS_ROWS), n_heads, n_windows), 256 threads: thread (r, c) owns rows r and r + 16 of the CTA's
// block and the frames c, c + 16, c + 32, c + 48 of every tile; its online (max, sum-exp) pairs are merged over c by a
// butterfly.
template <typename T>
__global__ void __launch_bounds__(256) align_rowstats_kernel(Windows<oasr_align_window> windows, float* row_stats_base) {
  __shared__ float qs[RS_ROWS * KPAD];
  __shared__ float ks[RS_FR * KPAD];
  const oasr_align_window win = windows.get(blockIdx.z);
  const int n_tok = win.n_tok, n_frames = win.n_frames;
  const int row0 = blockIdx.x * RS_ROWS;
  if (row0 >= n_tok) return;   // a shorter window of a batched call
  float* row_stats = row_stats_base + win.row_stats;
  const oasr_align_head hd = win.heads[blockIdx.y];
  const T* q = (const T*)hd.q;
  const T* k = (const T*)hd.k;
  const int tid = threadIdx.x, r = tid >> 4, c = tid & 15;
  for (int i = tid; i < RS_ROWS * HD; i += 256) {
    const int rr = i / HD, d = i % HD;
    qs[rr * KPAD + d] = (row0 + rr < n_tok) ? ld16(q + (int64_t)(row0 + rr) * hd.ldq + d) : 0.f;
  }
  float m[2] = {-INFINITY, -INFINITY}, s[2] = {0.f, 0.f};
  for (int f0 = 0; f0 < n_frames; f0 += RS_FR) {
    __syncthreads();
    for (int i = tid; i < RS_FR * HD; i += 256) {
      const int ff = i / HD, d = i % HD;
      ks[ff * KPAD + d] = (f0 + ff < n_frames) ? ld16(k + (int64_t)(f0 + ff) * hd.ldk + d) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int a = 0; a < 2; ++a) {
      const float* qa = qs + (r + 16 * a) * KPAD;
#pragma unroll
      for (int b = 0; b < RS_FR / 16; ++b) {
        const int ff = c + 16 * b;
        if (f0 + ff >= n_frames) continue;
        const float x = qk_dot(qa, ks + ff * KPAD);
        if (x > m[a]) {
          s[a] = s[a] * expf(m[a] - x) + 1.f;
          m[a] = x;
        } else {
          s[a] += expf(x - m[a]);
        }
      }
    }
  }
#pragma unroll
  for (int a = 0; a < 2; ++a) {
#pragma unroll
    for (int o = 1; o < 16; o <<= 1) {   // within the 16 lanes of one row
      const float mo = __shfl_xor_sync(0xffffffffu, m[a], o), so = __shfl_xor_sync(0xffffffffu, s[a], o);
      const float mn = fmaxf(m[a], mo);
      const float sa = (m[a] == -INFINITY) ? 0.f : s[a] * expf(m[a] - mn);
      const float sb = (mo == -INFINITY) ? 0.f : so * expf(mo - mn);
      // the same operand order in both lanes of a pair, so the pair ends with one value
      s[a] = (c & o) ? sb + sa : sa + sb;
      m[a] = mn;
    }
    const int row = row0 + r + 16 * a;
    if (c == 0 && row < n_tok) {
      float* out = row_stats + ((int64_t)blockIdx.y * n_tok + row) * 2;
      out[0] = m[a];
      out[1] = s[a];
    }
  }
}

// ---- the cost tile: probabilities, column normalisation, median, head mean ----------------------------------------
constexpr int CT_F = 16;                        // output frames per CTA
constexpr int CT_HALO = MAX_MEDFILT / 2;        // 3
constexpr int CT_C = CT_F + 2 * CT_HALO;        // 22 columns of probabilities per head
constexpr int CT_PLD = CT_C + 1;                // padded row of the probability tile
constexpr int CT_QROWS = 32;                    // query rows staged per step
constexpr int CT_THREADS = 256;

__host__ __device__ constexpr size_t cost_smem_floats(int n_tok) {
  return (size_t)n_tok * CT_PLD              // probabilities -> normalised weights
         + (size_t)(n_tok - 2) * CT_F        // head sum
         + (size_t)CT_C * KPAD               // k tile
         + (size_t)CT_QROWS * KPAD           // q rows
         + 2 * CT_C;                         // column mean / 1/std
}

__device__ __forceinline__ int reflect(int g, int n) {   // F.pad(mode="reflect") index, n > half width
  if (g < 0) g = -g;
  if (g >= n) g = 2 * (n - 1) - g;
  return g;
}

// grid (ceil(max n_frames / CT_F), n_windows) CTAs; heads are processed one after the other in table order, so the head
// sum adds them in ascending (layer, head) order for a table built that way.
template <typename T>
__global__ void __launch_bounds__(CT_THREADS, 1) align_cost_kernel(Windows<oasr_align_window> windows, int n_heads,
                                                                int medfilt_width, const float* row_stats_base) {
  extern __shared__ float sm[];
  const oasr_align_window win = windows.get(blockIdx.y);
  const int n_tok = win.n_tok, n_frames = win.n_frames;
  if ((int)blockIdx.x * CT_F >= n_frames) return;   // a shorter window of a batched call
  const oasr_align_head* heads = win.heads;
  const float* row_stats = row_stats_base + win.row_stats;
  float* cost = win.cost;
  const int64_t ld_cost = win.ld_cost;
  float* P = sm;
  float* acc = P + (size_t)n_tok * CT_PLD;
  float* ks = acc + (size_t)(n_tok - 2) * CT_F;
  float* qs = ks + CT_C * KPAD;
  float* cmean = qs + CT_QROWS * KPAD;
  float* crstd = cmean + CT_C;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int f0 = blockIdx.x * CT_F;
  const int g0 = f0 - CT_HALO;                             // frame of column 0
  const int n_out = n_tok - 2;
  const int half = medfilt_width / 2;
  const bool filter = half > 0 && n_frames > half;         // median_filter returns its input when n <= pad width
  // columns whose frames this tile reads: [clo, chi)
  const int clo = max(0, -g0), chi = min(CT_C, n_frames - g0);
  for (int i = tid; i < n_out * CT_F; i += CT_THREADS) acc[i] = 0.f;

  for (int h = 0; h < n_heads; ++h) {
    const oasr_align_head hd = heads[h];
    const T* q = (const T*)hd.q;
    const T* k = (const T*)hd.k;
    const float* stats = row_stats + (int64_t)h * n_tok * 2;
    __syncthreads();   // previous head's P fully consumed
    for (int i = tid; i < CT_C * HD; i += CT_THREADS) {
      const int cc = i / HD, d = i % HD;
      ks[cc * KPAD + d] = (cc >= clo && cc < chi) ? ld16(k + (int64_t)(g0 + cc) * hd.ldk + d) : 0.f;
    }
    for (int r0 = 0; r0 < n_tok; r0 += CT_QROWS) {
      __syncthreads();
      for (int i = tid; i < CT_QROWS * HD; i += CT_THREADS) {
        const int rr = i / HD, d = i % HD;
        qs[rr * KPAD + d] = (r0 + rr < n_tok) ? ld16(q + (int64_t)(r0 + rr) * hd.ldq + d) : 0.f;
      }
      __syncthreads();
      for (int i = tid; i < CT_QROWS * CT_C; i += CT_THREADS) {
        const int rr = i / CT_C, cc = i % CT_C, row = r0 + rr;
        if (row >= n_tok || cc < clo || cc >= chi) continue;
        const float x = qk_dot(qs + rr * KPAD, ks + cc * KPAD);
        P[row * CT_PLD + cc] = expf(x - stats[2 * row]) / stats[2 * row + 1];
      }
    }
    __syncthreads();
    // column mean and std over all n_tok rows (two passes, unbiased=False): one warp per column
    for (int cc = clo + warp; cc < chi; cc += CT_THREADS / 32) {
      float sum = 0.f;
      for (int r = lane; r < n_tok; r += 32) sum += P[r * CT_PLD + cc];
      sum = warp_sum(sum);
      const float mean = sum / (float)n_tok;
      float sq = 0.f;
      for (int r = lane; r < n_tok; r += 32) {
        const float dv = P[r * CT_PLD + cc] - mean;
        sq = __fmaf_rn(dv, dv, sq);
      }
      sq = warp_sum(sq);
      if (lane == 0) {
        cmean[cc] = mean;
        crstd[cc] = sqrtf(sq / (float)n_tok);
      }
    }
    __syncthreads();
    for (int i = tid; i < n_tok * CT_C; i += CT_THREADS) {
      const int r = i / CT_C, cc = i % CT_C;
      if (cc >= clo && cc < chi) P[r * CT_PLD + cc] = (P[r * CT_PLD + cc] - cmean[cc]) / crstd[cc];
    }
    __syncthreads();
    // median of the reflect-padded window (a selection: exact), accumulated per (row, frame) in head order
    for (int i = tid; i < n_out * CT_F; i += CT_THREADS) {
      const int r = 1 + i / CT_F, ff = i % CT_F, f = f0 + ff;
      if (f >= n_frames) continue;
      const float* row = P + r * CT_PLD;
      float med;
      if (!filter) {
        med = row[f - g0];
      } else {
        // the window padded to 7 with -inf / +inf on either side has the same median; a fixed compare-exchange
        // network keeps it in registers
        float w[MAX_MEDFILT];
#pragma unroll
        for (int o = 0; o < MAX_MEDFILT; ++o) {
          const int off = o - CT_HALO;
          w[o] = (off < -half) ? -INFINITY : (off > half) ? INFINITY : row[reflect(f + off, n_frames) - g0];
        }
#pragma unroll
        for (int a = 0; a < MAX_MEDFILT - 1; ++a)
#pragma unroll
          for (int b = 0; b < MAX_MEDFILT - 1 - a; ++b) {
            const float lo = fminf(w[b], w[b + 1]), hi = fmaxf(w[b], w[b + 1]);
            w[b] = lo;
            w[b + 1] = hi;
          }
        med = w[CT_HALO];
      }
      acc[i] += med;
    }
  }
  __syncthreads();
  for (int i = tid; i < n_out * CT_F; i += CT_THREADS) {
    const int r = i / CT_F, f = f0 + i % CT_F;
    if (f < n_frames) cost[(int64_t)r * ld_cost + f] = -(acc[i] / (float)n_heads);
  }
}

// ---- dynamic time warping ------------------------------------------------------------------------------------------
// One CTA per window walks the anti-diagonals d = i + j of the (rows + 1) x (cols + 1) cost table; three diagonals live
// in shared memory (indexed by i), the trace goes to global memory, then thread 0 backtracks.
constexpr int DTW_THREADS = 1024;

__global__ void __launch_bounds__(DTW_THREADS) dtw_kernel(Windows<oasr_dtw_window> windows) {
  extern __shared__ float diag[];   // 3 x (rows + 1)
  const oasr_dtw_window win = windows.get(blockIdx.x);
  const float* x = win.x;
  const int64_t ldx = win.ldx;
  const int rows = win.rows, cols = win.cols;
  uint8_t* trace = win.trace;
  int32_t* text_idx = win.text_idx;
  int32_t* time_idx = win.time_idx;
  const int R = rows + 1;
  const int64_t tld = cols + 1;
  for (int i = threadIdx.x; i < 3 * R; i += DTW_THREADS) diag[i] = INFINITY;
  __syncthreads();
  if (threadIdx.x == 0) diag[0] = 0.f;   // d = 0: cost[0][0]
  __syncthreads();
  for (int d = 2; d <= rows + cols; ++d) {
    float* cur = diag + (d % 3) * R;
    const float* p1 = diag + ((d + 2) % 3) * R;   // d - 1
    const float* p2 = diag + ((d + 1) % 3) * R;   // d - 2
    for (int i = threadIdx.x; i < R; i += DTW_THREADS) {
      const int j = d - i;
      float v = INFINITY;
      if (i >= 1 && j >= 1 && j <= cols) {
        const float c0 = p2[i - 1], c1 = p1[i - 1], c2 = p1[i];
        float c;
        uint8_t t;
        if (c0 < c1 && c0 < c2) {
          c = c0; t = 0;
        } else if (c1 < c0 && c1 < c2) {
          c = c1; t = 1;
        } else {
          c = c2; t = 2;
        }
        v = __fadd_rn(x[(int64_t)(i - 1) * ldx + (j - 1)], c);
        trace[(int64_t)i * tld + j] = t;
      }
      cur[i] = v;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    int i = rows, j = cols, n = 0;
    while (i > 0 || j > 0) {
      text_idx[n] = i - 1;
      time_idx[n] = j - 1;
      ++n;
      const int t = (i == 0) ? 2 : (j == 0) ? 1 : trace[(int64_t)i * tld + j];   // trace[0, :] = 2, trace[:, 0] = 1
      if (t == 0) {
        --i; --j;
      } else if (t == 1) {
        --i;
      } else {
        --j;
      }
    }
    *win.path_len = n;
    diag[0] = __int_as_float(n);
  }
  __syncthreads();
  const int n = __float_as_int(diag[0]);
  for (int a = threadIdx.x; a < n / 2; a += DTW_THREADS) {   // backtrace order -> path order
    const int b = n - 1 - a;
    const int32_t ti = text_idx[a], tj = time_idx[a];
    text_idx[a] = text_idx[b];
    time_idx[a] = time_idx[b];
    text_idx[b] = ti;
    time_idx[b] = tj;
  }
}

template <typename T>
int launch_align(Windows<oasr_align_window> windows, int n_windows, int n_heads, int max_tok, int max_frames,
                 int medfilt_width, float* row_stats, cudaStream_t st) {
  const dim3 rs_grid((unsigned)ceil_div(max_tok, RS_ROWS), (unsigned)n_heads, (unsigned)n_windows);
  align_rowstats_kernel<T><<<rs_grid, 256, 0, st>>>(windows, row_stats);
  OASR_LAUNCH_CHECK();
  const size_t smem = cost_smem_floats(max_tok) * sizeof(float);
  OASR_CUDA_OK(cudaFuncSetAttribute(align_cost_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const dim3 ct_grid((unsigned)ceil_div(max_frames, CT_F), (unsigned)n_windows);
  align_cost_kernel<T><<<ct_grid, CT_THREADS, smem, st>>>(windows, n_heads, medfilt_width, row_stats);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

int launch_dtw(Windows<oasr_dtw_window> windows, int n_windows, int max_rows, cudaStream_t st) {
  const size_t smem = (size_t)3 * (max_rows + 1) * sizeof(float);
  if (smem > 48 * 1024) OASR_CUDA_OK(cudaFuncSetAttribute(dtw_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dtw_kernel<<<(unsigned)n_windows, DTW_THREADS, smem, st>>>(windows);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

constexpr int DTW_MAX_ROWS = (int)(200 * 1024 / 12) - 1;   // three diagonals of rows + 1 floats in 200 KB
constexpr int MAX_WINDOWS = 65535;                          // the grid dimension that walks the windows

}  // namespace
}  // namespace oasr

using namespace oasr;

#define OASR_REQUIRE_ALIGN_SHAPE(n_heads, head_dim, n_tok, n_frames, medfilt_width)                                      \
  OASR_REQUIRE(head_dim == HD, "align_cost: head_dim must be %d (got %d)", HD, head_dim);                               \
  OASR_REQUIRE(n_heads >= 1, "align_cost: need at least one head (got %d)", n_heads);                                  \
  OASR_REQUIRE(n_tok >= 3 && n_tok <= ALIGN_MAX_TOK, "align_cost: 3 <= n_tok <= %d (got %d)", ALIGN_MAX_TOK, n_tok);   \
  OASR_REQUIRE(n_frames >= 1 && n_frames <= 1500, "align_cost: 1 <= n_frames <= 1500 (got %d)", n_frames);             \
  OASR_REQUIRE(medfilt_width >= 1 && medfilt_width <= MAX_MEDFILT && (medfilt_width & 1),                              \
               "align_cost: medfilt_width must be odd and <= %d (got %d)", MAX_MEDFILT, medfilt_width)

extern "C" int oasr_align_cost(const oasr_align_head* heads, int32_t n_heads, int32_t head_dim, int32_t n_tok,
                               int32_t n_frames, int32_t medfilt_width, float* row_stats, float* cost, int64_t ld_cost,
                               int dtype, void* stream) {
  OASR_REQUIRE(heads && row_stats && cost, "align_cost: null tensor");
  OASR_REQUIRE_ALIGN_SHAPE(n_heads, head_dim, n_tok, n_frames, medfilt_width);
  OASR_REQUIRE(ld_cost >= n_frames, "align_cost: ld_cost < n_frames");
  Windows<oasr_align_window> one{nullptr, {heads, cost, ld_cost, 0, n_tok, n_frames}};
  return OASR_BY_DTYPE16(dtype, launch_align, one, 1, n_heads, n_tok, n_frames, medfilt_width, row_stats,
                         (cudaStream_t)stream);
}

extern "C" int oasr_align_cost_batched(const oasr_align_window* windows, int32_t n_windows, int32_t n_heads,
                                       int32_t head_dim, int32_t max_tok, int32_t max_frames, int32_t medfilt_width,
                                       float* row_stats, int dtype, void* stream) {
  OASR_REQUIRE(windows && row_stats, "align_cost_batched: null tensor");
  OASR_REQUIRE(n_windows >= 1 && n_windows <= MAX_WINDOWS, "align_cost_batched: 1 <= n_windows <= %d (got %d)",
               MAX_WINDOWS, n_windows);
  OASR_REQUIRE_ALIGN_SHAPE(n_heads, head_dim, max_tok, max_frames, medfilt_width);
  Windows<oasr_align_window> table{windows, {}};
  return OASR_BY_DTYPE16(dtype, launch_align, table, n_windows, n_heads, max_tok, max_frames, medfilt_width, row_stats,
                         (cudaStream_t)stream);
}

extern "C" int oasr_dtw(const float* x, int64_t ldx, int32_t rows, int32_t cols, uint8_t* trace, int32_t* text_idx,
                        int32_t* time_idx, int32_t* path_len, void* stream) {
  OASR_REQUIRE(x && trace && text_idx && time_idx && path_len, "dtw: null tensor");
  OASR_REQUIRE(rows >= 1 && cols >= 1, "dtw: empty matrix (%d x %d)", rows, cols);
  OASR_REQUIRE(ldx >= cols, "dtw: ldx < cols");
  OASR_REQUIRE(rows <= DTW_MAX_ROWS, "dtw: rows <= %d (got %d)", DTW_MAX_ROWS, rows);
  Windows<oasr_dtw_window> one{nullptr, {x, ldx, trace, text_idx, time_idx, path_len, rows, cols}};
  return launch_dtw(one, 1, rows, (cudaStream_t)stream);
}

extern "C" int oasr_dtw_batched(const oasr_dtw_window* windows, int32_t n_windows, int32_t max_rows, void* stream) {
  OASR_REQUIRE(windows, "dtw_batched: null tensor");
  OASR_REQUIRE(n_windows >= 1 && n_windows <= MAX_WINDOWS, "dtw_batched: 1 <= n_windows <= %d (got %d)", MAX_WINDOWS,
               n_windows);
  OASR_REQUIRE(max_rows >= 1 && max_rows <= DTW_MAX_ROWS, "dtw_batched: 1 <= max_rows <= %d (got %d)", DTW_MAX_ROWS,
               max_rows);
  return launch_dtw(Windows<oasr_dtw_window>{windows, {}}, n_windows, max_rows, (cudaStream_t)stream);
}
