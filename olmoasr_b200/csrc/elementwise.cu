// HBM-bound glue kernels: weight casts, embedding gather/scatter, conv-stem im2col / col2im,
// positional add, bias-gradient column sums.  All vectorised to 16-byte accesses where alignment allows.
#include "common.cuh"

namespace oasr {
namespace {

// ------------------------------------------------------------------ fp32 -> bf16 casts (weights)
// Linear.forward casts the fp32 master weight to the activation dtype on every call
// (olmoasr/model.py:97-101); we do it once per optimizer step into a persistent bf16 shadow.
__global__ void cast_f32_bf16_kernel(const float* __restrict__ src, bf16* __restrict__ dst, int64_t n) {
  const int64_t i = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) * 8;
  if (i + 8 <= n) {
    const float4 a = *reinterpret_cast<const float4*>(src + i);
    const float4 b = *reinterpret_cast<const float4*>(src + i + 4);
    uint4 u;
    u.x = pack_bf16x2(a.x, a.y); u.y = pack_bf16x2(a.z, a.w);
    u.z = pack_bf16x2(b.x, b.y); u.w = pack_bf16x2(b.z, b.w);
    *reinterpret_cast<uint4*>(dst + i) = u;
  } else {
    for (int64_t j = i; j < n; ++j) dst[j] = __float2bfloat16_rn(src[j]);
  }
}

// Conv1d weight (C_out, C_in, 3) f32 -> (C_out, 3, C_in) T so that im2col rows are plain slabs.
template <typename T>
__global__ void cast_conv_weight_kernel(const float* __restrict__ src, T* __restrict__ dst, int c_out, int c_in) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;  // index into dst
  const int64_t n = static_cast<int64_t>(c_out) * 3 * c_in;
  if (i >= n) return;
  const int c = i % c_in;
  const int k = (i / c_in) % 3;
  const int64_t o = i / (3 * c_in);
  dst[i] = Act16<T>::from_f(src[(o * c_in + c) * 3 + k]);
}
// and its inverse for the weight gradient: (C_out, 3, C_in) f32 -> (C_out, C_in, 3) f32
__global__ void unpermute_conv_wgrad_kernel(const float* __restrict__ src, float* __restrict__ dst, int c_out, int c_in,
                                            int accumulate) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;  // index into dst
  const int64_t n = static_cast<int64_t>(c_out) * 3 * c_in;
  if (i >= n) return;
  const int k = i % 3;
  const int c = (i / 3) % c_in;
  const int64_t o = i / (3 * c_in);
  const float v = src[(o * 3 + k) * c_in + c];
  dst[i] = accumulate ? dst[i] + v : v;
}

// ------------------------------------------------------------------ padding mask -> per-sample key count
// The reference hands the decoder a dense additive mask (B, S, S) f32 whose columns >= len(text_input) are -inf on every
// row (scripts/training/train_timestamps.py:314-315; added to the causal mask at olmoasr/model.py:740-743).  The
// attention kernels want the key count.  One block per sample: count the zeros of row 0, then verify that every row has
// exactly that structure; any other additive mask raises err[0] (reported by the host as a ValueError).
__global__ void __launch_bounds__(256)
mask_to_kvlen_kernel(const float* __restrict__ mask, int32_t* __restrict__ kv_len, int32_t* __restrict__ err, int S) {
  // grid (batch, slices): every block recounts the zeros of row 0 (S floats), then verifies its slice of rows with
  // 16-byte loads (the first version used one block per sample: 0.44 ms for the 25.7 MB mask of a 32-clip batch)
  const float* m = mask + static_cast<int64_t>(blockIdx.x) * S * S;
  __shared__ int s_len;
  __shared__ int s_bad;
  if (threadIdx.x == 0) { s_len = 0; s_bad = 0; }
  __syncthreads();
  int cnt = 0;
  for (int c = threadIdx.x; c < S; c += blockDim.x) cnt += (m[c] == 0.f);
  cnt = warp_sum(cnt);
  if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(&s_len, cnt);
  __syncthreads();
  const int len = s_len;
  const int rows_per = (S + gridDim.y - 1) / gridDim.y;
  const int r0 = blockIdx.y * rows_per, r1 = min(S, r0 + rows_per);
  int bad = 0;
  if ((S & 3) == 0 && (reinterpret_cast<uintptr_t>(m) & 15) == 0) {
    const int vec = S >> 2;
    for (int64_t i = static_cast<int64_t>(r0) * vec + threadIdx.x; i < static_cast<int64_t>(r1) * vec; i += blockDim.x) {
      const int c = static_cast<int>(i % vec) * 4;
      const float4 v = *reinterpret_cast<const float4*>(m + i * 4);
      const float x[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) bad |= (c + j < len) ? (x[j] != 0.f) : !(x[j] < -1e30f);
    }
  } else {
    for (int64_t i = static_cast<int64_t>(r0) * S + threadIdx.x; i < static_cast<int64_t>(r1) * S; i += blockDim.x) {
      const int c = static_cast<int>(i % S);
      const float v = m[i];
      bad |= (c < len) ? (v != 0.f) : !(v < -1e30f);
    }
  }
  if (bad) s_bad = 1;
  __syncthreads();
  if (threadIdx.x == 0) {
    if (blockIdx.y == 0) kv_len[blockIdx.x] = len;
    if (s_bad) atomicOr(err, 1);
  }
}

// ------------------------------------------------------------------ embedding
// x = (token_embedding(ids) + positional_embedding[offset : offset+S]).to(T)   (model.py:728-732)
// Packed batches (src_rows set): output row r is dense row src_rows[r] = b*S + t of ids.
template <typename T>
__global__ void embed_fwd_kernel(const int64_t* __restrict__ ids, const float* __restrict__ emb,
                                 const float* __restrict__ pos, T* __restrict__ out, int64_t rows, int S,
                                 int d, int pos_offset, int64_t n_rows_emb, const int32_t* __restrict__ src_rows = nullptr) {
  const int64_t row = blockIdx.x;
  if (row >= rows) return;
  const int64_t src = src_rows ? src_rows[row] : row;
  int64_t id = ids[src];
  if (id < 0 || id >= n_rows_emb) id = 0;  // guarded like a clamped gather; callers validate ids
  const int s = static_cast<int>(src % S) + pos_offset;
  const float4* e = reinterpret_cast<const float4*>(emb + id * d);
  const float4* p = reinterpret_cast<const float4*>(pos + static_cast<int64_t>(s) * d);
  uint2* o = reinterpret_cast<uint2*>(out + row * d);
  for (int v = threadIdx.x; v < (d >> 2); v += blockDim.x) {
    const float4 a = __ldg(e + v), b = __ldg(p + v);
    uint2 u;
    u.x = Act16<T>::pack2(a.x + b.x, a.y + b.y);
    u.y = Act16<T>::pack2(a.z + b.z, a.w + b.w);
    o[v] = u;
  }
}
// dE[id] += dx (skipping padding_idx), dP[s] += dx   (autograd of the above; nn.Embedding padding_idx, model.py:665-667)
// One block per row, sums taken in row order so that the result does not depend on scheduling: the block of a row
// with b == 0 writes dP[s] (sum over the batch), the block of the FIRST row carrying an id writes dE[id] (sum over
// every row with that id, gathered 128 rows at a time).
// Packed batches (src_rows / cu set): dx holds the N = rows packed rows, row r being dense row src_rows[r] of ids and
// sample b owning rows [cu[b], cu[b+1]); the grid covers max(rows, S) blocks.  The sums run over the same rows in the same
// order as the dense kernel's minus the padded rows.
constexpr int EMB_COLS = 10;   // columns per thread: 128 threads cover d <= 1280 (every OLMoASR width)
template <typename T>
__global__ void __launch_bounds__(128)
embed_bwd_kernel(const int64_t* __restrict__ ids, const T* __restrict__ dx,
                 float* __restrict__ demb, float* __restrict__ dpos, int64_t rows, int S, int d,
                 int64_t padding_idx, int64_t n_rows_emb, const int32_t* __restrict__ src_rows = nullptr,
                 const int32_t* __restrict__ cu = nullptr, int n_seq = 0) {
  __shared__ int64_t s_rows[128];
  __shared__ int s_cnt[4];
  const int64_t row = blockIdx.x;
  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  if (row < S && dpos) {   // a null dpos / demb (a frozen parameter) skips its sums
    if (cu) {
      for (int c = t; c < d; c += blockDim.x) {
        float v = 0.f;
        for (int b = 0; b < n_seq; ++b)
          if (cu[b] + row < cu[b + 1]) v += Act16<T>::to_f(dx[(cu[b] + row) * d + c]);
        dpos[row * d + c] += v;
      }
    } else {
      const int64_t batch = rows / S;
      for (int c = t; c < d; c += blockDim.x) {
        float v = 0.f;
        for (int64_t b = 0; b < batch; ++b) v += Act16<T>::to_f(dx[(b * S + row) * d + c]);
        dpos[row * d + c] += v;
      }
    }
  }
  if (row >= rows || !demb) return;
  auto id_of = [&](int64_t r) { return ids[src_rows ? src_rows[r] : r]; };
  const int64_t id = id_of(row);
  if (id == padding_idx || id < 0 || id >= n_rows_emb) return;
  for (int64_t base = 0; base < row; base += blockDim.x)   // an earlier row with this id owns the sum
    if (__syncthreads_or(base + t < row && id_of(base + t) == id)) return;
  float acc[EMB_COLS];
#pragma unroll
  for (int j = 0; j < EMB_COLS; ++j) acc[j] = 0.f;
  for (int64_t base = row; base < rows; base += blockDim.x) {
    const bool hit = base + t < rows && id_of(base + t) == id;
    const unsigned bal = __ballot_sync(0xffffffffu, hit);
    if (lane == 0) s_cnt[warp] = __popc(bal);
    __syncthreads();
    int before = 0, total = 0;
    for (int w = 0; w < 4; ++w) { if (w < warp) before += s_cnt[w]; total += s_cnt[w]; }
    if (hit) s_rows[before + __popc(bal & ((1u << lane) - 1u))] = base + t;
    __syncthreads();
    for (int k = 0; k < total; ++k) {   // matches in row order
      const T* g = dx + s_rows[k] * d;
#pragma unroll
      for (int j = 0; j < EMB_COLS; ++j)
        if (t + j * 128 < d) acc[j] += Act16<T>::to_f(g[t + j * 128]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int j = 0; j < EMB_COLS; ++j)
    if (t + j * 128 < d) demb[id * d + t + j * 128] += acc[j];
}

// ------------------------------------------------------------------ conv stem data movement
// conv1 im2col: mel (B, C, T) f32 -> A (B*T, Kpad) E (bf16 / fp16) with A[b,t][k*C + c] = mel[b][c][t+k-1]  (k3, p1)
// Columns >= 3*C (Kpad padding for TMA row-stride alignment) are zero.
template <typename E>
__global__ void im2col_conv1_kernel(const float* __restrict__ mel, E* __restrict__ A, int C, int T, int kpad) {
  extern __shared__ float tile[];  // [C][34]
  const int b = blockIdx.y;
  const int t0 = blockIdx.x * 32;
  for (int i = threadIdx.x; i < C * 34; i += blockDim.x) {
    const int c = i / 34, j = i % 34;
    const int t = t0 + j - 1;
    tile[i] = (t >= 0 && t < T) ? mel[(static_cast<int64_t>(b) * C + c) * T + t] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 32 * kpad; i += blockDim.x) {
    const int tt = i / kpad, col = i % kpad;
    if (t0 + tt >= T) continue;
    float v = 0.f;
    if (col < 3 * C) {
      const int k = col / C, c = col % C;
      v = tile[c * 34 + tt + k];
    }
    A[(static_cast<int64_t>(b) * T + t0 + tt) * kpad + col] = Act16<E>::from_f(v);
  }
}
// conv2 im2col (k3, s2, p1) on time-major activations: A[b,t] = [h[b,2t-1], h[b,2t], h[b,2t+1]]  (each d wide)
__global__ void im2col_conv2_kernel(const uint16_t* __restrict__ h, uint16_t* __restrict__ A, int T_in, int T_out, int d) {
  const int64_t row = blockIdx.x;  // b * T_out + t
  const int b = row / T_out, t = row % T_out;
  const int nvec = d >> 3;
  for (int i = threadIdx.x; i < 3 * nvec; i += blockDim.x) {
    const int k = i / nvec, v = i % nvec;
    const int r = 2 * t + k - 1;
    uint4 u = make_uint4(0, 0, 0, 0);
    if (r >= 0 && r < T_in) u = reinterpret_cast<const uint4*>(h + (static_cast<int64_t>(b) * T_in + r) * d)[v];
    reinterpret_cast<uint4*>(A + row * 3 * d)[i] = u;
  }
}
// col2im of the conv2 input gradient fused with the GELU backward of conv1:
//   dpre1[b,r] = T( T(sum_{(t,k): 2t+k-1=r} dA[b,t][k]) * gelu'(pre1[b,r]) )
template <typename T>
__global__ void col2im_conv2_gelu_bwd_kernel(const T* __restrict__ dA, const T* __restrict__ pre1,
                                             T* __restrict__ dpre1, int T_in, int T_out, int d) {
  const int64_t row = blockIdx.x;  // b * T_in + r
  const int b = row / T_in, r = row % T_in;
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    float g = 0.f;
    if ((r & 1) == 0) {
      const int t = r >> 1;  // k = 1
      if (t < T_out) g = Act16<T>::to_f(dA[((static_cast<int64_t>(b) * T_out + t) * 3 + 1) * d + c]);
    } else {
      const int ta = (r + 1) >> 1;  // k = 0
      const int tb = (r - 1) >> 1;  // k = 2
      if (ta < T_out) g += Act16<T>::to_f(dA[((static_cast<int64_t>(b) * T_out + ta) * 3 + 0) * d + c]);
      if (tb >= 0 && tb < T_out) g += Act16<T>::to_f(dA[((static_cast<int64_t>(b) * T_out + tb) * 3 + 2) * d + c]);
    }
    const float p = Act16<T>::to_f(pre1[row * d + c]);
    dpre1[row * d + c] = Act16<T>::from_f(Act16<T>::round(g) * gelu_erf_grad(p));
  }
}

// x = (x + positional_embedding).to(E), positional rows repeat every T rows  (model.py:602)
template <typename E>
__global__ void add_pos_kernel(const E* __restrict__ x, const float* __restrict__ pos, E* __restrict__ out,
                               int64_t rows, int T, int d) {
  const int64_t nvec = rows * (d >> 3);
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t row = i / (d >> 3);
    const int v = i % (d >> 3);
    const uint4 u = reinterpret_cast<const uint4*>(x)[i];
    const float4* p = reinterpret_cast<const float4*>(pos + (row % T) * d) + 2 * v;
    const float4 p0 = __ldg(p), p1 = __ldg(p + 1);
    using A = Act16<E>;
    float2 a = A::unpack2(u.x), b = A::unpack2(u.y), c = A::unpack2(u.z), e = A::unpack2(u.w);
    uint4 o;
    o.x = A::pack2(a.x + p0.x, a.y + p0.y); o.y = A::pack2(b.x + p0.z, b.y + p0.w);
    o.z = A::pack2(c.x + p1.x, c.y + p1.y); o.w = A::pack2(e.x + p1.z, e.y + p1.w);
    reinterpret_cast<uint4*>(out)[i] = o;
  }
}

// dy * gelu'(pre) elementwise (conv2 backward, where the upstream gradient is not a GEMM output)
template <typename T>
__global__ void gelu_bwd_kernel(const T* __restrict__ dy, const T* __restrict__ pre, T* __restrict__ out, int64_t n) {
  for (int64_t i = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) * 8; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x * 8) {
    const uint4 a = *reinterpret_cast<const uint4*>(dy + i), b = *reinterpret_cast<const uint4*>(pre + i);
    const uint32_t av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
    uint32_t ov[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 g = Act16<T>::unpack2(av[j]), p = Act16<T>::unpack2(bv[j]);
      ov[j] = Act16<T>::pack2(g.x * gelu_erf_grad(p.x), g.y * gelu_erf_grad(p.y));
    }
    *reinterpret_cast<uint4*>(out + i) = make_uint4(ov[0], ov[1], ov[2], ov[3]);
  }
}

// ------------------------------------------------------------------ bias gradient: db[n] += sum_m dy[m,n]
// Block = 32 x 8 threads; tile = 256 columns (8 per thread, one 16-byte load) x a slab of rows.  Each slab of rows
// writes its column sums to part[slab][n]; add_partials adds the slabs in order.
template <typename T>
__global__ void __launch_bounds__(256)
colsum_kernel(const T* __restrict__ dy, float* __restrict__ part, int64_t M, int N, int64_t ld, int rows_per_block) {
  __shared__ float red[8][256 + 8];
  const int col = blockIdx.x * 256 + threadIdx.x * 8;
  const int64_t r0 = static_cast<int64_t>(blockIdx.y) * rows_per_block;
  const int64_t r1 = min(M, r0 + rows_per_block);
  float s[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) s[j] = 0.f;
  if (col + 8 <= N && (ld & 7) == 0 && (reinterpret_cast<uintptr_t>(dy) & 15) == 0) {
    int64_t r = r0 + threadIdx.y;
    for (; r + 8 < r1; r += 16) {  // two independent 16-byte loads in flight per thread
      const uint4 a = *reinterpret_cast<const uint4*>(dy + r * ld + col);
      const uint4 b = *reinterpret_cast<const uint4*>(dy + (r + 8) * ld + col);
      const uint32_t av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 p = Act16<T>::unpack2(av[j]), q = Act16<T>::unpack2(bv[j]);
        s[2 * j] += p.x + q.x; s[2 * j + 1] += p.y + q.y;
      }
    }
    for (; r < r1; r += 8) {
      const uint4 a = *reinterpret_cast<const uint4*>(dy + r * ld + col);
      const uint32_t av[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) { const float2 p = Act16<T>::unpack2(av[j]); s[2 * j] += p.x; s[2 * j + 1] += p.y; }
    }
  } else {
    for (int64_t r = r0 + threadIdx.y; r < r1; r += 8)
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (col + j < N) s[j] += Act16<T>::to_f(dy[r * ld + col + j]);
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[threadIdx.y][threadIdx.x * 8 + j] = s[j];
  __syncthreads();
  const int t = threadIdx.y * 32 + threadIdx.x;  // 256 threads -> 256 columns
  float a = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) a += red[j][t];
  if (blockIdx.x * 256 + t < N) part[static_cast<int64_t>(blockIdx.y) * N + blockIdx.x * 256 + t] = a;
}

}  // namespace
}  // namespace oasr

using namespace oasr;

// The vectorised kernels below read and write whole 8- or 16-byte words: a view that starts inside one is refused.
static inline bool aligned(const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }

static inline int grid_1d(int64_t n_items, int threads, int cap_mult = 32) {
  int64_t b = ceil_div(n_items, threads);
  const int64_t cap = static_cast<int64_t>(num_sms()) * cap_mult;
  return (int)(b < cap ? (b < 1 ? 1 : b) : cap);
}

extern "C" int oasr_cast_f32_to_bf16(const float* src, void* dst, int64_t n, void* stream) {
  OASR_REQUIRE(n > 0, "cast: empty");
  OASR_REQUIRE(((uintptr_t)src & 15) == 0 && ((uintptr_t)dst & 15) == 0, "cast: 16-byte alignment required");
  const int64_t threads_needed = ceil_div(n, 8);
  cast_f32_bf16_kernel<<<(unsigned)ceil_div(threads_needed, 256), 256, 0, (cudaStream_t)stream>>>(src, (bf16*)dst, n);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

template <typename T>
static int cast_conv_weight(const float* src, void* dst, int64_t c_out, int64_t c_in, void* stream) {
  const int64_t n = c_out * 3 * c_in;
  cast_conv_weight_kernel<T><<<(unsigned)ceil_div(n, 256), 256, 0, (cudaStream_t)stream>>>(src, (T*)dst, (int)c_out, (int)c_in);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

extern "C" int oasr_unpermute_conv_wgrad(const float* src, float* dst, int64_t c_out, int64_t c_in, int accumulate, void* stream) {
  const int64_t n = c_out * 3 * c_in;
  unpermute_conv_wgrad_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, (cudaStream_t)stream>>>(src, dst, (int)c_out, (int)c_in, accumulate);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

extern "C" int oasr_mask_to_kvlen(const float* mask, int32_t* kv_len, int32_t* err, int64_t batch, int64_t S, void* stream) {
  OASR_REQUIRE(batch > 0 && S > 0 && mask && kv_len && err, "mask_to_kvlen: bad arguments");
  mask_to_kvlen_kernel<<<dim3((unsigned)batch, 16), 256, 0, (cudaStream_t)stream>>>(mask, kv_len, err, (int)S);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

template <typename T>
static int embed_fwd(const int64_t* ids, const float* emb, const float* pos, void* out, int64_t batch, int64_t S, int64_t d,
              int64_t pos_offset, int64_t n_rows_emb, void* stream) {
  OASR_REQUIRE(batch > 0 && S > 0 && (d & 3) == 0, "embed_fwd: bad shape");
  OASR_REQUIRE(aligned(emb, 16) && aligned(pos, 16) && aligned(out, 8), "embed_fwd: emb / pos 16-byte, out 8-byte alignment required");
  embed_fwd_kernel<T><<<(unsigned)(batch * S), 128, 0, (cudaStream_t)stream>>>(ids, emb, pos, (T*)out, batch * S, (int)S, (int)d,
                                                                           (int)pos_offset, n_rows_emb);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

template <typename T>
static int embed_bwd(const int64_t* ids, const void* dx, float* demb, float* dpos, int64_t batch, int64_t S, int64_t d,
              int64_t padding_idx, int64_t n_rows_emb, void* stream) {
  OASR_REQUIRE(batch > 0 && S > 0 && d <= 128 * EMB_COLS, "embed_bwd: bad shape");
  embed_bwd_kernel<T><<<(unsigned)(batch * S), 128, 0, (cudaStream_t)stream>>>(ids, (const T*)dx, demb, dpos, batch * S, (int)S, (int)d,
                                                                           padding_idx, n_rows_emb);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

template <typename T>
static int embed_fwd_packed(const int64_t* ids, const float* emb, const float* pos, void* out, const int32_t* src_rows,
                            int64_t N, int64_t S, int64_t d, int64_t n_rows_emb, void* stream) {
  OASR_REQUIRE(src_rows && N > 0 && S > 0 && (d & 3) == 0, "embed_fwd_packed: bad shape");
  OASR_REQUIRE(aligned(emb, 16) && aligned(pos, 16) && aligned(out, 8), "embed_fwd_packed: emb / pos 16-byte, out 8-byte alignment required");
  embed_fwd_kernel<T><<<(unsigned)N, 128, 0, (cudaStream_t)stream>>>(ids, emb, pos, (T*)out, N, (int)S, (int)d, 0, n_rows_emb,
                                                                    src_rows);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

template <typename T>
static int embed_bwd_packed(const int64_t* ids, const void* dx, float* demb, float* dpos, const int32_t* src_rows,
                            const int32_t* cu, int64_t n_seq, int64_t N, int64_t S, int64_t d, int64_t padding_idx,
                            int64_t n_rows_emb, void* stream) {
  OASR_REQUIRE(src_rows && cu && n_seq > 0 && N > 0 && S > 0 && d <= 128 * EMB_COLS, "embed_bwd_packed: bad shape");
  embed_bwd_kernel<T><<<(unsigned)(N > S ? N : S), 128, 0, (cudaStream_t)stream>>>(ids, (const T*)dx, demb, dpos, N, (int)S,
                                                                                 (int)d, padding_idx, n_rows_emb, src_rows, cu,
                                                                                 (int)n_seq);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

template <typename E>
static int im2col_conv1(const float* mel, void* A, int64_t batch, int64_t C, int64_t T, int64_t kpad, void* stream) {
  OASR_REQUIRE(kpad >= 3 * C && (kpad & 7) == 0, "im2col_conv1: kpad must be >= 3C and a multiple of 8");
  dim3 grid((unsigned)ceil_div(T, 32), (unsigned)batch);
  im2col_conv1_kernel<E><<<grid, 256, C * 34 * sizeof(float), (cudaStream_t)stream>>>(mel, (E*)A, (int)C, (int)T, (int)kpad);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

extern "C" int oasr_im2col_conv2(const void* h, void* A, int64_t batch, int64_t T_in, int64_t T_out, int64_t d, void* stream) {
  OASR_REQUIRE((d & 7) == 0, "im2col_conv2: d must be a multiple of 8");
  OASR_REQUIRE(aligned(h, 16) && aligned(A, 16), "im2col_conv2: 16-byte alignment required");
  im2col_conv2_kernel<<<(unsigned)(batch * T_out), 128, 0, (cudaStream_t)stream>>>((const uint16_t*)h, (uint16_t*)A, (int)T_in, (int)T_out, (int)d);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

template <typename T>
static int col2im_conv2_gelu_bwd(const void* dA, const void* pre1, void* dpre1, int64_t batch, int64_t T_in, int64_t T_out, int64_t d,
                          void* stream) {
  col2im_conv2_gelu_bwd_kernel<T><<<(unsigned)(batch * T_in), 128, 0, (cudaStream_t)stream>>>((const T*)dA, (const T*)pre1,
                                                                                             (T*)dpre1, (int)T_in, (int)T_out, (int)d);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

template <typename E>
static int add_pos(const void* x, const float* pos, void* out, int64_t rows, int64_t T, int64_t d, void* stream) {
  OASR_REQUIRE((d & 7) == 0, "add_pos: d must be a multiple of 8");
  OASR_REQUIRE(aligned(x, 16) && aligned(pos, 16) && aligned(out, 16), "add_pos: 16-byte alignment required");
  add_pos_kernel<E><<<grid_1d(rows * (d >> 3), 256), 256, 0, (cudaStream_t)stream>>>((const E*)x, pos, (E*)out, rows, (int)T, (int)d);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

template <typename T>
static int gelu_bwd(const void* dy, const void* pre, void* out, int64_t n, void* stream) {
  OASR_REQUIRE((n & 7) == 0, "gelu_bwd: n must be a multiple of 8");
  OASR_REQUIRE(aligned(dy, 16) && aligned(pre, 16) && aligned(out, 16), "gelu_bwd: 16-byte alignment required");
  gelu_bwd_kernel<T><<<grid_1d(n >> 3, 256), 256, 0, (cudaStream_t)stream>>>((const T*)dy, (const T*)pre, (T*)out, n);
  OASR_LAUNCH_CHECK();
  return OASR_OK;
}

template <typename T>
static int colsum(const void* dy, float* db, int64_t M, int64_t N, int64_t ld, void* stream) {
  OASR_REQUIRE(M > 0 && N > 0 && (ld & 1) == 0, "colsum: bad shape");
  const int col_tiles = (int)ceil_div(N, 256);
  int row_blocks = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(M, 64), (num_sms() * 6) / col_tiles + 1));
  const int rows_per_block = (int)ceil_div(M, row_blocks);
  row_blocks = (int)ceil_div(M, rows_per_block);
  cudaStream_t st = (cudaStream_t)stream;
  float* part = static_cast<float*>(scratch_alloc(sizeof(float) * row_blocks * N, st));
  if (!part) return OASR_ERR_CUDA;
  colsum_kernel<T><<<dim3(col_tiles, row_blocks), dim3(32, 8), 0, st>>>((const T*)dy, part, M, (int)N, ld, rows_per_block);
  OASR_LAUNCH_CHECK();
  const int rc = add_partials(part, row_blocks, N, db, st);
  scratch_free(part, st);
  return rc;
}

extern "C" int oasr_cast_conv_weight(const float* src, void* dst, int64_t c_out, int64_t c_in, void* stream) {
  return cast_conv_weight<bf16>(src, dst, c_out, c_in, stream);
}
extern "C" int oasr_embed_fwd(const int64_t* ids, const float* emb, const float* pos, void* out, int64_t batch,
                              int64_t S, int64_t d, int64_t pos_offset, int64_t n_rows_emb, void* stream) {
  return embed_fwd<bf16>(ids, emb, pos, out, batch, S, d, pos_offset, n_rows_emb, stream);
}
extern "C" int oasr_embed_bwd(const int64_t* ids, const void* dx, float* demb, float* dpos, int64_t batch, int64_t S,
                              int64_t d, int64_t padding_idx, int64_t n_rows_emb, void* stream) {
  return embed_bwd<bf16>(ids, dx, demb, dpos, batch, S, d, padding_idx, n_rows_emb, stream);
}
extern "C" int oasr_im2col_conv1(const float* mel, void* A, int64_t batch, int64_t C, int64_t T, int64_t kpad, void* stream) {
  return im2col_conv1<bf16>(mel, A, batch, C, T, kpad, stream);
}
extern "C" int oasr_col2im_conv2_gelu_bwd(const void* dA, const void* pre1, void* dpre1, int64_t batch, int64_t T_in,
                                          int64_t T_out, int64_t d, void* stream) {
  return col2im_conv2_gelu_bwd<bf16>(dA, pre1, dpre1, batch, T_in, T_out, d, stream);
}
extern "C" int oasr_add_pos(const void* x, const float* pos, void* out, int64_t rows, int64_t T, int64_t d, void* stream) {
  return add_pos<bf16>(x, pos, out, rows, T, d, stream);
}
extern "C" int oasr_gelu_bwd(const void* dy, const void* pre, void* out, int64_t n, void* stream) {
  return gelu_bwd<bf16>(dy, pre, out, n, stream);
}
extern "C" int oasr_colsum_bf16(const void* dy, float* db, int64_t M, int64_t N, int64_t ld, void* stream) {
  return colsum<bf16>(dy, db, M, N, ld, stream);
}

extern "C" int oasr_cast_conv_weight16(const float* src, void* dst, int64_t c_out, int64_t c_in, int dtype, void* stream) {
  return OASR_BY_DTYPE16(dtype, cast_conv_weight, src, dst, c_out, c_in, stream);
}
extern "C" int oasr_embed_fwd16(const int64_t* ids, const float* emb, const float* pos, void* out, int64_t batch,
                                int64_t S, int64_t d, int64_t pos_offset, int64_t n_rows_emb, int dtype, void* stream) {
  return OASR_BY_DTYPE16(dtype, embed_fwd, ids, emb, pos, out, batch, S, d, pos_offset, n_rows_emb, stream);
}
extern "C" int oasr_embed_bwd16(const int64_t* ids, const void* dx, float* demb, float* dpos, int64_t batch, int64_t S,
                                int64_t d, int64_t padding_idx, int64_t n_rows_emb, int dtype, void* stream) {
  return OASR_BY_DTYPE16(dtype, embed_bwd, ids, dx, demb, dpos, batch, S, d, padding_idx, n_rows_emb, stream);
}
extern "C" int oasr_im2col_conv1_16(const float* mel, void* A, int64_t batch, int64_t C, int64_t T, int64_t kpad, int dtype,
                                    void* stream) {
  return OASR_BY_DTYPE16(dtype, im2col_conv1, mel, A, batch, C, T, kpad, stream);
}
extern "C" int oasr_col2im_conv2_gelu_bwd16(const void* dA, const void* pre1, void* dpre1, int64_t batch, int64_t T_in,
                                            int64_t T_out, int64_t d, int dtype, void* stream) {
  return OASR_BY_DTYPE16(dtype, col2im_conv2_gelu_bwd, dA, pre1, dpre1, batch, T_in, T_out, d, stream);
}
extern "C" int oasr_add_pos16(const void* x, const float* pos, void* out, int64_t rows, int64_t T, int64_t d, int dtype,
                              void* stream) {
  return OASR_BY_DTYPE16(dtype, add_pos, x, pos, out, rows, T, d, stream);
}
extern "C" int oasr_gelu_bwd16(const void* dy, const void* pre, void* out, int64_t n, int dtype, void* stream) {
  return OASR_BY_DTYPE16(dtype, gelu_bwd, dy, pre, out, n, stream);
}
extern "C" int oasr_colsum16(const void* dy, float* db, int64_t M, int64_t N, int64_t ld, int dtype, void* stream) {
  return OASR_BY_DTYPE16(dtype, colsum, dy, db, M, N, ld, stream);
}

extern "C" int oasr_embed_fwd_packed16(const int64_t* ids, const float* emb, const float* pos, void* out,
                                       const int32_t* src_rows, int64_t N, int64_t S, int64_t d, int64_t n_rows_emb, int dtype,
                                       void* stream) {
  return OASR_BY_DTYPE16(dtype, embed_fwd_packed, ids, emb, pos, out, src_rows, N, S, d, n_rows_emb, stream);
}
extern "C" int oasr_embed_bwd_packed16(const int64_t* ids, const void* dx, float* demb, float* dpos, const int32_t* src_rows,
                                       const int32_t* cu_seqlens, int64_t B, int64_t N, int64_t S, int64_t d,
                                       int64_t padding_idx, int64_t n_rows_emb, int dtype, void* stream) {
  return OASR_BY_DTYPE16(dtype, embed_bwd_packed, ids, dx, demb, dpos, src_rows, cu_seqlens, B, N, S, d, padding_idx,
                         n_rows_emb, stream);
}
