// nn_ops.cu — normalisation, pointwise and attention kernels shared by the s2mel / codec paths
// (channels-last fp32, see ops.h).  Reference semantics cited at each kernel.
#include "ops.h"
#include <cuda_bf16.h>

namespace {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// GEMM operands of the fp16 tensor-core path are written by the kernel that produces them: every pointwise kernel
// below takes an optional fp16 destination next to (or instead of) the fp32 one.
__device__ __forceinline__ void put(float* __restrict__ y, __half* __restrict__ y16, long long i, float v) {
  if (y) y[i] = v;
  if (y16) y16[i] = __float2half_rn(v);
}

// One warp per row.  MODE 0: LayerNorm (two-pass), MODE 1: RMSNorm (gpt_fast/model.py:317-333).
template <int MODE>
__global__ void rownorm_kernel(const float* __restrict__ x, float* __restrict__ y, long long rows, int T,
                               int C, const float* __restrict__ w, const float* __restrict__ b, float eps,
                               const float* __restrict__ m0, const float* __restrict__ m1, int mod_stride,
                               __half* __restrict__ y16) {
  pdl_wait();
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const int bidx = (int)(row / T);
  const float* xr = x + row * C;
  float s = 0.f;
  for (int i = lane; i < C; i += 32) s += xr[i];
  float mean = 0.f, q = 0.f;
  if (MODE == 0) {
    mean = warp_sum(s) / C;
    for (int i = lane; i < C; i += 32) { float d = xr[i] - mean; q += d * d; }
  } else {
    for (int i = lane; i < C; i += 32) q += xr[i] * xr[i];
  }
  const float rstd = rsqrtf(warp_sum(q) / C + eps);
  for (int i = lane; i < C; i += 32) {
    float v = (xr[i] - mean) * rstd;
    if (MODE == 0) {
      if (w) v = v * w[i] + (b ? b[i] : 0.f);
      // modulate(x, shift, scale) = x * (1 + scale) + shift   (diffusion_transformer.py:11-12)
      if (m0) v = v * (1.f + m0[(long long)bidx * mod_stride + i]) + m1[(long long)bidx * mod_stride + i];
    } else {
      v *= w[i];
      // AdaptiveLayerNorm: weight * norm(x) + bias             (gpt_fast/model.py:20-39)
      if (m0) v = m0[(long long)bidx * mod_stride + i] * v + m1[(long long)bidx * mod_stride + i];
    }
    put(y, y16, row * C + i, v);
  }
}

__global__ void gn_stats_kernel(const float* __restrict__ x, double* stats, long long n_per) {
  const int b = blockIdx.y;
  const float* xb = x + (long long)b * n_per;
  double s = 0, q = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_per; i += (long long)gridDim.x * blockDim.x) {
    const double v = xb[i];
    s += v; q += v * v;
  }
  __shared__ double ss[256], qq[256];
  ss[threadIdx.x] = s; qq[threadIdx.x] = q;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) { ss[threadIdx.x] += ss[threadIdx.x + o]; qq[threadIdx.x] += qq[threadIdx.x + o]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) { atomicAdd(&stats[2 * b], ss[0]); atomicAdd(&stats[2 * b + 1], qq[0]); }
}
__global__ void gn_apply_mish_kernel(const float* __restrict__ x, float* __restrict__ y, const double* stats,
                                     long long n_per, int C, const float* __restrict__ w,
                                     const float* __restrict__ bb, float eps) {
  const int b = blockIdx.y;
  const double mean = stats[2 * b] / n_per;
  const double var = stats[2 * b + 1] / n_per - mean * mean;
  const float rstd = (float)(1.0 / sqrt(var + (double)eps));
  const float fm = (float)mean;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_per; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    float v = (x[(long long)b * n_per + i] - fm) * rstd * w[c] + bb[c];
    const float sp = (v > 20.f) ? v : log1pf(expf(v));   // F.mish = x * tanh(softplus(x))
    y[(long long)b * n_per + i] = v * tanhf(sp);
  }
}

// Row-indexed kernels below take their rows from grid y with a grid-stride loop (row_grid): gridDim.y stops at 65535, and a
// packed CFM solve can hold more rows than that.
__global__ void dwconv_kernel(const float* __restrict__ x, float* __restrict__ y, int T, int C,
                              const float* __restrict__ w, const float* __restrict__ b, int k) {
  const int bi = blockIdx.z;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float* xb = x + (long long)bi * T * C;
  const int pad = (k - 1) / 2;
  for (int t = blockIdx.y; t < T; t += gridDim.y) {
    float acc = b ? b[c] : 0.f;
    for (int j = 0; j < k; ++j) {
      const int ts = t + j - pad;
      if (ts >= 0 && ts < T) acc = fmaf(xb[(long long)ts * C + c], w[c * k + j], acc);
    }
    y[((long long)bi * T + t) * C + c] = acc;
  }
}

__global__ void nearest_kernel(const float* __restrict__ x, float* __restrict__ y, int Tin, int Tout, int C) {
  const int bi = blockIdx.z;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  // aten nearest_idx: scale = (float)in/out; src = min((int)floorf(dst * scale), in - 1)
  const float scale = (float)Tin / (float)Tout;
  for (int t = blockIdx.y; t < Tout; t += gridDim.y) {
    int src = (int)floorf((float)t * scale);
    if (src > Tin - 1) src = Tin - 1;
    y[((long long)bi * Tout + t) * C + c] = x[((long long)bi * Tin + src) * C + c];
  }
}

// ids outside [0, nrows) never index the table: the row is zero-filled and the engine flag records the position
// (torch's F.embedding raises IndexError there; the ABI call returns IDX_ERR_ARG after the stream drains)
__global__ void embedding_kernel(const float* __restrict__ table, const int* __restrict__ ids, float* out, int C,
                                 int nrows, int* bad) {
  const int t = blockIdx.y;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  const int id = ids[t];
  const bool ok = id >= 0 && id < nrows;
  if (!ok && c == 0) atomicCAS(bad, 0, t + 1);
  if (c < C) out[(long long)t * C + c] = ok ? table[(long long)id * C + c] : 0.f;
}

__global__ void swiglu_kernel(const float* __restrict__ ab, float* __restrict__ y, long long rows, int N) {
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * N) return;
  const long long r = i / N;
  const int c = (int)(i % N);
  const float a = ab[r * 2 * N + c], b = ab[r * 2 * N + N + c];
  y[i] = a / (1.f + expf(-a)) * b;   // F.silu(w1 x) * (w3 x)  (gpt_fast/model.py:311-314)
}

__global__ void wn_gate_kernel(const float* __restrict__ xin, const float* __restrict__ g, int g_stride,
                               float* __restrict__ y, int T, int N) {
  pdl_wait();
  // fused_add_tanh_sigmoid_multiply (s2mel/modules/commons.py:132-141)
  const int bi = blockIdx.z;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)T * N) return;
  const long long t = i / N;
  const int c = (int)(i % N);
  const float* xr = xin + ((long long)bi * T + t) * 2 * N;
  const float a = xr[c] + g[(long long)bi * g_stride + c];
  const float s = xr[N + c] + g[(long long)bi * g_stride + N + c];
  y[((long long)bi * T + t) * N + c] = tanhf(a) * (1.f / (1.f + expf(-s)));
}

__global__ void copy_cols_kernel(const float* __restrict__ src, int lds, float* __restrict__ dst, int ldo,
                                 int col0, long long rows, int C, __half* __restrict__ dst16) {
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * C) return;
  const long long r = i / C;
  const int c = (int)(i % C);
  put(dst, dst16, r * ldo + col0 + c, src[r * lds + c]);
}
__global__ void bcast_cols_kernel(const float* __restrict__ vec, float* __restrict__ dst, int ldo, int col0,
                                  int T, int C) {
  const int bi = blockIdx.z;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)T * C) return;
  const long long t = i / C;
  const int c = (int)(i % C);
  dst[((long long)bi * T + t) * ldo + col0 + c] = vec[(long long)bi * C + c];
}
__global__ void silu_kernel(float* x, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) { const float v = x[i]; x[i] = v / (1.f + expf(-v)); }
}
// Source row of output row i of a reflect-padded frame of T rows (encodec.py pad1d): an input no longer than the larger pad
// is first zero-extended to Tr = max(left, right) + 1 rows, reflected, then cropped back.  Returns the row, or -1 where the
// frame holds one of those zeros.  For T > max(left, right) this is F.pad(mode='reflect').
__device__ __forceinline__ int reflect_src(int i, int T, int left, int right) {
  const int Tr = max(T, max(left, right) + 1);
  int t = i - left;
  if (t < 0) t = -t;
  if (t >= Tr) t = 2 * (Tr - 1) - t;
  return t < T ? t : -1;
}
__global__ void reflect_pad_kernel(const float* __restrict__ x, float* __restrict__ y, int T, int C, int left, int right,
                                   int Tout, __half* __restrict__ y16) {
  pdl_wait();
  const int bi = blockIdx.z;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  for (int i = blockIdx.y; i < Tout; i += gridDim.y) {
    const int t = reflect_src(i, T, left, right);
    put(y, y16, ((long long)bi * Tout + i) * C + c, t >= 0 ? x[((long long)bi * T + t) * C + c] : 0.f);
  }
}
// segment of row r in a layout where segment u starts at row off[u] + u * gap: the largest such u with start <= r
__device__ __forceinline__ int segment_of(const int* __restrict__ off, int n, int r, int gap) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (off[mid] + mid * gap <= r) lo = mid; else hi = mid - 1;
  }
  return lo;
}
__global__ void reflect_pad_seg_kernel(const float* __restrict__ x, __half* __restrict__ y16, int T, int C, int left, int gap,
                                       int Tout, const int* __restrict__ off, int n) {
  pdl_wait();
  const int bi = blockIdx.z;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  for (int i = blockIdx.y; i < Tout; i += gridDim.y) {
    const int u = segment_of(off, n, i, gap);
    const int t0 = off[u], Tu = off[u + 1] - t0;
    const int t = reflect_src(i - t0 - u * gap, Tu, left, gap - left);     // reflect_pad_kernel on the segment alone
    y16[((long long)bi * Tout + i) * C + c] = __float2half_rn(t >= 0 ? x[((long long)bi * T + t0 + t) * C + c] : 0.f);
  }
}
__global__ void compact_seg_kernel(const __half* __restrict__ x, __half* __restrict__ y, int T, int Mg, int C, int gap,
                                   const int* __restrict__ off, int n) {
  pdl_wait();
  const int bi = blockIdx.z;
  const int c = (blockIdx.x * blockDim.x + threadIdx.x) * 8;      // 16-byte vectors (C % 8 == 0)
  if (c >= C) return;
  for (int r = blockIdx.y; r < T; r += gridDim.y) {
    const int u = segment_of(off, n, r, 0);
    *(uint4*)(y + ((long long)bi * T + r) * C + c) = *(const uint4*)(x + ((long long)bi * Mg + r + u * gap) * C + c);
  }
}
__global__ void cfg_euler_rows_kernel(float* x, const float* vc, const float* vu, float dt, float rate, int T, int C,
                                      const unsigned char* __restrict__ zero_rows) {
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)T * C) return;
  const int t = (int)(i / C);
  const float d = (1.0f + rate) * vc[i] - rate * vu[i];      // cfg_euler_kernel, with each segment's own prompt rows
  x[i] = zero_rows[t] ? 0.f : x[i] + dt * d;
}
__global__ void zero_kernel(float* x, long long n) {
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) x[i] = 0.f;
}
__global__ void rope_table_kernel(float* tab, int T, int hd) {
  const int t = blockIdx.x;
  const int i = threadIdx.x;
  if (i >= hd / 2) return;
  // freqs = 1 / base^(2i/hd); angle = t * freq (fp32), cache = (cos, sin)   (model.py:336-346)
  const float freq = 1.0f / powf(10000.f, (float)(2 * i) / (float)hd);
  const float ang = (float)t * freq;
  tab[((long long)t * (hd / 2) + i) * 2] = cosf(ang);
  tab[((long long)t * (hd / 2) + i) * 2 + 1] = sinf(ang);
}
__global__ void cfg_euler_kernel(float* x, const float* vc, const float* vu, float dt, float rate, int T,
                                 int C, int P) {
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)T * C) return;
  const int t = (int)(i / C);
  // dphi = (1 + r) * dphi_cond - r * dphi_uncond ; x = x + dt * dphi ; x[:, :, :P] = 0
  // (flow_matching.py:96-113)
  const float d = (1.0f + rate) * vc[i] - rate * vu[i];
  x[i] = (t < P) ? 0.f : x[i] + dt * d;
}

// ------------------------------------------------------------------------ attention ----
// fp32 flash attention, 64 queries x 64 keys per tile, head_dim 64, RoPE applied on load
// (F.scaled_dot_product_attention, gpt_fast/model.py:293-306).
constexpr int AQ = 64, AK = 64, AD = 64;
__global__ void __launch_bounds__(256) attention_kernel(const float* __restrict__ qkv, float* __restrict__ out,
                                                        int T, int H, const float* __restrict__ rope) {
  extern __shared__ float sm[];
  float* Qt = sm;                 // [AD][AQ]
  float* Kt = Qt + AD * AQ;       // [AD][AK]
  float* Vs = Kt + AD * AK;       // [AK][AD]
  float* Pt = Vs + AK * AD;       // [AK][AQ]
  const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * AQ;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int ld = 3 * H * AD;
  const float* base = qkv + (long long)b * T * ld;
  // load + rotate Q (pairs), scaled by 1/sqrt(64)
  for (int i = tid; i < AQ * (AD / 2); i += 256) {
    const int r = i / (AD / 2), pi = i % (AD / 2);
    const int t = q0 + r;
    float a = 0.f, c = 0.f;
    if (t < T) {
      const float* qp = base + (long long)t * ld + h * AD + 2 * pi;
      const float cs = rope[((long long)t * (AD / 2) + pi) * 2], sn = rope[((long long)t * (AD / 2) + pi) * 2 + 1];
      const float x0 = qp[0], x1 = qp[1];
      a = (x0 * cs - x1 * sn) * 0.125f;
      c = (x1 * cs + x0 * sn) * 0.125f;
    }
    Qt[(2 * pi) * AQ + r] = a;
    Qt[(2 * pi + 1) * AQ + r] = c;
  }
  float m[4], l[4], o[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    m[i] = -INFINITY; l[i] = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) o[i][j] = 0.f;
  }
  for (int k0 = 0; k0 < T; k0 += AK) {
    __syncthreads();
    for (int i = tid; i < AK * (AD / 2); i += 256) {
      const int r = i / (AD / 2), pi = i % (AD / 2);
      const int t = k0 + r;
      float a = 0.f, c = 0.f, v0 = 0.f, v1 = 0.f;
      if (t < T) {
        const float* kp = base + (long long)t * ld + H * AD + h * AD + 2 * pi;
        const float cs = rope[((long long)t * (AD / 2) + pi) * 2], sn = rope[((long long)t * (AD / 2) + pi) * 2 + 1];
        const float x0 = kp[0], x1 = kp[1];
        a = x0 * cs - x1 * sn;
        c = x1 * cs + x0 * sn;
        const float* vp = kp + H * AD;
        v0 = vp[0]; v1 = vp[1];
      }
      Kt[(2 * pi) * AK + r] = a;
      Kt[(2 * pi + 1) * AK + r] = c;
      Vs[r * AD + 2 * pi] = v0;
      Vs[r * AD + 2 * pi + 1] = v1;
    }
    __syncthreads();
    float s[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
#pragma unroll 8
    for (int d = 0; d < AD; ++d) {
      const float4 qa = *(const float4*)(Qt + d * AQ + ty * 4);
      const float4 kb = *(const float4*)(Kt + d * AK + tx * 4);
      const float qv[4] = {qa.x, qa.y, qa.z, qa.w}, kv[4] = {kb.x, kb.y, kb.z, kb.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) s[i][j] = fmaf(qv[i], kv[j], s[i][j]);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (k0 + tx * 4 + j >= T) s[i][j] = -INFINITY;
        mx = fmaxf(mx, s[i][j]);
      }
#pragma unroll
      for (int xo = 1; xo <= 8; xo <<= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, xo));
      const float mn = fmaxf(m[i], mx);
      const float corr = (m[i] == -INFINITY) ? 0.f : __expf(m[i] - mn);
      float rs = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float p = (s[i][j] == -INFINITY) ? 0.f : __expf(s[i][j] - mn);
        s[i][j] = p;
        rs += p;
      }
#pragma unroll
      for (int xo = 1; xo <= 8; xo <<= 1) rs += __shfl_xor_sync(0xffffffffu, rs, xo);
      l[i] = l[i] * corr + rs;
      m[i] = mn;
#pragma unroll
      for (int j = 0; j < 4; ++j) o[i][j] *= corr;
#pragma unroll
      for (int j = 0; j < 4; ++j) Pt[(tx * 4 + j) * AQ + ty * 4 + i] = s[i][j];
    }
    __syncthreads();
#pragma unroll 8
    for (int k = 0; k < AK; ++k) {
      const float4 pa = *(const float4*)(Pt + k * AQ + ty * 4);
      const float4 vb = *(const float4*)(Vs + k * AD + tx * 4);
      const float pv[4] = {pa.x, pa.y, pa.z, pa.w}, vv[4] = {vb.x, vb.y, vb.z, vb.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) o[i][j] = fmaf(pv[i], vv[j], o[i][j]);
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int t = q0 + ty * 4 + i;
    if (t >= T) continue;
    const float inv = l[i] > 0.f ? 1.f / l[i] : 0.f;
    float4 r = make_float4(o[i][0] * inv, o[i][1] * inv, o[i][2] * inv, o[i][3] * inv);
    *(float4*)(out + ((long long)b * T + t) * H * AD + h * AD + tx * 4) = r;
  }
}

// ---- tensor-core attention: q / k rotated, q scaled by FLASH_Q_SCALE, and the heads split to fp16 Qr | Kr | Vb [B*H][T][64],
// the layout EPI_ROPE writes and the wgmma flash attention reads ----
__global__ void rope_split_fa_kernel(const float* __restrict__ qkv, const float* __restrict__ rope,
                                     __half* __restrict__ Qr, __half* __restrict__ Kr,
                                     __half* __restrict__ Vb, int T, int H) {
  pdl_wait();
  const int t = blockIdx.x, h = blockIdx.y, b = blockIdx.z, i = threadIdx.x;  // 64 threads
  const int ld = 3 * H * AD;
  const float* row = qkv + ((long long)b * T + t) * ld;
  const long long bh = (long long)b * H + h;
  if (i < AD / 2) {
    const float cs = rope[((long long)t * (AD / 2) + i) * 2], sn = rope[((long long)t * (AD / 2) + i) * 2 + 1];
    const float q0 = row[h * AD + 2 * i], q1 = row[h * AD + 2 * i + 1];
    const float k0 = row[H * AD + h * AD + 2 * i], k1 = row[H * AD + h * AD + 2 * i + 1];
    *(__half2*)(Qr + (bh * T + t) * AD + 2 * i) =
        __floats2half2_rn((q0 * cs - q1 * sn) * FLASH_Q_SCALE, (q1 * cs + q0 * sn) * FLASH_Q_SCALE);
    *(__half2*)(Kr + (bh * T + t) * AD + 2 * i) = __floats2half2_rn(k0 * cs - k1 * sn, k1 * cs + k0 * sn);
  }
  Vb[(bh * T + t) * AD + i] = __float2half_rn(row[2 * H * AD + h * AD + i]);
}

}  // namespace

#define LAUNCH_CHECK(e)            \
  do {                             \
    IDX_CUDA(cudaGetLastError());  \
    (e)->launches++;               \
  } while (0)

// grid y of the row-indexed kernels: one block row per row up to the hardware limit, the kernels loop beyond it
static unsigned row_grid(long long rows) { return (unsigned)std::min<long long>(rows, 65535); }

void layernorm(idx_engine* e, const float* x, float* y, int B, int T, int C, const float* w, const float* b,
               float eps, const float* scale, const float* shift, int mod_stride, __half* y16) {
  const long long rows = (long long)B * T;
  launch_pdl(e, rownorm_kernel<0>, dim3((unsigned)((rows + 7) / 8)), dim3(256), 0, x, y, rows, T, C, w, b, eps, scale, shift, mod_stride, y16);
  LAUNCH_CHECK(e);
}
void rmsnorm_adaln(idx_engine* e, const float* x, float* y, int B, int T, int C, const float* nw, const float* mw,
                   const float* mb, int mod_stride, float eps, __half* y16) {
  const long long rows = (long long)B * T;
  launch_pdl(e, rownorm_kernel<1>, dim3((unsigned)((rows + 7) / 8)), dim3(256), 0, x, y, rows, T, C, nw, (const float*)nullptr, eps, mw, mb, mod_stride, y16);
  LAUNCH_CHECK(e);
}
void groupnorm1_mish(idx_engine* e, const float* x, float* y, int B, int T, int C, const float* w, const float* b,
                     float eps) {
  double* stats = (double*)e->arena.alloc(sizeof(double) * 2 * B);
  IDX_CUDA(cudaMemsetAsync(stats, 0, sizeof(double) * 2 * B, e->stream));
  const long long n_per = (long long)T * C;
  dim3 grid((unsigned)std::min<long long>(296, (n_per + 255) / 256), B);
  gn_stats_kernel<<<grid, 256, 0, e->stream>>>(x, stats, n_per);
  LAUNCH_CHECK(e);
  gn_apply_mish_kernel<<<grid, 256, 0, e->stream>>>(x, y, stats, n_per, C, w, b, eps);
  LAUNCH_CHECK(e);
}
void dwconv1d(idx_engine* e, const float* x, float* y, int B, int T, int C, const float* w, const float* b, int k) {
  dim3 grid((C + 127) / 128, row_grid(T), B);
  dwconv_kernel<<<grid, 128, 0, e->stream>>>(x, y, T, C, w, b, k);
  LAUNCH_CHECK(e);
}
void nearest_interp(idx_engine* e, const float* x, float* y, int B, int Tin, int Tout, int C) {
  dim3 grid((C + 127) / 128, row_grid(Tout), B);
  nearest_kernel<<<grid, 128, 0, e->stream>>>(x, y, Tin, Tout, C);
  LAUNCH_CHECK(e);
}
void embedding_rows(idx_engine* e, const float* table, const int* ids, float* out, int n, int C, int nrows) {
  dim3 grid((C + 127) / 128, n);
  embedding_kernel<<<grid, 128, 0, e->stream>>>(table, ids, out, C, nrows, e->dev_flag);
  LAUNCH_CHECK(e);
}
void swiglu(idx_engine* e, const float* ab, float* y, long long rows, int N) {
  launch_pdl(e, swiglu_kernel, dim3((unsigned)((rows * N + 255) / 256)), dim3(256), 0, ab, y, rows, N);
  LAUNCH_CHECK(e);
}
void wn_gate(idx_engine* e, const float* xin, const float* g, int g_stride, float* y, int B, int T, int N) {
  dim3 grid((unsigned)(((long long)T * N + 255) / 256), 1, B);
  launch_pdl(e, wn_gate_kernel, grid, dim3(256), 0, xin, g, g_stride, y, T, N);
  LAUNCH_CHECK(e);
}
void copy_cols(idx_engine* e, const float* src, int lds, float* dst, int ldo, int col0, long long rows, int C, __half* dst16) {
  launch_pdl(e, copy_cols_kernel, dim3((unsigned)((rows * C + 255) / 256)), dim3(256), 0, src, lds, dst, ldo, col0, rows, C, dst16);
  LAUNCH_CHECK(e);
}
void bcast_cols(idx_engine* e, const float* vec, float* dst, int ldo, int col0, int B, int T, int C) {
  dim3 grid((unsigned)(((long long)T * C + 255) / 256), 1, B);
  bcast_cols_kernel<<<grid, 256, 0, e->stream>>>(vec, dst, ldo, col0, T, C);
  LAUNCH_CHECK(e);
}
void silu_inplace(idx_engine* e, float* x, long long n) {
  silu_kernel<<<(unsigned)((n + 255) / 256), 256, 0, e->stream>>>(x, n);
  LAUNCH_CHECK(e);
}
void fill_zero(idx_engine* e, float* x, long long n) {
  launch_pdl(e, zero_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, x, n);
  LAUNCH_CHECK(e);
}
void reflect_pad_rows(idx_engine* e, const float* x, float* y, int B, int T, int C, int left, int right, __half* y16) {
  const int Tout = T + left + right;
  dim3 grid((C + 127) / 128, row_grid(Tout), B);
  launch_pdl(e, reflect_pad_kernel, grid, dim3(128), 0, x, y, T, C, left, right, Tout, y16);
  LAUNCH_CHECK(e);
}
void reflect_pad_segments(idx_engine* e, const float* x, __half* y16, int B, int C, int left, int right, const Segments& sg) {
  const int gap = left + right, Tout = sg.total() + sg.n() * gap;
  dim3 grid((C + 127) / 128, row_grid(Tout), B);
  launch_pdl(e, reflect_pad_seg_kernel, grid, dim3(128), 0, x, y16, sg.total(), C, left, gap, Tout, (const int*)sg.d_off, sg.n());
  LAUNCH_CHECK(e);
}
void compact_segments16(idx_engine* e, const __half* x, __half* y, int B, int C, int gap, const Segments& sg) {
  IDX_CHECK(C % 8 == 0, IDX_ERR_ARG, "compact_segments16: C must be a multiple of 8");
  const int T = sg.total(), Mg = T + (sg.n() - 1) * gap;
  dim3 grid((C / 8 + 63) / 64, row_grid(T), B);
  launch_pdl(e, compact_seg_kernel, grid, dim3(64), 0, x, y, T, Mg, C, gap, (const int*)sg.d_off, sg.n());
  LAUNCH_CHECK(e);
}
void cfg_euler_rows(idx_engine* e, float* x, const float* v_cond, const float* v_uncond, float dt, float rate, int T, int C,
                    const unsigned char* zero_rows) {
  launch_pdl(e, cfg_euler_rows_kernel, dim3((unsigned)(((long long)T * C + 255) / 256)), dim3(256), 0, x, v_cond, v_uncond, dt,
             rate, T, C, zero_rows);
  LAUNCH_CHECK(e);
}
void segments_upload(idx_engine* e, Segments& sg) {
  std::vector<int4> tiles;
  for (int u = 0; u < sg.n(); ++u)
    for (int q = sg.off[u]; q < sg.off[u + 1]; q += 128) tiles.push_back(make_int4(q, sg.off[u], sg.off[u + 1], 0));
  sg.fa_tiles = (int)tiles.size();
  sg.d_off = e->arena.get<int>(sg.off.size());
  sg.d_fa_tiles = e->arena.get<int4>(tiles.size());
  idx_to_device(e, sg.d_off, sg.off.data(), sg.off.size() * sizeof(int));
  idx_to_device(e, sg.d_fa_tiles, tiles.data(), tiles.size() * sizeof(int4));
}
void rope_table(idx_engine* e, float* tab, int T, int hd) {
  rope_table_kernel<<<T, 32, 0, e->stream>>>(tab, T, hd);
  LAUNCH_CHECK(e);
}
void rope_table_segments(idx_engine* e, float* tab, const Segments& sg, int hd) {
  for (int u = 0; u < sg.n(); ++u) rope_table(e, tab + (size_t)sg.off[u] * hd, sg.len(u), hd);
}
void attention_rope(idx_engine* e, const float* qkv, float* out, int B, int T, int H, const float* rope) {
  if (gemm_default_backend(e) == 0) {
    // tensor cores: rotate / split once, then the wgmma flash attention
    const size_t mark = e->arena.off;
    const size_t n = (size_t)B * H * T * AD;
    __half* Qr = (__half*)e->arena.alloc(n * 2);
    __half* Kr = (__half*)e->arena.alloc(n * 2);
    __half* Vb = (__half*)e->arena.alloc(n * 2);
    launch_pdl(e, rope_split_fa_kernel, dim3(T, H, B), dim3(AD), 0, qkv, rope, Qr, Kr, Vb, T, H);
    LAUNCH_CHECK(e);
    flash_attention_wgmma(e, Qr, Kr, Vb, out, nullptr, B, T, H);
    e->arena.off = mark;
    return;
  }
  const int smem = 4 * AQ * AD * sizeof(float);
  if (!(e->attr_done & 8u)) {      // per engine = per device: function attributes live in the device's context
    IDX_CUDA(cudaFuncSetAttribute(attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    e->attr_done |= 8u;
  }
  dim3 grid((T + AQ - 1) / AQ, H, B);
  attention_kernel<<<grid, 256, smem, e->stream>>>(qkv, out, T, H, rope);
  LAUNCH_CHECK(e);
}
void cfg_euler(idx_engine* e, float* x, const float* v_cond, const float* v_uncond, float dt, float rate, int T,
               int C, int P) {
  launch_pdl(e, cfg_euler_kernel, dim3((unsigned)(((long long)T * C + 255) / 256)), dim3(256), 0, x, v_cond, v_uncond, dt, rate, T, C, P);
  LAUNCH_CHECK(e);
}

// ---- the unfused strict-fp32 attention pieces (emotion conformer, w2v-BERT encoder with gemm_backend 1) ----
namespace {
// exact-exp row softmax over the first T of Tp columns (columns T..Tp-1 set to 0: the K padding of the P V GEMM)
__global__ void softmax_rows_g_kernel(float* __restrict__ S, long long rows, int T, int Tp) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  float* r = S + row * Tp;
  float mx = -INFINITY;
  for (int i = lane; i < T; i += 32) mx = fmaxf(mx, r[i]);
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
  for (int i = lane; i < T; i += 32) { const float p = expf(r[i] - mx); r[i] = p; sum += p; }
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float inv = 1.f / sum;
  for (int i = lane; i < Tp; i += 32) r[i] = (i < T) ? r[i] * inv : 0.f;
}
__global__ void heads_merge_g_kernel(const float* __restrict__ O, float* __restrict__ out, int T, int H, int dk) {
  const int t = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  for (int i = threadIdx.x; i < dk; i += blockDim.x)
    out[((long long)b * T + t) * H * dk + h * dk + i] = O[(((long long)b * H + h) * T + t) * dk + i];
}
}  // namespace
void softmax_rows_exact(idx_engine* e, float* S, long long rows, int T, int Tp) {
  softmax_rows_g_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, e->stream>>>(S, rows, T, Tp);
  LAUNCH_CHECK(e);
}
void heads_merge(idx_engine* e, const float* O, float* out, int B, int T, int H, int dk) {
  heads_merge_g_kernel<<<dim3(T, H, B), 128, 0, e->stream>>>(O, out, T, H, dk);
  LAUNCH_CHECK(e);
}
