// ops.cu — generic multi-tap GEMM (Conv1d / ConvTranspose1d / Linear on channels-last fp32) and
// layout helpers.  Two back ends behind conv_gemm():
//   * wgmma implicit GEMM (gemm_tc.cu): TMA-staged operands, register accumulators, tf32 or fp16;
//   * a plain SIMT fp32 tile kernel (this file): bring-up / odd-shape path and the reference
//     the tensor-core path is tested against.  Both are CUDA; neither is a CPU fallback.
#include "stages.h"
#include <cstdlib>
#include <cstdio>

bool gemm_tc_supported(const ConvGemm& g);
void gemm_tc_launch(idx_engine* e, const ConvGemm& g);

namespace {

__device__ __forceinline__ float apply_act(float v, int act) {
  switch (act) {
    case ACT_GELU_ERF: return 0.5f * v * (1.f + erff(v * 0.70710678118654752f));
    case ACT_SILU: return v / (1.f + __expf(-v));
    case ACT_MISH: {
      float sp = (v > 20.f) ? v : log1pf(__expf(v));
      return v * tanhf(sp);
    }
    case ACT_GELU_TANH: {
      float u = 0.7978845608028654f * (v + 0.044715f * v * v * v);
      return 0.5f * v * (1.f + tanhf(u));
    }
    case ACT_RELU: return v > 0.f ? v : 0.f;
    default: return v;
  }
}

constexpr int BM = 64, BN = 64, BK = 16;

__global__ void __launch_bounds__(256) conv_gemm_simt_kernel(const ConvGemm g) {
  __shared__ float As[BK][BM + 4];
  __shared__ float Bs[BK][BN + 4];
  const int b = blockIdx.z;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const long long abs_ = g.a_bcast ? 0 : (g.a_batch_stride ? g.a_batch_stride : (long long)g.Tin * g.K);
  const int lda = g.lda ? g.lda : g.K;
  const float* Ab = g.A + (long long)b * abs_;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  const int ar = tid >> 2, ak = (tid & 3) * 4;   // A tile: row, k offset
  const int bk = tid >> 4, bn = (tid & 15) * 4;  // B tile: k, n offset
  for (int tap = 0; tap < g.taps; ++tap) {
    const int row = m0 + ar;
    int st = row + tap * g.dil - g.pad;
    if (g.reflect) {
      if (st < 0) st = -st;
      if (st >= g.Tin) st = 2 * (g.Tin - 1) - st;
    }
    const bool rvalid = row < g.M && st >= 0 && st < g.Tin;
    const float* arow = Ab + (long long)st * lda;
    for (int k0 = 0; k0 < g.K; k0 += BK) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int kk = k0 + ak + i;
        As[ak + i][ar] = (rvalid && kk < g.K) ? __ldg(arow + kk) : 0.f;
      }
      if (g.W) {
        const int kk = k0 + bk;
        const float* wrow = g.W + ((long long)tap * g.K + kk) * g.N;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int n = n0 + bn + i;
          Bs[bk][bn + i] = (kk < g.K && n < g.N) ? __ldg(wrow + n) : 0.f;
        }
      } else {
        // K-major weights only (per-batch "weights" such as K / V^T of attention)
        const int kk = k0 + bk;
        const int ldw = g.ldw ? g.ldw : g.taps * g.K;
        const float* wb = g.Wk + (long long)b * g.w_batch_stride + (long long)tap * g.K + kk;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int n = n0 + bn + i;
          Bs[bk][bn + i] = (kk < g.K && n < g.N) ? __ldg(wb + (long long)n * ldw) : 0.f;
        }
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < BK; ++k) {
        float a[4], w[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) a[i] = As[k][ty * 4 + i];
#pragma unroll
        for (int j = 0; j < 4; ++j) w[j] = Bs[k][tx * 4 + j];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], w[j], acc[i][j]);
      }
      __syncthreads();
    }
  }
  const int ldo = g.ldo ? g.ldo : g.N;
  const long long obs = g.out_batch_stride ? g.out_batch_stride : (long long)g.M * g.N;
  const long long valid = g.out_valid ? g.out_valid : (long long)g.M * ldo;
  const int biasN = g.biasN ? g.biasN : g.N;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= g.M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= g.N) continue;
      const long long flat = g.out_off + (long long)m * ldo + n;
      if (flat < 0 || flat >= valid) continue;
      float v = acc[i][j];
      if (g.bias) v += __ldg(g.bias + (n % biasN));
      v = apply_act(v, g.act);
      if (g.colscale) v *= __ldg(g.colscale + n);
      if (g.rowscale) v *= __ldg(g.rowscale + (long long)b * g.M + m);
      const long long o = (long long)b * obs + flat;
      if (g.res) v += g.res[o];
      if (g.accum) v += g.out[o];
      g.out[o] = v * g.scale;
    }
  }
}

__global__ void transpose_kernel(const float* in, float* out, int R, int Cc) {
  // in [B][R][Cc] -> out [B][Cc][R]
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const float* ib = in + (long long)b * R * Cc;
  float* ob = out + (long long)b * R * Cc;
  int c = blockIdx.x * 32 + threadIdx.x;
  for (int i = threadIdx.y; i < 32; i += 8) {
    int r = blockIdx.y * 32 + i;
    if (r < R && c < Cc) tile[i][threadIdx.x] = ib[(long long)r * Cc + c];
  }
  __syncthreads();
  int r = blockIdx.y * 32 + threadIdx.x;
  for (int i = threadIdx.y; i < 32; i += 8) {
    int cc = blockIdx.x * 32 + i;
    if (r < R && cc < Cc) ob[(long long)cc * R + r] = tile[threadIdx.x][i];
  }
}

}  // namespace


extern "C" int idx_set_option(idx_engine* e, const char* name, int value) {
  IDX_API_BEGIN
  IDX_CHECK(e && name, IDX_ERR_ARG, "null argument");
  const std::string n(name);
  if (n == "gemm_backend") {
    IDX_CHECK(value >= 0 && value <= 1, IDX_ERR_ARG, "gemm_backend: 0 = auto (wgmma tf32 where applicable), 1 = SIMT fp32");
    e->gemm_backend = value;       // per engine: another handle (another GPU, another thread) keeps its own
  } else if (n == "tail_f16") {
    IDX_CHECK(value >= 0 && value <= 1, IDX_ERR_ARG, "tail_f16: 1 = fp16 GEMM operands on the tensor-core path (default), 0 = tf32 over fp32 storage");
    e->tail_f16 = value;
  } else {
    throw IdxError(IDX_ERR_ARG, "unknown option: " + n);
  }
  IDX_API_END(e)
}

void conv_gemm(idx_engine* e, const ConvGemm& g) {
  IDX_CHECK((g.A || g.A16) && (g.out || g.out16) && g.M > 0 && g.N > 0 && g.K > 0, IDX_ERR_ARG, "conv_gemm: bad arguments");
  IDX_CHECK(g.epi == EPI_NONE || (g.A16 && g.Wk16), IDX_ERR_ARG, "conv_gemm: fused pair epilogues exist on the fp16 tensor-core path only");
  if (g.A16 && g.Wk16) {       // fp16 operands exist only for the tensor-core kernel
    IDX_CHECK(gemm_tc_supported(g), IDX_ERR_ARG, "conv_gemm: fp16 operands with a shape the tensor-core kernel does not take");
    gemm_tc_launch(e, g);
    return;
  }
  IDX_CHECK(g.A != nullptr, IDX_ERR_ARG, "conv_gemm: fp32 operand missing");
  if (e->force_backend == 2) {
    IDX_CHECK(g.Wk && !g.reflect, IDX_ERR_ARG, "conv_gemm: tensor-core path not applicable");
    gemm_tc_launch(e, g);
    return;
  }
  if (e->force_backend != 1 && !(e->force_backend == 0 && e->gemm_backend == 1) && g.Wk && gemm_tc_supported(g)) {
    gemm_tc_launch(e, g);
    return;
  }
  IDX_CHECK(g.W || g.Wk, IDX_ERR_ARG, "conv_gemm: weights missing");
  IDX_CHECK(g.W || true, IDX_ERR_ARG, "");
  dim3 grid((g.N + BN - 1) / BN, (g.M + BM - 1) / BM, g.B);
  conv_gemm_simt_kernel<<<grid, 256, 0, e->stream>>>(g);
  IDX_CUDA(cudaGetLastError());
  e->launches++;
}

void transpose_bct_to_btc(idx_engine* e, const float* in, float* out, int B, int C, int T) {
  dim3 grid((T + 31) / 32, (C + 31) / 32, B);
  transpose_kernel<<<grid, dim3(32, 8), 0, e->stream>>>(in, out, C, T);
  IDX_CUDA(cudaGetLastError());
  e->launches++;
}
void transpose_btc_to_bct(idx_engine* e, const float* in, float* out, int B, int T, int C) {
  dim3 grid((C + 31) / 32, (T + 31) / 32, B);
  transpose_kernel<<<grid, dim3(32, 8), 0, e->stream>>>(in, out, T, C);
  IDX_CUDA(cudaGetLastError());
  e->launches++;
}

// ------------------------------------------------------------------------ packed weights --
namespace {
__global__ void pack_conv_rows_kernel(const float* w, float* wsimt, float* wk, int Co, int Ci, int k, int row0) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long n = (long long)Co * Ci * k;
  if (i >= n) return;
  int kk = i % k;
  int ci = (i / k) % Ci;
  int co = i / ((long long)k * Ci);
  float v = w[(long long)row0 * Ci * k + i];
  wsimt[((long long)kk * Ci + ci) * Co + co] = v;
  wk[(long long)co * k * Ci + (long long)kk * Ci + ci] = v;
}
}  // namespace

float* WeightPool::alloc(size_t n) {
  float* p = nullptr;
  IDX_CUDA(cudaMalloc((void**)&p, n * sizeof(float)));
  owned.push_back(p);
  return p;
}
void WeightPool::release() {
  for (void* p : owned) cudaFree(p);
  owned.clear();
}

PackedW pack_conv1d(idx_engine* e, WeightPool& pool, const std::string& name, int dil, int row0, int rows) {
  const DevTensor& w = e->W(name + ".weight");
  IDX_CHECK(w.shape.size() == 3, IDX_ERR_ARG, name + ".weight must be [Co][Ci][k] (fold weight norm first)");
  PackedW p;
  const int Co = (int)w.shape[0];
  p.N = rows < 0 ? Co - row0 : rows;
  IDX_CHECK(row0 >= 0 && row0 + p.N <= Co, IDX_ERR_ARG, name + ": bad row range");
  p.K = (int)w.shape[1]; p.taps = (int)w.shape[2]; p.dil = dil;
  const size_t n = (size_t)p.N * p.K * p.taps;
  p.wsimt = pool.alloc(n);
  p.wk = pool.alloc(n);
  pack_conv_rows_kernel<<<(unsigned)((n + 255) / 256), 256, 0, e->stream>>>((const float*)w.d, p.wsimt, p.wk, p.N, p.K, p.taps, row0);
  IDX_CUDA(cudaGetLastError());
  if (e->has(name + ".bias")) p.bias = e->Wf(name + ".bias") + row0;
  return p;
}

PackedW pack_linear(idx_engine* e, WeightPool& pool, const std::string& name, int row0, int rows, bool with_bias) {
  const DevTensor& w = e->W(name + ".weight");
  IDX_CHECK(w.shape.size() == 2 || (w.shape.size() == 3 && w.shape[2] == 1), IDX_ERR_ARG, name + ".weight must be [N][K]");
  PackedW p;
  const int N = (int)w.shape[0];
  p.N = rows < 0 ? N - row0 : rows;
  IDX_CHECK(row0 >= 0 && row0 + p.N <= N, IDX_ERR_ARG, name + ": bad row range");
  p.K = (int)w.shape[1]; p.taps = 1;
  const size_t n = (size_t)p.N * p.K;
  p.wsimt = pool.alloc(n);
  p.wk = pool.alloc(n);
  pack_conv_rows_kernel<<<(unsigned)((n + 255) / 256), 256, 0, e->stream>>>((const float*)w.d, p.wsimt, p.wk, p.N, p.K, 1, row0);
  IDX_CUDA(cudaGetLastError());
  if (with_bias && e->has(name + ".bias")) p.bias = e->Wf(name + ".bias") + row0;
  return p;
}

ConvGemm gemm_of(const PackedW& w, const float* A, int B, int T, float* out) {
  ConvGemm g;
  g.A = A; g.B = B; g.Tin = T; g.K = w.K;
  g.W = w.wsimt; g.Wk = w.wk;
  g.taps = w.taps; g.dil = w.dil; g.pad = (w.taps * w.dil - w.dil) / 2;
  g.M = T; g.N = w.N; g.bias = w.bias; g.out = out;
  return g;
}

ConvGemm gemm_of16(const PackedW& w, const __half* A16, int B, int T, float* out) {
  ConvGemm g = gemm_of(w, nullptr, B, T, out);
  IDX_CHECK(w.wk16, IDX_ERR_STATE, "gemm_of16: the weight has no fp16 copy (pack_half)");
  g.A16 = A16; g.Wk16 = w.wk16;
  return g;
}

namespace {
__global__ void to_half_kernel(const float* __restrict__ x, __half* __restrict__ y, long long n) {
  pdl_wait();
  long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 2;
  if (i + 1 < n) *(__half2*)(y + i) = __floats2half2_rn(x[i], x[i + 1]);
  else if (i < n) y[i] = __float2half_rn(x[i]);
}
}  // namespace

void to_half(idx_engine* e, const float* x, __half* y, long long n) {
  if (n <= 0) return;
  launch_pdl(e, to_half_kernel, dim3((unsigned)((n / 2 + 256) / 256)), dim3(256), 0, x, y, n);
  e->launches++;
}

namespace {
__global__ void interleave_half_kernel(const float* __restrict__ wk, __half* __restrict__ dst, int N, long long KT) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)N * KT) return;
  const int r = (int)(i / KT);
  const long long k = i % KT;
  const int src = (r & 1) ? (N / 2 + (r >> 1)) : (r >> 1);
  dst[i] = __float2half_rn(wk[(long long)src * KT + k]);
}
__global__ void interleave_bias_kernel(const float* __restrict__ b, float* __restrict__ dst, int N) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < N) dst[r] = b[(r & 1) ? (N / 2 + (r >> 1)) : (r >> 1)];
}
}  // namespace

__half* pack_half_interleaved(idx_engine* e, WeightPool& pool, const PackedW& w, float** bias_out) {
  IDX_CHECK(w.wk && w.N % 2 == 0, IDX_ERR_ARG, "pack_half_interleaved: needs a K-major weight with an even row count");
  const long long KT = (long long)w.K * w.taps, n = (long long)w.N * KT;
  __half* dst = (__half*)pool.alloc((size_t)(n + 1) / 2 + 4);
  interleave_half_kernel<<<(unsigned)((n + 255) / 256), 256, 0, e->stream>>>(w.wk, dst, w.N, KT);
  IDX_CUDA(cudaGetLastError());
  if (bias_out) {
    *bias_out = nullptr;
    if (w.bias) {
      *bias_out = pool.alloc(w.N);
      interleave_bias_kernel<<<(w.N + 255) / 256, 256, 0, e->stream>>>(w.bias, *bias_out, w.N);
      IDX_CUDA(cudaGetLastError());
    }
  }
  return dst;
}

void pack_half(idx_engine* e, WeightPool& pool, PackedW& w) {
  if (w.wk16 || !w.wk) return;
  const size_t n = (size_t)w.N * w.K * w.taps;
  w.wk16 = (__half*)pool.alloc((n + 1) / 2 + 4);
  to_half(e, w.wk, w.wk16, (long long)n);
}

bool tail_half(const idx_engine* e) {
  return e->tail_f16 && e->gemm_backend == 0 && e->force_backend == 0;
}

namespace {
__global__ void kmajor_to_simt_kernel(const float* wk, float* ws, int N, int KT) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)N * KT) return;
  int n = (int)(i / KT), k = (int)(i % KT);
  ws[(long long)k * N + n] = wk[i];
}
}  // namespace

// Diagnostic entry (tests): run one multi-tap GEMM through a chosen back end, operand format and tile width
// (include/idxtts.h, idx_debug_gemm).  Every operand is staged into the arena; out / out16 travel with their guard bands.
extern "C" int idx_debug_conv_gemm(idx_engine* e, const idx_debug_gemm* d) {
  IDX_API_BEGIN
  IDX_CHECK(e && d && d->A && d->wk, IDX_ERR_ARG, "null argument");
  const bool fused = d->epi != EPI_NONE;
  IDX_CHECK(d->B > 0 && d->Tin > 0 && d->K > 0 && d->N > 0 && d->M > 0 && d->taps > 0, IDX_ERR_ARG, "idx_debug_conv_gemm: bad shape");
  IDX_CHECK(d->epi >= EPI_NONE && d->epi <= EPI_ROPE, IDX_ERR_ARG, "idx_debug_conv_gemm: unknown epi");
  IDX_CHECK(fused ? (d->out16 && d->operands == 1) : d->out != nullptr, IDX_ERR_ARG,
            "idx_debug_conv_gemm: epi 0 writes out; the fused epilogues write out16 and need fp16 operands");
  IDX_CHECK(d->operands == 0 || (d->operands == 1 && d->backend != 1), IDX_ERR_ARG,
            "idx_debug_conv_gemm: fp16 operands exist on the tensor-core path only");
  IDX_CHECK(d->tile_n == 0 || d->tile_n == 32 || d->tile_n == 64 || d->tile_n == 128, IDX_ERR_ARG,
            "idx_debug_conv_gemm: tile_n is 0, 32, 64 or 128");
  IDX_CHECK(d->guard >= 0 && d->guard % 8 == 0, IDX_ERR_ARG, "idx_debug_conv_gemm: guard must be a non-negative multiple of 8");
  IDX_CUDA(cudaSetDevice(e->device));
  const int B = d->B, M = d->M, N = d->N, KT = d->taps * d->K;
  const int lda = d->lda ? d->lda : d->K, ldw = d->ldw ? d->ldw : KT;
  IDX_CHECK(lda >= d->K && ldw >= KT, IDX_ERR_ARG, "idx_debug_conv_gemm: lda < K or ldw < taps*K");
  const size_t na = (size_t)(d->a_bcast ? 1 : B) * d->Tin * lda, nw = (size_t)(d->w_batched ? B : 1) * N * ldw;
  const size_t no = fused ? 0 : (size_t)B * d->out_elems_per_batch;
  const size_t no16 = d->epi == EPI_ROPE ? (size_t)B * M * N : (size_t)B * M * (N / 2);
  const int nbias = d->biasN ? d->biasN : N;
  size_t naux = 0;
  if (d->epi == EPI_ROPE) {
    IDX_CHECK(d->aux && d->heads > 0 && N == 3 * d->heads * 64, IDX_ERR_ARG, "idx_debug_conv_gemm: RoPE needs N = 3*heads*64 and a table");
    naux = (size_t)M * 64;
  } else if (d->epi == EPI_WNGATE) {
    IDX_CHECK(d->aux && d->aux_stride >= 0, IDX_ERR_ARG, "idx_debug_conv_gemm: the WaveNet gate needs g");
    naux = (size_t)(B - 1) * d->aux_stride + N;
  }
  if (d->epi == EPI_SWIGLU || d->epi == EPI_WNGATE)
    IDX_CHECK(!d->w_batched && ldw == KT, IDX_ERR_ARG, "idx_debug_conv_gemm: pair epilogues take one dense [N][taps*K] weight");
  const size_t g2 = 2 * (size_t)d->guard;
  // bytes: A fp32 + fp16, Wk fp32 + SIMT copy + fp16, out + res, out16, bias / aux / scales, alignment slack
  e->ensure_arena(6 * na + 10 * nw + 4 * (no + g2) + 4 * no + 2 * (no16 + g2) + 4 * (nbias + naux + (size_t)B * M + N) + (16 << 20));
  e->arena.reset();
  float* dA = e->arena.get<float>(na);
  float* dWk = e->arena.get<float>(nw);
  idx_to_device(e, dA, d->A, na * 4);
  idx_to_device(e, dWk, d->wk, nw * 4);
  auto stage = [&](const float* src, size_t n) -> float* {
    if (!src) return nullptr;
    float* p = e->arena.get<float>(n);
    idx_to_device(e, p, src, n * 4);
    return p;
  };
  float* dOut = nullptr;
  __half* dOut16 = nullptr;
  if (fused) {
    dOut16 = (__half*)e->arena.alloc((no16 + g2) * 2);
    idx_to_device(e, dOut16, d->out16 - d->guard, (no16 + g2) * 2);
  } else {
    dOut = stage(d->out - d->guard, no + g2);   // initial contents matter for accum / an in-place residual
  }
  const float* dRes = d->res_is_out ? (dOut ? dOut + d->guard : nullptr) : stage(d->res, no);
  const float* dBias = stage(d->bias, nbias);
  const float* dRow = stage(d->rowscale, (size_t)B * M);
  const float* dCol = stage(d->colscale, N);
  const float* dAux = stage(d->aux, naux);

  ConvGemm g;
  g.A = dA; g.B = B; g.Tin = d->Tin; g.K = d->K; g.lda = d->lda; g.a_bcast = d->a_bcast;
  g.Wk = dWk; g.ldw = d->ldw; g.w_batch_stride = d->w_batched ? (long long)N * ldw : 0;
  if (!d->w_batched && ldw == KT && !d->operands) {   // the SIMT kernel's [taps][K][N] copy
    float* dWs = e->arena.get<float>(nw);
    kmajor_to_simt_kernel<<<(unsigned)((nw + 255) / 256), 256, 0, e->stream>>>(dWk, dWs, N, KT);
    IDX_CUDA(cudaGetLastError());
    g.W = dWs;
  }
  g.taps = d->taps; g.dil = d->dil; g.pad = d->pad;
  g.M = M; g.N = N; g.bias = dBias; g.biasN = d->biasN; g.act = d->act; g.res = dRes; g.accum = d->accum;
  g.rowscale = dRow; g.colscale = dCol; g.scale = d->scale;
  g.out = dOut ? dOut + d->guard : nullptr;
  g.out_off = d->out_off; g.ldo = d->ldo; g.out_valid = d->out_valid; g.out_batch_stride = d->out_elems_per_batch;
  WeightPool pool;
  if (d->operands == 1) {      // fp16 operands on the tensor cores: round A and the K-major weights on the device
    __half* dA16 = (__half*)e->arena.alloc(na * 2);
    to_half(e, dA, dA16, (long long)na);
    g.A16 = dA16;
    if (d->epi == EPI_SWIGLU || d->epi == EPI_WNGATE) {
      PackedW w;
      w.wk = dWk; w.N = N; w.K = d->K; w.taps = d->taps; w.bias = dBias;
      float* bias_i = nullptr;
      g.Wk16 = pack_half_interleaved(e, pool, w, &bias_i);    // the pair layout the model's weights get at init
      g.bias = bias_i;
    } else {
      __half* dW16 = (__half*)e->arena.alloc(nw * 2);
      to_half(e, dWk, dW16, (long long)nw);
      g.Wk16 = dW16;
    }
    g.epi = d->epi;
    g.out16 = dOut16 ? dOut16 + d->guard : nullptr;
    g.aux = dAux;
    g.aux_stride = d->epi == EPI_ROPE ? d->heads : d->aux_stride;
    if (d->epi == EPI_ROPE && d->scale == 0.f) g.scale = FLASH_Q_SCALE;
  }
  DebugOverrides restore{e};
  e->force_backend = d->operands == 1 ? 0 : d->backend;
  e->force_tile_n = d->tile_n;
  conv_gemm(e, g);
  // timing loop (diagnostics): env IDX_GEMM_REPS=n repeats the launch between CUDA events
  static const int reps = getenv("IDX_GEMM_REPS") ? atoi(getenv("IDX_GEMM_REPS")) : 0;
  if (reps > 0) {
    cudaEvent_t a, b2;
    IDX_CUDA(cudaEventCreate(&a)); IDX_CUDA(cudaEventCreate(&b2));
    IDX_CUDA(cudaEventRecord(a, e->stream));
    for (int i = 0; i < reps; ++i) conv_gemm(e, g);
    IDX_CUDA(cudaEventRecord(b2, e->stream));
    IDX_CUDA(cudaEventSynchronize(b2));
    float ms = 0; IDX_CUDA(cudaEventElapsedTime(&ms, a, b2));
    fprintf(stderr, "[idx_debug_conv_gemm] backend %d operands %d B=%d M=%d N=%d K=%d taps=%d: %.2f us/launch, %.1f TFLOP/s\n",
            d->backend, d->operands, B, M, N, d->K, d->taps, ms * 1000.0 / reps,
            2.0 * B * M * (double)N * d->K * d->taps / (ms / reps * 1e-3) / 1e12);
    cudaEventDestroy(a); cudaEventDestroy(b2);
  }
  if (dOut) idx_from_device(e, d->out - d->guard, dOut, (no + g2) * 4);
  if (dOut16) idx_from_device(e, d->out16 - d->guard, dOut16, (no16 + g2) * 2);
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  pool.release();
  IDX_API_END(e)
}

// Diagnostic entry (tests): the wgmma flash attention on fp16 q / k / v [B*H][T][64] (include/idxtts.h).
extern "C" int idx_debug_flash_attention(idx_engine* e, const uint16_t* q16, const uint16_t* k16, const uint16_t* v16, int B,
                                         int T, int H, int kernel, long long guard, float* out, uint16_t* out16) {
  IDX_API_BEGIN
  IDX_CHECK(e && q16 && k16 && v16 && (out || out16), IDX_ERR_ARG, "null argument");
  IDX_CHECK(B > 0 && T > 0 && H > 0, IDX_ERR_ARG, "idx_debug_flash_attention: bad shape");
  IDX_CHECK(guard >= 0 && guard % 8 == 0, IDX_ERR_ARG, "idx_debug_flash_attention: guard must be a non-negative multiple of 8");
  IDX_CHECK(kernel == 0 || kernel == 2, IDX_ERR_ARG, "idx_debug_flash_attention: kernel is 0 or 2 (the wgmma flash attention)");
  IDX_CUDA(cudaSetDevice(e->device));
  const size_t n = (size_t)B * H * T * 64, ng = n + 2 * (size_t)guard;
  e->ensure_arena(3 * 2 * n + 6 * ng + (16 << 20));
  e->arena.reset();
  __half* dq = (__half*)e->arena.alloc(2 * n);
  __half* dk = (__half*)e->arena.alloc(2 * n);
  __half* dv = (__half*)e->arena.alloc(2 * n);
  idx_to_device(e, dq, q16, 2 * n);
  idx_to_device(e, dk, k16, 2 * n);
  idx_to_device(e, dv, v16, 2 * n);
  float* dOut = out ? e->arena.get<float>(ng) : nullptr;
  __half* dOut16 = out16 ? (__half*)e->arena.alloc(2 * ng) : nullptr;
  if (dOut) idx_to_device(e, dOut, out - guard, 4 * ng);
  if (dOut16) idx_to_device(e, dOut16, out16 - guard, 2 * ng);
  flash_attention_wgmma(e, dq, dk, dv, dOut ? dOut + guard : nullptr, dOut16 ? dOut16 + guard : nullptr, B, T, H);
  if (dOut) idx_from_device(e, out - guard, dOut, 4 * ng);
  if (dOut16) idx_from_device(e, out16 - guard, dOut16, 2 * ng);
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  IDX_API_END(e)
}

// Diagnostic entry (tests): the varlen wgmma flash attention on packed fp16 q / k / v [B*H][T][64] (include/idxtts.h).
extern "C" int idx_debug_flash_attention_varlen(idx_engine* e, const uint16_t* q16, const uint16_t* k16, const uint16_t* v16,
                                                int B, int H, const int32_t* seg_off, int n_seg, long long guard, float* out,
                                                uint16_t* out16) {
  IDX_API_BEGIN
  IDX_CHECK(e && q16 && k16 && v16 && seg_off && (out || out16), IDX_ERR_ARG, "null argument");
  IDX_CHECK(B > 0 && H > 0 && n_seg > 0 && seg_off[0] == 0, IDX_ERR_ARG, "idx_debug_flash_attention_varlen: bad shape");
  Segments sg;
  sg.off.assign(seg_off, seg_off + n_seg + 1);
  for (int u = 0; u < n_seg; ++u)
    IDX_CHECK(sg.off[u + 1] > sg.off[u], IDX_ERR_ARG, "idx_debug_flash_attention_varlen: segment offsets must increase");
  IDX_CHECK(guard >= 0 && guard % 8 == 0, IDX_ERR_ARG, "idx_debug_flash_attention_varlen: guard must be a non-negative multiple of 8");
  IDX_CUDA(cudaSetDevice(e->device));
  const int T = sg.total();
  const size_t n = (size_t)B * H * T * 64, ng = n + 2 * (size_t)guard;
  e->ensure_arena(3 * 2 * n + 6 * ng + 16 * (size_t)(n_seg + T / 128 + 2) + (16 << 20));
  e->arena.reset();
  __half* dq = (__half*)e->arena.alloc(2 * n);
  __half* dk = (__half*)e->arena.alloc(2 * n);
  __half* dv = (__half*)e->arena.alloc(2 * n);
  idx_to_device(e, dq, q16, 2 * n);
  idx_to_device(e, dk, k16, 2 * n);
  idx_to_device(e, dv, v16, 2 * n);
  float* dOut = out ? e->arena.get<float>(ng) : nullptr;
  __half* dOut16 = out16 ? (__half*)e->arena.alloc(2 * ng) : nullptr;
  if (dOut) idx_to_device(e, dOut, out - guard, 4 * ng);
  if (dOut16) idx_to_device(e, dOut16, out16 - guard, 2 * ng);
  segments_upload(e, sg);
  flash_attention_wgmma_varlen(e, dq, dk, dv, dOut ? dOut + guard : nullptr, dOut16 ? dOut16 + guard : nullptr, B, H, sg);
  if (dOut) idx_from_device(e, out - guard, dOut, 4 * ng);
  if (dOut16) idx_from_device(e, out16 - guard, dOut16, 2 * ng);
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  IDX_API_END(e)
}

// Diagnostic entry (tests): one of the tail's non-GEMM kernels through the host function the model calls
// (include/idxtts.h, idx_debug_tail).  Row-indexed inputs sit between NaN guard rows; outputs travel with their guard bands.
extern "C" int idx_debug_tail_op(idx_engine* e, const idx_debug_tail* d) {
  IDX_API_BEGIN
  IDX_CHECK(e && d, IDX_ERR_ARG, "null argument");
  IDX_CHECK(d->op >= 0 && d->op <= 12, IDX_ERR_ARG, "idx_debug_tail_op: unknown op");
  IDX_CHECK(d->B > 0 && d->T > 0 && d->C > 0, IDX_ERR_ARG, "idx_debug_tail_op: bad shape");
  IDX_CHECK(d->out || d->out16, IDX_ERR_ARG, "idx_debug_tail_op: no output");
  IDX_CHECK(d->guard >= 0 && d->guard % 8 == 0, IDX_ERR_ARG, "idx_debug_tail_op: guard must be a non-negative multiple of 8");
  IDX_CUDA(cudaSetDevice(e->device));
  const int op = d->op, B = d->B, T = d->T, C = d->C;
  Segments sg;
  if (op == 6 || op == 7 || (op == 10 && d->n_seg > 0)) {
    IDX_CHECK(d->seg_off && d->n_seg > 0 && d->seg_off[0] == 0, IDX_ERR_ARG, "idx_debug_tail_op: bad segment table");
    sg.off.assign(d->seg_off, d->seg_off + d->n_seg + 1);
    for (int u = 0; u < d->n_seg; ++u)
      IDX_CHECK(sg.off[u + 1] > sg.off[u], IDX_ERR_ARG, "idx_debug_tail_op: segment offsets must increase");
    IDX_CHECK(op == 7 || sg.total() == T, IDX_ERR_ARG, "idx_debug_tail_op: T must be the packed length");
  }
  // rows of x / x16 and of the output
  long long xrows = (long long)B * T, orows = (long long)B * T;
  int ocols = C;
  switch (op) {
    case 4: orows = (long long)B * d->n2; break;
    case 5: orows = (long long)B * (T + d->left + d->right); break;
    case 6: orows = (long long)B * (T + (long long)sg.n() * (d->left + d->right)); break;
    case 7: xrows = (long long)B * (sg.total() + (long long)(sg.n() - 1) * d->gap); orows = (long long)B * sg.total(); break;
    case 10: ocols = d->n2; break;
    case 12: ocols = 1; break;
    default: break;
  }
  IDX_CHECK((op == 8 || op == 9 || op == 10) ? B == 1 : true, IDX_ERR_ARG, "idx_debug_tail_op: ops 8-10 take B = 1");
  IDX_CHECK(op == 7 ? d->x16 != nullptr : (op == 10 || d->x != nullptr), IDX_ERR_ARG, "idx_debug_tail_op: input missing");
  IDX_CHECK((op != 8 && op != 9) || (d->x2 && d->x3 && (op == 8 || d->zero_rows)), IDX_ERR_ARG, "idx_debug_tail_op: cfg_euler inputs missing");
  IDX_CHECK((op != 1 && op != 2 && op != 3 && op != 11 && op != 12) || d->w, IDX_ERR_ARG, "idx_debug_tail_op: weight missing");
  IDX_CHECK((op != 2 && op != 11) || d->b, IDX_ERR_ARG, "idx_debug_tail_op: second parameter vector missing");
  IDX_CHECK(!d->m0 == !d->m1 && d->mod_stride >= 0, IDX_ERR_ARG, "idx_debug_tail_op: modulation needs both vectors");
  const bool f16_out = op == 0 || op == 1 || op == 5 || op == 6 || op == 7 || op == 11;
  const bool f32_out = !(op == 6 || op == 7);
  IDX_CHECK(f16_out || !d->out16, IDX_ERR_ARG, "idx_debug_tail_op: this op has no fp16 output");
  IDX_CHECK(f32_out || !d->out, IDX_ERR_ARG, "idx_debug_tail_op: this op has no fp32 output");
  IDX_CHECK(op != 10 || (d->n2 > 0 && d->n2 % 2 == 0 && d->n2 <= 64), IDX_ERR_ARG, "idx_debug_tail_op: rope head dim");
  IDX_CHECK(op != 3 || d->n2 > 0, IDX_ERR_ARG, "idx_debug_tail_op: dwconv kernel size");
  IDX_CHECK(op != 4 || d->n2 > 0, IDX_ERR_ARG, "idx_debug_tail_op: nearest output length");

  constexpr int G = 8;                              // NaN guard rows on each side of a row-indexed input
  const size_t nx = (size_t)xrows * C, gx = (size_t)G * C, no = (size_t)orows * ocols, g2 = 2 * (size_t)d->guard;
  const size_t nmod = d->m0 ? (size_t)(B - 1) * d->mod_stride + C : 0;
  const size_t nw = op == 3 ? (size_t)C * d->n2 : (op == 12 ? 7 * (size_t)C : C);
  e->ensure_arena(3 * 4 * (nx + 2 * gx) + 2 * (nx + 2 * gx) + 6 * (no + g2) + 4 * (2 * nw + 2 * nmod + 4 * (size_t)C) +
                  (size_t)T + 16 * (size_t)(sg.off.size() + T / 128 + 2) + (16 << 20));
  e->arena.reset();
  auto stage_rows = [&](const void* src, size_t esz) -> void* {     // [G NaN rows][rows][G NaN rows]
    if (!src) return nullptr;
    char* p = (char*)e->arena.alloc((nx + 2 * gx) * esz);
    IDX_CUDA(cudaMemsetAsync(p, 0xFF, (nx + 2 * gx) * esz, e->stream));   // all-ones: NaN in fp32 and fp16
    idx_to_device(e, p + gx * esz, src, nx * esz);
    return p + gx * esz;
  };
  auto stage = [&](const void* src, size_t bytes) -> void* {
    if (!src) return nullptr;
    void* p = e->arena.alloc(bytes);
    idx_to_device(e, p, src, bytes);
    return p;
  };
  const float* dx = (const float*)stage_rows(op == 7 ? nullptr : d->x, 4);
  const __half* dx16 = (const __half*)stage_rows(op == 7 ? d->x16 : nullptr, 2);
  const float* dx2 = (const float*)stage_rows(d->x2, 4);
  const float* dx3 = (const float*)stage_rows(d->x3, 4);
  const float* dw = (const float*)stage(d->w, nw * 4);
  const float* db = (const float*)stage(d->b, (op == 12 ? 1 : C) * 4);
  const float* dm0 = (const float*)stage(d->m0, nmod * 4);
  const float* dm1 = (const float*)stage(d->m1, nmod * 4);
  const unsigned char* dz = (op == 9) ? (const unsigned char*)stage(d->zero_rows, (size_t)T) : nullptr;
  float* dOut = d->out ? e->arena.get<float>(no + g2) : nullptr;
  __half* dOut16 = d->out16 ? (__half*)e->arena.alloc((no + g2) * 2) : nullptr;
  if (dOut) idx_to_device(e, dOut, d->out - d->guard, (no + g2) * 4);
  if (dOut16) idx_to_device(e, dOut16, d->out16 - d->guard, (no + g2) * 2);
  float* y = dOut ? dOut + d->guard : nullptr;
  __half* y16 = dOut16 ? dOut16 + d->guard : nullptr;
  if (!sg.off.empty()) segments_upload(e, sg);
  switch (op) {
    case 0: layernorm(e, dx, y, B, T, C, dw, db, d->eps, dm0, dm1, d->mod_stride, y16); break;
    case 1: rmsnorm_adaln(e, dx, y, B, T, C, dw, dm0, dm1, d->mod_stride, d->eps, y16); break;
    case 2: groupnorm1_mish(e, dx, y, B, T, C, dw, db, d->eps); break;
    case 3: dwconv1d(e, dx, y, B, T, C, dw, db, d->n2); break;
    case 4: nearest_interp(e, dx, y, B, T, d->n2, C); break;
    case 5: reflect_pad_rows(e, dx, y, B, T, C, d->left, d->right, y16); break;
    case 6: reflect_pad_segments(e, dx, y16, B, C, d->left, d->right, sg); break;
    case 7: compact_segments16(e, dx16, y16, B, C, d->gap, sg); break;
    case 8:
    case 9:
      IDX_CUDA(cudaMemcpyAsync(y, dx, nx * 4, cudaMemcpyDeviceToDevice, e->stream));    // the state is updated in place
      if (op == 8) cfg_euler(e, y, dx2, dx3, d->dt, d->rate, T, C, d->P);
      else cfg_euler_rows(e, y, dx2, dx3, d->dt, d->rate, T, C, dz);
      break;
    case 10:
      if (sg.off.empty()) rope_table(e, y, T, d->n2);
      else rope_table_segments(e, y, sg, d->n2);
      break;
    case 11: {
      float* ea = e->arena.get<float>(C);
      float* ib = e->arena.get<float>(C);
      snake_params_dev(e, dw, db, ea, ib, C, d->logscale);
      snake_act_dev(e, ea, ib, C, dx, y, B, T, y16);
      break;
    }
    case 12: conv_post_dev(e, dx, dw, db, y, B, T, C, d->use_tanh); break;
  }
  if (dOut) idx_from_device(e, d->out - d->guard, dOut, (no + g2) * 4);
  if (dOut16) idx_from_device(e, d->out16 - d->guard, dOut16, (no + g2) * 2);
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  IDX_API_END(e)
}
