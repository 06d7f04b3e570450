// ecapa.cu — ECAPA-TDNN speaker encoder of the IndexTTS v1 / v1.5 vocoder (SURVEY section 8 row a13).
//
// Replaces indextts/BigVGAN/ECAPA_TDNN.py:429-582 (ECAPA_TDNN.forward) for one full-length utterance:
//   TDNNBlock = Conv1d("same", reflect) -> ReLU -> BatchNorm1d(eval)            :79-128, nnet/CNN.py:411-470
//   SERes2NetBlock = tdnn1 -> Res2Net(8 slices) -> tdnn2 -> SE -> + residual      :131-242, :341-426
//   MFA tdnn over the concatenated block outputs, attentive statistics pooling
//   with global context, BatchNorm, 1x1 conv to the embedding                    :245-338, :543-582
// Activations are channels-last [T][C] fp32; every conv is a conv_gemm (ops.h) whose epilogue does the ReLU; the
// BatchNorm that follows the ReLU is a per-channel affine kernel.  The concatenation [x, mean, std] in front of the
// pooling attention is never materialised: the mean/std columns contribute a per-utterance bias vector.
#include "ops.h"
#include "stages.h"
#include <cmath>
#include <string>
#include <vector>

namespace {

__global__ void col_affine_kernel(float* x, int ld, const float* __restrict__ scale, const float* __restrict__ shift,
                                  long long rows, int C) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * C) return;
  const long long r = i / C;
  const int c = (int)(i % C);
  float* p = x + r * ld + c;
  *p = *p * scale[c] + shift[c];
}
__global__ void add_cols_kernel(const float* a, int lda, const float* b, int ldb, float* y, int ldy, long long rows, int C) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * C) return;
  const long long r = i / C;
  const int c = (int)(i % C);
  y[r * ldy + c] = a[r * lda + c] + b[r * ldb + c];
}
// per-channel mean (and optionally std = sqrt(clamp(E[(x-mean)^2], 1e-12))) over T rows; block (32, 8), 32 channels
__global__ void col_mean_std_kernel(const float* __restrict__ x, int ld, int T, int C, float* mean_out, float* std_out) {
  __shared__ float sh[8][33];
  const int c = blockIdx.x * 32 + threadIdx.x, ty = threadIdx.y;
  float s = 0.f;
  if (c < C)
    for (int t = ty; t < T; t += 8) s += x[(long long)t * ld + c];
  sh[ty][threadIdx.x] = s;
  __syncthreads();
  float m = 0.f;
  for (int q = 0; q < 8; ++q) m += sh[q][threadIdx.x];
  m /= (float)T;
  __syncthreads();
  if (std_out) {
    float v = 0.f;
    if (c < C)
      for (int t = ty; t < T; t += 8) { const float d = x[(long long)t * ld + c] - m; v += d * d; }
    sh[ty][threadIdx.x] = v;
    __syncthreads();
    float vs = 0.f;
    for (int q = 0; q < 8; ++q) vs += sh[q][threadIdx.x];
    if (ty == 0 && c < C) std_out[c] = sqrtf(fmaxf(vs / (float)T, 1e-12f));
  }
  if (ty == 0 && c < C) mean_out[c] = m;
}
// out[t][c] = s[c] * y[t][c] + res[t][c]   (SE scaling + residual of SERes2NetBlock)
__global__ void se_scale_res_kernel(const float* y, int ldy, const float* __restrict__ s, const float* res, int ldr,
                                    float* out, int ldo, long long rows, int C) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * C) return;
  const long long r = i / C;
  const int c = (int)(i % C);
  out[r * ldo + c] = s[c] * y[r * ldy + c] + res[r * ldr + c];
}
__global__ void sigmoid_kernel(float* x, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) x[i] = 1.f / (1.f + expf(-x[i]));
}
__global__ void tanh_kernel(float* x, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) x[i] = tanhf(x[i]);
}
// attentive statistics: per channel c, a = softmax_t(logit[t][c]); mean = sum a x; std = sqrt(clamp(sum a (x-mean)^2, 1e-12))
// out = [mean(C) | std(C)]; block (32, 8)
__global__ void asp_pool_kernel(const float* __restrict__ logit, const float* __restrict__ x, int T, int C, float* out) {
  __shared__ float sh[8][33];
  const int c = blockIdx.x * 32 + threadIdx.x, ty = threadIdx.y, tx = threadIdx.x;
  const bool on = c < C;
  float mx = -INFINITY;
  if (on) for (int t = ty; t < T; t += 8) mx = fmaxf(mx, logit[(long long)t * C + c]);
  sh[ty][tx] = mx;
  __syncthreads();
  mx = sh[0][tx];
  for (int q = 1; q < 8; ++q) mx = fmaxf(mx, sh[q][tx]);
  __syncthreads();
  float se = 0.f, sx = 0.f;
  if (on) for (int t = ty; t < T; t += 8) {
    const float p = expf(logit[(long long)t * C + c] - mx);
    se += p;
    sx += p * x[(long long)t * C + c];
  }
  sh[ty][tx] = se;
  __syncthreads();
  float tot = 0.f;
  for (int q = 0; q < 8; ++q) tot += sh[q][tx];
  __syncthreads();
  sh[ty][tx] = sx;
  __syncthreads();
  float mean = 0.f;
  for (int q = 0; q < 8; ++q) mean += sh[q][tx];
  mean /= tot;
  __syncthreads();
  float sv = 0.f;
  if (on) for (int t = ty; t < T; t += 8) {
    const float p = expf(logit[(long long)t * C + c] - mx);
    const float d = x[(long long)t * C + c] - mean;
    sv += p * d * d;
  }
  sh[ty][tx] = sv;
  __syncthreads();
  float var = 0.f;
  for (int q = 0; q < 8; ++q) var += sh[q][tx];
  if (ty == 0 && on) {
    out[c] = mean;
    out[C + c] = sqrtf(fmaxf(var / tot, 1e-12f));
  }
}

#define KCHK(e)                    \
  do {                             \
    IDX_CUDA(cudaGetLastError());  \
    (e)->launches++;               \
  } while (0)

}  // namespace

void ecapa_col_mean_std(idx_engine* e, const float* x, int ld, int T, int C, float* mean, float* std_out) {
  col_mean_std_kernel<<<(C + 31) / 32, dim3(32, 8), 0, e->stream>>>(x, ld, T, C, mean, std_out);
  KCHK(e);
}
void ecapa_asp_pool(idx_engine* e, const float* logit, const float* x, int T, int C, float* out) {
  asp_pool_kernel<<<(C + 31) / 32, dim3(32, 8), 0, e->stream>>>(logit, x, T, C, out);
  KCHK(e);
}

struct Tdnn {
  PackedW w;
  float *scale = nullptr, *shift = nullptr;   // BatchNorm(eval) after the ReLU
};
struct EcapaBlock {
  Tdnn tdnn1, tdnn2;
  std::vector<Tdnn> res2;     // scale - 1 slice convs
  PackedW se1, se2, shortcut;
  bool has_shortcut = false;
  int dil = 1;
};
struct EcapaState {
  WeightPool pool;
  int n_mels = 0, emb = 0, C = 512, Cm = 1536, scale = 8, att = 128;
  Tdnn first, mfa, asp_tdnn_x;          // asp_tdnn_x: the x columns of asp.tdnn (K = Cm); its BN lives here too
  PackedW asp_stats, asp_conv, fc;      // asp_stats: the [mean | std] columns of asp.tdnn as a [att][2 Cm] linear, no bias
  float *bn_scale = nullptr, *bn_shift = nullptr;   // asp_bn
  std::vector<EcapaBlock> blocks;
  std::vector<int> kernel_sizes, dilations;
};

static void bn_affine(idx_engine* e, WeightPool& pool, const std::string& name, int C, float** scale, float** shift) {
  std::vector<float> g(C), b(C), m(C), v(C), sc(C), sh(C);
  auto get = [&](const char* suf, std::vector<float>& dst) {
    const DevTensor& t = e->W(name + suf);
    IDX_CHECK((int)t.numel() == C, IDX_ERR_ARG, name + suf + ": bad size");
    IDX_CUDA(cudaMemcpy(dst.data(), t.d, (size_t)C * 4, cudaMemcpyDeviceToHost));
  };
  get(".weight", g); get(".bias", b); get(".running_mean", m); get(".running_var", v);
  for (int i = 0; i < C; ++i) {
    sc[i] = g[i] / std::sqrt(v[i] + 1e-5f);
    sh[i] = b[i] - m[i] * sc[i];
  }
  *scale = pool.alloc(C);
  *shift = pool.alloc(C);
  IDX_CUDA(cudaMemcpy(*scale, sc.data(), (size_t)C * 4, cudaMemcpyHostToDevice));
  IDX_CUDA(cudaMemcpy(*shift, sh.data(), (size_t)C * 4, cudaMemcpyHostToDevice));
}

static Tdnn pack_tdnn(idx_engine* e, EcapaState* s, const std::string& name, int dil) {
  Tdnn t;
  t.w = pack_conv1d(e, s->pool, name + ".conv.conv", dil);
  bn_affine(e, s->pool, name + ".norm.norm", t.w.N, &t.scale, &t.shift);
  return t;
}

// columns [k0, k1) of a [N][K][1] conv weight as an own [N][k1-k0] linear (temporary registry entry)
static PackedW pack_kslice(idx_engine* e, WeightPool& pool, const std::string& name, int k0, int k1, bool with_bias) {
  const DevTensor& w = e->W(name + ".weight");
  const int N = (int)w.shape[0], K = (int)w.shape[1];
  IDX_CHECK(w.shape.size() == 3 && w.shape[2] == 1 && k0 >= 0 && k1 <= K && k0 < k1, IDX_ERR_ARG, name + ": bad column slice");
  std::vector<float> h((size_t)N * K), sl((size_t)N * (k1 - k0));
  IDX_CUDA(cudaMemcpy(h.data(), w.d, h.size() * 4, cudaMemcpyDeviceToHost));
  for (int n = 0; n < N; ++n)
    for (int k = k0; k < k1; ++k) sl[(size_t)n * (k1 - k0) + (k - k0)] = h[(size_t)n * K + k];
  const std::string tmp = "__ecapa_slice_tmp__";
  int64_t sh[2] = {N, k1 - k0};
  IDX_CHECK(idx_load_weight(e, (tmp + ".weight").c_str(), sl.data(), IDX_F32, 2, sh) == 0, IDX_ERR_ARG, e->err);
  PackedW p = pack_linear(e, pool, tmp, 0, -1, false);
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  if (with_bias && e->has(name + ".bias")) p.bias = e->Wf(name + ".bias");
  return p;
}

EcapaState* ecapa_build(idx_engine* e, const std::string& prefix, int n_mels, int emb) {
  EcapaState* s = new EcapaState();
  s->n_mels = n_mels; s->emb = emb;
  s->kernel_sizes = {5, 3, 3, 3, 1};
  s->dilations = {1, 2, 3, 4, 1};
  const std::string q = prefix;
  s->first = pack_tdnn(e, s, q + "blocks.0", s->dilations[0]);
  IDX_CHECK(s->first.w.K == n_mels && s->first.w.N == s->C && s->first.w.taps == 5, IDX_ERR_ARG, "ECAPA blocks.0 shape");
  for (int i = 1; i <= 3; ++i) {
    const std::string p = q + "blocks." + std::to_string(i);
    EcapaBlock b;
    b.dil = s->dilations[i];
    b.tdnn1 = pack_tdnn(e, s, p + ".tdnn1", 1);
    for (int j = 0; j < s->scale - 1; ++j)
      b.res2.push_back(pack_tdnn(e, s, p + ".res2net_block.blocks." + std::to_string(j), b.dil));
    b.tdnn2 = pack_tdnn(e, s, p + ".tdnn2", 1);
    b.se1 = pack_conv1d(e, s->pool, p + ".se_block.conv1.conv", 1);
    b.se2 = pack_conv1d(e, s->pool, p + ".se_block.conv2.conv", 1);
    b.has_shortcut = e->has(p + ".shortcut.conv.weight");
    if (b.has_shortcut) b.shortcut = pack_conv1d(e, s->pool, p + ".shortcut.conv", 1);
    IDX_CHECK(b.tdnn1.w.N == s->C && b.res2[0].w.N == s->C / s->scale && b.res2[0].w.taps == 3, IDX_ERR_ARG, p + ": shape");
    s->blocks.push_back(b);
  }
  s->mfa = pack_tdnn(e, s, q + "mfa", 1);
  IDX_CHECK(s->mfa.w.K == 3 * s->C && s->mfa.w.N == s->Cm, IDX_ERR_ARG, "ECAPA mfa shape");
  // asp.tdnn over [x | mean | std]: x columns as the GEMM, the statistics columns as a per-utterance bias
  s->asp_tdnn_x.w = pack_kslice(e, s->pool, q + "asp.tdnn.conv.conv", 0, s->Cm, false);
  s->asp_stats = pack_kslice(e, s->pool, q + "asp.tdnn.conv.conv", s->Cm, 3 * s->Cm, true);
  bn_affine(e, s->pool, q + "asp.tdnn.norm.norm", s->att, &s->asp_tdnn_x.scale, &s->asp_tdnn_x.shift);
  s->asp_conv = pack_conv1d(e, s->pool, q + "asp.conv.conv", 1);
  bn_affine(e, s->pool, q + "asp_bn.norm", 2 * s->Cm, &s->bn_scale, &s->bn_shift);
  s->fc = pack_conv1d(e, s->pool, q + "fc.conv", 1);
  IDX_CHECK(s->fc.N == emb && s->fc.K == 2 * s->Cm, IDX_ERR_ARG, "ECAPA fc shape");
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  return s;
}

void ecapa_destroy(EcapaState* s) {
  if (!s) return;
  s->pool.release();
  delete s;
}

size_t ecapa_arena_bytes(const EcapaState* s, int T) {
  return 4 * ((size_t)T * (s->C * 3 + s->C * 3 + 3 * s->C + s->C / s->scale + 2 * s->Cm + s->att + s->n_mels) + 16 * (size_t)s->Cm) + (1 << 20);
}

// conv -> ReLU (GEMM epilogue) -> BatchNorm affine, reading columns of a wider matrix and writing a column slice
static void tdnn_run(idx_engine* e, const Tdnn& t, const float* in, int lda, int T, float* out, int ldo, int col0) {
  ConvGemm g = gemm_of(t.w, in, 1, T, out);
  g.lda = lda;
  g.reflect = t.w.taps > 1;           // speechbrain "same" padding with padding_mode="reflect" (nnet/CNN.py:458-470)
  g.act = ACT_RELU;
  g.ldo = ldo;
  g.out_off = col0;
  g.out_valid = (long long)T * ldo;
  conv_gemm(e, g);
  const long long n = (long long)T * t.w.N;
  col_affine_kernel<<<(unsigned)((n + 255) / 256), 256, 0, e->stream>>>(out + col0, ldo, t.scale, t.shift, T, t.w.N);
  KCHK(e);
}

// mel (device, [T][n_mels]) -> emb (device, [emb])
void ecapa_forward_dev(idx_engine* e, EcapaState* s, const float* d_mel, int T, float* d_emb) {
  const int C = s->C, Cm = s->Cm, W = C / s->scale;
  IDX_CHECK(T >= 5, IDX_ERR_ARG, "reference mel too short for the reflect-padded convolutions (needs > 4 frames)");
  float* x0 = e->arena.get<float>((size_t)T * C);
  float* cat = e->arena.get<float>((size_t)T * 3 * C);      // outputs of blocks 1..3 side by side (the MFA input)
  float* y = e->arena.get<float>((size_t)T * C);
  float* z = e->arena.get<float>((size_t)T * C);
  float* y2 = e->arena.get<float>((size_t)T * C);
  float* tmp = e->arena.get<float>((size_t)T * W);
  float* sv = e->arena.get<float>(5 * (size_t)Cm);
  tdnn_run(e, s->first, d_mel, s->n_mels, T, x0, C, 0);
  const float* xin = x0;
  int ldin = C;
  for (int i = 0; i < 3; ++i) {
    const EcapaBlock& b = s->blocks[i];
    IDX_CHECK(!b.has_shortcut, IDX_ERR_ARG, "ECAPA shortcut convs (in != out channels) are not wired");
    tdnn_run(e, b.tdnn1, xin, ldin, T, y, C, 0);
    // Res2Net (:179-191): slice 0 passes through, slice j >= 1 = tdnn(slice_j [+ previous output])
    copy_cols(e, y, C, z, C, 0, T, W);
    for (int j = 1; j < s->scale; ++j) {
      const float* src = y + j * W;
      int lds = C;
      if (j >= 2) {
        const long long n = (long long)T * W;
        add_cols_kernel<<<(unsigned)((n + 255) / 256), 256, 0, e->stream>>>(y + j * W, C, z + (j - 1) * W, C, tmp, W, T, W);
        KCHK(e);
        src = tmp; lds = W;
      }
      tdnn_run(e, b.res2[j - 1], src, lds, T, z, C, j * W);
    }
    tdnn_run(e, b.tdnn2, z, C, T, y2, C, 0);
    // SE (:228-242, full-length utterance): s = sigmoid(conv2(relu(conv1(mean_t y2))))
    float* mean = sv;
    float* h1 = sv + Cm;
    float* sc = sv + 2 * Cm;
    ecapa_col_mean_std(e, y2, C, T, C, mean, nullptr);
    { ConvGemm g = gemm_of(b.se1, mean, 1, 1, h1); g.act = ACT_RELU; conv_gemm(e, g); }
    conv_gemm(e, gemm_of(b.se2, h1, 1, 1, sc));
    sigmoid_kernel<<<(C + 127) / 128, 128, 0, e->stream>>>(sc, C);
    KCHK(e);
    const long long n = (long long)T * C;
    se_scale_res_kernel<<<(unsigned)((n + 255) / 256), 256, 0, e->stream>>>(y2, C, sc, xin, ldin, cat + i * C, 3 * C, T, C);
    KCHK(e);
    xin = cat + i * C;
    ldin = 3 * C;
  }
  float* xm = e->arena.get<float>((size_t)T * Cm);
  float* att = e->arena.get<float>((size_t)T * s->att);
  float* lg = e->arena.get<float>((size_t)T * Cm);
  tdnn_run(e, s->mfa, cat, 3 * C, T, xm, Cm, 0);
  // attentive statistics pooling with global context (:282-338)
  float* stats = sv;                 // [mean | std] of xm, uniform weights
  float* bvec = sv + 2 * Cm;         // W_stats . [mean | std] + bias  -> per-utterance bias of the attention TDNN
  float* pooled = sv + 2 * Cm + s->att;   // needs 2*Cm floats: sv holds 4*Cm
  ecapa_col_mean_std(e, xm, Cm, T, Cm, stats, stats + Cm);
  conv_gemm(e, gemm_of(s->asp_stats, stats, 1, 1, bvec));
  {
    ConvGemm g = gemm_of(s->asp_tdnn_x.w, xm, 1, T, att);
    g.bias = bvec;
    g.act = ACT_RELU;
    conv_gemm(e, g);
    const long long n = (long long)T * s->att;
    col_affine_kernel<<<(unsigned)((n + 255) / 256), 256, 0, e->stream>>>(att, s->att, s->asp_tdnn_x.scale, s->asp_tdnn_x.shift, T, s->att);
    KCHK(e);
    tanh_kernel<<<(unsigned)((n + 255) / 256), 256, 0, e->stream>>>(att, n);
    KCHK(e);
  }
  conv_gemm(e, gemm_of(s->asp_conv, att, 1, T, lg));
  ecapa_asp_pool(e, lg, xm, T, Cm, pooled);
  col_affine_kernel<<<(2 * Cm + 255) / 256, 256, 0, e->stream>>>(pooled, 2 * Cm, s->bn_scale, s->bn_shift, 1, 2 * Cm);
  KCHK(e);
  conv_gemm(e, gemm_of(s->fc, pooled, 1, 1, d_emb));
}
