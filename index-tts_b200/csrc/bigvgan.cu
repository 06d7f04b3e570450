// bigvgan.cu — BigVGAN-v2 generator (22 kHz, 80 band, 256x) on sm_90a.
//
// Replaces (SURVEY.md §8a row a12):
//   BigVGAN.forward / AMPBlock1.forward   indextts/s2mel/modules/bigvgan/bigvgan.py:360-386,132-141
//   Activation1d = UpSample1d → SnakeBeta → DownSample1d
//       alias_free_activation/torch/act.py:8-30, resample.py:10-58, filter.py:30-101,
//       activations.py:104-119   (and the reference's own CUDA kernel K1/K2,
//       alias_free_activation/cuda/anti_alias_activation_cuda.cu:43-181)
//
// Layout: activations are channels-last fp32 [B][T][C] so that
//   * every Conv1d is a multi-tap GEMM with M = time, N = C_out, K = C_in (ops.h), zero padding
//     comes from the row bounds of the A operand (TMA out-of-bounds fill on the wgmma path);
//   * ConvTranspose1d(k = n*u, stride u, pad (k - u)/2) is the SAME n-tap GEMM with N = u*C_out (n = 2
//     in BigVGAN-v2; the v1.5 generator also has k = u, n = 1): output phase r of frame q lands at
//     flat offset (q*u + r - pad)*C_out + co, i.e. the GEMM's row q is a contiguous run of the
//     upsampled signal (shifted by -pad*C_out) — no scatter;
//   * the anti-aliased SnakeBeta is ONE fused kernel (2x FIR upsample → snake → FIR downsample)
//     that reads x once and writes once; threads map to channels (coalesced) and slide along
//     time with a 6-sample input window and a 12-sample activated window in registers.
#include "stages.h"
#include <cmath>
#include <cstring>

namespace {

struct Taps { float f[12]; };

// Fused Activation1d(SnakeBeta).  x,y: [B][T][C].  ea = exp(alpha), ib = 1/(exp(beta)+1e-9).
// u[2j]   = 2*sum_q x[clamp(j-3+q)] * f[11-2q]     (UpSample1d, resample.py:29-40)
// u[2j+1] = 2*sum_q x[clamp(j-2+q)] * f[10-2q]
// a[m]    = u[m] + ib * sin^2(u[m]*ea)             (activations.py:104-119)
// y[t]    = sum_k a[clamp(2t-5+k)] * f[k]          (DownSample1d / LowPassFilter1d, filter.py:93-101)
template <int TT>
__global__ void __launch_bounds__(256) snake_act_kernel(const float* __restrict__ x,
                                                        float* __restrict__ y,
                                                        const float* __restrict__ ea,
                                                        const float* __restrict__ ib, int T, int C,
                                                        int CB, Taps taps, __half* __restrict__ y16) {
  pdl_wait();
  const int b = blockIdx.z;
  const int lanes_t = 256 / CB;
  const int c = blockIdx.x * CB + threadIdx.x % CB;
  const int tl = threadIdx.x / CB;
  if (tl >= lanes_t || c >= C) return;
  const int t0 = (blockIdx.y * lanes_t + tl) * TT;
  if (t0 >= T) return;
  const float* xb = x + (long long)b * T * C + c;
  float* yb = y ? y + (long long)b * T * C + c : nullptr;
  __half* yh = y16 ? y16 + (long long)b * T * C + c : nullptr;
  const float eac = __ldg(ea + c), ibc = __ldg(ib + c);
  const float* f = taps.f;
  auto X = [&](int t) { return __ldg(xb + (long long)min(max(t, 0), T - 1) * C); };
  auto snake = [&](float u) {
    // sin with an explicit two-constant 2*pi reduction, then the SFU sine on |r| <= pi
    // (abs error ~5e-7, inside the 1e-5 Activation1d parity bound; the reference CUDA kernel
    // builds with --use_fast_math, anti_alias_activation_cuda.cu / load.py:48-79)
    const float x = u * eac;
    const float k = rintf(x * 0.15915494309189535f);
    float r = fmaf(k, -6.2831855f, x);
    r = fmaf(k, 1.7484555e-7f, r);
    const float s = __sinf(r);
    return u + ibc * s * s;
  };
  // activated sample a[m] for any m in [0, 2T): recomputed from x (used for the window warm-up)
  auto A_at = [&](int m) {
    const int j = m >> 1;
    float u = 0.f;
    if (m & 1) {
#pragma unroll
      for (int q = 0; q < 6; ++q) u += X(j - 2 + q) * f[10 - 2 * q];
    } else {
#pragma unroll
      for (int q = 0; q < 6; ++q) u += X(j - 3 + q) * f[11 - 2 * q];
    }
    return snake(2.f * u);
  };
  // a-window holds a[clamp(2t-5+k)], k = 0..11
  float aw[12];
#pragma unroll
  for (int k = 0; k < 12; ++k) aw[k] = A_at(min(max(2 * t0 - 5 + k, 0), 2 * T - 1));
  // x-window xw[i] = x[clamp(t+1+i)], i = 0..5 : inputs of a[2(t+1)+5], a[2(t+1)+6]
  float xw[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) xw[i] = X(t0 + 1 + i);
  const int tend = min(t0 + TT, T);
  for (int t = t0; t < tend; ++t) {
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < 12; ++k) acc = fmaf(aw[k], f[k], acc);
    if (yb) yb[(long long)t * C] = acc;
    if (yh) yh[(long long)t * C] = __float2half_rn(acc);     // operand of the following conv (fp16 tensor-core path)
    // slide: next window is a[clamp(2t-3+k)]
#pragma unroll
    for (int k = 0; k < 10; ++k) aw[k] = aw[k + 2];
    const int m1 = 2 * t + 7, m2 = 2 * t + 8;  // new samples (odd j = t+3 ; even j = t+4)
    if (m2 <= 2 * T - 1) {
      // both in range: u[2j+1] with j=t+3 uses x[t+1..t+6]; u[2j] with j=t+4 uses x[t+1..t+6]
      float uo = 0.f, ue = 0.f;
#pragma unroll
      for (int q = 0; q < 6; ++q) {
        uo = fmaf(xw[q], f[10 - 2 * q], uo);
        ue = fmaf(xw[q], f[11 - 2 * q], ue);
      }
      aw[10] = snake(2.f * uo);
      aw[11] = snake(2.f * ue);
    } else {
      aw[10] = A_at(min(m1, 2 * T - 1));
      aw[11] = A_at(min(m2, 2 * T - 1));
    }
#pragma unroll
    for (int i = 0; i < 5; ++i) xw[i] = xw[i + 1];
    xw[5] = X(t + 7);
  }
}

__global__ void exp_params_kernel(const float* alpha, const float* beta, float* ea, float* ib, int n,
                                  int logscale) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float a = alpha[i], b = beta[i];
  if (logscale) { a = expf(a); b = expf(b); }
  ea[i] = a;
  ib[i] = 1.0f / (b + 1e-9f);
}

// conv_post: Conv1d(C -> 1, k=7, pad 3, no bias unless given) + clamp / tanh.  x [B][T][C] -> y [B][T]
__global__ void conv_post_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                 const float* __restrict__ bias, float* __restrict__ y, int T, int C,
                                 int use_tanh) {
  const int b = blockIdx.y;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  const float* xb = x + (long long)b * T * C;
  float acc = bias ? bias[0] : 0.f;
  for (int k = 0; k < 7; ++k) {
    const int ts = t + k - 3;
    if (ts < 0 || ts >= T) continue;
    const float* xr = xb + (long long)ts * C;
    for (int c = 0; c < C; ++c) acc = fmaf(__ldg(xr + c), __ldg(w + k * C + c), acc);
  }
  y[(long long)b * T + t] = use_tanh ? tanhf(acc) : fminf(fmaxf(acc, -1.f), 1.f);
}

// weight re-layout kernels ------------------------------------------------------------
// Conv1d weight [Co][Ci][k]  ->  Wsimt [k][Ci][Co]  and  Wk [Co][k*Ci]
__global__ void pack_conv_kernel(const float* w, float* wsimt, float* wk, int Co, int Ci, int k) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long n = (long long)Co * Ci * k;
  if (i >= n) return;
  int kk = i % k;
  int ci = (i / k) % Ci;
  int co = i / ((long long)k * Ci);
  float v = w[i];
  wsimt[((long long)kk * Ci + ci) * Co + co] = v;
  wk[(long long)co * k * Ci + (long long)kk * Ci + ci] = v;
}
// ConvTranspose1d weight [Ci][Co][nt*u] -> nt-tap GEMM weights with N = u*Co:
//   tap t (x[q-t]) : W[ci][co][r + t*u]
//   Wsimt [nt][Ci][u*Co],  Wk [u*Co][nt*Ci]
__global__ void pack_convT_kernel(const float* w, float* wsimt, float* wk, int Ci, int Co, int u, int nt) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long n = (long long)Ci * Co * nt * u;
  if (i >= n) return;
  int kk = i % (nt * u);
  int co = (i / (nt * u)) % Co;
  int ci = i / ((long long)nt * u * Co);
  int tap = kk / u, r = kk % u;
  float v = w[i];
  int j = r * Co + co;
  wsimt[((long long)tap * Ci + ci) * ((long long)u * Co) + j] = v;
  wk[(long long)j * nt * Ci + (long long)tap * Ci + ci] = v;
}

}  // namespace

struct ConvW {
  float *wsimt = nullptr, *wk = nullptr;
  __half* wk16 = nullptr;      // fp16 copy of wk (resblock convs: their input is written as fp16 by the Snake kernel)
  const float* bias = nullptr;
  int Co = 0, Ci = 0, k = 0, dil = 1;
};
struct ActP {
  float *ea = nullptr, *ib = nullptr;
  int C = 0;
};

struct BigvganState {
  idx_bigvgan_config cfg;
  std::vector<void*> owned;
  ConvW conv_pre;
  std::vector<ConvW> ups;                 // [num_upsamples]
  std::vector<ConvW> convs1, convs2;      // [num_upsamples*num_kernels*3]
  std::vector<ActP> acts;                 // [num_upsamples*num_kernels*6]
  ActP act_post;
  float* conv_post_w = nullptr;           // [7][C]
  const float* conv_post_b = nullptr;
  Taps taps;
  int total_up = 1;
  double last_ms = 0;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
};

void bigvgan_destroy(BigvganState* s) {
  if (!s) return;
  for (void* p : s->owned) cudaFree(p);
  if (s->ev0) cudaEventDestroy(s->ev0);
  if (s->ev1) cudaEventDestroy(s->ev1);
  delete s;
}

static float* balloc(BigvganState* s, size_t n) {
  float* p = nullptr;
  IDX_CUDA(cudaMalloc((void**)&p, n * sizeof(float)));
  s->owned.push_back(p);
  return p;
}

static ConvW pack_conv(idx_engine* e, BigvganState* s, const std::string& name, int dil) {
  const DevTensor& w = e->W(name + ".weight");
  IDX_CHECK(w.shape.size() == 3, IDX_ERR_ARG, name + ".weight must be 3-D (weight norm must be folded)");
  ConvW c;
  c.Co = (int)w.shape[0]; c.Ci = (int)w.shape[1]; c.k = (int)w.shape[2]; c.dil = dil;
  size_t n = w.numel();
  c.wsimt = balloc(s, n);
  c.wk = balloc(s, n);
  pack_conv_kernel<<<(unsigned)((n + 255) / 256), 256, 0, e->stream>>>((const float*)w.d, c.wsimt, c.wk, c.Co, c.Ci, c.k);
  IDX_CUDA(cudaGetLastError());
  if (c.Ci % 8 == 0) {
    c.wk16 = (__half*)balloc(s, n / 2 + 4);
    to_half(e, c.wk, c.wk16, (long long)n);
  }
  c.bias = e->has(name + ".bias") ? e->Wf(name + ".bias") : nullptr;
  return c;
}

static ActP pack_act(idx_engine* e, BigvganState* s, const std::string& name, int logscale) {
  const DevTensor& a = e->W(name + ".act.alpha");
  const DevTensor& b = e->W(name + ".act.beta");
  ActP p;
  p.C = (int)a.numel();
  IDX_CHECK(b.numel() == a.numel(), IDX_ERR_ARG, name + ": alpha/beta size mismatch");
  p.ea = balloc(s, p.C);
  p.ib = balloc(s, p.C);
  exp_params_kernel<<<(p.C + 127) / 128, 128, 0, e->stream>>>((const float*)a.d, (const float*)b.d, p.ea, p.ib, p.C, logscale);
  IDX_CUDA(cudaGetLastError());
  return p;
}

// kaiser_sinc_filter1d(cutoff=0.25, half_width=0.3, kernel_size=12) — filter.py:30-70; used
// when the checkpoint does not carry the registered filter buffers.
static void kaiser_sinc_taps(float* out) {
  const int K = 12, half = 6;
  const double cutoff = 0.25, half_width = 0.3;
  const double delta_f = 4 * half_width;
  const double A = 2.285 * (half - 1) * M_PI * delta_f + 7.95;
  double beta = (A > 50.0) ? 0.1102 * (A - 8.7) : (A >= 21.0 ? 0.5842 * pow(A - 21, 0.4) + 0.07886 * (A - 21.0) : 0.0);
  auto i0 = [](double x) {
    double s = 1, t = 1;
    for (int k = 1; k < 64; ++k) { t *= (x / (2.0 * k)) * (x / (2.0 * k)); s += t; }
    return s;
  };
  double f[12], sum = 0;
  for (int n = 0; n < K; ++n) {
    double r = 2.0 * n / (K - 1) - 1.0;
    double win = i0(beta * sqrt(fmax(0.0, 1 - r * r))) / i0(beta);
    double t = (n - half) + 0.5;
    double xx = 2 * cutoff * t;
    double sinc = (xx == 0) ? 1.0 : sin(M_PI * xx) / (M_PI * xx);
    f[n] = 2 * cutoff * win * sinc;
    sum += f[n];
  }
  for (int n = 0; n < K; ++n) out[n] = (float)(f[n] / sum);
}

static void kaiser_sinc_taps(float* out);

// builds a generator from the registered tensors `prefix + conv_pre.weight`, ...; *slot owns it (freed on failure by the
// engine teardown, like every module state)
static void bigvgan_build(idx_engine* e, const idx_bigvgan_config* cfg, const std::string& P, BigvganState** slot) {
  if (*slot) { bigvgan_destroy(*slot); *slot = nullptr; }
  BigvganState* s = new BigvganState();
  *slot = s;
  s->cfg = *cfg;
  IDX_CHECK(cfg->num_upsamples >= 1 && cfg->num_upsamples <= 8 && cfg->num_kernels >= 1 && cfg->num_kernels <= 4, IDX_ERR_ARG, "bad bigvgan config");
  s->conv_pre = pack_conv(e, s, P + "conv_pre", 1);
  IDX_CHECK(s->conv_pre.k == 7 && s->conv_pre.Ci == cfg->num_mels && s->conv_pre.Co == cfg->upsample_initial_channel, IDX_ERR_ARG, "conv_pre shape");
  int ch = cfg->upsample_initial_channel;
  for (int i = 0; i < cfg->num_upsamples; ++i) {
    const int u = cfg->upsample_rates[i], k = cfg->upsample_kernel_sizes[i];
    IDX_CHECK(u >= 1 && k >= u && k % u == 0 && (k - u) % 2 == 0, IDX_ERR_ARG,
              "ConvTranspose1d kernel must be a multiple of its stride, with an even difference (padding (k - u) / 2)");
    const std::string name = P + "ups." + std::to_string(i) + ".0";
    const DevTensor& w = e->W(name + ".weight");
    IDX_CHECK(w.shape.size() == 3 && w.shape[0] == ch && w.shape[1] == ch / 2 && w.shape[2] == k, IDX_ERR_ARG, name + ".weight shape");
    ConvW c;
    c.Ci = ch; c.Co = ch / 2; c.k = k;
    size_t n = w.numel();
    c.wsimt = balloc(s, n);
    c.wk = balloc(s, n);
    pack_convT_kernel<<<(unsigned)((n + 255) / 256), 256, 0, e->stream>>>((const float*)w.d, c.wsimt, c.wk, c.Ci, c.Co, u, k / u);
    IDX_CUDA(cudaGetLastError());
    c.bias = e->has(name + ".bias") ? e->Wf(name + ".bias") : nullptr;
    s->ups.push_back(c);
    ch /= 2;
    for (int j = 0; j < cfg->num_kernels; ++j) {
      const int rb = i * cfg->num_kernels + j;
      const std::string rp = P + "resblocks." + std::to_string(rb) + ".";
      for (int m = 0; m < 3; ++m) {
        ConvW c1 = pack_conv(e, s, rp + "convs1." + std::to_string(m), cfg->resblock_dilations[j][m]);
        ConvW c2 = pack_conv(e, s, rp + "convs2." + std::to_string(m), 1);
        IDX_CHECK(c1.k == cfg->resblock_kernel_sizes[j] && c1.Co == ch && c1.Ci == ch && c2.k == c1.k, IDX_ERR_ARG, rp + " conv shape");
        s->convs1.push_back(c1);
        s->convs2.push_back(c2);
      }
      for (int q = 0; q < 6; ++q)
        s->acts.push_back(pack_act(e, s, rp + "activations." + std::to_string(q), cfg->snake_logscale));
    }
    s->total_up *= u;
  }
  s->act_post = pack_act(e, s, P + "activation_post", cfg->snake_logscale);
  {
    const DevTensor& w = e->W(P + "conv_post.weight");
    IDX_CHECK(w.shape.size() == 3 && w.shape[0] == 1 && w.shape[1] == ch && w.shape[2] == 7, IDX_ERR_ARG, "conv_post shape");
    // [1][C][7] -> [7][C]
    std::vector<float> h(w.numel()), t(w.numel());
    IDX_CUDA(cudaMemcpy(h.data(), w.d, w.numel() * 4, cudaMemcpyDeviceToHost));
    for (int c = 0; c < ch; ++c)
      for (int k = 0; k < 7; ++k) t[(size_t)k * ch + c] = h[(size_t)c * 7 + k];
    s->conv_post_w = balloc(s, w.numel());
    IDX_CUDA(cudaMemcpy(s->conv_post_w, t.data(), w.numel() * 4, cudaMemcpyHostToDevice));
    s->conv_post_b = (cfg->use_bias_at_final && e->has(P + "conv_post.bias")) ? e->Wf(P + "conv_post.bias") : nullptr;
  }
  // FIR taps: the registered buffer of the checkpoint if present (bit-identical to torch), else computed
  if (e->has(P + "activation_post.upsample.filter")) {
    const DevTensor& f = e->W(P + "activation_post.upsample.filter");
    IDX_CHECK(f.numel() == 12, IDX_ERR_ARG, "filter must have 12 taps");
    IDX_CUDA(cudaMemcpy(s->taps.f, f.d, 48, cudaMemcpyDeviceToHost));
  } else {
    kaiser_sinc_taps(s->taps.f);
  }
  IDX_CUDA(cudaEventCreate(&s->ev0));
  IDX_CUDA(cudaEventCreate(&s->ev1));
  IDX_CUDA(cudaStreamSynchronize(e->stream));
}

extern "C" int idx_bigvgan_init(idx_engine* e, const idx_bigvgan_config* cfg) {
  IDX_API_BEGIN
  IDX_CHECK(e && cfg, IDX_ERR_ARG, "null argument");
  IDX_CUDA(cudaSetDevice(e->device));
  bigvgan_build(e, cfg, "bigvgan.", &e->bigvgan);
  IDX_API_END(e)
}

static void run_act(idx_engine* e, const BigvganState* s, const ActP& a, const float* x, float* y, int B, int T, __half* y16 = nullptr) {
  const int C = a.C;
  const int CB = C >= 32 ? 32 : C;
  const int lanes_t = 256 / CB;
  constexpr int TT = 32;
  dim3 grid((C + CB - 1) / CB, (T + lanes_t * TT - 1) / (lanes_t * TT), B);
  launch_pdl(e, snake_act_kernel<TT>, grid, dim3(256), 0, x, y, (const float*)a.ea, (const float*)a.ib, T, C, CB, s->taps, y16);
  e->launches++;
}

void snake_params_dev(idx_engine* e, const float* alpha, const float* beta, float* ea, float* ib, int C, int logscale) {
  exp_params_kernel<<<(C + 127) / 128, 128, 0, e->stream>>>(alpha, beta, ea, ib, C, logscale);
  IDX_CUDA(cudaGetLastError());
  e->launches++;
}

void snake_act_dev(idx_engine* e, const float* ea, const float* ib, int C, const float* x, float* y, int B, int T, __half* y16) {
  BigvganState tmp;
  if (e->bigvgan) tmp.taps = e->bigvgan->taps; else kaiser_sinc_taps(tmp.taps.f);
  ActP a; a.ea = (float*)ea; a.ib = (float*)ib; a.C = C;
  run_act(e, &tmp, a, x, y, B, T, y16);
}

void conv_post_dev(idx_engine* e, const float* x, const float* w, const float* bias, float* y, int B, int T, int C, int use_tanh) {
  dim3 grid((T + 127) / 128, B);
  conv_post_kernel<<<grid, 128, 0, e->stream>>>(x, w, bias, y, T, C, use_tanh);
  IDX_CUDA(cudaGetLastError());
  e->launches++;
}

static void run_conv(idx_engine* e, const ConvW& c, const float* x, float* out, int B, int T, const float* res, int accum, float scale,
                     const __half* x16 = nullptr) {
  ConvGemm g;
  g.A = x; g.B = B; g.Tin = T; g.K = c.Ci;
  g.W = c.wsimt; g.Wk = c.wk;
  if (x16) { g.A16 = x16; g.Wk16 = c.wk16; }
  g.taps = c.k; g.dil = c.dil; g.pad = (c.k * c.dil - c.dil) / 2;  // get_padding, bigvgan/utils.py:57-58
  g.M = T; g.N = c.Co; g.bias = c.bias;
  g.res = res; g.accum = accum; g.scale = scale; g.out = out;
  conv_gemm(e, g);
}

static void run_convT(idx_engine* e, const ConvW& c, int u, const float* x, float* out, int B, int T) {
  // nt = k / u taps; rows q = 0..T+nt-2, tap t reads x[q-t] (zero outside 0..T-1)
  const int nt = c.k / u;
  ConvGemm g;
  g.A = x; g.B = B; g.Tin = T; g.K = c.Ci;
  g.W = c.wsimt; g.Wk = c.wk;
  g.taps = nt; g.dil = -1; g.pad = 0;
  g.M = T + nt - 1; g.N = u * c.Co; g.bias = c.bias; g.biasN = c.Co;
  const int pad = (c.k - u) / 2;
  g.out = out;
  g.ldo = u * c.Co;
  g.out_off = -(long long)pad * c.Co;
  g.out_valid = (long long)T * u * c.Co;
  g.out_batch_stride = (long long)T * u * c.Co;
  conv_gemm(e, g);
}

static size_t bigvgan_maxel(const BigvganState* s, int F) {
  const idx_bigvgan_config& cfg = s->cfg;
  size_t maxel = (size_t)F * cfg.upsample_initial_channel;
  int T = F, ch = cfg.upsample_initial_channel;
  for (int i = 0; i < cfg.num_upsamples; ++i) {
    T *= cfg.upsample_rates[i]; ch /= 2;
    maxel = std::max(maxel, (size_t)T * ch);
  }
  return maxel;
}
size_t bigvgan_arena_bytes(const BigvganState* s, int B, int F) {
  return 6 * (size_t)B * bigvgan_maxel(s, F) * 4 + 2 * (size_t)B * s->cfg.num_mels * F * 4 +
         (size_t)B * F * s->total_up * 4 + (1 << 20);
}
int bigvgan_total_up(const BigvganState* s) { return s->total_up; }
void bigvgan_set_ms(BigvganState* s, double ms) { s->last_ms = ms; }

// channels_last_in: d_mel is already [B][F][num_mels] (the v1 latents); pre_bias / up_bias[i]: per-call replacements of the
// conv_pre / ups[i] biases (the speaker conditioning of the v1 generator, BigVGAN/models.py:230-240, folded into biases)
static void bigvgan_forward_impl(idx_engine* e, BigvganState* s, const float* d_mel, int B, int F, float* d_wav,
                                 bool channels_last_in, const float* pre_bias, const float* const* up_bias) {
  const idx_bigvgan_config& cfg = s->cfg;
  const int nm = cfg.num_mels;
  const size_t bufel = (size_t)B * bigvgan_maxel(s, F);
  float* d_melT = e->arena.get<float>((size_t)B * nm * F);
  float* buf[6];
  for (int i = 0; i < 6; ++i) buf[i] = e->arena.get<float>(bufel);
  if (channels_last_in) IDX_CUDA(cudaMemcpyAsync(d_melT, d_mel, (size_t)B * nm * F * 4, cudaMemcpyDeviceToDevice, e->stream));
  else transpose_bct_to_btc(e, d_mel, d_melT, B, nm, F);
  // P: stage input, and — once the transposed conv has consumed it — the accumulator of the
  // resblock outputs (= next stage's input).  Q: the upsampled stage signal read by all blocks.
  float *P = buf[0], *Q = buf[1], *xb0 = buf[2], *xb1 = buf[3], *ta = buf[4], *tc = buf[5];
  // fp16 operand mode: the Snake outputs inside the resblocks exist only as fp16 (they are read by a conv and nothing else)
  const bool hf = tail_half(e);
  __half* ta16 = (__half*)ta;
  {
    ConvW pre = s->conv_pre;
    if (pre_bias) pre.bias = pre_bias;
    run_conv(e, pre, d_melT, P, B, F, nullptr, 0, 1.f);
  }
  int T = F;
  for (int i = 0; i < cfg.num_upsamples; ++i) {
    const int u = cfg.upsample_rates[i];
    float* xst = Q;
    float* xsum = P;
    {
      ConvW up = s->ups[i];
      if (up_bias && up_bias[i]) up.bias = up_bias[i];
      run_convT(e, up, u, P, xst, B, T);
    }
    T *= u;
    for (int j = 0; j < cfg.num_kernels; ++j) {
      const int rb = i * cfg.num_kernels + j;
      const float* xcur = xst;
      for (int m = 0; m < 3; ++m) {
        const ActP& a1 = s->acts[rb * 6 + 2 * m];
        const ActP& a2 = s->acts[rb * 6 + 2 * m + 1];
        const ConvW &c1 = s->convs1[rb * 3 + m], &c2 = s->convs2[rb * 3 + m];
        const bool h1 = hf && c1.wk16, h2 = hf && c2.wk16;
        run_act(e, s, a1, xcur, h1 ? nullptr : ta, B, T, h1 ? ta16 : nullptr);
        run_conv(e, c1, ta, tc, B, T, nullptr, 0, 1.f, h1 ? ta16 : nullptr);
        run_act(e, s, a2, tc, h2 ? nullptr : ta, B, T, h2 ? ta16 : nullptr);
        if (m < 2) {
          float* xo = (m == 0) ? xb0 : xb1;
          run_conv(e, c2, ta, xo, B, T, xcur, 0, 1.f, h2 ? ta16 : nullptr);  // x = xt + x
          xcur = xo;
        } else {
          // last conv of the block: xs (+)= xt + x ; the /num_kernels average is folded into the
          // last block's epilogue (bigvgan.py:368-376)
          const bool last = (j == cfg.num_kernels - 1);
          run_conv(e, c2, ta, xsum, B, T, xcur, j > 0, last ? 1.0f / cfg.num_kernels : 1.f, h2 ? ta16 : nullptr);
        }
      }
    }
  }
  // NOTE: accumulate-then-scale: (xs0 + xs1 + xs2)/3 computed as ((xs0 + xs1) + xs2) * (1/3)
  run_act(e, s, s->act_post, P, ta, B, T);
  conv_post_dev(e, ta, s->conv_post_w, s->conv_post_b, d_wav, B, T, s->act_post.C, cfg.use_tanh_at_final);
}

void bigvgan_forward_dev(idx_engine* e, BigvganState* s, const float* d_mel, int B, int F, float* d_wav) {
  bigvgan_forward_impl(e, s, d_mel, B, F, d_wav, false, nullptr, nullptr);
}

// ------------------------------------------------------------------ v1 / v1.5 vocoder (SURVEY section 8 row a13) --
// indextts/BigVGAN/models.py:129-249: ECAPA-TDNN(mel_ref) -> speaker embedding -> cond_layer / conds[i] (1x1 convs)
// added after conv_pre / ups[i]; GPT latents [T][gpt_dim] in, tanh(wav) out.
struct V1VocoderState {
  BigvganState* gen = nullptr;
  EcapaState* ecapa = nullptr;
  WeightPool pool;
  PackedW cond_layer;
  std::vector<PackedW> conds;
  int n_mels = 0, emb = 0, cond_each = 1;
};
void v1voc_destroy(V1VocoderState* s) {
  if (!s) return;
  if (s->gen) bigvgan_destroy(s->gen);
  ecapa_destroy(s->ecapa);
  s->pool.release();
  delete s;
}

extern "C" int idx_v1_vocoder_init(idx_engine* e, const idx_bigvgan_config* gen_cfg, int n_mels, int speaker_embedding_dim,
                                   int cond_in_each_up_layer) {
  IDX_API_BEGIN
  IDX_CHECK(e && gen_cfg && n_mels >= 1 && speaker_embedding_dim >= 1, IDX_ERR_ARG, "bad arguments");
  IDX_CUDA(cudaSetDevice(e->device));
  if (e->v1voc) { v1voc_destroy(e->v1voc); e->v1voc = nullptr; }
  V1VocoderState* s = new V1VocoderState();
  e->v1voc = s;
  s->n_mels = n_mels; s->emb = speaker_embedding_dim; s->cond_each = cond_in_each_up_layer;
  const std::string P = "bigvgan_v1.";
  idx_bigvgan_config cfg = *gen_cfg;       // num_mels = gpt_dim (the latent width), tanh at the end (models.py:247)
  cfg.use_tanh_at_final = 1;
  bigvgan_build(e, &cfg, P, &s->gen);
  s->ecapa = ecapa_build(e, P + "speaker_encoder.", n_mels, speaker_embedding_dim);
  s->cond_layer = pack_conv1d(e, s->pool, P + "cond_layer", 1);
  IDX_CHECK(s->cond_layer.K == speaker_embedding_dim && s->cond_layer.N == cfg.upsample_initial_channel, IDX_ERR_ARG, "cond_layer shape");
  if (cond_in_each_up_layer)
    for (int i = 0; i < cfg.num_upsamples; ++i) s->conds.push_back(pack_conv1d(e, s->pool, P + "conds." + std::to_string(i), 1));
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  IDX_API_END(e)
}

extern "C" int idx_v1_speaker_embedding(idx_engine* e, const float* mel_ref, int Tm, float* emb_out) {
  IDX_API_BEGIN
  IDX_CHECK(e && e->v1voc, IDX_ERR_STATE, "idx_v1_vocoder_init has not been called");
  IDX_CHECK(mel_ref && emb_out && Tm >= 5, IDX_ERR_ARG, "bad arguments (the reference mel needs at least 5 frames)");
  IDX_CUDA(cudaSetDevice(e->device));
  V1VocoderState* s = e->v1voc;
  e->ensure_arena(ecapa_arena_bytes(s->ecapa, Tm) + (size_t)Tm * s->n_mels * 4 + (1 << 16));
  e->arena.reset();
  float* d_mel = e->arena.get<float>((size_t)Tm * s->n_mels);
  float* d_emb = e->arena.get<float>(s->emb);
  idx_to_device(e, d_mel, mel_ref, (size_t)Tm * s->n_mels * 4);
  ecapa_forward_dev(e, s->ecapa, d_mel, Tm, d_emb);
  idx_from_device(e, emb_out, d_emb, (size_t)s->emb * 4);
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  IDX_API_END(e)
}

namespace {
__global__ void add_vec_kernel(const float* a, const float* b, float* y, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] = (a ? a[i] : 0.f) + b[i];
}
}  // namespace

extern "C" int idx_v1_vocode(idx_engine* e, const float* latent, int T, const float* mel_ref, int Tm, float* wav_out) {
  IDX_API_BEGIN
  IDX_CHECK(e && e->v1voc, IDX_ERR_STATE, "idx_v1_vocoder_init has not been called");
  IDX_CHECK(latent && mel_ref && wav_out && T >= 1 && Tm >= 5, IDX_ERR_ARG, "bad arguments");
  IDX_CUDA(cudaSetDevice(e->device));
  V1VocoderState* s = e->v1voc;
  BigvganState* g = s->gen;
  const idx_bigvgan_config& cfg = g->cfg;
  const int gd = cfg.num_mels, nup = cfg.num_upsamples;
  const size_t out_n = (size_t)T * g->total_up;
  e->ensure_arena(bigvgan_arena_bytes(g, 1, T) + ecapa_arena_bytes(s->ecapa, Tm) + (size_t)(Tm * s->n_mels + T * gd) * 4 +
                  16 * (size_t)cfg.upsample_initial_channel * 4 + (1 << 16));
  e->arena.reset();
  float* d_lat = e->arena.get<float>((size_t)T * gd);
  float* d_mel = e->arena.get<float>((size_t)Tm * s->n_mels);
  float* d_emb = e->arena.get<float>(s->emb);
  float* d_wav = e->arena.get<float>(out_n);
  float* d_bias = e->arena.get<float>(4 * (size_t)cfg.upsample_initial_channel);
  idx_to_device(e, d_lat, latent, (size_t)T * gd * 4);
  idx_to_device(e, d_mel, mel_ref, (size_t)Tm * s->n_mels * 4);
  IDX_CUDA(cudaEventRecord(g->ev0, e->stream));
  ecapa_forward_dev(e, s->ecapa, d_mel, Tm, d_emb);
  // speaker conditioning as bias vectors: bias' = bias + cond(spk)
  const float* up_bias[8] = {nullptr};
  float* bp = d_bias;
  float* pre_bias = bp;
  {
    const int C0 = cfg.upsample_initial_channel;
    conv_gemm(e, gemm_of(s->cond_layer, d_emb, 1, 1, bp));
    add_vec_kernel<<<(C0 + 127) / 128, 128, 0, e->stream>>>(g->conv_pre.bias, bp, bp, C0);
    IDX_CUDA(cudaGetLastError()); e->launches++;
    bp += C0;
    int ch = C0;
    for (int i = 0; i < nup && s->cond_each; ++i) {
      ch /= 2;
      conv_gemm(e, gemm_of(s->conds[i], d_emb, 1, 1, bp));
      add_vec_kernel<<<(ch + 127) / 128, 128, 0, e->stream>>>(g->ups[i].bias, bp, bp, ch);
      IDX_CUDA(cudaGetLastError()); e->launches++;
      up_bias[i] = bp;
      bp += ch;
    }
  }
  bigvgan_forward_impl(e, g, d_lat, 1, T, d_wav, true, pre_bias, up_bias);
  IDX_CUDA(cudaEventRecord(g->ev1, e->stream));
  idx_from_device(e, wav_out, d_wav, out_n * 4);
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  float ms = 0;
  IDX_CUDA(cudaEventElapsedTime(&ms, g->ev0, g->ev1));
  g->last_ms = ms;
  IDX_API_END(e)
}

extern "C" int idx_bigvgan_forward(idx_engine* e, const float* mel, int B, int F, float* wav) {
  IDX_API_BEGIN
  IDX_CHECK(e && e->bigvgan, IDX_ERR_STATE, "idx_bigvgan_init has not been called");
  IDX_CHECK(mel && wav && B >= 1 && F >= 1, IDX_ERR_ARG, "bad arguments");
  IDX_CUDA(cudaSetDevice(e->device));
  BigvganState* s = e->bigvgan;
  const int nm = s->cfg.num_mels;
  const size_t out_n = (size_t)B * F * s->total_up;
  e->ensure_arena(bigvgan_arena_bytes(s, B, F) + (size_t)B * nm * F * 4);
  e->arena.reset();
  float* d_mel = e->arena.get<float>((size_t)B * nm * F);
  float* d_wav = e->arena.get<float>(out_n);
  idx_to_device(e, d_mel, mel, (size_t)B * nm * F * 4);
  IDX_CUDA(cudaEventRecord(s->ev0, e->stream));
  bigvgan_forward_dev(e, s, d_mel, B, F, d_wav);
  IDX_CUDA(cudaEventRecord(s->ev1, e->stream));
  idx_from_device(e, wav, d_wav, out_n * 4);
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  float ms = 0;
  IDX_CUDA(cudaEventElapsedTime(&ms, s->ev0, s->ev1));
  s->last_ms = ms;
  IDX_API_END(e)
}

extern "C" int idx_bigvgan_last_ms(const idx_engine* e, double* ms) {
  if (!e || !e->bigvgan || !ms) return IDX_ERR_STATE;
  *ms = e->bigvgan->last_ms;
  return IDX_OK;
}

extern "C" int idx_antialias_snake(idx_engine* e, const float* x, const float* alpha, const float* beta,
                                   int B, int C, int T, int logscale, float* y) {
  IDX_API_BEGIN
  IDX_CHECK(e && x && alpha && beta && y && B >= 1 && C >= 1 && T >= 1, IDX_ERR_ARG, "bad arguments");
  IDX_CUDA(cudaSetDevice(e->device));
  const size_t n = (size_t)B * C * T;
  e->ensure_arena(3 * n * 4 + 4 * (size_t)C * 4 + (1 << 16));
  e->arena.reset();
  float* d_x = e->arena.get<float>(n);
  float* d_xt = e->arena.get<float>(n);
  float* d_yt = e->arena.get<float>(n);
  float* d_a = e->arena.get<float>(C);
  float* d_b = e->arena.get<float>(C);
  float* d_ea = e->arena.get<float>(C);
  float* d_ib = e->arena.get<float>(C);
  idx_to_device(e, d_x, x, n * 4);
  idx_to_device(e, d_a, alpha, (size_t)C * 4);
  idx_to_device(e, d_b, beta, (size_t)C * 4);
  snake_params_dev(e, d_a, d_b, d_ea, d_ib, C, logscale);
  transpose_bct_to_btc(e, d_x, d_xt, B, C, T);
  snake_act_dev(e, d_ea, d_ib, C, d_xt, d_yt, B, T, nullptr);
  transpose_btc_to_bct(e, d_yt, d_x, B, T, C);
  idx_from_device(e, y, d_x, n * 4);
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  IDX_API_END(e)
}
