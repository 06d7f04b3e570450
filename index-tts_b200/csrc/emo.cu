// emo.cu — emotion-vector path of UnifiedVoice (SURVEY.md §8a row a7) on sm_90a, fp32/tf32.
//
// Replaces:
//   merge_emovec / get_emovec / get_emo_conditioning   indextts/gpt/model_v2.py:827-838,588-593
//   ConformerEncoder (conv2d2 front-end, rel-pos MHA, conv module, FFN)
//                                                      indextts/gpt/conformer_encoder.py:56-167,232-313,389-437
//                                                      gpt/conformer/subsampling.py:135-187, attention.py:189-312
//   PerceiverResampler (1 latent, GEGLU FF, RMSNorm)    indextts/gpt/perceiver.py:140-317
// The reference recomputes this for every text segment with identical inputs (trap P11); callers cache the
// result per (speaker, emotion, alpha), so it runs once per reference audio.  All GEMMs go through
// conv_gemm (wgmma tf32 where the shape allows); lengths follow the reference's all-valid mask (P10).
#include "ops.h"
#include <cmath>

namespace {

// Conv2d(1 -> C, k3, s2) + ReLU on x [T][F], written directly in the layout of
// x.transpose(1,2).view(b, t, c*f): y[t2][c*Fs + f2]      (subsampling.py:144-146,181-185)
__global__ void conv2d_sub2_relu_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                        const float* __restrict__ bias, float* __restrict__ y, int T, int F_,
                                        int T2, int Fs, int C) {
  const int t2 = blockIdx.y, c = blockIdx.z;
  const int f2 = blockIdx.x * blockDim.x + threadIdx.x;
  if (f2 >= Fs) return;
  float acc = bias[c];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) acc = fmaf(w[c * 9 + i * 3 + j], x[(long long)(2 * t2 + i) * F_ + 2 * f2 + j], acc);
  y[(long long)t2 * C * Fs + (long long)c * Fs + f2] = fmaxf(acc, 0.f);
}

__global__ void pos_table_kernel(float* pe, int T, int d) {
  // PositionalEncoding.pe (embedding.py:47-53): pe[:, 0::2] = sin(pos*div), pe[:, 1::2] = cos(pos*div)
  const int t = blockIdx.x;
  for (int i = threadIdx.x; i < d / 2; i += blockDim.x) {
    const float div = expf((float)(2 * i) * -(logf(10000.0f) / (float)d));
    pe[(long long)t * d + 2 * i] = sinf((float)t * div);
    pe[(long long)t * d + 2 * i + 1] = cosf((float)t * div);
  }
}

// A' [H][T][2dk] = [q+u | q+v], B' [H][T][2dk] = [k | p], Vt [H][dk][Tp]
__global__ void relpos_split_kernel(const float* __restrict__ qkv, const float* __restrict__ pp,
                                    const float* __restrict__ u, const float* __restrict__ v, float* __restrict__ Ap,
                                    float* __restrict__ Bp, float* __restrict__ Vt, int T, int Tp, int H, int dk) {
  const int t = blockIdx.x, h = blockIdx.y;
  const int od = H * dk;
  for (int i = threadIdx.x; i < dk; i += blockDim.x) {
    const float q = qkv[(long long)t * 3 * od + h * dk + i];
    const float k = qkv[(long long)t * 3 * od + od + h * dk + i];
    const float vv = qkv[(long long)t * 3 * od + 2 * od + h * dk + i];
    float* ap = Ap + ((long long)h * T + t) * 2 * dk;
    float* bp = Bp + ((long long)h * T + t) * 2 * dk;
    ap[i] = q + u[h * dk + i];
    ap[dk + i] = q + v[h * dk + i];
    bp[i] = k;
    bp[dk + i] = pp[(long long)t * od + h * dk + i];
    Vt[((long long)h * dk + i) * Tp + t] = vv;
  }
}
__global__ void glu_kernel(const float* __restrict__ x, float* __restrict__ y, long long rows, int C) {
  // F.glu(dim=channels): first half * sigmoid(second half)  (conformer_encoder.py:151-152)
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * C) return;
  const long long r = i / C;
  const int c = (int)(i % C);
  const float a = x[r * 2 * C + c], b = x[r * 2 * C + C + c];
  y[i] = a * (1.f / (1.f + expf(-b)));
}
__global__ void geglu_kernel(const float* __restrict__ x, float* __restrict__ y, int N) {
  // GEGLU: x, gate = chunk(2); gelu(gate) * x   (perceiver.py:197-200)
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const float a = x[i], g = x[N + i];
  y[i] = 0.5f * g * (1.f + erff(g * 0.70710678118654752f)) * a;
}
// single-query attention of the perceiver latent: one block per head
__global__ void latent_attn_kernel(const float* __restrict__ q, const float* __restrict__ kv, float* __restrict__ out,
                                   int n, int H, int dh) {
  extern __shared__ float sc[];
  const int h = blockIdx.x, inner = H * dh;
  q += (long long)blockIdx.y * inner;          // one latent per blockIdx.y (32 of them in the v1 prompt encoder)
  out += (long long)blockIdx.y * inner;
  const float scale = rsqrtf((float)dh);
  float lmax = -INFINITY;
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    float s = 0.f;
    for (int d = 0; d < dh; ++d) s = fmaf(q[h * dh + d], kv[(long long)j * 2 * inner + h * dh + d], s);
    s *= scale;
    sc[j] = s;
    lmax = fmaxf(lmax, s);
  }
  __shared__ float red[32];
  for (int o = 16; o > 0; o >>= 1) lmax = fmaxf(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = lmax;
  __syncthreads();
  float mx = -INFINITY;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) mx = fmaxf(mx, red[i]);
  __syncthreads();
  float lsum = 0.f;
  for (int j = threadIdx.x; j < n; j += blockDim.x) { const float p = expf(sc[j] - mx); sc[j] = p; lsum += p; }
  for (int o = 16; o > 0; o >>= 1) lsum += __shfl_xor_sync(0xffffffffu, lsum, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = lsum;
  __syncthreads();
  float sum = 0.f;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) sum += red[i];
  for (int d = threadIdx.x; d < dh; d += blockDim.x) {
    float a = 0.f;
    for (int j = 0; j < n; ++j) a = fmaf(sc[j], kv[(long long)j * 2 * inner + inner + h * dh + d], a);
    out[h * dh + d] = a / sum;
  }
}
__global__ void l2norm_scale_kernel(const float* __restrict__ x, const float* __restrict__ gamma, float* __restrict__ y,
                                    int d) {
  // RMSNorm of the perceiver: F.normalize(x, dim=-1) * sqrt(d) * gamma   (perceiver.py:166-176)
  __shared__ float red[32];
  float s = 0.f;
  for (int i = threadIdx.x; i < d; i += blockDim.x) s += x[i] * x[i];
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  float tot = 0.f;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) tot += red[i];
  const float inv = 1.f / fmaxf(sqrtf(tot), 1e-12f);
  for (int i = threadIdx.x; i < d; i += blockDim.x) y[i] = x[i] * inv * sqrtf((float)d) * gamma[i];
}
__global__ void lerp_kernel(const float* base, const float* emo, float alpha, float* out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = base[i] + alpha * (emo[i] - base[i]);   // model_v2.py:837
}

}  // namespace

struct EmoBlock {
  PackedW qkv, pos, out, w1, w2, pw1, pw2;
  const float *u, *v, *dw_w, *dw_b;
  const float *n_mha_w, *n_mha_b, *n_conv_w, *n_conv_b, *n_ff_w, *n_ff_b, *n_fin_w, *n_fin_b, *cn_w, *cn_b;
};
struct EmoPLayer { PackedW to_q, to_kv, to_out, ff0, ff2; };
struct EmoState {
  idx_emo_config cfg;
  WeightPool pool;
  const float *conv_w, *conv_b;
  PackedW embed_out, proj_ctx, emovec, emol;
  std::vector<EmoBlock> blocks;
  std::vector<EmoPLayer> pl;
  const float *after_w, *after_b, *latents, *gamma;
  int n_latents = 1;
  bool has_heads = true;        // emovec_layer / emo_layer (v2.5 emotion path); the v1 prompt encoder has none
};
static EmoState* g_emo_of(idx_engine* e);

#define KCHECK(e)                  \
  do {                             \
    IDX_CUDA(cudaGetLastError());  \
    (e)->launches++;               \
  } while (0)

static EmoState* g_emo_of(idx_engine* e) { return e->emo; }

void emo_destroy(EmoState* s) {
  if (!s) return;
  s->pool.release();
  delete s;
}

// stack q,k,v linears into one [3*od][od] packed weight
PackedW pack3(idx_engine* e, WeightPool& pool, const std::string& a, const std::string& b, const std::string& c) {
  const DevTensor& wa = e->W(a + ".weight");
  const int od = (int)wa.shape[0], K = (int)wa.shape[1];
  std::vector<float> h((size_t)3 * od * K), hb((size_t)3 * od);
  int r = 0;
  for (const std::string* n : {&a, &b, &c}) {
    IDX_CUDA(cudaMemcpy(h.data() + (size_t)r * od * K, e->W(*n + ".weight").d, (size_t)od * K * 4, cudaMemcpyDeviceToHost));
    IDX_CUDA(cudaMemcpy(hb.data() + (size_t)r * od, e->W(*n + ".bias").d, (size_t)od * 4, cudaMemcpyDeviceToHost));
    ++r;
  }
  const std::string tmp = "__emo_qkv_tmp__";
  int64_t sh[2] = {3 * od, K}, shb[1] = {3 * od};
  IDX_CHECK(idx_load_weight(e, (tmp + ".weight").c_str(), h.data(), IDX_F32, 2, sh) == 0, IDX_ERR_ARG, e->err);
  PackedW p = pack_linear(e, pool, tmp, 0, -1, false);
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  float* bias = pool.alloc(3 * od);
  IDX_CUDA(cudaMemcpy(bias, hb.data(), (size_t)3 * od * 4, cudaMemcpyHostToDevice));
  p.bias = bias;
  (void)shb;
  return p;
}

static size_t emo_arena_bytes(const EmoState* s, int T);
static void cond_encode_dev(idx_engine* e, EmoState* s, const float* d_x, int T, float* d_lat_out);

// conformer + perceiver from the tensors under E / Q; *slot owns the state
static void cond_build(idx_engine* e, const idx_emo_config* cfg, const std::string& E, const std::string& Q, int n_latents,
                       bool has_heads, EmoState** slot) {
  emo_destroy(*slot);
  *slot = nullptr;
  EmoState* s = new EmoState();
  *slot = s;
  s->cfg = *cfg;
  s->n_latents = n_latents;
  s->has_heads = has_heads;
  s->conv_w = e->Wf(E + "embed.conv.0.weight");
  s->conv_b = e->Wf(E + "embed.conv.0.bias");
  s->embed_out = pack_linear(e, s->pool, E + "embed.out.0");
  for (int i = 0; i < cfg->blocks; ++i) {
    const std::string p = E + "encoders." + std::to_string(i) + ".";
    EmoBlock b;
    b.qkv = pack3(e, s->pool, p + "self_attn.linear_q", p + "self_attn.linear_k", p + "self_attn.linear_v");
    b.pos = pack_linear(e, s->pool, p + "self_attn.linear_pos");
    b.out = pack_linear(e, s->pool, p + "self_attn.linear_out");
    b.u = e->Wf(p + "self_attn.pos_bias_u"); b.v = e->Wf(p + "self_attn.pos_bias_v");
    b.w1 = pack_linear(e, s->pool, p + "feed_forward.w_1");
    b.w2 = pack_linear(e, s->pool, p + "feed_forward.w_2");
    b.pw1 = pack_linear(e, s->pool, p + "conv_module.pointwise_conv1");
    b.pw2 = pack_linear(e, s->pool, p + "conv_module.pointwise_conv2");
    b.dw_w = e->Wf(p + "conv_module.depthwise_conv.weight"); b.dw_b = e->Wf(p + "conv_module.depthwise_conv.bias");
    b.cn_w = e->Wf(p + "conv_module.norm.weight"); b.cn_b = e->Wf(p + "conv_module.norm.bias");
    b.n_mha_w = e->Wf(p + "norm_mha.weight"); b.n_mha_b = e->Wf(p + "norm_mha.bias");
    b.n_conv_w = e->Wf(p + "norm_conv.weight"); b.n_conv_b = e->Wf(p + "norm_conv.bias");
    b.n_ff_w = e->Wf(p + "norm_ff.weight"); b.n_ff_b = e->Wf(p + "norm_ff.bias");
    b.n_fin_w = e->Wf(p + "norm_final.weight"); b.n_fin_b = e->Wf(p + "norm_final.bias");
    s->blocks.push_back(b);
  }
  s->after_w = e->Wf(E + "after_norm.weight"); s->after_b = e->Wf(E + "after_norm.bias");
  s->proj_ctx = pack_linear(e, s->pool, Q + "proj_context");
  s->latents = e->Wf(Q + "latents");
  IDX_CHECK((int)e->W(Q + "latents").numel() == n_latents * cfg->p_dim, IDX_ERR_ARG, Q + "latents: unexpected size");
  for (int i = 0; i < cfg->p_depth; ++i) {
    const std::string p = Q + "layers." + std::to_string(i) + ".";
    EmoPLayer l;
    l.to_q = pack_linear(e, s->pool, p + "0.to_q");
    l.to_kv = pack_linear(e, s->pool, p + "0.to_kv");
    l.to_out = pack_linear(e, s->pool, p + "0.to_out");
    l.ff0 = pack_linear(e, s->pool, p + "1.0");
    l.ff2 = pack_linear(e, s->pool, p + "1.2");
    s->pl.push_back(l);
  }
  s->gamma = e->Wf(Q + "norm.gamma");
  if (has_heads) {
    s->emovec = pack_linear(e, s->pool, "gpt.emovec_layer");
    s->emol = pack_linear(e, s->pool, "gpt.emo_layer");
  }
  IDX_CUDA(cudaStreamSynchronize(e->stream));
}

extern "C" int idx_emo_init(idx_engine* e, const idx_emo_config* cfg) {
  IDX_API_BEGIN
  IDX_CHECK(e && cfg, IDX_ERR_ARG, "null argument");
  IDX_CUDA(cudaSetDevice(e->device));
  cond_build(e, cfg, "gpt.emo_conditioning_encoder.", "gpt.emo_perceiver_encoder.", 1, true, &e->emo);
  IDX_API_END(e)
}

// ---- v1 / v1.5 prompt encoder (gpt/model.py:352-363, get_conditioning :493-503): conformer over the 100-bin mel +
// perceiver with 32 latents -> conds [32][model_dim] that open the GPT prompt
extern "C" int idx_v1_cond_init(idx_engine* e, const idx_emo_config* cfg, int n_latents) {
  IDX_API_BEGIN
  IDX_CHECK(e && cfg && n_latents >= 1 && n_latents <= 64, IDX_ERR_ARG, "bad arguments");
  IDX_CHECK(cfg->p_dim == cfg->model_dim, IDX_ERR_ARG, "the v1 perceiver works at model_dim");
  IDX_CUDA(cudaSetDevice(e->device));
  cond_build(e, cfg, "gpt.conditioning_encoder.", "gpt.perceiver_encoder.", n_latents, false, &e->v1cond);
  IDX_API_END(e)
}

extern "C" int idx_v1_get_conditioning(idx_engine* e, const float* mel, int T, float* conds_out) {
  IDX_API_BEGIN
  EmoState* s = e ? e->v1cond : nullptr;
  IDX_CHECK(s, IDX_ERR_STATE, "idx_v1_cond_init has not been called");
  IDX_CHECK(mel && conds_out && T >= 3, IDX_ERR_ARG, "bad arguments");
  IDX_CUDA(cudaSetDevice(e->device));
  const idx_emo_config& c = s->cfg;
  e->ensure_arena(emo_arena_bytes(s, T) + 4 * ((size_t)T * c.idim + (size_t)s->n_latents * c.p_dim) + (1 << 16));
  e->arena.reset();
  float* d_x = e->arena.get<float>((size_t)T * c.idim);
  float* d_o = e->arena.get<float>((size_t)s->n_latents * c.p_dim);
  idx_to_device(e, d_x, mel, (size_t)T * c.idim * 4);
  cond_encode_dev(e, s, d_x, T, d_o);
  idx_from_device(e, conds_out, d_o, (size_t)s->n_latents * c.p_dim * 4);
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  IDX_API_END(e)
}

// feats (device [T][idim]) -> normalised perceiver latents (device [n_latents][p_dim])
static void cond_encode_dev(idx_engine* e, EmoState* s, const float* d_x, int T, float* d_lat_out) {
  const idx_emo_config& c = s->cfg;
  const int od = c.odim, H = c.heads, dk = od / H;
  const int T2 = (T - 3) / 2 + 1, Fs = (c.idim - 3) / 2 + 1;
  IDX_CHECK(T >= 3 && T2 >= 1, IDX_ERR_ARG, "emotion features too short");
  const int Tp = (T2 + 3) & ~3;
  float* sub = e->arena.get<float>((size_t)T2 * od * Fs);
  float* y = e->arena.get<float>((size_t)T2 * od);
  float* hbuf = e->arena.get<float>((size_t)T2 * od);
  float* big = e->arena.get<float>((size_t)T2 * std::max(3 * od, std::max(2 * od, c.linear_units)));
  float* pe = e->arena.get<float>((size_t)T2 * od);
  float* pp = e->arena.get<float>((size_t)T2 * od);
  float* Ap = e->arena.get<float>((size_t)H * T2 * 2 * dk);
  float* Bp = e->arena.get<float>((size_t)H * T2 * 2 * dk);
  float* Vt = e->arena.get<float>((size_t)H * dk * Tp);
  float* S = e->arena.get<float>((size_t)H * T2 * Tp);
  float* O = e->arena.get<float>((size_t)H * T2 * dk);
  float* att = e->arena.get<float>((size_t)T2 * od);
  conv2d_sub2_relu_kernel<<<dim3((Fs + 127) / 128, T2, od), 128, 0, e->stream>>>(d_x, s->conv_w, s->conv_b, sub, T, c.idim, T2, Fs, od);
  KCHECK(e);
  {
    ConvGemm g = gemm_of(s->embed_out, sub, 1, T2, y);
    g.scale = sqrtf((float)od);                       // x * xscale (embedding.py:139)
    conv_gemm(e, g);
  }
  pos_table_kernel<<<T2, 128, 0, e->stream>>>(pe, T2, od);
  KCHECK(e);
  fill_zero(e, Vt, (long long)H * dk * Tp);
  for (auto& b : s->blocks) {
    layernorm(e, y, hbuf, 1, T2, od, b.n_mha_w, b.n_mha_b, 1e-5f, nullptr, nullptr, 0);
    conv_gemm(e, gemm_of(b.qkv, hbuf, 1, T2, big));
    conv_gemm(e, gemm_of(b.pos, pe, 1, T2, pp));
    relpos_split_kernel<<<dim3(T2, H), 128, 0, e->stream>>>(big, pp, b.u, b.v, Ap, Bp, Vt, T2, Tp, H, dk);
    KCHECK(e);
    ConvGemm g1;
    g1.A = Ap; g1.B = H; g1.Tin = T2; g1.K = 2 * dk; g1.Wk = Bp; g1.w_batch_stride = (long long)T2 * 2 * dk;
    g1.M = T2; g1.N = T2; g1.out = S; g1.ldo = Tp; g1.out_batch_stride = (long long)T2 * Tp;
    g1.scale = 1.0f / sqrtf((float)dk);               // (ac + bd) / sqrt(d_k)  (attention.py:307-308)
    conv_gemm(e, g1);
    softmax_rows_exact(e, S, (long long)H * T2, T2, Tp);
    ConvGemm g2;
    g2.A = S; g2.B = H; g2.Tin = T2; g2.K = Tp; g2.Wk = Vt; g2.w_batch_stride = (long long)dk * Tp;
    g2.M = T2; g2.N = dk; g2.out = O;
    conv_gemm(e, g2);
    heads_merge(e, O, att, 1, T2, H, dk);
    { ConvGemm g = gemm_of(b.out, att, 1, T2, y); g.res = y; conv_gemm(e, g); }
    // convolution module (conformer_encoder.py:113-167)
    layernorm(e, y, hbuf, 1, T2, od, b.n_conv_w, b.n_conv_b, 1e-5f, nullptr, nullptr, 0);
    conv_gemm(e, gemm_of(b.pw1, hbuf, 1, T2, big));
    glu_kernel<<<(unsigned)(((long long)T2 * od + 255) / 256), 256, 0, e->stream>>>(big, hbuf, T2, od);
    KCHECK(e);
    dwconv1d(e, hbuf, att, 1, T2, od, b.dw_w, b.dw_b, c.cnn_kernel);
    layernorm(e, att, hbuf, 1, T2, od, b.cn_w, b.cn_b, 1e-5f, nullptr, nullptr, 0);
    silu_inplace(e, hbuf, (long long)T2 * od);
    { ConvGemm g = gemm_of(b.pw2, hbuf, 1, T2, y); g.res = y; conv_gemm(e, g); }
    // feed forward
    layernorm(e, y, hbuf, 1, T2, od, b.n_ff_w, b.n_ff_b, 1e-5f, nullptr, nullptr, 0);
    { ConvGemm g = gemm_of(b.w1, hbuf, 1, T2, big); g.act = ACT_SILU; conv_gemm(e, g); }
    { ConvGemm g = gemm_of(b.w2, big, 1, T2, y); g.res = y; conv_gemm(e, g); }
    layernorm(e, y, y, 1, T2, od, b.n_fin_w, b.n_fin_b, 1e-5f, nullptr, nullptr, 0);
  }
  layernorm(e, y, y, 1, T2, od, s->after_w, s->after_b, 1e-5f, nullptr, nullptr, 0);
  // perceiver resampler with one latent (perceiver.py:224-274)
  const int pd = c.p_dim, inner = c.p_heads * c.p_dim_head;
  const int di = (int)(pd * c.p_ff_mult * 2 / 3);
  const int nl = s->n_latents;
  float* ctx = e->arena.get<float>((size_t)(nl + T2) * pd);    // rows 0..nl-1 = the latents (cross_attn_include_queries)
  float* kv = e->arena.get<float>((size_t)(nl + T2) * 2 * inner);
  float* q = e->arena.get<float>((size_t)nl * inner);
  float* ao = e->arena.get<float>((size_t)nl * inner);
  float* ff = e->arena.get<float>((size_t)nl * 2 * di);
  float* fg = e->arena.get<float>((size_t)nl * di);
  float* lat = ctx;                                             // the latents live in the first rows of ctx
  conv_gemm(e, gemm_of(s->proj_ctx, y, 1, T2, ctx + (size_t)nl * pd));
  IDX_CUDA(cudaMemcpyAsync(lat, s->latents, (size_t)nl * pd * 4, cudaMemcpyDeviceToDevice, e->stream));
  for (auto& l : s->pl) {
    conv_gemm(e, gemm_of(l.to_q, lat, 1, nl, q));
    conv_gemm(e, gemm_of(l.to_kv, ctx, 1, nl + T2, kv));
    latent_attn_kernel<<<dim3(c.p_heads, nl), 128, (size_t)(nl + T2) * 4, e->stream>>>(q, kv, ao, nl + T2, c.p_heads, c.p_dim_head);
    KCHECK(e);
    { ConvGemm g = gemm_of(l.to_out, ao, 1, nl, lat); g.res = lat; conv_gemm(e, g); }
    conv_gemm(e, gemm_of(l.ff0, lat, 1, nl, ff));
    for (int r = 0; r < nl; ++r) {
      geglu_kernel<<<(di + 127) / 128, 128, 0, e->stream>>>(ff + (size_t)r * 2 * di, fg + (size_t)r * di, di);
      KCHECK(e);
    }
    { ConvGemm g = gemm_of(l.ff2, fg, 1, nl, lat); g.res = lat; conv_gemm(e, g); }
  }
  for (int r = 0; r < nl; ++r) {
    l2norm_scale_kernel<<<1, 256, 0, e->stream>>>(lat + (size_t)r * pd, s->gamma, d_lat_out + (size_t)r * pd, pd);
    KCHECK(e);
  }
}

// feats (device [T][idim]) -> emovec (device [model_dim])
static void emovec_dev(idx_engine* e, EmoState* s, const float* d_x, int T, float* d_out) {
  const idx_emo_config& c = s->cfg;
  float* ln = e->arena.get<float>(c.p_dim);
  float* ev = e->arena.get<float>(c.model_dim);
  cond_encode_dev(e, s, d_x, T, ln);
  conv_gemm(e, gemm_of(s->emovec, ln, 1, 1, ev));               // emovec_layer (model_v2.py:829)
  conv_gemm(e, gemm_of(s->emol, ev, 1, 1, d_out));              // emo_layer    (model_v2.py:830)
}

static size_t emo_arena_bytes(const EmoState* s, int T) {
  const idx_emo_config& c = s->cfg;
  const size_t T2 = (size_t)((T - 3) / 2 + 1), Fs = (size_t)((c.idim - 3) / 2 + 1), Tp = (T2 + 3) & ~(size_t)3;
  const size_t od = c.odim, H = c.heads, dk = od / H;
  return 4 * (T2 * od * Fs + T2 * od * 6 + T2 * (size_t)std::max<int>(3 * od, c.linear_units) + H * T2 * 5 * dk + H * dk * Tp +
              H * T2 * Tp + ((size_t)s->n_latents + T2) * (size_t)(c.p_dim + 2 * c.p_heads * c.p_dim_head) + 8 * (size_t)s->n_latents * c.p_dim * c.p_ff_mult +
              4 * (size_t)s->n_latents * c.p_heads * c.p_dim_head +
              4 * (size_t)c.model_dim) + 64 * 256 + (1 << 20);
}

extern "C" int idx_merge_emovec(idx_engine* e, const float* spk_feats, int Ts, const float* emo_feats, int Te,
                                float alpha, float* emo_vec_out) {
  IDX_API_BEGIN
  EmoState* s = e ? g_emo_of(e) : nullptr;
  IDX_CHECK(s, IDX_ERR_STATE, "idx_emo_init has not been called");
  IDX_CHECK(spk_feats && emo_vec_out && Ts >= 3, IDX_ERR_ARG, "bad arguments");
  IDX_CUDA(cudaSetDevice(e->device));
  const idx_emo_config& c = s->cfg;
  const bool same = (emo_feats == nullptr) || (emo_feats == spk_feats && Te == Ts);
  const int Tm = std::max(Ts, same ? Ts : Te);
  e->ensure_arena(emo_arena_bytes(s, Tm) + 4 * (size_t)(Ts + (same ? 0 : Te)) * c.idim + 16 * (size_t)c.model_dim + (1 << 20));
  e->arena.reset();
  float* d_s = e->arena.get<float>((size_t)Ts * c.idim);
  float* d_e = same ? d_s : e->arena.get<float>((size_t)Te * c.idim);
  float* base = e->arena.get<float>(c.model_dim);
  float* emo = e->arena.get<float>(c.model_dim);
  float* out = e->arena.get<float>(c.model_dim);
  idx_to_device(e, d_s, spk_feats, (size_t)Ts * c.idim * 4);
  if (!same) idx_to_device(e, d_e, emo_feats, (size_t)Te * c.idim * 4);
  const size_t mark = e->arena.off;
  emovec_dev(e, s, d_s, Ts, base);
  if (same) {
    // identical inputs give identical vectors: base + alpha * (base - base) == base exactly
    IDX_CUDA(cudaMemcpyAsync(out, base, (size_t)c.model_dim * 4, cudaMemcpyDeviceToDevice, e->stream));
  } else {
    e->arena.off = mark;
    emovec_dev(e, s, d_e, Te, emo);
    lerp_kernel<<<(c.model_dim + 127) / 128, 128, 0, e->stream>>>(base, emo, alpha, out, c.model_dim);
    KCHECK(e);
  }
  idx_from_device(e, emo_vec_out, out, (size_t)c.model_dim * 4);
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  IDX_API_END(e)
}
