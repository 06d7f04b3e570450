// s2mel.cu — semantic-codec decode → length regulator → flow-matching CFM (DiT + WaveNet) Euler
// solver of IndexTTS-2 / 2.5 on sm_90a, fp32 (the reference disables autocast here, P5).
//
// Replaces (SURVEY.md §8a rows a8–a11):
//   EnhancedCodec.decode               indextts/codec/models.py:205-231
//   InterpolateRegulator.forward       indextts/s2mel/modules/length_regulator.py:90-141
//   BASECFM.inference / solve_euler    indextts/s2mel/modules/flow_matching.py:30-115
//   DiT.forward                        indextts/s2mel/modules/diffusion_transformer.py:186-257
//   Transformer/Block/Attention/FFN    indextts/s2mel/modules/gpt_fast/model.py:121-360
//   WN                                 indextts/s2mel/modules/wavenet.py:103-166
//
// Structure exploited (none of it changes the arithmetic per element):
//   * everything that depends only on the timestep — the two TimestepEmbedder MLPs, all 27 adaLN
//     projections, the WaveNet cond_layer and the FinalLayer modulation — is evaluated ONCE for all
//     n_steps timesteps as a few M = n_steps GEMMs before the Euler loop;
//   * the time-invariant part of cond_x_merge_linear ([prompt | cond | style] columns) is folded
//     into a per-solve constant C0, so each step starts with a K = 80 GEMM;
//   * the cond / uncond CFG pair runs as batch 2 exactly like the reference (flow_matching.py:88-104).
#include "stages.h"
#include <algorithm>
#include <cmath>
#include <cstring>

namespace {

__global__ void timestep_embed_kernel(const float* t, const float* freqs, float* out, int half) {
  // TimestepEmbedder.timestep_embedding: args = 1000 * t * freqs; [cos | sin]  (dit.py:38-56)
  const int k = blockIdx.x, i = threadIdx.x;
  if (i >= half) return;
  const float a = 1000.f * t[k] * freqs[i];
  out[(long long)k * 2 * half + i] = cosf(a);
  out[(long long)k * 2 * half + half + i] = sinf(a);
}

__global__ void gamma_residual_kernel(const float* y, const float* gamma, float* x, long long rows, int C) {
  // ConvNeXtBlock tail: x = residual + gamma * y   (vocos.py:521-526)
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * C) return;
  x[i] += gamma[i % C] * y[i];
}

}  // namespace

struct AdaLN {
  const float* norm_w = nullptr;
  int mod_off = 0;  // offset of (weight | bias) inside the per-timestep modulation row
};

struct S2melState {
  idx_s2mel_config cfg;
  idx_codec_config ccfg;
  bool has_s2mel = false, has_codec = false;
  WeightPool pool;
  int inter = 0;
  // DiT
  std::vector<PackedW> wqkv, wo, w13, w2, skip_in;
  std::vector<AdaLN> attn_norm, ffn_norm;
  AdaLN final_norm;
  PackedW mod_stack;      // all adaLN project_layers stacked: [nmod*2H][H]
  PackedW cond_proj, merge_x, merge_rest, skip_linear, conv1, res_proj, fl_linear, conv2, fl_mod;
  PackedW te_mlp0, te_mlp2, te2_mlp0, te2_mlp2, wn_cond;
  const float *te_freqs = nullptr, *te2_freqs = nullptr;
  std::vector<PackedW> wn_in, wn_res, wn_skip;
  // fused-epilogue weight layouts of the fp16 path (rows of the two halves interleaved): w1|w3 and the WaveNet in_layers
  std::vector<__half*> w13_i16, wn_in_i16;
  std::vector<float*> wn_in_bias_i;
  int mod_width = 0;
  // length regulator
  PackedW lr_in_proj, lr_out;
  std::vector<PackedW> lr_conv;
  std::vector<const float*> lr_gn_w, lr_gn_b;
  // codec
  PackedW cd_out_proj, cd_embed, cd_head, cd_up;
  const float* cd_codebook = nullptr;
  const float *cd_norm_w = nullptr, *cd_norm_b = nullptr, *cd_fnorm_w = nullptr, *cd_fnorm_b = nullptr;
  struct CNX { const float *dw_w, *dw_b, *n_w, *n_b, *gamma; PackedW pw1, pw2; };
  std::vector<CNX> cnx;
  double ms_codec = 0, ms_lr = 0, ms_cfm = 0;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
};

void s2mel_destroy(S2melState* s) {
  if (!s) return;
  s->pool.release();
  if (s->ev0) cudaEventDestroy(s->ev0);
  if (s->ev1) cudaEventDestroy(s->ev1);
  delete s;
}

static S2melState* state(idx_engine* e) {
  if (!e->s2mel) {
    e->s2mel = new S2melState();
    IDX_CUDA(cudaEventCreate(&e->s2mel->ev0));
    IDX_CUDA(cudaEventCreate(&e->s2mel->ev1));
  }
  return e->s2mel;
}

// stack several [rows_i][K] linear layers into one packed weight (rows concatenated)
static PackedW pack_stacked(idx_engine* e, WeightPool& pool, const std::vector<std::string>& names, float** bias_out) {
  int K = -1, N = 0;
  for (auto& n : names) {
    const DevTensor& w = e->W(n + ".weight");
    IDX_CHECK(w.shape.size() >= 2, IDX_ERR_ARG, n + ": bad shape");
    if (K < 0) K = (int)w.shape[1];
    IDX_CHECK((int)w.shape[1] == K, IDX_ERR_ARG, n + ": K mismatch in stacked pack");
    N += (int)w.shape[0];
  }
  // build a temporary concatenated [N][K] master, register it under a synthetic name, pack, drop
  float* cat = nullptr;
  IDX_CUDA(cudaMalloc((void**)&cat, (size_t)N * K * 4));
  float* bias = pool.alloc(N);
  IDX_CUDA(cudaMemsetAsync(bias, 0, (size_t)N * 4, e->stream));
  int r = 0;
  for (auto& n : names) {
    const DevTensor& w = e->W(n + ".weight");
    const int rows = (int)w.shape[0];
    IDX_CUDA(cudaMemcpyAsync(cat + (size_t)r * K, w.d, (size_t)rows * K * 4, cudaMemcpyDeviceToDevice, e->stream));
    if (e->has(n + ".bias"))
      IDX_CUDA(cudaMemcpyAsync(bias + r, e->W(n + ".bias").d, (size_t)rows * 4, cudaMemcpyDeviceToDevice, e->stream));
    r += rows;
  }
  DevTensor t;
  t.d = cat; t.dtype = IDX_F32; t.shape = {N, K};
  const std::string tmpname = "__stack_tmp__";
  e->weights.erase(tmpname);
  e->weights.emplace(tmpname + ".weight", t);
  PackedW p = pack_linear(e, pool, tmpname, 0, -1, false);
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  e->weights.erase(tmpname + ".weight");
  cudaFree(cat);
  p.bias = bias;
  if (bias_out) *bias_out = bias;
  return p;
}

extern "C" int idx_s2mel_init(idx_engine* e, const idx_s2mel_config* cfg) {
  IDX_API_BEGIN
  IDX_CHECK(e && cfg, IDX_ERR_ARG, "null argument");
  IDX_CUDA(cudaSetDevice(e->device));
  S2melState* s = state(e);
  s->cfg = *cfg;
  const int H = cfg->hidden, Dn = cfg->depth, WH = cfg->wn_hidden, NL = cfg->wn_layers, C = cfg->in_channels;
  IDX_CHECK(H == cfg->heads * 64, IDX_ERR_ARG, "DiT head_dim must be 64");
  IDX_CHECK(WH == H, IDX_ERR_ARG, "FinalLayer requires wavenet.hidden_dim == DiT.hidden_dim (diffusion_transformer.py:84-101)");
  s->inter = ((int)(2 * 4 * H / 3) + 255) / 256 * 256;  // gpt_fast/model.py:59-63
  const std::string E = "s2mel.cfm.estimator.";
  std::vector<std::string> mods;
  s->wqkv.clear(); s->wo.clear(); s->w13.clear(); s->w2.clear(); s->skip_in.clear();
  s->attn_norm.clear(); s->ffn_norm.clear();
  for (int l = 0; l < Dn; ++l) {
    const std::string p = E + "transformer.layers." + std::to_string(l) + ".";
    s->wqkv.push_back(pack_linear(e, s->pool, p + "attention.wqkv"));
    s->wo.push_back(pack_linear(e, s->pool, p + "attention.wo"));
    s->w13.push_back(pack_stacked(e, s->pool, {p + "feed_forward.w1", p + "feed_forward.w3"}, nullptr));
    s->w13.back().bias = nullptr;
    s->w2.push_back(pack_linear(e, s->pool, p + "feed_forward.w2"));
    s->skip_in.push_back(pack_linear(e, s->pool, p + "skip_in_linear"));
    AdaLN a; a.norm_w = e->Wf(p + "attention_norm.norm.weight"); a.mod_off = (int)mods.size() * 2 * H;
    mods.push_back(p + "attention_norm.project_layer");
    AdaLN f; f.norm_w = e->Wf(p + "ffn_norm.norm.weight"); f.mod_off = (int)mods.size() * 2 * H;
    mods.push_back(p + "ffn_norm.project_layer");
    s->attn_norm.push_back(a);
    s->ffn_norm.push_back(f);
  }
  s->final_norm.norm_w = e->Wf(E + "transformer.norm.norm.weight");
  s->final_norm.mod_off = (int)mods.size() * 2 * H;
  mods.push_back(E + "transformer.norm.project_layer");
  s->mod_stack = pack_stacked(e, s->pool, mods, nullptr);
  s->mod_width = (int)mods.size() * 2 * H;
  s->cond_proj = pack_linear(e, s->pool, E + "cond_projection");
  // cond_x_merge_linear columns: [x(80) | prompt_x(80) | cond(H) | style]  (dit.py:214-225)
  {
    const DevTensor& w = e->W(E + "cond_x_merge_linear.weight");
    const int Kall = (int)w.shape[1];
    IDX_CHECK(Kall == H + 2 * C + cfg->style_dim, IDX_ERR_ARG, "cond_x_merge_linear shape");
    // split by columns: copy into two masters
    std::vector<float> h((size_t)H * Kall);
    IDX_CUDA(cudaMemcpy(h.data(), w.d, h.size() * 4, cudaMemcpyDeviceToHost));
    std::vector<float> hx((size_t)H * C), hr((size_t)H * (Kall - C));
    for (int r = 0; r < H; ++r) {
      memcpy(&hx[(size_t)r * C], &h[(size_t)r * Kall], (size_t)C * 4);
      memcpy(&hr[(size_t)r * (Kall - C)], &h[(size_t)r * Kall + C], (size_t)(Kall - C) * 4);
    }
    int64_t shx[2] = {H, C}, shr[2] = {H, Kall - C};
    IDX_CHECK(idx_load_weight(e, "__merge_x.weight", hx.data(), IDX_F32, 2, shx) == 0, IDX_ERR_ARG, e->err);
    IDX_CHECK(idx_load_weight(e, "__merge_rest.weight", hr.data(), IDX_F32, 2, shr) == 0, IDX_ERR_ARG, e->err);
    s->merge_x = pack_linear(e, s->pool, "__merge_x", 0, -1, false);
    s->merge_rest = pack_linear(e, s->pool, "__merge_rest", 0, -1, false);
    s->merge_rest.bias = e->Wf(E + "cond_x_merge_linear.bias");
  }
  s->skip_linear = pack_linear(e, s->pool, E + "skip_linear");
  s->conv1 = pack_linear(e, s->pool, E + "conv1");
  s->res_proj = pack_linear(e, s->pool, E + "res_projection");
  s->fl_linear = pack_linear(e, s->pool, E + "final_layer.linear");
  s->fl_mod = pack_linear(e, s->pool, E + "final_layer.adaLN_modulation.1");
  s->conv2 = pack_linear(e, s->pool, E + "conv2");
  s->te_mlp0 = pack_linear(e, s->pool, E + "t_embedder.mlp.0");
  s->te_mlp2 = pack_linear(e, s->pool, E + "t_embedder.mlp.2");
  s->te2_mlp0 = pack_linear(e, s->pool, E + "t_embedder2.mlp.0");
  s->te2_mlp2 = pack_linear(e, s->pool, E + "t_embedder2.mlp.2");
  s->te_freqs = e->Wf(E + "t_embedder.freqs");
  s->te2_freqs = e->Wf(E + "t_embedder2.freqs");
  s->wn_cond = pack_linear(e, s->pool, E + "wavenet.cond_layer.conv.conv");
  s->wn_in.clear(); s->wn_res.clear(); s->wn_skip.clear();
  for (int i = 0; i < NL; ++i) {
    const std::string wi = E + "wavenet.in_layers." + std::to_string(i) + ".conv.conv";
    const std::string wr = E + "wavenet.res_skip_layers." + std::to_string(i) + ".conv.conv";
    s->wn_in.push_back(pack_conv1d(e, s->pool, wi, 1));
    IDX_CHECK(s->wn_in.back().taps == cfg->wn_kernel, IDX_ERR_ARG, "wavenet kernel size");
    if (i < NL - 1) {
      s->wn_res.push_back(pack_linear(e, s->pool, wr, 0, WH));
      s->wn_skip.push_back(pack_linear(e, s->pool, wr, WH, WH));
    } else {
      s->wn_res.push_back(PackedW());
      s->wn_skip.push_back(pack_linear(e, s->pool, wr, 0, WH));
    }
  }
  // length regulator
  const std::string R = "s2mel.length_regulator.";
  s->lr_in_proj = pack_linear(e, s->pool, R + "content_in_proj");
  s->lr_conv.clear(); s->lr_gn_w.clear(); s->lr_gn_b.clear();
  for (int i = 0; i < cfg->lr_convs; ++i) {
    s->lr_conv.push_back(pack_conv1d(e, s->pool, R + "model." + std::to_string(3 * i), 1));
    s->lr_gn_w.push_back(e->Wf(R + "model." + std::to_string(3 * i + 1) + ".weight"));
    s->lr_gn_b.push_back(e->Wf(R + "model." + std::to_string(3 * i + 1) + ".bias"));
  }
  s->lr_out = pack_linear(e, s->pool, R + "model." + std::to_string(3 * cfg->lr_convs));
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  // fp16 K-major copies for the tensor-core path with fp16 operands (DiT + WaveNet GEMMs; made once)
  for (auto* v : {&s->wqkv, &s->wo, &s->w13, &s->w2, &s->skip_in, &s->wn_in, &s->wn_res, &s->wn_skip})
    for (auto& w : *v) pack_half(e, s->pool, w);
  for (auto* w : {&s->skip_linear, &s->conv1, &s->res_proj, &s->fl_linear, &s->conv2}) pack_half(e, s->pool, *w);
  s->w13_i16.clear(); s->wn_in_i16.clear(); s->wn_in_bias_i.clear();
  for (auto& w : s->w13) s->w13_i16.push_back(pack_half_interleaved(e, s->pool, w, nullptr));
  for (auto& w : s->wn_in) {
    float* bi = nullptr;
    s->wn_in_i16.push_back(pack_half_interleaved(e, s->pool, w, &bi));
    s->wn_in_bias_i.push_back(bi);
  }
  s->has_s2mel = true;
  IDX_API_END(e)
}

extern "C" int idx_codec_init(idx_engine* e, const idx_codec_config* cfg) {
  IDX_API_BEGIN
  IDX_CHECK(e && cfg, IDX_ERR_ARG, "null argument");
  IDX_CUDA(cudaSetDevice(e->device));
  S2melState* s = state(e);
  s->ccfg = *cfg;
  const std::string Q = "codec.quantizer.quantizers.0.", D = "codec.decoder.0.";
  s->cd_codebook = e->Wf(Q + "codebook.weight");
  s->cd_out_proj = pack_linear(e, s->pool, Q + "out_project");
  s->cd_embed = pack_conv1d(e, s->pool, D + "embed", 1);
  s->cd_norm_w = e->Wf(D + "norm.weight"); s->cd_norm_b = e->Wf(D + "norm.bias");
  s->cd_fnorm_w = e->Wf(D + "final_layer_norm.weight"); s->cd_fnorm_b = e->Wf(D + "final_layer_norm.bias");
  s->cnx.clear();
  for (int l = 0; l < cfg->vocos_num_layers; ++l) {
    const std::string p = D + "convnext." + std::to_string(l) + ".";
    S2melState::CNX c;
    c.dw_w = e->Wf(p + "dwconv.weight"); c.dw_b = e->Wf(p + "dwconv.bias");
    c.n_w = e->Wf(p + "norm.weight"); c.n_b = e->Wf(p + "norm.bias");
    c.gamma = e->Wf(p + "gamma");
    c.pw1 = pack_linear(e, s->pool, p + "pwconv1");
    c.pw2 = pack_linear(e, s->pool, p + "pwconv2");
    s->cnx.push_back(c);
  }
  s->cd_head = pack_linear(e, s->pool, "codec.decoder.1");
  s->cd_up = pack_conv1d(e, s->pool, "codec.up", 1);
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  s->has_codec = true;
  IDX_API_END(e)
}

// ------------------------------------------------------------------ device-side stages --
// codes (device int32 [n]) -> S_infer (device [2n][hidden])
void codec_decode_dev(idx_engine* e, S2melState* s, const int* d_codes, int n, float* d_out) {
  const idx_codec_config& c = s->ccfg;
  const int Hs = c.hidden_size, Vd = c.vocos_dim, Vi = c.vocos_intermediate_dim;
  float* emb = e->arena.get<float>((size_t)n * c.codebook_dim);
  float* q = e->arena.get<float>((size_t)n * Hs);
  float* x = e->arena.get<float>((size_t)n * Vd);
  float* y = e->arena.get<float>((size_t)n * Vd);
  float* hbuf = e->arena.get<float>((size_t)n * Vi);
  float* up = e->arena.get<float>((size_t)2 * n * Hs);
  embedding_rows(e, s->cd_codebook, d_codes, emb, n, c.codebook_dim, c.codebook_size);
  conv_gemm(e, gemm_of(s->cd_out_proj, emb, 1, n, q));
  conv_gemm(e, gemm_of(s->cd_embed, q, 1, n, y));
  layernorm(e, y, x, 1, n, Vd, s->cd_norm_w, s->cd_norm_b, 1e-6f, nullptr, nullptr, 0);
  for (auto& b : s->cnx) {
    dwconv1d(e, x, y, 1, n, Vd, b.dw_w, b.dw_b, 7);
    layernorm(e, y, y, 1, n, Vd, b.n_w, b.n_b, 1e-6f, nullptr, nullptr, 0);
    ConvGemm g1 = gemm_of(b.pw1, y, 1, n, hbuf);
    g1.act = ACT_GELU_ERF;
    conv_gemm(e, g1);
    ConvGemm g2 = gemm_of(b.pw2, hbuf, 1, n, x);   // x = residual + gamma * (pw2(h) + bias)
    g2.colscale = b.gamma; g2.res = x;
    conv_gemm(e, g2);
  }
  layernorm(e, x, y, 1, n, Vd, s->cd_fnorm_w, s->cd_fnorm_b, 1e-6f, nullptr, nullptr, 0);
  conv_gemm(e, gemm_of(s->cd_head, y, 1, n, q));
  nearest_interp(e, q, up, 1, n, 2 * n, Hs);
  conv_gemm(e, gemm_of(s->cd_up, up, 1, 2 * n, d_out));
}

// S (device [n_in][lr_in]) -> cond (device rows written at d_out with row stride = content_dim)
void length_regulate_dev(idx_engine* e, S2melState* s, const float* d_S, int n_in, int ylen, float* d_out) {
  const idx_s2mel_config& c = s->cfg;
  const int C = c.content_dim;
  float* a = e->arena.get<float>((size_t)n_in * C);
  float* x = e->arena.get<float>((size_t)ylen * C);
  float* y = e->arena.get<float>((size_t)ylen * C);
  conv_gemm(e, gemm_of(s->lr_in_proj, d_S, 1, n_in, a));
  nearest_interp(e, a, x, 1, n_in, ylen, C);
  for (int i = 0; i < c.lr_convs; ++i) {
    conv_gemm(e, gemm_of(s->lr_conv[i], x, 1, ylen, y));
    groupnorm1_mish(e, y, x, 1, ylen, C, s->lr_gn_w[i], s->lr_gn_b[i], 1e-5f);
  }
  conv_gemm(e, gemm_of(s->lr_out, x, 1, ylen, d_out));
}

struct DitBuffers {
  float *h[16], *a, *qkv, *att, *ff, *cat, *xres, *wy, *wpad, *wxin, *wacts, *wout, *z, *v, *rope;
  // fp16 images of the GEMM operands (tail_half mode): written by the kernel that produces the operand
  __half *a16 = nullptr, *att16 = nullptr, *ffh16 = nullptr, *cat16 = nullptr, *xres16 = nullptr, *wpad16 = nullptr,
         *wacts16 = nullptr, *z16 = nullptr, *wy16 = nullptr, *qkv16 = nullptr;     // qkv16: Qr | Kr | Vb [B*H][T][64] each
  // packed solve (two or more segments; null otherwise): the utterances' segments along T, and the gapped WaveNet gate
  // output (see dit_eval)
  const Segments* sg = nullptr;
  __half* wacts16g = nullptr;
};

// one DiT evaluation for batch Bn. x_t [T][80] (shared when x_bcast), C0 [Bn][T][H] constant part
// of the merge linear, mod/wncond/flmod: rows of the per-timestep tables. out v [Bn][T][80].
static void dit_eval(idx_engine* e, S2melState* s, DitBuffers& b, int Bn, int T, const float* x_t, int x_bcast,
                     const float* C0, const float* mod, const float* wncond, const float* flmod) {
  const idx_s2mel_config& c = s->cfg;
  const int H = c.hidden, Dn = c.depth, WH = c.wn_hidden, NL = c.wn_layers, C = c.in_channels, nh = c.heads;
  // h0 = x · Wx^T + C0
  {
    ConvGemm g = gemm_of(s->merge_x, x_t, Bn, T, b.h[0]);
    g.a_bcast = x_bcast; g.res = C0;
    conv_gemm(e, g);
  }
  const bool hf = b.a16 != nullptr;     // fp16 GEMM operands and the fused pair epilogues (alloc_dit decides: cfm_half)
  auto G = [&](const PackedW& w, const float* A32, const __half* A16, int Bb, int Tt, float* out) {
    return hf ? gemm_of16(w, A16, Bb, Tt, out) : gemm_of(w, A32, Bb, Tt, out);
  };
  float* h = b.h[0];
  int nskip = 0;
  float* skips[16];
  for (int l = 0; l < Dn; ++l) {
    if (l > Dn / 2) {   // layers_receive_skip (gpt_fast/model.py:166-167)
      float* sk = skips[--nskip];
      copy_cols(e, h, H, hf ? nullptr : b.cat, 2 * H, 0, (long long)Bn * T, H, b.cat16);
      copy_cols(e, sk, H, hf ? nullptr : b.cat, 2 * H, H, (long long)Bn * T, H, b.cat16);
      float* hn = b.h[8 + (l & 1)];
      conv_gemm(e, G(s->skip_in[l], b.cat, b.cat16, Bn, T, hn));
      h = hn;
    }
    rmsnorm_adaln(e, h, hf ? nullptr : b.a, Bn, T, H, s->attn_norm[l].norm_w, mod + s->attn_norm[l].mod_off,
                  mod + s->attn_norm[l].mod_off + H, 0, 1e-5f, b.a16);
    if (hf) {
      // wqkv with the RoPE / q scale / head split in its epilogue: fp16 Qr | Kr | Vb go straight to the flash attention
      ConvGemm g = gemm_of16(s->wqkv[l], b.a16, Bn, T, nullptr);
      g.epi = EPI_ROPE; g.out16 = b.qkv16; g.aux = b.rope; g.aux_stride = nh; g.scale = FLASH_Q_SCALE;
      conv_gemm(e, g);
      const size_t one = (size_t)Bn * nh * T * 64;
      if (b.sg) flash_attention_wgmma_varlen(e, b.qkv16, b.qkv16 + one, b.qkv16 + 2 * one, nullptr, b.att16, Bn, nh, *b.sg);
      else flash_attention_wgmma(e, b.qkv16, b.qkv16 + one, b.qkv16 + 2 * one, nullptr, b.att16, Bn, T, nh);
    } else {
      conv_gemm(e, gemm_of(s->wqkv[l], b.a, Bn, T, b.qkv));
      attention_rope(e, b.qkv, b.att, Bn, T, nh, b.rope);
    }
    // layer output buffer: emitted skips (l < Dn/2) keep their own buffer
    float* hout = (l < Dn / 2) ? b.h[1 + l] : b.h[10 + (l & 1)];
    {
      ConvGemm g = G(s->wo[l], b.att, b.att16, Bn, T, hout);
      g.res = h;
      conv_gemm(e, g);
    }
    rmsnorm_adaln(e, hout, hf ? nullptr : b.a, Bn, T, H, s->ffn_norm[l].norm_w, mod + s->ffn_norm[l].mod_off,
                  mod + s->ffn_norm[l].mod_off + H, 0, 1e-5f, b.a16);
    if (hf) {
      ConvGemm g = gemm_of16(s->w13[l], b.a16, Bn, T, nullptr);       // SwiGLU in the epilogue (w1 / w3 rows interleaved)
      g.Wk16 = s->w13_i16[l]; g.bias = nullptr; g.epi = EPI_SWIGLU; g.out16 = b.ffh16;
      conv_gemm(e, g);
    } else {
      conv_gemm(e, gemm_of(s->w13[l], b.a, Bn, T, b.ff));
      swiglu(e, b.ff, b.qkv, (long long)Bn * T, s->inter);
    }
    {
      ConvGemm g = G(s->w2[l], b.qkv, b.ffh16, Bn, T, hout);
      g.res = hout;
      conv_gemm(e, g);
    }
    h = hout;
    if (l < Dn / 2) skips[nskip++] = h;
  }
  rmsnorm_adaln(e, h, b.a, Bn, T, H, s->final_norm.norm_w, mod + s->final_norm.mod_off,
                mod + s->final_norm.mod_off + H, 0, 1e-5f);
  // long skip: x_res = skip_linear(cat[h, x])   (dit.py:242-243)
  copy_cols(e, b.a, H, hf ? nullptr : b.cat, H + C, 0, (long long)Bn * T, H, b.cat16);
  for (int bi = 0; bi < Bn; ++bi)
    copy_cols(e, x_bcast ? x_t : x_t + (size_t)bi * T * C, C, hf ? nullptr : b.cat + (size_t)bi * T * (H + C), H + C, H, T, C,
              hf ? b.cat16 + (size_t)bi * T * (H + C) : nullptr);
  conv_gemm(e, G(s->skip_linear, b.cat, b.cat16, Bn, T, b.xres));
  if (hf) to_half(e, b.xres, b.xres16, (long long)Bn * T * H);          // operand of conv1 and res_projection
  conv_gemm(e, G(s->conv1, b.xres, b.xres16, Bn, T, b.wy));
  // WaveNet (wavenet.py:132-166), masks are all-ones for full-length sequences
  fill_zero(e, b.wout, (long long)Bn * T * WH);
  for (int i = 0; i < NL; ++i) {
    // SConv1d pad_mode='reflect' (encodec.py:196-229): materialise the reflected halo rows so the
    // conv is a plain zero-pad-free multi-tap GEMM (tensor-core path; TMA cannot reflect)
    const int kk = s->wn_in[i].taps, pl = (kk - 1) - (kk - 1) / 2, pr = (kk - 1) / 2;
    if (b.sg) {
      // packed: each segment gets its own reflected frame (kk - 1 rows more than the segment, so no tap reaches another
      // utterance); the conv runs once over the gapped frames and the gate output is compacted back to the packed rows
      const int gap = kk - 1, ng = b.sg->n();
      reflect_pad_segments(e, b.wy, b.wpad16, Bn, WH, pl, pr, *b.sg);
      ConvGemm gi = gemm_of16(s->wn_in[i], b.wpad16, Bn, T + ng * gap, nullptr);
      gi.pad = 0; gi.M = T + (ng - 1) * gap;
      gi.Wk16 = s->wn_in_i16[i]; gi.bias = s->wn_in_bias_i[i];
      gi.epi = EPI_WNGATE; gi.out16 = b.wacts16g; gi.aux = wncond + (size_t)i * 2 * WH; gi.aux_stride = 0;
      conv_gemm(e, gi);
      compact_segments16(e, b.wacts16g, b.wacts16, Bn, WH, gap, *b.sg);
    } else {
      reflect_pad_rows(e, b.wy, hf ? nullptr : b.wpad, Bn, T, WH, pl, pr, b.wpad16);
      ConvGemm gi = G(s->wn_in[i], b.wpad, b.wpad16, Bn, T + kk - 1, b.wxin);
      gi.pad = 0; gi.M = T;
      if (hf) {                 // the gate in the epilogue (tanh / sigmoid halves interleaved): fp16 acts, no [T][2 WH] round trip
        gi.Wk16 = s->wn_in_i16[i]; gi.bias = s->wn_in_bias_i[i]; gi.out = nullptr;
        gi.epi = EPI_WNGATE; gi.out16 = b.wacts16; gi.aux = wncond + (size_t)i * 2 * WH; gi.aux_stride = 0;
        conv_gemm(e, gi);
      } else {
        conv_gemm(e, gi);
        wn_gate(e, b.wxin, wncond + (size_t)i * 2 * WH, 0, b.wacts, Bn, T, WH);
      }
    }
    if (i < NL - 1) {
      ConvGemm gr = G(s->wn_res[i], b.wacts, b.wacts16, Bn, T, b.wy);
      gr.res = b.wy;
      conv_gemm(e, gr);
    }
    ConvGemm gs = G(s->wn_skip[i], b.wacts, b.wacts16, Bn, T, b.wout);
    gs.accum = 1;
    conv_gemm(e, gs);
  }
  {
    ConvGemm g = G(s->res_proj, b.xres, b.xres16, Bn, T, b.wout);   // + res_projection(x_res)
    g.accum = 1;
    conv_gemm(e, g);
  }
  // FinalLayer: modulate(LN(x), shift, scale) -> linear ; then conv2 (1x1)
  layernorm(e, b.wout, hf ? nullptr : b.z, Bn, T, WH, nullptr, nullptr, 1e-6f, flmod + WH, flmod, 0, b.z16);
  conv_gemm(e, G(s->fl_linear, b.z, b.z16, Bn, T, b.wy));
  if (hf) to_half(e, b.wy, b.wy16, (long long)Bn * T * WH);
  conv_gemm(e, G(s->conv2, b.wy, b.wy16, Bn, T, b.v));
}

// sg with more than one segment (packed solve, fp16 mode only): RoPE positions restart at every segment, room for the
// per-segment WaveNet frames.  One segment (or none) is the single-sequence layout.
static void alloc_dit(idx_engine* e, S2melState* s, DitBuffers& b, int Bn, int T, const Segments* sg = nullptr) {
  const idx_s2mel_config& c = s->cfg;
  const int H = c.hidden, WH = c.wn_hidden, C = c.in_channels;
  const size_t bt = (size_t)Bn * T;
  if (sg && sg->n() == 1) sg = nullptr;
  for (int i = 0; i < 12; ++i) b.h[i] = e->arena.get<float>(bt * H);
  b.a = e->arena.get<float>(bt * H);
  b.qkv = e->arena.get<float>(bt * (size_t)std::max(3 * H, s->inter));
  b.att = e->arena.get<float>(bt * H);
  b.ff = e->arena.get<float>(bt * 2 * s->inter);
  b.cat = e->arena.get<float>(bt * 2 * H);
  b.xres = e->arena.get<float>(bt * H);
  b.wy = e->arena.get<float>(bt * WH);
  const size_t padT = (size_t)T + 8 * (sg ? sg->n() : 1);
  b.wpad = e->arena.get<float>((size_t)Bn * padT * WH);
  b.wxin = e->arena.get<float>(bt * 2 * WH);
  b.wacts = e->arena.get<float>(bt * WH);
  b.wout = e->arena.get<float>(bt * WH);
  b.z = e->arena.get<float>(bt * WH);
  b.v = e->arena.get<float>(bt * C);
  b.rope = e->arena.get<float>((size_t)T * 64);
  if (cfm_half(e, s)) {
    auto hb = [&](size_t n) { return (__half*)e->arena.alloc(n * sizeof(__half) + 16); };
    b.a16 = hb(bt * H); b.att16 = hb(bt * H); b.ffh16 = hb(bt * s->inter); b.cat16 = hb(bt * 2 * H);
    b.xres16 = hb(bt * H); b.wpad16 = hb((size_t)Bn * padT * WH); b.wacts16 = hb(bt * WH); b.z16 = hb(bt * WH);
    b.wy16 = hb(bt * WH);
    b.qkv16 = hb(3 * bt * H);
  }
  b.sg = sg;
  if (sg) {
    IDX_CHECK(b.a16, IDX_ERR_STATE, "packed solve outside the fp16 tail mode");
    b.wacts16g = (__half*)e->arena.alloc((size_t)Bn * padT * WH * sizeof(__half) + 16);
    rope_table_segments(e, b.rope, *sg, 64);
  } else {
    rope_table(e, b.rope, T, 64);
  }
}
// alloc_dit over nseg segments, plus the scratch attention_rope takes when the solve is not packed: linear in the length
static size_t dit_arena_bytes(const S2melState* s, int Bn, int T, int nseg) {
  const idx_s2mel_config& c = s->cfg;
  const size_t bt = (size_t)Bn * T, pad = (size_t)Bn * (T + 8 * (size_t)nseg) * c.wn_hidden;
  const size_t Tp = (size_t)((T + 3) & ~3);
  const size_t attn = nseg > 1 ? 0 : 4 * (size_t)Bn * c.heads * (3 * (size_t)T * 64 + 64 * Tp) + 8 * 256;
  const size_t half_bytes = 2 * (bt * c.hidden * 8 + bt * s->inter + bt * c.wn_hidden * 3 + (nseg > 1 ? 2 : 1) * pad) + 16 * 512;
  return attn + half_bytes + 4 * (bt * c.hidden * 20 + bt * 3 * s->inter + bt * c.wn_hidden * 6 + pad + bt * c.in_channels +
                                  (size_t)T * 64) + 64 * 256;
}

// timestep tables for a list of nt timesteps (device float [nt])
struct TimeTables { float *mod, *wncond, *flmod; };
static TimeTables time_tables(idx_engine* e, S2melState* s, const float* d_t, int nt) {
  const idx_s2mel_config& c = s->cfg;
  const int H = c.hidden, WH = c.wn_hidden;
  float* emb = e->arena.get<float>((size_t)nt * 256);
  float* t1a = e->arena.get<float>((size_t)nt * H);
  float* t1 = e->arena.get<float>((size_t)nt * H);
  float* t2a = e->arena.get<float>((size_t)nt * WH);
  float* t2 = e->arena.get<float>((size_t)nt * WH);
  TimeTables tt;
  tt.mod = e->arena.get<float>((size_t)nt * s->mod_width);
  tt.wncond = e->arena.get<float>((size_t)nt * 2 * WH * c.wn_layers);
  tt.flmod = e->arena.get<float>((size_t)nt * 2 * WH);
  timestep_embed_kernel<<<nt, 128, 0, e->stream>>>(d_t, s->te_freqs, emb, 128);
  IDX_CUDA(cudaGetLastError()); e->launches++;
  ConvGemm g = gemm_of(s->te_mlp0, emb, 1, nt, t1a); g.act = ACT_SILU; conv_gemm(e, g);
  conv_gemm(e, gemm_of(s->te_mlp2, t1a, 1, nt, t1));
  timestep_embed_kernel<<<nt, 128, 0, e->stream>>>(d_t, s->te2_freqs, emb, 128);
  IDX_CUDA(cudaGetLastError()); e->launches++;
  g = gemm_of(s->te2_mlp0, emb, 1, nt, t2a); g.act = ACT_SILU; conv_gemm(e, g);
  conv_gemm(e, gemm_of(s->te2_mlp2, t2a, 1, nt, t2));
  conv_gemm(e, gemm_of(s->mod_stack, t1, 1, nt, tt.mod));          // all adaLN project_layers
  conv_gemm(e, gemm_of(s->wn_cond, t2, 1, nt, tt.wncond));         // WN cond_layer(g)
  silu_inplace(e, t1, (long long)nt * H);                          // FinalLayer: SiLU then Linear
  conv_gemm(e, gemm_of(s->fl_mod, t1, 1, nt, tt.flmod));
  return tt;
}

// C0[b] = [prompt_x | cond_projection(mu_b) | style_b] · W_rest^T + bias   for b in {cond, uncond}
// sg with more than one segment (packed): d_style is [Bn][n][style], one style per segment
static float* merge_const(idx_engine* e, S2melState* s, int Bn, int T, const float* d_prompt_x /*[Bn][T][80]*/,
                          const float* d_mu /*[Bn][T][content]*/, const float* d_style /*[Bn][style]*/,
                          const Segments* sg = nullptr) {
  const idx_s2mel_config& c = s->cfg;
  const int H = c.hidden, C = c.in_channels, Sd = c.style_dim;
  const int Kr = C + H + Sd;
  float* rest = e->arena.get<float>((size_t)Bn * T * Kr);
  float* cp = e->arena.get<float>((size_t)Bn * T * H);
  float* C0 = e->arena.get<float>((size_t)Bn * T * H);
  conv_gemm(e, gemm_of(s->cond_proj, d_mu, Bn, T, cp));
  copy_cols(e, d_prompt_x, C, rest, Kr, 0, (long long)Bn * T, C);
  copy_cols(e, cp, H, rest, Kr, C, (long long)Bn * T, H);
  if (sg && sg->n() > 1) {
    for (int bi = 0; bi < Bn; ++bi)
      for (int u = 0; u < sg->n(); ++u)
        bcast_cols(e, d_style + ((size_t)bi * sg->n() + u) * Sd, rest + ((size_t)bi * T + sg->off[u]) * Kr, Kr, C + H, 1,
                   sg->len(u), Sd);
  } else {
    bcast_cols(e, d_style, rest, Kr, C + H, Bn, T, Sd);
  }
  conv_gemm(e, gemm_of(s->merge_rest, rest, Bn, T, C0));
  return C0;
}

// torch.linspace(0, 1, n+1) in fp32 (ATen symmetric formula) and the t = t + dt accumulation
static void euler_times(int n, std::vector<float>& t, std::vector<float>& dt) {
  const int steps = n + 1;
  std::vector<float> span(steps);
  const float step = (1.0f - 0.0f) / (float)(steps - 1);
  const int half = steps / 2;
  for (int i = 0; i < steps; ++i) span[i] = (i < half) ? 0.0f + step * (float)i : 1.0f - step * (float)(steps - i - 1);
  t.resize(n); dt.resize(n);
  float tc = span[0];
  for (int k = 1; k <= n; ++k) {
    dt[k - 1] = span[k] - span[k - 1];
    t[k - 1] = tc;
    tc = tc + dt[k - 1];
  }
}

CfmInputs cfm_inputs(idx_engine* e, const S2melState* s, int T, int n) {
  const idx_s2mel_config& c = s->cfg;
  CfmInputs in;
  in.x = e->arena.get<float>((size_t)T * c.in_channels);
  in.px = e->arena.get<float>((size_t)2 * T * c.in_channels);
  in.mu2 = e->arena.get<float>((size_t)2 * T * c.content_dim);
  in.st = e->arena.get<float>((size_t)2 * n * c.style_dim);
  fill_zero(e, in.px, (long long)2 * T * c.in_channels);
  fill_zero(e, in.mu2, (long long)2 * T * c.content_dim);
  fill_zero(e, in.st, (long long)2 * n * c.style_dim);
  return in;
}

void cfm_stage(idx_engine* e, const S2melState* s, const CfmInputs& in, int u, int o, int Tu, int P, const float* z,
               const float* ref_mel, const float* mu, int mu_rows, const float* style) {
  const idx_s2mel_config& c = s->cfg;
  const int C = c.in_channels, Cd = c.content_dim, Sd = c.style_dim;
  const size_t mark = e->arena.off;
  float* d_z = e->arena.get<float>((size_t)C * Tu);
  idx_to_device(e, d_z, z, (size_t)C * Tu * 4);
  transpose_bct_to_btc(e, d_z, in.x + (size_t)o * C, 1, C, Tu);
  if (P > 0) {
    float* d_prompt = e->arena.get<float>((size_t)C * P);
    idx_to_device(e, d_prompt, ref_mel, (size_t)C * P * 4);
    transpose_bct_to_btc(e, d_prompt, in.px + (size_t)o * C, 1, C, P);
    fill_zero(e, in.x + (size_t)o * C, (long long)P * C);          // x[..., :prompt_len] = 0
  }
  idx_to_device(e, in.mu2 + (size_t)o * Cd, mu, (size_t)mu_rows * Cd * 4);
  idx_to_device(e, in.st + (size_t)u * Sd, style, (size_t)Sd * 4);
  e->arena.off = mark;
}

void cfm_solve_dev(idx_engine* e, S2melState* s, Segments& sg, const int* P, const CfmInputs& in, int n_steps, float rate) {
  const idx_s2mel_config& c = s->cfg;
  const int C = c.in_channels, T = sg.total(), Bn = 2;
  unsigned char* zero_rows = nullptr;       // packed: 1 on each segment's own prompt frames
  if (sg.n() > 1) {
    segments_upload(e, sg);
    std::vector<unsigned char> zr(T, 0);
    for (int u = 0; u < sg.n(); ++u) std::fill(zr.begin() + sg.off[u], zr.begin() + sg.off[u] + P[u], 1);
    zero_rows = (unsigned char*)e->arena.alloc(T);
    idx_to_device(e, zero_rows, zr.data(), T);
  }
  std::vector<float> ts, dts;
  euler_times(n_steps, ts, dts);
  float* d_t = e->arena.get<float>(n_steps);
  IDX_CUDA(cudaMemcpyAsync(d_t, ts.data(), (size_t)n_steps * 4, cudaMemcpyHostToDevice, e->stream));
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  TimeTables tt = time_tables(e, s, d_t, n_steps);
  float* C0 = merge_const(e, s, Bn, T, in.px, in.mu2, in.st, &sg);
  DitBuffers b;
  alloc_dit(e, s, b, Bn, T, &sg);
  for (int k = 0; k < n_steps; ++k) {
    dit_eval(e, s, b, Bn, T, in.x, 1, C0, tt.mod + (size_t)k * s->mod_width,
             tt.wncond + (size_t)k * 2 * c.wn_hidden * c.wn_layers, tt.flmod + (size_t)k * 2 * c.wn_hidden);
    if (zero_rows) cfg_euler_rows(e, in.x, b.v, b.v + (size_t)T * C, dts[k], rate, T, C, zero_rows);
    else cfg_euler(e, in.x, b.v, b.v + (size_t)T * C, dts[k], rate, T, C, P[0]);
  }
}
size_t cfm_arena_bytes(const S2melState* s, const Segments& sg, int n_steps) {
  const idx_s2mel_config& c = s->cfg;
  const int T = sg.total(), n = sg.n();
  return dit_arena_bytes(s, 2, T, n) + 4 * (size_t)T * (8 * c.in_channels + 3 * c.content_dim + 6 * c.hidden + 2 * c.style_dim) +
         4 * (size_t)n_steps * (s->mod_width + 2 * c.wn_hidden * (c.wn_layers + 1) + 6 * c.hidden + 512) +
         (n > 1 ? (size_t)T + 16 * ((size_t)T / 128 + 2 * (size_t)n + 1) + 768 : 0) + (4 << 20);   // segment tables, zero_rows
}
bool cfm_half(const idx_engine* e, const S2melState* s) {
  const idx_s2mel_config& c = s->cfg;
  return tail_half(e) && c.hidden % 8 == 0 && c.wn_hidden % 8 == 0 && (c.hidden + c.in_channels) % 8 == 0 && s->inter % 8 == 0;
}

size_t codec_arena_bytes(const S2melState* s, int n) {
  const idx_codec_config& c = s->ccfg;
  return 4 * (size_t)n * (c.codebook_dim + 5 * c.hidden_size + 2 * c.vocos_dim + c.vocos_intermediate_dim) + (1 << 20);
}
size_t lr_arena_bytes(const S2melState* s, int n_in, int ylen) {
  const idx_s2mel_config& c = s->cfg;
  return 4 * ((size_t)n_in * (c.lr_in + c.content_dim) + 4 * (size_t)ylen * c.content_dim) + (1 << 20);
}
int s2mel_style_dim(const S2melState* s) { return s->cfg.style_dim; }
int s2mel_content_dim(const S2melState* s) { return s->cfg.content_dim; }
int s2mel_codec_hidden(const S2melState* s) { return s->ccfg.hidden_size; }
bool s2mel_ready(const S2melState* s) { return s && s->has_s2mel && s->has_codec; }
void s2mel_set_ms(S2melState* s, double codec, double lr, double cfm) { s->ms_codec = codec; s->ms_lr = lr; s->ms_cfm = cfm; }

// ------------------------------------------------------------------------------ C-ABI --
extern "C" int idx_codec_decode(idx_engine* e, const int32_t* codes, int n, float* S_out) {
  IDX_API_BEGIN
  IDX_CHECK(e && e->s2mel && e->s2mel->has_codec, IDX_ERR_STATE, "idx_codec_init has not been called");
  IDX_CHECK(codes && S_out && n >= 1, IDX_ERR_ARG, "bad arguments");
  IDX_CUDA(cudaSetDevice(e->device));
  S2melState* s = e->s2mel;
  const idx_codec_config& c = s->ccfg;
  e->ensure_arena(codec_arena_bytes(s, n) + 8 * (size_t)n * c.hidden_size);
  e->arena.reset();
  int* d_codes = e->arena.get<int>(n);
  float* d_out = e->arena.get<float>((size_t)2 * n * c.hidden_size);
  idx_to_device(e, d_codes, codes, (size_t)n * 4);
  IDX_CUDA(cudaEventRecord(s->ev0, e->stream));
  codec_decode_dev(e, s, d_codes, n, d_out);
  IDX_CUDA(cudaEventRecord(s->ev1, e->stream));
  idx_from_device(e, S_out, d_out, (size_t)2 * n * c.hidden_size * 4);
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  e->check_flag("semantic code outside the codebook (codes must be cut before the stop token, infer_v2_5.py:809-821)");
  float ms; IDX_CUDA(cudaEventElapsedTime(&ms, s->ev0, s->ev1)); s->ms_codec = ms;
  IDX_API_END(e)
}

extern "C" int idx_length_regulate(idx_engine* e, const float* S, int n_in, int ylen, float* cond_out) {
  IDX_API_BEGIN
  IDX_CHECK(e && e->s2mel && e->s2mel->has_s2mel, IDX_ERR_STATE, "idx_s2mel_init has not been called");
  IDX_CHECK(S && cond_out && n_in >= 1 && ylen >= 1, IDX_ERR_ARG, "bad arguments");
  IDX_CUDA(cudaSetDevice(e->device));
  S2melState* s = e->s2mel;
  const idx_s2mel_config& c = s->cfg;
  e->ensure_arena(4 * ((size_t)n_in * (c.lr_in + c.content_dim) + 4 * (size_t)ylen * c.content_dim) + (1 << 20));
  e->arena.reset();
  float* d_S = e->arena.get<float>((size_t)n_in * c.lr_in);
  float* d_out = e->arena.get<float>((size_t)ylen * c.content_dim);
  idx_to_device(e, d_S, S, (size_t)n_in * c.lr_in * 4);
  IDX_CUDA(cudaEventRecord(s->ev0, e->stream));
  length_regulate_dev(e, s, d_S, n_in, ylen, d_out);
  IDX_CUDA(cudaEventRecord(s->ev1, e->stream));
  idx_from_device(e, cond_out, d_out, (size_t)ylen * c.content_dim * 4);
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  float ms; IDX_CUDA(cudaEventElapsedTime(&ms, s->ev0, s->ev1)); s->ms_lr = ms;
  IDX_API_END(e)
}

extern "C" int idx_dit_forward(idx_engine* e, const float* x, const float* prompt_x, const float* t,
                               const float* style, const float* cond, int B, int T, float* out) {
  IDX_API_BEGIN
  IDX_CHECK(e && e->s2mel && e->s2mel->has_s2mel, IDX_ERR_STATE, "idx_s2mel_init has not been called");
  IDX_CHECK(x && prompt_x && t && style && cond && out && B >= 1 && T >= 1, IDX_ERR_ARG, "bad arguments");
  IDX_CUDA(cudaSetDevice(e->device));
  S2melState* s = e->s2mel;
  const idx_s2mel_config& c = s->cfg;
  const int C = c.in_channels;
  e->ensure_arena(dit_arena_bytes(s, B, T, 1) + 4 * (size_t)B * T * (4 * C + c.content_dim + 3 * c.hidden + c.style_dim) +
                  4 * (size_t)B * (s->mod_width + 2 * c.wn_hidden * (c.wn_layers + 1) + 6 * c.hidden + 512) + (4 << 20));
  e->arena.reset();
  float* d_x = e->arena.get<float>((size_t)B * C * T);
  float* d_p = e->arena.get<float>((size_t)B * C * T);
  float* d_xt = e->arena.get<float>((size_t)B * C * T);
  float* d_pt = e->arena.get<float>((size_t)B * C * T);
  float* d_t = e->arena.get<float>(B);
  float* d_style = e->arena.get<float>((size_t)B * c.style_dim);
  float* d_cond = e->arena.get<float>((size_t)B * T * c.content_dim);
  idx_to_device(e, d_x, x, (size_t)B * C * T * 4);
  idx_to_device(e, d_p, prompt_x, (size_t)B * C * T * 4);
  idx_to_device(e, d_t, t, (size_t)B * 4);
  idx_to_device(e, d_style, style, (size_t)B * c.style_dim * 4);
  idx_to_device(e, d_cond, cond, (size_t)B * T * c.content_dim * 4);
  transpose_bct_to_btc(e, d_x, d_xt, B, C, T);
  transpose_bct_to_btc(e, d_p, d_pt, B, C, T);
  // per-sample timesteps: evaluate each batch entry with its own table row
  TimeTables tt = time_tables(e, s, d_t, B);
  float* C0 = merge_const(e, s, B, T, d_pt, d_cond, d_style);
  float* d_v = e->arena.get<float>((size_t)B * T * C);
  for (int bi = 0; bi < B; ++bi) {
    DitBuffers b;
    const size_t mark = e->arena.off;
    alloc_dit(e, s, b, 1, T);
    dit_eval(e, s, b, 1, T, d_xt + (size_t)bi * T * C, 0, C0 + (size_t)bi * T * c.hidden,
             tt.mod + (size_t)bi * s->mod_width, tt.wncond + (size_t)bi * 2 * c.wn_hidden * c.wn_layers,
             tt.flmod + (size_t)bi * 2 * c.wn_hidden);
    IDX_CUDA(cudaMemcpyAsync(d_v + (size_t)bi * T * C, b.v, (size_t)T * C * 4, cudaMemcpyDeviceToDevice, e->stream));
    e->arena.off = mark;
  }
  transpose_btc_to_bct(e, d_v, d_x, B, T, C);
  idx_from_device(e, out, d_x, (size_t)B * C * T * 4);
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  IDX_API_END(e)
}

extern "C" int idx_cfm_solve(idx_engine* e, const float* mu, int T, const float* prompt, int P,
                             const float* style, const float* z, int n_steps, float cfg_rate, float* mel_out) {
  IDX_API_BEGIN
  IDX_CHECK(e && e->s2mel && e->s2mel->has_s2mel, IDX_ERR_STATE, "idx_s2mel_init has not been called");
  IDX_CHECK(mu && style && z && mel_out && T >= 1 && n_steps >= 1 && (P == 0 || prompt), IDX_ERR_ARG, "bad arguments");
  IDX_CHECK(P >= 0 && P <= T, IDX_ERR_ARG, "prompt longer than sequence");
  IDX_CHECK(cfg_rate > 0.f, IDX_ERR_ARG, "inference_cfg_rate must be > 0 (the CFG pair path is the one built)");
  IDX_CUDA(cudaSetDevice(e->device));
  S2melState* s = e->s2mel;
  const int C = s->cfg.in_channels;
  Segments sg;
  sg.off = {0, T};
  e->ensure_arena(cfm_arena_bytes(s, sg, n_steps));     // with room for the staged inputs and the mel
  e->arena.reset();
  float* d_mel = e->arena.get<float>((size_t)C * T);
  CfmInputs in = cfm_inputs(e, s, T, 1);
  cfm_stage(e, s, in, 0, 0, T, P, z, prompt, mu, T, style);
  IDX_CUDA(cudaEventRecord(s->ev0, e->stream));
  cfm_solve_dev(e, s, sg, &P, in, n_steps, cfg_rate);
  transpose_btc_to_bct(e, in.x, d_mel, 1, T, C);
  IDX_CUDA(cudaEventRecord(s->ev1, e->stream));
  idx_from_device(e, mel_out, d_mel, (size_t)C * T * 4);
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  float ms; IDX_CUDA(cudaEventElapsedTime(&ms, s->ev0, s->ev1)); s->ms_cfm = ms;
  IDX_API_END(e)
}

extern "C" int idx_s2mel_last_ms(const idx_engine* e, double* ms3) {
  if (!e || !e->s2mel || !ms3) return IDX_ERR_STATE;
  ms3[0] = e->s2mel->ms_codec; ms3[1] = e->s2mel->ms_lr; ms3[2] = e->s2mel->ms_cfm;
  return IDX_OK;
}
