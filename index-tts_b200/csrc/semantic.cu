// semantic.cu — the w2v-BERT 2.0 prompt encoder behind IndexTTS2.get_emb (SURVEY.md §8f, DESIGN row f1) on sm_90a.
//
// Replaces:
//   IndexTTS2.get_emb                                   indextts/infer_v2_5.py:281-290
//   Wav2Vec2BertModel (feature projection + the first `layers` conformer layers, hidden_states[layers])
//                                                       transformers models/wav2vec2_bert/modeling_wav2vec2_bert.py
// and the (feat - semantic_mean) / semantic_std that follows, folded into the last layer's final_layer_norm at init.
//
// Default path: fp16 GEMM operands (written by the producing kernel), fp32 accumulate, fp32 residual stream; the attention is
// the wgmma flash kernel in its RELKEY mode (gemm_tc.cu), the conv module one fused kernel after pointwise_conv1.
// Strict path (gemm_backend 1 or IDX_NO_TC): fp32 everywhere, the attention unfused (batched GEMMs + exact softmax).
// The tail diagnostics tail_f16 / IDX_TAIL_F16, IDX_FA_WGMMA and IDX_ATTN_UNFUSED do not apply here.
// Padding: rows t >= lens[b] are zeroed at entry and before the depthwise conv, and masked as keys — what the HF encoder
// does with a prefix attention mask; those rows are still computed, as HF computes them.
#include "ops.h"
#include <cmath>

namespace {

constexpr int CM_ROWS = 8;        // output rows per CTA of the conv-module kernel
constexpr int CM_KMAX = 31;       // depthwise taps held in registers (shorter kernels are left-padded with zero taps)
constexpr int QE_W = 80;          // floats per row of qe = Q E^T (left_max + right_max + 1 <= 80)

// conv module after pointwise_conv1 (modeling_wav2vec2_bert.py:195-225), for CM_ROWS rows of one batch entry:
//   x [B][T][2C] pointwise_conv1 output -> GLU -> causal depthwise conv (rows t >= lens[b] and t < 0 read as zero, never
//   loaded) -> LayerNorm over C -> swish -> y [B][T][C] fp32 and / or y16 fp16 (the operand of pointwise_conv2).
// dw [C][CM_KMAX]: tap k multiplies row t - (CM_KMAX - 1) + k.  Each output row sums its taps in the order k = 0 .. 30,
// independently of the other rows and batch entries.
__global__ void __launch_bounds__(256)
conv_module_kernel(const float* __restrict__ x, const int* __restrict__ lens, const float* __restrict__ dw,
                   const float* __restrict__ lw, const float* __restrict__ lb, float eps, float* __restrict__ y,
                   __half* __restrict__ y16, int T, int C) {
  extern __shared__ float ys[];   // [CM_ROWS][C] depthwise conv output
  const int b = blockIdx.y, r0 = blockIdx.x * CM_ROWS, len = lens[b];
  const float* xb = x + (size_t)b * T * 2 * C;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float w[CM_KMAX], acc[CM_ROWS];
#pragma unroll
    for (int k = 0; k < CM_KMAX; ++k) w[k] = __ldg(dw + (size_t)c * CM_KMAX + k);
#pragma unroll
    for (int r = 0; r < CM_ROWS; ++r) acc[r] = 0.f;
#pragma unroll
    for (int s = 0; s < CM_ROWS + CM_KMAX - 1; ++s) {
      const int t = r0 - (CM_KMAX - 1) + s;
      float g = 0.f;
      if (t >= 0 && t < len) {
        const float a = xb[(size_t)t * 2 * C + c], gt = xb[(size_t)t * 2 * C + C + c];
        g = a * (1.f / (1.f + expf(-gt)));                     // nn.GLU(dim=channels)
      }
#pragma unroll
      for (int r = 0; r < CM_ROWS; ++r) {
        const int k = s - r;
        if (k >= 0 && k < CM_KMAX) acc[r] = fmaf(w[k], g, acc[r]);
      }
    }
#pragma unroll
    for (int r = 0; r < CM_ROWS; ++r) ys[r * C + c] = acc[r];
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int r = warp; r < CM_ROWS; r += blockDim.x >> 5) {
    const int t = r0 + r;
    if (t >= T) break;
    const float* v = ys + r * C;
    float s = 0.f;
    for (int c = lane; c < C; c += 32) s += v[c];
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s / C;
    float q = 0.f;
    for (int c = lane; c < C; c += 32) { const float d = v[c] - mean; q += d * d; }
    for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float rstd = rsqrtf(q / C + eps);
    const size_t o0 = ((size_t)b * T + t) * C;
    for (int c = lane; c < C; c += 32) {
      float u = (v[c] - mean) * rstd * __ldg(lw + c) + __ldg(lb + c);
      u = u / (1.f + expf(-u));                                 // swish
      if (y) y[o0 + c] = u;
      if (y16) y16[o0 + c] = __float2half_rn(u);
    }
  }
}

// rows t >= lens[b] of x [B][T][C] set to zero (the encoder's entry masked_fill)
__global__ void mask_rows_kernel(float* __restrict__ x, const int* __restrict__ lens, int T, int C) {
  const int t = blockIdx.x, b = blockIdx.y;
  if (t < lens[b]) return;
  for (int c = threadIdx.x; c < C; c += blockDim.x) x[((size_t)b * T + t) * C + c] = 0.f;
}

// strict path: q | k | v [B][T][3*H*64] -> Q, K [B*H][T][64], Vt [B*H][64][Tp]
__global__ void qkv_split_kernel(const float* __restrict__ qkv, float* __restrict__ Q, float* __restrict__ K,
                                 float* __restrict__ Vt, int T, int Tp, int H) {
  const int t = blockIdx.x, h = blockIdx.y, b = blockIdx.z, i = threadIdx.x;     // 64 threads
  const float* row = qkv + ((size_t)b * T + t) * 3 * H * 64;
  const size_t bh = (size_t)b * H + h;
  Q[(bh * T + t) * 64 + i] = row[h * 64 + i];
  K[(bh * T + t) * 64 + i] = row[(H + h) * 64 + i];
  Vt[(bh * 64 + i) * Tp + t] = row[(2 * H + h) * 64 + i];
}

// strict path: S [B*H][T][Tp] holds q.k / 8; adds (q . E[clamp(j - i, -L, R) + L]) / 8 and masks keys j >= lens[b] with
// -inf (HF adds finfo.min: the same zero after the softmax).  One CTA per (query row i, b*H + h).
__global__ void relkey_bias_kernel(float* __restrict__ S, const float* __restrict__ Q, const float* __restrict__ E,
                                   const int* __restrict__ lens, int T, int Tp, int H, int L, int R) {
  __shared__ float qe[QE_W];
  const int i = blockIdx.x, bh = blockIdx.y, len = lens[bh / H];
  const float* q = Q + ((size_t)bh * T + i) * 64;
  for (int d = threadIdx.x; d <= L + R; d += blockDim.x) {
    float s = 0.f;
    for (int k = 0; k < 64; ++k) s = fmaf(q[k], E[d * 64 + k], s);
    qe[d] = s * 0.125f;
  }
  __syncthreads();
  float* row = S + ((size_t)bh * T + i) * Tp;
  for (int j = threadIdx.x; j < T; j += blockDim.x) row[j] = j < len ? row[j] + qe[min(max(j - i, -L), R) + L] : -INFINITY;
}

}  // namespace

struct SemLayer {
  PackedW f1a, f1b, qkv, out, pw1, pw2, f2a, f2b;
  const float *ln1_w, *ln1_b, *lna_w, *lna_b, *lnc_w, *lnc_b, *dln_w, *dln_b, *ln2_w, *ln2_b, *fin_w, *fin_b;
  float* dw;       // [C][CM_KMAX] depthwise taps, left-padded with zeros
  float* E;        // [QE_W][64] distance_embedding rows, zero-padded
  __half* E16;     // the same in fp16 (the weight of the qe GEMM)
};
struct SemanticState {
  idx_semantic_config cfg;
  WeightPool pool;
  const float *fp_ln_w, *fp_ln_b;
  PackedW proj;
  std::vector<SemLayer> layers;
  float* half_col = nullptr;   // [hidden] of 0.5: the half-step residual of both FFNs (colscale)
  float* ident = nullptr;      // identity RoPE table [ident_T][32][2] = (1, 0): EPI_ROPE then only splits q | k | v
  int ident_T = 0;
};

void semantic_destroy(SemanticState* s) {
  if (!s) return;
  s->pool.release();
  delete s;
}

namespace {

// the encoder runs on fp16 tensor-core operands unless the engine is in strict fp32 mode
bool sem_half(const idx_engine* e) {
  static const bool no_tc = getenv("IDX_NO_TC") != nullptr;
  return e->gemm_backend == 0 && e->force_backend == 0 && !no_tc;
}

float* upload(WeightPool& pool, const std::vector<float>& h) {
  float* d = pool.alloc(h.size());
  IDX_CUDA(cudaMemcpy(d, h.data(), h.size() * 4, cudaMemcpyHostToDevice));
  return d;
}
std::vector<float> download(const idx_engine* e, const std::string& name, size_t n) {
  const DevTensor& t = e->W(name);
  IDX_CHECK(t.numel() == n, IDX_ERR_ARG, name + ": unexpected size");
  std::vector<float> h(n);
  IDX_CUDA(cudaMemcpy(h.data(), e->Wf(name), n * 4, cudaMemcpyDeviceToHost));
  return h;
}

void conv_module(idx_engine* e, const float* x, const int* lens, const SemLayer& l, float eps, float* y, __half* y16, int B,
                 int T, int C) {
  const size_t smem = (size_t)CM_ROWS * C * 4;
  if (smem > 48 * 1024 && !(e->attr_done & (1u << 23))) {
    IDX_CUDA(cudaFuncSetAttribute(conv_module_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    e->attr_done |= 1u << 23;
  }
  conv_module_kernel<<<dim3((T + CM_ROWS - 1) / CM_ROWS, B), 256, smem, e->stream>>>(x, lens, l.dw, l.dln_w, l.dln_b, eps, y,
                                                                                      y16, T, C);
  IDX_CUDA(cudaGetLastError());
  e->launches++;
}

size_t sem_arena_bytes(const idx_semantic_config& c, int B, int T, bool half) {
  const size_t BT = (size_t)B * T, C = c.hidden, H = c.heads, Tp = (T + 3) & ~3;
  size_t f = BT * c.feat_dim + BT * C * 2 + BT * std::max<size_t>(c.ffn, 3 * C) + BT * 2 * C + BT * 16 + B;
  size_t h = BT * c.feat_dim + BT * C + BT * std::max<size_t>(c.ffn, 3 * C);     // fp16 buffers (in floats: x 2 bytes / 4)
  if (half) f += H * BT * QE_W;
  else f += 2 * H * BT * 64 + H * B * 64 * Tp + H * BT * Tp + H * BT * 64;
  return 4 * f + 2 * h + 64 * 256 + (1 << 20);
}

// feats [B][T][feat_dim] (device), lens [B] (device) -> out [B][T][hidden] (device)
void encode_dev(idx_engine* e, SemanticState* s, const float* feats, const int* lens, int B, int T, float* out) {
  const idx_semantic_config& c = s->cfg;
  const int C = c.hidden, H = c.heads, BT = B * T, F = c.feat_dim;
  const bool half = sem_half(e);
  const float eps = c.eps;
  float* x = out;                                             // the residual stream lives in the output buffer
  float* hb = e->arena.get<float>((size_t)BT * C);            // LN output (strict) / attention output (strict)
  float* big = e->arena.get<float>((size_t)BT * std::max(c.ffn, 3 * C));
  float* pw = e->arena.get<float>((size_t)BT * 2 * C);        // pointwise_conv1 output
  __half* a16 = half ? (__half*)e->arena.alloc((size_t)BT * std::max(F, C) * 2) : nullptr;
  __half* big16 = half ? (__half*)e->arena.alloc((size_t)BT * std::max(c.ffn, 3 * C) * 2) : nullptr;
  float* fin = e->arena.get<float>((size_t)BT * F);
  // feature projection (modeling_wav2vec2_bert.py:125-130), then the encoder's entry mask (:491-493)
  layernorm(e, feats, half ? nullptr : fin, 1, BT, F, s->fp_ln_w, s->fp_ln_b, eps, nullptr, nullptr, 0, a16);
  conv_gemm(e, half ? gemm_of16(s->proj, a16, 1, BT, x) : gemm_of(s->proj, fin, 1, BT, x));
  mask_rows_kernel<<<dim3(T, B), 256, 0, e->stream>>>(x, lens, T, C);
  IDX_CUDA(cudaGetLastError());
  e->launches++;
  // attention buffers
  float* qe = nullptr;
  float *Q = nullptr, *K = nullptr, *Vt = nullptr, *S = nullptr, *O = nullptr;
  const int Tp = (T + 3) & ~3;
  if (half) {
    qe = e->arena.get<float>((size_t)H * BT * QE_W);
    if (s->ident_T < T) {                                     // identity table for EPI_ROPE, grown on demand
      std::vector<float> id((size_t)T * 64);
      for (size_t i = 0; i < id.size(); ++i) id[i] = (i & 1) ? 0.f : 1.f;
      s->ident = upload(s->pool, id);
      s->ident_T = T;
    }
  } else {
    Q = e->arena.get<float>((size_t)H * BT * 64);
    K = e->arena.get<float>((size_t)H * BT * 64);
    Vt = e->arena.get<float>((size_t)H * B * 64 * Tp);
    S = e->arena.get<float>((size_t)H * BT * Tp);
    O = e->arena.get<float>((size_t)H * BT * 64);
    if (Tp != T) fill_zero(e, Vt, (long long)H * B * 64 * Tp);
  }
  // x += 0.5 * FFN(LN x)
  auto ffn = [&](const float* lw, const float* lb, const PackedW& wa, const PackedW& wb) {
    if (half) {
      layernorm(e, x, nullptr, 1, BT, C, lw, lb, eps, nullptr, nullptr, 0, a16);
      { ConvGemm g = gemm_of16(wa, a16, 1, BT, big); g.act = ACT_SILU; conv_gemm(e, g); }
      to_half(e, big, big16, (long long)BT * c.ffn);
      { ConvGemm g = gemm_of16(wb, big16, 1, BT, x); g.res = x; g.colscale = s->half_col; conv_gemm(e, g); }
    } else {
      layernorm(e, x, hb, 1, BT, C, lw, lb, eps, nullptr, nullptr, 0);
      { ConvGemm g = gemm_of(wa, hb, 1, BT, big); g.act = ACT_SILU; conv_gemm(e, g); }
      { ConvGemm g = gemm_of(wb, big, 1, BT, x); g.res = x; g.colscale = s->half_col; conv_gemm(e, g); }
    }
  };
  for (const SemLayer& l : s->layers) {
    ffn(l.ln1_w, l.ln1_b, l.f1a, l.f1b);
    // x += MHA(LN x) with relative_key positions (:262-336)
    if (half) {
      layernorm(e, x, nullptr, 1, BT, C, l.lna_w, l.lna_b, eps, nullptr, nullptr, 0, a16);
      __half* Qr = big16;                                     // Qr | Kr | Vb [B*H][T][64] each
      {
        ConvGemm g = gemm_of16(l.qkv, a16, B, T, nullptr);
        g.epi = EPI_ROPE; g.out16 = Qr; g.aux = s->ident; g.aux_stride = H;
        g.scale = 0.125f * 1.4426950408889634f;              // 1/sqrt(64) and log2(e): the kernel's softmax is in 2^x
        conv_gemm(e, g);
      }
      {
        ConvGemm g;                                           // qe = Qr E^T, from the same fp16 q
        g.A16 = Qr; g.B = 1; g.Tin = H * BT; g.K = 64; g.Wk16 = l.E16; g.M = H * BT; g.N = QE_W; g.out = qe;
        conv_gemm(e, g);
      }
      const size_t n = (size_t)H * BT * 64;
      flash_attention_wgmma_relkey(e, Qr, Qr + n, Qr + 2 * n, qe, lens, c.left_max, c.right_max, a16, B, T, H);
      { ConvGemm g = gemm_of16(l.out, a16, 1, BT, x); g.res = x; conv_gemm(e, g); }
    } else {
      layernorm(e, x, hb, 1, BT, C, l.lna_w, l.lna_b, eps, nullptr, nullptr, 0);
      conv_gemm(e, gemm_of(l.qkv, hb, 1, BT, big));
      qkv_split_kernel<<<dim3(T, H, B), 64, 0, e->stream>>>(big, Q, K, Vt, T, Tp, H);
      IDX_CUDA(cudaGetLastError());
      e->launches++;
      ConvGemm g1;
      g1.A = Q; g1.B = H * B; g1.Tin = T; g1.K = 64; g1.Wk = K; g1.w_batch_stride = (long long)T * 64;
      g1.M = T; g1.N = T; g1.out = S; g1.ldo = Tp; g1.out_batch_stride = (long long)T * Tp; g1.scale = 0.125f;
      conv_gemm(e, g1);
      relkey_bias_kernel<<<dim3(T, H * B), 128, 0, e->stream>>>(S, Q, l.E, lens, T, Tp, H, c.left_max, c.right_max);
      IDX_CUDA(cudaGetLastError());
      e->launches++;
      softmax_rows_exact(e, S, (long long)H * BT, T, Tp);
      ConvGemm g2;
      g2.A = S; g2.B = H * B; g2.Tin = T; g2.K = Tp; g2.Wk = Vt; g2.w_batch_stride = (long long)64 * Tp;
      g2.M = T; g2.N = 64; g2.out = O;
      conv_gemm(e, g2);
      heads_merge(e, O, hb, B, T, H, 64);
      { ConvGemm g = gemm_of(l.out, hb, 1, BT, x); g.res = x; conv_gemm(e, g); }
    }
    // x += Conv(x) (:195-225): LN -> pointwise_conv1 -> fused GLU / masked causal depthwise / LN / swish -> pointwise_conv2
    if (half) {
      layernorm(e, x, nullptr, 1, BT, C, l.lnc_w, l.lnc_b, eps, nullptr, nullptr, 0, a16);
      conv_gemm(e, gemm_of16(l.pw1, a16, 1, BT, pw));
      conv_module(e, pw, lens, l, eps, nullptr, a16, B, T, C);
      { ConvGemm g = gemm_of16(l.pw2, a16, 1, BT, x); g.res = x; conv_gemm(e, g); }
    } else {
      layernorm(e, x, hb, 1, BT, C, l.lnc_w, l.lnc_b, eps, nullptr, nullptr, 0);
      conv_gemm(e, gemm_of(l.pw1, hb, 1, BT, pw));
      conv_module(e, pw, lens, l, eps, hb, nullptr, B, T, C);
      { ConvGemm g = gemm_of(l.pw2, hb, 1, BT, x); g.res = x; conv_gemm(e, g); }
    }
    ffn(l.ln2_w, l.ln2_b, l.f2a, l.f2b);
    layernorm(e, x, x, 1, BT, C, l.fin_w, l.fin_b, eps, nullptr, nullptr, 0);
  }
}

}  // namespace

extern "C" int idx_semantic_init(idx_engine* e, const idx_semantic_config* cfg) {
  IDX_API_BEGIN
  IDX_CHECK(e && cfg, IDX_ERR_ARG, "null argument");
  const idx_semantic_config& c = *cfg;
  IDX_CHECK(c.hidden > 0 && c.heads > 0 && c.hidden == 64 * c.heads, IDX_ERR_ARG, "idx_semantic_init: head size must be 64");
  IDX_CHECK(c.left_max >= 0 && c.right_max >= 0 && c.left_max + c.right_max + 1 <= QE_W, IDX_ERR_ARG,
            "idx_semantic_init: left_max + right_max + 1 must be <= 80");
  IDX_CHECK(c.feat_dim > 0 && c.feat_dim % 8 == 0 && c.hidden % 8 == 0 && c.ffn > 0 && c.ffn % 8 == 0 && c.layers >= 1,
            IDX_ERR_ARG, "idx_semantic_init: feat_dim, hidden and ffn must be positive multiples of 8, layers >= 1");
  IDX_CHECK(c.conv_kernel >= 1 && c.conv_kernel <= CM_KMAX, IDX_ERR_ARG, "idx_semantic_init: conv_kernel must be 1..31");
  IDX_CHECK(c.eps > 0.f, IDX_ERR_ARG, "idx_semantic_init: eps must be positive");
  IDX_CUDA(cudaSetDevice(e->device));
  semantic_destroy(e->semantic);
  e->semantic = nullptr;
  SemanticState* s = new SemanticState();
  e->semantic = s;
  s->cfg = c;
  const int C = c.hidden, KS = c.conv_kernel, NE = c.left_max + c.right_max + 1;
  const std::string P = "semantic.";
  s->fp_ln_w = e->Wf(P + "feature_projection.layer_norm.weight");
  s->fp_ln_b = e->Wf(P + "feature_projection.layer_norm.bias");
  s->proj = pack_linear(e, s->pool, P + "feature_projection.projection");
  s->half_col = upload(s->pool, std::vector<float>(C, 0.5f));
  const std::vector<float> mean = download(e, P + "semantic_mean", C), stdv = download(e, P + "semantic_std", C);
  for (int i = 0; i < c.layers; ++i) {
    const std::string p = P + "encoder.layers." + std::to_string(i) + ".";
    SemLayer l;
    l.f1a = pack_linear(e, s->pool, p + "ffn1.intermediate_dense");
    l.f1b = pack_linear(e, s->pool, p + "ffn1.output_dense");
    l.f2a = pack_linear(e, s->pool, p + "ffn2.intermediate_dense");
    l.f2b = pack_linear(e, s->pool, p + "ffn2.output_dense");
    l.qkv = pack3(e, s->pool, p + "self_attn.linear_q", p + "self_attn.linear_k", p + "self_attn.linear_v");
    l.out = pack_linear(e, s->pool, p + "self_attn.linear_out");
    l.pw1 = pack_linear(e, s->pool, p + "conv_module.pointwise_conv1");
    l.pw2 = pack_linear(e, s->pool, p + "conv_module.pointwise_conv2");
    IDX_CHECK(l.f1a.K == C && l.f1a.N == c.ffn && l.qkv.N == 3 * C && l.pw1.N == 2 * C && l.pw2.K == C && !l.pw1.bias &&
              !l.pw2.bias, IDX_ERR_ARG, p + ": weight shapes do not match the config");
    auto ln = [&](const std::string& n, const float** w, const float** b) {
      *w = e->Wf(p + n + ".weight");
      *b = e->Wf(p + n + ".bias");
    };
    ln("ffn1_layer_norm", &l.ln1_w, &l.ln1_b);
    ln("self_attn_layer_norm", &l.lna_w, &l.lna_b);
    ln("conv_module.layer_norm", &l.lnc_w, &l.lnc_b);
    ln("conv_module.depthwise_layer_norm", &l.dln_w, &l.dln_b);
    ln("ffn2_layer_norm", &l.ln2_w, &l.ln2_b);
    ln("final_layer_norm", &l.fin_w, &l.fin_b);
    {
      const std::vector<float> w = download(e, p + "conv_module.depthwise_conv.weight", (size_t)C * KS);
      std::vector<float> wp((size_t)C * CM_KMAX, 0.f);
      for (int ch = 0; ch < C; ++ch)
        for (int k = 0; k < KS; ++k) wp[(size_t)ch * CM_KMAX + CM_KMAX - KS + k] = w[(size_t)ch * KS + k];
      l.dw = upload(s->pool, wp);
    }
    {
      std::vector<float> E = download(e, p + "self_attn.distance_embedding.weight", (size_t)NE * 64);
      E.resize((size_t)QE_W * 64, 0.f);
      l.E = upload(s->pool, E);
      l.E16 = (__half*)s->pool.alloc((size_t)QE_W * 32);
      to_half(e, l.E, l.E16, (long long)QE_W * 64);
    }
    if (i == c.layers - 1) {
      // (LN(x) * w + b - mean) / std = LN(x) * (w / std) + (b - mean) / std
      std::vector<float> w = download(e, p + "final_layer_norm.weight", C), b = download(e, p + "final_layer_norm.bias", C);
      for (int j = 0; j < C; ++j) { w[j] /= stdv[j]; b[j] = (b[j] - mean[j]) / stdv[j]; }
      l.fin_w = upload(s->pool, w);
      l.fin_b = upload(s->pool, b);
    }
    for (PackedW* w : {&l.f1a, &l.f1b, &l.f2a, &l.f2b, &l.qkv, &l.out, &l.pw1, &l.pw2}) pack_half(e, s->pool, *w);
    s->layers.push_back(l);
  }
  pack_half(e, s->pool, s->proj);
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  IDX_API_END(e)
}

extern "C" int idx_semantic_encode(idx_engine* e, const float* feats, const int32_t* lens, int B, int T, float* out) {
  IDX_API_BEGIN
  SemanticState* s = e ? e->semantic : nullptr;
  IDX_CHECK(s, IDX_ERR_STATE, "idx_semantic_init has not been called");
  IDX_CHECK(feats && lens && out && B >= 1 && T >= 1, IDX_ERR_ARG, "idx_semantic_encode: bad arguments");
  IDX_CUDA(cudaSetDevice(e->device));
  std::vector<int32_t> hl(B);
  if (idx_is_device_ptr(lens)) {
    IDX_CUDA(cudaMemcpyAsync(hl.data(), lens, (size_t)B * 4, cudaMemcpyDeviceToHost, e->stream));
    IDX_CUDA(cudaStreamSynchronize(e->stream));
  } else {
    std::copy(lens, lens + B, hl.begin());
  }
  for (int b = 0; b < B; ++b)
    IDX_CHECK(hl[b] >= 1 && hl[b] <= T, IDX_ERR_ARG, "idx_semantic_encode: length " + std::to_string(hl[b]) + " of entry " +
                                                         std::to_string(b) + " is outside 1..T");
  const idx_semantic_config& c = s->cfg;
  const size_t nin = (size_t)B * T * c.feat_dim, nout = (size_t)B * T * c.hidden;
  e->ensure_arena(sem_arena_bytes(c, B, T, sem_half(e)) + 4 * (nin + nout) + 4 * (size_t)B + (1 << 20));
  e->arena.reset();
  float* d_in = e->arena.get<float>(nin);
  float* d_out = e->arena.get<float>(nout);
  int* d_lens = e->arena.get<int>(B);
  idx_to_device(e, d_in, feats, nin * 4);
  idx_to_device(e, d_lens, hl.data(), (size_t)B * 4);
  encode_dev(e, s, d_in, d_lens, B, T, d_out);
  idx_from_device(e, out, d_out, nout * 4);
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  IDX_API_END(e)
}

// Diagnostic entry (tests): the RELKEY flash attention alone (include/idxtts.h).
extern "C" int idx_debug_flash_attention_relkey(idx_engine* e, const uint16_t* q16, const uint16_t* k16, const uint16_t* v16,
                                                const uint16_t* E16, const int32_t* lens, int B, int T, int H, int left,
                                                int right, long long guard, uint16_t* out16) {
  IDX_API_BEGIN
  IDX_CHECK(e && q16 && k16 && v16 && E16 && lens && out16, IDX_ERR_ARG, "null argument");
  IDX_CHECK(B > 0 && T > 0 && H > 0 && left >= 0 && right >= 0 && left + right + 1 <= QE_W, IDX_ERR_ARG,
            "idx_debug_flash_attention_relkey: bad shape");
  IDX_CHECK(guard >= 0 && guard % 8 == 0, IDX_ERR_ARG, "idx_debug_flash_attention_relkey: guard must be a non-negative multiple of 8");
  for (int b = 0; b < B; ++b) IDX_CHECK(lens[b] >= 1 && lens[b] <= T, IDX_ERR_ARG, "idx_debug_flash_attention_relkey: bad length");
  IDX_CUDA(cudaSetDevice(e->device));
  const size_t n = (size_t)B * H * T * 64, ng = n + 2 * (size_t)guard, nq = (size_t)B * H * T * QE_W;
  e->ensure_arena(3 * 2 * n + 2 * ng + 4 * nq + 2 * QE_W * 64 + 4 * (size_t)B + (16 << 20));
  e->arena.reset();
  __half* dq = (__half*)e->arena.alloc(2 * n);
  __half* dk = (__half*)e->arena.alloc(2 * n);
  __half* dv = (__half*)e->arena.alloc(2 * n);
  __half* dE = (__half*)e->arena.alloc(2 * QE_W * 64);
  float* qe = e->arena.get<float>(nq);
  int* dl = e->arena.get<int>(B);
  __half* dOut16 = (__half*)e->arena.alloc(2 * ng);
  idx_to_device(e, dq, q16, 2 * n);
  idx_to_device(e, dk, k16, 2 * n);
  idx_to_device(e, dv, v16, 2 * n);
  IDX_CUDA(cudaMemsetAsync(dE, 0, 2 * QE_W * 64, e->stream));
  idx_to_device(e, dE, E16, 2 * (size_t)(left + right + 1) * 64);
  idx_to_device(e, dl, lens, 4 * (size_t)B);
  idx_to_device(e, dOut16, out16 - guard, 2 * ng);
  ConvGemm g;                                                 // qe = q E^T, as the encoder computes it
  g.A16 = dq; g.B = 1; g.Tin = B * H * T; g.K = 64; g.Wk16 = dE; g.M = B * H * T; g.N = QE_W; g.out = qe;
  conv_gemm(e, g);
  flash_attention_wgmma_relkey(e, dq, dk, dv, qe, dl, left, right, dOut16 + guard, B, T, H);
  idx_from_device(e, out16 - guard, dOut16, 2 * ng);
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  IDX_API_END(e)
}

// Diagnostic entry (tests): the fused conv-module kernel alone, each batch entry's rows staged between 8 NaN rows.
extern "C" int idx_debug_conv_module(idx_engine* e, const float* x, const int32_t* lens, const float* dw, const float* ln_w,
                                     const float* ln_b, float eps, int B, int T, int C, int kernel, long long guard,
                                     float* out, uint16_t* out16) {
  IDX_API_BEGIN
  IDX_CHECK(e && x && lens && dw && ln_w && ln_b && (out || out16), IDX_ERR_ARG, "null argument");
  IDX_CHECK(B > 0 && T > 0 && C > 0 && kernel >= 1 && kernel <= CM_KMAX, IDX_ERR_ARG, "idx_debug_conv_module: bad shape");
  IDX_CHECK(guard >= 0 && guard % 8 == 0, IDX_ERR_ARG, "idx_debug_conv_module: guard must be a non-negative multiple of 8");
  for (int b = 0; b < B; ++b) IDX_CHECK(lens[b] >= 1 && lens[b] <= T, IDX_ERR_ARG, "idx_debug_conv_module: bad length");
  IDX_CUDA(cudaSetDevice(e->device));
  constexpr int G = 8;
  const size_t row = 2 * (size_t)C, per = (size_t)(T + 2 * G) * row, no = (size_t)B * T * C, g2 = 2 * (size_t)guard;
  e->ensure_arena(4 * (B * per + (size_t)C * CM_KMAX + 2 * (size_t)C + B) + 6 * (no + g2) + (16 << 20));
  e->arena.reset();
  // [B][G NaN rows | T rows | G NaN rows][2C]; the kernel sees the T rows of each entry through a [B][T + 2G] view
  float* dx = e->arena.get<float>(B * per);
  IDX_CUDA(cudaMemsetAsync(dx, 0xFF, B * per * 4, e->stream));
  for (int b = 0; b < B; ++b) idx_to_device(e, dx + b * per + G * row, x + (size_t)b * T * row, (size_t)T * row * 4);
  std::vector<float> wp((size_t)C * CM_KMAX, 0.f);
  for (int ch = 0; ch < C; ++ch)
    for (int k = 0; k < kernel; ++k) wp[(size_t)ch * CM_KMAX + CM_KMAX - kernel + k] = dw[(size_t)ch * kernel + k];
  SemLayer l;
  l.dw = e->arena.get<float>(wp.size());
  float* dlw = e->arena.get<float>(C);
  float* dlb = e->arena.get<float>(C);
  int* dl = e->arena.get<int>(B);
  idx_to_device(e, l.dw, wp.data(), wp.size() * 4);
  idx_to_device(e, dlw, ln_w, (size_t)C * 4);
  idx_to_device(e, dlb, ln_b, (size_t)C * 4);
  l.dln_w = dlw; l.dln_b = dlb;
  float* dOut = out ? e->arena.get<float>(no + g2) : nullptr;
  __half* dOut16 = out16 ? (__half*)e->arena.alloc((no + g2) * 2) : nullptr;
  if (dOut) idx_to_device(e, dOut, out - guard, (no + g2) * 4);
  if (dOut16) idx_to_device(e, dOut16, out16 - guard, (no + g2) * 2);
  // one launch per entry: entry b reads its own staged block (rows before 0 / past T would be NaN)
  idx_to_device(e, dl, lens, (size_t)B * 4);
  for (int b = 0; b < B; ++b) {
    conv_module(e, dx + b * per + G * row, dl + b, l, eps, dOut ? dOut + guard + (size_t)b * T * C : nullptr,
                dOut16 ? dOut16 + guard + (size_t)b * T * C : nullptr, 1, T, C);
  }
  if (dOut) idx_from_device(e, out - guard, dOut, (no + g2) * 4);
  if (dOut16) idx_from_device(e, out16 - guard, dOut16, (no + g2) * 2);
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  IDX_API_END(e)
}
