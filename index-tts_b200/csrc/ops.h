// ops.h — generic building blocks shared by the vocoder / s2mel / codec paths.
// Activations are channels-last fp32: a [B][T][C] tensor is a row-major [B*T, C] matrix whose
// rows are time steps, so every Conv1d / Linear is a (multi-tap) GEMM with K = C contiguous.
#pragma once
#include "engine.h"
#include <cuda_fp16.h>
#include <cstdlib>
#include <string>
#include <utility>
#include <vector>

enum { EPI_NONE = 0, EPI_SWIGLU = 1, EPI_WNGATE = 2, EPI_ROPE = 3 };
enum { ACT_NONE = 0, ACT_GELU_ERF = 1, ACT_SILU = 2, ACT_MISH = 3, ACT_GELU_TANH = 4, ACT_RELU = 5 };
// the scale EPI_ROPE applies to q for the wgmma flash attention: 1/sqrt(64), times log2(e) because its softmax is in 2^x
constexpr float FLASH_Q_SCALE = 0.125f * 1.4426950408889634f;

// D[b][m][j] = epi( sum_{tap} sum_{k} A[b][m + tap*dil - pad][k] * W[tap][k][j] )
// rows of A outside [0, Tin) read as zero (Conv1d zero padding) or are reflected (SConv1d).
struct ConvGemm {
  const float* A = nullptr;   // [B][Tin][K]
  int B = 1, Tin = 0, K = 0;
  long long a_batch_stride = 0;  // elements; 0 → Tin*K
  int a_bcast = 0;               // 1 → every batch entry reads the same A (stride 0)
  int lda = 0;                   // row stride of A in elements; 0 → K
  const float* W = nullptr;   // [taps][K][N]  (N contiguous)  — SIMT layout
  const float* Wk = nullptr;  // [N][taps*K]   (K contiguous)  — tensor-core layout (optional)
  // fp16 operand path (wgmma .f16): both set -> the tensor-core kernel reads these instead of A / Wk (same shapes,
  // strides given in ELEMENTS as for the fp32 operands).  Written by the producing kernel of A / converted once at init.
  const __half* A16 = nullptr;
  const __half* Wk16 = nullptr;
  // fused pair epilogues of the tensor-core kernel (fp16 results straight into the operand of the next GEMM / the attention):
  //   EPI_SWIGLU : columns (2j, 2j+1) = (w1 x, w3 x)_j (weight rows interleaved at pack time) -> out16[row][j] = silu(a) * b
  //   EPI_WNGATE : columns (2j, 2j+1) = (a_j, c_j) of the WaveNet in_layer -> out16[row][j] = tanh(a + g[b][j]) * sigmoid(c + g[b][N/2 + j])
  //   EPI_ROPE   : columns = q | k | v of the fused wqkv: interleaved-pair RoPE (table aux [T][32][2]) on q (x scale) and k, v as is,
  //                written head-major as fp16 Qr | Kr | Vb [B*H][T][64] (out16 = Qr; the three tensors are contiguous)
  int epi = 0;
  __half* out16 = nullptr;
  const float* aux = nullptr;      // EPI_WNGATE: g [B][aux_stride] ; EPI_ROPE: rope table
  int aux_stride = 0;              // EPI_WNGATE: floats per batch entry of g ; EPI_ROPE: heads
  long long w_batch_stride = 0;  // elements between the Wk matrices of consecutive batch entries (0: shared)
  int ldw = 0;                   // row stride of Wk in elements; 0 → taps*K
  int taps = 1, dil = 1, pad = 0, reflect = 0;
  int M = 0;                  // output rows per batch
  int N = 0;
  const float* bias = nullptr;
  int biasN = 0;              // bias index = j % biasN (0 → N)
  int act = ACT_NONE;
  const float* res = nullptr;   // optional residual, indexed like out
  const float* rowscale = nullptr;  // optional per-(b,m) multiplier (masks), [B][M]
  const float* colscale = nullptr;  // optional per-column multiplier applied to (acc+bias) (layer scale)
  int accum = 0;              // out = scale * (v + out_old)
  float scale = 1.f;
  float* out = nullptr;
  long long out_batch_stride = 0;  // elements; 0 → M*N
  long long out_off = 0;           // flat offset added to m*ldo + j (may be negative: ConvTranspose)
  long long out_valid = 0;         // writes only where 0 <= flat < out_valid (0 → M*ldo)
  int ldo = 0;                     // 0 → N
};

void conv_gemm(idx_engine* e, const ConvGemm& g);
inline int gemm_default_backend(const idx_engine* e) { return e->gemm_backend; }   // 0 auto (wgmma), 1 SIMT fp32

// [B][C][T] <-> [B][T][C]
void transpose_bct_to_btc(idx_engine* e, const float* in, float* out, int B, int C, int T);
void transpose_btc_to_bct(idx_engine* e, const float* in, float* out, int B, int T, int C);

// ------------------------------------------------------------- programmatic dependent launch --
// The tail is ~4000 short kernels per utterance.  Kernels launched through launch_pdl() carry the programmatic-stream-
// serialization attribute: their CTAs may be scheduled while the previous kernel of the stream is still draining, so launch
// latency and the kernel's own prologue (barrier init, descriptor prefetch) overlap with it.  Such a kernel
// executes pdl_wait() — every thread — before it touches global memory, and pdl_trigger() as soon as it has nothing left that
// the NEXT kernel could disturb (the next kernel's own pdl_wait still waits for this grid to finish completely).
#ifdef __CUDACC__
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
template <typename... KArgs, typename... Args>
inline void launch_pdl(idx_engine* e, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, Args&&... args) {
  static const bool off = getenv("IDX_PDL") && atoi(getenv("IDX_PDL")) == 0;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = e->stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = off ? 0 : 1;
  IDX_CUDA(cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...));
}
#endif

// ---------------------------------------------------------------- normalisation / pointwise --
// y = LayerNorm(x) [* w + b] [ * (1 + scale[b]) + shift[b] ]   rows of C, x/y [B][T][C]
void layernorm(idx_engine* e, const float* x, float* y, int B, int T, int C, const float* w,
               const float* b, float eps, const float* scale, const float* shift, int mod_stride, __half* y16 = nullptr);
// y = mw[b] * (x * rsqrt(mean(x^2)+eps) * nw) + mb[b]          (AdaptiveLayerNorm over RMSNorm)
void rmsnorm_adaln(idx_engine* e, const float* x, float* y, int B, int T, int C, const float* nw,
                   const float* mw, const float* mb, int mod_stride, float eps, __half* y16 = nullptr);
// GroupNorm(1 group) over each sample's [T][C] block, affine per channel, followed by Mish
void groupnorm1_mish(idx_engine* e, const float* x, float* y, int B, int T, int C, const float* w,
                     const float* b, float eps);
// depthwise Conv1d (groups = C), zero padding (k-1)/2; w [C][k]
void dwconv1d(idx_engine* e, const float* x, float* y, int B, int T, int C, const float* w,
              const float* b, int k);
// y[b][t][:] = x[b][src(t)][:], src(t) = min(floor(t * Tin/Tout), Tin-1)  (F.interpolate nearest)
void nearest_interp(idx_engine* e, const float* x, float* y, int B, int Tin, int Tout, int C);
// out[t][:] = table[ids[t]][:]
void embedding_rows(idx_engine* e, const float* table, const int* ids, float* out, int n, int C, int nrows);
// y = silu(a) * b where ab [rows][2*N] holds a | b side by side
void swiglu(idx_engine* e, const float* ab, float* y, long long rows, int N);
// y = tanh(a + ga[b]) * sigmoid(c + gc[b]),  xin [B][T][2N] = a | c ; g [B][*] with stride
void wn_gate(idx_engine* e, const float* xin, const float* g, int g_stride, float* y, int B, int T, int N);
// copy a [rows][C] block into columns [col0, col0+C) of a [rows][ldo] matrix (concat by columns)
void copy_cols(idx_engine* e, const float* src, int lds, float* dst, int ldo, int col0, long long rows, int C, __half* dst16 = nullptr);
// broadcast a per-batch vector [B][C] over T rows into columns of dst
void bcast_cols(idx_engine* e, const float* vec, float* dst, int ldo, int col0, int B, int T, int C);
// y = silu(x)
void silu_inplace(idx_engine* e, float* x, long long n);
// RoPE table [T][hd/2][2] (cos, sin), base 1e4 (gpt_fast/model.py:336-346)
void rope_table(idx_engine* e, float* tab, int T, int hd);
// full (non-causal) attention with interleaved-pair RoPE on q,k: the wgmma flash attention on fp16 q / k / v (gemm_backend 0)
// or the fp32 SIMT kernel (gemm_backend 1).  qkv [B][T][3*H*64] (q | k | v), out [B][T][H*64]
void attention_rope(idx_engine* e, const float* qkv, float* out, int B, int T, int H, const float* rope);
// x[b][t][c] (+)= ... CFG + Euler: x += dt * ((1+r) * v[0] - r * v[1]); rows t < P zeroed. x,v: [T][C]
void cfg_euler(idx_engine* e, float* x, const float* v_cond, const float* v_uncond, float dt, float rate,
               int T, int C, int P);
void fill_zero(idx_engine* e, float* x, long long n);
// restores the engine's diagnostic overrides (force_backend, force_tile_n) however a debug entry leaves
struct DebugOverrides {
  idx_engine* e;
  ~DebugOverrides() { e->force_backend = 0; e->force_tile_n = 0; }
};
// y[b][i][:] = x[b][reflect(i - left)][:], i in [0, T + left + right)   (encodec.py pad1d mode='reflect': F.pad's reflection,
// with an input no longer than max(left, right) zero-extended to max(left, right) + 1 rows first)
void reflect_pad_rows(idx_engine* e, const float* x, float* y, int B, int T, int C, int left, int right, __half* y16 = nullptr);

// ------------------------------------------------------------------------ packed weights --
struct PackedW {
  float* wsimt = nullptr;  // [taps][K][N]
  float* wk = nullptr;     // [N][taps*K]
  __half* wk16 = nullptr;  // [N][taps*K] fp16 copy of wk (made on demand by pack_half)
  const float* bias = nullptr;
  int N = 0, K = 0, taps = 1, dil = 1;
};
struct WeightPool {
  std::vector<void*> owned;
  float* alloc(size_t n);
  void release();
};
// nn.Linear weight [N][K] (optionally only rows [row0, row0+rows))
PackedW pack_linear(idx_engine* e, WeightPool& pool, const std::string& name, int row0 = 0, int rows = -1,
                    bool with_bias = true);
// nn.Conv1d weight [Co][Ci][k] (optionally only output rows [row0, row0+rows))
PackedW pack_conv1d(idx_engine* e, WeightPool& pool, const std::string& name, int dil = 1, int row0 = 0,
                    int rows = -1);
// convenience: D = A·W^T (+bias) for a channels-last activation with optional epilogue fields preset in g
ConvGemm gemm_of(const PackedW& w, const float* A, int B, int T, float* out);
// same GEMM with fp16 operands: A16 is the fp16 image of the activation (the fp32 pointer may be null)
ConvGemm gemm_of16(const PackedW& w, const __half* A16, int B, int T, float* out);
// fp16 copy of a K-major weight matrix (w.wk must exist); idempotent
void pack_half(idx_engine* e, WeightPool& pool, PackedW& w);
// fp16 K-major copy of w.wk with the two halves of the output rows interleaved (row 2j = row j, row 2j+1 = row N/2 + j): the
// weight layout of the EPI_SWIGLU / EPI_WNGATE pair epilogues; bias_out (optional) receives the bias interleaved the same way
__half* pack_half_interleaved(idx_engine* e, WeightPool& pool, const PackedW& w, float** bias_out);
// the fused flash attention on already rotated / split fp16 tensors Qr | Kr | Vb [B*H][T][64] (what EPI_ROPE writes), on
// wgmma (gemm_tc.cu: S and O in registers, P fed back as a register operand)
void flash_attention_wgmma(idx_engine* e, const __half* Qr, const __half* Kr, const __half* Vb, float* out, __half* out16,
                           int B, int T, int H);
// ------------------------------------------------------------------- packed sequences --
// Sequences of different lengths packed along T (the batched CFM solve): segment u owns rows [off[u], off[u+1]) of every
// batch entry.  segments_upload() puts the offsets and the query-tile list of the varlen flash attention on the device
// (arena memory, one upload per packed solve).
struct Segments {
  std::vector<int> off;            // o_0 = 0 .. o_n = total rows
  int* d_off = nullptr;            // device copy of off
  int4* d_fa_tiles = nullptr;      // (first query row, segment start, segment end) of every 128-row query tile
  int fa_tiles = 0;
  int n() const { return (int)off.size() - 1; }
  int total() const { return off.back(); }
  int len(int u) const { return off[u + 1] - off[u]; }
};
void segments_upload(idx_engine* e, Segments& sg);
// flash_attention_wgmma over packed sequences: attention never crosses a segment boundary (see fa_wgmma_kernel)
void flash_attention_wgmma_varlen(idx_engine* e, const __half* Qr, const __half* Kr, const __half* Vb, float* out, __half* out16,
                                  int B, int H, const Segments& sg);
// reflect_pad_rows per segment into a gapped layout: segment u's padded frame of len(u) + left + right rows starts at row
// off[u] + u * (left + right) of each batch entry [B][total + n * (left + right)][C] (fp16 only)
void reflect_pad_segments(idx_engine* e, const float* x, __half* y16, int B, int C, int left, int right, const Segments& sg);
// undo the gaps: y[b][off[u] + t] = x[b][off[u] + u * gap + t], x [B][total + n * gap - gap][C] fp16 (the rows a
// multi-tap GEMM over the gapped layout produces), y [B][total][C]
void compact_segments16(idx_engine* e, const __half* x, __half* y, int B, int C, int gap, const Segments& sg);
// rope_table per segment: segment u's positions restart at 0 in rows [off[u], off[u+1]) of tab [total][hd/2][2]
void rope_table_segments(idx_engine* e, float* tab, const Segments& sg, int hd);
// cfg_euler with the rows listed in zero_rows (1 = prompt frame of its segment) zeroed
void cfg_euler_rows(idx_engine* e, float* x, const float* v_cond, const float* v_uncond, float dt, float rate, int T, int C,
                    const unsigned char* zero_rows);
// the unfused fp32 attention (emotion conformer, strict w2v-BERT encoder): exact-exp softmax over the first T of Tp columns of
// each row (columns T..Tp-1 zeroed), and O [B*H][T][dk] -> out [B][T][H*dk]
void softmax_rows_exact(idx_engine* e, float* S, long long rows, int T, int Tp);
void heads_merge(idx_engine* e, const float* O, float* out, int B, int T, int H, int dk);
// the wgmma flash attention with w2v-BERT's relative_key positions and a key-length mask (see fa_wgmma_kernel, RELKEY):
// qe [B*H][T][80] = Qr E^T (fp32), lens [B] valid keys (device); out16 [B][T][H*64]
void flash_attention_wgmma_relkey(idx_engine* e, const __half* Qr, const __half* Kr, const __half* Vb, const float* qe,
                                  const int* lens, int rel_l, int rel_r, __half* out16, int B, int T, int H);
// q | k | v Linears of one attention stacked into one [3*od][K] weight with its bias
PackedW pack3(idx_engine* e, WeightPool& pool, const std::string& a, const std::string& b, const std::string& c);
// fp32 -> fp16 (round to nearest), n elements
void to_half(idx_engine* e, const float* x, __half* y, long long n);
// true when the engine runs the tail with fp16 GEMM operands (gemm_backend 0 and tail_f16 1)
bool tail_half(const idx_engine* e);
