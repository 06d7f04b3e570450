// gpt_decode.cu — the autoregressive speech-token path of UnifiedVoice as ONE persistent
// sm_90a kernel per group of decode steps.
//
// Replaces, for the v2/v2.5 GPT (SURVEY.md §8a rows a2–a6):
//   GPT2InferenceModel.forward            indextts/gpt/model_v2.py:121-198
//   stock HF GPT2Model/Block/Attention/MLP indextts/gpt/transformers_gpt2.py:189-227,571-667
//   lm_head = Sequential(final_norm, mel_head) model_v2.py:54,408-410   (double LayerNorm, P3)
//   GenerationMixin._sample greedy loop     transformers_generation_utils.py:3123-3297
//   RepetitionPenaltyLogitsProcessor        (transformers.generation.logits_process)
//
// Design (batch-1 decode is pure weight streaming — 965.6 MB bf16 per token):
//   * one CTA per SM (cooperative launch), 8 compute warps + 1 producer warp;
//   * every CTA owns a fixed slice of output columns of every GEMV phase; its weights for
//     ALL layers/phases are pre-packed into one contiguous byte stream in consumption order,
//     so the producer warp streams it with cp.async.bulk (UBLKCP) into a shared-memory ring,
//     completely decoupled from the grid barriers — HBM stays busy while the SMs sit at a
//     barrier or run the tiny attention / LayerNorm / sampling phases;
//   * 5 grid barriers per layer (QKV | attention | O-proj+res | FC+gelu | proj+res), head,
//     sampling; repetition penalty, argmax, stop check and the next-token embedding happen on
//     the device, the host polls one flag per launch (no per-step D2H sync);
//   * prefill reuses the same kernel: a "step" is then a tile of up to B_TILE consecutive
//     prompt positions of one sequence (causality falls out of the KV-cache position bound).
//
// Numerics follow the reference's bf16 path (infer_v2_5.py:143-146,758 — weights .bfloat16()
// under autocast): bf16 weights, fp32 accumulation, and a round-to-bf16 at every point where
// autocast materialises a bf16 tensor (after each Conv1D/Linear, after each elementwise op of
// NewGELUActivation); LayerNorm is fp32 in / fp32 out; the residual stream is fp32 (the fp32
// zeros of null_position_embeddings promote it, model_v2.py:23-24 — trap P12); logits are bf16
// values upcast to fp32 (P5).  See DESIGN.md "GPT numerics".
#include "engine.h"
#include "ops.h"
#include "ptx.cuh"
#include <cooperative_groups.h>
#include <algorithm>
#include <cstring>
#include <cmath>
#include <type_traits>

namespace {

constexpr int NCW = 8;                      // compute warps
constexpr int NCT = NCW * 32;               // compute threads
constexpr int NTHREADS = NCT + 32;          // + producer warp
constexpr int UPC = 8;                      // weight units (one K-segment of D bf16) per chunk
constexpr int MAXPL = 40;                   // max LayerNorm elements per lane (D <= 1280)
constexpr int HD = 64;                      // head dim (fixed)
constexpr int PART_STRIDE = 66;             // attention partial: m, l, o[64]
constexpr int CMAX = 128;                   // candidates the samplers keep after TopK (1 <= top_k <= CMAX, checked by the host)
#define RED_FLOATS(BT) (((BT) == 1 ? 7 * NCW * 8 : 2 * NCW * 64) > (NCW * PART_STRIDE) ? ((BT) == 1 ? 7 * NCW * 8 : 2 * NCW * 64) : (NCW * PART_STRIDE))

struct PrefillTile {
  int seq, pos0, nrows, src_row;
};

struct GptParams {
  int L, D, H, V, FF, G;
  int B;            // valid rows this launch (<= B_TILE)
  int mode;         // 0 prefill tiles, 1 decode
  int nsteps;       // steps (or tiles) in this launch
  int step0;        // decode: global index of the first step of this launch
  int max_new;      // decode: max tokens per sequence
  int start_tok, stop_tok, forbid_stop_before;
  float rep_penalty;
  int do_sample, top_k;       // do_sample: temperature -> top-k -> top-p -> multinomial (HF warper order)
  float top_p, temperature;
  unsigned long long seed;
  int round_bf16;   // 1: emulate autocast bf16 rounding points
  int nst;          // ring stages
  int bar_flavor;   // 0: fence after the grid barrier, 1: none (consumers use ld.cg)
  int bias_cap;     // floats reserved for the per-CTA bias table
  int ocap;         // max O-proj columns per CTA
  // packed weights
  const __nv_bfloat16* wstream;   // all CTA streams
  const long long* stream_off;    // [G] unit offset of CTA i's stream
  // small fp32 parameters
  const float *ln1_w, *ln1_b, *ln2_w, *ln2_b;      // [L][D]
  const float *qkv_b, *o_b, *fc_b, *proj_b;        // [L][3D],[L][D],[L][FF],[L][D]
  const float *lnf_w, *lnf_b, *fn_w, *fn_b, *head_b;
  const float *mel_emb, *mel_pos;                  // [V][D], [P][D]  (f32 masters)
  // KV cache [L][nseq][maxpos][D] bf16
  __nv_bfloat16 *kc, *vc;
  int nseq, maxpos;
  // activations (global, L2 resident)
  float* xg;            // [8][D]   residual stream
  float* qg;            // [8][D]   q of the current layer
  __nv_bfloat16* fg;    // [8][FF]  gelu(fc) of the current layer
  float* part;          // [B*H*nsplit][66] attention partials
  float* logits;        // [8][V]
  // per-sequence state
  int* tok;             // [8] token to feed next
  int* nout;            // [8] tokens generated so far
  int* finished;        // [8]
  int* prompt_len;      // [8]
  unsigned* seen;       // [8][ceil(V/32)] repetition-penalty bitmap
  int* codes;           // [8][max_new]
  const int* forced;    // [8][max_new] or null
  float* logits_dump;   // [8][max_new][V] or null
  int* done;            // [1] all sequences finished
  int* flag;            // engine error word: set to step + 1 when more than CMAX tokens tie at the top-k boundary
  // prefill
  const float* prompt;  // [rows][D] f32
  float* hidden_out;    // prefill only, optional: [rows][D] residual stream after the last block (v1 latent pass)
  const PrefillTile* tiles;
  unsigned* barrier;    // grid barrier counter (zeroed before each launch)
  // tag-in-data dataflow for the residual stream (batch-1 decode): x[c] travels as {value, epoch} in one 8-byte word
  // (the NCCL LL idea), consumers poll the words instead of waiting at a grid barrier
  uint2* xt;            // [D] tagged residual stream, or null: grid barriers everywhere
  unsigned* ft;         // [FF] gelu(fc) as {bf16 value, 16-bit tag} words (same mode)
  unsigned* pflag;      // [B*H*nsplit] epoch of the attention partial of each (row, head, key split)
  uint2* qt;            // [D] tagged q of the current layer
  uint2* kvt;           // [2][D] tagged k, v (bf16-valued) of the position being decoded
  unsigned epoch0;      // first epoch of this launch (2 per layer per step)
  int seq_base;         // global index of row 0 (requests beyond one decode group run as consecutive groups)
  int pos_plain;        // 1: mel position k at step k (decoding without a cache, infer.py:101); 0: trap P1 (k + 1)
  // beam search (beam_step_kernel runs between single-step launches)
  int ext_sample;       // 1: leave the logits in p.logits and skip the sampling phase
  int beams;            // rows per utterance (also set for the beam driver's prefill launch: the prefill probe's request index)
  int phys_stride;
  const unsigned char* phys;   // [8][phys_stride]: cache slot of generated position t of row b's lineage, or null
  long long* prof;      // optional: globaltimer stamps of CTA 0 for the last step of the launch
  // second-generation batch-1 decode kernel (gpt_decode1.cuh)
  const __nv_bfloat16* wstream1;  // per-CTA row streams in tile order
  const long long* stream_off1;   // [G] row offset of CTA i's stream
  int ring_rows;                  // R: rows of D bf16 in the shared-memory ring
  int dbg;                        // diagnostics (IDX_GPT_DBG): 1 skip the MMA loops, 2 skip the attention key loop, 4 do not wait in polls
  uint2* ot;                      // [D] tagged normalised attention output (one CTA per head)
  uint2* partt;                   // [H * 7][66] tagged (m, l, o) partials (long contexts: key splits)
  uint2* cand;                    // [G][2] tagged per-CTA argmax candidate (score, index) / sampling flags
  uint2* tokt;                    // [1] tagged sampled token
  long long* prof2;     // optional: [G][64] fine globaltimer stamps of every CTA for layer prof2_layer of the last step
  int prof2_layer;
  // attention probe (idx_gpt_probe_attention for decode launches, idx_gpt_probe_prefill for prefill launches), null when disarmed
  float* probe;         // decode: [max_new][probed layers][probe_seqs][2][D]; prefill: [probe_seqs][probe_rows][probed layers][2][D]
                        // (q as the attention reads it | normalised attention output)
  int* probe_ns;        // decode: [max_new][probed layers]: key splits of the step
  int probe_layer;      // the probed layer, -1: all layers
  int probe_seqs;
  int probe_rows;       // prefill: prompt positions per request
};

// Probe slot of (decode step k, layer l), or -1 when the probe is disarmed or does not record layer l
__device__ __forceinline__ long long probe_slot(const GptParams& p, int k, int l) {
  if (!p.probe || (p.probe_layer >= 0 && l != p.probe_layer)) return -1;
  return p.probe_layer >= 0 ? (long long)k : (long long)k * p.L + l;
}

// gpt_fused_kernel: probe record ([0] = q, [1] = attention output: 2 * D floats) of row b at the first probed layer, or null.
// Decode: row b of step k.  Prefill: prompt position `pos` of the request whose first cache slot is `seq` (beam search:
// seq / beams).  fused_probe_at moves it to layer l (null when l is not probed).
__device__ __forceinline__ float* fused_probe_row(const GptParams& p, int k, int b, int seq, int pos) {
  const long long D2 = 2LL * p.D;
  if (p.mode == 1) return p.probe + (probe_slot(p, k, max(p.probe_layer, 0)) * p.probe_seqs + b) * D2;
  const int nl = p.probe_layer >= 0 ? 1 : p.L, req = p.beams > 1 ? seq / p.beams : seq;
  return p.probe + ((long long)req * p.probe_rows + pos) * nl * D2;
}
__device__ __forceinline__ float* fused_probe_at(const GptParams& p, float* row, int l) {
  if (p.probe_layer >= 0) return l == p.probe_layer ? row : nullptr;
  return row + (long long)l * 2 * p.D * (p.mode == 1 ? p.probe_seqs : 1);
}

__device__ __forceinline__ float bf16r(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }
__device__ __forceinline__ float rnd(float v, int on) { return on ? bf16r(v) : v; }
__device__ __forceinline__ float lo_bf(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float hi_bf(uint32_t v) { return __uint_as_float(v & 0xffff0000u); }

__device__ __forceinline__ long long gtimer() {
  long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

// Philox4x32-10 (Salmon et al.), counter = (step, sequence, 0, 0), key = seed.  The device sampler's
// RNG contract (documented in DESIGN.md): NOT bit-compatible with torch.multinomial's stream.
__device__ __forceinline__ void philox4x32_10(unsigned long long seed, unsigned c0, unsigned c1, unsigned (&out)[4]) {
  unsigned k0 = (unsigned)seed, k1 = (unsigned)(seed >> 32);
  unsigned x0 = c0, x1 = c1, x2 = 0u, x3 = 0u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const unsigned long long p0 = (unsigned long long)0xD2511F53u * x0;
    const unsigned long long p1 = (unsigned long long)0xCD9E8D57u * x2;
    const unsigned n0 = (unsigned)(p1 >> 32) ^ x1 ^ k0;
    const unsigned n1 = (unsigned)p1;
    const unsigned n2 = (unsigned)(p0 >> 32) ^ x3 ^ k1;
    const unsigned n3 = (unsigned)p0;
    x0 = n0; x1 = n1; x2 = n2; x3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  out[0] = x0; out[1] = x1; out[2] = x2; out[3] = x3;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(ptx::smem_u32(smem_dst)), "l"(gsrc)
               : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
// 16-byte copy that writes zeros when !valid (src-size 0; the address must still be a valid one)
__device__ __forceinline__ void cp_async16_zfill(void* smem_dst, const void* gsrc, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(ptx::smem_u32(smem_dst)), "l"(gsrc), "r"(valid ? 16 : 0)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait_group() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ unsigned ld_relaxed_gpu(const unsigned* p) {
  unsigned v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

__device__ __forceinline__ void st_tagged(uint2* p, float v, unsigned epoch) {
  asm volatile("st.relaxed.gpu.global.v2.u32 [%0], {%1, %2};" ::"l"(p), "r"(__float_as_uint(v)), "r"(epoch) : "memory");
}
// Poll N tagged words together (thread-strided slice of x): all loads of one round are in flight at once, so a
// round costs one L2 round trip; repeat until every word carries `epoch`.
// 8-byte aligned vector accesses are single-copy atomic on the hardware (the NCCL LL protocol relies on the same).
template <int N>
__device__ __forceinline__ void ld_tagged_slice(const uint2* base, int first, unsigned epoch, float (&v)[N], bool nowait = false) {
  unsigned val[N], tag[N], spins = 0;
  bool ok;
  do {
#pragma unroll
    for (int j = 0; j < N; ++j)
      asm volatile("ld.relaxed.gpu.global.v2.u32 {%0, %1}, [%2];" : "=r"(val[j]), "=r"(tag[j]) : "l"(base + first + 32 * j) : "memory");
    ok = true;
#pragma unroll
    for (int j = 0; j < N; ++j) ok &= (tag[j] == epoch);
    if (++spins > (1u << 26)) __trap();
  } while (!ok && !nowait);
#pragma unroll
  for (int j = 0; j < N; ++j) v[j] = __uint_as_float(val[j]);
}

// Grid-wide barrier among the compute warps of all CTAs (monotonic counter).  All cross-CTA
// data is read with ld.global.cg (L2), so no L1 invalidation is needed on the consumer side.
// Every thread also drains its cp.async prefetches (LayerNorm parameters of the next phase)
// before the closing CTA barrier, so they are visible to the whole CTA afterwards.
__device__ __forceinline__ void st_release_gpu(unsigned* p, unsigned v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void grid_sync(unsigned* ctr, unsigned& target, int G, int flavor) {
  ptx::named_bar_sync(1, NCT);
  if (flavor == 2) {
    // flag barrier: one arrival word per CTA (no same-address atomics, which L2 serialises at
    // ~27 cycles each: one arrival per SM on one counter costs ~2 us), polled by the 32 lanes of warp 0.
    if (threadIdx.x < 32) {
      unsigned* flags = ctr + 32;
      target += 1u;
      if (threadIdx.x == 0) st_release_gpu(flags + blockIdx.x, target);   // cumulative over the CTA (bar.sync above)
      unsigned spins = 0;
      for (int i = threadIdx.x; i < G; i += 32) {
        while (ld_relaxed_gpu(flags + i) < target) {
          if (++spins > (1u << 28)) __trap();
        }
      }
      __syncwarp();
    }
  } else if (threadIdx.x == 0) {
    target += (unsigned)G;
    if (flavor == 3) {
      // release-reduction: no returned value to wait for, release ordering instead of a separate fence
      asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(ctr), "r"(1u) : "memory");
    } else {
      __threadfence();                      // release: the CTA's stores of this phase
      atomicAdd(ctr, 1u);
    }
    unsigned spins = 0;
    while (ld_relaxed_gpu(ctr) < target) {
      if (++spins > (1u << 28)) __trap();
    }
    if (flavor == 0) __threadfence();     // acquire
  }
  cp_async_wait_all();
  ptx::named_bar_sync(1, NCT);
}

// LayerNorm of one row by one warp, fp32, two-pass from registers.
// Element i of the row lives in lane (i % 32), slot (i / 32); slots >= npl are unused.
template <int NPL>
__device__ __forceinline__ void ln_row(const float (&v_in)[NPL], float (&v_out)[NPL],
                                       const float* w, const float* b, int lane) {
  constexpr float invD = 1.0f / (float)(NPL * 32);
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < NPL; ++j) s += v_in[j];
  const float mean = warp_sum(s) * invD;
  float q = 0.f;
#pragma unroll
  for (int j = 0; j < NPL; ++j) {
    const float d = v_in[j] - mean;
    q += d * d;
  }
  const float var = warp_sum(q) * invD;
  const float rstd = rsqrtf(var + 1e-5f);
#pragma unroll
  for (int j = 0; j < NPL; ++j) {
    const int i = lane + 32 * j;
    v_out[j] = (v_in[j] - mean) * rstd * w[i] + b[i];
  }
}

template <int NPL>
__device__ __forceinline__ void load_row(float (&v)[NPL], const float* x, int lane) {
#pragma unroll
  for (int j = 0; j < NPL; ++j) v[j] = __ldcg(x + lane + 32 * j);
}
// Activation rows in shared memory (the B operand of the GEMV MMAs) are stored with the 16-byte
// chunk index XOR-ed by (row & 7), like the weight rows in the ring: the 8 row addresses of an
// ldmatrix 8x8 tile then hit 8 different bank groups (rows are 10 KB / 2.5 KB apart = 0 mod 128 B).
__device__ __forceinline__ int xs_idx(int b, int k) { return (((k >> 3) ^ (b & 7)) << 3) | (k & 7); }

template <int NPL>
__device__ __forceinline__ void store_row_bf16(const float (&v)[NPL], __nv_bfloat16* xs_row, int b, int lane) {
#pragma unroll
  for (int j = 0; j < NPL; ++j) xs_row[xs_idx(b, lane + 32 * j)] = __float2bfloat16_rn(v[j]);
}

__device__ __forceinline__ void ldmatrix_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldmatrix_x2(uint32_t addr, uint32_t& r0, uint32_t& r1) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0,%1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(addr));
}
__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                               uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// NewGELUActivation with a bf16 round after every tensor op (transformers activations.py,
// evaluated on a bf16 tensor under autocast); plain fp32 formula when rounding is off.
__device__ __forceinline__ float gelu_new(float x, int r) {
  float t1 = rnd(x * x * x, r);
  float t2 = rnd(0.044715f * t1, r);
  float t3 = rnd(x + t2, r);
  float t4 = rnd(0.7978845608028654f * t3, r);
  float t5 = rnd(tanhf(t4), r);
  float t6 = rnd(1.0f + t5, r);
  float t7 = rnd(0.5f * x, r);
  return rnd(t7 * t6, r);
}

template <int BT>
struct Smem {
  // carved from dynamic shared memory
  __nv_bfloat16* xs;    // [BT][FF]  GEMV input rows (bf16)
  __nv_bfloat16* ring;  // [nst][UPC][D]
  float* red;           // [2][UPC][BT] K-split partial sums / attention warp merge [NCW][66]
  uint64_t* full;       // [nst]
  uint64_t* empty;      // [nst]
  int* flags;           // [4]: 0 exit flag for producer, 1 broadcast slot
  float* bias_s;        // per-CTA biases of every layer/phase + head, loaded once per launch
  float* xres;          // [BT][ocap] this CTA's slice of the fp32 residual stream
  float* lnp;           // [2][2][D] LayerNorm (weight,bias) double buffer, filled by cp.async
  unsigned* seen_s;     // [(V+31)/32] repetition-penalty bitmap of the sequence being sampled
};

// Cooperative LayerNorm of ONE row by all 8 compute warps (batch-1 decode, where a warp-per-row
// LayerNorm would leave 7 warps idle on the critical path).  Shifted one-pass statistics with a
// per-warp shift K_w = the warp's first element (a single global shift x[0] would make every thread of
// every CTA poll the same word of the tagged stream): S1_w = sum(x-K_w), S2_w = sum((x-K_w)^2);
// mean = sum_w(S1_w + n K_w) / D,  var = sum_w(S2_w + 2 (K_w-mean) S1_w + n (K_w-mean)^2) / D.
template <int NPL>
__device__ __forceinline__ void ln_block(float (&v)[NPL / 8], const float* w, const float* b,
                                         float* red, int warp, int lane) {
  constexpr int NPT = NPL / 8;
  constexpr float invD = 1.0f / (float)(NPL * 32);
  constexpr float nwarp = (float)(NPT * 32);
  const float K = __shfl_sync(0xffffffffu, v[0], 0);
  float s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int j = 0; j < NPT; ++j) {
    const float d = v[j] - K;
    s1 += d;
    s2 = fmaf(d, d, s2);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    s2 += __shfl_xor_sync(0xffffffffu, s2, o);
  }
  if (lane == 0) { red[3 * warp] = s1; red[3 * warp + 1] = s2; red[3 * warp + 2] = K; }
  ptx::named_bar_sync(1, NCT);
  float tot = 0.f;
#pragma unroll
  for (int q = 0; q < NCW; ++q) tot += red[3 * q] + nwarp * red[3 * q + 2];
  const float mean = tot * invD;
  float va = 0.f;
#pragma unroll
  for (int q = 0; q < NCW; ++q) {
    const float d = red[3 * q + 2] - mean;
    va += red[3 * q + 1] + 2.f * d * red[3 * q] + nwarp * d * d;
  }
  const float var = fmaxf(va * invD, 0.f);
  const float rstd = rsqrtf(var + 1e-5f);
#pragma unroll
  for (int j = 0; j < NPT; ++j) {
    const int i = warp * (NPL * 4) + lane + 32 * j;
    v[j] = (v[j] - mean) * rstd * w[i] + b[i];
  }
}

// One GEMV phase over this CTA's column slice on the tensor cores (mma.sync m16n8k16, bf16 in,
// fp32 accumulate).  The slice is cut into groups of <= 8 columns; one ring chunk holds the 8 weight
// rows of a group for one K-segment of D (pre-swizzled at pack time).  The MMA's M = 16 rows are the 8
// weight rows (rows 8..15 alias them), N = 8 are the activation rows of the step (batch / prompt
// positions; a 1-row step aliases row 0), K runs over the segment: warp w owns k-steps
// [w*KS, (w+1)*KS), so every warp issues KS x (ldmatrix A, ldmatrix B, mma) per chunk and the 8 partial
// accumulators are summed through shared memory.  A tile of M = 8 weight rows per 20 KB stage is what
// keeps the prefetch ring deep; wgmma's minimum M = 64 would need 160 KB stages.
// EPI: 0 QKV, 1 O-proj(+residual), 2 FC(+gelu), 3 PROJ(+residual), 4 HEAD
template <int BT, int EPI, int D>
__device__ __forceinline__ void gemv_phase(const GptParams& p, const Smem<BT>& sm, int layer,
                                           int col0, int ncols, int nseg, unsigned& cons_idx,
                                           const int* row_seq, const int* row_pos,
                                           const int* row_valid, int warp, int lane,
                                           const float* bias_ph, int o0, long long* fine = nullptr,
                                           unsigned x_epoch = 0) {
  constexpr int GMAX = (BT == 1) ? 7 : 2;           // column groups in flight
  constexpr int KS = (D / 16) / NCW;                // k-steps per warp per segment
  constexpr int FFc = 4 * D;
  const int ngroups = (ncols + 7) >> 3;
  const int gpb = max(1, min(GMAX, (p.nst - 1) / nseg));
  // per-lane ldmatrix coordinates
  const int a_r = lane & 7, a_hi = (lane >> 4) & 1;            // A: row in tile, k-half (matrices 2,3)
  const int b_n = min(lane & 7, BT - 1), b_hi = (lane >> 3) & 1;
  const uint32_t ring_base = ptx::smem_u32(sm.ring);
  const uint32_t xs_base = ptx::smem_u32(sm.xs) + (uint32_t)b_n * FFc * 2;
  const int g = lane >> 2, t4 = lane & 3;
  for (int g0 = 0; g0 < ngroups; g0 += gpb) {
    const int nb = min(gpb, ngroups - g0);
    float acc[GMAX][4];
#pragma unroll
    for (int gi = 0; gi < GMAX; ++gi) { acc[gi][0] = acc[gi][1] = acc[gi][2] = acc[gi][3] = 0.f; }
#pragma unroll
    for (int gi = 0; gi < GMAX; ++gi) {
      if (gi < nb) {
        for (int sgi = 0; sgi < nseg; ++sgi) {
          const unsigned n = cons_idx + gi * nseg + sgi;
          const int stage = n % p.nst;
          ptx::mbar_wait(&sm.full[stage], (n / p.nst) & 1u);
          if (fine && threadIdx.x == 0 && g0 == 0 && gi == 0 && sgi == 0) fine[0] = gtimer();
          const uint32_t a_row = ring_base + (uint32_t)((stage * UPC + a_r) * D * 2);
          const uint32_t b_row = xs_base + (uint32_t)(sgi * D * 2);
#pragma unroll
          for (int ks = 0; ks < KS; ++ks) {
            const int kc = 2 * (warp * KS + ks);                 // 16-byte chunk index of k0
            uint32_t a0, a1, a2, a3, b0, b1;
            ldmatrix_x4(a_row + (uint32_t)(((kc + a_hi) ^ a_r) << 4), a0, a1, a2, a3);
            ldmatrix_x2(b_row + (uint32_t)(((kc + b_hi) ^ (b_n & 7)) << 4), b0, b1);
            // x4 matrix order is (rows, k-lo), (rows+8, k-lo), (rows, k-hi), (rows+8, k-hi): the lane ->
            // address map above gives matrices 0,1 the k-lo chunk and 2,3 the k-hi chunk of the same rows
            mma_bf16_16816(acc[gi], a0, a1, a2, a3, b0, b1);
          }
        }
      }
    }
    // the weights of these chunks are consumed: hand the stages back to the producer
    if (fine && threadIdx.x == 0 && g0 == 0) fine[1] = gtimer();
    __syncwarp();
    if (lane == 0)
      for (int i = 0; i < nb * nseg; ++i) ptx::mbar_arrive(&sm.empty[(cons_idx + i) % p.nst]);
    cons_idx += nb * nseg;

    // cross-warp K reduction: red[gi][warp][row g][col]
    float* red = sm.red;
#pragma unroll
    for (int gi = 0; gi < GMAX; ++gi) {
      if (gi < nb) {
        if (BT == 1) {
          if (t4 == 0) red[(gi * NCW + warp) * 8 + g] = acc[gi][0];
        } else {
          float* rp = red + ((gi * NCW + warp) * 8 + g) * 8 + 2 * t4;
          rp[0] = acc[gi][0];
          rp[1] = acc[gi][1];
        }
      }
    }
    ptx::named_bar_sync(1, NCT);
    if (fine && threadIdx.x == 0 && g0 == 0) fine[2] = gtimer();
    const int nout = nb * 8 * BT;
    for (int idx = threadIdx.x; idx < nout; idx += NCT) {
      const int gi = idx / (8 * BT), r = (idx / BT) & 7, b = idx % BT;
      const int cl = (g0 + gi) * 8 + r;                         // column index inside the slice
      if (cl >= ncols || !row_valid[b]) continue;
      float a = 0.f;
#pragma unroll
      for (int w = 0; w < NCW; ++w)
        a += (BT == 1) ? red[(gi * NCW + w) * 8 + r] : red[((gi * NCW + w) * 8 + r) * 8 + b];
      const int c = col0 + cl;
      const int rr = p.round_bf16;
      if (EPI == 0) {
        float v = rnd(a + bias_ph[cl], rr);
        if (c < D) {
          p.qg[(size_t)b * D + c] = v;
          if (BT == 1 && x_epoch) st_tagged(p.qt + c, v, x_epoch);
        } else {
          size_t base = (((size_t)layer * p.nseq + row_seq[b]) * p.maxpos + row_pos[b]) * D;
          const __nv_bfloat16 kvb = __float2bfloat16_rn(v);
          if (c < 2 * D) p.kc[base + (c - D)] = kvb;
          else p.vc[base + (c - 2 * D)] = kvb;
          if (BT == 1 && x_epoch) st_tagged(p.kvt + (c - D), __bfloat162float(kvb), x_epoch);
        }
      } else if (EPI == 1 || EPI == 3) {
        // the residual stream is fp32 even on the bf16 path (trap P12): only the branch is rounded
        float o = rnd(a + bias_ph[cl], rr);
        float xn = sm.xres[b * p.ocap + (c - o0)] + o;
        sm.xres[b * p.ocap + (c - o0)] = xn;
        p.xg[(size_t)b * D + c] = xn;
        if (BT == 1 && x_epoch) st_tagged(p.xt + c, xn, x_epoch);
      } else if (EPI == 2) {
        float f = rnd(a + bias_ph[cl], rr);
        const __nv_bfloat16 fv = __float2bfloat16_rn(gelu_new(f, rr));
        p.fg[(size_t)b * FFc + c] = fv;
        if (BT == 1 && x_epoch)
          asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p.ft + c),
                       "r"((unsigned)__bfloat16_as_ushort(fv) | (x_epoch << 16)) : "memory");
      } else {
        p.logits[(size_t)b * p.V + c] = rnd(a + bias_ph[cl], rr);
      }
    }
    if (fine && threadIdx.x == 0 && g0 + gpb >= ngroups) fine[3] = gtimer();
    ptx::named_bar_sync(1, NCT);   // red is reused by the next batch of groups
  }
  if (fine && threadIdx.x == 0) fine[4] = gtimer();
}

#define PROF_STAMP()                                                        \
  do {                                                                      \
    if (p.prof && cta == 0 && tid == 0 && step == p.nsteps - 1 && pi < 256) \
      p.prof[pi++] = gtimer();                                              \
  } while (0)

__device__ __forceinline__ int col_begin(int N, int i, int G) {
  return (int)(((long long)N * i) / G);
}

// PROBE: the instantiation launched while an attention / prefill probe is armed (the other one has no probe code at all)
template <int BT, int NPL, bool PROBE>
__global__ void __launch_bounds__(NTHREADS, 1) gpt_fused_kernel(const GptParams p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  constexpr int D = NPL * 32, FF = 4 * D;
  const int G = p.G, L = p.L, H = p.H, V = p.V;
  const int cta = blockIdx.x;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  Smem<BT> sm;
  {
    unsigned char* q = smem_raw;
    sm.ring = (__nv_bfloat16*)q;  q += (size_t)p.nst * UPC * D * 2;
    sm.xs = (__nv_bfloat16*)q;    q += (size_t)BT * FF * 2;
    sm.red = (float*)q;           q += sizeof(float) * RED_FLOATS(BT);
    sm.full = (uint64_t*)q;       q += sizeof(uint64_t) * p.nst;
    sm.empty = (uint64_t*)q;      q += sizeof(uint64_t) * p.nst;
    sm.flags = (int*)q;           q += 16;
    sm.bias_s = (float*)q;        q += sizeof(float) * (size_t)p.bias_cap;
    sm.xres = (float*)q;          q += sizeof(float) * (size_t)BT * p.ocap;
    sm.seen_s = (unsigned*)q;     q += sizeof(unsigned) * (size_t)((V + 31) / 32);
    q = (unsigned char*)(((uintptr_t)q + 15) & ~(uintptr_t)15);
    sm.lnp = (float*)q;
  }
  if (tid == 0) {
    for (int s = 0; s < p.nst; ++s) {
      ptx::mbar_init(&sm.full[s], 1);
      ptx::mbar_init(&sm.empty[s], NCW);
    }
    sm.flags[0] = 0;
    ptx::fence_mbar_init();
  }
  __syncthreads();

  // column slices of this CTA
  const int q0 = col_begin(3 * D, cta, G), q1 = col_begin(3 * D, cta + 1, G);
  const int o0 = col_begin(D, cta, G), o1 = col_begin(D, cta + 1, G);
  const int f0 = col_begin(FF, cta, G), f1 = col_begin(FF, cta + 1, G);
  const int h0 = col_begin(V, cta, G), h1 = col_begin(V, cta + 1, G);
  const int nseg_proj = FF / D;
  const int units_head = (p.mode == 1) ? (h1 - h0) : 0;
  // per-CTA bias table: [L][ qkv | o | fc | proj ] then head — epilogues never wait on L2
  const int nq = q1 - q0, no = o1 - o0, nf = f1 - f0, nh = h1 - h0;
  const int bstride = nq + 2 * no + nf;
  if (warp < NCW) {
    for (int i = tid; i < L * bstride; i += NCT) {
      const int l = i / bstride, j = i % bstride;
      float v;
      if (j < nq) v = p.qkv_b[(size_t)l * 3 * D + q0 + j];
      else if (j < nq + no) v = p.o_b[(size_t)l * D + o0 + (j - nq)];
      else if (j < nq + no + nf) v = p.fc_b[(size_t)l * FF + f0 + (j - nq - no)];
      else v = p.proj_b[(size_t)l * D + o0 + (j - nq - no - nf)];
      sm.bias_s[i] = v;
    }
    for (int i = tid; i < nh; i += NCT) sm.bias_s[L * bstride + i] = p.head_b[h0 + i];
  }
  __syncthreads();

  // =============================================================== producer warp ====
  if (warp == NCW) {
    if (lane == 0) {
      const uint64_t pol = ptx::policy_evict_first();
      const __nv_bfloat16* base = p.wstream + (size_t)p.stream_off[cta] * D;
      unsigned prod_idx = 0;
      bool stop = false;
      const int phase_cols[4] = {nq, no, nf, no};
      const int phase_nseg[4] = {1, 1, 1, nseg_proj};
      for (int step = 0; step < p.nsteps && !stop; ++step) {
        size_t uoff = 0;
        for (int l = 0; l <= L && !stop; ++l) {
          const int nph = (l < L) ? 4 : 1;
          for (int ph = 0; ph < nph && !stop; ++ph) {
            const int ncol = (l < L) ? phase_cols[ph] : units_head;
            const int nsg = (l < L) ? phase_nseg[ph] : 1;
            for (int c0 = 0; c0 < ncol && !stop; c0 += 8) {
              const int rows = min(8, ncol - c0);
              for (int sgi = 0; sgi < nsg; ++sgi) {
                const int stage = prod_idx % p.nst;
                const unsigned parity = ((prod_idx / p.nst) & 1u) ^ 1u;
                unsigned spins = 0;
                while (!ptx::mbar_try_wait(&sm.empty[stage], parity)) {
                  if (*((volatile int*)&sm.flags[0])) { stop = true; break; }
                  if (++spins > (1u << 26)) __trap();
                }
                if (stop) break;
                const uint32_t bytes = (uint32_t)rows * D * 2;
                ptx::mbar_arrive_expect_tx(&sm.full[stage], bytes);
                ptx::bulk_g2s(sm.ring + (size_t)stage * UPC * D, base + uoff * D, bytes, &sm.full[stage], pol);
                ++prod_idx;
                uoff += rows;
              }
            }
          }
        }
      }
      sm.flags[2] = (int)prod_idx;  // chunks issued (read by the drain below)
    }
    __syncwarp();
  } else {
    // ============================================================ compute warps ====
    unsigned cons_idx = 0;
    unsigned bar_target = 0;
    __shared__ int row_seq[8], row_pos[8], row_valid[8], row_posidx[8];
    __shared__ float* prb_row[8];   // PROBE: record of row b of the current step at its first probed layer, or null
    const int nsplit = min(8, max(1, G / (p.B * H)));

    int pi = 0;
    // cp.async prefetch of a LayerNorm (weight, bias) pair into lnp buffer `buf`
    auto prefetch_ln = [&](int buf, const float* w, const float* b) {
      float* dst = sm.lnp + (size_t)buf * 2 * D;
      const int n4 = D / 4;
      for (int i = tid; i < 2 * n4; i += NCT) {
        const int which = i / n4, off = (i % n4) * 4;
        cp_async16(dst + which * D + off, (which ? b : w) + off);
      }
    };
    const float* lnA = sm.lnp;
    const float* lnB = sm.lnp + 2 * D;
    for (int step = 0; step < p.nsteps; ++step) {
      PROF_STAMP();
      if (step == 0) prefetch_ln(0, p.ln1_w, p.ln1_b);
      // ---- step prologue: row descriptors + input embedding -> xg (own columns only) ----
      if (tid < 8) {
        int b = tid;
        if (p.mode == 0) {
          PrefillTile t = p.tiles[step];
          row_seq[b] = t.seq;
          row_pos[b] = t.pos0 + b;
          row_valid[b] = (b < t.nrows);
          row_posidx[b] = t.src_row + b;
        } else {
          int k = p.step0 + step;
          row_seq[b] = b;
          row_pos[b] = (b < p.B) ? p.prompt_len[b] + k : 0;
          row_valid[b] = (b < p.B);
          row_posidx[b] = (k == 0 || p.pos_plain) ? k : k + 1;  // P1: mel position k+1 with KV cache
        }
        if constexpr (PROBE) {
          // probe records of this step's rows (published to the attention phases by the barriers below)
          prb_row[b] = (b < p.B && row_valid[b]) ? fused_probe_row(p, p.step0 + step, b, row_seq[b], row_pos[b]) : nullptr;
          if (p.mode == 1 && cta == 0 && b == 0)
            for (int l = 0; l < L; ++l)
              if (probe_slot(p, p.step0 + step, l) >= 0) p.probe_ns[probe_slot(p, p.step0 + step, l)] = nsplit;
        }
      }
      ptx::named_bar_sync(1, NCT);
      // every CTA writes the input rows for its own O-proj column slice [o0,o1)
      for (int idx = tid; idx < BT * (o1 - o0); idx += NCT) {
        int b = idx / (o1 - o0), c = o0 + idx % (o1 - o0);
        if (b < BT && row_valid[b]) {
          float v;
          if (p.mode == 0) {
            v = p.prompt[(size_t)row_posidx[b] * D + c];
          } else {
            int t = __ldcg(p.tok + b);
            v = rnd(__ldg(p.mel_emb + (size_t)t * D + c) +
                        __ldg(p.mel_pos + (size_t)row_posidx[b] * D + c), p.round_bf16);
          }
          p.xg[(size_t)b * D + c] = v;
          sm.xres[b * p.ocap + (c - o0)] = v;
        }
      }
      PROF_STAMP();
      grid_sync(p.barrier, bar_target, G, p.bar_flavor);
      PROF_STAMP();

      for (int l = 0; l < L; ++l) {
        // Data-flow hand-overs (batch-1 decode): no grid barrier inside a layer.  Epochs are unique per (step, layer).
        // Write-after-read safety without extra synchronisation — the next writer of every buffer transitively depends on
        // data that all CTAs produce only after their own reads of it (program order + CTA barriers inside a CTA):
        //   xt  (O-proj -> FC, PROJ -> next QKV): PROJ(l) starts on a CTA once it holds every ft word of FC(l), which each
        //        CTA writes after its FC(l) read of xt; O-proj(l+1) needs the attention partials of all heads, hence
        //        q/k/v columns from every CTA's QKV(l+1), each written after that CTA's read of xt;
        //   ft  (FC -> PROJ): FC(l+1) needs every xt word of O-proj(l+1), which follows each CTA's PROJ(l) read of ft;
        //   qt, kvt (QKV -> attention) and part/pflag (attention -> O-proj): QKV(l+1) needs every xt word of PROJ(l),
        //        which follows each CTA's attention(l) and O-proj(l) reads.
        // Steps are separated by the grid barriers around the head and the sampling phase.
        // tagged residual stream (batch-1 decode): epochs of the two x hand-overs of this layer
        const bool tagged = (BT == 1) && p.xt != nullptr;
        long long* f2 = (p.prof2 && l == p.prof2_layer && step == p.nsteps - 1) ? p.prof2 + (size_t)cta * 64 : nullptr;
#define F2(i) do { if (f2 && tid == 0) f2[(i)] = gtimer(); } while (0)
        F2(0);
        const unsigned ep_base = p.epoch0 + (unsigned)(step * L + l) * 2u;
        const unsigned ep_oproj = ep_base + 1u;      // O-proj -> FC of this layer
        const unsigned ep_proj = ep_base + 2u;       // PROJ -> QKV of the next layer (== ep_base of l + 1)
        const unsigned f_tag = ((ep_base >> 1) % 65535u) + 1u;   // 16-bit tag of this layer's gelu(fc) words, never 0
        // ---------------- P1: LN1 -> QKV ----------------
        prefetch_ln(1, p.ln2_w + (size_t)l * D, p.ln2_b + (size_t)l * D);  // for P4
        if constexpr (BT == 1) {
          float v[NPL / 8];
          if (tagged && l > 0) {
            ld_tagged_slice<NPL / 8>(p.xt, warp * (NPL * 4) + lane, ep_base, v);
            F2(1);
          } else {
#pragma unroll
            for (int j = 0; j < NPL / 8; ++j) v[j] = __ldcg(p.xg + warp * (NPL * 4) + lane + 32 * j);
          }
          ln_block<NPL>(v, lnA, lnA + D, sm.red, warp, lane);
          F2(2);
#pragma unroll
          for (int j = 0; j < NPL / 8; ++j)
            sm.xs[warp * (NPL * 4) + lane + 32 * j] = __float2bfloat16_rn(v[j]);
        } else {
          for (int b = warp; b < BT; b += NCW) {
            float v[NPL], o[NPL];
            load_row<NPL>(v, p.xg + (size_t)b * D, lane);
            ln_row<NPL>(v, o, lnA, lnA + D, lane);
            store_row_bf16<NPL>(o, sm.xs + (size_t)b * FF, b, lane);
          }
        }
        ptx::named_bar_sync(1, NCT);
        F2(3);
        gemv_phase<BT, 0, D>(p, sm, l, q0, nq, 1, cons_idx, row_seq, row_pos, row_valid,
                          warp, lane, sm.bias_s + l * bstride, o0,
                          f2 ? f2 + 4 : nullptr, tagged ? ep_oproj : 0u);
        F2(9);
        PROF_STAMP();
        if (!tagged) grid_sync(p.barrier, bar_target, G, p.bar_flavor);   // tagged: attention polls q and the new k, v
        PROF_STAMP();

        // ---------------- P2: attention over the KV cache ----------------
        {
          const int nitems = p.B * H * nsplit;
          const int g4 = lane >> 3, sub = lane & 7;
          for (int it = cta; it < nitems; it += G) {
            const int b = it / (H * nsplit);
            const int h = (it / nsplit) % H;
            const int sp = it % nsplit;
            float* pout = p.part + (size_t)it * PART_STRIDE;
            if (!row_valid[b]) continue;
            const int ctx = row_pos[b] + 1;
            const int k0 = (int)(((long long)ctx * sp) / nsplit);
            const int k1 = (int)(((long long)ctx * (sp + 1)) / nsplit);
            float qv[8];
            if (tagged) {
              const uint2* qp = p.qt + h * HD + sub * 8;
              unsigned val[8], tg[8], spins = 0;
              bool ok;
              do {
#pragma unroll
                for (int i = 0; i < 8; ++i)
                  asm volatile("ld.relaxed.gpu.global.v2.u32 {%0, %1}, [%2];" : "=r"(val[i]), "=r"(tg[i]) : "l"(qp + i) : "memory");
                ok = true;
#pragma unroll
                for (int i = 0; i < 8; ++i) ok &= (tg[i] == ep_oproj);
                if (++spins > (1u << 26)) __trap();
              } while (!ok);
              F2(10);
#pragma unroll
              for (int i = 0; i < 8; ++i) qv[i] = __uint_as_float(val[i]);
            } else {
              const float* qp = p.qg + (size_t)b * D + h * HD + sub * 8;
#pragma unroll
              for (int i = 0; i < 8; ++i) qv[i] = __ldcg(qp + i);
            }
            if (PROBE && sp == 0 && warp == 0 && g4 == 0) {
              float* const pr = prb_row[b];
              if (pr) {
                float* const pl = fused_probe_at(p, pr, l);
                if (pl)
#pragma unroll
                  for (int i = 0; i < 8; ++i) pl[h * HD + sub * 8 + i] = qv[i];
              }
            }
            // tagged mode: the position being decoded comes from the tagged words, not from the cache
            const int kend = tagged ? min(k1, ctx - 1) : k1;
            float m = -INFINITY, lsum = 0.f, ov[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) ov[i] = 0.f;
            // beam search: prompt positions live in the utterance's first slot, generated ones where p.phys says.
            // Two instantiations of the key loop so that the plain path keeps its single address stream.
            const size_t cbase = ((size_t)l * p.nseq + row_seq[b]) * p.maxpos;
            auto key_loop = [&](auto beamed_tag) {
              constexpr bool BEAMED = decltype(beamed_tag)::value;
              int plen_b = 0, base_seq = 0;
              const unsigned char* phys_b = nullptr;
              if constexpr (BEAMED) {
                plen_b = __ldg(p.prompt_len + b);
                base_seq = (b / p.beams) * p.beams;
                phys_b = p.phys + (size_t)b * p.phys_stride;
              }
              for (int j0 = k0 + warp * 4; j0 < kend; j0 += NCW * 4) {
                const int j = j0 + g4;
                const bool valid = j < kend;
                float s = 0.f;
                uint4 vv = make_uint4(0, 0, 0, 0);
                if (valid) {
                  size_t off;
                  if constexpr (BEAMED) {
                    const int sj = (j < plen_b) ? base_seq : (int)phys_b[j - plen_b];
                    off = ((((size_t)l * p.nseq + sj) * p.maxpos) + j) * D + h * HD + sub * 8;
                  } else {
                    off = (cbase + j) * D + h * HD + sub * 8;
                  }
                  uint4 kk = __ldcg((const uint4*)(p.kc + off));
                  vv = __ldcg((const uint4*)(p.vc + off));
                  s = qv[0] * lo_bf(kk.x) + qv[1] * hi_bf(kk.x) + qv[2] * lo_bf(kk.y) +
                      qv[3] * hi_bf(kk.y) + qv[4] * lo_bf(kk.z) + qv[5] * hi_bf(kk.z) +
                      qv[6] * lo_bf(kk.w) + qv[7] * hi_bf(kk.w);
                }
                s += __shfl_xor_sync(0xffffffffu, s, 1);
                s += __shfl_xor_sync(0xffffffffu, s, 2);
                s += __shfl_xor_sync(0xffffffffu, s, 4);
                if (valid) {
                  s *= 0.125f;
                  const float mn = fmaxf(m, s);
                  const float corr = __expf(m - mn);
                  const float pr = __expf(s - mn);
                  lsum = lsum * corr + pr;
                  const float vf[8] = {lo_bf(vv.x), hi_bf(vv.x), lo_bf(vv.y), hi_bf(vv.y),
                                       lo_bf(vv.z), hi_bf(vv.z), lo_bf(vv.w), hi_bf(vv.w)};
#pragma unroll
                  for (int i = 0; i < 8; ++i) ov[i] = ov[i] * corr + pr * vf[i];
                  m = mn;
                }
              }
            };
            if (p.phys) key_loop(std::true_type{}); else key_loop(std::false_type{});
            F2(11);
            if (tagged && k1 == ctx && warp == 0 && g4 == 0) {
              // the new position (owned by the last key split): k and v straight from the QKV epilogue's tagged words
              const uint2* kp = p.kvt + h * HD + sub * 8;
              const uint2* vp = p.kvt + D + h * HD + sub * 8;
              unsigned kvv[16], tg[16], spins = 0;
              bool ok;
              do {
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                  asm volatile("ld.relaxed.gpu.global.v2.u32 {%0, %1}, [%2];" : "=r"(kvv[i]), "=r"(tg[i]) : "l"(kp + i) : "memory");
                  asm volatile("ld.relaxed.gpu.global.v2.u32 {%0, %1}, [%2];" : "=r"(kvv[8 + i]), "=r"(tg[8 + i]) : "l"(vp + i) : "memory");
                }
                ok = true;
#pragma unroll
                for (int i = 0; i < 16; ++i) ok &= (tg[i] == ep_oproj);
                if (++spins > (1u << 26)) __trap();
              } while (!ok);
              float s = 0.f;
#pragma unroll
              for (int i = 0; i < 8; ++i) s += qv[i] * __uint_as_float(kvv[i]);
              s += __shfl_xor_sync(0xffu, s, 1);
              s += __shfl_xor_sync(0xffu, s, 2);
              s += __shfl_xor_sync(0xffu, s, 4);
              s *= 0.125f;
              const float mn = fmaxf(m, s);
              const float corr = __expf(m - mn);
              const float pr = __expf(s - mn);
              lsum = lsum * corr + pr;
#pragma unroll
              for (int i = 0; i < 8; ++i) ov[i] = ov[i] * corr + pr * __uint_as_float(kvv[8 + i]);
              m = mn;
            }
            __syncwarp();
            F2(12);
            // merge the 4 key groups of the warp
#pragma unroll
            for (int xo = 8; xo <= 16; xo <<= 1) {
              const float m2 = __shfl_xor_sync(0xffffffffu, m, xo);
              const float l2 = __shfl_xor_sync(0xffffffffu, lsum, xo);
              const float mn = fmaxf(m, m2);
              const float c1 = (m == -INFINITY) ? 0.f : __expf(m - mn);
              const float c2 = (m2 == -INFINITY) ? 0.f : __expf(m2 - mn);
              lsum = lsum * c1 + l2 * c2;
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                const float o2 = __shfl_xor_sync(0xffffffffu, ov[i], xo);
                ov[i] = ov[i] * c1 + o2 * c2;
              }
              m = mn;
            }
            // merge the 8 warps through shared memory
            float* red = sm.red;
            ptx::named_bar_sync(1, NCT);  // previous item's merge buffer is free
            if (lane < 8) {
              float* rw = red + warp * PART_STRIDE;
              if (lane == 0) { rw[0] = m; rw[1] = lsum; }
#pragma unroll
              for (int i = 0; i < 8; ++i) rw[2 + lane * 8 + i] = ov[i];
            }
            ptx::named_bar_sync(1, NCT);
            F2(13);
            if (warp == 0) {
              float mm = -INFINITY;
              for (int w = 0; w < NCW; ++w) mm = fmaxf(mm, red[w * PART_STRIDE]);
              float lt = 0.f, oa = 0.f, ob = 0.f;
              for (int w = 0; w < NCW; ++w) {
                const float mw = red[w * PART_STRIDE];
                const float c = (mw == -INFINITY) ? 0.f : __expf(mw - mm);
                lt += red[w * PART_STRIDE + 1] * c;
                oa += red[w * PART_STRIDE + 2 + lane] * c;
                ob += red[w * PART_STRIDE + 2 + 32 + lane] * c;
              }
              if (lane == 0) { pout[0] = mm; pout[1] = lt; }
              pout[2 + lane] = oa;
              pout[2 + 32 + lane] = ob;
              if (tagged) {
                // publish the partial: the release is cumulative over the warp's stores ordered by __syncwarp
                __syncwarp();
                if (lane == 0) st_release_gpu(p.pflag + (size_t)it * 32, ep_oproj);   // one 128-byte line per flag: no hot line
              }
            }
          }
        }
        F2(14);
        PROF_STAMP();
        if (!tagged) grid_sync(p.barrier, bar_target, G, p.bar_flavor);   // tagged: O-proj polls the partials' flags
        PROF_STAMP();

        // ---------------- P3: merge attention splits -> O-proj + residual ----------------
        // one warp per (row, head): the nsplit partials of a head are contiguous (66 floats
        // each); every load below is independent so they all fly together (one L2 round trip)
        for (int bh0 = warp; bh0 < BT * H; bh0 += 3 * NCW) {
          if (tagged) {
            // lanes 0..23 poll the flags of (head r3 = lane / 8, split lane % 8) of this round together
            const int r3f = lane >> 3, sf = lane & 7;
            const int bhf = bh0 + r3f * NCW;
            const bool onf = r3f < 3 && bhf < BT * H && sf < nsplit && row_valid[bhf / H];
            const unsigned* fp = p.pflag + ((size_t)bhf * nsplit + sf) * 32;
            unsigned spins = 0;
            for (;;) {
              unsigned fv = ep_oproj;
              if (onf) asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(fv) : "l"(fp) : "memory");
              if (__all_sync(0xffffffffu, fv == ep_oproj)) break;
              if (++spins > (1u << 26)) __trap();
            }
            if (bh0 == warp) F2(16);
          }
          float ms[3][8], ls[3][8], oa[3][8], ob[3][8];
#pragma unroll
          for (int r3 = 0; r3 < 3; ++r3) {
            const int bh = bh0 + r3 * NCW;
            const int b = bh / H, h = bh % H;
            const bool rowon = bh < BT * H && b < p.B && row_valid[b];
            const float* pp = p.part + (size_t)((b * H + h) * nsplit) * PART_STRIDE;
#pragma unroll
            for (int s = 0; s < 8; ++s) {
              const bool on = rowon && s < nsplit;
              ms[r3][s] = on ? __ldcg(pp + s * PART_STRIDE) : -INFINITY;
              ls[r3][s] = on ? __ldcg(pp + s * PART_STRIDE + 1) : 0.f;
              oa[r3][s] = on ? __ldcg(pp + s * PART_STRIDE + 2 + lane) : 0.f;
              ob[r3][s] = on ? __ldcg(pp + s * PART_STRIDE + 34 + lane) : 0.f;
            }
          }
#pragma unroll
          for (int r3 = 0; r3 < 3; ++r3) {
            const int bh = bh0 + r3 * NCW;
            if (bh >= BT * H) continue;
            const int b = bh / H, h = bh % H;
            float mm = -INFINITY;
#pragma unroll
            for (int s = 0; s < 8; ++s) mm = fmaxf(mm, ms[r3][s]);
            float lt = 0.f, o0v = 0.f, o1v = 0.f;
#pragma unroll
            for (int s = 0; s < 8; ++s) {
              const float cc = (ms[r3][s] == -INFINITY) ? 0.f : __expf(ms[r3][s] - mm);
              lt += ls[r3][s] * cc;
              o0v += oa[r3][s] * cc;
              o1v += ob[r3][s] * cc;
            }
            const float inv = (lt > 0.f) ? 1.0f / lt : 0.f;
            sm.xs[(size_t)b * FF + xs_idx(b, h * HD + lane)] = __float2bfloat16_rn(o0v * inv);
            sm.xs[(size_t)b * FF + xs_idx(b, h * HD + 32 + lane)] = __float2bfloat16_rn(o1v * inv);
            float* const pr = PROBE ? prb_row[b] : nullptr;
            if (PROBE && pr && cta == 0) {
              float* const pl = fused_probe_at(p, pr, l);
              if (pl) { pl[D + h * HD + lane] = o0v * inv; pl[D + h * HD + 32 + lane] = o1v * inv; }
            }
          }
        }
        ptx::named_bar_sync(1, NCT);
        F2(17);
        gemv_phase<BT, 1, D>(p, sm, l, o0, no, 1, cons_idx, row_seq, row_pos, row_valid,
                          warp, lane, sm.bias_s + l * bstride + nq, o0, f2 ? f2 + 18 : nullptr, tagged ? ep_oproj : 0u);
        F2(23);
        PROF_STAMP();
        if (!tagged) grid_sync(p.barrier, bar_target, G, p.bar_flavor);   // tagged: FC polls the x words instead
        PROF_STAMP();

        // ---------------- P4: LN2 -> FC + gelu_new ----------------
        // buffer A was last read in P1 of this layer: refill it for the next LN1 / ln_f
        if (l + 1 < L) prefetch_ln(0, p.ln1_w + (size_t)(l + 1) * D, p.ln1_b + (size_t)(l + 1) * D);
        else if (p.mode == 1) prefetch_ln(0, p.lnf_w, p.lnf_b);
        else prefetch_ln(0, p.ln1_w, p.ln1_b);
        if constexpr (BT == 1) {
          float v[NPL / 8];
          if (tagged) {
            ld_tagged_slice<NPL / 8>(p.xt, warp * (NPL * 4) + lane, ep_oproj, v);
            F2(24);
            cp_async_wait_all();   // ln_2 parameters prefetched in P1 (ln_block's own CTA barrier publishes them)
          } else {
#pragma unroll
            for (int j = 0; j < NPL / 8; ++j) v[j] = __ldcg(p.xg + warp * (NPL * 4) + lane + 32 * j);
          }
          ln_block<NPL>(v, lnB, lnB + D, sm.red, warp, lane);
          F2(25);
#pragma unroll
          for (int j = 0; j < NPL / 8; ++j)
            sm.xs[warp * (NPL * 4) + lane + 32 * j] = __float2bfloat16_rn(v[j]);
        } else {
          for (int b = warp; b < BT; b += NCW) {
            float v[NPL], o[NPL];
            load_row<NPL>(v, p.xg + (size_t)b * D, lane);
            ln_row<NPL>(v, o, lnB, lnB + D, lane);
            store_row_bf16<NPL>(o, sm.xs + (size_t)b * FF, b, lane);
          }
        }
        ptx::named_bar_sync(1, NCT);
        F2(26);
        gemv_phase<BT, 2, D>(p, sm, l, f0, nf, 1, cons_idx, row_seq, row_pos, row_valid,
                          warp, lane, sm.bias_s + l * bstride + nq + no, o0,
                          f2 ? f2 + 27 : nullptr, tagged ? f_tag : 0u);
        F2(32);
        PROF_STAMP();
        if (!tagged) grid_sync(p.barrier, bar_target, G, p.bar_flavor);   // tagged: PROJ polls the {value, tag} words
        PROF_STAMP();

        // ---------------- P5: proj + residual ----------------
        if (l + 1 == L && p.mode == 1) prefetch_ln(1, p.fn_w, p.fn_b);  // final_norm for the head
        if (tagged) {
          // chunks of 8 words {bf16, tag}: all loads of a round in flight together, repeat until every tag matches
          constexpr int CPR = FF / 8, NCH = (CPR + NCT - 1) / NCT;
          uint4 lo[NCH], hi[NCH];
          const unsigned want = f_tag << 16;
          unsigned spins = 0;
          bool ok;
          do {
            ok = true;
#pragma unroll
            for (int q = 0; q < NCH; ++q) {
              const int c = tid + q * NCT;
              if (c < CPR) {
                const unsigned* src = p.ft + (size_t)c * 8;
                asm volatile("ld.relaxed.gpu.global.v4.u32 {%0, %1, %2, %3}, [%4];"
                             : "=r"(lo[q].x), "=r"(lo[q].y), "=r"(lo[q].z), "=r"(lo[q].w) : "l"(src) : "memory");
                asm volatile("ld.relaxed.gpu.global.v4.u32 {%0, %1, %2, %3}, [%4];"
                             : "=r"(hi[q].x), "=r"(hi[q].y), "=r"(hi[q].z), "=r"(hi[q].w) : "l"(src + 4) : "memory");
              }
            }
#pragma unroll
            for (int q = 0; q < NCH; ++q) {
              if (tid + q * NCT < CPR)
                ok &= ((lo[q].x & 0xffff0000u) == want) & ((lo[q].y & 0xffff0000u) == want) &
                      ((lo[q].z & 0xffff0000u) == want) & ((lo[q].w & 0xffff0000u) == want) &
                      ((hi[q].x & 0xffff0000u) == want) & ((hi[q].y & 0xffff0000u) == want) &
                      ((hi[q].z & 0xffff0000u) == want) & ((hi[q].w & 0xffff0000u) == want);
            }
            if (++spins > (1u << 26)) __trap();
          } while (!ok);
          F2(33);
#pragma unroll
          for (int q = 0; q < NCH; ++q) {
            const int c = tid + q * NCT;
            if (c < CPR)
              ((uint4*)sm.xs)[c] = make_uint4((lo[q].x & 0xffffu) | (lo[q].y << 16), (lo[q].z & 0xffffu) | (lo[q].w << 16),
                                              (hi[q].x & 0xffffu) | (hi[q].y << 16), (hi[q].z & 0xffffu) | (hi[q].w << 16));
          }
          cp_async_wait_all();     // the LayerNorm parameters prefetched in P4 (the barrier used to drain them)
        } else {
          constexpr int CPR = FF / 8;   // 16-byte chunks per row
          for (int idx = tid; idx < BT * CPR; idx += NCT) {
            const int b = idx / CPR, c = idx % CPR;
            ((uint4*)sm.xs)[b * CPR + (c ^ (b & 7))] = __ldcg(((const uint4*)p.fg) + idx);
          }
        }
        ptx::named_bar_sync(1, NCT);
        F2(34);
        const bool tag_proj = tagged && l + 1 < L;   // the last layer hands over to the head through a barrier
        gemv_phase<BT, 3, D>(p, sm, l, o0, no, nseg_proj, cons_idx, row_seq, row_pos,
                          row_valid, warp, lane, sm.bias_s + l * bstride + nq + no + nf, o0, f2 ? f2 + 35 : nullptr,
                          tag_proj ? ep_proj : 0u);
        F2(40);
        PROF_STAMP();
        if (!tag_proj) grid_sync(p.barrier, bar_target, G, p.bar_flavor);
        PROF_STAMP();
      }

      if (p.mode == 0 && p.hidden_out) {
        // v1 latent pass: every CTA writes its own column slice of the final residual stream (kept in xres by the
        // PROJ epilogue), so no other CTA's data is touched and the next tile may start at once
        for (int idx = tid; idx < BT * (o1 - o0); idx += NCT) {
          const int b = idx / (o1 - o0), c = o0 + idx % (o1 - o0);
          if (row_valid[b]) p.hidden_out[(size_t)row_posidx[b] * D + c] = sm.xres[b * p.ocap + (c - o0)];
        }
        ptx::named_bar_sync(1, NCT);
      }
      if (p.mode == 1) {
        // ---------------- head: ln_f -> final_norm -> mel_head ----------------
        if constexpr (BT == 1) {
          float v[NPL / 8];
#pragma unroll
          for (int j = 0; j < NPL / 8; ++j) v[j] = __ldcg(p.xg + warp * (NPL * 4) + lane + 32 * j);
          ln_block<NPL>(v, lnA, lnA + D, sm.red, warp, lane);
          ln_block<NPL>(v, lnB, lnB + D, sm.red + 3 * NCW, warp, lane);
#pragma unroll
          for (int j = 0; j < NPL / 8; ++j)
            sm.xs[warp * (NPL * 4) + lane + 32 * j] = __float2bfloat16_rn(v[j]);
        } else {
          for (int b = warp; b < BT; b += NCW) {
            float v[NPL], o[NPL];
            load_row<NPL>(v, p.xg + (size_t)b * D, lane);
            ln_row<NPL>(v, o, lnA, lnA + D, lane);
            ln_row<NPL>(o, v, lnB, lnB + D, lane);
            store_row_bf16<NPL>(v, sm.xs + (size_t)b * FF, b, lane);
          }
        }
        ptx::named_bar_sync(1, NCT);
        gemv_phase<BT, 4, D>(p, sm, 0, h0, nh, 1, cons_idx, row_seq, row_pos, row_valid,
                          warp, lane, sm.bias_s + L * bstride, o0);
        PROF_STAMP();
        grid_sync(p.barrier, bar_target, G, p.bar_flavor);
        PROF_STAMP();

        // ---------------- sampling: CTA b handles sequence b ----------------
        prefetch_ln(0, p.ln1_w, p.ln1_b);  // layer 0 of the next step (buffer A is free again)
        if (cta < p.B && !p.ext_sample) {
          const int b = cta;
          const int k = p.step0 + step;
          const float* lg = p.logits + (size_t)b * V;
          if (p.logits_dump) {
            float* dst = p.logits_dump + ((size_t)b * p.max_new + k) * V;
            for (int i = tid; i < V; i += NCT) dst[i] = __ldcg(lg + i);
          }
          for (int i = tid; i < (V + 31) / 32; i += NCT)
            sm.seen_s[i] = p.seen[(size_t)b * ((V + 31) / 32) + i];
          ptx::named_bar_sync(1, NCT);
#define FINE_STAMP(n) do { if (p.prof && cta == 0 && tid == 0 && step == p.nsteps - 1) p.prof[256 + (n)] = gtimer(); } while (0)
          FINE_STAMP(32);
          const unsigned* seen = sm.seen_s;
          // processed scores of this thread's slice stay in registers: s = rep_penalty(logit) [/ temperature]
          constexpr int VPT = 40;   // ceil(V / 256) for V <= 10240
          float sv[VPT];
          const float inv_temp = (p.do_sample && p.temperature > 0.f) ? 1.0f / p.temperature : 1.0f;
          // two passes: all loads first (they then fly together: one L2 round trip instead of one per element —
          // fused into one loop the compiler serialised load -> test -> next load, 10.8 us of the 14 us of this phase)
#pragma unroll
          for (int j = 0; j < VPT; ++j) {
            const int i = tid + j * NCT;
            sv[j] = (i < V) ? __ldcg(lg + i) : -INFINITY;
          }
#pragma unroll
          for (int j = 0; j < VPT; ++j) {
            const int i = tid + j * NCT;
            if (i < V) {
              float sc = sv[j];
              if ((seen[i >> 5] >> (i & 31)) & 1u) sc = (sc < 0.f) ? sc * p.rep_penalty : sc / p.rep_penalty;
              if (i == p.stop_tok && k < p.forbid_stop_before) sc = -INFINITY;
              if (p.do_sample) sc *= inv_temp;
              sv[j] = sc;
            }
          }
          float* red = sm.red;
          // block argmax with lowest-index tie break; `extract` removes the winner from its owner's registers
          auto block_argmax = [&](float& bestv, int& besti) {
            float best = -INFINITY;
            int bi = 0x7fffffff;
#pragma unroll
            for (int j = 0; j < VPT; ++j) {
              const int i = tid + j * NCT;
              if (sv[j] > best || (sv[j] == best && i < bi && sv[j] > -INFINITY)) { best = sv[j]; bi = i; }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
              const float b2 = __shfl_xor_sync(0xffffffffu, best, o);
              const int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
              if (b2 > best || (b2 == best && i2 < bi)) { best = b2; bi = i2; }
            }
            ptx::named_bar_sync(1, NCT);
            if (lane == 0) { red[warp * 2] = best; ((int*)red)[warp * 2 + 1] = bi; }
            ptx::named_bar_sync(1, NCT);
            for (int w = 0; w < NCW; ++w) {
              const float b2 = red[w * 2];
              const int i2 = ((int*)red)[w * 2 + 1];
              if (w == 0 || b2 > best || (b2 == best && i2 < bi)) { best = b2; bi = i2; }
            }
            bestv = best; besti = bi;
          };
          FINE_STAMP(33);
          float best; int besti;
          block_argmax(best, besti);
          FINE_STAMP(34);
          if (p.do_sample) {
            // top-k: extract candidates in descending order (ties at the k-th value are kept, like
            // TopKLogitsWarper's `scores < kth` test); the host rejects top_k outside 1..CMAX, and a tie that would
            // need more than CMAX slots sets the error flag (the call is refused, never silently capped)
            float* cv = red + 32;                    // [CMAX] candidate scores
            int* ci = (int*)(red + 32 + CMAX);       // [CMAX] candidate ids
            const int kk = min(max(p.top_k, 1), CMAX);
            int nc = 0;
            float kth = best;
            while (nc < CMAX && best > -INFINITY && (nc < kk || best == kth)) {
              if (tid == 0) { cv[nc] = best; ci[nc] = besti; }
              if (nc < kk) kth = best;
              ++nc;
#pragma unroll
              for (int j = 0; j < VPT; ++j)
                if (tid + j * NCT == besti) sv[j] = -INFINITY;
              block_argmax(best, besti);
            }
            if (tid == 0 && nc == CMAX && best == kth && best > -INFINITY && !p.finished[b]) *p.flag = k + 1;
            ptx::named_bar_sync(1, NCT);
            if (tid == 0) {
              // softmax over the kept candidates, top-p filter (TopPLogitsWarper: drop while the
              // ascending cumulative probability <= 1 - top_p, keep at least one), multinomial
              const float mx = cv[0];
              float tot = 0.f;
              for (int i = 0; i < nc; ++i) { cv[i] = expf(cv[i] - mx); tot += cv[i]; }
              int keep = nc;
              if (p.top_p < 1.0f) {
                float tail = 0.f;
                for (int i = nc - 1; i >= 1; --i) {
                  tail += cv[i] / tot;
                  if (tail <= 1.0f - p.top_p) keep = i; else break;
                }
              }
              float kt = 0.f;
              for (int i = 0; i < keep; ++i) kt += cv[i];
              unsigned rnd4[4];
              philox4x32_10(p.seed, (unsigned)k, (unsigned)(b + p.seq_base), rnd4);
              const float u = (float)(rnd4[0] >> 8) * (1.0f / 16777216.0f) * kt;
              float acc = 0.f;
              int pick = keep - 1;
              for (int i = 0; i < keep; ++i) { acc += cv[i]; if (u < acc) { pick = i; break; } }
              besti = ci[pick];
            }
          }
          if (tid == 0) {
            const int fin = p.finished[b];
            if (!fin) {
              p.codes[(size_t)b * p.max_new + k] = besti;
              p.nout[b] = k + 1;
              int feed = besti;
              if (p.forced) feed = p.forced[(size_t)b * p.max_new + k];
              else if (besti == p.stop_tok) p.finished[b] = 1;
              if (k + 1 >= p.max_new) p.finished[b] = 1;
              p.tok[b] = feed;
              p.seen[(size_t)b * ((V + 31) / 32) + (feed >> 5)] |= 1u << (feed & 31);
            }
          }
          FINE_STAMP(35);
          ptx::named_bar_sync(1, NCT);
        }
        PROF_STAMP();
        grid_sync(p.barrier, bar_target, G, p.bar_flavor);
        PROF_STAMP();
        // all-finished check (every CTA reads the same flags after the barrier)
        if (tid == 0) {
          int alldone = 1;
          for (int b = 0; b < p.B; ++b) alldone &= __ldcg(p.finished + b);
          sm.flags[1] = alldone;
          if (alldone && cta == 0) *p.done = 1;
        }
        ptx::named_bar_sync(1, NCT);
        if (sm.flags[1]) break;
      }
    }
    // tell the producer to stop prefetching
    if (tid == 0) { *((volatile int*)&sm.flags[0]) = 1; sm.flags[3] = (int)cons_idx; }
  }
  __syncthreads();
  // drain: bulk copies issued beyond what was consumed must land before the CTA exits
  if (tid == 0) {
    const unsigned issued = (unsigned)sm.flags[2], consumed = (unsigned)sm.flags[3];
    for (unsigned n = consumed; n < issued; ++n)
      ptx::mbar_wait(&sm.full[n % p.nst], (n / p.nst) & 1u);
  }
  __syncthreads();
}

#include "gpt_decode1.cuh"
#include "gpt_decode8.cuh"

// -------------------------------------------------------------------- packing kernel --
struct PackUnit {
  const float* src;
  long long base;      // element offset of (k = 0)
  long long kstride;   // element stride along K
  long long row;       // row of the unit inside its 8-row chunk (swizzle key)
};
__global__ void pack_units_kernel(const PackUnit* units, __nv_bfloat16* dst, int D, long long n) {
  long long u = blockIdx.x;
  if (u >= n) return;
  PackUnit pu = units[u];
  const int r = (int)(pu.row & 7);
  for (int k = threadIdx.x; k < D; k += blockDim.x) {
    const int kp = (((k >> 3) ^ r) << 3) | (k & 7);   // 16-byte chunk index XOR row: ldmatrix bank spread
    dst[u * D + kp] = __float2bfloat16_rn(pu.src[pu.base + (long long)k * pu.kstride]);
  }
}

__global__ void round_bf16_kernel(float* x, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) x[i] = __bfloat162float(__float2bfloat16_rn(x[i]));
}

__global__ void concat_rows_kernel(float* dst, const float* src, int D, int rows) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < (size_t)rows * D) dst[i] = src[i];
}

// prepare_gpt_inputs (gpt/model_v2.py:648-714 + :754-768) for one utterance.
__global__ void prepare_inputs_kernel(const float* style, const float* emo_vec,
                                      const int* text_ids, int n_text, int lang,
                                      const float* spk_w, const float* spk_b,
                                      const float* text_emb, const float* text_pos,
                                      const float* lang_emb, int D, int r, float* out, int text_rows, int* bad) {
  const int row = blockIdx.x;
  for (int c = threadIdx.x; c < D; c += blockDim.x) {
    float v = 0.f;
    if (row == 0) {
      float acc = 0.f;
      for (int k = 0; k < 192; ++k) acc += rnd(style[k], r) * spk_w[(size_t)c * 192 + k];
      v = rnd(rnd(acc + spk_b[c], r) + emo_vec[c], r);
    } else if (row >= 3) {
      const int j = row - 3;
      int id = (j == 0) ? 0 : (j == n_text + 1 ? 1 : text_ids[j - 1]);
      if (id < 0 || id >= text_rows) {      // nn.Embedding raises IndexError here; flagged, never dereferenced
        if (c == 0) atomicCAS(bad, 0, j);
        id = 0;
      }
      v = rnd(text_emb[(size_t)id * D + c] + text_pos[(size_t)j * D + c], r);
      if (lang_emb) v = rnd(v + lang_emb[(size_t)lang * D + c], r);
    }
    out[(size_t)row * D + c] = v;
  }
}


// ============================================================================================
// Strict fp32 path (idx_gpt_config.weights_bf16 = 0): the reference's default `use_bf16=False`
// arithmetic (fp32 weights, fp32 activations, fp32 KV cache) as plain per-op kernels, one sequence
// at a time.  It exists for token-for-token parity against the fp32 oracle (DESIGN.md section 5); the
// fused persistent kernel above is the performance path.  Same call sites, same sampler contract.
// ============================================================================================
__global__ void strict_embed_kernel(float* x, const float* prompt_row, const float* mel_emb, const float* mel_pos,
                                    const int* tok, int posidx, int D) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= D) return;
  x[c] = prompt_row ? prompt_row[c] : mel_emb[(size_t)tok[0] * D + c] + mel_pos[(size_t)posidx * D + c];
}

// LayerNorm(eps 1e-5) of one row, statistics accumulated in double
__global__ void strict_ln_kernel(const float* x, const float* w, const float* b, float* y, int D) {
  __shared__ double sh[64];
  const int tid = threadIdx.x;
  double s = 0.0;
  for (int i = tid; i < D; i += blockDim.x) s += (double)x[i];
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((tid & 31) == 0) sh[tid >> 5] = s;
  __syncthreads();
  double tot = 0.0;
  for (int q = 0; q < (int)(blockDim.x >> 5); ++q) tot += sh[q];
  const double mean = tot / D;
  __syncthreads();
  double v = 0.0;
  for (int i = tid; i < D; i += blockDim.x) { const double d = (double)x[i] - mean; v += d * d; }
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((tid & 31) == 0) sh[32 + (tid >> 5)] = v;
  __syncthreads();
  double vt = 0.0;
  for (int q = 0; q < (int)(blockDim.x >> 5); ++q) vt += sh[32 + q];
  const float rstd = (float)(1.0 / sqrt(vt / D + 1e-5));
  const float mf = (float)mean;
  for (int i = tid; i < D; i += blockDim.x) y[i] = (x[i] - mf) * rstd * w[i] + b[i];
}

// y[c] = act(sum_k x[k] W[k][c] + bias[c]) (+ res[c]);  W is HF Conv1D [K][N] (trap P4).  Block (32, 32):
// warp ty owns k = ty, ty + 32, ...; a warp reads one 128-byte row segment per k.
__global__ void strict_gemv_kn_kernel(const float* __restrict__ x, const float* __restrict__ W,
                                      const float* __restrict__ bias, const float* res, float* y, int K, int N, int act) {
  __shared__ float part[32][33];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int c = blockIdx.x * 32 + tx;
  float acc = 0.f;
  if (c < N)
    for (int k = ty; k < K; k += 32) acc = fmaf(x[k], W[(size_t)k * N + c], acc);
  part[ty][tx] = acc;
  __syncthreads();
  if (ty == 0 && c < N) {
    float s = 0.f;
#pragma unroll
    for (int q = 0; q < 32; ++q) s += part[q][tx];
    s += bias[c];
    if (act == 1) s = gelu_new(s, 0);
    if (res) s += res[c];
    y[c] = s;
  }
}

// nn.Linear [N][K]: one warp per output row
__global__ void strict_gemv_nk_kernel(const float* __restrict__ x, const float* __restrict__ W,
                                      const float* __restrict__ bias, float* y, int K, int N) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= N) return;
  float acc = 0.f;
  for (int k = lane; k < K; k += 32) acc = fmaf(x[k], W[(size_t)row * K + k], acc);
  acc = warp_sum(acc);
  if (lane == 0) y[row] = acc + bias[row];
}

// one head per block: append (k, v) of this position to the fp32 cache, softmax(q k^T / 8) v over positions 0..pos
__global__ void strict_attn_kernel(const float* qkv, float* kc, float* vc, int pos, float* out, int D) {
  extern __shared__ float sc[];           // [pos + 1] scores, then [128] merge buffer
  __shared__ float redv[8];
  const int h = blockIdx.x, tid = threadIdx.x;
  if (tid < HD) {
    kc[(size_t)pos * D + h * HD + tid] = qkv[D + h * HD + tid];
    vc[(size_t)pos * D + h * HD + tid] = qkv[2 * D + h * HD + tid];
  }
  __syncthreads();
  const float* q = qkv + h * HD;
  float mx = -INFINITY;
  for (int j = tid; j <= pos; j += blockDim.x) {
    const float* kr = kc + (size_t)j * D + h * HD;
    float s = 0.f;
#pragma unroll 8
    for (int d = 0; d < HD; ++d) s = fmaf(q[d], kr[d], s);
    s *= 0.125f;
    sc[j] = s;
    mx = fmaxf(mx, s);
  }
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((tid & 31) == 0) redv[tid >> 5] = mx;
  __syncthreads();
  mx = redv[0];
  for (int q2 = 1; q2 < (int)(blockDim.x >> 5); ++q2) mx = fmaxf(mx, redv[q2]);
  __syncthreads();
  float sum = 0.f;
  for (int j = tid; j <= pos; j += blockDim.x) { const float p = expf(sc[j] - mx); sc[j] = p; sum += p; }
  sum = warp_sum(sum);
  if ((tid & 31) == 0) redv[4 + (tid >> 5)] = sum;
  __syncthreads();
  float tot = 0.f;
  for (int q2 = 0; q2 < (int)(blockDim.x >> 5); ++q2) tot += redv[4 + q2];
  const int d = tid & (HD - 1), half = tid / HD;      // 128 threads: two interleaved halves of the positions
  float acc = 0.f;
  for (int j = half; j <= pos; j += 2) acc = fmaf(sc[j], vc[(size_t)j * D + h * HD + d], acc);
  float* mg = sc + pos + 1;
  mg[tid] = acc;
  __syncthreads();
  if (tid < HD) out[h * HD + tid] = (mg[tid] + mg[tid + HD]) / tot;
}

// RepetitionPenalty -> (forbid stop) -> [Temperature -> TopK -> TopP -> multinomial | argmax]; same order, tie rules
// and Philox contract as the sampling phase of the fused kernel.
__global__ void strict_sample_kernel(const float* logits, unsigned* seen, int V, int k, int seq, float rep_penalty,
                                     int stop_tok, int forbid_stop_before, int do_sample, int top_k, float top_p,
                                     float temperature, unsigned long long seed, int* codes, int max_new, int* nout,
                                     int* finished, int* tok, const int* forced, float* ldump, int* flag) {
  extern __shared__ float sv[];            // [V] processed scores
  __shared__ float rb[16];
  __shared__ int ri[16];
  __shared__ float cv[CMAX];
  __shared__ int ci[CMAX];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  const float inv_temp = (do_sample && temperature > 0.f) ? 1.0f / temperature : 1.0f;
  for (int i = tid; i < V; i += blockDim.x) {
    float s = logits[i];
    if (ldump) ldump[i] = s;
    if ((seen[i >> 5] >> (i & 31)) & 1u) s = (s < 0.f) ? s * rep_penalty : s / rep_penalty;
    if (i == stop_tok && k < forbid_stop_before) s = -INFINITY;
    if (do_sample) s *= inv_temp;
    sv[i] = s;
  }
  __syncthreads();
  auto block_argmax = [&](float& bestv, int& besti) {
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = tid; i < V; i += blockDim.x)
      if (sv[i] > best || (sv[i] == best && i < bi && sv[i] > -INFINITY)) { best = sv[i]; bi = i; }
    for (int o = 16; o > 0; o >>= 1) {
      const float b2 = __shfl_xor_sync(0xffffffffu, best, o);
      const int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
      if (b2 > best || (b2 == best && i2 < bi)) { best = b2; bi = i2; }
    }
    __syncthreads();
    if (lane == 0) { rb[warp] = best; ri[warp] = bi; }
    __syncthreads();
    for (int w = 0; w < nw; ++w)
      if (w == 0 || rb[w] > best || (rb[w] == best && ri[w] < bi)) { best = rb[w]; bi = ri[w]; }
    bestv = best; besti = bi;
  };
  float best; int besti;
  block_argmax(best, besti);
  if (do_sample) {
    const int kk = min(max(top_k, 1), CMAX);
    int nc = 0;
    float kth = best;
    while (nc < CMAX && best > -INFINITY && (nc < kk || best == kth)) {
      if (tid == 0) { cv[nc] = best; ci[nc] = besti; sv[besti] = -INFINITY; }
      if (nc < kk) kth = best;
      ++nc;
      __syncthreads();
      block_argmax(best, besti);
    }
    // more than CMAX tokens tie at the k-th score: TopKLogitsWarper would keep them all, so the call is refused
    if (tid == 0 && nc == CMAX && best == kth && best > -INFINITY && !finished[0]) *flag = k + 1;
    __syncthreads();
    if (tid == 0) {
      const float mx = cv[0];
      float tot = 0.f;
      for (int i = 0; i < nc; ++i) { cv[i] = expf(cv[i] - mx); tot += cv[i]; }
      int keep = nc;
      if (top_p < 1.0f) {
        float tail = 0.f;
        for (int i = nc - 1; i >= 1; --i) {
          tail += cv[i] / tot;
          if (tail <= 1.0f - top_p) keep = i; else break;
        }
      }
      float kt = 0.f;
      for (int i = 0; i < keep; ++i) kt += cv[i];
      unsigned rnd4[4];
      philox4x32_10(seed, (unsigned)k, (unsigned)seq, rnd4);
      const float u = (float)(rnd4[0] >> 8) * (1.0f / 16777216.0f) * kt;
      float acc = 0.f;
      int pick = keep - 1;
      for (int i = 0; i < keep; ++i) { acc += cv[i]; if (u < acc) { pick = i; break; } }
      besti = ci[pick];
    }
  }
  if (tid == 0 && !finished[0]) {
    codes[k] = besti;
    nout[0] = k + 1;
    int feed = besti;
    if (forced) feed = forced[k];
    else if (besti == stop_tok) finished[0] = 1;
    if (k + 1 >= max_new) finished[0] = 1;
    tok[0] = feed;
    seen[feed >> 5] |= 1u << (feed & 31);
  }
}


// ============================================================================================
// Beam-sample (the reference's default decoding mode: num_beams = 3, do_sample = True).
// `GenerationMixin._beam_search` transformers_generation_utils.py:3325-3609 + `BeamSearchScorer.process`
// transformers_beam_search.py:215-320 + `BeamHypotheses` :930-1010, one CTA per utterance, run between
// single-step launches of the fused kernel (which then skips its own sampling phase: ext_sample).
// The beams are rows u*m .. u*m+m-1 of the fused kernel; instead of HF's index_select of the KV cache, row i
// keeps writing into its own cache slot and `phys[i][t]` names the slot that holds generated position t of its
// lineage (prompt positions live once, in the utterance's first slot).
// RNG contract (DESIGN.md section 5, oracle/beam.py): 2m successive draws without replacement by inverse CDF over the
// union of the kept candidates (beam-major, descending score), Philox counter (step, 0x10000 + 16 u + draw).
// ============================================================================================
struct BeamParams {
  const float* logits;     // [8][V]
  int V, m, k, max_new, stop_tok, forbid_stop_before, top_k, hist_stride, utt_base;
  float rep_penalty, inv_temp, top_p;
  double length_penalty;
  unsigned long long seed;
  int do_sample;
  float* beam_scores;                              // [8]
  const unsigned* seen_cur; unsigned* seen_nxt;    // [8][wv]
  const int* hist_cur; int* hist_nxt;              // [8][hist_stride]
  const unsigned char* phys_cur; unsigned char* phys_nxt;   // [8][hist_stride]
  int* tok;                                        // [8]
  double* hyp_score;  // [nutt][m+1]
  int* hyp_len;       // [nutt][m+1]
  int* hyp_tok;       // [nutt][m+1][hist_stride]
  int* hyp_order;     // [nutt][m+1] physical slots in list order
  int* nhyp;          // [nutt]
  double* worst;      // [nutt]
  int* done_u;        // [nutt]
  float* ldump;       // [max_new][8][V] or null
  int* flag;          // engine error word: set to step + 1 when more than CMAX tokens tie at the top-k boundary
  int* trace_pt;     // [max_new][8][2] or null
  float* trace_sc;    // [max_new][8] or null
};

constexpr int BEAM_MAX = 4;

__global__ void __launch_bounds__(256) beam_step_kernel(const BeamParams p) {
  constexpr int VPT = 40;
  __shared__ float red[16];
  __shared__ int redi[16];
  __shared__ float cs[BEAM_MAX][CMAX];   // processed score (+ beam score after top-p)
  __shared__ int ci[BEAM_MAX][CMAX];
  __shared__ int keepn[BEAM_MAX];
  __shared__ float nb_score[BEAM_MAX];
  __shared__ int nb_tok[BEAM_MAX], nb_par[BEAM_MAX];
  __shared__ int sh_done;
  const int u = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int V = p.V, m = p.m, k = p.k, wv = (V + 31) / 32, hs = p.hist_stride;
  const int r0 = u * m;

  if (p.done_u[u]) {
    // finished utterance: identity reorder, pad token (transformers_beam_search.py:258-266)
    for (int i = 0; i < m; ++i) {
      const int r = r0 + i;
      for (int t = tid; t <= k; t += 256) {
        p.phys_nxt[r * hs + t] = p.phys_cur[r * hs + t];
        if (t < k) p.hist_nxt[r * hs + t] = p.hist_cur[r * hs + t];
      }
      for (int t = tid; t < wv; t += 256) p.seen_nxt[(size_t)r * wv + t] = p.seen_cur[(size_t)r * wv + t];
      if (tid == 0) {
        p.hist_nxt[r * hs + k] = p.stop_tok;
        p.phys_nxt[r * hs + k + 1] = (unsigned char)r;
        p.tok[r] = p.stop_tok;
        if (p.trace_pt) {           // the trace records the identity reorder too (the beam score is left as it was)
          p.trace_pt[((size_t)k * 8 + r) * 2] = i;
          p.trace_pt[((size_t)k * 8 + r) * 2 + 1] = p.stop_tok;
          p.trace_sc[(size_t)k * 8 + r] = p.beam_scores[r];
        }
      }
    }
    return;
  }

  auto block_max = [&](float v) {
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float r = red[0];
    for (int w = 1; w < 8; ++w) r = fmaxf(r, red[w]);
    return r;
  };
  auto block_sum = [&](float v) {
    v = warp_sum(v);
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float r = 0.f;
    for (int w = 0; w < 8; ++w) r += red[w];
    return r;
  };

  // ---- phase A: per beam, processed scores and the kept candidate list ----
  for (int j = 0; j < m; ++j) {
    const int r = r0 + j;
    const float* lg = p.logits + (size_t)r * V;
    const unsigned* seen = p.seen_cur + (size_t)r * wv;
    float sv[VPT];
    float mx = -INFINITY;
#pragma unroll
    for (int q = 0; q < VPT; ++q) {
      const int i = tid + q * 256;
      sv[q] = (i < V) ? __ldcg(lg + i) : -INFINITY;
      mx = fmaxf(mx, sv[q]);
    }
    if (p.ldump)
      for (int q = 0; q < VPT; ++q) {
        const int i = tid + q * 256;
        if (i < V) p.ldump[((size_t)k * 8 + r) * V + i] = sv[q];
      }
    mx = block_max(mx);
    float se = 0.f;
#pragma unroll
    for (int q = 0; q < VPT; ++q)
      if (tid + q * 256 < V) se += expf(sv[q] - mx);
    se = block_sum(se);
    const float lse = mx + logf(se);
#pragma unroll
    for (int q = 0; q < VPT; ++q) {
      const int i = tid + q * 256;
      if (i < V) {
        float s = sv[q] - lse;                                             // log_softmax
        if ((seen[i >> 5] >> (i & 31)) & 1u) s = (s < 0.f) ? s * p.rep_penalty : s / p.rep_penalty;
        if (i == p.stop_tok && k < p.forbid_stop_before) s = -INFINITY;
        sv[q] = s * p.inv_temp;
      }
    }
    auto block_argmax = [&](float& bestv, int& besti) {
      float best = -INFINITY;
      int bi = 0x7fffffff;
#pragma unroll
      for (int q = 0; q < VPT; ++q) {
        const int i = tid + q * 256;
        if (sv[q] > best || (sv[q] == best && i < bi && sv[q] > -INFINITY)) { best = sv[q]; bi = i; }
      }
      for (int o = 16; o > 0; o >>= 1) {
        const float b2 = __shfl_xor_sync(0xffffffffu, best, o);
        const int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
        if (b2 > best || (b2 == best && i2 < bi)) { best = b2; bi = i2; }
      }
      __syncthreads();
      if (lane == 0) { red[warp] = best; redi[warp] = bi; }
      __syncthreads();
      for (int w = 0; w < 8; ++w)
        if (w == 0 || red[w] > best || (red[w] == best && redi[w] < bi)) { best = red[w]; bi = redi[w]; }
      bestv = best; besti = bi;
    };
    float best; int besti;
    block_argmax(best, besti);
    const int kk = (p.top_k > 0) ? min(max(p.top_k, 2), CMAX) : CMAX;  // min_tokens_to_keep = 2 with beams; plain beam search (top_k = 0) keeps CMAX >= 2m candidates per beam
    int nc = 0;
    float kth = best;
    while (nc < CMAX && best > -INFINITY && (nc < kk || best == kth)) {
      if (tid == 0) { cs[j][nc] = best; ci[j][nc] = besti; }
      if (nc < kk) kth = best;
      ++nc;
#pragma unroll
      for (int q = 0; q < VPT; ++q)
        if (tid + q * 256 == besti) sv[q] = -INFINITY;
      block_argmax(best, besti);
    }
    // beam-sample top-k keeps every tie at the k-th score; more than CMAX of them is refused (plain beam search,
    // top_k = 0, needs only the best 2m candidates and keeps no ties)
    if (tid == 0 && p.top_k > 0 && nc == CMAX && best == kth && best > -INFINITY) *p.flag = k + 1;
    __syncthreads();
    if (tid == 0) {
      int keep = nc;
      if (p.top_p < 1.0f) {
        float ev[CMAX];
        const float m0 = cs[j][0];
        float tot = 0.f;
        for (int i = 0; i < nc; ++i) { ev[i] = expf(cs[j][i] - m0); tot += ev[i]; }
        float tail = 0.f;
        for (int i = nc - 1; i >= 2; --i) {
          tail += ev[i] / tot;
          if (tail <= 1.0f - p.top_p) keep = i; else break;
        }
      }
      keepn[j] = keep;
      const float bsc = p.beam_scores[r];
      for (int i = 0; i < keep; ++i) cs[j][i] += bsc;
    }
    __syncthreads();
  }

  // ---- phase B (thread 0): union -> 2m draws without replacement -> sort -> scorer.process ----
  if (tid == 0) {
    float w[BEAM_MAX * CMAX];
    unsigned char used[BEAM_MAX * CMAX];
    int ub[BEAM_MAX + 1];
    ub[0] = 0;
    for (int j = 0; j < m; ++j) ub[j + 1] = ub[j] + keepn[j];
    const int nu = ub[m];
    auto usc = [&](int i) { int j = 0; while (i >= ub[j + 1]) ++j; return cs[j][i - ub[j]]; };
    auto utok = [&](int i) { int j = 0; while (i >= ub[j + 1]) ++j; return ci[j][i - ub[j]]; };
    auto upar = [&](int i) { int j = 0; while (i >= ub[j + 1]) ++j; return j; };
    float umax = -INFINITY;
    for (int i = 0; i < nu; ++i) umax = fmaxf(umax, usc(i));
    for (int i = 0; i < nu; ++i) { w[i] = expf(usc(i) - umax); used[i] = 0; }
    int picks[2 * BEAM_MAX];
    const int nd = 2 * m;
    for (int d = 0; d < nd; ++d) {
      float tot = 0.f;
      for (int i = 0; i < nu; ++i) if (!used[i]) tot += w[i];
      int pick = -1;
      if (tot > 0.f && p.do_sample) {      // do_sample = 0: plain beam search = torch.topk of the union (:3527-3530)
        unsigned rnd4[4];
        philox4x32_10(p.seed, (unsigned)k, 0x10000u + 16u * (unsigned)(u + p.utt_base) + (unsigned)d, rnd4);
        const float uu = (float)(rnd4[0] >> 8) * (1.0f / 16777216.0f) * tot;
        float acc = 0.f;
        int last = -1;
        for (int i = 0; i < nu; ++i) {
          if (used[i] || w[i] == 0.f) continue;
          acc += w[i]; last = i;
          if (uu < acc) { pick = i; break; }
        }
        if (pick < 0) pick = last;
      }
      if (pick < 0) {       // fewer positive-probability candidates than draws: best remaining score, lowest index
        for (int i = 0; i < nu; ++i)
          if (!used[i] && (pick < 0 || usc(i) > usc(pick))) pick = i;
      }
      used[pick] = 1;
      picks[d] = pick;
    }
    for (int a = 1; a < nd; ++a) {          // stable insertion sort, descending score
      const int x = picks[a];
      int b = a - 1;
      while (b >= 0 && usc(picks[b]) < usc(x)) { picks[b + 1] = picks[b]; --b; }
      picks[b + 1] = x;
    }
    // scorer.process
    const int gen_len = k + 1;
    const double lp_den = pow((double)gen_len, p.length_penalty);
    double* hs_ = p.hyp_score + (size_t)u * (m + 1);
    int* hl = p.hyp_len + (size_t)u * (m + 1);
    int* ho = p.hyp_order + (size_t)u * (m + 1);
    int nh = p.nhyp[u];
    double worst = p.worst[u];
    int nbn = 0;
    for (int rank = 0; rank < nd && nbn < m; ++rank) {
      const int i = picks[rank];
      const int tk = utok(i), par = upar(i);
      const float sc = usc(i);
      if (tk == p.stop_tok) {
        if (rank >= m) continue;
        const double score = (double)sc / lp_den;
        if (nh < m || score > worst) {
          // free physical slot = the one not in the order list
          bool taken[BEAM_MAX + 1];
          for (int q = 0; q <= m; ++q) taken[q] = false;
          for (int q = 0; q < nh; ++q) taken[ho[q]] = true;
          int slot = 0;
          while (taken[slot]) ++slot;
          hs_[slot] = score;
          hl[slot] = k;
          const int* src = p.hist_cur + (size_t)(r0 + par) * hs;
          int* dst = p.hyp_tok + ((size_t)u * (m + 1) + slot) * hs;
          for (int t = 0; t < k; ++t) dst[t] = src[t];
          ho[nh++] = slot;
          if (nh > m) {
            int lo = 0;                         // smallest (score, list index)
            for (int q = 1; q < nh; ++q) if (hs_[ho[q]] < hs_[ho[lo]]) lo = q;
            for (int q = lo; q + 1 < nh; ++q) ho[q] = ho[q + 1];
            --nh;
            double w2 = hs_[ho[0]];
            for (int q = 1; q < nh; ++q) w2 = fmin(w2, hs_[ho[q]]);
            worst = w2;
          } else {
            worst = fmin(score, worst);
          }
        }
      } else {
        nb_score[nbn] = sc; nb_tok[nbn] = tk; nb_par[nbn] = par;
        ++nbn;
      }
    }
    // (nbn == m always: every beam keeps >= 2 candidates, so at most m of the 2m draws can be the stop token)
    p.nhyp[u] = nh;
    p.worst[u] = worst;
    int done = 0;
    if (nh >= m) {
      const double highest = (double)usc(picks[0]) / lp_den;
      done = worst >= highest;
    }
    sh_done = done;
    p.done_u[u] = done;
  }
  __syncthreads();

  // ---- phase C: reorder histories, cache maps and repetition bitmaps; publish the next inputs ----
  for (int i = 0; i < m; ++i) {
    const int r = r0 + i, pr = r0 + nb_par[i], tk = nb_tok[i];
    for (int t = tid; t <= k; t += 256) {
      p.phys_nxt[r * hs + t] = p.phys_cur[pr * hs + t];
      if (t < k) p.hist_nxt[r * hs + t] = p.hist_cur[pr * hs + t];
    }
    for (int t = tid; t < wv; t += 256) {
      unsigned v = p.seen_cur[(size_t)pr * wv + t];
      if (t == (tk >> 5)) v |= 1u << (tk & 31);
      p.seen_nxt[(size_t)r * wv + t] = v;
    }
    if (tid == 0) {
      p.hist_nxt[r * hs + k] = tk;
      p.phys_nxt[r * hs + k + 1] = (unsigned char)r;
      p.tok[r] = tk;
      p.beam_scores[r] = nb_score[i];
      if (p.trace_pt) {
        p.trace_pt[((size_t)k * 8 + r) * 2] = nb_par[i];
        p.trace_pt[((size_t)k * 8 + r) * 2 + 1] = tk;
        p.trace_sc[(size_t)k * 8 + r] = nb_score[i];
      }
    }
  }
}

}  // namespace

// ------------------------------------------------------------------------ host state --
struct GptStrict;
struct GptState {
  idx_gpt_config cfg;
  GptStrict* strict = nullptr;   // fp32 per-op path (weights_bf16 = 0)
  struct BeamTrace* beam_trace = nullptr;
  int seq_base = 0;             // first request of the decode group being run (idx_gpt_generate splits large calls)
  int G = 0, FF = 0, nst1 = 0, nst8 = 0, bias_cap = 0, ocap = 0, bar_flavor = 0;
  size_t smem1 = 0, smem8 = 0;
  __nv_bfloat16* wstream = nullptr;
  long long* stream_off = nullptr;
  float *ln1_w = nullptr, *ln1_b = nullptr, *ln2_w = nullptr, *ln2_b = nullptr;
  float *qkv_b = nullptr, *o_b = nullptr, *fc_b = nullptr, *proj_b = nullptr;
  float *mel_emb = nullptr, *mel_pos = nullptr;
  __nv_bfloat16 *kc = nullptr, *vc = nullptr;
  int maxpos = 0;
  float *xg = nullptr, *qg = nullptr, *part = nullptr, *logits = nullptr;
  uint2* xt = nullptr;          // tagged residual stream (batch-1 decode)
  unsigned* ft = nullptr;       // tagged gelu(fc) words
  uint2 *qt = nullptr, *kvt = nullptr;
  unsigned* pflag = nullptr;
  // second-generation batch-1 decode kernel
  int v2 = 0, ring_rows = 0;
  int v8 = 0, ring_rows8 = 0;       // gpt_decode8_kernel (2..8 sequences per group)
  size_t smem_v8 = 0;
  size_t smem_v2 = 0;
  __nv_bfloat16* wstream1 = nullptr;
  long long* stream_off1 = nullptr;
  uint2 *ot = nullptr, *partt = nullptr, *cand = nullptr, *tokt = nullptr;
  unsigned epoch = 0;           // epochs handed out so far
  int dataflow = 1;
  __nv_bfloat16* fg = nullptr;
  int *tok = nullptr, *nout = nullptr, *finished = nullptr, *prompt_len = nullptr, *done = nullptr;
  unsigned* seen = nullptr;
  unsigned* barrier = nullptr;
  long long* prof = nullptr;
  long long* prof2 = nullptr;
  int prof_on = 0;
  // attention probe armed by idx_gpt_probe_attention for the next generate call (caller buffers, host or device)
  int probe_armed = 0, probe_layer = -1, probe_steps = 0, probe_seqs = 0;
  float* probe_out = nullptr;
  int32_t* probe_ns_out = nullptr;
  // prefill probe armed by idx_gpt_probe_prefill for the next generate call
  int pprobe_armed = 0, pprobe_layer = -1, pprobe_rows = 0, pprobe_seqs = 0;
  float* pprobe_out = nullptr;
  std::vector<void*> owned;
  double t_prefill_ms = 0, t_decode_ms = 0;
  int last_steps = 0, last_launches = 0;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev2 = nullptr;
};

static void beam_trace_free(GptState* g);
void gpt_destroy(GptState* g) {
  if (!g) return;
  delete g->strict;
  beam_trace_free(g);
  for (void* p : g->owned) cudaFree(p);
  if (g->ev0) cudaEventDestroy(g->ev0);
  if (g->ev1) cudaEventDestroy(g->ev1);
  if (g->ev2) cudaEventDestroy(g->ev2);
  delete g;
}

template <typename T>
static T* galloc(GptState* g, size_t n) {
  T* p = nullptr;
  IDX_CUDA(cudaMalloc((void**)&p, n * sizeof(T)));
  IDX_CUDA(cudaMemset(p, 0, n * sizeof(T)));
  g->owned.push_back(p);
  return p;
}

// the samplers' error flag: a top-k boundary tie wider than the CMAX candidate slots
static const char* const kTieOverflow = "more than 128 tokens tie at the top-k boundary";

// ------------------------------------------------------------------ strict fp32 host path --
struct StrictLayer {
  const float *ln1_w, *ln1_b, *wqkv, *bqkv, *wo, *bo, *ln2_w, *ln2_b, *wfc, *bfc, *wproj, *bproj;
};
struct GptStrict {
  std::vector<StrictLayer> layers;
  float *kc = nullptr, *vc = nullptr;                 // [L][maxpos][D] fp32, one sequence at a time
  float *x = nullptr, *h = nullptr, *qkv = nullptr, *att = nullptr, *f = nullptr, *logits = nullptr;
};

static void strict_init(idx_engine* e, GptState* g) {
  const idx_gpt_config& c = g->cfg;
  const int L = c.layers, D = c.model_dim, V = c.number_mel_codes, FF = 4 * D;
  GptStrict* s = new GptStrict();
  g->strict = s;
  auto lname = [&](int l, const char* n) { return "gpt.gpt.h." + std::to_string(l) + "." + n; };
  for (int l = 0; l < L; ++l) {
    StrictLayer y;
    IDX_CHECK(e->W(lname(l, "attn.c_attn.weight")).numel() == (size_t)D * 3 * D, IDX_ERR_ARG, "c_attn.weight shape");
    IDX_CHECK(e->W(lname(l, "mlp.c_fc.weight")).numel() == (size_t)D * FF, IDX_ERR_ARG, "c_fc.weight shape");
    y.ln1_w = e->Wf(lname(l, "ln_1.weight")); y.ln1_b = e->Wf(lname(l, "ln_1.bias"));
    y.wqkv = e->Wf(lname(l, "attn.c_attn.weight")); y.bqkv = e->Wf(lname(l, "attn.c_attn.bias"));
    y.wo = e->Wf(lname(l, "attn.c_proj.weight")); y.bo = e->Wf(lname(l, "attn.c_proj.bias"));
    y.ln2_w = e->Wf(lname(l, "ln_2.weight")); y.ln2_b = e->Wf(lname(l, "ln_2.bias"));
    y.wfc = e->Wf(lname(l, "mlp.c_fc.weight")); y.bfc = e->Wf(lname(l, "mlp.c_fc.bias"));
    y.wproj = e->Wf(lname(l, "mlp.c_proj.weight")); y.bproj = e->Wf(lname(l, "mlp.c_proj.bias"));
    s->layers.push_back(y);
  }
  IDX_CHECK(e->W("gpt.mel_head.weight").numel() == (size_t)V * D, IDX_ERR_ARG, "mel_head.weight shape");
  g->maxpos = c.max_prompt + c.max_mel_positions + 8;
  s->kc = galloc<float>(g, (size_t)L * g->maxpos * D);
  s->vc = galloc<float>(g, (size_t)L * g->maxpos * D);
  s->x = galloc<float>(g, D); s->h = galloc<float>(g, D); s->qkv = galloc<float>(g, 3 * (size_t)D);
  s->att = galloc<float>(g, D); s->f = galloc<float>(g, FF); s->logits = galloc<float>(g, V);
  g->tok = galloc<int>(g, 8); g->nout = galloc<int>(g, 8); g->finished = galloc<int>(g, 8);
  g->seen = galloc<unsigned>(g, (size_t)((V + 31) / 32));
  IDX_CUDA(cudaFuncSetAttribute(strict_attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
  IDX_CHECK((size_t)(g->maxpos + 129) * 4 <= 96 * 1024, IDX_ERR_ARG, "context too long for the strict attention kernel");
}

// one position through the 24 blocks (x in s->x, updated in place); pos = its index in the KV cache
static void strict_layers(idx_engine* e, GptState* g, int pos) {
  GptStrict* s = g->strict;
  const int D = g->cfg.model_dim, H = g->cfg.heads, FF = 4 * D;
  cudaStream_t st = e->stream;
  const dim3 blk(32, 32);
  for (int l = 0; l < g->cfg.layers; ++l) {
    const StrictLayer& y = s->layers[l];
    float* kc = s->kc + (size_t)l * g->maxpos * D;
    float* vc = s->vc + (size_t)l * g->maxpos * D;
    strict_ln_kernel<<<1, 256, 0, st>>>(s->x, y.ln1_w, y.ln1_b, s->h, D);
    strict_gemv_kn_kernel<<<(3 * D + 31) / 32, blk, 0, st>>>(s->h, y.wqkv, y.bqkv, nullptr, s->qkv, D, 3 * D, 0);
    strict_attn_kernel<<<H, 128, (size_t)(pos + 1 + 128) * 4, st>>>(s->qkv, kc, vc, pos, s->att, D);
    strict_gemv_kn_kernel<<<(D + 31) / 32, blk, 0, st>>>(s->att, y.wo, y.bo, s->x, s->x, D, D, 0);
    strict_ln_kernel<<<1, 256, 0, st>>>(s->x, y.ln2_w, y.ln2_b, s->h, D);
    strict_gemv_kn_kernel<<<(FF + 31) / 32, blk, 0, st>>>(s->h, y.wfc, y.bfc, nullptr, s->f, D, FF, 1);
    strict_gemv_kn_kernel<<<(D + 31) / 32, blk, 0, st>>>(s->f, y.wproj, y.bproj, s->x, s->x, FF, D, 0);
    e->launches += 7;
    g->last_launches += 7;
  }
  IDX_CUDA(cudaGetLastError());
}

static void strict_generate(idx_engine* e, GptState* g, const idx_gpt_request* reqs, int nreq, const idx_sampling* sp) {
  GptStrict* s = g->strict;
  const idx_gpt_config& c = g->cfg;
  const int D = c.model_dim, V = c.number_mel_codes, max_new = sp->max_new_tokens;
  cudaStream_t st = e->stream;
  const size_t wv = (size_t)((V + 31) / 32);
  const float* mel_emb = e->Wf("gpt.mel_embedding.weight");
  const float* mel_pos = e->Wf("gpt.mel_pos_embedding.emb.weight");
  int maxn = 0;
  IDX_CUDA(cudaEventRecord(g->ev0, st));
  IDX_CUDA(cudaEventRecord(g->ev1, st));
  for (int i = 0; i < nreq; ++i) {
    const int plen = reqs[i].prompt_len;
    IDX_CHECK(reqs[i].prompt_emb && plen >= 1 && plen <= c.max_prompt, IDX_ERR_ARG, "bad prompt");
    IDX_CHECK(plen + max_new + 1 <= g->maxpos, IDX_ERR_ARG, "KV cache too small");
    size_t need = (size_t)plen * D * 4 + 2 * (size_t)max_new * 4 + 4096;
    if (reqs[i].logits_out) need += (size_t)max_new * V * 4;
    e->ensure_arena(need + (1 << 20));
    e->arena.reset();
    float* d_prompt = e->arena.get<float>((size_t)plen * D);
    int* d_codes = e->arena.get<int>(max_new);
    int* d_forced = reqs[i].forced_codes ? e->arena.get<int>(max_new) : nullptr;
    float* d_ldump = reqs[i].logits_out ? e->arena.get<float>((size_t)max_new * V) : nullptr;
    idx_to_device(e, d_prompt, reqs[i].prompt_emb, (size_t)plen * D * 4);
    if (d_forced) idx_to_device(e, d_forced, reqs[i].forced_codes, (size_t)max_new * 4);
    {
      std::vector<unsigned> h_seen(wv, 0u);
      h_seen[1 >> 5] |= 1u << 1;                                            // trap P2: fake ids {1, start_mel}
      h_seen[c.start_mel_token >> 5] |= 1u << (c.start_mel_token & 31);
      const int h_tok = c.start_mel_token, zero = 0;
      IDX_CUDA(cudaMemcpyAsync(g->seen, h_seen.data(), wv * 4, cudaMemcpyHostToDevice, st));
      IDX_CUDA(cudaMemcpyAsync(g->tok, &h_tok, 4, cudaMemcpyHostToDevice, st));
      IDX_CUDA(cudaMemcpyAsync(g->nout, &zero, 4, cudaMemcpyHostToDevice, st));
      IDX_CUDA(cudaMemcpyAsync(g->finished, &zero, 4, cudaMemcpyHostToDevice, st));
      IDX_CUDA(cudaStreamSynchronize(st));
    }
    for (int pos = 0; pos < plen; ++pos) {                                   // prompt positions, one at a time
      strict_embed_kernel<<<(D + 255) / 256, 256, 0, st>>>(s->x, d_prompt + (size_t)pos * D, nullptr, nullptr, nullptr, 0, D);
      strict_layers(e, g, pos);
    }
    int* h_fin = (int*)e->pinned_buf(64);
    int k = 0;
    for (; k < max_new; ++k) {
      strict_embed_kernel<<<(D + 255) / 256, 256, 0, st>>>(s->x, nullptr, mel_emb, mel_pos, g->tok, (k == 0 || sp->mel_pos_mode == 1) ? k : k + 1, D);   // trap P1 / no-cache rule
      strict_layers(e, g, plen + k);
      strict_ln_kernel<<<1, 256, 0, st>>>(s->x, e->Wf("gpt.gpt.ln_f.weight"), e->Wf("gpt.gpt.ln_f.bias"), s->h, D);
      strict_ln_kernel<<<1, 256, 0, st>>>(s->h, e->Wf("gpt.final_norm.weight"), e->Wf("gpt.final_norm.bias"), s->att, D);   // trap P3
      strict_gemv_nk_kernel<<<(V + 7) / 8, 256, 0, st>>>(s->att, e->Wf("gpt.mel_head.weight"), e->Wf("gpt.mel_head.bias"), s->logits, D, V);
      strict_sample_kernel<<<1, 256, (size_t)V * 4, st>>>(s->logits, g->seen, V, k, i + g->seq_base, sp->repetition_penalty, c.stop_mel_token,
                                                          sp->forbid_stop_before, sp->do_sample, sp->top_k, sp->top_p,
                                                          sp->temperature, sp->seed, d_codes, max_new, g->nout, g->finished,
                                                          g->tok, d_forced, d_ldump ? d_ldump + (size_t)k * V : nullptr,
                                                          e->dev_flag);
      IDX_CUDA(cudaGetLastError());
      e->launches += 5;
      g->last_launches += 5;
      IDX_CUDA(cudaMemcpyAsync(h_fin, g->finished, 4, cudaMemcpyDeviceToHost, st));
      IDX_CUDA(cudaStreamSynchronize(st));
      if (*h_fin) break;
    }
    e->check_flag(kTieOverflow);
    int h_nout = 0;
    IDX_CUDA(cudaMemcpyAsync(&h_nout, g->nout, 4, cudaMemcpyDeviceToHost, st));
    IDX_CUDA(cudaStreamSynchronize(st));
    maxn = std::max(maxn, h_nout);
    if (reqs[i].n_codes_out) *reqs[i].n_codes_out = h_nout;
    if (reqs[i].codes_out) idx_from_device(e, reqs[i].codes_out, d_codes, (size_t)h_nout * 4);
    if (reqs[i].logits_out) idx_from_device(e, reqs[i].logits_out, d_ldump, (size_t)h_nout * V * 4);
    IDX_CUDA(cudaStreamSynchronize(st));
  }
  IDX_CUDA(cudaEventRecord(g->ev2, st));
  IDX_CUDA(cudaStreamSynchronize(st));
  float ms = 0;
  IDX_CUDA(cudaEventElapsedTime(&ms, g->ev0, g->ev2));
  g->t_prefill_ms = 0;
  g->t_decode_ms = ms;
  g->last_steps = maxn;
}

static size_t smem_bytes(int BT, int D, int FF, int nst, int bias_cap, int ocap, int V) {
  size_t red = sizeof(float) * (size_t)RED_FLOATS(BT);
  return (size_t)nst * UPC * D * 2 + (size_t)BT * FF * 2 + red + 16 * (size_t)nst + 16 +
         4 * (size_t)bias_cap + 4 * (size_t)BT * ocap + 4 * (size_t)((V + 31) / 32) + 16 +
         sizeof(float) * 4 * (size_t)D + 64;
}

static void reset_tagged_fwd(idx_engine* e, GptState* g, const GptParams& p);
template <int BT, int NPL>
static void launch_fused_t(idx_engine* e, GptState* g, GptParams& p) {
  p.nst = (BT == 1) ? g->nst1 : g->nst8;
  p.bias_cap = g->bias_cap;
  p.ocap = g->ocap;
  p.bar_flavor = g->bar_flavor;
  size_t smem = smem_bytes(BT, p.D, p.FF, p.nst, g->bias_cap, g->ocap, p.V);
  IDX_CUDA(cudaMemsetAsync(g->barrier, 0, (32 + 256) * sizeof(unsigned), e->stream));
  p.xt = nullptr;
  if (BT == 1 && p.mode == 1 && g->dataflow) {
    const unsigned need = (unsigned)p.nsteps * (unsigned)p.L * 2u + 2u;
    if (g->epoch > 0xF0000000u - need) reset_tagged_fwd(e, g, p);   // epochs never repeat while a stale word could still carry them
    p.xt = g->xt;
    p.ft = g->ft;
    p.qt = g->qt;
    p.pflag = g->pflag;
    p.kvt = g->kvt;
    p.epoch0 = g->epoch;
    g->epoch += need;
  }
  void* args[] = {(void*)&p};
  const void* fn = p.probe ? (const void*)gpt_fused_kernel<BT, NPL, true> : (const void*)gpt_fused_kernel<BT, NPL, false>;
  IDX_CUDA(cudaLaunchCooperativeKernel(fn, dim3(g->G), dim3(NTHREADS),
                                       args, smem, e->stream));
  e->launches++;
  g->last_launches++;
}

static void launch_fused_bt(idx_engine* e, GptState* g, GptParams& p, int BT) {
  // instantiated geometries: model_dim 1280 (IndexTTS GPT) and 256 (unit-test size)
  const int npl = p.D / 32;
  if (npl == 40) { if (BT == 1) launch_fused_t<1, 40>(e, g, p); else launch_fused_t<8, 40>(e, g, p); }
  else if (npl == 8) { if (BT == 1) launch_fused_t<1, 8>(e, g, p); else launch_fused_t<8, 8>(e, g, p); }
  else throw IdxError(IDX_ERR_ARG, "model_dim must be 1280 or 256 (instantiated kernel geometries)");
}
// second-generation batch-1 decode launch (same epoch bookkeeping as the tagged mode of gpt_fused_kernel<1, .>)
static size_t smem_bytes_v2(int D, int FF, int R, int bias_cap, int ocap, int V) {
  return (size_t)R * D * 2 + (size_t)FF * 2 + sizeof(float) * (size_t)RED1_FLOATS + 8 * (size_t)NBAR + 5 * sizeof(Phase1) + 32 +
         4 * (size_t)bias_cap + 4 * (size_t)ocap + 4 * (size_t)((V + 31) / 32) + 16 + sizeof(float) * 4 * (size_t)D + 64;
}
static void reset_tagged(idx_engine* e, GptState* g, const GptParams& p) {
  IDX_CUDA(cudaMemsetAsync(g->xt, 0, (size_t)p.D * sizeof(uint2), e->stream));
  IDX_CUDA(cudaMemsetAsync(g->ft, 0, (size_t)p.FF * sizeof(unsigned), e->stream));
  IDX_CUDA(cudaMemsetAsync(g->qt, 0, (size_t)p.D * sizeof(uint2), e->stream));
  IDX_CUDA(cudaMemsetAsync(g->pflag, 0, 32 * (size_t)(8 * p.H * std::max(1, p.G / p.H) + p.G) * sizeof(unsigned), e->stream));
  IDX_CUDA(cudaMemsetAsync(g->kvt, 0, 2 * (size_t)p.D * sizeof(uint2), e->stream));
  if (g->ot) {
    IDX_CUDA(cudaMemsetAsync(g->ot, 0, (size_t)p.D * sizeof(uint2), e->stream));
    IDX_CUDA(cudaMemsetAsync(g->partt, 0, (size_t)p.H * 7 * PART_STRIDE * sizeof(uint2), e->stream));
    IDX_CUDA(cudaMemsetAsync(g->cand, 0, 2 * (size_t)p.G * sizeof(uint2), e->stream));
    IDX_CUDA(cudaMemsetAsync(g->tokt, 0, sizeof(uint2), e->stream));
  }
  g->epoch = 0;
}
static void reset_tagged_fwd(idx_engine* e, GptState* g, const GptParams& p) { reset_tagged(e, g, p); }
static void launch_decode1(idx_engine* e, GptState* g, GptParams& p) {
  p.bias_cap = g->bias_cap;
  p.ocap = g->ocap;
  p.xt = g->xt; p.ft = g->ft; p.qt = g->qt; p.pflag = g->pflag; p.kvt = g->kvt;
  const unsigned need = (unsigned)p.nsteps * (unsigned)p.L * 2u + 2u;
  if (g->epoch > 0xF0000000u - need) reset_tagged(e, g, p);   // epochs never repeat while a stale word could still carry them
  p.epoch0 = g->epoch;
  g->epoch += need;
  void* args[] = {(void*)&p};
  const void* fn = (p.D / 32 == 40) ? (const void*)gpt_decode1_kernel<40> : (const void*)gpt_decode1_kernel<8>;
  IDX_CUDA(cudaLaunchCooperativeKernel(fn, dim3(g->G), dim3(NCT), args, g->smem_v2, e->stream));   // 8 warps: no producer warp
  e->launches++;
  g->last_launches++;
}

// 2..8 sequences per group on the tile / ring structure (gpt_decode8.cuh)
static size_t smem_bytes_v8(int D, int R, int bias_cap, int ocap, int V) {
  return (size_t)R * D * 2 + (size_t)B8 * D * 2 + sizeof(float) * (size_t)(RED8_FLOATS + NCW * PART_STRIDE) + 8 * (size_t)NBAR +
         5 * sizeof(Phase1) + 32 + 4 * (size_t)bias_cap + 4 * (size_t)B8 * ocap + 4 * (size_t)((V + 31) / 32) + 16 +
         sizeof(float) * 4 * (size_t)D + 64;
}
static void launch_decode8(idx_engine* e, GptState* g, GptParams& p) {
  p.bias_cap = g->bias_cap;
  p.ocap = g->ocap;
  p.ring_rows = g->ring_rows8;
  IDX_CUDA(cudaMemsetAsync(g->barrier, 0, (32 + 256) * sizeof(unsigned), e->stream));
  void* args[] = {(void*)&p};
  const void* fn = (p.D / 32 == 40) ? (const void*)gpt_decode8_kernel<40> : (const void*)gpt_decode8_kernel<8>;
  IDX_CUDA(cudaLaunchCooperativeKernel(fn, dim3(g->G), dim3(NCT), args, g->smem_v8, e->stream));
  e->launches++;
  g->last_launches++;
}

template <int BT>
static void set_smem_attr(int npl, size_t bytes) {
  if (npl == 40) {
    IDX_CUDA(cudaFuncSetAttribute(gpt_fused_kernel<BT, 40, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    IDX_CUDA(cudaFuncSetAttribute(gpt_fused_kernel<BT, 40, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  } else {
    IDX_CUDA(cudaFuncSetAttribute(gpt_fused_kernel<BT, 8, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    IDX_CUDA(cudaFuncSetAttribute(gpt_fused_kernel<BT, 8, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  }
}

extern "C" int idx_gpt_init(idx_engine* e, const idx_gpt_config* cfg) {
  IDX_API_BEGIN
  IDX_CHECK(e && cfg, IDX_ERR_ARG, "null argument");
  IDX_CUDA(cudaSetDevice(e->device));
  if (e->gpt) { gpt_destroy(e->gpt); e->gpt = nullptr; }
  // built into a local state and published only on success: a failed init must not leave a half-built e->gpt that passes the
  // "idx_gpt_init has not been called" guards (ADVICE r1)
  struct Guard {
    GptState* g; idx_engine* e; bool ok = false;
    ~Guard() { if (ok) e->gpt = g; else gpt_destroy(g); }
  } guard{new GptState(), e};
  GptState* g = guard.g;
  g->cfg = *cfg;
  const int L = cfg->layers, D = cfg->model_dim, H = cfg->heads, V = cfg->number_mel_codes;
  const int FF = 4 * D;
  g->FF = FF;
  IDX_CHECK(D == 1280 || D == 256, IDX_ERR_ARG, "model_dim must be 1280 or 256 (instantiated kernel geometries)");
  IDX_CHECK(D == H * HD, IDX_ERR_ARG, "head_dim must be 64");
  IDX_CHECK(cfg->max_batch >= 1 && cfg->max_batch <= 8, IDX_ERR_ARG, "max_batch must be 1..8 (per decode group)");
  const int G = e->num_sms;
  g->G = G;
  if (!cfg->weights_bf16) {
    strict_init(e, g);
    IDX_CUDA(cudaEventCreate(&g->ev0));
    IDX_CUDA(cudaEventCreate(&g->ev1));
    IDX_CUDA(cudaEventCreate(&g->ev2));
    IDX_CUDA(cudaStreamSynchronize(e->stream));
    guard.ok = true;
    return IDX_OK;
  }

  // ---- ring depth from the shared-memory budget ----
  int dev_smem = 0;
  IDX_CUDA(cudaDeviceGetAttribute(&dev_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, e->device));
  auto cdiv = [](int a, int b) { return (a + b - 1) / b; };
  g->ocap = cdiv(D, G) + 1;
  g->bias_cap = L * (cdiv(3 * D, G) + 1 + 2 * g->ocap + cdiv(FF, G) + 1) + cdiv(V, G) + 1;
  g->bar_flavor = getenv("IDX_GPT_BAR_FLAVOR") ? atoi(getenv("IDX_GPT_BAR_FLAVOR")) : 1;   // flavor 2 (per-CTA flags) measured slower: 839 vs 683 us/step
  auto pick_nst = [&](int BT) {
    int nst = 2;
    while (nst < 32 && smem_bytes(BT, D, FF, nst + 1, g->bias_cap, g->ocap, V) <= (size_t)dev_smem - 1024) ++nst;
    return nst;
  };
  g->nst1 = pick_nst(1);
  g->nst8 = pick_nst(8);
  g->smem1 = smem_bytes(1, D, FF, g->nst1, g->bias_cap, g->ocap, V);
  g->smem8 = smem_bytes(8, D, FF, g->nst8, g->bias_cap, g->ocap, V);
  IDX_CHECK(g->smem8 <= (size_t)dev_smem, IDX_ERR_ARG, "shared memory budget exceeded");
  set_smem_attr<1>(D / 32, g->smem1);
  set_smem_attr<8>(D / 32, g->smem8);

  // ---- build the per-CTA unit table in consumption order ----
  std::vector<PackUnit> units;
  std::vector<long long> off(G + 1, 0);
  auto lname = [&](int l, const char* s) { return "gpt.gpt.h." + std::to_string(l) + "." + s; };
  for (int l = 0; l < L; ++l) {
    const DevTensor& wq = e->W(lname(l, "attn.c_attn.weight"));
    IDX_CHECK(wq.shape.size() == 2 && wq.shape[0] == D && wq.shape[1] == 3 * D, IDX_ERR_ARG, "c_attn.weight shape");
    const DevTensor& wo = e->W(lname(l, "attn.c_proj.weight"));
    IDX_CHECK(wo.shape[0] == D && wo.shape[1] == D, IDX_ERR_ARG, "attn.c_proj.weight shape");
    const DevTensor& wf = e->W(lname(l, "mlp.c_fc.weight"));
    IDX_CHECK(wf.shape[0] == D && wf.shape[1] == FF, IDX_ERR_ARG, "c_fc.weight shape");
    const DevTensor& wp = e->W(lname(l, "mlp.c_proj.weight"));
    IDX_CHECK(wp.shape[0] == FF && wp.shape[1] == D, IDX_ERR_ARG, "mlp.c_proj.weight shape");
  }
  const DevTensor& wh = e->W("gpt.mel_head.weight");
  IDX_CHECK(wh.shape[0] == V && wh.shape[1] == D, IDX_ERR_ARG, "mel_head.weight shape");
  for (int i = 0; i < G; ++i) {
    off[i] = (long long)units.size();
    const int q0 = (int)(((long long)3 * D * i) / G), q1 = (int)(((long long)3 * D * (i + 1)) / G);
    const int o0 = (int)(((long long)D * i) / G), o1 = (int)(((long long)D * (i + 1)) / G);
    const int f0 = (int)(((long long)FF * i) / G), f1 = (int)(((long long)FF * (i + 1)) / G);
    const int h0 = (int)(((long long)V * i) / G), h1 = (int)(((long long)V * (i + 1)) / G);
    for (int l = 0; l < L; ++l) {
      const float* wq = (const float*)e->W(lname(l, "attn.c_attn.weight")).d;
      const float* wo = (const float*)e->W(lname(l, "attn.c_proj.weight")).d;
      const float* wf = (const float*)e->W(lname(l, "mlp.c_fc.weight")).d;
      const float* wp = (const float*)e->W(lname(l, "mlp.c_proj.weight")).d;
      // HF Conv1D keeps weight as [in, out] (P4): element (k, c) at k*N + c
      for (int c = q0; c < q1; ++c) units.push_back({wq, c, 3LL * D, (c - q0) & 7});
      for (int c = o0; c < o1; ++c) units.push_back({wo, c, (long long)D, (c - o0) & 7});
      for (int c = f0; c < f1; ++c) units.push_back({wf, c, (long long)FF, (c - f0) & 7});
      // PROJ: chunks are (8-column group, K-segment): group-major, then segment, then column
      for (int g0 = o0; g0 < o1; g0 += 8)
        for (int s = 0; s < FF / D; ++s)
          for (int c = g0; c < std::min(g0 + 8, o1); ++c)
            units.push_back({wp, (long long)s * D * D + c, (long long)D, (c - g0) & 7});
    }
    // nn.Linear keeps weight as [out, in]
    for (int c = h0; c < h1; ++c) units.push_back({(const float*)wh.d, (long long)c * D, 1LL, (c - h0) & 7});
  }
  off[G] = (long long)units.size();
  const long long nunits = (long long)units.size();
  PackUnit* d_units = nullptr;
  IDX_CUDA(cudaMalloc((void**)&d_units, nunits * sizeof(PackUnit)));
  IDX_CUDA(cudaMemcpyAsync(d_units, units.data(), nunits * sizeof(PackUnit), cudaMemcpyHostToDevice, e->stream));
  g->wstream = galloc<__nv_bfloat16>(g, (size_t)nunits * D + 64);
  pack_units_kernel<<<(unsigned)nunits, 128, 0, e->stream>>>(d_units, g->wstream, D, nunits);
  IDX_CUDA(cudaGetLastError());
  g->stream_off = galloc<long long>(g, G + 1);
  IDX_CUDA(cudaMemcpyAsync(g->stream_off, off.data(), (G + 1) * sizeof(long long), cudaMemcpyHostToDevice, e->stream));
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  cudaFree(d_units);

  // ---- second-generation batch-1 decode kernel (gpt_decode1.cuh): its own row stream in tile order ----
  {
    auto cdiv2 = [](int a, int b) { return (a + b - 1) / b; };
    const int mq = cdiv2(3 * D, G) + 1, mo = cdiv2(D, G) + 1, mf = cdiv2(FF, G) + 1, mh = cdiv2(V, G) + 1;
    // G >= H: the attention phase needs at least one CTA per head
    const bool fits = mo <= TROWS && cdiv2(mq, TROWS) <= MAXIT && cdiv2(mf, TROWS) <= MAXIT && cdiv2(mh, TROWS) <= MAXIT &&
                      FF / D <= MAXIT && G <= NCT && G >= H;
    g->v2 = fits && !(getenv("IDX_GPT_V2") && atoi(getenv("IDX_GPT_V2")) == 0);
    if (g->v2) {
      int R = 0;
      while (smem_bytes_v2(D, FF, R + 1, g->bias_cap, g->ocap, V) <= (size_t)dev_smem - 1024) ++R;
      if (getenv("IDX_GPT_RING")) R = std::min(R, atoi(getenv("IDX_GPT_RING")));
      IDX_CHECK(R >= std::max(std::max(mq, mf), std::max((FF / D) * mo, mh)), IDX_ERR_ARG, "shared memory too small for the decode ring");
      g->ring_rows = R;
      g->smem_v2 = smem_bytes_v2(D, FF, R, g->bias_cap, g->ocap, V);
      if (D / 32 == 40) IDX_CUDA(cudaFuncSetAttribute(gpt_decode1_kernel<40>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)g->smem_v2));
      else IDX_CUDA(cudaFuncSetAttribute(gpt_decode1_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)g->smem_v2));
      std::vector<PackUnit> u1;
      std::vector<long long> off1(G + 1, 0);
      auto tile_rows = [&](int c0, int n, int nt, auto&& emit) {     // column tiles of <= TROWS rows; the swizzle key is the row in the tile
        for (int j = 0; j < nt; ++j) {
          const int b0 = (n * j) / nt, b1 = (n * (j + 1)) / nt;
          for (int r = 0; r < b1 - b0; ++r) emit(c0 + b0 + r, r);
        }
      };
      for (int i = 0; i < G; ++i) {
        off1[i] = (long long)u1.size();
        const int q0 = (int)(((long long)3 * D * i) / G), q1 = (int)(((long long)3 * D * (i + 1)) / G);
        const int o0 = (int)(((long long)D * i) / G), o1 = (int)(((long long)D * (i + 1)) / G);
        const int f0 = (int)(((long long)FF * i) / G), f1 = (int)(((long long)FF * (i + 1)) / G);
        const int h0 = (int)(((long long)V * i) / G), h1 = (int)(((long long)V * (i + 1)) / G);
        for (int l = 0; l < L; ++l) {
          const float* wq = (const float*)e->W(lname(l, "attn.c_attn.weight")).d;
          const float* wo = (const float*)e->W(lname(l, "attn.c_proj.weight")).d;
          const float* wf = (const float*)e->W(lname(l, "mlp.c_fc.weight")).d;
          const float* wp = (const float*)e->W(lname(l, "mlp.c_proj.weight")).d;
          tile_rows(q0, q1 - q0, cdiv2(q1 - q0, TROWS), [&](int c, int r) { u1.push_back({wq, c, 3LL * D, r}); });
          tile_rows(o0, o1 - o0, 1, [&](int c, int r) { u1.push_back({wo, c, (long long)D, r}); });
          tile_rows(f0, f1 - f0, cdiv2(f1 - f0, TROWS), [&](int c, int r) { u1.push_back({wf, c, (long long)FF, r}); });
          for (int sg = 0; sg < FF / D; ++sg)        // PROJ: one tile per K-segment of D rows of c_proj.weight
            tile_rows(o0, o1 - o0, 1, [&](int c, int r) { u1.push_back({wp, (long long)sg * D * D + c, (long long)D, r}); });
        }
        tile_rows(h0, h1 - h0, cdiv2(h1 - h0, TROWS), [&](int c, int r) { u1.push_back({(const float*)wh.d, (long long)c * D, 1LL, r}); });
      }
      off1[G] = (long long)u1.size();
      const long long n1 = (long long)u1.size();
      PackUnit* d_u1 = nullptr;
      IDX_CUDA(cudaMalloc((void**)&d_u1, n1 * sizeof(PackUnit)));
      IDX_CUDA(cudaMemcpyAsync(d_u1, u1.data(), n1 * sizeof(PackUnit), cudaMemcpyHostToDevice, e->stream));
      g->wstream1 = galloc<__nv_bfloat16>(g, (size_t)n1 * D + 64);
      pack_units_kernel<<<(unsigned)n1, 128, 0, e->stream>>>(d_u1, g->wstream1, D, n1);
      IDX_CUDA(cudaGetLastError());
      g->stream_off1 = galloc<long long>(g, G + 1);
      IDX_CUDA(cudaMemcpyAsync(g->stream_off1, off1.data(), (G + 1) * sizeof(long long), cudaMemcpyHostToDevice, e->stream));
      IDX_CUDA(cudaStreamSynchronize(e->stream));
      cudaFree(d_u1);
      // the 8-row decode kernel shares the row stream; its ring is smaller (8 activation rows and 8-wide partial sums in shared memory)
      g->v8 = (H % 2 == 0) && 8 * (H / 2) <= G && !(getenv("IDX_GPT_V8") && atoi(getenv("IDX_GPT_V8")) == 0);
      if (g->v8) {
        int R8 = 0;
        while (smem_bytes_v8(D, R8 + 1, g->bias_cap, g->ocap, V) <= (size_t)dev_smem - 1024) ++R8;
        if (getenv("IDX_GPT_RING")) R8 = std::min(R8, atoi(getenv("IDX_GPT_RING")));
        if (R8 >= std::max(std::max(mq, mf), std::max((FF / D) * mo, mh))) {
          g->ring_rows8 = R8;
          g->smem_v8 = smem_bytes_v8(D, R8, g->bias_cap, g->ocap, V);
          if (D / 32 == 40) IDX_CUDA(cudaFuncSetAttribute(gpt_decode8_kernel<40>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)g->smem_v8));
          else IDX_CUDA(cudaFuncSetAttribute(gpt_decode8_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)g->smem_v8));
        } else {
          g->v8 = 0;
        }
      }
      g->ot = galloc<uint2>(g, (size_t)D);
      g->partt = galloc<uint2>(g, (size_t)H * 7 * PART_STRIDE);
      g->cand = galloc<uint2>(g, 2 * (size_t)G);
      g->tokt = galloc<uint2>(g, 1);
    }
  }

  // ---- small parameters gathered into [L][..] arrays ----
  auto gather = [&](const char* suffix, int n) {
    float* dst = galloc<float>(g, (size_t)L * n);
    for (int l = 0; l < L; ++l) {
      const DevTensor& t = e->W(lname(l, suffix));
      IDX_CHECK((int)t.numel() == n, IDX_ERR_ARG, std::string("bad size for ") + suffix);
      IDX_CUDA(cudaMemcpyAsync(dst + (size_t)l * n, t.d, (size_t)n * 4, cudaMemcpyDeviceToDevice, e->stream));
    }
    return dst;
  };
  g->ln1_w = gather("ln_1.weight", D);
  g->ln1_b = gather("ln_1.bias", D);
  g->ln2_w = gather("ln_2.weight", D);
  g->ln2_b = gather("ln_2.bias", D);
  g->qkv_b = gather("attn.c_attn.bias", 3 * D);
  g->o_b = gather("attn.c_proj.bias", D);
  g->fc_b = gather("mlp.c_fc.bias", FF);
  g->proj_b = gather("mlp.c_proj.bias", D);
  // weights .bfloat16(): biases/LN params/embeddings are bf16-valued too
  auto round_inplace = [&](float* p, size_t n) {
    round_bf16_kernel<<<(unsigned)((n + 255) / 256), 256, 0, e->stream>>>(p, n);
  };
  for (float* p : {g->ln1_w, g->ln1_b, g->ln2_w, g->ln2_b, g->o_b, g->proj_b}) round_inplace(p, (size_t)L * D);
  round_inplace(g->qkv_b, (size_t)L * 3 * D);
  round_inplace(g->fc_b, (size_t)L * FF);
  auto copy_round = [&](const std::string& name, size_t expect) {
    const DevTensor& t = e->W(name);
    IDX_CHECK(expect == 0 || t.numel() == expect, IDX_ERR_ARG, "bad size for " + name);
    float* dst = galloc<float>(g, t.numel());
    IDX_CUDA(cudaMemcpyAsync(dst, t.d, t.numel() * 4, cudaMemcpyDeviceToDevice, e->stream));
    round_inplace(dst, t.numel());
    return dst;
  };
  g->mel_emb = copy_round("gpt.mel_embedding.weight", (size_t)V * D);
  IDX_CHECK(e->W("gpt.mel_pos_embedding.emb.weight").shape[0] >= cfg->max_mel_positions, IDX_ERR_ARG, "mel_pos rows");
  g->mel_pos = copy_round("gpt.mel_pos_embedding.emb.weight", 0);

  // ---- KV cache + activations ----
  g->maxpos = cfg->max_prompt + cfg->max_mel_positions + 8;
  const size_t kvn = (size_t)L * cfg->max_batch * g->maxpos * D;
  g->kc = galloc<__nv_bfloat16>(g, kvn);
  g->vc = galloc<__nv_bfloat16>(g, kvn);
  g->xg = galloc<float>(g, 8 * (size_t)D);
  g->xt = galloc<uint2>(g, (size_t)D);
  g->ft = galloc<unsigned>(g, (size_t)FF);
  g->qt = galloc<uint2>(g, (size_t)D);
  g->pflag = galloc<unsigned>(g, 32 * (size_t)(8 * H * std::max(1, G / H) + G));
  g->kvt = galloc<uint2>(g, 2 * (size_t)D);
  g->dataflow = getenv("IDX_GPT_DATAFLOW") ? atoi(getenv("IDX_GPT_DATAFLOW")) : 1;
  g->qg = galloc<float>(g, 8 * (size_t)D);
  g->fg = galloc<__nv_bfloat16>(g, 8 * (size_t)FF);
  g->part = galloc<float>(g, (size_t)(8 * H * std::max(1, G / H) + G) * PART_STRIDE);
  g->logits = galloc<float>(g, 8 * (size_t)V);
  g->tok = galloc<int>(g, 8);
  g->nout = galloc<int>(g, 8);
  g->finished = galloc<int>(g, 8);
  g->prompt_len = galloc<int>(g, 8);
  g->done = galloc<int>(g, 1);
  g->seen = galloc<unsigned>(g, 8 * (size_t)((V + 31) / 32));
  g->barrier = galloc<unsigned>(g, 32 + 256);   // [0] counter (flavors 0/1), [32..] per-CTA arrival flags (flavor 2)
  g->prof = galloc<long long>(g, 320);
  g->prof2 = galloc<long long>(g, (size_t)G * 64);
  IDX_CUDA(cudaEventCreate(&g->ev0));
  IDX_CUDA(cudaEventCreate(&g->ev1));
  IDX_CUDA(cudaEventCreate(&g->ev2));
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  guard.ok = true;
  IDX_API_END(e)
}

static void fill_common(idx_engine* e, GptState* g, GptParams& p) {
  const idx_gpt_config& c = g->cfg;
  memset(&p, 0, sizeof(p));
  p.L = c.layers; p.D = c.model_dim; p.H = c.heads; p.V = c.number_mel_codes; p.FF = g->FF; p.G = g->G;
  p.start_tok = c.start_mel_token; p.stop_tok = c.stop_mel_token;
  p.round_bf16 = c.weights_bf16;
  p.wstream = g->wstream; p.stream_off = g->stream_off;
  p.ln1_w = g->ln1_w; p.ln1_b = g->ln1_b; p.ln2_w = g->ln2_w; p.ln2_b = g->ln2_b;
  p.qkv_b = g->qkv_b; p.o_b = g->o_b; p.fc_b = g->fc_b; p.proj_b = g->proj_b;
  p.lnf_w = e->Wf("gpt.gpt.ln_f.weight"); p.lnf_b = e->Wf("gpt.gpt.ln_f.bias");
  p.fn_w = e->Wf("gpt.final_norm.weight"); p.fn_b = e->Wf("gpt.final_norm.bias");
  p.head_b = e->Wf("gpt.mel_head.bias");
  p.mel_emb = g->mel_emb; p.mel_pos = g->mel_pos;
  p.kc = g->kc; p.vc = g->vc; p.nseq = c.max_batch; p.maxpos = g->maxpos;
  p.xg = g->xg; p.qg = g->qg; p.fg = g->fg; p.part = g->part; p.logits = g->logits;
  p.tok = g->tok; p.nout = g->nout; p.finished = g->finished; p.prompt_len = g->prompt_len;
  p.seen = g->seen; p.done = g->done; p.barrier = g->barrier; p.flag = e->dev_flag;
  p.wstream1 = g->wstream1; p.stream_off1 = g->stream_off1; p.ring_rows = g->ring_rows;
  p.dbg = getenv("IDX_GPT_DBG") ? atoi(getenv("IDX_GPT_DBG")) : 0;
  p.ot = g->ot; p.partt = g->partt; p.cand = g->cand; p.tokt = g->tokt;
  p.prof = g->prof_on ? g->prof : nullptr;
  p.prof2 = g->prof_on ? g->prof2 : nullptr;
  p.prof2_layer = c.layers / 2;
}

// Device buffers of the probes armed for one generate call (idx_gpt_probe_attention / idx_gpt_probe_prefill); the
// caller's buffers are written by probe_copy_out when the call has run.
struct ProbeBufs {
  float* q = nullptr;     // decode records
  int* ns = nullptr;      // decode split counts
  float* pf = nullptr;    // prefill records
  size_t nq = 0, nns = 0, npf = 0;
  ~ProbeBufs() { if (q) cudaFree(q); if (ns) cudaFree(ns); if (pf) cudaFree(pf); }
};

static void probe_arm_prefill(idx_engine* e, GptState* g, GptParams& p, ProbeBufs& pb) {
  const int nl = (g->pprobe_layer >= 0) ? 1 : g->cfg.layers;
  pb.npf = (size_t)g->pprobe_seqs * g->pprobe_rows * nl * 2 * g->cfg.model_dim;
  IDX_CUDA(cudaMalloc(&pb.pf, pb.npf * sizeof(float)));
  IDX_CUDA(cudaMemsetAsync(pb.pf, 0, pb.npf * sizeof(float), e->stream));
  p.probe = pb.pf;
  p.probe_layer = g->pprobe_layer;
  p.probe_seqs = g->pprobe_seqs;
  p.probe_rows = g->pprobe_rows;
}

static void probe_arm_decode(idx_engine* e, GptState* g, GptParams& p, ProbeBufs& pb, int max_new) {
  const int nl = (g->probe_layer >= 0) ? 1 : g->cfg.layers;
  pb.nq = (size_t)max_new * nl * g->probe_seqs * 2 * g->cfg.model_dim;
  pb.nns = (size_t)max_new * nl;
  IDX_CUDA(cudaMalloc(&pb.q, pb.nq * sizeof(float)));
  IDX_CUDA(cudaMalloc(&pb.ns, pb.nns * sizeof(int)));
  IDX_CUDA(cudaMemsetAsync(pb.q, 0, pb.nq * sizeof(float), e->stream));
  IDX_CUDA(cudaMemsetAsync(pb.ns, 0, pb.nns * sizeof(int), e->stream));
  p.probe = pb.q;
  p.probe_ns = pb.ns;
  p.probe_layer = g->probe_layer;
  p.probe_seqs = g->probe_seqs;
}

static void probe_copy_out(idx_engine* e, GptState* g, const ProbeBufs& pb) {
  if (pb.q) {
    idx_from_device(e, g->probe_out, pb.q, pb.nq * sizeof(float));
    idx_from_device(e, g->probe_ns_out, pb.ns, pb.nns * sizeof(int));
  }
  if (pb.pf) idx_from_device(e, g->pprobe_out, pb.pf, pb.npf * sizeof(float));
}

// ------------------------------------------------------------------ beam-sample host driver --
struct BeamTrace {
  int nutt = 0, m = 0, steps = 0, max_new = 0;
  std::vector<int> pt;        // [steps][8][2] (parent, token)
  std::vector<float> sc;      // [steps][8]
  double final_score[8] = {0};
};

static void beam_trace_free(GptState* g) { delete g->beam_trace; g->beam_trace = nullptr; }

static void beam_generate(idx_engine* e, GptState* g, const idx_gpt_request* reqs, int nreq, const idx_sampling* sp,
                          bool probe_on, bool pprobe_on) {
  const idx_gpt_config& c = g->cfg;
  const int D = c.model_dim, V = c.number_mel_codes, max_new = sp->max_new_tokens, m = sp->num_beams;
  IDX_CHECK(m >= 2 && m <= BEAM_MAX, IDX_ERR_ARG, "num_beams must be 1..4");
  IDX_CHECK(nreq * m <= 8 && nreq * m <= c.max_batch, IDX_ERR_ARG,
            "beam search needs num_beams rows per request: nreq * num_beams must be <= max_batch (<= 8)");
  IDX_CHECK(V <= 40 * 256, IDX_ERR_ARG, "vocabulary too large for the device sampler");
  cudaStream_t st = e->stream;
  const int rows = nreq * m, wv = (V + 31) / 32, hs = max_new + 2;
  bool want_logits = false;
  for (int i = 0; i < nreq; ++i) want_logits |= reqs[i].logits_out != nullptr;

  int total_rows = 0;
  std::vector<int> plen(8, 0), row0(8, 0), plen_rows(8, 0);
  for (int i = 0; i < nreq; ++i) {
    IDX_CHECK(reqs[i].prompt_emb && reqs[i].prompt_len >= 1 && reqs[i].prompt_len <= c.max_prompt, IDX_ERR_ARG, "bad prompt");
    IDX_CHECK(reqs[i].prompt_len + max_new + 1 <= g->maxpos, IDX_ERR_ARG, "KV cache too small");
    IDX_CHECK(!reqs[i].forced_codes, IDX_ERR_ARG, "forced_codes is not defined for beam search");
    plen[i] = reqs[i].prompt_len;
    row0[i] = total_rows;
    total_rows += plen[i];
    for (int j = 0; j < m; ++j) plen_rows[i * m + j] = plen[i];
  }
  std::vector<PrefillTile> tiles;
  for (int i = 0; i < nreq; ++i)
    for (int p0 = 0; p0 < plen[i]; p0 += 8)
      tiles.push_back({i * m, p0, std::min(8, plen[i] - p0), row0[i] + p0});     // prompt KV lives in the first beam's slot

  size_t need = (size_t)(total_rows + 8) * D * 4 + tiles.size() * sizeof(PrefillTile) + 2 * 8 * (size_t)wv * 4 +
                2 * 8 * (size_t)hs * 4 + 2 * 8 * (size_t)hs + (size_t)nreq * (m + 1) * hs * 4 + 8 * (size_t)max_new * 12 + (1 << 16);
  if (want_logits) need += (size_t)max_new * 8 * V * 4;
  e->ensure_arena(need + (1 << 20));
  e->arena.reset();
  float* d_prompt = e->arena.get<float>((size_t)(total_rows + 8) * D);
  PrefillTile* d_tiles = e->arena.get<PrefillTile>(tiles.size());
  unsigned* d_seen[2] = {e->arena.get<unsigned>(8 * (size_t)wv), e->arena.get<unsigned>(8 * (size_t)wv)};
  int* d_hist[2] = {e->arena.get<int>(8 * (size_t)hs), e->arena.get<int>(8 * (size_t)hs)};
  unsigned char* d_phys[2] = {e->arena.get<unsigned char>(8 * (size_t)hs + 16), e->arena.get<unsigned char>(8 * (size_t)hs + 16)};
  float* d_bscore = e->arena.get<float>(8);
  double* d_hscore = e->arena.get<double>((size_t)nreq * (m + 1) + 2);
  double* d_worst = e->arena.get<double>(nreq + 2);
  int* d_hlen = e->arena.get<int>((size_t)nreq * (m + 1));
  int* d_horder = e->arena.get<int>((size_t)nreq * (m + 1));
  int* d_nhyp = e->arena.get<int>(nreq);
  int* d_done = e->arena.get<int>(nreq);
  int* d_htok = e->arena.get<int>((size_t)nreq * (m + 1) * hs);
  int* d_trpt = e->arena.get<int>((size_t)max_new * 16);
  float* d_trsc = e->arena.get<float>((size_t)max_new * 8);
  float* d_ldump = want_logits ? e->arena.get<float>((size_t)max_new * 8 * V) : nullptr;

  IDX_CUDA(cudaEventRecord(g->ev0, st));
  for (int i = 0; i < nreq; ++i)
    idx_to_device(e, d_prompt + (size_t)row0[i] * D, reqs[i].prompt_emb, (size_t)plen[i] * D * 4);
  IDX_CUDA(cudaMemcpyAsync(d_tiles, tiles.data(), tiles.size() * sizeof(PrefillTile), cudaMemcpyHostToDevice, st));
  {
    std::vector<int> h_tok(8, c.start_mel_token), zeros(16, 0);
    std::vector<unsigned> h_seen(8 * (size_t)wv, 0u);
    std::vector<float> h_bs(8, -1e9f);
    std::vector<unsigned char> h_phys(8 * (size_t)hs + 16, 0);
    std::vector<double> h_worst(nreq + 2, 1e9);
    for (int r = 0; r < rows; ++r) {
      h_seen[(size_t)r * wv + (1 >> 5)] |= 1u << 1;                                      // trap P2
      h_seen[(size_t)r * wv + (c.start_mel_token >> 5)] |= 1u << (c.start_mel_token & 31);
      if (r % m == 0) h_bs[r] = 0.f;          // only the first beam carries probability mass at step 0 (:3408-3410)
      h_phys[(size_t)r * hs] = (unsigned char)r;
    }
    IDX_CUDA(cudaMemcpyAsync(g->tok, h_tok.data(), 32, cudaMemcpyHostToDevice, st));
    IDX_CUDA(cudaMemcpyAsync(g->finished, zeros.data(), 32, cudaMemcpyHostToDevice, st));
    IDX_CUDA(cudaMemcpyAsync(g->done, zeros.data(), 4, cudaMemcpyHostToDevice, st));
    IDX_CUDA(cudaMemcpyAsync(g->prompt_len, plen_rows.data(), 32, cudaMemcpyHostToDevice, st));
    IDX_CUDA(cudaMemcpyAsync(d_seen[0], h_seen.data(), h_seen.size() * 4, cudaMemcpyHostToDevice, st));
    IDX_CUDA(cudaMemcpyAsync(d_bscore, h_bs.data(), 32, cudaMemcpyHostToDevice, st));
    IDX_CUDA(cudaMemcpyAsync(d_phys[0], h_phys.data(), h_phys.size(), cudaMemcpyHostToDevice, st));
    IDX_CUDA(cudaMemcpyAsync(d_worst, h_worst.data(), h_worst.size() * 8, cudaMemcpyHostToDevice, st));
    IDX_CUDA(cudaMemsetAsync(d_nhyp, 0, nreq * 4, st));
    IDX_CUDA(cudaMemsetAsync(d_done, 0, nreq * 4, st));
    IDX_CUDA(cudaMemsetAsync(d_hlen, 0, (size_t)nreq * (m + 1) * 4, st));
    IDX_CUDA(cudaStreamSynchronize(st));
  }

  GptParams p;
  ProbeBufs pb;
  fill_common(e, g, p);
  p.B = 8; p.mode = 0; p.nsteps = (int)tiles.size(); p.prompt = d_prompt; p.tiles = d_tiles;
  p.max_new = max_new; p.rep_penalty = sp->repetition_penalty;
  p.beams = m;                                   // the prefill probe's request index is the tile's slot / m
  if (pprobe_on) probe_arm_prefill(e, g, p, pb);
  launch_fused_bt(e, g, p, 8);
  IDX_CUDA(cudaEventRecord(g->ev1, st));

  fill_common(e, g, p);
  p.B = rows; p.mode = 1; p.max_new = max_new; p.ext_sample = 1; p.beams = m; p.phys_stride = hs;
  p.pos_plain = sp->mel_pos_mode == 1;
  if (probe_on) probe_arm_decode(e, g, p, pb, max_new);
  BeamParams bp;
  memset(&bp, 0, sizeof(bp));
  bp.logits = g->logits; bp.V = V; bp.m = m; bp.max_new = max_new; bp.stop_tok = c.stop_mel_token;
  bp.forbid_stop_before = sp->forbid_stop_before; bp.hist_stride = hs;
  bp.rep_penalty = sp->repetition_penalty;
  bp.do_sample = sp->do_sample;
  bp.top_k = sp->do_sample ? sp->top_k : 0;
  bp.top_p = sp->do_sample ? sp->top_p : 1.0f;
  bp.inv_temp = (sp->do_sample && sp->temperature > 0.f) ? 1.0f / sp->temperature : 1.0f;
  bp.length_penalty = sp->length_penalty; bp.seed = sp->seed; bp.utt_base = g->seq_base;
  bp.beam_scores = d_bscore; bp.tok = g->tok;
  bp.hyp_score = d_hscore; bp.hyp_len = d_hlen; bp.hyp_tok = d_htok; bp.hyp_order = d_horder; bp.nhyp = d_nhyp;
  bp.worst = d_worst; bp.done_u = d_done; bp.ldump = d_ldump; bp.trace_pt = d_trpt; bp.trace_sc = d_trsc;
  bp.flag = e->dev_flag;
  int* h_done = (int*)e->pinned_buf(64);
  int steps = 0;
  for (int k = 0; k < max_new; ++k) {
    const int cur = k & 1, nxt = cur ^ 1;
    p.step0 = k; p.nsteps = 1; p.phys = d_phys[cur];
    launch_fused_bt(e, g, p, 8);
    bp.k = k;
    bp.seen_cur = d_seen[cur]; bp.seen_nxt = d_seen[nxt];
    bp.hist_cur = d_hist[cur]; bp.hist_nxt = d_hist[nxt];
    bp.phys_cur = d_phys[cur]; bp.phys_nxt = d_phys[nxt];
    beam_step_kernel<<<nreq, 256, 0, st>>>(bp);
    IDX_CUDA(cudaGetLastError());
    e->launches++;
    g->last_launches++;
    steps = k + 1;
    if ((k & 7) == 7 || k + 1 == max_new) {
      IDX_CUDA(cudaMemcpyAsync(h_done, d_done, nreq * 4, cudaMemcpyDeviceToHost, st));
      IDX_CUDA(cudaStreamSynchronize(st));
      bool all = true;
      for (int i = 0; i < nreq; ++i) all &= h_done[i] != 0;
      if (all) break;
    }
  }
  IDX_CUDA(cudaEventRecord(g->ev2, st));
  e->check_flag(kTieOverflow);

  // ---- BeamSearchScorer.finalize (transformers_beam_search.py:322-420) on the host ----
  const int fin = steps & 1;      // buffers written by the last beam step
  std::vector<int> h_hist(8 * (size_t)hs), h_hlen((size_t)nreq * (m + 1)), h_horder((size_t)nreq * (m + 1)), h_nhyp(nreq), h_dn(nreq);
  std::vector<int> h_htok((size_t)nreq * (m + 1) * hs);
  std::vector<double> h_hscore((size_t)nreq * (m + 1) + 2);
  std::vector<float> h_bs(8);
  BeamTrace* tr = g->beam_trace ? g->beam_trace : (g->beam_trace = new BeamTrace());
  tr->nutt = nreq; tr->m = m; tr->steps = steps; tr->max_new = max_new;
  tr->pt.assign((size_t)steps * 16, 0); tr->sc.assign((size_t)steps * 8, 0.f);
  IDX_CUDA(cudaMemcpyAsync(h_hist.data(), d_hist[fin], h_hist.size() * 4, cudaMemcpyDeviceToHost, st));
  IDX_CUDA(cudaMemcpyAsync(h_hlen.data(), d_hlen, h_hlen.size() * 4, cudaMemcpyDeviceToHost, st));
  IDX_CUDA(cudaMemcpyAsync(h_horder.data(), d_horder, h_horder.size() * 4, cudaMemcpyDeviceToHost, st));
  IDX_CUDA(cudaMemcpyAsync(h_nhyp.data(), d_nhyp, nreq * 4, cudaMemcpyDeviceToHost, st));
  IDX_CUDA(cudaMemcpyAsync(h_dn.data(), d_done, nreq * 4, cudaMemcpyDeviceToHost, st));
  IDX_CUDA(cudaMemcpyAsync(h_htok.data(), d_htok, h_htok.size() * 4, cudaMemcpyDeviceToHost, st));
  IDX_CUDA(cudaMemcpyAsync(h_hscore.data(), d_hscore, (size_t)nreq * (m + 1) * 8, cudaMemcpyDeviceToHost, st));
  IDX_CUDA(cudaMemcpyAsync(h_bs.data(), d_bscore, 32, cudaMemcpyDeviceToHost, st));
  IDX_CUDA(cudaMemcpyAsync(tr->pt.data(), d_trpt, tr->pt.size() * 4, cudaMemcpyDeviceToHost, st));
  IDX_CUDA(cudaMemcpyAsync(tr->sc.data(), d_trsc, tr->sc.size() * 4, cudaMemcpyDeviceToHost, st));
  probe_copy_out(e, g, pb);
  IDX_CUDA(cudaStreamSynchronize(st));
  int maxn = 0;
  for (int u = 0; u < nreq; ++u) {
    struct Hyp { double score; const int* tok; int len; };
    std::vector<Hyp> list;
    for (int q = 0; q < h_nhyp[u]; ++q) {
      const int slot = h_horder[(size_t)u * (m + 1) + q];
      list.push_back({h_hscore[(size_t)u * (m + 1) + slot], &h_htok[((size_t)u * (m + 1) + slot) * hs], h_hlen[(size_t)u * (m + 1) + slot]});
    }
    double worst = 1e9;
    for (auto& h : list) worst = std::min(worst, h.score);
    if (!h_dn[u]) {
      for (int j = 0; j < m; ++j) {           // add the live beams (:345-356); generated_len = steps
        const double score = (double)h_bs[u * m + j] / std::pow((double)steps, (double)sp->length_penalty);
        if ((int)list.size() < m || score > worst) {
          list.push_back({score, &h_hist[(size_t)(u * m + j) * hs], steps});
          if ((int)list.size() > m) {
            size_t lo = 0;
            for (size_t q = 1; q < list.size(); ++q) if (list[q].score < list[lo].score) lo = q;
            list.erase(list.begin() + lo);
            worst = 1e9;
            for (auto& h : list) worst = std::min(worst, h.score);
          } else {
            worst = std::min(worst, score);
          }
        }
      }
    }
    // sorted(candidate_beams, key=score).pop(): the LAST of the maximal scores in list order
    size_t best = 0;
    for (size_t q = 1; q < list.size(); ++q) if (list[q].score >= list[best].score) best = q;
    std::vector<int> codes(list[best].tok, list[best].tok + list[best].len);
    if ((int)codes.size() < max_new) codes.push_back(c.stop_mel_token);
    tr->final_score[u] = list[best].score;
    maxn = std::max(maxn, (int)codes.size());
    if (reqs[u].n_codes_out) *reqs[u].n_codes_out = (int)codes.size();
    if (reqs[u].codes_out) {
      IDX_CUDA(cudaMemcpyAsync(d_trpt, codes.data(), codes.size() * 4, cudaMemcpyHostToDevice, st));
      IDX_CUDA(cudaStreamSynchronize(st));
      idx_from_device(e, reqs[u].codes_out, d_trpt, codes.size() * 4);
      IDX_CUDA(cudaStreamSynchronize(st));
    }
    if (reqs[u].logits_out) {
      // [steps][m][V]: the raw logits every beam of this utterance saw at each step
      for (int k = 0; k < steps; ++k)
        idx_from_device(e, reqs[u].logits_out + ((size_t)k * m) * V, d_ldump + ((size_t)k * 8 + u * m) * V, (size_t)m * V * 4);
    }
  }
  IDX_CUDA(cudaStreamSynchronize(st));
  float ms01 = 0, ms12 = 0;
  IDX_CUDA(cudaEventElapsedTime(&ms01, g->ev0, g->ev1));
  IDX_CUDA(cudaEventElapsedTime(&ms12, g->ev1, g->ev2));
  g->t_prefill_ms = ms01;
  g->t_decode_ms = ms12;
  g->last_steps = steps;
}

extern "C" int idx_gpt_generate(idx_engine* e, const idx_gpt_request* reqs, int nreq,
                                const idx_sampling* sp) {
  IDX_API_BEGIN
  IDX_CHECK(e && e->gpt, IDX_ERR_STATE, "idx_gpt_init has not been called");
  IDX_CHECK(reqs && sp && nreq >= 1, IDX_ERR_ARG, "bad request");
  GptState* g = e->gpt;
  const idx_gpt_config& c = g->cfg;
  IDX_CHECK(sp->num_beams >= 1, IDX_ERR_ARG, "num_beams must be >= 1");
  // HF semantics are kept exactly or refused: top_k = 0 (warper disabled) or top_k > CMAX would need more candidate slots
  // than the device samplers hold, and capping them silently would change the support of the top-p / multinomial step
  IDX_CHECK(!sp->do_sample || (sp->top_k >= 1 && sp->top_k <= CMAX), IDX_ERR_ARG,
            "do_sample needs 1 <= top_k <= 128 (the reference default is 30; top_k = 0 / larger values are not built)");
  // the values HF's processors refuse are refused here too (greedy ignores temperature and top_p, as HF does)
  IDX_CHECK(std::isfinite(sp->repetition_penalty) && sp->repetition_penalty > 0.f, IDX_ERR_ARG,
            "repetition_penalty must be a finite number > 0");
  IDX_CHECK(!sp->do_sample || (std::isfinite(sp->temperature) && sp->temperature > 0.f), IDX_ERR_ARG,
            "do_sample needs a finite temperature > 0");
  IDX_CHECK(!sp->do_sample || (sp->top_p >= 0.f && sp->top_p <= 1.f), IDX_ERR_ARG, "do_sample needs 0 <= top_p <= 1");
  // an armed attention probe is consumed by this call, whatever its outcome
  const int probe_on = g->probe_armed, pprobe_on = g->pprobe_armed;
  g->probe_armed = g->pprobe_armed = 0;
  const int rows = nreq * sp->num_beams;      // decode rows of one group
  if (probe_on) {
    const bool dec1 = nreq == 1 && g->v2, dec8 = nreq > 1 && g->v8;
    IDX_CHECK(!g->strict && (sp->num_beams > 1 || dec1 || dec8) && rows <= c.max_batch, IDX_ERR_ARG,
              "the attention probe records one decode group of gpt_decode1 / gpt_decode8 (num_beams = 1) or of gpt_fused_kernel "
              "(num_beams > 1), bf16 path");
    IDX_CHECK(rows <= g->probe_seqs && sp->max_new_tokens <= g->probe_steps, IDX_ERR_ARG, "attention probe buffer too small");
  }
  if (pprobe_on) {
    IDX_CHECK(!g->strict && rows <= c.max_batch, IDX_ERR_ARG, "the prefill probe records the prefill of one decode group (bf16 path)");
    IDX_CHECK(nreq <= g->pprobe_seqs, IDX_ERR_ARG, "prefill probe buffer too small");
    for (int i = 0; i < nreq; ++i)
      IDX_CHECK(reqs[i].prompt_len <= g->pprobe_rows, IDX_ERR_ARG, "prefill probe buffer too small");
  }
  {
    // more requests than one decode group holds (max_batch rows, num_beams rows per request): run consecutive groups;
    // the sampler's sequence index stays the request's global index, so the result does not depend on the grouping
    const int cap = g->strict ? nreq : std::max(0, c.max_batch / sp->num_beams);
    IDX_CHECK(cap >= 1, IDX_ERR_ARG, "max_batch is smaller than num_beams (every request needs num_beams rows)");
    if (nreq > cap) {
      double tp = 0, td = 0;
      int steps = 0, launches = 0, rc = IDX_OK;
      const int base0 = g->seq_base;
      for (int i0 = 0; i0 < nreq && rc == IDX_OK; i0 += cap) {
        g->seq_base = base0 + i0;
        rc = idx_gpt_generate(e, reqs + i0, std::min(cap, nreq - i0), sp);
        tp += g->t_prefill_ms; td += g->t_decode_ms;
        steps = std::max(steps, g->last_steps); launches += g->last_launches;
      }
      g->seq_base = base0;
      g->t_prefill_ms = tp; g->t_decode_ms = td; g->last_steps = steps; g->last_launches = launches;
      return rc;
    }
  }
  IDX_CHECK(c.number_mel_codes <= 40 * 256, IDX_ERR_ARG, "vocabulary too large for the device sampler");
  IDX_CHECK(sp->max_new_tokens >= 1 && sp->max_new_tokens + 2 <= c.max_mel_positions, IDX_ERR_ARG,
            "max_new_tokens must satisfy k+1 <= mel_pos rows - 1 (SURVEY A.3)");
  IDX_CUDA(cudaSetDevice(e->device));
  const int D = c.model_dim, V = c.number_mel_codes, max_new = sp->max_new_tokens;
  const int BT = (nreq == 1) ? 1 : 8;
  g->last_launches = 0;
  if (g->strict) {
    IDX_CHECK(sp->num_beams == 1, IDX_ERR_ARG, "the strict fp32 path decodes one sequence at a time (num_beams = 1)");
    strict_generate(e, g, reqs, nreq, sp);
    return IDX_OK;
  }
  if (sp->num_beams > 1) {
    beam_generate(e, g, reqs, nreq, sp, probe_on, pprobe_on);
    return IDX_OK;
  }

  // ---- stage prompts ----
  int total_rows = 0;
  std::vector<int> plen(8, 0), row0(8, 0);
  for (int i = 0; i < nreq; ++i) {
    IDX_CHECK(reqs[i].prompt_emb && reqs[i].prompt_len >= 1 && reqs[i].prompt_len <= c.max_prompt, IDX_ERR_ARG, "bad prompt");
    IDX_CHECK(reqs[i].prompt_len + max_new + 1 <= g->maxpos, IDX_ERR_ARG, "KV cache too small");
    plen[i] = reqs[i].prompt_len;
    row0[i] = total_rows;
    total_rows += plen[i];
  }
  std::vector<PrefillTile> tiles;
  for (int i = 0; i < nreq; ++i)
    for (int p0 = 0; p0 < plen[i]; p0 += 8)
      tiles.push_back({i, p0, std::min(8, plen[i] - p0), row0[i] + p0});
  const size_t wv = (size_t)((V + 31) / 32);
  size_t need = (size_t)(total_rows + 8) * D * 4 + tiles.size() * sizeof(PrefillTile) + 8 * (size_t)max_new * 8 + 4096;
  bool want_logits = false, want_forced = false;
  for (int i = 0; i < nreq; ++i) { want_logits |= reqs[i].logits_out != nullptr; want_forced |= reqs[i].forced_codes != nullptr; }
  if (want_logits) need += 8 * (size_t)max_new * V * 4;
  e->ensure_arena(need + (1 << 20));
  e->arena.reset();
  float* d_prompt = e->arena.get<float>((size_t)(total_rows + 8) * D);
  PrefillTile* d_tiles = e->arena.get<PrefillTile>(tiles.size());
  int* d_codes = e->arena.get<int>(8 * (size_t)max_new);
  int* d_forced = want_forced ? e->arena.get<int>(8 * (size_t)max_new) : nullptr;
  float* d_ldump = want_logits ? e->arena.get<float>(8 * (size_t)max_new * V) : nullptr;

  IDX_CUDA(cudaEventRecord(g->ev0, e->stream));
  for (int i = 0; i < nreq; ++i)
    idx_to_device(e, d_prompt + (size_t)row0[i] * D, reqs[i].prompt_emb, (size_t)plen[i] * D * 4);
  IDX_CUDA(cudaMemcpyAsync(d_tiles, tiles.data(), tiles.size() * sizeof(PrefillTile), cudaMemcpyHostToDevice, e->stream));
  if (want_forced) {
    IDX_CUDA(cudaMemsetAsync(d_forced, 0, 8 * (size_t)max_new * 4, e->stream));
    for (int i = 0; i < nreq; ++i) {
      IDX_CHECK(reqs[i].forced_codes, IDX_ERR_ARG, "forced_codes must be given for all requests or none");
      idx_to_device(e, d_forced + (size_t)i * max_new, reqs[i].forced_codes, (size_t)max_new * 4);
    }
  }
  // per-sequence state
  {
    std::vector<int> h_tok(8, c.start_mel_token), zeros(8, 0);
    std::vector<unsigned> h_seen(8 * wv, 0u);
    for (int i = 0; i < nreq; ++i) {
      // P2: the fake prompt ids [1,...,1, start_mel] are part of input_ids
      h_seen[i * wv + (1 >> 5)] |= 1u << 1;
      h_seen[i * wv + (c.start_mel_token >> 5)] |= 1u << (c.start_mel_token & 31);
    }
    IDX_CUDA(cudaMemcpyAsync(g->tok, h_tok.data(), 32, cudaMemcpyHostToDevice, e->stream));
    IDX_CUDA(cudaMemcpyAsync(g->nout, zeros.data(), 32, cudaMemcpyHostToDevice, e->stream));
    IDX_CUDA(cudaMemcpyAsync(g->finished, zeros.data(), 32, cudaMemcpyHostToDevice, e->stream));
    IDX_CUDA(cudaMemcpyAsync(g->done, zeros.data(), 4, cudaMemcpyHostToDevice, e->stream));
    IDX_CUDA(cudaMemcpyAsync(g->prompt_len, plen.data(), 32, cudaMemcpyHostToDevice, e->stream));
    IDX_CUDA(cudaMemcpyAsync(g->seen, h_seen.data(), h_seen.size() * 4, cudaMemcpyHostToDevice, e->stream));
    IDX_CUDA(cudaStreamSynchronize(e->stream));  // host vectors go out of scope
  }

  // ---- prefill: tiles of 8 prompt positions through the same fused kernel ----
  GptParams p;
  fill_common(e, g, p);
  p.B = 8; p.mode = 0; p.nsteps = (int)tiles.size(); p.prompt = d_prompt; p.tiles = d_tiles;
  p.max_new = max_new; p.rep_penalty = sp->repetition_penalty;
  ProbeBufs pb;
  if (pprobe_on) probe_arm_prefill(e, g, p, pb);
  launch_fused_bt(e, g, p, 8);
  IDX_CUDA(cudaEventRecord(g->ev1, e->stream));

  // ---- decode ----
  fill_common(e, g, p);
  p.B = nreq; p.mode = 1; p.max_new = max_new; p.rep_penalty = sp->repetition_penalty;
  p.forbid_stop_before = sp->forbid_stop_before;
  p.do_sample = sp->do_sample; p.top_k = sp->top_k; p.top_p = sp->top_p; p.temperature = sp->temperature;
  p.seed = sp->seed;
  p.seq_base = g->seq_base;
  p.pos_plain = sp->mel_pos_mode == 1;
  p.codes = d_codes; p.forced = d_forced; p.logits_dump = d_ldump;
  if (probe_on) probe_arm_decode(e, g, p, pb, max_new);
  const int SPL = (BT == 1 && g->v2) ? 64 : 32;  // steps per launch: the host looks at one flag every SPL steps
  int steps_done = 0;
  int* h_done = (int*)e->pinned_buf(64);
  while (steps_done < max_new) {
    p.step0 = steps_done;
    p.nsteps = std::min(SPL, max_new - steps_done);
    if (BT == 1 && g->v2) launch_decode1(e, g, p);
    else if (BT == 8 && g->v8) launch_decode8(e, g, p);
    else launch_fused_bt(e, g, p, BT);
    IDX_CUDA(cudaMemcpyAsync(h_done, g->done, 4, cudaMemcpyDeviceToHost, e->stream));
    IDX_CUDA(cudaStreamSynchronize(e->stream));
    steps_done += p.nsteps;
    if (*h_done) break;
  }
  IDX_CUDA(cudaEventRecord(g->ev2, e->stream));
  e->check_flag(kTieOverflow);

  // ---- results ----
  int h_nout[8];
  IDX_CUDA(cudaMemcpyAsync(h_nout, g->nout, 32, cudaMemcpyDeviceToHost, e->stream));
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  int maxn = 0;
  for (int i = 0; i < nreq; ++i) {
    maxn = std::max(maxn, h_nout[i]);
    if (reqs[i].n_codes_out) *reqs[i].n_codes_out = h_nout[i];
    if (reqs[i].codes_out) idx_from_device(e, reqs[i].codes_out, d_codes + (size_t)i * max_new, (size_t)h_nout[i] * 4);
    if (reqs[i].logits_out)
      idx_from_device(e, reqs[i].logits_out, d_ldump + (size_t)i * max_new * V, (size_t)h_nout[i] * V * 4);
  }
  probe_copy_out(e, g, pb);
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  float ms01 = 0, ms12 = 0;
  IDX_CUDA(cudaEventElapsedTime(&ms01, g->ev0, g->ev1));
  IDX_CUDA(cudaEventElapsedTime(&ms12, g->ev1, g->ev2));
  g->t_prefill_ms = ms01;
  g->t_decode_ms = ms12;
  g->last_steps = maxn;
  IDX_API_END(e)
}

extern "C" int idx_gpt_last_timing(const idx_engine* e, double* out4) {
  if (!e || !e->gpt || !out4) return IDX_ERR_STATE;
  out4[0] = e->gpt->t_prefill_ms;
  out4[1] = e->gpt->t_decode_ms;
  out4[2] = e->gpt->last_steps;
  out4[3] = e->gpt->last_launches;
  return IDX_OK;
}

extern "C" int idx_gpt_prepare_inputs(idx_engine* e, const float* style, const float* emo_vec,
                                      const int32_t* text_ids, int n_text, int lang, float* out) {
  IDX_API_BEGIN
  IDX_CHECK(e && e->gpt, IDX_ERR_STATE, "idx_gpt_init has not been called");
  IDX_CUDA(cudaSetDevice(e->device));
  GptState* g = e->gpt;
  const int D = g->cfg.model_dim;
  const int rows = 3 + n_text + 2;
  const DevTensor& tpos = e->W("gpt.text_pos_embedding.emb.weight");
  IDX_CHECK(n_text + 2 <= tpos.shape[0], IDX_ERR_ARG, "text longer than text_pos_embedding");
  e->ensure_arena((size_t)rows * D * 4 + 4 * (size_t)n_text + 192 * 4 + D * 4 + (1 << 16));
  e->arena.reset();
  float* d_style = e->arena.get<float>(192);
  float* d_emo = e->arena.get<float>(D);
  int* d_ids = e->arena.get<int>(n_text + 1);
  float* d_out = e->arena.get<float>((size_t)rows * D);
  idx_to_device(e, d_style, style, 192 * 4);
  idx_to_device(e, d_emo, emo_vec, (size_t)D * 4);
  idx_to_device(e, d_ids, text_ids, (size_t)n_text * 4);
  const float* lang_emb = e->has("gpt.lang_embedding.weight") ? e->Wf("gpt.lang_embedding.weight") : nullptr;
  prepare_inputs_kernel<<<rows, 256, 0, e->stream>>>(
      d_style, d_emo, d_ids, n_text, lang, e->Wf("gpt.spk_emb_proj.weight"), e->Wf("gpt.spk_emb_proj.bias"),
      e->Wf("gpt.text_embedding.weight"), (const float*)tpos.d, lang_emb, D, g->cfg.weights_bf16, d_out,
      (int)e->W("gpt.text_embedding.weight").shape[0], e->dev_flag);
  IDX_CUDA(cudaGetLastError());
  e->launches++;
  idx_from_device(e, out, d_out, (size_t)rows * D * 4);
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  e->check_flag("text token id outside text_embedding");
  IDX_API_END(e)
}

extern "C" int idx_gpt_profile(idx_engine* e, int enable, int64_t* stamps_out, int n) {
  IDX_API_BEGIN
  IDX_CHECK(e && e->gpt, IDX_ERR_STATE, "idx_gpt_init has not been called");
  IDX_CUDA(cudaSetDevice(e->device));
  GptState* g = e->gpt;
  g->prof_on = enable;
  if (stamps_out && n > 0 && g->prof) {
    IDX_CUDA(cudaStreamSynchronize(e->stream));
    IDX_CUDA(cudaMemcpy(stamps_out, g->prof, sizeof(long long) * (size_t)std::min(n, 320), cudaMemcpyDeviceToHost));
  }
  IDX_API_END(e)
}

// diagnostics: [G][64] fine globaltimer stamps of every CTA for the middle layer of the last decode step (see F2 in the kernel)
extern "C" int idx_gpt_profile_fine(idx_engine* e, int64_t* stamps_out, int n) {
  IDX_API_BEGIN
  IDX_CHECK(e && e->gpt && e->gpt->prof2, IDX_ERR_STATE, "idx_gpt_init (bf16 path) has not been called");
  IDX_CUDA(cudaSetDevice(e->device));
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  IDX_CUDA(cudaMemcpy(stamps_out, e->gpt->prof2, sizeof(long long) * (size_t)std::min(n, e->gpt->G * 64), cudaMemcpyDeviceToHost));
  IDX_API_END(e)
}

extern "C" int idx_gpt_probe_attention(idx_engine* e, int layer, int max_steps, int max_seqs, float* qo_out, int32_t* nsplit_out) {
  IDX_API_BEGIN
  IDX_CHECK(e && e->gpt && !e->gpt->strict, IDX_ERR_STATE, "idx_gpt_init (bf16 path) has not been called");
  GptState* g = e->gpt;
  IDX_CHECK(layer >= -1 && layer < g->cfg.layers, IDX_ERR_ARG, "layer must be -1 (all) or a layer index");
  IDX_CHECK(max_steps >= 1 && max_seqs >= 1 && max_seqs <= 8 && qo_out && nsplit_out, IDX_ERR_ARG, "bad probe buffers");
  g->probe_layer = layer;
  g->probe_steps = max_steps;
  g->probe_seqs = max_seqs;
  g->probe_out = qo_out;
  g->probe_ns_out = nsplit_out;
  g->probe_armed = 1;
  IDX_API_END(e)
}

extern "C" int idx_gpt_probe_prefill(idx_engine* e, int layer, int max_rows, int max_seqs, float* qo_out) {
  IDX_API_BEGIN
  IDX_CHECK(e && e->gpt && !e->gpt->strict, IDX_ERR_STATE, "idx_gpt_init (bf16 path) has not been called");
  GptState* g = e->gpt;
  IDX_CHECK(layer >= -1 && layer < g->cfg.layers, IDX_ERR_ARG, "layer must be -1 (all) or a layer index");
  IDX_CHECK(max_rows >= 1 && max_seqs >= 1 && max_seqs <= 8 && qo_out, IDX_ERR_ARG, "bad probe buffers");
  g->pprobe_layer = layer;
  g->pprobe_rows = max_rows;
  g->pprobe_seqs = max_seqs;
  g->pprobe_out = qo_out;
  g->pprobe_armed = 1;
  IDX_API_END(e)
}

extern "C" int idx_gpt_debug_kv(idx_engine* e, int layer, int seq, int pos0, int n, float* k_out, float* v_out) {
  IDX_API_BEGIN
  IDX_CHECK(e && e->gpt && !e->gpt->strict, IDX_ERR_STATE, "idx_gpt_init (bf16 path) has not been called");
  GptState* g = e->gpt;
  const idx_gpt_config& c = g->cfg;
  IDX_CHECK(layer >= 0 && layer < c.layers && seq >= 0 && seq < c.max_batch && pos0 >= 0 && n >= 1 && pos0 + n <= g->maxpos &&
                k_out && v_out, IDX_ERR_ARG, "bad KV-cache range");
  IDX_CUDA(cudaSetDevice(e->device));
  const size_t D = (size_t)c.model_dim, off = (((size_t)layer * c.max_batch + seq) * g->maxpos + pos0) * D, cnt = (size_t)n * D;
  std::vector<uint16_t> raw(cnt);
  std::vector<float> f(cnt);
  for (int which = 0; which < 2; ++which) {
    IDX_CUDA(cudaStreamSynchronize(e->stream));
    IDX_CUDA(cudaMemcpy(raw.data(), (which ? g->vc : g->kc) + off, cnt * 2, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < cnt; ++i) {         // bf16 -> fp32 is exact: the bf16 bits are the high half of the fp32 word
      const uint32_t u = (uint32_t)raw[i] << 16;
      memcpy(&f[i], &u, 4);
    }
    IDX_CUDA(cudaMemcpy(which ? v_out : k_out, f.data(), cnt * 4, cudaMemcpyDefault));
  }
  IDX_API_END(e)
}

extern "C" int idx_gpt_beam_trace(const idx_engine* e, int utterance, int32_t* parents_tokens, float* scores,
                                  int max_steps, int32_t* steps_out, double* final_score) {
  if (!e || !e->gpt || !e->gpt->beam_trace) return IDX_ERR_STATE;
  const BeamTrace* t = e->gpt->beam_trace;
  if (utterance < 0 || utterance >= t->nutt) return IDX_ERR_ARG;
  const int n = std::min(max_steps, t->steps), m = t->m;
  for (int k = 0; k < n; ++k)
    for (int j = 0; j < m; ++j) {
      const int r = utterance * m + j;
      if (parents_tokens) {
        parents_tokens[((size_t)k * m + j) * 2] = t->pt[((size_t)k * 8 + r) * 2];
        parents_tokens[((size_t)k * m + j) * 2 + 1] = t->pt[((size_t)k * 8 + r) * 2 + 1];
      }
      if (scores) scores[(size_t)k * m + j] = t->sc[(size_t)k * 8 + r];
    }
  if (steps_out) *steps_out = t->steps;
  if (final_score) *final_score = t->final_score[utterance];
  return IDX_OK;
}

// ------------------------------------------------------------------ v1 / v1.5 GPT side (row a13) --
namespace {
// rows r < n_lat: conds[r]; then j = r - n_lat over [start_text, text.., stop_text]: text_emb[id] + text_pos[j];
// with n_codes >= 0 also the mel part [start_mel, codes.., stop_mel]: mel_emb[tok] + mel_pos[i]  (model.py:565-578)
__global__ void v1_rows_kernel(const float* conds, int n_lat, const int* text_ids, int n_text, const int* codes, int n_codes,
                               const float* text_emb, const float* text_pos, const float* mel_emb, const float* mel_pos,
                               int start_mel, int stop_mel, int D, int r16, float* out, int text_rows, int mel_rows, int* bad) {
  const int row = blockIdx.x;
  for (int c = threadIdx.x; c < D; c += blockDim.x) {
    float v;
    if (row < n_lat) {
      v = conds[(size_t)row * D + c];
    } else if (row < n_lat + n_text + 2) {
      const int j = row - n_lat;
      int id = (j == 0) ? 0 : (j == n_text + 1 ? 1 : text_ids[j - 1]);
      if (id < 0 || id >= text_rows) { if (c == 0) atomicCAS(bad, 0, j); id = 0; }
      v = rnd(text_emb[(size_t)id * D + c] + text_pos[(size_t)j * D + c], r16);
    } else {
      const int i = row - (n_lat + n_text + 2);
      int tok = (i == 0) ? start_mel : (i == n_codes + 1 ? stop_mel : codes[i - 1]);
      if (tok < 0 || tok >= mel_rows) { if (c == 0) atomicCAS(bad, 0, n_text + 2 + i); tok = 0; }
      v = rnd(mel_emb[(size_t)tok * D + c] + mel_pos[(size_t)i * D + c], r16);
    }
    out[(size_t)row * D + c] = v;
  }
}
}  // namespace

static void v1_rows(idx_engine* e, GptState* g, const float* d_conds, int n_lat, const int* d_ids, int n_text, const int* d_codes,
                    int n_codes, float* d_out) {
  const int D = g->cfg.model_dim;
  const DevTensor& tpos = e->W("gpt.text_pos_embedding.emb.weight");
  IDX_CHECK(n_text + 2 <= tpos.shape[0], IDX_ERR_ARG, "text longer than text_pos_embedding");
  const int rows = n_lat + n_text + 2 + (n_codes >= 0 ? n_codes + 2 : 0);
  if (n_codes >= 0)
    IDX_CHECK(n_codes + 2 <= e->W("gpt.mel_pos_embedding.emb.weight").shape[0], IDX_ERR_ARG, "codes longer than mel_pos_embedding");
  v1_rows_kernel<<<rows, 256, 0, e->stream>>>(d_conds, n_lat, d_ids, n_text, d_codes, n_codes, e->Wf("gpt.text_embedding.weight"),
                                              (const float*)tpos.d, e->Wf("gpt.mel_embedding.weight"),
                                              e->Wf("gpt.mel_pos_embedding.emb.weight"), g->cfg.start_mel_token,
                                              g->cfg.stop_mel_token, D, g->cfg.weights_bf16, d_out,
                                              (int)e->W("gpt.text_embedding.weight").shape[0],
                                              (int)e->W("gpt.mel_embedding.weight").shape[0], e->dev_flag);
  IDX_CUDA(cudaGetLastError());
  e->launches++;
}

extern "C" int idx_gpt_prepare_inputs_v1(idx_engine* e, const float* conds, int n_latents, const int32_t* text_ids, int n_text,
                                         float* out) {
  IDX_API_BEGIN
  IDX_CHECK(e && e->gpt, IDX_ERR_STATE, "idx_gpt_init has not been called");
  IDX_CHECK(conds && out && n_latents >= 1 && n_text >= 0 && (n_text == 0 || text_ids), IDX_ERR_ARG, "bad arguments");
  IDX_CUDA(cudaSetDevice(e->device));
  GptState* g = e->gpt;
  const int D = g->cfg.model_dim, rows = n_latents + n_text + 2;
  e->ensure_arena(4 * ((size_t)(rows + n_latents) * D + (size_t)n_text + 16) + (1 << 16));
  e->arena.reset();
  float* d_c = e->arena.get<float>((size_t)n_latents * D);
  int* d_ids = e->arena.get<int>(n_text + 1);
  float* d_out = e->arena.get<float>((size_t)rows * D);
  idx_to_device(e, d_c, conds, (size_t)n_latents * D * 4);
  if (n_text) idx_to_device(e, d_ids, text_ids, (size_t)n_text * 4);
  v1_rows(e, g, d_c, n_latents, d_ids, n_text, nullptr, -1, d_out);
  idx_from_device(e, out, d_out, (size_t)rows * D * 4);
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  e->check_flag("text token id outside text_embedding");
  IDX_API_END(e)
}

extern "C" int idx_gpt_latents_v1(idx_engine* e, const float* conds, int n_latents, const int32_t* text_ids, int n_text,
                                  const int32_t* codes, int n_codes, float* latents_out) {
  IDX_API_BEGIN
  IDX_CHECK(e && e->gpt, IDX_ERR_STATE, "idx_gpt_init has not been called");
  IDX_CHECK(conds && codes && latents_out && n_latents >= 1 && n_text >= 0 && n_codes >= 1, IDX_ERR_ARG, "bad arguments");
  IDX_CUDA(cudaSetDevice(e->device));
  GptState* g = e->gpt;
  GptStrict* s = g->strict;
  const int D = g->cfg.model_dim, R = n_latents + n_text + 2 + n_codes + 2;
  IDX_CHECK(R <= g->maxpos, IDX_ERR_ARG, "sequence longer than the KV cache");
  for (int i = 0; i < n_codes; ++i) (void)i;
  e->ensure_arena(4 * ((size_t)(2 * R + n_latents + 2 * n_codes + 2) * D + (size_t)n_text + n_codes + 32) +
                  (size_t)(R / 8 + 2) * sizeof(PrefillTile) + (1 << 16));
  e->arena.reset();
  float* d_c = e->arena.get<float>((size_t)n_latents * D);
  int* d_ids = e->arena.get<int>(n_text + 1);
  int* d_codes = e->arena.get<int>(n_codes);
  float* d_rows = e->arena.get<float>((size_t)R * D);
  float* d_lat = e->arena.get<float>((size_t)n_codes * D);
  idx_to_device(e, d_c, conds, (size_t)n_latents * D * 4);
  if (n_text) idx_to_device(e, d_ids, text_ids, (size_t)n_text * 4);
  idx_to_device(e, d_codes, codes, (size_t)n_codes * 4);
  v1_rows(e, g, d_c, n_latents, d_ids, n_text, d_codes, n_codes, d_rows);
  const int first = R - (n_codes + 2);                 // first mel row; latents = rows first .. first + n_codes - 1
  cudaStream_t st = e->stream;
  g->last_launches = 0;
  if (!s) {
    // bf16 path: one prefill sweep of the fused kernel (tiles of 8 rows, sequence slot 0) that dumps the residual stream
    std::vector<PrefillTile> tiles;
    for (int p0 = 0; p0 < R - 2; p0 += 8) tiles.push_back({0, p0, std::min(8, R - 2 - p0), p0});
    PrefillTile* d_tiles = e->arena.get<PrefillTile>(tiles.size());
    float* d_hid = e->arena.get<float>((size_t)R * D);
    float* d_tmp = e->arena.get<float>((size_t)n_codes * D);
    IDX_CUDA(cudaMemcpyAsync(d_tiles, tiles.data(), tiles.size() * sizeof(PrefillTile), cudaMemcpyHostToDevice, st));
    IDX_CUDA(cudaStreamSynchronize(st));
    GptParams p;
    fill_common(e, g, p);
    p.B = 8; p.mode = 0; p.nsteps = (int)tiles.size(); p.prompt = d_rows; p.tiles = d_tiles; p.hidden_out = d_hid;
    p.max_new = 1; p.rep_penalty = 1.f;
    launch_fused_bt(e, g, p, 8);
    layernorm(e, d_hid + (size_t)first * D, d_tmp, 1, n_codes, D, e->Wf("gpt.gpt.ln_f.weight"), e->Wf("gpt.gpt.ln_f.bias"), 1e-5f,
              nullptr, nullptr, 0);
    layernorm(e, d_tmp, d_lat, 1, n_codes, D, e->Wf("gpt.final_norm.weight"), e->Wf("gpt.final_norm.bias"), 1e-5f, nullptr, nullptr, 0);
    idx_from_device(e, latents_out, d_lat, (size_t)n_codes * D * 4);
    IDX_CUDA(cudaStreamSynchronize(e->stream));
    e->check_flag("text token id or speech code outside its embedding table");
    return IDX_OK;
  }
  // strict fp32: one teacher-forced sweep, position by position (the KV cache of the strict path is the causal mask)
  for (int pos = 0; pos < R - 2; ++pos) {              // the last two rows are dropped by the caller of get_logits (:583)
    strict_embed_kernel<<<(D + 255) / 256, 256, 0, st>>>(s->x, d_rows + (size_t)pos * D, nullptr, nullptr, nullptr, 0, D);
    strict_layers(e, g, pos);
    if (pos >= first) {
      strict_ln_kernel<<<1, 256, 0, st>>>(s->x, e->Wf("gpt.gpt.ln_f.weight"), e->Wf("gpt.gpt.ln_f.bias"), s->h, D);
      strict_ln_kernel<<<1, 256, 0, st>>>(s->h, e->Wf("gpt.final_norm.weight"), e->Wf("gpt.final_norm.bias"),
                                          d_lat + (size_t)(pos - first) * D, D);
      e->launches += 2;
    }
  }
  IDX_CUDA(cudaGetLastError());
  idx_from_device(e, latents_out, d_lat, (size_t)n_codes * D * 4);
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  e->check_flag("text token id outside text_embedding");
  IDX_API_END(e)
}
