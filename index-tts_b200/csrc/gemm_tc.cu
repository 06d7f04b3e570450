// gemm_tc.cu — wgmma implicit-GEMM back end of conv_gemm() for sm_90a.
//
//   D[b][m][n] = epi( sum_tap sum_k A[b][m + tap*dil - pad][k] * Wk[n][tap*K + k] )
//
// One CTA computes a 128 x BN output tile (M = time rows, N = output channels) with 160 threads:
//   warps 0..3  one warpgroup: issues wgmma (two M = 64 halves, N = BN, K = 8 tf32 / 16 fp16 per instruction, 4 K steps
//               per stage) from shared-memory descriptors into register accumulators, one commit group per stage, and frees
//               a stage as soon as the group that read it has retired; then the epilogue: the accumulator tile goes through
//               shared memory (the operand ring is dead by then) so that each warp applies bias / activation / layer-scale /
//               residual / accumulate / scale to 32 rows and stores with the generic (out_off, ldo, out_valid) mapping that
//               also serves ConvTranspose1d;
//   warp 4      TMA producer: per (tap, k-chunk) one 3-D box of the activations [B][T][K] (128 bytes along K x 128 rows,
//               SWIZZLE_128B; rows outside [0,T) and columns >= K are zero-filled by TMA = Conv1d zero padding / ragged K
//               for free) and one box of the K-major weights, into a ring of shared-memory stages (mbarrier full/empty).
// Two operand formats share the kernel (template EB = operand element bytes):
//   EB = 4: fp32 in HBM, tensor maps TFLOAT32 (the TMA unit rounds to tf32 on load), wgmma .tf32, K = 8 per MMA;
//   EB = 2: fp16 in HBM (activations written as fp16 by their producing kernel, weights converted once at init),
//           wgmma .f16, K = 16 per MMA: the same 10-bit mantissa as tf32 at half the bytes per operand — the tf32 tiles of
//           this kernel are bound by L2 -> shared-memory operand traffic (DESIGN.md), so halving the bytes is what counts.
// A 128-byte swizzle row holds 32 fp32 or 64 fp16 along K; a stage is always A 16 KB + B BN x 128 B.
#include "ops.h"
#include "ptx.cuh"
#include <cuda.h>
#include <cudaTypedefs.h>
#include <map>
#include <mutex>
#include <tuple>
#include <cstdlib>

namespace {

constexpr int BM = 128;
constexpr int BKB = 128; // bytes along K per stage row = one SWIZZLE_128B row (32 tf32 or 64 fp16 elements)
constexpr int GEMM_THREADS = 160;

__device__ __forceinline__ float apply_act_tc(float v, int act) {
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

struct TcParams {
  int M, N, K, taps, dil, pad, a_bcast, w_batched;
  int n_kchunks;        // ceil(K / (BKB / EB))
  const float* bias; int biasN; int act;
  const float* res; const float* rowscale; const float* colscale;
  int accum; float scale;
  float* out; long long out_batch_stride, out_off, out_valid; int ldo;
  int stages; int ring_bytes;   // ring_bytes = max(stages x stage, accumulator tile), a multiple of 1024
  int epi; __half* out16; const float* aux; int aux_stride;
};

// bytes of the fp32 accumulator tile staged for the epilogue: 128 rows x (BN + 1) (odd pitch: conflict-free row and column reads)
constexpr int acc_tile_bytes(int BN) { return BM * (BN + 1) * 4; }

template <int BN, int EB>
__global__ void __launch_bounds__(GEMM_THREADS, 2)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const TcParams p) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  // carve: stages x (A 16 KB | B BN*128 B) (later the accumulator tile), then barriers
  unsigned char* base = (unsigned char*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  constexpr int BK = BKB / EB;       // elements along K per stage
  constexpr int A_BYTES = BM * BKB;
  constexpr int B_BYTES = BN * BKB;
  constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  constexpr int TP = BN + 1;         // accumulator tile pitch (floats)
  uint64_t* full = (uint64_t*)(base + p.ring_bytes);
  uint64_t* empty = full + p.stages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n0 = blockIdx.x * BN, m0 = blockIdx.y * BM, b = blockIdx.z;
  const int n_iters = p.taps * p.n_kchunks;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      ptx::mbar_init(&full[s], 1);
      ptx::mbar_init(&empty[s], 4);   // lane 0 of each MMA warp, after its wgmma group that read the stage retired
    }
    ptx::fence_mbar_init();
  }
  __syncthreads();
  // everything above overlapped with the previous kernel of the stream (programmatic dependent launch); from here on
  // this grid reads what that kernel wrote
  pdl_wait();
  pdl_trigger();

  if (warp == 4) {
    if (lane == 0) {
      ptx::prefetch_tensormap(&tmA);
      ptx::prefetch_tensormap(&tmB);
      for (int it = 0; it < n_iters; ++it) {
        const int s = it % p.stages;
        const uint32_t ph = (it / p.stages) & 1u;
        ptx::mbar_wait(&empty[s], ph ^ 1u);
        const int tap = it / p.n_kchunks, kc = it % p.n_kchunks;
        unsigned char* sa = base + (size_t)s * STAGE_BYTES;
        unsigned char* sb = sa + A_BYTES;
        ptx::mbar_arrive_expect_tx(&full[s], STAGE_BYTES);
        ptx::tma_load_3d(sa, &tmA, &full[s], kc * BK, m0 + tap * p.dil - p.pad, p.a_bcast ? 0 : b);
        ptx::tma_load_3d(sb, &tmB, &full[s], tap * p.K + kc * BK, n0, p.w_batched ? b : 0);
      }
    }
    return;
  }

  // ---------------- MMA warpgroup (warps 0..3): rows 0..63 in acc0, 64..127 in acc1 ----------------
  float acc0[BN / 2], acc1[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; }
  for (int it = 0; it < n_iters; ++it) {
    const int s = it % p.stages;
    const uint32_t ph = (it / p.stages) & 1u;
    ptx::mbar_wait(&full[s], ph);
    const uint32_t sa = ptx::smem_u32(base + (size_t)s * STAGE_BYTES);
    const uint32_t sb = sa + A_BYTES;
    const uint64_t da = ptx::make_desc_sw128(sa), db = ptx::make_desc_sw128(sb);
    ptx::fence_regs(acc0);
    ptx::fence_regs(acc1);
    ptx::wgmma_fence();
#pragma unroll
    for (int k = 0; k < BKB / 32; ++k) {
      // one MMA consumes 32 bytes of K (8 tf32 / 16 fp16) inside the 128-byte swizzle row: +2 in 16-byte units;
      // the second M half starts 64 rows x 128 B = 8 KB further (+512)
      ptx::wgmma_ss<BN, EB>(acc0, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), 1u);
      ptx::wgmma_ss<BN, EB>(acc1, da + (uint64_t)(512 + 2 * k), db + (uint64_t)(2 * k), 1u);
    }
    ptx::wgmma_commit();
    ptx::wgmma_wait<1>();           // the group of stage it-1 has retired: its operands may be overwritten
    ptx::fence_regs(acc0);
    ptx::fence_regs(acc1);
    if (it > 0 && lane == 0) ptx::mbar_arrive(&empty[(it - 1) % p.stages]);
  }
  ptx::wgmma_wait<0>();
  ptx::fence_regs(acc0);
  ptx::fence_regs(acc1);

  // ---------------- epilogue: accumulators -> shared tile [128][BN + 1] -> 32 rows per warp ----------------
  // every stage has been consumed, so the ring is dead; the named barrier makes sure no warp still reads it
  ptx::named_bar_sync(1, 128);
  float* tile = (float*)base;
  {
    const int r0 = warp * 16 + (lane >> 2), c = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      float* t0 = tile + (size_t)r0 * TP + 8 * j + c;
      t0[0] = acc0[4 * j]; t0[1] = acc0[4 * j + 1];
      t0[8 * TP] = acc0[4 * j + 2]; t0[8 * TP + 1] = acc0[4 * j + 3];
      t0[64 * TP] = acc1[4 * j]; t0[64 * TP + 1] = acc1[4 * j + 1];
      t0[72 * TP] = acc1[4 * j + 2]; t0[72 * TP + 1] = acc1[4 * j + 3];
    }
  }
  ptx::named_bar_sync(1, 128);
  const int q = warp;                 // this warp's 32 rows of the tile
  const long long obs = p.out_batch_stride;
  const int biasN = p.biasN ? p.biasN : p.N;
  const int mrow0 = m0 + q * 32;
#pragma unroll 1
  for (int c0 = 0; c0 < BN; c0 += 32) {
    if (n0 + c0 >= p.N) break;
    const float* trow = tile + (size_t)(q * 32) * TP + c0;   // element (row rr, column j) of the chunk at trow[rr * TP + j]
    const int n = n0 + c0 + lane;
    if (p.epi != EPI_NONE) {
      // fused pair epilogues, thread = accumulator row: both columns of every pair are read by this thread, no shuffle;
      // each thread writes 16 or 32 fp16 values = whole 32-byte sectors.
      // (N is a multiple of 32 for these GEMMs: whole 32-column chunks only.)
      const int row = mrow0 + lane;
      if (row < p.M) {
        const int nb = n0 + c0;                                // first column of this chunk
        float v[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = trow[lane * TP + j] + (p.bias ? __ldg(p.bias + nb + j) : 0.f);
        if (p.epi == EPI_ROPE) {
          const int HD = 64, Hh = p.aux_stride, HW = Hh * HD;
          const int which = nb / HW, hh = (nb % HW) / HD, d0 = nb % HD;      // q | k | v, head, first dim of the chunk
          __half* dst = p.out16 + (size_t)which * ((size_t)gridDim.z * Hh * p.M * HD) + (((size_t)b * Hh + hh) * (size_t)p.M + row) * HD + d0;
          uint32_t o[16];
          if (which < 2) {
            const float4* tab = (const float4*)(p.aux + ((size_t)row * (HD / 2) + (d0 >> 1)) * 2);   // (cos, sin) pairs
            const float sc = (which == 0) ? p.scale : 1.0f;      // FLASH_Q_SCALE for the flash attention
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const float4 t4 = __ldg(tab + i);
              const float a0 = v[4 * i], a1 = v[4 * i + 1], b0 = v[4 * i + 2], b1 = v[4 * i + 3];
              __half2 h0 = __floats2half2_rn((a0 * t4.x - a1 * t4.y) * sc, (a1 * t4.x + a0 * t4.y) * sc);
              __half2 h1 = __floats2half2_rn((b0 * t4.z - b1 * t4.w) * sc, (b1 * t4.z + b0 * t4.w) * sc);
              o[2 * i] = *(uint32_t*)&h0;
              o[2 * i + 1] = *(uint32_t*)&h1;
            }
          } else {
#pragma unroll
            for (int i = 0; i < 16; ++i) {
              __half2 h = __floats2half2_rn(v[2 * i], v[2 * i + 1]);
              o[i] = *(uint32_t*)&h;
            }
          }
#pragma unroll
          for (int i = 0; i < 4; ++i) ((uint4*)dst)[i] = make_uint4(o[4 * i], o[4 * i + 1], o[4 * i + 2], o[4 * i + 3]);
        } else {
          const int NH = p.N >> 1, j0 = nb >> 1;
          uint32_t o[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            float r0, r1;
            if (p.epi == EPI_SWIGLU) {                          // F.silu(w1 x) * (w3 x)
              r0 = __fdividef(v[4 * i], 1.f + __expf(-v[4 * i])) * v[4 * i + 1];
              r1 = __fdividef(v[4 * i + 2], 1.f + __expf(-v[4 * i + 2])) * v[4 * i + 3];
            } else {                                            // fused_add_tanh_sigmoid_multiply
              const float* ga = p.aux + (size_t)b * p.aux_stride + j0 + 2 * i;
              r0 = tanhf(v[4 * i] + __ldg(ga)) * __fdividef(1.f, 1.f + __expf(-(v[4 * i + 1] + __ldg(ga + NH))));
              r1 = tanhf(v[4 * i + 2] + __ldg(ga + 1)) * __fdividef(1.f, 1.f + __expf(-(v[4 * i + 3] + __ldg(ga + NH + 1))));
            }
            __half2 h = __floats2half2_rn(r0, r1);
            o[i] = *(uint32_t*)&h;
          }
          uint4* dst = (uint4*)(p.out16 + ((size_t)b * p.M + row) * NH + j0);
          dst[0] = make_uint4(o[0], o[1], o[2], o[3]);
          dst[1] = make_uint4(o[4], o[5], o[6], o[7]);
        }
      }
    } else if (n < p.N) {
      // thread = column: every global load / store of this epilogue is a coalesced 128-byte row segment
      const float bv = p.bias ? __ldg(p.bias + (n % biasN)) : 0.f;
      const float cs = (p.colscale ? __ldg(p.colscale + n) : 1.f);
      const long long flat0 = p.out_off + (long long)mrow0 * p.ldo + n;     // row rr adds rr*ldo
      const int rows = min(32, p.M - mrow0);
      // fast path: the 32-row x 32-col chunk lies wholly inside the valid output range
      const bool interior = rows == 32 && (p.out_off + (long long)mrow0 * p.ldo + n0 + c0) >= 0 &&
                            (p.out_off + (long long)(mrow0 + 31) * p.ldo + n0 + c0 + 31) < p.out_valid;
      float* op = p.out + (long long)b * obs + flat0;
      const float* rp = p.res ? p.res + (long long)b * obs + flat0 : nullptr;
      if (interior && p.act == ACT_NONE && !p.rowscale) {
        const float sc = p.scale;
        if (!rp && !p.accum) {
#pragma unroll 8
          for (int rr = 0; rr < 32; ++rr) op[(long long)rr * p.ldo] = (trow[rr * TP + lane] + bv) * cs * sc;
        } else {
          // res may alias out (in-place residual): fetch the whole 32-row column into registers first so the
          // 32 L2 round trips overlap instead of serialising behind the stores
          float addv[32];
#pragma unroll
          for (int rr = 0; rr < 32; ++rr) {
            float a = 0.f;
            if (rp) a = rp[(long long)rr * p.ldo];
            if (p.accum) a += op[(long long)rr * p.ldo];
            addv[rr] = a;
          }
#pragma unroll
          for (int rr = 0; rr < 32; ++rr)
            op[(long long)rr * p.ldo] = ((trow[rr * TP + lane] + bv) * cs + addv[rr]) * sc;
        }
      } else {
        for (int rr = 0; rr < rows; ++rr) {
          const long long flat = flat0 + (long long)rr * p.ldo;
          if (flat < 0 || flat >= p.out_valid) continue;
          float v = trow[rr * TP + lane] + bv;
          v = apply_act_tc(v, p.act) * cs;
          if (p.rowscale) v *= __ldg(p.rowscale + (long long)b * p.M + mrow0 + rr);
          if (rp) v += rp[(long long)rr * p.ldo];
          if (p.accum) v += op[(long long)rr * p.ldo];
          op[(long long)rr * p.ldo] = v * p.scale;
        }
      }
    }
  }
}

PFN_cuTensorMapEncodeTiled get_encode() {
  static PFN_cuTensorMapEncodeTiled fn = nullptr;
  if (!fn) {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qres) != cudaSuccess || !f)
      throw IdxError(IDX_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
    fn = (PFN_cuTensorMapEncodeTiled)f;
  }
  return fn;
}

using MapKey = std::tuple<const void*, long long, long long, long long, long long, int, int>;
std::map<MapKey, CUtensorMap>& map_cache() {
  static std::map<MapKey, CUtensorMap> c;
  return c;
}

CUtensorMap make_map(const void* ptr, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                     const cuuint32_t* box, bool half = false) {
  static const bool plain_f32 = getenv("IDX_TMA_F32") != nullptr;
  MapKey key(ptr, (long long)dims[0], (long long)dims[1], rank > 2 ? (long long)dims[2] : 0,
             (long long)strides_bytes[0] ^ ((rank > 2 ? (long long)strides_bytes[1] : 0) << 20), (int)box[1] | ((int)box[0] << 12), rank | (half ? 16 : 0));
  // process-wide cache (keys carry the unique UVA address): engines may be driven from different threads
  static std::mutex mu;
  std::lock_guard<std::mutex> lock(mu);
  auto& cache = map_cache();
  auto it = cache.find(key);
  if (it != cache.end()) return it->second;
  CUtensorMap m;
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = get_encode()(&m, half ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : (plain_f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_TFLOAT32),
                            (cuuint32_t)rank, const_cast<void*>(ptr), dims, strides_bytes, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    throw IdxError(IDX_ERR_CUDA, "cuTensorMapEncodeTiled failed with code " + std::to_string((int)r));
  if (cache.size() > 20000) cache.clear();
  cache.emplace(key, m);
  return m;
}

template <int BN, int EB>
void launch_bn(idx_engine* e, const ConvGemm& g, const CUtensorMap& tmA, const CUtensorMap& tmB) {
  constexpr int BK = BKB / EB;
  TcParams p;
  p.M = g.M; p.N = g.N; p.K = g.K; p.taps = g.taps; p.dil = g.dil; p.pad = g.pad; p.a_bcast = g.a_bcast;
  p.w_batched = g.w_batch_stride != 0;
  p.n_kchunks = (g.K + BK - 1) / BK;
  p.bias = g.bias; p.biasN = g.biasN; p.act = g.act;
  p.res = g.res; p.rowscale = g.rowscale; p.colscale = g.colscale;
  p.accum = g.accum; p.scale = g.scale; p.out = g.out;
  p.ldo = g.ldo ? g.ldo : g.N;
  p.out_batch_stride = g.out_batch_stride ? g.out_batch_stride : (long long)g.M * g.N;
  p.out_off = g.out_off;
  p.out_valid = g.out_valid ? g.out_valid : (long long)g.M * p.ldo;
  p.epi = g.epi; p.out16 = g.out16; p.aux = g.aux; p.aux_stride = g.aux_stride;
  if (g.epi != EPI_NONE)
    IDX_CHECK(g.out16 && g.N % 32 == 0 && !g.res && !g.accum && g.act == ACT_NONE && (g.epi == EPI_SWIGLU || g.aux), IDX_ERR_ARG,
              "conv_gemm: bad fused-epilogue arguments");
  constexpr int STAGE = BM * BKB + BN * BKB;
  const int n_iters = p.taps * p.n_kchunks;
  static const int occ = getenv("IDX_GEMM_OCC") ? atoi(getenv("IDX_GEMM_OCC")) : 2;
  int stages = ((occ == 1 ? 208 : 104) * 1024) / STAGE;   // two CTAs per SM: one's epilogue overlaps the other's mainloop
  if (stages > 8) stages = 8;
  if (stages > n_iters) stages = n_iters < 2 ? 2 : n_iters;
  p.stages = stages;
  p.ring_bytes = ((stages * STAGE > acc_tile_bytes(BN) ? stages * STAGE : acc_tile_bytes(BN)) + 1023) & ~1023;
  const size_t smem = (size_t)p.ring_bytes + 1024 + 2 * stages * 8;
  const unsigned bit = (BN == 32 ? 1u : (BN == 64 ? 2u : 4u)) << (EB == 2 ? 8 : 0);
  if (!(e->attr_done & bit)) {     // per engine = per device: function attributes live in the device's context
    IDX_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<BN, EB>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
    e->attr_done |= bit;
  }
  dim3 grid((g.N + BN - 1) / BN, (g.M + BM - 1) / BM, g.B);
  launch_pdl(e, gemm_tc_kernel<BN, EB>, grid, dim3(GEMM_THREADS), smem, tmA, tmB, p);
  e->launches++;
}


// ================================================================================================================
// wgmma flash attention for the DiT (full attention, head dim 64, fp16 operands, fp32 softmax and accumulation).
//   gpt_fast/model.py:293-303 (F.scaled_dot_product_attention over all T keys; q arrives pre-scaled by log2(e)/8 and
//   rotated — EPI_ROPE above).
// One CTA = 128 queries of one (batch, head), 288 threads:
//   warps 0..7  two warpgroups of 64 query rows each.  Per key tile of 128: S = Q K_j^T (4 x wgmma M64 N128 K16, both
//               operands K-major in shared memory) into registers; online softmax in the log2 domain on the registers
//               (a row's 128 scores are spread over the 4 lanes of a quad); P_j packed to fp16 in place — the accumulator
//               layout of S is the register-operand layout of A — and O (+)= P_j V_j (8 x wgmma M64 N64 K16: A = P from
//               registers, B = V straight from its [key][dim] rows = MN-major operand);
//   warp 8      TMA: Q tile once, then K_j / V_j tiles of 128 keys into a 2-stage ring (SWIZZLE_128B rows of 64 fp16).
// The two warpgroups (and the two CTAs an SM holds) fill each other's softmax bubbles on the tensor cores.
// VARLEN: several sequences packed along T (the batched CFM solve).  CTA x takes query tile tiles[x] = (first query row,
// segment start, segment end), which lies inside one segment; its key tiles start at the segment start, so they align as in
// a solo run of that sequence, keys at or past the segment end are masked and query rows at or past it are not stored.
// RELKEY: the w2v-BERT encoder's attention (transformers wav2vec2_bert, position_embeddings_type "relative_key").  Keys at
// or past lens[b] are masked (the padding mask; every query row of the T is stored), and query row i adds
// qe[bh][i][clamp(j - i, -rel_l, rel_r) + rel_l] to its score against key j, where qe = Q E^T was computed from the same
// pre-scaled fp16 q, so it lands in the log2 domain of S.  A key tile wholly left (right) of a row's band adds the row's
// constant qe[..][0] (qe[..][rel_l + rel_r]); only the tiles that cross the band gather.
constexpr int FA_Q = 128, FA_K = 128, FA_D = 64;
constexpr int FA_THREADS = 288;
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t pack_half2(float lo, float hi) {
  __half2 h = __floats2half2_rn(lo, hi);
  return *(uint32_t*)&h;
}
struct FaParams {
  int T, H; float* out; __half* out16; const int4* tiles;
  const int* lens; const float* qe; int rel_l, rel_r;    // RELKEY only
};
// RELKEY: adds the relative-position term to the elements of S that belong to query row r (SEL 0: S[4c], S[4c + 1]; SEL 2:
// S[4c + 2], S[4c + 3]); element 4c + SEL + i is key k0 + 8c + 2 t4 + i.  qr = row r of qe [80], staged in shared memory
// (32-bit addresses: the gathers then fit next to S, O and P in the 168 registers of this kernel).
template <int SEL>
__device__ __forceinline__ void fa_add_relkey(float (&S)[FA_K / 2], const float* qr, int r, int k0, int t4, int L, int R) {
  if (k0 + FA_K - 1 - r <= -L || k0 - r >= R) {
    const float c = qr[k0 - r >= R ? L + R : 0];
#pragma unroll
    for (int c8 = 0; c8 < FA_K / 8; ++c8) { S[4 * c8 + SEL] += c; S[4 * c8 + SEL + 1] += c; }
  } else {
#pragma unroll
    for (int c8 = 0; c8 < FA_K / 8; ++c8) {
      const int d = k0 + 8 * c8 + 2 * t4 - r;
      S[4 * c8 + SEL] += qr[min(max(d, -L), R) + L];
      S[4 * c8 + SEL + 1] += qr[min(max(d + 1, -L), R) + L];
    }
  }
}
constexpr int FA_QE = 80;              // RELKEY: floats per row of qe (left + right + 1 <= 80)
template <bool VARLEN, bool RELKEY = false>
__global__ void __launch_bounds__(FA_THREADS, 1)
fa_wgmma_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                const FaParams p) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  unsigned char* base = (unsigned char*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  constexpr int TILE = FA_K * FA_D * 2;                  // 16 KB: 128 rows x 128 bytes
  unsigned char* sQ = base;
  unsigned char* sK = base + TILE;                       // [2][TILE]
  unsigned char* sV = base + 3 * TILE;                   // [2][TILE]
  uint64_t* bars = (uint64_t*)(base + 5 * TILE);
  uint64_t *q_full = bars, *kv_full = bars + 1, *kv_empty = bars + 3;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int bh = blockIdx.y;
  int q0 = blockIdx.x * FA_Q;
  const int T = p.T;
  int kbeg = 0, kend = T, ntiles = (T + FA_K - 1) / FA_K;
  if (threadIdx.x == 0) {
    ptx::mbar_init(q_full, 1);
    for (int s = 0; s < 2; ++s) { ptx::mbar_init(&kv_full[s], 1); ptx::mbar_init(&kv_empty[s], 8); }
    ptx::fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_trigger();
  if constexpr (VARLEN) {
    const int4 tl = p.tiles[blockIdx.x];
    q0 = tl.x; kbeg = tl.y; kend = tl.z;
    ntiles = (kend - kbeg + FA_K - 1) / FA_K;
  }
  if constexpr (RELKEY) {
    kend = p.lens[bh / p.H];
    ntiles = (kend + FA_K - 1) / FA_K;
  }

  if (warp == 8) {
    if (lane == 0) {
      ptx::prefetch_tensormap(&tmQ); ptx::prefetch_tensormap(&tmK); ptx::prefetch_tensormap(&tmV);
      ptx::mbar_arrive_expect_tx(q_full, TILE);
      ptx::tma_load_3d(sQ, &tmQ, q_full, 0, q0, bh);
      for (int j = 0; j < ntiles; ++j) {
        const int s = j & 1;
        ptx::mbar_wait(&kv_empty[s], ((j >> 1) & 1) ^ 1u);
        ptx::mbar_arrive_expect_tx(&kv_full[s], 2 * TILE);
        ptx::tma_load_3d(sK + s * TILE, &tmK, &kv_full[s], 0, kbeg + j * FA_K, bh);
        ptx::tma_load_3d(sV + s * TILE, &tmV, &kv_full[s], 0, kbeg + j * FA_K, bh);
      }
    }
    return;
  }

  const int wg = warp >> 2;                             // 64-row half of the query tile
  const int g = lane >> 2, t4 = lane & 3;
  // this thread's rows of the tile: rA = 64 wg + 16 (warp % 4) + g and rA + 8
  const int rA = wg * 64 + (warp & 3) * 16 + g;
  float S[FA_K / 2], O[FA_D / 2];
#pragma unroll
  for (int i = 0; i < FA_D / 2; ++i) O[i] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // running row max (log2 domain), this thread's share of the row sum
  if constexpr (RELKEY) {
    // this tile's 128 rows of qe into shared memory (rows past T repeat row T - 1; they are not stored)
    float* sqe = (float*)(base + 5 * TILE + 64);
    const float* qe = p.qe + (size_t)bh * T * FA_QE;
    for (int i = threadIdx.x; i < FA_Q * FA_QE; i += 256)
      sqe[i] = __ldg(qe + (size_t)min(q0 + i / FA_QE, T - 1) * FA_QE + i % FA_QE);
    ptx::named_bar_sync(1, 256);
  }
  ptx::mbar_wait(q_full, 0);
  const uint64_t dq = ptx::make_desc_sw128(ptx::smem_u32(sQ + wg * 64 * 128));
  for (int j = 0; j < ntiles; ++j) {
    const int s = j & 1;
    ptx::mbar_wait(&kv_full[s], (j >> 1) & 1u);
    const uint64_t dk = ptx::make_desc_sw128(ptx::smem_u32(sK + s * TILE));
    ptx::fence_regs(S);
    ptx::wgmma_fence();
#pragma unroll
    for (int k = 0; k < FA_D / 16; ++k) ptx::wgmma_ss<FA_K, 2>(S, dq + (uint64_t)(2 * k), dk + (uint64_t)(2 * k), k > 0 ? 1u : 0u);
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>();
    ptx::fence_regs(S);
    if constexpr (RELKEY) {
      const float* sqe = (const float*)(base + 5 * TILE + 64);
      fa_add_relkey<0>(S, sqe + rA * FA_QE, q0 + rA, j * FA_K, t4, p.rel_l, p.rel_r);
      fa_add_relkey<2>(S, sqe + (rA + 8) * FA_QE, q0 + rA + 8, j * FA_K, t4, p.rel_l, p.rel_r);
    }
    // keys beyond the sequence end (zero-filled rows past T, or the next packed sequence) are masked;
    // element 4c + i is key 8c + 2 t4 + (i & 1)
    const int nvalid = kend - kbeg - j * FA_K;
    if (nvalid < FA_K) {
#pragma unroll
      for (int c = 0; c < FA_K / 8; ++c) {
        const int key = 8 * c + 2 * t4;
        if (key >= nvalid) { S[4 * c] = -INFINITY; S[4 * c + 2] = -INFINITY; }
        if (key + 1 >= nvalid) { S[4 * c + 1] = -INFINITY; S[4 * c + 3] = -INFINITY; }
      }
    }
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int c = 0; c < FA_K / 8; ++c) {
      mx0 = fmaxf(mx0, fmaxf(S[4 * c], S[4 * c + 1]));
      mx1 = fmaxf(mx1, fmaxf(S[4 * c + 2], S[4 * c + 3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
    const float c0 = ex2_approx(m0 - mn0), c1 = ex2_approx(m1 - mn1);   // 0 at the first tile (m = -inf)
    // p = 2^(s - mn) packed to fp16 pairs: P[2c] = row rA keys (8c + 2 t4, +1), P[2c + 1] = row rA + 8, same keys
    uint32_t P[FA_K / 4];
    float rs0 = 0.f, rs1 = 0.f;
#pragma unroll
    for (int c = 0; c < FA_K / 8; ++c) {
      const float p0 = ex2_approx(S[4 * c] - mn0), p1 = ex2_approx(S[4 * c + 1] - mn0);
      const float p2 = ex2_approx(S[4 * c + 2] - mn1), p3 = ex2_approx(S[4 * c + 3] - mn1);
      rs0 += p0 + p1;
      rs1 += p2 + p3;
      P[2 * c] = pack_half2(p0, p1);
      P[2 * c + 1] = pack_half2(p2, p3);
    }
    l0 = l0 * c0 + rs0;
    l1 = l1 * c1 + rs1;
    m0 = mn0;
    m1 = mn1;
#pragma unroll
    for (int c = 0; c < FA_D / 8; ++c) { O[4 * c] *= c0; O[4 * c + 1] *= c0; O[4 * c + 2] *= c1; O[4 * c + 3] *= c1; }
    const uint64_t dv = ptx::make_desc_sw128(ptx::smem_u32(sV + s * TILE));
    ptx::fence_regs(O);
    ptx::wgmma_fence();
#pragma unroll
    for (int k = 0; k < FA_K / 16; ++k) {               // 16 keys per MMA: A = keys 16k..16k+15 of P, B = 16 V rows = 2048 bytes
      const uint32_t a[4] = {P[4 * k], P[4 * k + 1], P[4 * k + 2], P[4 * k + 3]};
      ptx::wgmma_rs_f16_n64_tb(O, a, dv + (uint64_t)(128 * k), 1u);
    }
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>();
    ptx::fence_regs(O);
    __syncwarp();
    if (lane == 0) ptx::mbar_arrive(&kv_empty[s]);      // K_j / V_j consumed by this warp
  }
  // epilogue: O / l -> fp16 (operand of the output projection) and / or fp32, [B][T][H*64]
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = l0 > 0.f ? 1.f / l0 : 0.f, i1 = l1 > 0.f ? 1.f / l1 : 0.f;
  const int b = bh / p.H, h = bh % p.H;
  const int t0 = q0 + rA, t1 = t0 + 8;
  if constexpr (RELKEY) kend = T;                 // masked keys, but every query row is stored
  const size_t o0 = ((size_t)b * T + t0) * (size_t)p.H * FA_D + (size_t)h * FA_D;
  const size_t o1 = o0 + (size_t)8 * p.H * FA_D;
#pragma unroll
  for (int c = 0; c < FA_D / 8; ++c) {
    const int d = 8 * c + 2 * t4;
    if (p.out16) {
      if (t0 < kend) *(uint32_t*)(p.out16 + o0 + d) = pack_half2(O[4 * c] * i0, O[4 * c + 1] * i0);
      if (t1 < kend) *(uint32_t*)(p.out16 + o1 + d) = pack_half2(O[4 * c + 2] * i1, O[4 * c + 3] * i1);
    }
    if (p.out) {
      if (t0 < kend) *(float2*)(p.out + o0 + d) = make_float2(O[4 * c] * i0, O[4 * c + 1] * i0);
      if (t1 < kend) *(float2*)(p.out + o1 + d) = make_float2(O[4 * c + 2] * i1, O[4 * c + 3] * i1);
    }
  }
}

}  // namespace

// wgmma flash attention on the rotated / split fp16 tensors Qr | Kr | Vb [B*H][T][64] (see fa_wgmma_kernel)
void flash_attention_wgmma(idx_engine* e, const __half* Qr, const __half* Kr, const __half* Vb, float* out, __half* out16,
                           int B, int T, int H) {
  const int BH = B * H;
  cuuint64_t dims[3] = {(cuuint64_t)FA_D, (cuuint64_t)T, (cuuint64_t)BH};
  cuuint64_t str[2] = {(cuuint64_t)FA_D * 2, (cuuint64_t)T * FA_D * 2};
  cuuint32_t box[3] = {FA_D, FA_K, 1};
  CUtensorMap tq = make_map(Qr, 3, dims, str, box, true), tk = make_map(Kr, 3, dims, str, box, true), tv = make_map(Vb, 3, dims, str, box, true);
  FaParams p;
  p.T = T; p.H = H; p.out = out; p.out16 = out16; p.tiles = nullptr;
  const size_t smem = 5 * (size_t)(FA_K * FA_D * 2) + 1024 + 64;
  if (!(e->attr_done & (1u << 20))) {
    IDX_CUDA(cudaFuncSetAttribute(fa_wgmma_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    e->attr_done |= 1u << 20;
  }
  launch_pdl(e, fa_wgmma_kernel<false>, dim3((T + FA_Q - 1) / FA_Q, BH), dim3(FA_THREADS), smem, tq, tk, tv, p);
  e->launches++;
}

void flash_attention_wgmma_varlen(idx_engine* e, const __half* Qr, const __half* Kr, const __half* Vb, float* out, __half* out16,
                                  int B, int H, const Segments& sg) {
  const int BH = B * H, T = sg.total();
  cuuint64_t dims[3] = {(cuuint64_t)FA_D, (cuuint64_t)T, (cuuint64_t)BH};
  cuuint64_t str[2] = {(cuuint64_t)FA_D * 2, (cuuint64_t)T * FA_D * 2};
  cuuint32_t box[3] = {FA_D, FA_K, 1};
  CUtensorMap tq = make_map(Qr, 3, dims, str, box, true), tk = make_map(Kr, 3, dims, str, box, true), tv = make_map(Vb, 3, dims, str, box, true);
  FaParams p;
  p.T = T; p.H = H; p.out = out; p.out16 = out16; p.tiles = sg.d_fa_tiles;
  const size_t smem = 5 * (size_t)(FA_K * FA_D * 2) + 1024 + 64;
  if (!(e->attr_done & (1u << 21))) {
    IDX_CUDA(cudaFuncSetAttribute(fa_wgmma_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    e->attr_done |= 1u << 21;
  }
  launch_pdl(e, fa_wgmma_kernel<true>, dim3(sg.fa_tiles, BH), dim3(FA_THREADS), smem, tq, tk, tv, p);
  e->launches++;
}

void flash_attention_wgmma_relkey(idx_engine* e, const __half* Qr, const __half* Kr, const __half* Vb, const float* qe,
                                  const int* lens, int rel_l, int rel_r, __half* out16, int B, int T, int H) {
  const int BH = B * H;
  cuuint64_t dims[3] = {(cuuint64_t)FA_D, (cuuint64_t)T, (cuuint64_t)BH};
  cuuint64_t str[2] = {(cuuint64_t)FA_D * 2, (cuuint64_t)T * FA_D * 2};
  cuuint32_t box[3] = {FA_D, FA_K, 1};
  CUtensorMap tq = make_map(Qr, 3, dims, str, box, true), tk = make_map(Kr, 3, dims, str, box, true), tv = make_map(Vb, 3, dims, str, box, true);
  FaParams p;
  p.T = T; p.H = H; p.out = nullptr; p.out16 = out16; p.tiles = nullptr;
  p.lens = lens; p.qe = qe; p.rel_l = rel_l; p.rel_r = rel_r;
  const size_t smem = 5 * (size_t)(FA_K * FA_D * 2) + 1024 + 64 + (size_t)FA_Q * FA_QE * 4;
  if (!(e->attr_done & (1u << 22))) {
    IDX_CUDA(cudaFuncSetAttribute(fa_wgmma_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    e->attr_done |= 1u << 22;
  }
  launch_pdl(e, fa_wgmma_kernel<false, true>, dim3((T + FA_Q - 1) / FA_Q, BH), dim3(FA_THREADS), smem, tq, tk, tv, p);
  e->launches++;
}

bool gemm_tc_supported(const ConvGemm& g) {
  const bool half = g.A16 && g.Wk16;
  if (g.reflect || (!g.Wk && !half)) return false;
  const int al = half ? 8 : 4;                                // 16-byte global strides: 8 fp16 / 4 fp32 elements
  if (g.K % al != 0) return false;
  const int lda = g.lda ? g.lda : g.K;
  if (lda % al != 0) return false;
  if (half ? (((uintptr_t)g.A16 & 15) || ((uintptr_t)g.Wk16 & 15)) : (((uintptr_t)g.A & 15) || ((uintptr_t)g.Wk & 15))) return false;
  const long long abs_ = g.a_batch_stride ? g.a_batch_stride : (long long)g.Tin * lda;
  if (abs_ % al != 0) return false;
  if ((g.ldw && g.ldw % al) || (g.w_batch_stride % al)) return false;
  if (!half && (long long)g.M * g.N * g.K * g.taps < (1 << 18)) return false;   // tiny problems: SIMT (fp16 operands have no SIMT twin)
  return true;
}

void gemm_tc_launch(idx_engine* e, const ConvGemm& g) {
  const bool half = g.A16 && g.Wk16;
  const int EBh = half ? 2 : 4;
  const int lda = g.lda ? g.lda : g.K;
  const long long abs_ = g.a_bcast ? (long long)g.Tin * lda : (g.a_batch_stride ? g.a_batch_stride : (long long)g.Tin * lda);
  // A: [B][Tin][K], dims (K, Tin, B)
  cuuint64_t adims[3] = {(cuuint64_t)g.K, (cuuint64_t)g.Tin, (cuuint64_t)(g.a_bcast ? 1 : g.B)};
  cuuint64_t astr[2] = {(cuuint64_t)lda * EBh, (cuuint64_t)abs_ * EBh};
  cuuint32_t abox[3] = {(cuuint32_t)(BKB / EBh), BM, 1};
  CUtensorMap tmA = make_map(half ? (const void*)g.A16 : (const void*)g.A, 3, adims, astr, abox, half);
  // B: Wk [nb][N][taps*K], dims (taps*K, N, nb)   (nb = 1 for shared weights)
  const int ldw = g.ldw ? g.ldw : g.taps * g.K;
  const long long wbs = g.w_batch_stride ? g.w_batch_stride : (long long)g.N * ldw;
  cuuint64_t bdims[3] = {(cuuint64_t)g.taps * g.K, (cuuint64_t)g.N, (cuuint64_t)(g.w_batch_stride ? g.B : 1)};
  cuuint64_t bstr[2] = {(cuuint64_t)ldw * EBh, (cuuint64_t)wbs * EBh};
  int BN = g.N <= 32 ? 32 : (g.N <= 64 ? 64 : 128);
  {
    // fewer 128-wide tiles than SMs: halve the tile so every SM gets work (2 CTAs/SM are resident anyway)
    static const int bn64 = getenv("IDX_GEMM_BN64") ? atoi(getenv("IDX_GEMM_BN64")) : 1;
    const long long tiles128 = (long long)((g.N + 127) / 128) * ((g.M + BM - 1) / BM) * g.B;
    if (bn64 && BN == 128 && tiles128 < e->num_sms) BN = 64;
  }
  if (e->force_tile_n) BN = e->force_tile_n;
  cuuint32_t bbox[3] = {(cuuint32_t)(BKB / EBh), (cuuint32_t)BN, 1};
  CUtensorMap tmB = make_map(half ? (const void*)g.Wk16 : (const void*)g.Wk, 3, bdims, bstr, bbox, half);
  if (half) {
    if (BN == 32) launch_bn<32, 2>(e, g, tmA, tmB);
    else if (BN == 64) launch_bn<64, 2>(e, g, tmA, tmB);
    else launch_bn<128, 2>(e, g, tmA, tmB);
  } else {
    if (BN == 32) launch_bn<32, 4>(e, g, tmA, tmB);
    else if (BN == 64) launch_bn<64, 4>(e, g, tmA, tmB);
    else launch_bn<128, 4>(e, g, tmA, tmB);
  }
}
