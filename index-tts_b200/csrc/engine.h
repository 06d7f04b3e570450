// engine.h — internal state of libidxtts.so (not part of the C-ABI; see include/idxtts.h).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <string>
#include <vector>
#include <unordered_map>
#include <stdexcept>
#include "../../include/idxtts.h"

struct IdxError : std::runtime_error {
  int code;
  IdxError(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

#define IDX_CUDA(call)                                                                    \
  do {                                                                                    \
    cudaError_t err__ = (call);                                                           \
    if (err__ != cudaSuccess)                                                             \
      throw IdxError(IDX_ERR_CUDA, std::string(#call) + " failed: " +                     \
                                       cudaGetErrorString(err__) + " at " + __FILE__ +   \
                                       ":" + std::to_string(__LINE__));                  \
  } while (0)

#define IDX_CHECK(cond, code, msg)                                                        \
  do {                                                                                    \
    if (!(cond)) throw IdxError((code), std::string(msg));                                \
  } while (0)

struct DevTensor {
  void* d = nullptr;  // device pointer owned by the engine
  int dtype = IDX_F32;
  std::vector<int64_t> shape;
  size_t numel() const {
    size_t n = 1;
    for (auto s : shape) n *= (size_t)s;
    return n;
  }
};

static inline size_t idx_dtype_size(int dt) {
  switch (dt) {
    case IDX_F32: return 4;
    case IDX_BF16: return 2;
    case IDX_F16: return 2;
    case IDX_I32: return 4;
    case IDX_I64: return 8;
  }
  return 0;
}

struct GptState;      // gpt_decode.cu
struct EmoState;      // emo.cu
struct V1VocoderState; // bigvgan.cu (latent-conditioned BigVGAN + ECAPA-TDNN, row a13)
struct BigvganState;  // bigvgan.cu
struct S2melState;    // s2mel.cu
struct SemanticState; // semantic.cu

// Bump allocator for per-call activations: reset at the start of each forward call.
struct Arena {
  char* base = nullptr;
  size_t cap = 0, off = 0, high = 0;
  void* alloc(size_t bytes) {
    size_t a = (off + 255) & ~(size_t)255;
    if (a + bytes > cap)
      throw IdxError(IDX_ERR_ARG, "arena exhausted: need " + std::to_string(a + bytes) +
                                      " of " + std::to_string(cap));
    off = a + bytes;
    if (off > high) high = off;
    return base + a;
  }
  template <typename T>
  T* get(size_t n) { return (T*)alloc(n * sizeof(T)); }
  void reset() { off = 0; }
};

struct idx_engine {
  int device = 0;
  int num_sms = 0;
  cudaStream_t stream = nullptr;
  std::string err;
  int64_t launches = 0;
  std::unordered_map<std::string, DevTensor> weights;
  Arena arena;
  // pinned staging for host<->device copies
  void* pinned = nullptr;
  size_t pinned_cap = 0;
  cudaEvent_t events[16] = {};
  cudaEvent_t order_ev = nullptr;   // idx_wait_stream: orders the engine stream after a caller stream
  int gemm_backend = 0;         // idx_set_option("gemm_backend"): 0 auto (wgmma tf32 where applicable), 1 SIMT fp32 (IDX_NO_TC)
  int force_backend = 0;        // diagnostics (idx_debug_conv_gemm): 0 none, 1 SIMT, 2 tensor core
  int force_tile_n = 0;         // diagnostics (idx_debug_conv_gemm): tensor-core tile width, 0 automatic, 32 / 64 / 128
  int tail_f16 = 1;             // idx_set_option("tail_f16"): 1 fp16 GEMM operands on the tensor-core path (default), 0 tf32 over fp32 storage (IDX_TAIL_F16=0)
  unsigned attr_done = 0;       // bit i: >48 KB dynamic-smem attribute of kernel family i set on this engine's device
  int* dev_flag = nullptr;      // device word set by kernels that meet invalid input (index out of range)
  GptState* gpt = nullptr;
  BigvganState* bigvgan = nullptr;
  S2melState* s2mel = nullptr;
  EmoState* emo = nullptr;
  EmoState* v1cond = nullptr;   // v1 prompt encoder (32-latent conformer-perceiver)
  V1VocoderState* v1voc = nullptr;
  SemanticState* semantic = nullptr;   // w2v-BERT 2.0 prompt encoder (get_emb)

  const DevTensor& W(const std::string& name) const {
    auto it = weights.find(name);
    if (it == weights.end()) throw IdxError(IDX_ERR_ARG, "missing weight: " + name);
    return it->second;
  }
  bool has(const std::string& name) const { return weights.find(name) != weights.end(); }
  // f32 view of a weight (converted copy is made at load time for non-f32 inputs)
  const float* Wf(const std::string& name) const {
    const DevTensor& t = W(name);
    IDX_CHECK(t.dtype == IDX_F32, IDX_ERR_ARG, "weight not f32: " + name);
    return (const float*)t.d;
  }
  void ensure_arena(size_t bytes);
  void* pinned_buf(size_t bytes);
  // read-and-clear dev_flag after the stream is idle; throws IdxError(IDX_ERR_ARG, what) when it was set
  void check_flag(const char* what);
};

// true if p is a device (or managed) pointer
bool idx_is_device_ptr(const void* p);
// copy `bytes` from a host-or-device pointer into a device buffer on the engine stream
void idx_to_device(idx_engine* e, void* dst_dev, const void* src, size_t bytes);
// copy from device buffer to host-or-device pointer (synchronises if dst is host)
void idx_from_device(idx_engine* e, void* dst, const void* src_dev, size_t bytes);

// module teardown hooks
void gpt_destroy(GptState*);
void bigvgan_destroy(BigvganState*);
void s2mel_destroy(S2melState*);
void emo_destroy(EmoState*);
void v1voc_destroy(V1VocoderState*);
void semantic_destroy(SemanticState*);

#define IDX_API_BEGIN try {
#define IDX_API_END(e)                                     \
  }                                                        \
  catch (const IdxError& ex) {                             \
    if (e) (e)->err = ex.what();                           \
    return ex.code;                                        \
  }                                                        \
  catch (const std::exception& ex) {                       \
    if (e) (e)->err = ex.what();                           \
    return IDX_ERR_ARG;                                    \
  }                                                        \
  return IDX_OK;
