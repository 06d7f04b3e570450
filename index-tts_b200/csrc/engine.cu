// engine.cu — lifecycle, weight registry and host<->device staging of libidxtts.so.
#include "engine.h"
#include <cstdlib>
#include <cstring>
#include <mutex>

static std::string g_create_err;
static std::mutex g_mu;

bool idx_is_device_ptr(const void* p) {
  cudaPointerAttributes a;
  cudaError_t err = cudaPointerGetAttributes(&a, p);
  if (err != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

void idx_engine::ensure_arena(size_t bytes) {
  if (arena.cap >= bytes) return;
  IDX_CUDA(cudaStreamSynchronize(stream));
  if (arena.base) IDX_CUDA(cudaFree(arena.base));
  arena.base = nullptr;
  IDX_CUDA(cudaMalloc((void**)&arena.base, bytes));
  arena.cap = bytes;
  arena.off = 0;
}

void idx_engine::check_flag(const char* what) {
  int v = 0;
  IDX_CUDA(cudaMemcpyAsync(&v, dev_flag, 4, cudaMemcpyDeviceToHost, stream));
  IDX_CUDA(cudaStreamSynchronize(stream));
  if (v) {
    IDX_CUDA(cudaMemsetAsync(dev_flag, 0, 4, stream));
    throw IdxError(IDX_ERR_ARG, std::string(what) + " (first offending position " + std::to_string(v - 1) + ")");
  }
}

void* idx_engine::pinned_buf(size_t bytes) {
  if (pinned_cap < bytes) {
    if (pinned) cudaFreeHost(pinned);
    pinned = nullptr;
    size_t cap = bytes < (1u << 20) ? (1u << 20) : bytes;
    IDX_CUDA(cudaMallocHost(&pinned, cap));
    pinned_cap = cap;
  }
  return pinned;
}

void idx_to_device(idx_engine* e, void* dst_dev, const void* src, size_t bytes) {
  if (bytes == 0) return;
  if (idx_is_device_ptr(src)) {
    IDX_CUDA(cudaMemcpyAsync(dst_dev, src, bytes, cudaMemcpyDeviceToDevice, e->stream));
  } else {
    // host memory: works for pageable and pinned alike; ordered on the engine stream
    IDX_CUDA(cudaMemcpyAsync(dst_dev, src, bytes, cudaMemcpyHostToDevice, e->stream));
  }
}

void idx_from_device(idx_engine* e, void* dst, const void* src_dev, size_t bytes) {
  if (bytes == 0) return;
  if (idx_is_device_ptr(dst)) {
    IDX_CUDA(cudaMemcpyAsync(dst, src_dev, bytes, cudaMemcpyDeviceToDevice, e->stream));
  } else {
    IDX_CUDA(cudaMemcpyAsync(dst, src_dev, bytes, cudaMemcpyDeviceToHost, e->stream));
    IDX_CUDA(cudaStreamSynchronize(e->stream));
  }
}

__global__ void cvt_to_f32_kernel(const void* src, float* dst, size_t n, int dtype) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t stride = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    float v;
    if (dtype == IDX_BF16) v = __bfloat162float(((const __nv_bfloat16*)src)[i]);
    else if (dtype == IDX_F16) v = __half2float(((const __half*)src)[i]);
    else v = ((const float*)src)[i];
    dst[i] = v;
  }
}

extern "C" {

const char* idx_version(void) { return "idxtts 0.1 (sm_90a; cuda " "12.9" ")"; }

int idx_create(int device, idx_engine** out) {
  idx_engine* e = nullptr;
  try {
    int n = 0;
    cudaError_t err = cudaGetDeviceCount(&n);
    if (err != cudaSuccess || n == 0) {
      cudaGetLastError();
      throw IdxError(IDX_ERR_NOGPU,
                     "no CUDA device visible: libidxtts has no CPU fallback (sm_90a only)");
    }
    IDX_CHECK(device >= 0 && device < n, IDX_ERR_ARG, "bad device index");
    IDX_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    IDX_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)
      throw IdxError(IDX_ERR_NOGPU, std::string("device is sm_") + std::to_string(prop.major) +
                                        std::to_string(prop.minor) +
                                        ", libidxtts is built for sm_90a only");
    e = new idx_engine();
    e->device = device;
    e->num_sms = prop.multiProcessorCount;
    // initial precision options; idx_set_option changes them afterwards
    if (getenv("IDX_NO_TC")) e->gemm_backend = 1;
    if (getenv("IDX_TAIL_F16") && atoi(getenv("IDX_TAIL_F16")) == 0) e->tail_f16 = 0;
    IDX_CUDA(cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking));
    IDX_CUDA(cudaMalloc((void**)&e->dev_flag, 4));
    IDX_CUDA(cudaMemset(e->dev_flag, 0, 4));
    *out = e;
  } catch (const IdxError& ex) {
    std::lock_guard<std::mutex> lk(g_mu);
    g_create_err = ex.what();
    delete e;
    *out = nullptr;
    return ex.code;
  }
  return IDX_OK;
}

void idx_destroy(idx_engine* e) {
  if (!e) return;
  cudaSetDevice(e->device);
  cudaStreamSynchronize(e->stream);
  if (e->gpt) gpt_destroy(e->gpt);
  if (e->bigvgan) bigvgan_destroy(e->bigvgan);
  if (e->s2mel) s2mel_destroy(e->s2mel);
  if (e->emo) emo_destroy(e->emo);
  if (e->v1cond) emo_destroy(e->v1cond);
  if (e->semantic) semantic_destroy(e->semantic);
  if (e->v1voc) v1voc_destroy(e->v1voc);
  if (e->sjoin) stream_join_destroy(e->sjoin);
  for (auto& kv : e->weights) cudaFree(kv.second.d);
  for (auto ev : e->events) if (ev) cudaEventDestroy(ev);
  if (e->order_ev) cudaEventDestroy(e->order_ev);
  if (e->arena.base) cudaFree(e->arena.base);
  if (e->pinned) cudaFreeHost(e->pinned);
  if (e->dev_flag) cudaFree(e->dev_flag);
  cudaStreamDestroy(e->stream);
  delete e;
}

const char* idx_last_error(const idx_engine* e) {
  if (e) return e->err.c_str();
  return g_create_err.c_str();
}

int64_t idx_launch_count(const idx_engine* e) { return e ? e->launches : 0; }

int idx_sync(idx_engine* e) {
  IDX_API_BEGIN
  IDX_CUDA(cudaSetDevice(e->device));
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  IDX_API_END(e)
}

int idx_wait_stream(idx_engine* e, void* cuda_stream) {
  IDX_API_BEGIN
  IDX_CHECK(e, IDX_ERR_ARG, "null engine");
  IDX_CUDA(cudaSetDevice(e->device));
  if (!e->order_ev) IDX_CUDA(cudaEventCreateWithFlags(&e->order_ev, cudaEventDisableTiming));
  IDX_CUDA(cudaEventRecord(e->order_ev, (cudaStream_t)cuda_stream));
  IDX_CUDA(cudaStreamWaitEvent(e->stream, e->order_ev, 0));
  IDX_API_END(e)
}

int idx_event_record(idx_engine* e, int slot) {
  IDX_API_BEGIN
  IDX_CHECK(e && slot >= 0 && slot < 16, IDX_ERR_ARG, "bad event slot");
  IDX_CUDA(cudaSetDevice(e->device));
  if (!e->events[slot]) IDX_CUDA(cudaEventCreate(&e->events[slot]));
  IDX_CUDA(cudaEventRecord(e->events[slot], e->stream));
  IDX_API_END(e)
}

int idx_event_elapsed_ms(idx_engine* e, int slot_a, int slot_b, double* ms) {
  IDX_API_BEGIN
  IDX_CHECK(e && ms && slot_a >= 0 && slot_a < 16 && slot_b >= 0 && slot_b < 16 && e->events[slot_a] && e->events[slot_b],
            IDX_ERR_ARG, "bad event slots");
  IDX_CUDA(cudaSetDevice(e->device));
  IDX_CUDA(cudaEventSynchronize(e->events[slot_b]));
  float f = 0;
  IDX_CUDA(cudaEventElapsedTime(&f, e->events[slot_a], e->events[slot_b]));
  *ms = f;
  IDX_API_END(e)
}

int idx_load_weight(idx_engine* e, const char* name, const void* data, int dtype, int ndim,
                    const int64_t* shape) {
  IDX_API_BEGIN
  IDX_CHECK(e && name && data, IDX_ERR_ARG, "null argument");
  IDX_CHECK(dtype == IDX_F32 || dtype == IDX_BF16 || dtype == IDX_F16, IDX_ERR_ARG,
            "weights must be f32/bf16/f16");
  IDX_CUDA(cudaSetDevice(e->device));
  DevTensor t;
  t.dtype = IDX_F32;  // registry keeps f32 masters; modules repack to their own layouts
  for (int i = 0; i < ndim; ++i) t.shape.push_back(shape[i]);
  size_t n = t.numel();
  IDX_CHECK(n > 0, IDX_ERR_ARG, "empty weight");
  IDX_CUDA(cudaMalloc(&t.d, n * sizeof(float)));
  if (dtype == IDX_F32) {
    idx_to_device(e, t.d, data, n * 4);
  } else {
    void* tmp = nullptr;
    IDX_CUDA(cudaMalloc(&tmp, n * 2));
    idx_to_device(e, tmp, data, n * 2);
    cvt_to_f32_kernel<<<256, 256, 0, e->stream>>>(tmp, (float*)t.d, n, dtype);
    IDX_CUDA(cudaGetLastError());
    IDX_CUDA(cudaStreamSynchronize(e->stream));
    cudaFree(tmp);
  }
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  auto it = e->weights.find(name);
  if (it != e->weights.end()) {
    cudaFree(it->second.d);
    e->weights.erase(it);
  }
  e->weights.emplace(name, std::move(t));
  IDX_API_END(e)
}

}  // extern "C"
