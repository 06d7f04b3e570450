// pipeline.cu — the per-segment "codes → waveform" tail of IndexTTS2.infer as one C-ABI call for one request or several:
// semantic-codec decode → length regulator → cat(prompt_condition) → CFM solve → crop the prompt
// frames → BigVGAN → clamp/int16.  Replaces indextts/infer_v2_5.py:827-856 (one text segment per request);
// every intermediate stays in HBM, the host sees only the requests and the waveforms.
#include "stages.h"
#include <algorithm>

namespace {
__global__ void crop_cols_kernel(const float* src, int ld_src, int col0, float* dst, int ncols, int rows) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)rows * ncols) return;
  const int r = (int)(i / ncols), c = (int)(i % ncols);
  dst[i] = src[(long long)r * ld_src + col0 + c];
}
__global__ void pcm16_kernel(const float* wav, int16_t* pcm, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  // wav = clamp(32767 * wav, -32767, 32767) (infer_v2_5.py:855) ; .type(torch.int16) truncates
  float v = fminf(fmaxf(32767.f * wav[i], -32767.f), 32767.f);
  pcm[i] = (int16_t)v;
}
// why the tail refuses a request, or nullptr
const char* request_error(const idx_vocode_request* r) {
  if (!(r->codes && r->n_codes >= 1 && r->F >= 1 && r->P >= 0 && r->style && r->z)) return "bad request";
  if (!(r->P == 0 || (r->prompt_condition && r->ref_mel))) return "prompt tensors missing";
  return nullptr;
}
// CUDA events of one call, destroyed with it
struct CallEvents {
  std::vector<cudaEvent_t> ev;
  cudaEvent_t record(cudaStream_t st) {
    cudaEvent_t x;
    IDX_CUDA(cudaEventCreate(&x));
    ev.push_back(x);
    IDX_CUDA(cudaEventRecord(x, st));
    return x;
  }
  ~CallEvents() { for (auto x : ev) cudaEventDestroy(x); }
};
float elapsed_ms(cudaEvent_t a, cudaEvent_t b) {
  float ms;
  IDX_CUDA(cudaEventElapsedTime(&ms, a, b));
  return ms;
}

// one CFM solve of a call: the requests [u0, u0 + sg.n()) packed along T, with their staged inputs
struct Solve {
  int u0 = 0;
  Segments sg;
  std::vector<int> P;
  CfmInputs in;
};

// The tail of n requests: every request's codec decode and length regulator, then the CFM solves, then per request the
// prompt-frame crop, BigVGAN and pcm16.  Where cfm_half() holds, ONE solve runs over the frames of all requests
// packed along T (request u owns rows [o_u, o_u + T_u) of both CFG batch entries; with one request that is the solo
// layout); in the other tail modes each request gets a solve of its own.  Outputs are written only after every stage has
// run and the codes have been checked.  batch: the error of a bad request names its index.
void codes_to_wav(idx_engine* e, const idx_vocode_request* reqs, int n, int n_steps, float cfg_rate, bool batch) {
  IDX_CHECK(s2mel_ready(e->s2mel) && e->bigvgan, IDX_ERR_STATE, "s2mel / codec / bigvgan not initialised");
  for (int u = 0; u < n; ++u)
    if (const char* why = request_error(&reqs[u]))
      throw IdxError(IDX_ERR_ARG, batch ? "request " + std::to_string(u) + ": " + why : why);
  IDX_CHECK(cfg_rate > 0.f, IDX_ERR_ARG, "inference_cfg_rate must be > 0 (the CFG pair path is the one built)");
  IDX_CUDA(cudaSetDevice(e->device));
  S2melState* s = e->s2mel;
  BigvganState* bv = e->bigvgan;
  const int Cd = s2mel_content_dim(s), Hs = s2mel_codec_hidden(s), C = 80, up = bigvgan_total_up(bv), Sd = s2mel_style_dim(s);
  const bool packed = cfm_half(e, s);
  std::vector<Solve> solves;
  for (int u = 0; u < n; ++u) {
    if (u == 0 || !packed) {
      solves.emplace_back();
      solves.back().u0 = u;
      solves.back().sg.off = {0};
    }
    solves.back().sg.off.push_back(solves.back().sg.total() + reqs[u].P + reqs[u].F);
    solves.back().P.push_back(reqs[u].P);
  }
  auto solve_of = [&](int u) -> Solve& { return solves[packed ? 0 : u]; };
  // persistent buffers, then the largest scratch of each phase (the phases reuse the arena above the persistent part)
  size_t keep = 0, scratch = 0;
  for (const Solve& v : solves) {
    const size_t T = v.sg.total();
    keep += 4 * (3 * T * C + 2 * T * Cd + 2 * v.P.size() * Sd) + 4 * 256;
    scratch = std::max(scratch, cfm_arena_bytes(s, v.sg, n_steps));
  }
  for (int u = 0; u < n; ++u) {
    const idx_vocode_request& r = reqs[u];
    const size_t Tu = (size_t)r.P + r.F;
    keep += 4 * (size_t)r.n_codes + 4 * (size_t)C * r.F + 6 * (size_t)r.F * up + 4 * 256;
    scratch = std::max(scratch, 4 * (size_t)C * (Tu + r.P) + 1024);
    scratch = std::max(scratch, codec_arena_bytes(s, r.n_codes) + lr_arena_bytes(s, 2 * r.n_codes, r.F) + 8 * (size_t)r.n_codes * Hs);
    scratch = std::max(scratch, 4 * (size_t)C * Tu + bigvgan_arena_bytes(bv, 1, r.F) + 1024);
  }
  e->ensure_arena(keep + scratch + (8 << 20));
  e->arena.reset();
  for (Solve& v : solves) v.in = cfm_inputs(e, s, v.sg.total(), v.sg.n());
  std::vector<int*> d_codes(n);
  std::vector<float*> d_melF(n), d_wav(n);
  std::vector<int16_t*> d_pcm(n);
  for (int u = 0; u < n; ++u) {
    const idx_vocode_request& r = reqs[u];
    d_codes[u] = e->arena.get<int>(r.n_codes);
    d_melF[u] = e->arena.get<float>((size_t)C * r.F);
    d_wav[u] = e->arena.get<float>((size_t)r.F * up);
    d_pcm[u] = (int16_t*)e->arena.alloc((size_t)r.F * up * 2);
  }
  const size_t mark = e->arena.off;
  for (int u = 0; u < n; ++u) {
    const idx_vocode_request& r = reqs[u];
    Solve& v = solve_of(u);
    const int k = u - v.u0;
    idx_to_device(e, d_codes[u], r.codes, (size_t)r.n_codes * 4);
    cfm_stage(e, s, v.in, k, v.sg.off[k], r.P + r.F, r.P, r.z, r.ref_mel, r.prompt_condition, r.P, r.style);
  }
  CallEvents ev;
  std::vector<cudaEvent_t> t_codec(n + 1), t_lr(n);
  for (int u = 0; u < n; ++u) {
    const idx_vocode_request& r = reqs[u];
    Solve& v = solve_of(u);
    float* d_S = e->arena.get<float>((size_t)2 * r.n_codes * Hs);
    t_codec[u] = ev.record(e->stream);
    codec_decode_dev(e, s, d_codes[u], r.n_codes, d_S);                                          // infer_v2_5.py:832
    t_lr[u] = ev.record(e->stream);
    length_regulate_dev(e, s, d_S, 2 * r.n_codes, r.F, v.in.mu2 + (size_t)(v.sg.off[u - v.u0] + r.P) * Cd);   // :835-840
    e->arena.off = mark;
  }
  t_codec[n] = ev.record(e->stream);
  for (Solve& v : solves) {
    cfm_solve_dev(e, s, v.sg, v.P.data(), v.in, n_steps, cfg_rate);                             // :841-845
    e->arena.off = mark;
  }
  cudaEvent_t t_cfm = ev.record(e->stream);
  std::vector<cudaEvent_t> t_bv(2 * n);
  for (int u = 0; u < n; ++u) {
    const idx_vocode_request& r = reqs[u];
    const Solve& v = solve_of(u);
    const int P = r.P, F = r.F, Tu = P + F;
    float* d_mel = e->arena.get<float>((size_t)C * Tu);
    transpose_btc_to_bct(e, v.in.x + (size_t)v.sg.off[u - v.u0] * C, d_mel, 1, Tu, C);
    t_bv[2 * u] = ev.record(e->stream);
    crop_cols_kernel<<<(unsigned)(((long long)C * F + 255) / 256), 256, 0, e->stream>>>(d_mel, Tu, P, d_melF[u], F, C);  // :846
    IDX_CUDA(cudaGetLastError()); e->launches++;
    bigvgan_forward_dev(e, bv, d_melF[u], 1, F, d_wav[u]);                                      // :850
    t_bv[2 * u + 1] = ev.record(e->stream);
    if (r.pcm16_out) {
      pcm16_kernel<<<(unsigned)(((long long)F * up + 255) / 256), 256, 0, e->stream>>>(d_wav[u], d_pcm[u], (long long)F * up);
      IDX_CUDA(cudaGetLastError()); e->launches++;
    }
    e->arena.off = mark;
  }
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  e->check_flag("semantic code outside the codebook (codes must be cut before the stop token, infer_v2_5.py:809-821)");
  for (int u = 0; u < n; ++u) {
    const idx_vocode_request& r = reqs[u];
    if (r.mel_out) idx_from_device(e, r.mel_out, d_melF[u], (size_t)C * r.F * 4);
    if (r.wav_out) idx_from_device(e, r.wav_out, d_wav[u], (size_t)r.F * up * 4);
    if (r.pcm16_out) idx_from_device(e, r.pcm16_out, d_pcm[u], (size_t)r.F * up * 2);
  }
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  double ms_codec = 0, ms_lr = 0, ms_bv = 0;
  for (int u = 0; u < n; ++u) {
    ms_codec += elapsed_ms(t_codec[u], t_lr[u]);
    ms_lr += elapsed_ms(t_lr[u], t_codec[u + 1]);
    ms_bv += elapsed_ms(t_bv[2 * u], t_bv[2 * u + 1]);
  }
  s2mel_set_ms(s, ms_codec, ms_lr, elapsed_ms(t_codec[n], t_cfm));
  bigvgan_set_ms(bv, ms_bv);
}
}  // namespace

extern "C" int idx_codes_to_wav(idx_engine* e, const idx_vocode_request* r, int n_steps, float cfg_rate) {
  IDX_API_BEGIN
  IDX_CHECK(e && r, IDX_ERR_ARG, "null argument");
  codes_to_wav(e, r, 1, n_steps, cfg_rate, false);
  IDX_API_END(e)
}

extern "C" int idx_codes_to_wav_batch(idx_engine* e, const idx_vocode_request* reqs, int n, int n_steps, float cfg_rate) {
  IDX_API_BEGIN
  IDX_CHECK(e && reqs && n >= 1, IDX_ERR_ARG, "idx_codes_to_wav_batch: null argument or n < 1");
  codes_to_wav(e, reqs, n, n_steps, cfg_rate, true);
  IDX_API_END(e)
}
