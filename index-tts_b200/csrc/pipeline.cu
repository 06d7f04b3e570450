// pipeline.cu — the per-segment "codes → waveform" tail of IndexTTS2.infer as one C-ABI call:
// semantic-codec decode → length regulator → cat(prompt_condition) → CFM solve → crop the prompt
// frames → BigVGAN → clamp/int16.  Replaces indextts/infer_v2_5.py:827-856 (one text segment);
// every intermediate stays in HBM, the host sees only the request and the waveform.
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
// why idx_codes_to_wav refuses a request, or nullptr
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
}  // namespace

extern "C" int idx_codes_to_wav(idx_engine* e, const idx_vocode_request* r, int n_steps, float cfg_rate) {
  IDX_API_BEGIN
  IDX_CHECK(e && r, IDX_ERR_ARG, "null argument");
  IDX_CHECK(s2mel_ready(e->s2mel) && e->bigvgan, IDX_ERR_STATE, "s2mel / codec / bigvgan not initialised");
  if (const char* why = request_error(r)) throw IdxError(IDX_ERR_ARG, why);
  IDX_CUDA(cudaSetDevice(e->device));
  S2melState* s = e->s2mel;
  BigvganState* bv = e->bigvgan;
  const int n = r->n_codes, F = r->F, P = r->P, T = P + F;
  const int Cd = s2mel_content_dim(s), Hs = s2mel_codec_hidden(s), C = 80, up = bigvgan_total_up(bv);
  const int Sd = s2mel_style_dim(s);        // 192 for IndexTTS-2.5 (infer_v2_5.py:218); the caller's buffer holds exactly this many
  const size_t need = codec_arena_bytes(s, n) + lr_arena_bytes(s, 2 * n, F) + cfm_arena_bytes(s, T, n_steps) +
                      bigvgan_arena_bytes(bv, 1, F) +
                      4 * ((size_t)2 * n * Hs + (size_t)T * Cd + (size_t)C * (2 * T + P + F) + Sd + (size_t)F * up * 2) +
                      (8 << 20);
  e->ensure_arena(need);
  e->arena.reset();
  int* d_codes = e->arena.get<int>(n);
  float* d_S = e->arena.get<float>((size_t)2 * n * Hs);
  float* d_mu = e->arena.get<float>((size_t)T * Cd);
  float* d_prompt = e->arena.get<float>((size_t)C * std::max(P, 1));
  float* d_style = e->arena.get<float>(Sd);
  float* d_z = e->arena.get<float>((size_t)C * T);
  float* d_mel = e->arena.get<float>((size_t)C * T);
  float* d_melF = e->arena.get<float>((size_t)C * F);
  float* d_wav = e->arena.get<float>((size_t)F * up);
  int16_t* d_pcm = (int16_t*)e->arena.alloc((size_t)F * up * 2);
  idx_to_device(e, d_codes, r->codes, (size_t)n * 4);
  if (P > 0) {
    idx_to_device(e, d_mu, r->prompt_condition, (size_t)P * Cd * 4);
    idx_to_device(e, d_prompt, r->ref_mel, (size_t)C * P * 4);
  }
  idx_to_device(e, d_style, r->style, (size_t)Sd * 4);
  idx_to_device(e, d_z, r->z, (size_t)C * T * 4);
  auto stamp = [&](int slot) {
    if (!e->events[slot]) IDX_CUDA(cudaEventCreate(&e->events[slot]));
    IDX_CUDA(cudaEventRecord(e->events[slot], e->stream));
  };
  stamp(10);
  codec_decode_dev(e, s, d_codes, n, d_S);                              // infer_v2_5.py:832
  stamp(11);
  length_regulate_dev(e, s, d_S, 2 * n, F, d_mu + (size_t)P * Cd);      // :835-840 (cat with prompt_condition)
  stamp(12);
  cfm_solve_dev(e, s, d_mu, T, d_prompt, P, d_style, d_z, n_steps, cfg_rate, d_mel);   // :841-845
  stamp(13);
  crop_cols_kernel<<<(unsigned)(((long long)C * F + 255) / 256), 256, 0, e->stream>>>(d_mel, T, P, d_melF, F, C);  // :846
  IDX_CUDA(cudaGetLastError()); e->launches++;
  bigvgan_forward_dev(e, bv, d_melF, 1, F, d_wav);                      // :850
  stamp(14);
  if (r->mel_out) idx_from_device(e, r->mel_out, d_melF, (size_t)C * F * 4);
  if (r->wav_out) idx_from_device(e, r->wav_out, d_wav, (size_t)F * up * 4);
  if (r->pcm16_out) {
    pcm16_kernel<<<(unsigned)(((long long)F * up + 255) / 256), 256, 0, e->stream>>>(d_wav, d_pcm, (long long)F * up);
    IDX_CUDA(cudaGetLastError()); e->launches++;
    idx_from_device(e, r->pcm16_out, d_pcm, (size_t)F * up * 2);
  }
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  float m0, m1, m2, m3;
  IDX_CUDA(cudaEventElapsedTime(&m0, e->events[10], e->events[11]));
  IDX_CUDA(cudaEventElapsedTime(&m1, e->events[11], e->events[12]));
  IDX_CUDA(cudaEventElapsedTime(&m2, e->events[12], e->events[13]));
  IDX_CUDA(cudaEventElapsedTime(&m3, e->events[13], e->events[14]));
  s2mel_set_ms(s, m0, m1, m2);
  bigvgan_set_ms(bv, m3);
  e->check_flag("semantic code outside the codebook (codes must be cut before the stop token, infer_v2_5.py:809-821)");
  IDX_API_END(e)
}

// Every request's codec decode and length regulator, then ONE CFM solve over all their frames packed along T
// (utterance u owns rows [o_u, o_u + T_u) of both CFG batch entries), then per request the prompt-frame crop, BigVGAN and
// pcm16.  Outputs are written only after every stage has run and the codes have been checked.
extern "C" int idx_codes_to_wav_batch(idx_engine* e, const idx_vocode_request* reqs, int n, int n_steps, float cfg_rate) {
  IDX_API_BEGIN
  IDX_CHECK(e && reqs && n >= 1, IDX_ERR_ARG, "idx_codes_to_wav_batch: null argument or n < 1");
  IDX_CHECK(s2mel_ready(e->s2mel) && e->bigvgan, IDX_ERR_STATE, "s2mel / codec / bigvgan not initialised");
  for (int u = 0; u < n; ++u)
    if (const char* why = request_error(&reqs[u])) throw IdxError(IDX_ERR_ARG, "request " + std::to_string(u) + ": " + why);
  IDX_CHECK(cfg_rate > 0.f, IDX_ERR_ARG, "inference_cfg_rate must be > 0 (the CFG pair path is the one built)");
  IDX_CUDA(cudaSetDevice(e->device));
  S2melState* s = e->s2mel;
  BigvganState* bv = e->bigvgan;
  if (!cfm_packed_supported(e, s)) {
    // the reference modes (tf32, SIMT, unfused, mma.sync attention) have no packed solve: one request at a time
    double ms[3] = {0, 0, 0}, bms = 0;
    for (int u = 0; u < n; ++u) {
      const int rc = idx_codes_to_wav(e, &reqs[u], n_steps, cfg_rate);
      if (rc != IDX_OK) throw IdxError(rc, "request " + std::to_string(u) + ": " + e->err);
      double m3[3], mb;
      idx_s2mel_last_ms(e, m3);
      idx_bigvgan_last_ms(e, &mb);
      for (int i = 0; i < 3; ++i) ms[i] += m3[i];
      bms += mb;
    }
    s2mel_set_ms(s, ms[0], ms[1], ms[2]);
    bigvgan_set_ms(bv, bms);
    return IDX_OK;
  }
  const int Cd = s2mel_content_dim(s), Hs = s2mel_codec_hidden(s), C = 80, up = bigvgan_total_up(bv), Sd = s2mel_style_dim(s);
  Segments sg;
  sg.off.push_back(0);
  for (int u = 0; u < n; ++u) sg.off.push_back(sg.off.back() + reqs[u].P + reqs[u].F);
  const int T = sg.total();
  // persistent buffers, then the largest scratch of each phase (the phases reuse the arena above the persistent part)
  size_t keep = 4 * ((size_t)5 * T * C + 2 * (size_t)T * Cd + 2 * (size_t)n * Sd) + T + 256 * (size_t)(4 * n + 16) +
                (sizeof(int) + 16) * (size_t)(n + 1 + (T + 127) / 128 + n), scratch = 0;
  for (int u = 0; u < n; ++u) {
    const idx_vocode_request& r = reqs[u];
    const size_t Tu = (size_t)r.P + r.F;
    keep += 4 * (size_t)r.n_codes + 4 * (size_t)C * r.F + 6 * (size_t)r.F * up;
    scratch = std::max(scratch, codec_arena_bytes(s, r.n_codes) + lr_arena_bytes(s, 2 * r.n_codes, r.F) + 8 * (size_t)r.n_codes * Hs);
    scratch = std::max(scratch, 4 * (size_t)C * (Tu + r.P) + 1024);
    scratch = std::max(scratch, 4 * (size_t)C * Tu + bigvgan_arena_bytes(bv, 1, r.F) + 1024);
  }
  scratch = std::max(scratch, cfm_packed_arena_bytes(s, T, n, n_steps));
  e->ensure_arena(keep + scratch + (8 << 20));
  e->arena.reset();
  float* x = e->arena.get<float>((size_t)T * C);               // the solve state [T][80], the mel when it returns
  float* px = e->arena.get<float>((size_t)2 * T * C);
  float* mu2 = e->arena.get<float>((size_t)2 * T * Cd);
  float* st = e->arena.get<float>((size_t)2 * n * Sd);
  unsigned char* zero_rows = (unsigned char*)e->arena.alloc(T);
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
  segments_upload(e, sg);
  const size_t mark = e->arena.off;
  {
    std::vector<unsigned char> zr(T, 0);
    for (int u = 0; u < n; ++u) std::fill(zr.begin() + sg.off[u], zr.begin() + sg.off[u] + reqs[u].P, 1);
    idx_to_device(e, zero_rows, zr.data(), T);
  }
  fill_zero(e, px, (long long)2 * T * C);
  fill_zero(e, mu2, (long long)2 * T * Cd);
  fill_zero(e, st, (long long)2 * n * Sd);
  for (int u = 0; u < n; ++u) {     // the inputs cfm_solve_dev stacks, at each utterance's rows
    const idx_vocode_request& r = reqs[u];
    const int P = r.P, Tu = P + r.F, o = sg.off[u];
    float* d_z = e->arena.get<float>((size_t)C * Tu);
    idx_to_device(e, d_codes[u], r.codes, (size_t)r.n_codes * 4);
    idx_to_device(e, d_z, r.z, (size_t)C * Tu * 4);
    transpose_bct_to_btc(e, d_z, x + (size_t)o * C, 1, C, Tu);
    if (P > 0) {
      float* d_prompt = e->arena.get<float>((size_t)C * P);
      idx_to_device(e, d_prompt, r.ref_mel, (size_t)C * P * 4);
      transpose_bct_to_btc(e, d_prompt, px + (size_t)o * C, 1, C, P);
      fill_zero(e, x + (size_t)o * C, (long long)P * C);
      idx_to_device(e, mu2 + (size_t)o * Cd, r.prompt_condition, (size_t)P * Cd * 4);
    }
    idx_to_device(e, st + (size_t)u * Sd, r.style, (size_t)Sd * 4);
    e->arena.off = mark;
  }
  CallEvents ev;
  std::vector<cudaEvent_t> t_codec(n + 1), t_lr(n);
  for (int u = 0; u < n; ++u) {
    const idx_vocode_request& r = reqs[u];
    float* d_S = e->arena.get<float>((size_t)2 * r.n_codes * Hs);
    t_codec[u] = ev.record(e->stream);
    codec_decode_dev(e, s, d_codes[u], r.n_codes, d_S);
    t_lr[u] = ev.record(e->stream);
    length_regulate_dev(e, s, d_S, 2 * r.n_codes, r.F, mu2 + (size_t)(sg.off[u] + r.P) * Cd);
    e->arena.off = mark;
  }
  t_codec[n] = ev.record(e->stream);
  cfm_solve_packed_dev(e, s, sg, x, px, mu2, st, zero_rows, n_steps, cfg_rate);
  cudaEvent_t t_cfm = ev.record(e->stream);
  e->arena.off = mark;
  std::vector<cudaEvent_t> t_bv(2 * n);
  for (int u = 0; u < n; ++u) {
    const idx_vocode_request& r = reqs[u];
    const int P = r.P, F = r.F, Tu = P + F;
    float* d_mel = e->arena.get<float>((size_t)C * Tu);
    transpose_btc_to_bct(e, x + (size_t)sg.off[u] * C, d_mel, 1, Tu, C);
    t_bv[2 * u] = ev.record(e->stream);
    crop_cols_kernel<<<(unsigned)(((long long)C * F + 255) / 256), 256, 0, e->stream>>>(d_mel, Tu, P, d_melF[u], F, C);
    IDX_CUDA(cudaGetLastError()); e->launches++;
    bigvgan_forward_dev(e, bv, d_melF[u], 1, F, d_wav[u]);
    t_bv[2 * u + 1] = ev.record(e->stream);
    if (r.pcm16_out) {
      pcm16_kernel<<<(unsigned)(((long long)F * up + 255) / 256), 256, 0, e->stream>>>(d_wav[u], d_pcm[u], (long long)F * up);
      IDX_CUDA(cudaGetLastError()); e->launches++;
    }
    e->arena.off = mark;
  }
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  e->check_flag("semantic code outside the codebook (codes must be cut before the stop token, infer_v2_5.py:809-821)");
  double ms_codec = 0, ms_lr = 0, ms_bv = 0;
  for (int u = 0; u < n; ++u) {
    ms_codec += elapsed_ms(t_codec[u], t_lr[u]);
    ms_lr += elapsed_ms(t_lr[u], t_codec[u + 1]);
    ms_bv += elapsed_ms(t_bv[2 * u], t_bv[2 * u + 1]);
  }
  s2mel_set_ms(s, ms_codec, ms_lr, elapsed_ms(t_codec[n], t_cfm));
  bigvgan_set_ms(bv, ms_bv);
  for (int u = 0; u < n; ++u) {
    const idx_vocode_request& r = reqs[u];
    if (r.mel_out) idx_from_device(e, r.mel_out, d_melF[u], (size_t)C * r.F * 4);
    if (r.wav_out) idx_from_device(e, r.wav_out, d_wav[u], (size_t)r.F * up * 4);
    if (r.pcm16_out) idx_from_device(e, r.pcm16_out, d_pcm[u], (size_t)r.F * up * 2);
  }
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  IDX_API_END(e)
}
