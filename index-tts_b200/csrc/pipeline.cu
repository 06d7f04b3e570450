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
// The windows of one idx_stream_vocode_batch call (at most one per slot), each joined onto the tail its slot kept
// (include/idxtts.h idx_stream_vocode), with the rules of the reference's StreamingDecoder.generate: out[i] = tail[i] *
// fade_out[i] + wav[i] * fade_in[i] for i < nb (the two halves of np.hanning(2 nb)), wav[src0 + i - nb] after that; the
// last 512 samples scaled by np.linspace(1, 0, 512) when `fade`; int16 with the truncation of pcm16_kernel.  In double,
// as numpy computes the blend.  blockIdx.y: the window.
struct JoinWin {
  const float* wav;
  const float* tail;
  int16_t* pcm;
  long long src0, n_out;
  int nb, fade;
};
struct JoinTable { JoinWin w[8]; };
__global__ void stream_join_kernel(JoinTable t) {
  const JoinWin& w = t.w[blockIdx.y];
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= w.n_out) return;
  const int nb = w.nb;
  double v;
  if (i < nb) {
    const double c = 6.283185307179586 / (2.0 * nb - 1.0);
    const double fade_in = 0.5 - 0.5 * cos(c * (double)i), fade_out = 0.5 - 0.5 * cos(c * (double)(nb + i));
    v = (double)w.tail[i] * fade_out + (double)w.wav[i] * fade_in;
  } else {
    v = (double)w.wav[w.src0 + i - nb];
  }
  if (w.fade && i >= w.n_out - 512) v *= 1.0 - (double)(i - (w.n_out - 512)) / 511.0;
  v = fmin(fmax(32767.0 * v, -32767.0), 32767.0);
  w.pcm[i] = (int16_t)v;
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

// idx_stream_vocode(_batch)'s device state: per slot the last overlap_samples of its previous window (kept until its next
// window blends them in), and the windows' waveform and int16 buffers, all engine-owned: the tail runs of the windows
// reset the arena.
struct StreamJoin {
  struct Slot {
    float* tail = nullptr;
    long long tail_len = 0, tail_cap = 0;
    bool has_tail = false;    // false: the slot's next window is joined as the first one
  } slot[IDX_STREAM_SLOTS];
  float* wav = nullptr;
  int16_t* pcm = nullptr;
  long long wav_cap = 0, pcm_cap = 0;
};

void stream_join_destroy(StreamJoin* j) {
  if (!j) return;
  for (auto& s : j->slot) cudaFree(s.tail);
  cudaFree(j->wav);
  cudaFree(j->pcm);
  delete j;
}

namespace {
// grow a device buffer to n elements, keeping its first `keep` elements
template <typename T>
void grow(idx_engine* e, T*& buf, long long& cap, long long n, long long keep) {
  if (cap >= n) return;
  T* nb = nullptr;
  IDX_CUDA(cudaMalloc((void**)&nb, (size_t)n * sizeof(T)));
  if (keep > 0) IDX_CUDA(cudaMemcpyAsync(nb, buf, (size_t)keep * sizeof(T), cudaMemcpyDeviceToDevice, e->stream));
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  cudaFree(buf);
  buf = nb;
  cap = n;
}

// What one window of a call emits: nb blended samples, then wav[src0, src0 + n_out - nb); len = its waveform's samples.
struct WinPlan {
  long long len = 0, nb = 0, src0 = 0, n_out = 0, wav_off = 0, pcm_off = 0;
  bool first = false, last = false;
};

void stream_vocode_batch(idx_engine* e, const idx_stream_window* w, int n, int n_steps, float cfg_rate) {
  IDX_CHECK(e && w && n >= 1 && n <= IDX_STREAM_SLOTS, IDX_ERR_ARG, "idx_stream_vocode: null argument or n not in 1..8");
  IDX_CUDA(cudaSetDevice(e->device));
  if (!e->sjoin) e->sjoin = new StreamJoin();
  StreamJoin* j = e->sjoin;
  // every window is checked before any work: a refused call emits nothing and keeps every slot's tail
  std::vector<WinPlan> plan(n);
  std::vector<idx_vocode_request> reqs;
  bool used[IDX_STREAM_SLOTS] = {};
  long long wav_total = 0, pcm_total = 0;
  for (int i = 0; i < n; ++i) {
    const idx_stream_window& x = w[i];
    const std::string at = n > 1 ? "idx_stream_vocode_batch: window " + std::to_string(i) + ": " : "idx_stream_vocode: ";
    auto need = [&](bool ok, const char* why) { if (!ok) throw IdxError(IDX_ERR_ARG, at + why); };
    need(x.pcm_out && x.n_pcm, "null argument");
    need(x.slot >= 0 && x.slot < IDX_STREAM_SLOTS, "slot must be 0..7");
    need(!used[x.slot], "the slot is used by another window of the call");
    used[x.slot] = true;
    need((x.flags & ~(IDX_STREAM_FIRST | IDX_STREAM_LAST)) == 0, "unknown flags");
    WinPlan& q = plan[i];
    q.first = x.flags & IDX_STREAM_FIRST;
    q.last = x.flags & IDX_STREAM_LAST;
    need(x.window || q.last, "a NULL window is the flush and needs IDX_STREAM_LAST");
    need(x.overlap_samples >= 0, "overlap_samples must be >= 0");
    const StreamJoin::Slot& sl = j->slot[x.slot];
    const bool joined = !q.first && sl.has_tail;      // a window without a kept tail is joined as the first one
    const long long kept = joined ? sl.tail_len : 0, ovlp = x.overlap_samples;
    if (x.window) {
      IDX_CHECK(e->bigvgan, IDX_ERR_STATE, "s2mel / codec / bigvgan not initialised");
      if (const char* why = request_error(x.window)) need(false, why);
      q.len = (long long)x.window->F * bigvgan_total_up(e->bigvgan);
      need(q.last || q.len >= 2 * ovlp, "a window that is not the last needs F * 256 >= 2 * overlap_samples");
    }
    need((long long)*x.n_pcm >= q.len + kept,
         "*n_pcm (the capacity of pcm_out) must be >= F * 256 plus the kept tail (at most the previous window's "
         "overlap_samples)");
    if (!x.window) {
      q.n_out = kept;
    } else if (!joined) {
      q.n_out = q.last ? q.len : q.len - ovlp;
    } else {
      const long long head = std::min(ovlp, q.len), rest = std::max(0LL, q.len - ovlp);
      q.nb = std::min(kept, head);
      q.src0 = std::min(ovlp, q.len);
      q.n_out = q.last ? q.nb + rest : q.nb + rest - ovlp;
    }
    q.wav_off = wav_total;
    q.pcm_off = pcm_total;
    wav_total += q.len;
    pcm_total += q.n_out;
  }
  grow(e, j->pcm, j->pcm_cap, std::max(pcm_total, 1LL), 0);
  grow(e, j->wav, j->wav_cap, std::max(wav_total, 1LL), 0);
  for (int i = 0; i < n; ++i)
    if (w[i].window) {
      reqs.push_back(*w[i].window);                   // the windows' tail: the driver of idx_codes_to_wav(_batch)
      reqs.back().wav_out = j->wav + plan[i].wav_off;
    }
  if (!reqs.empty()) codes_to_wav(e, reqs.data(), (int)reqs.size(), n_steps, cfg_rate, n > 1);
  for (int i = 0; i < n; ++i)
    if (w[i].window && w[i].window->wav_out)
      idx_from_device(e, w[i].window->wav_out, j->wav + plan[i].wav_off, (size_t)plan[i].len * 4);
  // one launch joins every window (the flush reads its slot's kept tail), before any slot keeps a new tail
  JoinTable t;
  memset(&t, 0, sizeof(t));
  long long max_out = 0;
  for (int i = 0; i < n; ++i) {
    const WinPlan& q = plan[i];
    const float* tail = j->slot[w[i].slot].tail;
    t.w[i] = {w[i].window ? j->wav + q.wav_off : tail, tail, j->pcm + q.pcm_off, q.src0, q.n_out, (int)q.nb,
              q.last && q.n_out > 512};
    max_out = std::max(max_out, q.n_out);
  }
  if (max_out > 0) {
    stream_join_kernel<<<dim3((unsigned)((max_out + 255) / 256), (unsigned)n), 256, 0, e->stream>>>(t);
    IDX_CUDA(cudaGetLastError()); e->launches++;
    for (int i = 0; i < n; ++i)
      if (plan[i].n_out > 0) idx_from_device(e, w[i].pcm_out, j->pcm + plan[i].pcm_off, (size_t)plan[i].n_out * 2);
  }
  for (int i = 0; i < n; ++i) {                       // keep each window's last overlap_samples for its slot's next one
    const WinPlan& q = plan[i];
    StreamJoin::Slot& sl = j->slot[w[i].slot];
    const long long ovlp = w[i].overlap_samples;
    if (w[i].window && !q.last) {
      grow(e, sl.tail, sl.tail_cap, std::max(ovlp, 1LL), 0);
      if (ovlp > 0)
        IDX_CUDA(cudaMemcpyAsync(sl.tail, j->wav + q.wav_off + (q.len - ovlp), (size_t)ovlp * 4, cudaMemcpyDeviceToDevice,
                                 e->stream));
    }
  }
  IDX_CUDA(cudaStreamSynchronize(e->stream));
  for (int i = 0; i < n; ++i) {
    StreamJoin::Slot& sl = j->slot[w[i].slot];
    sl.has_tail = w[i].window && !plan[i].last;
    sl.tail_len = sl.has_tail ? w[i].overlap_samples : 0;
    *w[i].n_pcm = (int32_t)plan[i].n_out;
  }
}
}  // namespace

extern "C" int idx_stream_vocode_batch(idx_engine* e, const idx_stream_window* w, int n, int n_steps, float cfg_rate) {
  IDX_API_BEGIN
  stream_vocode_batch(e, w, n, n_steps, cfg_rate);
  IDX_API_END(e)
}

extern "C" int idx_stream_vocode(idx_engine* e, const idx_vocode_request* r, int n_steps, float cfg_rate,
                                 int32_t overlap_samples, int32_t flags, int16_t* pcm_out, int32_t* n_pcm) {
  IDX_API_BEGIN
  const idx_stream_window w = {0, r, overlap_samples, flags, pcm_out, n_pcm};
  stream_vocode_batch(e, &w, 1, n_steps, cfg_rate);
  IDX_API_END(e)
}

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
