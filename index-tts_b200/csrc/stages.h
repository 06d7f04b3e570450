// stages.h — device-level entry points of the pipeline stages (all pointers are device memory
// taken from the engine arena or owned by the caller; no host synchronisation inside).
#pragma once
#include "ops.h"

struct S2melState;
struct BigvganState;

size_t codec_arena_bytes(const S2melState* s, int n);
void codec_decode_dev(idx_engine* e, S2melState* s, const int* d_codes, int n, float* d_out);
size_t lr_arena_bytes(const S2melState* s, int n_in, int ylen);
void length_regulate_dev(idx_engine* e, S2melState* s, const float* d_S, int n_in, int ylen, float* d_out);
// The inputs of one CFM solve over T rows holding n utterances, in the CFG pair layout (cond, uncond): x [T][80] (the
// noise; the mel [T][80] when the solve returns), px / mu2 [2][T][80 | content] and st [2][n][style].
struct CfmInputs { float *x, *px, *mu2, *st; };
// takes them from the arena, px / mu2 / st zeroed (the uncond entry stays zero)
CfmInputs cfm_inputs(idx_engine* e, const S2melState* s, int T, int n);
// utterance u at rows [o, o + Tu): x = z^T with the first P frames zeroed, cond px = ref_mel^T, the first mu_rows cond rows
// of mu2 = mu, cond style u.  z [80][Tu], ref_mel [80][P], mu [mu_rows][content], style: host or device memory.
void cfm_stage(idx_engine* e, const S2melState* s, const CfmInputs& in, int u, int o, int Tu, int P, const float* z,
               const float* ref_mel, const float* mu, int mu_rows, const float* style);
// The CFM solve of the utterances of sg as ONE solve over their frames packed along T: segment u owns rows
// [off[u], off[u+1]) of both CFG batch entries and its first P[u] rows are prompt frames (include/idxtts.h
// idx_codes_to_wav_batch).  One segment issues the launches of a single-utterance solve; two or more upload sg and take
// the packed kernels, which exist only where cfm_half() holds.
void cfm_solve_dev(idx_engine* e, S2melState* s, Segments& sg, const int* P, const CfmInputs& in, int n_steps, float rate);
// arena of cfm_solve_dev over sg, with room for its staged inputs
size_t cfm_arena_bytes(const S2melState* s, const Segments& sg, int n_steps);
// true when the CFM solve runs the DiT / WaveNet on fp16 GEMM operands with the fused pair epilogues: tail_half() and shapes
// the fp16 kernels take.  The default mode, and the only one with the packed solve.
bool cfm_half(const idx_engine* e, const S2melState* s);
int s2mel_content_dim(const S2melState* s);
int s2mel_style_dim(const S2melState* s);
int s2mel_codec_hidden(const S2melState* s);
bool s2mel_ready(const S2melState* s);

size_t bigvgan_arena_bytes(const BigvganState* s, int B, int F);
int bigvgan_total_up(const BigvganState* s);
// d_mel [B][num_mels][F] (NCT) -> d_wav [B][F*total_up]
void bigvgan_forward_dev(idx_engine* e, BigvganState* s, const float* d_mel, int B, int F, float* d_wav);
// BigVGAN's fused Activation1d(SnakeBeta) over x [B][T][C] with the per-channel ea = exp(alpha) (or alpha) and
// ib = 1 / (exp(beta) (or beta) + 1e-9) of snake_params_dev; FIR taps of the loaded generator, else the computed ones
void snake_params_dev(idx_engine* e, const float* alpha, const float* beta, float* ea, float* ib, int C, int logscale);
void snake_act_dev(idx_engine* e, const float* ea, const float* ib, int C, const float* x, float* y, int B, int T, __half* y16);
// BigVGAN conv_post: Conv1d(C -> 1, k 7, pad 3) with w [7][C], optional bias [1], then tanh or a clamp to [-1, 1]; y [B][T]
void conv_post_dev(idx_engine* e, const float* x, const float* w, const float* bias, float* y, int B, int T, int C, int use_tanh);
void s2mel_set_ms(S2melState* s, double codec, double lr, double cfm);
void bigvgan_set_ms(BigvganState* s, double ms);

// v1 / v1.5 vocoder side (row a13): ECAPA-TDNN speaker encoder (ecapa.cu)
struct EcapaState;
EcapaState* ecapa_build(idx_engine* e, const std::string& prefix, int n_mels, int emb);
void ecapa_destroy(EcapaState* s);
size_t ecapa_arena_bytes(const EcapaState* s, int T);
// d_mel [T][n_mels] -> d_emb [emb]
void ecapa_forward_dev(idx_engine* e, EcapaState* s, const float* d_mel, int T, float* d_emb);
// per-channel statistics over the T rows of x [T][ld] (columns < C): mean [C] and, when std_out is given,
// std = sqrt(max(E[(x - mean)^2], 1e-12)) [C]
void ecapa_col_mean_std(idx_engine* e, const float* x, int ld, int T, int C, float* mean, float* std_out);
// attentive statistics pooling: per channel c, a = softmax over t of logit[t][c]; out [2C] = sum_t a x | sqrt(max(sum_t a (x -
// mean)^2, 1e-12)); logit, x [T][C]
void ecapa_asp_pool(idx_engine* e, const float* logit, const float* x, int T, int C, float* out);
