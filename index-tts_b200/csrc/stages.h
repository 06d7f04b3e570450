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
size_t cfm_arena_bytes(const S2melState* s, int T, int n_steps);
void cfm_solve_dev(idx_engine* e, S2melState* s, const float* d_mu, int T, const float* d_prompt, int P,
                   const float* d_style, const float* d_z, int n_steps, float rate, float* d_mel);
// several utterances' solves as one solve over their frames packed along T (s2mel.cu)
bool cfm_packed_supported(const idx_engine* e, const S2melState* s);
size_t cfm_packed_arena_bytes(const S2melState* s, int T, int nseg, int n_steps);
void cfm_solve_packed_dev(idx_engine* e, S2melState* s, const Segments& sg, float* x, const float* px, const float* mu2,
                          const float* st, const unsigned char* zero_rows, int n_steps, float rate);
int s2mel_content_dim(const S2melState* s);
int s2mel_style_dim(const S2melState* s);
int s2mel_codec_hidden(const S2melState* s);
bool s2mel_ready(const S2melState* s);

size_t bigvgan_arena_bytes(const BigvganState* s, int B, int F);
int bigvgan_total_up(const BigvganState* s);
// d_mel [B][num_mels][F] (NCT) -> d_wav [B][F*total_up]
void bigvgan_forward_dev(idx_engine* e, BigvganState* s, const float* d_mel, int B, int F, float* d_wav);
void s2mel_set_ms(S2melState* s, double codec, double lr, double cfm);
void bigvgan_set_ms(BigvganState* s, double ms);

// v1 / v1.5 vocoder side (row a13): ECAPA-TDNN speaker encoder (ecapa.cu)
struct EcapaState;
EcapaState* ecapa_build(idx_engine* e, const std::string& prefix, int n_mels, int emb);
void ecapa_destroy(EcapaState* s);
size_t ecapa_arena_bytes(const EcapaState* s, int T);
// d_mel [T][n_mels] -> d_emb [emb]
void ecapa_forward_dev(idx_engine* e, EcapaState* s, const float* d_mel, int T, float* d_emb);
