// gpt_decode8.cuh — decode of 2..8 sequences per group on the round-2 tile / ring structure (included by gpt_decode.cu
// after gpt_decode1.cuh, inside its anonymous namespace).
//
// Takes plain (non-beam) multi-sequence decode off `gpt_fused_kernel` — BASELINE configs 3 and 5 decode 8
// utterances per group.  The round-1 kernel spent 47 us per layer (profile of round 2: O-proj 11.7 us merging key splits for
// 8 x 20 (row, head) pairs, attention 8.6, FC 6.4, QKV 5.3, barriers 10.9): 1.1 ms per 8-row step.  Here:
//   * the m16n8k16 MMA's N = 8 columns are the 8 sequences (they were 7/8 wasted at batch 1), 16 real weight rows per tile,
//     all tiles of a phase in flight, the same row-granular bulk-copy weight ring and phase barriers as gpt_decode1_kernel;
//   * LayerNorm: one warp per sequence row; the normalised bf16 rows go to shared memory (swizzled for ldmatrix) and one B
//     fragment per k-step serves every tile of the phase;
//   * phases without a LayerNorm (O-proj, PROJ) take their B fragments straight from global memory into registers: the
//     producing epilogues store bf16 in FRAGMENT ORDER (frag_idx below), so a thread's operands of two k-steps are one
//     16-byte load and all loads of the phase are in flight before the first MMA (no 80 KB staging buffer);
//   * attention: one CTA per (sequence, head PAIR), the two heads on two groups of four warps, every key of the head
//     (no split, no merge pass), the normalised output written once;
//   * hand-overs between phases are grid barriers (the tagged-word protocol of the 1-row kernel would poll 8x the data);
//     the first LayerNorm of a step builds its input rows from the embedding tables, so a step has 5 L + 2 barriers.
// Same arithmetic, rounding points, sampler contract and KV-cache layout as the other GPT kernels; prefill stays on
// gpt_fused_kernel<8, .>, which leaves the cache and the per-sequence state exactly as this kernel expects them.

constexpr int B8 = 8;                                   // rows of the group (N of the MMA)
constexpr int RED8_FLOATS = MAXIT * NCW * 16 * B8;      // K-split partial sums [item][warp][16 weight rows][8 sequences]

struct Smem8 {
  __nv_bfloat16* ring;  // [R][D]
  __nv_bfloat16* xs;    // [8][D] LayerNorm output rows (bf16, 16-byte chunks XOR-swizzled by the row)
  float* red;           // [RED8_FLOATS]
  float* att;           // [NCW][66] attention merge
  uint64_t* full;       // [NBAR]
  Phase1* pht;          // [5]
  float* bias_s;
  float* xres;          // [8][ocap]
  unsigned* seen_s;     // [(V+31)/32] repetition bitmap of the sequence this CTA samples
  float* lnp;           // [2][2][D]
};

// Fragment order of an activation row that is consumed as the MMA's B operand straight from global memory: element k
// (k-step kk = k / 16) is stored so that thread t4's {b0, b1} of k-steps 2j and 2j + 1 are the four consecutive 32-bit
// words 16 j + 4 t4 .. + 3.
__device__ __forceinline__ int frag_idx(int k) {
  const int kk = k >> 4, r = k & 15;
  const int word = (kk >> 1) * 16 + ((r & 7) >> 1) * 4 + (kk & 1) * 2 + (r >> 3);
  return word * 2 + (r & 1);
}

// All MMAs of one phase for 8 sequences.  REGB = false: B from the swizzled rows in shared memory (ldmatrix.x2, one
// fragment per k-step for all tiles); REGB = true: B of item i from breg[i][.] (preloaded 16-byte fragments).
template <int D, int NIT, bool REGB>
__device__ __forceinline__ void mma8_n(const Smem8& sm, const Phase1& ph, int row0, unsigned phase_idx, int R, int warp, int lane,
                                       const uint4 (&breg)[REGB ? NIT : 1][(D / 16) / NCW / 2]) {
  constexpr int KS = (D / 16) / NCW;
  static_assert(KS % 2 == 0, "k-steps per warp must pair up");
  const uint32_t ring_base = ptx::smem_u32(sm.ring);
  const uint32_t xs_base = ptx::smem_u32(sm.xs);
  const int g = lane >> 2, t4 = lane & 3;
  const int lrow = (lane & 7) + ((lane >> 3) & 1) * 8, khalf = lane >> 4;
  const int bn = lane & 7, bhi = (lane >> 3) & 1;
  const uint32_t b_row = xs_base + (uint32_t)(bn * D * 2);
  uint32_t a_base[NIT];
  int key[NIT];
  float acc[NIT][4];
#pragma unroll
  for (int i = 0; i < NIT; ++i) {
    acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
    const int rr = min(lrow, max(ph.nrows[i] - 1, 0));     // rows beyond the tile read a valid row; their results are unused
    int slot = row0 + ph.off[i] + rr;
    if (slot >= R) slot -= R;
    a_base[i] = ring_base + (uint32_t)(slot * (D * 2));
    key[i] = rr & 7;
  }
  ptx::mbar_wait(&sm.full[phase_idx % NBAR], (phase_idx / NBAR) & 1u);
  uint32_t a[2][NIT][4], b[2][2];
#pragma unroll
  for (int i = 0; i < NIT; ++i)
    ldmatrix_x4(a_base[i] + (uint32_t)(((2 * (warp * KS) + khalf) ^ key[i]) << 4), a[0][i][0], a[0][i][1], a[0][i][2], a[0][i][3]);
  if constexpr (!REGB) ldmatrix_x2(b_row + (uint32_t)(((2 * (warp * KS) + bhi) ^ bn) << 4), b[0][0], b[0][1]);
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) {
    const int kk = warp * KS + ks;
    if (ks + 1 < KS) {
#pragma unroll
      for (int i = 0; i < NIT; ++i)
        ldmatrix_x4(a_base[i] + (uint32_t)(((2 * (kk + 1) + khalf) ^ key[i]) << 4), a[(ks + 1) & 1][i][0], a[(ks + 1) & 1][i][1],
                    a[(ks + 1) & 1][i][2], a[(ks + 1) & 1][i][3]);
      if constexpr (!REGB) ldmatrix_x2(b_row + (uint32_t)(((2 * (kk + 1) + bhi) ^ bn) << 4), b[(ks + 1) & 1][0], b[(ks + 1) & 1][1]);
    }
#pragma unroll
    for (int i = 0; i < NIT; ++i) {
      uint32_t b0, b1;
      if constexpr (REGB) {
        const uint4 w = breg[i][ks >> 1];
        b0 = (ks & 1) ? w.z : w.x;
        b1 = (ks & 1) ? w.w : w.y;
      } else {
        b0 = b[ks & 1][0];
        b1 = b[ks & 1][1];
      }
      mma_bf16_16816(acc[i], a[ks & 1][i][0], a[ks & 1][i][1], a[ks & 1][i][2], a[ks & 1][i][3], b0, b1);
    }
  }
  __syncwarp();
  // c0, c1: weight row g, sequences 2 t4, 2 t4 + 1 ; c2, c3: weight row g + 8
#pragma unroll
  for (int i = 0; i < NIT; ++i) {
    float* rp = sm.red + ((i * NCW + warp) * 16) * B8;
    *(float2*)(rp + g * B8 + 2 * t4) = make_float2(acc[i][0], acc[i][1]);
    *(float2*)(rp + (g + 8) * B8 + 2 * t4) = make_float2(acc[i][2], acc[i][3]);
  }
  ptx::named_bar_sync(1, NCT);
}

template <int D>
__device__ __forceinline__ void mma8_smem(const Smem8& sm, const Phase1& ph, int row0, unsigned phase_idx, int R, int warp, int lane) {
  const uint4 none[1][(D / 16) / NCW / 2] = {};
  switch (ph.nitems) {       // CTA-uniform
    case 1: mma8_n<D, 1, false>(sm, ph, row0, phase_idx, R, warp, lane, none); break;
    case 2: mma8_n<D, 2, false>(sm, ph, row0, phase_idx, R, warp, lane, none); break;
    case 3: mma8_n<D, 3, false>(sm, ph, row0, phase_idx, R, warp, lane, none); break;
    default: mma8_n<D, 4, false>(sm, ph, row0, phase_idx, R, warp, lane, none); break;
  }
}

__device__ __forceinline__ float red8_sum(const float* red, int item, int row, int b) {
  float a = 0.f;
#pragma unroll
  for (int w = 0; w < NCW; ++w) a += red[((item * NCW + w) * 16 + row) * B8 + b];
  return a;
}

template <int NPL>
__global__ void __launch_bounds__(NCT, 1) gpt_decode8_kernel(const GptParams p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  constexpr int D = NPL * 32, FF = 4 * D, NSEG = FF / D, KS = (D / 16) / NCW;
  static_assert(NSEG <= MAXIT, "PROJ K-segments must fit the item slots");
  const int G = p.G, L = p.L, H = p.H, V = p.V, R = p.ring_rows, B = p.B;
  const int cta = blockIdx.x;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wv = (V + 31) / 32;

  Smem8 sm;
  {
    unsigned char* q = smem_raw;
    sm.ring = (__nv_bfloat16*)q;  q += (size_t)R * D * 2;
    sm.xs = (__nv_bfloat16*)q;    q += (size_t)B8 * D * 2;
    sm.red = (float*)q;           q += sizeof(float) * RED8_FLOATS;
    sm.lnp = (float*)q;           q += sizeof(float) * 4 * (size_t)D;      // xs | red | lnp are contiguous: the attention phase stages K/V there
    sm.att = (float*)q;           q += sizeof(float) * NCW * PART_STRIDE;
    sm.full = (uint64_t*)q;       q += sizeof(uint64_t) * NBAR;
    sm.pht = (Phase1*)q;          q += 5 * sizeof(Phase1);
    q = (unsigned char*)(((uintptr_t)q + 15) & ~(uintptr_t)15);
    sm.bias_s = (float*)q;        q += sizeof(float) * (size_t)p.bias_cap;
    sm.xres = (float*)q;          q += sizeof(float) * (size_t)B8 * p.ocap;
    sm.seen_s = (unsigned*)q;     q += sizeof(unsigned) * (size_t)wv;
  }
  __shared__ int s_plen[B8], s_tok[B8], s_fin[B8], s_step0[B8], s_seq[B8];
  if (tid == 0) {
    for (int s = 0; s < NBAR; ++s) ptx::mbar_init(&sm.full[s], 1);
    ptx::fence_mbar_init();
  }
  // column slices of this CTA (same ownership as the other GPT kernels)
  const int q0 = col_begin(3 * D, cta, G), q1 = col_begin(3 * D, cta + 1, G);
  const int o0 = col_begin(D, cta, G), o1 = col_begin(D, cta + 1, G);
  const int f0 = col_begin(FF, cta, G), f1 = col_begin(FF, cta + 1, G);
  const int h0 = col_begin(V, cta, G), h1 = col_begin(V, cta + 1, G);
  const int nq = q1 - q0, no = o1 - o0, nf = f1 - f0, nh = h1 - h0;
  Sched1 sc;
  sc.L = L; sc.nseg = NSEG; sc.nq = nq; sc.no = no; sc.nf = nf; sc.nh = nh;
  sc.ntq = (nq + TROWS - 1) / TROWS; sc.ntf = (nf + TROWS - 1) / TROWS; sc.nth = (nh + TROWS - 1) / TROWS;
  const int bstride = nq + 2 * no + nf;
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
  if (cta < B)
    for (int i = tid; i < wv; i += NCT) sm.seen_s[i] = p.seen[(size_t)cta * wv + i];
  if (tid < B8) {
    s_plen[tid] = (tid < B) ? p.prompt_len[tid] : 0;
    s_tok[tid] = (tid < B) ? p.tok[tid] : 0;
    s_fin[tid] = (tid < B) ? p.finished[tid] : 1;
    s_step0[tid] = p.row_step0[tid];
    s_seq[tid] = p.row_seqidx[tid];
  }
  // Row b's own step at group step k.  Ordinary groups: k itself (k < max_new).  A finished or empty row of a serving
  // group runs on as a masked column for as long as the group does: the cap keeps its KV write, attention context and
  // mel position inside its own slot's rows.
  auto row_k = [&](int b, int k) { return min(k - s_step0[b], p.max_new - 1); };
  auto mel_row = [&](int kb) { return (kb == 0 || p.pos_plain) ? kb : kb + 1; };   // P1: mel position kb+1 with the KV cache
  auto make_phase = [&](int ncols, int nt, int nseg) {
    Phase1 ph;
    ph.nitems = nt * nseg;
    int r = 0;
#pragma unroll
    for (int i = 0; i < MAXIT; ++i) {
      const int rows = (i < ph.nitems) ? ((nseg > 1) ? ncols : split_rows(ncols, nt, i)) : 0;
      ph.off[i] = r; ph.nrows[i] = rows; ph.seg[i] = (nseg > 1) ? i : 0;
      r += rows;
    }
    ph.total = r;
    return ph;
  };
  if (tid == 0) {
    sm.pht[0] = make_phase(nq, sc.ntq, 1);
    sm.pht[1] = make_phase(no, 1, 1);
    sm.pht[2] = make_phase(nf, sc.ntf, 1);
    sm.pht[3] = make_phase(no, 1, NSEG);
    sm.pht[4] = make_phase(nh, sc.nth, 1);
  }
  __syncthreads();
  const Phase1 &ph_q = sm.pht[0], &ph_o = sm.pht[1], &ph_f = sm.pht[2], &ph_p = sm.pht[3], &ph_h = sm.pht[4];

  // ---- the weight stream: the last thread issues every phase that fits, at the start and whenever rows are released ----
  const bool is_prod = (tid == NCT - 1);
  const uint64_t pol = ptx::policy_evict_first();
  const __nv_bfloat16* wbase = p.wstream1 + (size_t)p.stream_off1[cta] * D;
  const int pps = sc.phases_per_step();
  unsigned tix = 0, cons_tile = 0, bar_target = 0;
  int fill = 0, wpos = 0, pstep = 0, pidx = 0, cons_row = 0;
  size_t uoff = 0;
  // A phase is issued in instalments when only part of it fits (>= MINPART rows): the ring (62 rows at model_dim 1280) is
  // smaller than FC + PROJ of one CTA (66-71 rows), and a PROJ requested only after FC had been consumed arrived late.
  // Pacing: one call issues at most `cap` rows.  Round-2 timeline: with every freed row refilled at once, the grid barriers
  // that followed a big release (FC: 3.9 us, PROJ: 3.3 us, QKV: 2.5 us) cost two to three times the barrier after the
  // attention phase (1.0-1.3 us, no refill in flight) although all CTAs arrived within 0.3 us — every CTA x up to 150 KB of
  // bulk copies queue in front of the barrier's atomics and polls.  Smaller instalments at more points of the layer keep
  // the ring ahead of the consumption (~4.4 rows / us) without such bursts.
  constexpr int MINPART = 4;
  const int cap = ((p.dbg >> 8) & 0xff) ? ((p.dbg >> 8) & 0xff) : 6;
  int part = 0;                       // rows of phase pidx already issued
  auto issue_fitting = [&](int budget = 0) {
    if (!is_prod) return;
    if (budget <= 0) budget = cap;
    while (pstep < p.nsteps && tix - cons_tile < (unsigned)NBAR && budget > 0) {
      const int n = sc.rows(pidx) - part;
      const int avail = min(R - fill, budget);
      const bool last = avail >= n;
      const int m = last ? n : avail;
      if (!last && m < MINPART) break;
      uint64_t* bar = &sm.full[tix % NBAR];
      if (last) ptx::mbar_arrive_expect_tx(bar, (uint32_t)m * D * 2);
      else ptx::mbar_expect_tx(bar, (uint32_t)m * D * 2);
      const int n1 = min(m, R - wpos);
      ptx::bulk_g2s(sm.ring + (size_t)wpos * D, wbase + uoff * D, (uint32_t)n1 * D * 2, bar, pol);
      if (n1 < m) ptx::bulk_g2s(sm.ring, wbase + (uoff + n1) * D, (uint32_t)(m - n1) * D * 2, bar, pol);
      wpos += m;
      if (wpos >= R) wpos -= R;
      fill += m;
      uoff += m;
      budget -= m;
      if (!last) { part += m; break; }
      part = 0;
      ++tix;
      if (++pidx == pps) { pidx = 0; uoff = 0; ++pstep; }
    }
  };
  // called right after the phase's MMAs (which end with a CTA barrier: every warp is done with the rows)
  auto advance = [&](const Phase1& ph) {
    const int tot = ph.total;
    cons_row += tot;
    if (cons_row >= R) cons_row -= R;
    ++cons_tile;
    fill -= tot;
    issue_fitting(tix == cons_tile ? max(cap, sc.rows(pidx) - part) : cap);      // the phase consumed next is not complete yet: all of it, now
  };
  int pi = 0;
  int step = 0;
#define FINE8(n) do { if (p.prof2 && tid == 0 && step == p.nsteps - 1 && l == p.prof2_layer) p.prof2[(size_t)cta * 64 + (n)] = gtimer(); } while (0)
  auto gsync = [&]() {
    PROF_STAMP();
    grid_sync(p.barrier, bar_target, G, 1);
    PROF_STAMP();
    issue_fitting();
  };
  auto prefetch_ln = [&](int buf, const float* w, const float* bb) {
    float* dst = sm.lnp + (size_t)buf * 2 * D;
    const int n4 = D / 4;
    for (int i = tid; i < 2 * n4; i += NCT) {
      const int which = i / n4, off = (i % n4) * 4;
      cp_async16(dst + which * D + off, (which ? bb : w) + off);
    }
  };
  const float* lnA = sm.lnp;
  const float* lnB = sm.lnp + 2 * D;
  const int rr = p.round_bf16;
  // LayerNorm of sequence row `warp` (one warp per row) into the swizzled bf16 rows; emb: build the row from the embedding
  // tables (first layer of a step) instead of the residual stream; w2: the head's second LayerNorm.  Lane owns the elements
  // 4 lane + 128 j .. + 3: 16-byte loads of the row and of the parameters, 8-byte stores (the scalar version spent 1.5-1.7 us
  // of a 3.2-3.7 us phase here).
  constexpr int NV = D / 128;
  auto ln_stats = [&](const float4 (&v)[NV], float& mean, float& rstd) {
    constexpr float invD = 1.0f / (float)D;
    float sacc = 0.f;
#pragma unroll
    for (int j = 0; j < NV; ++j) sacc += (v[j].x + v[j].y) + (v[j].z + v[j].w);
    mean = warp_sum(sacc) * invD;
    float qacc = 0.f;
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      const float d0 = v[j].x - mean, d1 = v[j].y - mean, d2 = v[j].z - mean, d3 = v[j].w - mean;
      qacc += (d0 * d0 + d1 * d1) + (d2 * d2 + d3 * d3);
    }
    rstd = rsqrtf(warp_sum(qacc) * invD + 1e-5f);
  };
  auto ln_apply = [&](float4 (&v)[NV], float mean, float rstd, const float* w, const float* bb) {
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      const float4 ww = *(const float4*)(w + 4 * lane + 128 * j), b4 = *(const float4*)(bb + 4 * lane + 128 * j);
      v[j].x = (v[j].x - mean) * rstd * ww.x + b4.x;
      v[j].y = (v[j].y - mean) * rstd * ww.y + b4.y;
      v[j].z = (v[j].z - mean) * rstd * ww.z + b4.z;
      v[j].w = (v[j].w - mean) * rstd * ww.w + b4.w;
    }
  };
  auto ln_rows = [&](bool emb, int k, const float* w1, const float* b1, const float* w2, const float* b2) {
    float4 v[NV];
    if (warp < B) {
      if (emb) {
        const float4* er = (const float4*)(p.mel_emb + (size_t)s_tok[warp] * D) + lane;
        const float4* pr = (const float4*)(p.mel_pos + (size_t)mel_row(row_k(warp, k)) * D) + lane;
#pragma unroll
        for (int j = 0; j < NV; ++j) {
          const float4 a4 = __ldg(er + 32 * j), c4 = __ldg(pr + 32 * j);
          v[j] = make_float4(rnd(a4.x + c4.x, rr), rnd(a4.y + c4.y, rr), rnd(a4.z + c4.z, rr), rnd(a4.w + c4.w, rr));
        }
      } else {
        const float4* xr = (const float4*)(p.xg + (size_t)warp * D) + lane;
#pragma unroll
        for (int j = 0; j < NV; ++j) v[j] = __ldcg(xr + 32 * j);
      }
      float mean, rstd;
      ln_stats(v, mean, rstd);
      ln_apply(v, mean, rstd, w1, b1);
      if (w2) {
        ln_stats(v, mean, rstd);
        ln_apply(v, mean, rstd, w2, b2);
      }
    } else {
#pragma unroll
      for (int j = 0; j < NV; ++j) v[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __nv_bfloat16* xrow = sm.xs + (size_t)warp * D;
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      const int k = 4 * lane + 128 * j;
      __nv_bfloat162 lo = __floats2bfloat162_rn(v[j].x, v[j].y), hi = __floats2bfloat162_rn(v[j].z, v[j].w);
      *(uint2*)(xrow + ((((k >> 3) ^ (warp & 7)) << 3) | (k & 7))) = make_uint2(*(uint32_t*)&lo, *(uint32_t*)&hi);
    }
  };

  issue_fitting(R);
  prefetch_ln(0, p.ln1_w, p.ln1_b);
  bool alldone = true;
  for (int b = 0; b < B; ++b) alldone &= (s_fin[b] != 0);
  __nv_bfloat16* ob = (__nv_bfloat16*)p.part;      // [8][D] attention output, bf16 in fragment order (`part` is free in this kernel)

  for (; step < p.nsteps && !alldone; ++step) {
    const int k = p.step0 + step;                // the group's step; row b is at its own step row_k(b, k)
    PROF_STAMP();
    // this CTA's slice of the residual stream of the 8 input rows
    for (int idx = tid; idx < B8 * no; idx += NCT) {
      const int b = idx / no, cl = idx % no;
      float v = 0.f;
      if (b < B)
        v = rnd(__ldg(p.mel_emb + (size_t)s_tok[b] * D + o0 + cl) + __ldg(p.mel_pos + (size_t)mel_row(row_k(b, k)) * D + o0 + cl),
                rr);
      sm.xres[b * p.ocap + cl] = v;
    }
    PROF_STAMP();
    PROF_STAMP();

    for (int l = 0; l < L; ++l) {
      const long long pslot = probe_slot(p, k, l);
      float* const prb = (pslot >= 0) ? p.probe + pslot * p.probe_seqs * 2 * D : nullptr;   // [B][2][D]: q | attention output
      // ---------------- P1: LN1 -> QKV ----------------
      FINE8(0);
      cp_async_wait_all();
      ptx::named_bar_sync(1, NCT);                 // LN1 parameters (buffer A) visible
      ln_rows(l == 0, k, lnA, lnA + D, nullptr, nullptr);
      ptx::named_bar_sync(1, NCT);
      issue_fitting();
      FINE8(1);
      ptx::mbar_wait(&sm.full[cons_tile % NBAR], (cons_tile / NBAR) & 1u);
      FINE8(2);
      mma8_smem<D>(sm, ph_q, cons_row, cons_tile, R, warp, lane);
      FINE8(3);
      advance(ph_q);
      for (int idx = tid; idx < nq * B8; idx += NCT) {
        const int cl = idx / B8, b = idx % B8;
        if (b >= B) continue;
        int j = 0;
        while (j + 1 < sc.ntq && cl >= split_begin(nq, sc.ntq, j + 1)) ++j;
        const float v = rnd(red8_sum(sm.red, j, cl - split_begin(nq, sc.ntq, j), b) + sm.bias_s[l * bstride + cl], rr);
        const int c = q0 + cl;
        if (c < D) {
          p.qg[(size_t)b * D + c] = v;
          if (prb) prb[(size_t)b * 2 * D + c] = v;
        } else {
          const size_t base = (((size_t)l * p.nseq + b) * p.maxpos + (s_plen[b] + row_k(b, k))) * D;
          const __nv_bfloat16 kvb = __float2bfloat16_rn(v);
          if (c < 2 * D) p.kc[base + (c - D)] = kvb;
          else p.vc[base + (c - 2 * D)] = kvb;
        }
      }
      FINE8(4);
      gsync();

      // ---------------- P2: attention: (sequence, head pair) = CTA, one head per group of four warps ----------------
      FINE8(5);
      if (cta < B * (H / 2)) {
        const int b = cta / (H / 2), h = 2 * (cta % (H / 2)) + (warp >> 2);
        const int w4 = warp & 3;
        const int ctx = s_plen[b] + row_k(b, k) + 1;
        const int g4 = lane >> 3, sub = lane & 7;
        const size_t cbase = ((size_t)l * p.nseq + b) * p.maxpos;
        const size_t coff = (size_t)h * HD + sub * 8;
        // K/V rows travel through shared memory with cp.async, DEP iterations (of 16 keys per head) deep per warp, in the
        // space of xs | red | lnp (dead in this phase).  Register prefetch did not scale: 4 or 12 iterations of __ldcg in
        // flight ran at one memory round trip per 4 iterations either way (10.6 / 11.6 us per layer at 580 keys — the loads
        // share the warp's six scoreboards with the shuffles and MUFUs of the loop), and the cache of 8 sequences does not
        // fit in L2.  Every lane copies and reads back only its own 16-byte slots: no barrier inside the loop.
        constexpr int STG_BYTES = B8 * D * 2 + RED8_FLOATS * 4 + 4 * D * 4;
        constexpr int DEP = STG_BYTES / (NCW * 1024), GP = 2, STRIDE = 16;      // 4 warps x 4 key groups per iteration
        static_assert(DEP > GP, "K/V staging too small");
        const int jbase = w4 * 4 + g4;
        uint4* stg = (uint4*)sm.xs + (size_t)warp * (DEP * 64) + lane;       // stage: [K: 32 lanes][V: 32 lanes] x 16 bytes
        const __nv_bfloat16* kp = p.kc + cbase * D + coff;
        const __nv_bfloat16* vp = p.vc + cbase * D + coff;
        int st_w = 0;                                                           // stage the next copy lands in
        auto issue = [&](int it) {
          const int j = jbase + STRIDE * it;
          const bool valid = j < ctx;
          const size_t off = (size_t)(valid ? j : 0) * D;
          cp_async16_zfill(stg + st_w * 64, kp + off, valid);
          cp_async16_zfill(stg + st_w * 64 + 32, vp + off, valid);
          cp_async_commit();
          st_w = (st_w + 1 == DEP) ? 0 : st_w + 1;
        };
#pragma unroll
        for (int it = 0; it < DEP; ++it) issue(it);
        float qv[8];
        {
          const float4* qp = (const float4*)(p.qg + (size_t)b * D + h * HD + sub * 8);
          const float4 qa = __ldcg(qp), qb = __ldcg(qp + 1);
          qv[0] = qa.x; qv[1] = qa.y; qv[2] = qa.z; qv[3] = qa.w;
          qv[4] = qb.x; qv[5] = qb.y; qv[6] = qb.z; qv[7] = qb.w;
        }
        float m = -INFINITY, lsum = 0.f, ov[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) ov[i] = 0.f;
        const int span = ctx - w4 * 4;
        const int niter = span > 0 ? (span + STRIDE - 1) / STRIDE : 0;        // warp-uniform
        int st_r = 0;
        for (int it0 = 0; it0 < niter; it0 += GP) {
          cp_async_wait_group<DEP - GP>();
          // GP keys per lane group at once: independent dot products and shuffles, ONE rescale of the running state
          float s[GP];
          uint4 vv[GP];
#pragma unroll
          for (int u = 0; u < GP; ++u) {
            const int j = jbase + STRIDE * (it0 + u);
            const uint4 kk = stg[st_r * 64];
            vv[u] = stg[st_r * 64 + 32];
            st_r = (st_r + 1 == DEP) ? 0 : st_r + 1;
            float d = qv[0] * lo_bf(kk.x) + qv[1] * hi_bf(kk.x) + qv[2] * lo_bf(kk.y) + qv[3] * hi_bf(kk.y) +
                      qv[4] * lo_bf(kk.z) + qv[5] * hi_bf(kk.z) + qv[6] * lo_bf(kk.w) + qv[7] * hi_bf(kk.w);
            d += __shfl_xor_sync(0xffffffffu, d, 1);
            d += __shfl_xor_sync(0xffffffffu, d, 2);
            d += __shfl_xor_sync(0xffffffffu, d, 4);
            s[u] = (j < ctx) ? d * 0.125f : -INFINITY;
          }
          float mn = m;
#pragma unroll
          for (int u = 0; u < GP; ++u) mn = fmaxf(mn, s[u]);
          if (mn > -INFINITY) {
            const float corr = __expf(m - mn);              // m = -inf (first keys): 0
            float pr[GP], ps = 0.f;
#pragma unroll
            for (int u = 0; u < GP; ++u) { pr[u] = __expf(s[u] - mn); ps += pr[u]; }
            lsum = lsum * corr + ps;
#pragma unroll
            for (int i = 0; i < 8; ++i) ov[i] *= corr;
#pragma unroll
            for (int u = 0; u < GP; ++u) {
              const float vf[8] = {lo_bf(vv[u].x), hi_bf(vv[u].x), lo_bf(vv[u].y), hi_bf(vv[u].y),
                                   lo_bf(vv[u].z), hi_bf(vv[u].z), lo_bf(vv[u].w), hi_bf(vv[u].w)};
#pragma unroll
              for (int i = 0; i < 8; ++i) ov[i] += pr[u] * vf[i];
            }
            m = mn;
          }
          // refill the stages just read (their values are in registers: the accumulations above depend on them)
#pragma unroll
          for (int u = 0; u < GP; ++u) issue(it0 + DEP + u);
        }
        cp_async_wait_all();
        __syncwarp();
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
        if (lane < 8) {
          float* rw = sm.att + warp * PART_STRIDE;
          if (lane == 0) { rw[0] = m; rw[1] = lsum; }
#pragma unroll
          for (int i = 0; i < 8; ++i) rw[2 + lane * 8 + i] = ov[i];
        }
        ptx::named_bar_sync(1, NCT);
        if (tid < 2 * HD) {
          // 64 threads per head merge its four warps and write the normalised output (bf16: the operand it becomes)
          const int hg = tid >> 6, d = tid & 63;
          const float* base = sm.att + hg * 4 * PART_STRIDE;
          float mm = -INFINITY;
#pragma unroll
          for (int w = 0; w < 4; ++w) mm = fmaxf(mm, base[w * PART_STRIDE]);
          float lt = 0.f, oa = 0.f;
#pragma unroll
          for (int w = 0; w < 4; ++w) {
            const float mw = base[w * PART_STRIDE];
            const float c = (mw == -INFINITY) ? 0.f : __expf(mw - mm);
            lt += base[w * PART_STRIDE + 1] * c;
            oa += base[w * PART_STRIDE + 2 + d] * c;
          }
          const int hh = 2 * (cta % (H / 2)) + hg;
          const float o = oa * ((lt > 0.f) ? 1.0f / lt : 0.f);
          ob[(size_t)b * D + frag_idx(hh * HD + d)] = __float2bfloat16_rn(o);
          if (prb) prb[((size_t)b * 2 + 1) * D + hh * HD + d] = o;
        }
      }
      issue_fitting();
      FINE8(6);
      gsync();

      // ---------------- P3: O-proj + residual ----------------
      {
        FINE8(7);
        uint4 bo[1][KS / 2];
        const uint4* src = (const uint4*)(ob + (size_t)(lane >> 2) * D) + (warp * KS / 2) * 4 + (lane & 3);
#pragma unroll
        for (int j = 0; j < KS / 2; ++j) bo[0][j] = __ldcg(src + j * 4);
        ptx::mbar_wait(&sm.full[cons_tile % NBAR], (cons_tile / NBAR) & 1u);
        FINE8(8);
        mma8_n<D, 1, true>(sm, ph_o, cons_row, cons_tile, R, warp, lane, bo);
        FINE8(9);
        advance(ph_o);
        for (int idx = tid; idx < no * B8; idx += NCT) {
          const int cl = idx / B8, b = idx % B8;
          if (b >= B) continue;
          const float o = rnd(red8_sum(sm.red, 0, cl, b) + sm.bias_s[l * bstride + nq + cl], rr);
          const float xn = sm.xres[b * p.ocap + cl] + o;
          sm.xres[b * p.ocap + cl] = xn;
          p.xg[(size_t)b * D + o0 + cl] = xn;
        }
      }
      // LayerNorm parameters: LN2 of this layer (P4) and LN1 of the next (both buffers are dead during the attention phase,
      // which stages K/V over them)
      prefetch_ln(1, p.ln2_w + (size_t)l * D, p.ln2_b + (size_t)l * D);
      if (l + 1 < L) prefetch_ln(0, p.ln1_w + (size_t)(l + 1) * D, p.ln1_b + (size_t)(l + 1) * D);
      else prefetch_ln(0, p.lnf_w, p.lnf_b);
      FINE8(10);
      gsync();

      // ---------------- P4: LN2 -> FC + gelu_new ----------------
      FINE8(11);
      ln_rows(false, 0, lnB, lnB + D, nullptr, nullptr);
      ptx::named_bar_sync(1, NCT);
      issue_fitting();
      FINE8(12);
      ptx::mbar_wait(&sm.full[cons_tile % NBAR], (cons_tile / NBAR) & 1u);
      FINE8(13);
      mma8_smem<D>(sm, ph_f, cons_row, cons_tile, R, warp, lane);
      FINE8(14);
      advance(ph_f);
      {
        // outputs tid and tid + 256 (nf <= 2 x 32 columns) computed together: the two gelu chains overlap
        float fv[2];
        int fdst[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int idx = tid + u * NCT;
          const int cl = min(idx / B8, nf - 1), b = idx % B8;
          int j = 0;
          while (j + 1 < sc.ntf && cl >= split_begin(nf, sc.ntf, j + 1)) ++j;
          fv[u] = rnd(red8_sum(sm.red, j, cl - split_begin(nf, sc.ntf, j), b) + sm.bias_s[l * bstride + nq + no + cl], rr);
          const int c = f0 + cl;
          fdst[u] = (idx < nf * B8 && b < B) ? (b * FF + (c / D) * D + frag_idx(c % D)) : -1;
        }
        const float g0 = gelu_new(fv[0], rr), g1 = gelu_new(fv[1], rr);
        if (fdst[0] >= 0) p.fg[fdst[0]] = __float2bfloat16_rn(g0);
        if (fdst[1] >= 0) p.fg[fdst[1]] = __float2bfloat16_rn(g1);
      }
      if (l + 1 == L) prefetch_ln(1, p.fn_w, p.fn_b);
      FINE8(15);
      gsync();

      // ---------------- P5: PROJ + residual ----------------
      {
        uint4 bf[NSEG][KS / 2];
        const uint4* src = (const uint4*)(p.fg + (size_t)(lane >> 2) * FF) + (warp * KS / 2) * 4 + (lane & 3);
#pragma unroll
        for (int s = 0; s < NSEG; ++s)
#pragma unroll
          for (int j = 0; j < KS / 2; ++j) bf[s][j] = __ldcg(src + s * (D / 8) + j * 4);
        FINE8(16);
        ptx::mbar_wait(&sm.full[cons_tile % NBAR], (cons_tile / NBAR) & 1u);
        FINE8(17);
        mma8_n<D, NSEG, true>(sm, ph_p, cons_row, cons_tile, R, warp, lane, bf);
        FINE8(18);
        advance(ph_p);
        for (int idx = tid; idx < no * B8; idx += NCT) {
          const int cl = idx / B8, b = idx % B8;
          if (b >= B) continue;
          float a = 0.f;
#pragma unroll
          for (int s = 0; s < NSEG; ++s) a += red8_sum(sm.red, s, cl, b);
          const float o = rnd(a + sm.bias_s[l * bstride + nq + no + nf + cl], rr);
          const float xn = sm.xres[b * p.ocap + cl] + o;
          sm.xres[b * p.ocap + cl] = xn;
          p.xg[(size_t)b * D + o0 + cl] = xn;
        }
      }
      FINE8(19);
      gsync();
      FINE8(20);
    }

    // ---------------- head: ln_f -> final_norm -> mel_head ----------------
    ln_rows(false, 0, lnA, lnA + D, lnB, lnB + D);
    ptx::named_bar_sync(1, NCT);
    prefetch_ln(0, p.ln1_w, p.ln1_b);          // layer 0 of the next step (drained by the barriers below)
    mma8_smem<D>(sm, ph_h, cons_row, cons_tile, R, warp, lane);
    advance(ph_h);
    for (int idx = tid; idx < nh * B8; idx += NCT) {
      const int cl = idx / B8, b = idx % B8;
      if (b >= B) continue;
      int j = 0;
      while (j + 1 < sc.nth && cl >= split_begin(nh, sc.nth, j + 1)) ++j;
      const float lg = rnd(red8_sum(sm.red, j, cl - split_begin(nh, sc.nth, j), b) + sm.bias_s[L * bstride + cl], rr);
      p.logits[(size_t)b * V + h0 + cl] = lg;
      if (p.logits_dump) p.logits_dump[((size_t)b * p.max_new + row_k(b, k)) * V + h0 + cl] = lg;
    }
    gsync();

    // ---------------- sampling: CTA b decides for sequence b ----------------
    if (cta < B) {
      const int b = cta, kb = row_k(b, k);
      SampleArgs sa = sample_args(p, s_fin[b]);
      sa.seq_base = 0;                          // the Philox counter is (kb, row_seqidx[b])
      const int tk = pick_token(sa, sm.red, sm.seen_s, p.logits + (size_t)b * V, kb, s_seq[b]);
      if (tid == 0 && !s_fin[b]) {
        p.codes[(size_t)b * p.max_new + kb] = tk;
        p.nout[b] = kb + 1;
        int feed = tk;
        int fin = 0;
        if (p.forced) feed = p.forced[(size_t)b * p.max_new + kb];
        else if (tk == p.stop_tok) fin = 1;
        if (kb + 1 >= p.max_new) fin = 1;
        p.tok[b] = feed;
        if (fin) p.finished[b] = 1;
        sm.seen_s[feed >> 5] |= 1u << (feed & 31);
        p.seen[(size_t)b * wv + (feed >> 5)] |= 1u << (feed & 31);
      }
    }
    gsync();
    if (tid < B8) {
      s_tok[tid] = (tid < B) ? __ldcg(p.tok + tid) : 0;
      s_fin[tid] = (tid < B) ? __ldcg(p.finished + tid) : 1;
    }
    ptx::named_bar_sync(1, NCT);
    alldone = true;
    for (int b = 0; b < B; ++b) alldone &= (s_fin[b] != 0);
    if (alldone && cta == 0 && tid == 0) *p.done = 1;
  }
  // drain: bulk copies issued beyond what was consumed must land before the CTA exits
  if (is_prod) {
    if (part > 0) { ptx::mbar_arrive(&sm.full[tix % NBAR]); ++tix; }     // a partly issued phase: close it so that its bytes can be waited for
    for (unsigned n = cons_tile; n < tix; ++n) ptx::mbar_wait(&sm.full[n % NBAR], (n / NBAR) & 1u);
  }
  __syncthreads();
}
