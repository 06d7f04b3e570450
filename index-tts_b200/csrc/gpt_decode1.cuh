// gpt_decode1.cuh — second-generation batch-1 decode kernel (round 2).  Included by gpt_decode.cu inside its
// anonymous namespace: it reuses GptParams, the tagged-word helpers, ln_block, gelu_new and the Philox sampler.
//
// What it replaces: the <1, NPL> instantiation of gpt_fused_kernel for `nreq == 1, num_beams == 1` decode (the
// BASELINE config-2 hot loop).  Same arithmetic, same rounding points, same sampler contract, same KV-cache layout;
// prefill, multi-row decode and beam search stay on gpt_fused_kernel<8, NPL>.
//
// Why: the per-CTA timeline of round 1 (profiles/r02_gpt_fine_timeline_before.txt; 26 us per layer against 6 us of
// pure weight streaming) showed where the time of a layer went:
//   * 6.9 us in the GEMV MMAs: one dependent ldmatrix -> mma chain per 8-row chunk, chunks processed one after
//     the other, and the 9th column of the 1280-wide phases costing a whole second chain
//       -> here a tile is 16 REAL weight rows (m16n8k16 with all 16 A rows used), every tile of a phase is in flight
//          at once (<= 4 independent accumulators per warp, k-steps outermost), so a phase costs KS dependent MMAs;
//   * 2.2 us in the O-proj merge of the 7 key-splits per head (flag poll -> data loads: two L2 round trips)
//       -> contexts up to 640 positions use ONE CTA per head which hands over the normalised head output as tagged
//          words (one round trip, same protocol as the residual stream); longer contexts split the keys and
//          hand over tagged (m, l, o) partials;
//   * 1.0 us in the serial cross-warp merge of the attention partials  -> merged by 64 threads in parallel;
//   * K/V loads only issued after q had arrived  -> first iterations preloaded before the q poll;
//   * 1.0-1.5 us waiting for weights in PROJ: a ring stage held ONE chunk (a 1-row chunk wasted 17.5 KB)
//       -> the ring is row-granular (R rows of D bf16), tiles are mbarrier-tracked independently of the rows;
//   * 22 us per step in embedding / head / sampling with four grid barriers
//       -> no grid barrier at all: every CTA reduces the per-CTA argmax candidates (tagged words) itself, so
//          every CTA knows the next token and builds the next input row locally; sampling (do_sample) keeps a
//          CTA-0 sampler fed by release/acquire flags.
//
// Shared-memory ring protocol.  The CTA's weights of one decode step are a fixed sequence of PHASES
// (per layer: QKV, O-proj, FC, PROJ; then the head), each a run of consecutive stream rows (its MMA tiles back to back).
// Phase g lands in ring rows [row(g) mod R ...) with ONE bulk copy (two when it wraps) and completes full[g mod NBAR];
// There is no producer warp and no "empty" barrier: a phase is free again once all 8 warps have passed the CTA barrier that
// ends its MMAs, and right there ONE thread (the last one, never an epilogue thread) issues every following phase that
// now fits (fewer than NBAR outstanding, rows fit behind the consumed ones).  8 warps = 256 threads also lifts the
// register cap from 168 (288 threads are allocated like 384) to 255 per thread.

constexpr int TROWS = 16;       // weight rows per MMA tile
constexpr int NBAR = 8;         // phase barrier slots
constexpr int MAXIT = 4;        // (column tile, K segment) items per phase
constexpr int RED1_MMA = MAXIT * NCW * 16;                 // per-warp partial sums of the phase's tiles
constexpr int RED1_FLOATS = 2 * RED1_MMA + 48 + 64 + NCW * PART_STRIDE;   // the MMA partials are double-buffered by phase parity   // + LayerNorm statistics + head scores + attention merge

__device__ __forceinline__ int split_rows(int n, int nt, int j) { return (n * (j + 1)) / nt - (n * j) / nt; }
__device__ __forceinline__ int split_begin(int n, int nt, int j) { return (n * j) / nt; }

// per-CTA tile schedule of one decode step, in stream order
struct Sched1 {
  int L, nseg, nq, no, nf, nh, ntq, ntf, nth;
  __device__ __forceinline__ int phases_per_step() const { return 4 * L + 1; }
  // stream rows of phase i (0 <= i < phases_per_step): QKV | O | FC | PROJ (nseg K-segments) per layer, then the head
  __device__ __forceinline__ int rows(int i) const {
    if (i >= 4 * L) return nh;
    const int j = i & 3;
    return j == 0 ? nq : (j == 1 ? no : (j == 2 ? nf : no * nseg));
  }
};

// MMA tiles of one phase, precomputed once per CTA: item i = rows [off[i], off[i] + nrows[i]) of the phase, K-segment seg[i]
struct Phase1 {
  int nitems, total, nrows[MAXIT], off[MAXIT], seg[MAXIT];
};

struct Smem1 {
  __nv_bfloat16* ring;  // [R][D]
  __nv_bfloat16* xs;    // [FF] GEMV input row (bf16, plain layout)
  float* red;           // [2][RED1_MMA] K-split partial sums, by phase parity: phase n + 1 may write while the epilogue of phase n reads
  float* red_ln;        // [48] LayerNorm statistics (two sets)
  float* cs;            // [64] processed scores of this CTA's head columns
  float* red_att;       // [NCW][66] attention merge / sampler scratch
  uint64_t* full;       // [NBAR]
  Phase1* pht;          // [5] MMA tiles of the QKV / O / FC / PROJ / head phases
  float* bias_s;
  float* xres;          // [ocap] this CTA's slice of the fp32 residual stream
  unsigned* seen_s;     // [(V+31)/32]
  float* lnp;           // [2][2][D]
};

// All MMAs of one phase: its tiles in flight together, k-steps outermost, A fragments of k-step ks + 1 loaded (ldmatrix)
// before the MMAs of k-step ks are issued — with the asm statements volatile the compiler keeps this order, so every
// HMMA waits only for an LDSM issued a whole k-step earlier.  (Round-2 measurement: with LDSM -> HMMA back to back into
// one register set the loop cost 55-100 cycles per pair, 100 us of a 505 us step.)
// Phase rows start at ring row `row0` (< R); leaves the per-warp partial sums in red[(i * NCW + warp) * 16 + row] and
// synchronises the compute warps.
// NIT (the number of tiles) is a template parameter: with a run-time bound the compiler kept the fragment arrays in local
// memory (an STL after every LDSM, an LDL before every HMMA: 5400 cycles for a two-tile phase instead of ~500).
template <int D, int NIT>
__device__ __forceinline__ void mma_items_n(const Smem1& sm, float* red, const Phase1& ph, int row0, unsigned phase_idx, int R, int warp, int lane,
                                            long long* st, int dbg) {
  constexpr int KS = (D / 16) / NCW;
  const uint32_t ring_base = ptx::smem_u32(sm.ring);
  const int g = lane >> 2, t4 = lane & 3;
  const int lrow = (lane & 7) + ((lane >> 3) & 1) * 8, khalf = lane >> 4;
  uint32_t a_base[NIT];
  int key[NIT], sgo[NIT];
  float acc[NIT][4];
#pragma unroll
  for (int i = 0; i < NIT; ++i) {
    acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
    const int rr = min(lrow, max(ph.nrows[i] - 1, 0));     // rows beyond the tile read a valid row; their results are unused
    int slot = row0 + ph.off[i] + rr;
    if (slot >= R) slot -= R;
    a_base[i] = ring_base + (uint32_t)(slot * (D * 2));
    key[i] = rr & 7;
    sgo[i] = ph.seg[i] * (D / 2);
  }
  ptx::mbar_wait(&sm.full[phase_idx % NBAR], (phase_idx / NBAR) & 1u);
  if (st && threadIdx.x == 0) { st[0] = gtimer(); st[32] = clock64(); }
  const uint32_t* xw = (const uint32_t*)sm.xs;
  if (!(dbg & 1)) {
    uint32_t a[2][NIT][4];
#pragma unroll
    for (int i = 0; i < NIT; ++i)
      ldmatrix_x4(a_base[i] + (uint32_t)(((2 * (warp * KS) + khalf) ^ key[i]) << 4), a[0][i][0], a[0][i][1], a[0][i][2], a[0][i][3]);
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
      const int kk = warp * KS + ks;                        // k-step: k0 = 16 * kk
      if (ks + 1 < KS) {
#pragma unroll
        for (int i = 0; i < NIT; ++i)
          ldmatrix_x4(a_base[i] + (uint32_t)(((2 * (kk + 1) + khalf) ^ key[i]) << 4), a[(ks + 1) & 1][i][0], a[(ks + 1) & 1][i][1],
                        a[(ks + 1) & 1][i][2], a[(ks + 1) & 1][i][3]);
      }
      uint32_t b0[NIT], b1[NIT];
#pragma unroll
      for (int i = 0; i < NIT; ++i)
      {
        const uint32_t* xb = xw + sgo[i] + kk * 8 + t4;      // B: the one activation row in every n column
        b0[i] = xb[0];
        b1[i] = xb[4];
      }
#pragma unroll
      for (int i = 0; i < NIT; ++i)
        mma_bf16_16816(acc[i], a[ks & 1][i][0], a[ks & 1][i][1], a[ks & 1][i][2], a[ks & 1][i][3], b0[i], b1[i]);
    }
  }
  __syncwarp();
  if (st && threadIdx.x == 0) { st[1] = gtimer(); st[33] = clock64(); }
  if (t4 == 0) {
#pragma unroll
    for (int i = 0; i < NIT; ++i)
    {
      red[(i * NCW + warp) * 16 + g] = acc[i][0];
      red[(i * NCW + warp) * 16 + g + 8] = acc[i][2];
    }
  }
  ptx::named_bar_sync(1, NCT);
  if (st && threadIdx.x == 0) { st[2] = gtimer(); st[34] = clock64(); }
}

template <int D>
__device__ __forceinline__ float* mma_items(const Smem1& sm, const Phase1& ph, int row0, unsigned phase_idx, int R, int warp, int lane,
                                          long long* st = nullptr, int dbg = 0) {
  float* red = sm.red + (phase_idx & 1u) * RED1_MMA;
  switch (ph.nitems) {       // CTA-uniform
    case 1: mma_items_n<D, 1>(sm, red, ph, row0, phase_idx, R, warp, lane, st, dbg); break;
    case 2: mma_items_n<D, 2>(sm, red, ph, row0, phase_idx, R, warp, lane, st, dbg); break;
    case 3: mma_items_n<D, 3>(sm, red, ph, row0, phase_idx, R, warp, lane, st, dbg); break;
    default: mma_items_n<D, 4>(sm, red, ph, row0, phase_idx, R, warp, lane, st, dbg); break;
  }
  return red;
}

__device__ __forceinline__ float red_sum(const float* red, int item, int row) {
  float a = 0.f;
#pragma unroll
  for (int w = 0; w < NCW; ++w) a += red[(item * NCW + w) * 16 + row];
  return a;
}

// Hand-over polls.  Round-2 measurement: the LAST producer's words became visible to the pollers 2-3 us after they were
// stored when all 256 threads of all CTAs re-read their whole slice in every round — CTAs x 4 sector reads per 128-byte
// line per round queue at the L2 slice that holds the line, in front of the very stores the pollers wait for.  So a warp
// first spins on ONE word (all lanes the same address = one request per warp per round, the word chosen per (CTA, warp)
// so the spinners spread over the lines) and only then checks its whole slice.
template <int N>
__device__ __forceinline__ void poll_slice(const uint2* base, int first, unsigned epoch, float (&v)[N], int spin_idx, bool nowait) {
  if (!nowait) {
    unsigned spins = 0, tag;
    do {
      asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(tag) : "l"((const unsigned*)(base + spin_idx) + 1) : "memory");
      if (++spins > (1u << 26)) __trap();
    } while (tag != epoch);
  }
  ld_tagged_slice<N>(base, first, epoch, v, nowait);
}

__device__ __forceinline__ uint2 ld_tagged_word(const uint2* p) {
  uint2 v;
  asm volatile("ld.relaxed.gpu.global.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p) : "memory");
  return v;
}

// The sampling phase of gpt_fused_kernel as a function (same processor order, tie rules and Philox contract):
// RepetitionPenalty -> (forbid stop) -> Temperature -> TopK (ties kept) -> TopP -> multinomial.  Called by the 8 compute
// warps of ONE CTA; `red` is >= 32 + 2 * CMAX floats of scratch.  The pick is valid in thread 0.
struct SampleArgs {
  int V, stop_tok, forbid_stop_before, top_k, seq_base;
  float rep_penalty, temperature, top_p;
  unsigned long long seed;
  int* flag;    // set to k + 1 when more than CMAX tokens tie at the top-k boundary; null: the sequence has finished
};
__device__ __noinline__ int sample_block(const SampleArgs p, float* red, const unsigned* seen, const float* lg, int k, int b,
                                         int tid, int lane, int warp) {
  constexpr int VPT = 40;   // ceil(V / 256) for V <= 10240
  const int V = p.V;
  float sv[VPT];
  const float inv_temp = (p.temperature > 0.f) ? 1.0f / p.temperature : 1.0f;
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
      sv[j] = sc * inv_temp;
    }
  }
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
  float best; int besti;
  block_argmax(best, besti);
  float* cv = red + 32;
  int* ci = (int*)(red + 32 + CMAX);
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
  // more than CMAX tokens tie at the k-th score: TopKLogitsWarper would keep them all, so the call is refused
  if (tid == 0 && p.flag && nc == CMAX && best == kth && best > -INFINITY) *p.flag = k + 1;
  ptx::named_bar_sync(1, NCT);
  if (tid == 0) {
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
  return besti;
}

template <int NPL>
__global__ void __launch_bounds__(NCT, 1) gpt_decode1_kernel(const GptParams p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  constexpr int D = NPL * 32, FF = 4 * D, NSEG = FF / D;
  static_assert(NSEG <= MAXIT, "PROJ K-segments must fit the item slots");
  const int G = p.G, L = p.L, H = p.H, V = p.V, R = p.ring_rows;
  const int cta = blockIdx.x;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  Smem1 sm;
  {
    unsigned char* q = smem_raw;
    sm.ring = (__nv_bfloat16*)q;  q += (size_t)R * D * 2;
    sm.xs = (__nv_bfloat16*)q;    q += (size_t)FF * 2;
    sm.red = (float*)q;           q += sizeof(float) * RED1_FLOATS;
    sm.red_ln = sm.red + 2 * RED1_MMA;
    sm.cs = sm.red_ln + 48;
    sm.red_att = sm.cs + 64;
    sm.full = (uint64_t*)q;       q += sizeof(uint64_t) * NBAR;
    sm.pht = (Phase1*)q;          q += 5 * sizeof(Phase1);
    q = (unsigned char*)(((uintptr_t)q + 15) & ~(uintptr_t)15);
    sm.bias_s = (float*)q;        q += sizeof(float) * (size_t)p.bias_cap;
    sm.xres = (float*)q;          q += sizeof(float) * (size_t)p.ocap;
    sm.seen_s = (unsigned*)q;     q += sizeof(unsigned) * (size_t)((V + 31) / 32);
    q = (unsigned char*)(((uintptr_t)q + 15) & ~(uintptr_t)15);
    sm.lnp = (float*)q;
  }
  if (tid == 0) {
    for (int s = 0; s < NBAR; ++s) ptx::mbar_init(&sm.full[s], 1);
    ptx::fence_mbar_init();
  }
  __syncthreads();

  // column slices of this CTA (same ownership as gpt_fused_kernel)
  const int q0 = col_begin(3 * D, cta, G), q1 = col_begin(3 * D, cta + 1, G);
  const int o0 = col_begin(D, cta, G), o1 = col_begin(D, cta + 1, G);
  const int f0 = col_begin(FF, cta, G), f1 = col_begin(FF, cta + 1, G);
  const int h0 = col_begin(V, cta, G), h1 = col_begin(V, cta + 1, G);
  const int nq = q1 - q0, no = o1 - o0, nf = f1 - f0, nh = h1 - h0;
  Sched1 sc;
  sc.L = L; sc.nseg = NSEG; sc.nq = nq; sc.no = no; sc.nf = nf; sc.nh = nh;
  sc.ntq = (nq + TROWS - 1) / TROWS; sc.ntf = (nf + TROWS - 1) / TROWS; sc.nth = (nh + TROWS - 1) / TROWS;
  const int bstride = nq + 2 * no + nf;
  {
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
    for (int i = tid; i < (V + 31) / 32; i += NCT) sm.seen_s[i] = p.seen[i];
  }
  __syncthreads();

  {
    // ---- the weight stream: issued by the last thread at the points where ring rows become free ----
    const bool is_prod = (tid == NCT - 1);
    const uint64_t pol = ptx::policy_evict_first();
    const __nv_bfloat16* wbase = p.wstream1 + (size_t)p.stream_off1[cta] * D;
    const int pps = sc.phases_per_step();
    unsigned tix = 0;                 // phases issued
    int fill = 0, wpos = 0;           // ring rows in flight or resident; ring row the next phase lands at
    int pstep = 0, pidx = 0;          // producer cursor: step, phase inside the step
    size_t uoff = 0;                  // stream row of that phase inside the step's stream
    unsigned cons_tile = 0;           // phases consumed
    int cons_row = 0;                 // ring row of the next phase to consume
    // A phase may be issued in instalments (mbarrier.expect_tx for all but the last, which arrives) and one call issues at
    // most `cap` rows: see gpt_decode8.cuh — bursts of one 60-150 KB bulk copy per CTA copies delay the latency-critical hand-over traffic.
    // Measured over 256 steps (us / step): whole phases only 445.2; instalments, no cap 433.1; cap 24: 432.8; cap 18: 425.5; cap 12: 436.5.
    constexpr int MINPART = 4;
    const int cap = ((p.dbg >> 8) & 0xff) ? ((p.dbg >> 8) & 0xff) : 18;
    int part = 0;                     // rows of phase pidx already issued
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
    const int b = 0;                  // the one sequence
    const int plen = __ldg(p.prompt_len + b);
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
    const int spin_x = warp * (NPL * 4) + (cta * 37 + warp * 13) % (NPL * 4);      // the word this warp spins on (inside its own slice)
    const int spin_f = ((cta * 5 + warp) % NSEG) * D + warp * (D / NCW) + (cta * 41) % (D / NCW);   // same for the gelu(fc) words (inside this warp's slices)
    const int split_at = ((p.dbg >> 16) & 0xff) ? ((p.dbg >> 16) & 0xff) * 32 : 640;     // IDX_GPT_DBG bits 16-23 / 24-30: experiment knobs
    const int split_len = ((p.dbg >> 24) & 0x7f) ? ((p.dbg >> 24) & 0x7f) * 32 : 320;
    const int max_split = min(7, G / H);        // partt holds 7 partials per head
    const bool nowait = (p.dbg & 4) != 0;      // diagnostics only: polls do not wait (results are garbage, timing = no dependencies)
    int feed = __ldcg(p.tok + b);
    const bool already_done = __ldcg(p.finished + b) != 0;
    // phase descriptors: either nt column tiles of one K-segment, or one column tile with nseg K-segments (computed once;
    // no division or modulo on the per-phase path)
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
    // called right after mma_items (which ends with a CTA barrier: every warp is done with the phase's rows)
    auto advance = [&](const Phase1& ph) {
      const int tot = ph.total;
      cons_row += tot;
      if (cons_row >= R) cons_row -= R;
      ++cons_tile;
      fill -= tot;
      if ((p.dbg & 8) || tix == cons_tile) issue_fitting(max(cap, sc.rows(pidx) - part));   // the phase consumed next is not (completely) issued: all of it at once; dbg 8 = always
    };
    // The freed rows are refilled a little later — right after this CTA's NEXT hand-over poll has completed: at the release
    // point all CTAs would start their 60-90 KB bulk copies together, exactly when the epilogue stores and the polls of
    // the hand-over (the latency-critical traffic) are in flight; the ring holds two to three phases, so the weights issued
    // one poll later still arrive long before they are consumed.
    auto refill = [&]() { if (!(p.dbg & 8)) issue_fitting(); };
    issue_fitting(R);                 // initial fill

    for (int step = 0; step < p.nsteps && !already_done; ++step) {
      const int k = p.step0 + step;
      const int posidx = (k == 0 || p.pos_plain) ? k : k + 1;   // P1: mel position k+1 with the KV cache
      const int pos = plen + k;                       // position of this token in the cache
      const int ctx = pos + 1;
      // key splits: one CTA per head up to split_at keys, then ceil(ctx / split_len) CTAs per head, at most
      // min(7, G / H): every (head, split) pair needs a CTA of the grid, or the P3 merge would wait for a partial no CTA computes
      const int nsplit = (ctx <= split_at || max_split < 2) ? 1 : min(max_split, (ctx + split_len - 1) / split_len);
      if (step == 0) prefetch_ln(0, p.ln1_w, p.ln1_b);
      // ---- input row: mel_emb[feed] + mel_pos[posidx], built locally by every CTA (no hand-over) ----
      float v0[NPL / 8];
      {
        const float* er = p.mel_emb + (size_t)feed * D;
        const float* pr = p.mel_pos + (size_t)posidx * D;
#pragma unroll
        for (int j = 0; j < NPL / 8; ++j) {
          const int i = warp * (NPL * 4) + lane + 32 * j;
          v0[j] = rnd(__ldg(er + i) + __ldg(pr + i), rr);
        }
        if (tid < no) sm.xres[tid] = rnd(__ldg(er + o0 + tid) + __ldg(pr + o0 + tid), rr);
      }

      for (int l = 0; l < L; ++l) {
        const unsigned ep_base = p.epoch0 + (unsigned)(step * L + l) * 2u;
        const unsigned ep_oproj = ep_base + 1u, ep_proj = ep_base + 2u;
        const unsigned f_tag = ((ep_base >> 1) % 65535u) + 1u;
        long long* f2 = (p.prof2 && l == p.prof2_layer && step == p.nsteps - 1) ? p.prof2 + (size_t)cta * 64 : nullptr;
#define G2(i) do { if (f2 && tid == 0) { f2[(i)] = gtimer(); f2[32 + (i)] = clock64(); } } while (0)
        const long long pslot = probe_slot(p, k, l);
        float* const prb = (pslot >= 0) ? p.probe + pslot * p.probe_seqs * 2 * D : nullptr;   // q | attention output
        if (prb && cta == 0 && tid == 0) p.probe_ns[pslot] = nsplit;
        G2(0);
        // ---------------- P1: LN1 -> QKV ----------------
        {
          float v[NPL / 8];
          if (l > 0) {
            poll_slice<NPL / 8>(p.xt, warp * (NPL * 4) + lane, ep_base, v, spin_x, nowait);
          } else {
#pragma unroll
            for (int j = 0; j < NPL / 8; ++j) v[j] = v0[j];
            cp_async_wait_all();          // LN1 parameters of layer 0 (prefetched in the previous step / above)
          }
          prefetch_ln(1, p.ln2_w + (size_t)l * D, p.ln2_b + (size_t)l * D);   // for P4 (drained there)
          G2(1);
          refill();
          ln_block<NPL>(v, lnA, lnA + D, sm.red_ln, warp, lane);
          G2(2);
#pragma unroll
          for (int j = 0; j < NPL / 8; ++j) sm.xs[warp * (NPL * 4) + lane + 32 * j] = __float2bfloat16_rn(v[j]);
        }
        // no CTA barrier: a warp's MMAs read exactly the k-slice of xs this warp has just written (k-steps warp*KS ..)
        __syncwarp();
        {
          const float* redp = mma_items<D>(sm, ph_q, cons_row, cons_tile, R, warp, lane, f2 ? f2 + 3 : nullptr, p.dbg);
          advance(ph_q);
          if (tid < nq) {
            const int cl = tid;
            int j = 0;
            while (j + 1 < sc.ntq && cl >= split_begin(nq, sc.ntq, j + 1)) ++j;
            const float a = red_sum(redp, j, cl - split_begin(nq, sc.ntq, j));
            const float v = rnd(a + sm.bias_s[l * bstride + cl], rr);
            const int c = q0 + cl;
            if (c < D) {
              st_tagged(p.qt + c, v, ep_oproj);
              if (prb) prb[c] = v;
            } else {
              const size_t base = (((size_t)l * p.nseq + b) * p.maxpos + pos) * D;
              const __nv_bfloat16 kvb = __float2bfloat16_rn(v);
              if (c < 2 * D) p.kc[base + (c - D)] = kvb;
              else p.vc[base + (c - 2 * D)] = kvb;
              st_tagged(p.kvt + (c - D), __bfloat162float(kvb), ep_oproj);
            }
          }
        }
        G2(6);

        // ---------------- P2: attention over the KV cache: (head, key split) = CTA ----------------
        if (cta < H * nsplit) {
          const int h = cta / nsplit, sp = cta % nsplit;
          const int k0 = (int)(((long long)ctx * sp) / nsplit);
          const int k1 = (int)(((long long)ctx * (sp + 1)) / nsplit);
          const int kend = min(k1, ctx - 1);        // the position being decoded comes from the tagged k, v words
          const int g4 = lane >> 3, sub = lane & 7;
          const size_t cbase = ((size_t)l * p.nseq + b) * p.maxpos;
          const size_t coff = (size_t)h * HD + sub * 8;
          // software pipeline, PF iterations deep (a key costs one L2 round trip: with one iteration in flight the loop
          // ran at ~1200 cycles per 32 keys); the first PF iterations are in flight before q has arrived
          constexpr int PF = 4;
          const int jbase = k0 + warp * 4 + g4;          // key of iteration it: jbase + 32 * it
          uint4 kb[PF], vb[PF];
#pragma unroll
          for (int u = 0; u < PF; ++u) {
            kb[u] = make_uint4(0, 0, 0, 0);
            vb[u] = make_uint4(0, 0, 0, 0);
            const int ju = jbase + NCW * 4 * u;
            if (ju < kend) {
              kb[u] = __ldcg((const uint4*)(p.kc + (cbase + ju) * D + coff));
              vb[u] = __ldcg((const uint4*)(p.vc + (cbase + ju) * D + coff));
            }
          }
          float qv[8];
          {
            const uint2* qp = p.qt + h * HD + sub * 8;
            uint2 w[8];
            unsigned spins = 0;
            bool ok;
            do {
#pragma unroll
              for (int i = 0; i < 8; ++i) w[i] = ld_tagged_word(qp + i);
              ok = true;
#pragma unroll
              for (int i = 0; i < 8; ++i) ok &= (w[i].y == ep_oproj);
              if (++spins > (1u << 26)) __trap();
            } while (!ok && !nowait);
#pragma unroll
            for (int i = 0; i < 8; ++i) qv[i] = __uint_as_float(w[i].x);
          }
          G2(7);
          float m = -INFINITY, lsum = 0.f, ov[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) ov[i] = 0.f;
          const int span = ((p.dbg & 2) ? 0 : kend) - (k0 + warp * 4);
          const int niter = span > 0 ? (span + NCW * 4 - 1) / (NCW * 4) : 0;        // warp-uniform
          for (int it0 = 0; it0 < niter; it0 += PF) {
#pragma unroll
            for (int u = 0; u < PF; ++u) {
              const int it = it0 + u;
              if (it < niter) {
                const int j = jbase + NCW * 4 * it;
                const bool valid = j < kend;
                const uint4 kk = kb[u], vv = vb[u];
                const int jn = j + NCW * 4 * PF;             // refill this slot: in flight for the next PF - 1 iterations
                kb[u] = make_uint4(0, 0, 0, 0);
                vb[u] = make_uint4(0, 0, 0, 0);
                if (jn < kend) {
                  kb[u] = __ldcg((const uint4*)(p.kc + (cbase + jn) * D + coff));
                  vb[u] = __ldcg((const uint4*)(p.vc + (cbase + jn) * D + coff));
                }
                float s = qv[0] * lo_bf(kk.x) + qv[1] * hi_bf(kk.x) + qv[2] * lo_bf(kk.y) + qv[3] * hi_bf(kk.y) +
                          qv[4] * lo_bf(kk.z) + qv[5] * hi_bf(kk.z) + qv[6] * lo_bf(kk.w) + qv[7] * hi_bf(kk.w);
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
            }
          }
          if (k1 == ctx && warp == 0 && g4 == 0) {
            // the new position (owned by the last key split): k and v straight from the QKV epilogue's tagged words
            const uint2* kp = p.kvt + h * HD + sub * 8;
            const uint2* vp = p.kvt + D + h * HD + sub * 8;
            uint2 wk[8], wv[8];
            unsigned spins = 0;
            bool ok;
            do {
#pragma unroll
              for (int i = 0; i < 8; ++i) { wk[i] = ld_tagged_word(kp + i); wv[i] = ld_tagged_word(vp + i); }
              ok = true;
#pragma unroll
              for (int i = 0; i < 8; ++i) ok &= (wk[i].y == ep_oproj) & (wv[i].y == ep_oproj);
              if (++spins > (1u << 26)) __trap();
            } while (!ok && !nowait);
            float s = 0.f;
#pragma unroll
            for (int i = 0; i < 8; ++i) s += qv[i] * __uint_as_float(wk[i].x);
            s += __shfl_xor_sync(0xffu, s, 1);
            s += __shfl_xor_sync(0xffu, s, 2);
            s += __shfl_xor_sync(0xffu, s, 4);
            s *= 0.125f;
            const float mn = fmaxf(m, s);
            const float corr = __expf(m - mn);
            const float pr = __expf(s - mn);
            lsum = lsum * corr + pr;
#pragma unroll
            for (int i = 0; i < 8; ++i) ov[i] = ov[i] * corr + pr * __uint_as_float(wv[i].x);
            m = mn;
          }
          __syncwarp();
          G2(8);
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
          // merge the 8 warps: every warp publishes (m, l, o[64]) in shared memory, 64 threads combine them in parallel
          float* red = sm.red_att;
          if (lane < 8) {
            float* rw = red + warp * PART_STRIDE;
            if (lane == 0) { rw[0] = m; rw[1] = lsum; }
#pragma unroll
            for (int i = 0; i < 8; ++i) rw[2 + lane * 8 + i] = ov[i];
          }
          ptx::named_bar_sync(1, NCT);
          G2(9);
          if (tid < HD) {
            float mm = -INFINITY;
#pragma unroll
            for (int w = 0; w < NCW; ++w) mm = fmaxf(mm, red[w * PART_STRIDE]);
            float lt = 0.f, oa = 0.f;
#pragma unroll
            for (int w = 0; w < NCW; ++w) {
              const float mw = red[w * PART_STRIDE];
              const float c = (mw == -INFINITY) ? 0.f : __expf(mw - mm);
              lt += red[w * PART_STRIDE + 1] * c;
              oa += red[w * PART_STRIDE + 2 + tid] * c;
            }
            if (nsplit == 1) {
              // one CTA saw every key of the head: hand over the normalised output (bf16-rounded like the operand it becomes)
              const float inv = (lt > 0.f) ? 1.0f / lt : 0.f;
              st_tagged(p.ot + h * HD + tid, oa * inv, ep_oproj);
              if (prb) prb[D + h * HD + tid] = oa * inv;
            } else {
              uint2* pw = p.partt + (size_t)cta * PART_STRIDE;
              st_tagged(pw + 2 + tid, oa, ep_oproj);
              if (tid == 0) { st_tagged(pw, mm, ep_oproj); st_tagged(pw + 1, lt, ep_oproj); }
            }
          }
        }
        G2(10);

        // ---------------- P3: attention output -> O-proj + residual ----------------
        if (nsplit == 1) {
          float v[NPL / 8];
          poll_slice<NPL / 8>(p.ot, warp * (NPL * 4) + lane, ep_oproj, v, spin_x, nowait);
          G2(11);
          refill();
#pragma unroll
          for (int j = 0; j < NPL / 8; ++j) sm.xs[warp * (NPL * 4) + lane + 32 * j] = __float2bfloat16_rn(v[j]);
          __syncwarp();          // own k-slice only: no CTA barrier
        } else {
          // one warp per head, all loads of a head (nsplit x (m, l, o[lane], o[lane + 32])) in flight together
          for (int h = warp; h < H; h += NCW) {
            const uint2* pp = p.partt + (size_t)h * nsplit * PART_STRIDE;
            uint2 wm[7], wl[7], wa[7], wb[7];
            unsigned spins = 0;
            bool ok;
            do {
              ok = true;
#pragma unroll
              for (int s = 0; s < 7; ++s)
                if (s < nsplit) {
                  wm[s] = ld_tagged_word(pp + s * PART_STRIDE);
                  wl[s] = ld_tagged_word(pp + s * PART_STRIDE + 1);
                  wa[s] = ld_tagged_word(pp + s * PART_STRIDE + 2 + lane);
                  wb[s] = ld_tagged_word(pp + s * PART_STRIDE + 34 + lane);
                }
#pragma unroll
              for (int s = 0; s < 7; ++s)
                if (s < nsplit) ok &= (wm[s].y == ep_oproj) & (wl[s].y == ep_oproj) & (wa[s].y == ep_oproj) & (wb[s].y == ep_oproj);
              if (++spins > (1u << 26)) __trap();
            } while (!ok && !nowait);
            float mm = -INFINITY;
#pragma unroll
            for (int s = 0; s < 7; ++s)
              if (s < nsplit) mm = fmaxf(mm, __uint_as_float(wm[s].x));
            float lt = 0.f, oa = 0.f, ob = 0.f;
#pragma unroll
            for (int s = 0; s < 7; ++s)
              if (s < nsplit) {
                const float ms = __uint_as_float(wm[s].x);
                const float cc = (ms == -INFINITY) ? 0.f : __expf(ms - mm);
                lt += __uint_as_float(wl[s].x) * cc;
                oa += __uint_as_float(wa[s].x) * cc;
                ob += __uint_as_float(wb[s].x) * cc;
              }
            const float inv = (lt > 0.f) ? 1.0f / lt : 0.f;
            sm.xs[h * HD + lane] = __float2bfloat16_rn(oa * inv);
            sm.xs[h * HD + 32 + lane] = __float2bfloat16_rn(ob * inv);
            if (prb && cta == 0) { prb[D + h * HD + lane] = oa * inv; prb[D + h * HD + 32 + lane] = ob * inv; }
          }
          G2(11);
          refill();
          ptx::named_bar_sync(1, NCT);     // heads are not aligned with the warps' k-slices here
        }
        {
          const float* redp = mma_items<D>(sm, ph_o, cons_row, cons_tile, R, warp, lane, f2 ? f2 + 12 : nullptr, p.dbg);
          advance(ph_o);
          if (tid < no) {
            // the residual stream is fp32 even on the bf16 path (trap P12): only the branch is rounded
            const float o = rnd(red_sum(redp, 0, tid) + sm.bias_s[l * bstride + nq + tid], rr);
            const float xn = sm.xres[tid] + o;
            sm.xres[tid] = xn;
            st_tagged(p.xt + o0 + tid, xn, ep_oproj);
          }
        }
        G2(15);

        // ---------------- P4: LN2 -> FC + gelu_new ----------------
        if (l + 1 < L) prefetch_ln(0, p.ln1_w + (size_t)(l + 1) * D, p.ln1_b + (size_t)(l + 1) * D);
        else prefetch_ln(0, p.lnf_w, p.lnf_b);
        {
          float v[NPL / 8];
          poll_slice<NPL / 8>(p.xt, warp * (NPL * 4) + lane, ep_oproj, v, spin_x, nowait);
          G2(16);
          refill();
          cp_async_wait_all();   // ln_2 parameters prefetched in P1 (ln_block's own CTA barrier publishes them)
          ln_block<NPL>(v, lnB, lnB + D, sm.red_ln, warp, lane);
          G2(17);
#pragma unroll
          for (int j = 0; j < NPL / 8; ++j) sm.xs[warp * (NPL * 4) + lane + 32 * j] = __float2bfloat16_rn(v[j]);
        }
        __syncwarp();
        {
          const float* redp = mma_items<D>(sm, ph_f, cons_row, cons_tile, R, warp, lane, f2 ? f2 + 18 : nullptr, p.dbg);
          advance(ph_f);
          if (tid < nf) {
            const int cl = tid;
            int j = 0;
            while (j + 1 < sc.ntf && cl >= split_begin(nf, sc.ntf, j + 1)) ++j;
            const float a = red_sum(redp, j, cl - split_begin(nf, sc.ntf, j));
            const float f = rnd(a + sm.bias_s[l * bstride + nq + no + cl], rr);
            const __nv_bfloat16 fv = __float2bfloat16_rn(gelu_new(f, rr));
            asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p.ft + f0 + cl),
                         "r"((unsigned)__bfloat16_as_ushort(fv) | (f_tag << 16)) : "memory");
          }
        }
        G2(21);

        // ---------------- P5: proj + residual ----------------
        if (l + 1 == L) prefetch_ln(1, p.fn_w, p.fn_b);   // final_norm for the head
        {
          // every warp polls exactly the gelu(fc) words of ITS k-slices (k-steps warp*KS .. of each of the NSEG segments),
          // repacks them to bf16 in xs and goes straight to its MMAs: no CTA barrier between the hand-over and the MMAs
          constexpr int CW = (D / NCW) / 8;                 // 8-word chunks per warp per K-segment
          constexpr int NCHW = (NSEG * CW + 31) / 32;       // chunks per lane
          uint4 lo[NCHW], hi[NCHW];
          int cidx[NCHW];
#pragma unroll
          for (int q = 0; q < NCHW; ++q) {
            const int i = lane + 32 * q;
            cidx[q] = (i < NSEG * CW) ? (i / CW) * (D / 8) + warp * CW + (i % CW) : -1;
          }
          const unsigned want = f_tag << 16;
          unsigned spins = 0;
          bool ok;
          if (!nowait) {
            unsigned wv;
            do {
              asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(wv) : "l"(p.ft + spin_f) : "memory");
              if (++spins > (1u << 26)) __trap();
            } while ((wv & 0xffff0000u) != want);
          }
          do {
            ok = true;
#pragma unroll
            for (int q = 0; q < NCHW; ++q) {
              if (cidx[q] >= 0) {
                const unsigned* src = p.ft + (size_t)cidx[q] * 8;
                asm volatile("ld.relaxed.gpu.global.v4.u32 {%0, %1, %2, %3}, [%4];"
                             : "=r"(lo[q].x), "=r"(lo[q].y), "=r"(lo[q].z), "=r"(lo[q].w) : "l"(src) : "memory");
                asm volatile("ld.relaxed.gpu.global.v4.u32 {%0, %1, %2, %3}, [%4];"
                             : "=r"(hi[q].x), "=r"(hi[q].y), "=r"(hi[q].z), "=r"(hi[q].w) : "l"(src + 4) : "memory");
              }
            }
#pragma unroll
            for (int q = 0; q < NCHW; ++q) {
              if (cidx[q] >= 0)
                ok &= ((lo[q].x & 0xffff0000u) == want) & ((lo[q].y & 0xffff0000u) == want) &
                      ((lo[q].z & 0xffff0000u) == want) & ((lo[q].w & 0xffff0000u) == want) &
                      ((hi[q].x & 0xffff0000u) == want) & ((hi[q].y & 0xffff0000u) == want) &
                      ((hi[q].z & 0xffff0000u) == want) & ((hi[q].w & 0xffff0000u) == want);
            }
            if (++spins > (1u << 26)) __trap();
          } while (!ok && !nowait);
          G2(22);
          refill();
#pragma unroll
          for (int q = 0; q < NCHW; ++q) {
            if (cidx[q] >= 0)
              ((uint4*)sm.xs)[cidx[q]] = make_uint4((lo[q].x & 0xffffu) | (lo[q].y << 16), (lo[q].z & 0xffffu) | (lo[q].w << 16),
                                                     (hi[q].x & 0xffffu) | (hi[q].y << 16), (hi[q].z & 0xffffu) | (hi[q].w << 16));
          }
          cp_async_wait_all();     // the LayerNorm parameters prefetched in P4 (published by the barrier that ends the MMAs)
        }
        __syncwarp();
        {
          const float* redp = mma_items<D>(sm, ph_p, cons_row, cons_tile, R, warp, lane, f2 ? f2 + 23 : nullptr, p.dbg);
          advance(ph_p);
          if (tid < no) {
            float a = 0.f;
#pragma unroll
            for (int s = 0; s < NSEG; ++s) a += red_sum(redp, s, tid);
            const float o = rnd(a + sm.bias_s[l * bstride + nq + no + nf + tid], rr);
            const float xn = sm.xres[tid] + o;
            sm.xres[tid] = xn;
            st_tagged(p.xt + o0 + tid, xn, ep_proj);
          }
        }
        G2(26);
      }

      // ---------------- head: ln_f -> final_norm -> mel_head ----------------
      const unsigned ep_head = p.epoch0 + (unsigned)(step * L + L - 1) * 2u + 2u;
      {
        float v[NPL / 8];
        poll_slice<NPL / 8>(p.xt, warp * (NPL * 4) + lane, ep_head, v, spin_x, nowait);
        refill();
        ln_block<NPL>(v, lnA, lnA + D, sm.red_ln, warp, lane);
        ln_block<NPL>(v, lnB, lnB + D, sm.red_ln + 3 * NCW, warp, lane);
#pragma unroll
        for (int j = 0; j < NPL / 8; ++j) sm.xs[warp * (NPL * 4) + lane + 32 * j] = __float2bfloat16_rn(v[j]);
      }
      __syncwarp();
      prefetch_ln(0, p.ln1_w, p.ln1_b);      // layer 0 of the next step (buffer A is free: both LNs above are done)
      int token = 0;
      {
        const float* redp = mma_items<D>(sm, ph_h, cons_row, cons_tile, R, warp, lane);
        advance(ph_h);
        float* cs = sm.cs;
        if (tid < nh) {
          const int cl = tid;
          int j = 0;
          while (j + 1 < sc.nth && cl >= split_begin(nh, sc.nth, j + 1)) ++j;
          const float lg = rnd(red_sum(redp, j, cl - split_begin(nh, sc.nth, j)) + sm.bias_s[L * bstride + cl], rr);
          const int i = h0 + cl;
          if (p.logits_dump) p.logits_dump[((size_t)b * p.max_new + k) * V + i] = lg;
          if (p.do_sample) {
            p.logits[(size_t)b * V + i] = lg;
          } else {
            float s = lg;
            if ((sm.seen_s[i >> 5] >> (i & 31)) & 1u) s = (s < 0.f) ? s * p.rep_penalty : s / p.rep_penalty;
            if (i == p.stop_tok && k < p.forbid_stop_before) s = -INFINITY;
            cs[cl] = s;
          }
        }
        ptx::named_bar_sync(1, NCT);
        if (!p.do_sample) {
          // greedy: this CTA's best (score, index), lowest index first among ties -> tagged candidate words;
          // every CTA then reduces all G candidates itself: no hand-over of the token, no barrier
          if (warp == 0) {
            float best = -INFINITY;
            int bi = 0x7fffffff;
            for (int c = lane; c < nh; c += 32) {
              const float s = cs[c];
              if (s > best) { best = s; bi = h0 + c; }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
              const float b2 = __shfl_xor_sync(0xffffffffu, best, o);
              const int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
              if (b2 > best || (b2 == best && i2 < bi)) { best = b2; bi = i2; }
            }
            if (lane == 0) {
              st_tagged(p.cand + 2 * cta, best, ep_head);
              st_tagged(p.cand + 2 * cta + 1, __int_as_float(bi), ep_head);
            }
          }
          float best = -INFINITY;
          int bi = 0x7fffffff;
          if (tid < G) {
            uint2 wv, wi;
            unsigned spins = 0;
            do {
              wv = ld_tagged_word(p.cand + 2 * tid);
              wi = ld_tagged_word(p.cand + 2 * tid + 1);
              if (++spins > (1u << 26)) __trap();
            } while ((wv.y != ep_head || wi.y != ep_head) && !nowait);
            best = __uint_as_float(wv.x);
            bi = (int)wi.x;
          }
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) {
            const float b2 = __shfl_xor_sync(0xffffffffu, best, o);
            const int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
            if (b2 > best || (b2 == best && i2 < bi)) { best = b2; bi = i2; }
          }
          float* rb = sm.red_ln;
          if (lane == 0) { rb[warp * 2] = best; ((int*)rb)[warp * 2 + 1] = bi; }
          ptx::named_bar_sync(1, NCT);
#pragma unroll
          for (int w = 0; w < NCW; ++w) {
            const float b2 = rb[w * 2];
            const int i2 = ((int*)rb)[w * 2 + 1];
            if (w == 0 || b2 > best || (b2 == best && i2 < bi)) { best = b2; bi = i2; }
          }
          token = nowait ? min(max(bi, 0), V - 1) : bi;
        } else {
          // sampling: logits -> global, flag with release; CTA 0 samples and publishes the token as a tagged word
          if (tid == 0) st_release_gpu((unsigned*)(p.cand + 2 * cta) + 1, ep_head);   // cumulative over the CTA (bar.sync above)
          if (cta == 0) {
            if (tid < G) {
              unsigned spins = 0;
              while (ld_relaxed_gpu((const unsigned*)(p.cand + 2 * tid) + 1) != ep_head)
                if (++spins > (1u << 26)) __trap();
            }
            __threadfence();
            ptx::named_bar_sync(1, NCT);
            SampleArgs sa;
            sa.V = V; sa.stop_tok = p.stop_tok; sa.forbid_stop_before = p.forbid_stop_before; sa.top_k = p.top_k;
            sa.seq_base = p.seq_base; sa.rep_penalty = p.rep_penalty; sa.temperature = p.temperature; sa.top_p = p.top_p;
            sa.seed = p.seed; sa.flag = p.flag;
            const int tk = sample_block(sa, sm.red_att, sm.seen_s, p.logits + (size_t)b * V, k, b, tid, lane, warp);
            if (tid == 0) st_tagged(p.tokt, __int_as_float(tk), ep_head);
            token = tk;
          }
          {
            uint2 w;
            unsigned spins = 0;
            do {
              w = ld_tagged_word(p.tokt);
              if (++spins > (1u << 26)) __trap();
            } while (w.y != ep_head);
            token = (int)w.x;
          }
        }
      }
      // ---------------- bookkeeping: every CTA knows the token ----------------
      int nfeed = token;
      if (p.forced) nfeed = __ldg(p.forced + (size_t)b * p.max_new + k);
      const bool fin = (!p.forced && token == p.stop_tok) || (k + 1 >= p.max_new);
      if (tid == 0) {
        sm.seen_s[nfeed >> 5] |= 1u << (nfeed & 31);
        if (cta == 0) {
          p.codes[(size_t)b * p.max_new + k] = token;
          p.nout[b] = k + 1;
          p.tok[b] = nfeed;
          p.seen[nfeed >> 5] |= 1u << (nfeed & 31);
          if (fin) { p.finished[b] = 1; *p.done = 1; }
        }
      }
      feed = nfeed;
      ptx::named_bar_sync(1, NCT);      // seen_s / red are reused by the next step
      if (fin) break;
    }
    // drain: bulk copies issued beyond what was consumed must land before the CTA exits
    if (is_prod) {
      if (part > 0) { ptx::mbar_arrive(&sm.full[tix % NBAR]); ++tix; }     // a partly issued phase: close it so that its bytes can be waited for
      for (unsigned n = cons_tile; n < tix; ++n) ptx::mbar_wait(&sm.full[n % NBAR], (n / NBAR) & 1u);
    }
  }
  __syncthreads();
}
