// ust_kernels.cu — the verification kernel of ApplyState and the auxiliary kernels of libust.so (sm_90a).
//
// ust_verify_kernel runs behind ust_stream_kernel (ust_stream.cu) on the same stream, launched with programmatic
// dependent launch: one small CTA per SM, resident (asleep in griddepcontrol.wait, 4.4 KiB transition table staged)
// while the streaming kernel runs. When that ends every CTA reads the shard's counters - on several GPUs: exchanges
// them through NVLink mailboxes, or takes the result of a host-launched NCCL all-reduce - derives the slot budget
// (GetUpgradesAvailable, common_manager.go:748-776) and judges the speculation the streaming kernel made. CTA 0 writes
// ust_counters. In the common case the speculation held, every output is final, and the kernel returns at once.
// Otherwise the CTAs re-evaluate, exactly, the tiles that need it: tiles before the cut with every upgrade candidate
// granted, tiles behind it with none, the cut tile with the ordered allocation of upgrade_inplace.go:71-109
// (candidate rank in slice order < slots left: warp-shuffle scan + per-step totals), and - when the call aborts -
// every tile with the reference's abort semantics (nodes the sequential passes had not reached stay untouched,
// common_manager.go:462-523).
// Around it: ust_pod_summary_kernel (pod lists -> one byte per node), ust_build_state*_kernel (BuildState),
// ust_patch_kernel / ust_splice_kernel / ust_reorder_kernel / ust_feedback_kernel (delta updates, membership changes,
// new node orders, rollout simulation), ust_pods_scatter_kernel / ust_pods_runs_kernel / ust_pods_relayout_kernel
// (replaced pod lists), ust_pods_reorder_runs_kernel / ust_pods_reorder_kernel (pod lists in a new node order),
// ust_diff_*_kernel (sparse outputs),
// ust_widen_kernel (packed host format).
// The auxiliary kernels share their building blocks, each written once: the BuildState join and counts (build_prologue,
// build_join, build_count, build_count_ds, build_spill, build_finish), the searches over sorted run / segment starts
// (last_le in global memory, last_le_from over a staged slice), the gathers of a new order (gather_runs for node columns,
// gather_pods for a pod-list CSR), and the compaction in index order behind a scan of CTA counts (cta_sum,
// cta_first_pos).
#include <climits>

#include "ust_common.cuh"

using namespace ustd;

namespace {

constexpr int kThreads = UST_THREADS;
constexpr int kWarps = kThreads / 32;
// the verification kernel: 12 warps per CTA, one CTA per SM beside the resident streaming kernel (register bound below)
constexpr int kVThreads = UST_VERIFY_THREADS;
constexpr int kVWarps = kVThreads / 32;
constexpr int kVStep = kVThreads * 4;
constexpr uint32_t kLutBytes = UST_LUT_WORDS * sizeof(uint32_t);  // table + 16 {x, y} meta pairs
constexpr int kSimNone = INT32_MIN;        // rollout simulation: no start-time annotation
constexpr int kSimLongAgo = -(1 << 30);    // ... one that timed out before the simulation began
constexpr int kDsSmem = 64;  // the kernel sits next to the streaming kernel on every SM: keep its shared memory small

struct __align__(128) Shared {
  uint32_t lut[UST_LUT_ENTRIES];  // + meta directly behind it: filled by ONE bulk (TMA) copy
  uint2 meta[16];
  unsigned long long mbar;        // mbarrier the bulk copy completes on
  unsigned long long xflag;       // fused exchange: the flag word CTA 0 published (other CTAs)
  int dsrev[kDsSmem + 1];         // DaemonSet revisions (larger tables are read from global memory: this is the rare path)
  unsigned int warp_tot[kVWarps];
  // the verdict, CTA-uniform
  unsigned long long abort_key;   // ~0 = none
  long long node_offset;          // global index of this shard's node 0
  long long slots;                // ordered path: slots left at the start of the tile being evaluated
  int redo, cut, lo, hi;
  DecideShared D;
};

// ------------------------------------------------------------------------------------------------
// per-node transition
// ------------------------------------------------------------------------------------------------
// table entry for one node. hb = hot byte, extra = derived bits (slot grant, pod-list summaries)
__device__ __forceinline__ uint32_t node_entry(const UstParams& P, const Shared& S, bool ds_smem, uint32_t hb, uint32_t fl, int rev,
                                               uint32_t di, uint32_t extra) {
  uint32_t w = (fl & UST_F_INPUT_MASK) | ((hb >> 3) & (UST_W_SKIP | UST_W_UNSCHEDULABLE)) | extra;
  // podRevisionHash == daemonsetRevisionHash (common_manager.go:318); a missing DaemonSet never matches
  bool synced;
  if (ds_smem) synced = (di < (uint32_t)P.n_ds) && (rev == S.dsrev[min(di, (uint32_t)P.n_ds)]);
  else synced = di < (uint32_t)P.n_ds && rev == __ldg(P.ds_rev + di);
  if (synced) w |= UST_W_SYNCED;
  const uint2 m = S.meta[hb & 15u];
  const uint32_t off = (__funnelshift_r(w, 0u, m.x) & (m.x >> 16)) | m.y;
  return *reinterpret_cast<const uint32_t*>(reinterpret_cast<const char*>(S.lut) + off);
}

// A node's pod-list summary byte `ps` (ust_pod_summary_kernel; layout: pods_apply() in ust_common.cuh) folded into its flags
// word `fl` and the derived bits `extra` node_entry takes: bit 4 says the list overrides UST_F_WAIT_PODS_RUNNING, which bit
// 0 then gives; bits 1-3 and 5-7 land at w bits 22-24 and 26-28. Every evaluation of a node with pod lists goes through it.
__device__ __forceinline__ void fold_podsum(uint32_t ps, uint32_t& fl, uint32_t& extra) {
  fl &= ~((ps & 0x10u) << 12);
  extra = extra | ((ps & 1u) << 16) | ((ps & 0xEEu) << 21);
}

__device__ __forceinline__ uint32_t noop_entry(uint32_t hb) { return ((hb & 15u) << 16) | 0xFF000000u; }

// abort semantics: nodes the sequential passes had not reached when the reference returned its error
// stay untouched; the aborting node carries UST_A_ERROR; an abort inside ProcessPodRestartNodes also
// drops the restarts collected so far, SchedulePodsRestart is only called after the loop
// (common_manager.go:462-523). A node that aborts in ProcessValidationRequiredNodes has already had its driver unblocked
// (UnblockLoading runs before Validate, common_manager.go:580-590).
__device__ __forceinline__ uint32_t apply_abort(const Shared& S, uint32_t ent, uint32_t hb, long long gidx) {
  const int pass = pass_of_state(hb & 15u);
  if (pass < 0) return ent;
  const unsigned long long key = UST_KEY(pass, (unsigned long long)gidx + 1ull);
  if (key >= S.abort_key) {
    const uint32_t kept = (key == S.abort_key && pass == 10) ? (ent & UST_A_UNBLOCK_SAFE_LOAD) : 0u;
    ent = noop_entry(hb) | kept;
    if (key == S.abort_key) ent |= UST_A_ERROR;
  } else if (pass == 8 && (S.abort_key >> 56) == 8) {
    ent &= ~(uint32_t)UST_A_RESTART_DRIVER_POD;
  }
  return ent;
}

// One step of kVStep nodes starting at `base`, bounds-checked against b1 (the end of the tile / the shard).
// EXACT: the ordered slot allocation - candidate = upgrade-required && !skip; rank = exclusive count of candidates in
// slice order from the start of the tile (`running` carries it from step to step); granted iff rank < S.slots
// (upgrade_inplace.go:71-109). Otherwise the grant is uniform. Abort masking and pod-list summaries as in the
// streaming pass.
template <bool EXACT>
__device__ void general_step(const UstParams& P, Shared& S, long long base, long long b1, uint32_t grant, long long& running) {
  const int t = threadIdx.x;
  const long long i0 = base + 4 * t;
  const bool aborting = S.abort_key != ~0ull;
  uint32_t hb[4], fl[4], di[4];
  int rev[4];
  int nvalid = 0;
  if (i0 + 4 <= b1) {
    nvalid = 4;
    const uint32_t h = __ldg(reinterpret_cast<const uint32_t*>(P.hot + i0));
    const uint4 f = __ldcs(reinterpret_cast<const uint4*>(P.flags + i0)), r = __ldcs(reinterpret_cast<const uint4*>(P.pod_rev + i0)),
                d = __ldcs(reinterpret_cast<const uint4*>(P.ds_idx + i0));
    hb[0] = h & 0xFFu; hb[1] = (h >> 8) & 0xFFu; hb[2] = (h >> 16) & 0xFFu; hb[3] = h >> 24;
    fl[0] = f.x; fl[1] = f.y; fl[2] = f.z; fl[3] = f.w;
    rev[0] = (int)r.x; rev[1] = (int)r.y; rev[2] = (int)r.z; rev[3] = (int)r.w;
    di[0] = d.x; di[1] = d.y; di[2] = d.z; di[3] = d.w;
  } else if (i0 < b1) {
    nvalid = (int)(b1 - i0);
    for (int k = 0; k < 4; k++) {
      const bool v = k < nvalid;
      hb[k] = v ? P.hot[i0 + k] : (uint32_t)UST_STATE_EXCLUDED;
      fl[k] = v ? P.flags[i0 + k] : 0u;
      rev[k] = v ? P.pod_rev[i0 + k] : 0;
      di[k] = v ? (uint32_t)P.ds_idx[i0 + k] : 0xFFFFFFFFu;
    }
  } else {
    for (int k = 0; k < 4; k++) { hb[k] = UST_STATE_EXCLUDED; fl[k] = 0; rev[k] = 0; di[k] = 0xFFFFFFFFu; }
  }

  uint32_t gbits[4] = {grant, grant, grant, grant};
  if (EXACT) {
    unsigned c[4], tc = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) {
      c[k] = ((hb[k] & 15u) == UST_STATE_UPGRADE_REQUIRED && !(hb[k] & UST_HOT_SKIP)) ? 1u : 0u;
      tc += c[k];
    }
    unsigned incl = tc;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned v = __shfl_up_sync(kFull, incl, o);
      if ((t & 31) >= o) incl += v;
    }
    if ((t & 31) == 31) S.warp_tot[t >> 5] = incl;
    __syncthreads();
    unsigned before = 0, step_total = 0;
#pragma unroll
    for (int w = 0; w < kVWarps; w++) {
      const unsigned v = S.warp_tot[w];
      if (w < (t >> 5)) before += v;
      step_total += v;
    }
    __syncthreads();
    long long rank = running + before + (incl - tc);
#pragma unroll
    for (int k = 0; k < 4; k++) {
      gbits[k] = (c[k] && rank < S.slots) ? UST_W_GRANTED : 0u;
      rank += c[k];
    }
    running += step_total;
  }

  if (nvalid == 0) return;
  const bool ds_smem = P.n_ds <= kDsSmem;
  uint32_t e[4];
#pragma unroll
  for (int k = 0; k < 4; k++) {
    uint32_t extra = gbits[k], f = fl[k];
    if (P.podsum && k < nvalid) fold_podsum(P.podsum[i0 + k], f, extra);  // pod-list summary of the node
    e[k] = node_entry(P, S, ds_smem, hb[k], f, rev[k], di[k], extra);
    if (aborting) e[k] = apply_abort(S, e[k], hb[k], S.node_offset + i0 + k);
  }
  uint32_t next4, out4;
  uint2 act4;
  pack4(e, next4, act4, out4);
  if (nvalid == 4) {
    __stcs(reinterpret_cast<uint32_t*>(P.next + i0), next4);
    __stcs(reinterpret_cast<uint2*>(P.actions + i0), act4);
    if (P.outcome) __stcs(reinterpret_cast<uint32_t*>(P.outcome + i0), out4);
  } else {
    for (int k = 0; k < nvalid; k++) {
      P.next[i0 + k] = (uint8_t)(e[k] >> 16);
      P.actions[i0 + k] = (uint16_t)e[k];
      if (P.outcome) P.outcome[i0 + k] = (uint8_t)(e[k] >> 24);
    }
  }
}

// A span of full steps with a uniform grant and no abort, software-pipelined: while the two steps (2048 nodes) of one
// iteration are evaluated, the loads of the next two are already in flight (two register buffers, the loop is unrolled
// over them). b0, b1: multiples of kVStep apart (the caller peels the ragged end).
struct SpanTile {
  uint32_t h[2], ps[2];
  uint4 f[2], r[2], d[2];
};
__device__ __forceinline__ void span_load(const UstParams& P, SpanTile& T, long long base, long long b1) {
  const int t = threadIdx.x;
#pragma unroll
  for (int j = 0; j < 2; j++) {
    const long long i = base + (long long)j * kVStep + 4 * t;
    const bool v = i < b1;   // warp-uniform: spans are multiples of kVStep
    const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
    T.h[j] = v ? __ldg(reinterpret_cast<const uint32_t*>(P.hot + i)) : 0x0E0E0E0Eu;
    T.ps[j] = (v && P.podsum) ? __ldcs(reinterpret_cast<const uint32_t*>(P.podsum + i)) : 0u;
    T.f[j] = v ? __ldcs(reinterpret_cast<const uint4*>(P.flags + i)) : zero;
    T.r[j] = v ? __ldcs(reinterpret_cast<const uint4*>(P.pod_rev + i)) : zero;
    T.d[j] = v ? __ldcs(reinterpret_cast<const uint4*>(P.ds_idx + i)) : zero;
  }
}
__device__ __forceinline__ void span_eval(const UstParams& P, Shared& S, const SpanTile& T, long long base, long long b1, uint32_t grant,
                                          bool ds_smem) {
  const int t = threadIdx.x;
#pragma unroll
  for (int j = 0; j < 2; j++) {
    const long long i = base + (long long)j * kVStep + 4 * t;
    if (i >= b1) continue;
    const uint32_t fl[4] = {T.f[j].x, T.f[j].y, T.f[j].z, T.f[j].w};
    const uint32_t rv[4] = {T.r[j].x, T.r[j].y, T.r[j].z, T.r[j].w};
    const uint32_t dv[4] = {T.d[j].x, T.d[j].y, T.d[j].z, T.d[j].w};
    uint32_t e[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const uint32_t hb = (T.h[j] >> (8 * k)) & 0xFFu, p = (T.ps[j] >> (8 * k)) & 0xFFu;
      uint32_t fk = fl[k], extra = grant;
      fold_podsum(p, fk, extra);
      e[k] = node_entry(P, S, ds_smem, hb, fk, (int)rv[k], dv[k], extra);
    }
    uint32_t next4, out4;
    uint2 act4;
    pack4(e, next4, act4, out4);
    __stcs(reinterpret_cast<uint32_t*>(P.next + i), next4);
    __stcs(reinterpret_cast<uint2*>(P.actions + i), act4);
    if (P.outcome) __stcs(reinterpret_cast<uint32_t*>(P.outcome + i), out4);
  }
}
__device__ void uniform_span(const UstParams& P, Shared& S, long long b0, long long b1, uint32_t grant) {
  const bool ds_smem = P.n_ds <= kDsSmem;
  constexpr long long kIter = 2LL * kVStep;
  SpanTile A, B;
  span_load(P, A, b0, b1);
  for (long long base = b0; base < b1; base += 2 * kIter) {
    span_load(P, B, base + kIter, b1);           // (all-invalid past the end: no loads are issued)
    span_eval(P, S, A, base, b1, grant, ds_smem);
    span_load(P, A, base + 2 * kIter, b1);
    span_eval(P, S, B, base + kIter, b1, grant, ds_smem);
  }
}

// candidates (upgrade-required && !skip, upgrade_inplace.go:82) among the nodes [b0, b1) - hot bytes only; b0 and
// b1 are multiples of kVStep apart inside one tile. Whole CTA; every thread returns the total.
__device__ long long count_candidates(const UstParams& P, Shared& S, long long b0, long long b1) {
  const int t = threadIdx.x;
  unsigned c = 0;
  for (long long i = b0 + 16LL * t; i < b1; i += 16LL * kVThreads) {  // b0: multiple of 1024, 16 t < 4096: aligned 16-byte loads
    const uint4 x = __ldg(reinterpret_cast<const uint4*>(P.hot + i));
    c += __popc(cand_mask4(x.x)) + __popc(cand_mask4(x.y)) + __popc(cand_mask4(x.z)) + __popc(cand_mask4(x.w));
  }
  c = __reduce_add_sync(kFull, c);
  __syncthreads();
  if ((t & 31) == 0) S.warp_tot[t >> 5] = c;
  __syncthreads();
  long long tot = 0;
#pragma unroll
  for (int w = 0; w < kVWarps; w++) tot += S.warp_tot[w];
  __syncthreads();
  return tot;
}

// Re-evaluate the steps [s0, s1) (kVStep nodes each) of one tile exactly, given where the slot budget cuts.
__device__ void redo_steps(const UstParams& P, Shared& S, int tile, int s0, int s1) {
  const long long t0 = (long long)tile * P.tile_nodes;
  long long t1 = t0 + P.tile_nodes;
  if (t1 > P.n) t1 = P.n;
  const long long b0 = t0 + (long long)s0 * kVStep;
  long long b1 = t0 + (long long)s1 * kVStep;
  if (b1 > t1) b1 = t1;
  if (b0 >= b1) return;
  const bool slotted = P.active && !P.requestor;
  const bool aborting = S.abort_key != ~0ull;
  if (slotted && tile == S.cut) {  // the cut tile: S.slots of its candidates get a slot, in slice order
    long long running = s0 > 0 ? count_candidates(P, S, t0, b0) : 0;  // candidates of the tile before this piece
    for (long long base = b0; base < b1; base += kVStep) general_step<true>(P, S, base, b1, 0u, running);
    return;
  }
  const uint32_t grant = (slotted && tile < S.cut) ? UST_W_GRANTED : 0u;
  long long running = 0, full_end = b0;
  if (!aborting) {
    full_end = b0 + ((b1 - b0) / kVStep) * kVStep;
    if (full_end > b0) uniform_span(P, S, b0, full_end, grant);
  }
  for (long long base = full_end; base < b1; base += kVStep) general_step<false>(P, S, base, b1, grant, running);
}

// Re-evaluate the tiles [ta, tb) - a contiguous run owned by one CTA when many tiles are redone. Without an abort and
// with tiles that are whole steps, the tiles before the cut and the tiles behind it are two node ranges that go
// through the pipelined span as a whole; the cut tile takes the ordered path.
__device__ void redo_range(const UstParams& P, Shared& S, int ta, int tb) {
  const int tn = P.tile_nodes;
  const int steps_per_tile = (tn + kVStep - 1) / kVStep;
  const bool aborting = S.abort_key != ~0ull;
  if (aborting || tn % kVStep != 0) {
    for (int tile = ta; tile < tb; tile++) { redo_steps(P, S, tile, 0, steps_per_tile); __syncthreads(); }
    return;
  }
  const bool slotted = P.active && !P.requestor;
  const int cut = slotted ? S.cut : 0x7FFFFFFF;
  for (int part = 0; part < 2; part++) {
    const int x = part == 0 ? ta : (cut + 1 > ta ? cut + 1 : ta);
    const int y = part == 0 ? (cut < tb ? cut : tb) : tb;
    if (x >= y) continue;
    const uint32_t grant = (slotted && part == 0) ? UST_W_GRANTED : 0u;
    const long long b0 = (long long)x * tn;
    long long b1 = (long long)y * tn;
    if (b1 > P.n) b1 = P.n;
    const long long full_end = b0 + ((b1 - b0) / kVStep) * kVStep;
    if (full_end > b0) uniform_span(P, S, b0, full_end, grant);
    long long running = 0;
    for (long long base = full_end; base < b1; base += kVStep) general_step<false>(P, S, base, b1, grant, running);
  }
  if (cut >= ta && cut < tb) { __syncthreads(); redo_steps(P, S, cut, 0, steps_per_tile); }
}

// ------------------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------------------
// Registers: an SM sub-partition has 16384. The streaming kernel's CTA puts 4 of its 13 warps (64 registers a thread) on
// one sub-partition = 8192; this kernel's 12 warps come 3 to a sub-partition, so they must stay within 8192 / 96 = 85
// registers a thread to be resident BESIDE the streaming CTA (asserted in ust_stream.cu). At 96 this
// kernel only got onto an SM when a streaming CTA left it - and the next call's streaming kernel, whose launch waits
// for every CTA here to have started, with it.
static_assert(sizeof(Shared) <= UST_VERIFY_SMEM_MAX, "the streaming kernel's residency arithmetic assumes this bound");

// this CTA is through with its call's parity set of the workspace (UstParams::verify_before; only counted where two
// streaming CTAs share an SM - with one, residency alone keeps calls k and k+2 apart, DESIGN.md §3.3)
__device__ __forceinline__ void verify_cta_done(const UstParams& P) {
  if (UST_STREAM_CTAS_PER_SM < 2) return;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(&P.ws->verify_done, 1ull);
  }
}

__global__ void __maxnreg__(UST_VERIFY_MAXREG) ust_verify_kernel(const __grid_constant__ UstParams P) {
  __shared__ Shared S;
  const int t = threadIdx.x;
  // prologue (overlaps the streaming kernel): the transition table (4.4 KiB) by one TMA bulk copy - it was uploaded by
  // a copy, not by a kernel, so it need not wait
  if (t == 0) {
    mbar_init(&S.mbar, 1);
    mbar_fence_init();
    mbar_arrive_expect_tx(&S.mbar, kLutBytes);
    bulk_g2s(S.lut, P.lut, kLutBytes, &S.mbar);
  }
  if (P.stamps && t == 0 && (blockIdx.x == 0 || blockIdx.x == gridDim.x - 1)) P.ws->dbg2[blockIdx.x == 0 ? 8 : 9] = now_ns();
  griddep_launch_dependents();  // the next call's streaming kernel may become resident (it waits for this grid itself)
  griddep_wait();               // the streaming kernel (and, split mode, the collective) has completed
  const bool lead = blockIdx.x == 0;
  if (P.stamps && lead && t == 0) P.ws->dbg2[0] = now_ns();
  bool comm_ok = true;
  if (P.split) {
    if (t < UST_V_LEN) S.D.V[t] = P.xchg[t];
  } else {
    load_local_vector(P, S.D);
    if (t < 32) {
      __syncwarp();
      if (t == 14) fix_excluded_lane(P, S.D);
    }
    if (P.fused_exchange) {
      // Only CTA 0 polls the peers' mailbox words. (Every CTA polling them - one CTA per SM x 84 x world threads spinning
      // on a few L2 lines that the peers' NVLink writes must get into - slows every step down.) The others wait for one
      // flag, one thread each.
      __syncthreads();
      const int par = (int)(P.epoch & 1);
      const unsigned long long tag = (unsigned long long)(unsigned)P.epoch << 32;
      if (lead) {
        comm_ok = exchange_vector(P, S.D, true);
        // the sum and its flag stay on this GPU: gpu scope, written by warps that issued no NVLink store (a system-scope
        // release - or a fence by a thread with peer stores in flight - waits for the peers' acknowledgements)
        if (t < UST_V_LEN) P.ws->xsum[par][t] = S.D.V[t];
        __syncthreads();
        if (t == 0) st_release_gpu(reinterpret_cast<long long*>(&P.ws->xflag[par]), (long long)(tag | (comm_ok ? 1ull : 0ull)));
      } else {
        if (t == 0) {
          const unsigned long long t0 = now_ns();
          unsigned long long v = (unsigned long long)ld_acquire_gpu(reinterpret_cast<const long long*>(&P.ws->xflag[par]));
          while ((v >> 32) != (tag >> 32)) {
            if (now_ns() - t0 > 2 * kCommTimeoutNs) { v = tag; break; }
            __nanosleep(100);
            v = (unsigned long long)ld_acquire_gpu(reinterpret_cast<const long long*>(&P.ws->xflag[par]));
          }
          S.xflag = v;
        }
        __syncthreads();
        comm_ok = (S.xflag & 1ull) != 0;
        if (t < UST_V_LEN) S.D.V[t] = __ldcg(&P.ws->xsum[par][t]);
      }
    }
  }
  if (t == 0) S.D.spec_cut = __ldcg(&P.ws->spec_used[P.parity]);
  __syncthreads();
  if (P.stamps && lead && t == 0) P.ws->dbg2[1] = now_ns();
  decide(P, S.D, lead, !comm_ok);
  if (P.stamps && lead && t == 0) P.ws->dbg2[2] = now_ns();
  const int redo = S.D.redo;
  mbar_wait(&S.mbar, 0);  // never leave with the bulk copy in flight (it landed long ago)
  if (redo == 0) { verify_cta_done(P); return; }  // the speculation held: every output of the streaming kernel is final
  if (t == 0) {
    S.redo = redo; S.cut = S.D.cut; S.lo = S.D.lo; S.hi = S.D.hi; S.slots = S.D.slots_left;
    S.abort_key = S.D.abort_key; S.node_offset = S.D.node_offset;
  }
  if (P.n_ds <= kDsSmem)
    for (int i = t; i <= P.n_ds; i += kVThreads) S.dsrev[i] = i < P.n_ds ? __ldg(P.ds_rev + i) : 0;
  __syncthreads();
  int first = S.lo, last = S.hi;
  if (redo == 2) { first = 0; last = P.n_tiles - 1; }
  const int m = last - first + 1;
  const int steps_per_tile = (P.tile_nodes + kVStep - 1) / kVStep;
  if (m >= (int)gridDim.x) {
    // many tiles: a contiguous run per CTA
    const int per = (m + (int)gridDim.x - 1) / (int)gridDim.x;
    const int ta = first + (int)blockIdx.x * per, tb = ta + per < last + 1 ? ta + per : last + 1;
    if (ta < tb) redo_range(P, S, ta, tb);
  } else {
    // a few tiles (the steady state: the one tile the budget cuts through): one step per CTA, so that the redo costs
    // one load round trip instead of one per step
    const int items = m * steps_per_tile;
    for (int it = (int)blockIdx.x; it < items; it += (int)gridDim.x) {
      const int tile = first + it / steps_per_tile, st = it % steps_per_tile;
      redo_steps(P, S, tile, st, st + 1);
      __syncthreads();
    }
  }
  if (P.stamps && lead && t == 0) P.ws->dbg2[3] = now_ns();
  verify_cta_done(P);
}

// Pod-list summaries (rows 12-14 of the scope table: pod_manager.go:256-391, :122-229, drain_manager.go:58-139).
// Only nodes whose actuator would look at its pods have their list read: wait-for-jobs, pod-deletion and
// drain-required nodes - everything else costs the hot byte. A CTA takes blocks of kPodBlock consecutive nodes:
// it compacts the nodes that need their list (in node order) into shared memory, then every thread walks the list
// of one such node with aligned 16-byte loads (8 pods each, all loads of a pass in flight together). A pod counts
// only if it matches the selector of the node's own actuator (wait-for-completion selector, deletion filter or drain
// selector: one bit of pod_flags each); those are mapped through the per-policy table of the pod's own eight bits
// (256 bytes in shared memory) and OR-ed, and the list is dropped as soon as every bit the node's state reads is set
// (the lookups of a 2 KiB table instead kept the LSU data pipe busy). One thread per list rather than one warp (the
// warp-per-node formulation executes several times the instructions).
// Neighbouring threads own neighbouring lists, so their loads share sectors. Output: one byte per node for the streaming pass (layout: pods_apply()), written
// coalesced per block.
constexpr int kPodBlock = 4096;            // nodes per block = 16 per thread
constexpr int kPodChunks = 6;              // 16-byte loads in flight per thread and pass (48 pods: a typical list in one pass)
// `validation` (UST_EVAL_VALIDATION): 0 = off, 1 = on with an empty selector (the byte carries the flag bits only),
// kValWalk = on: the validation pods are walked as well
constexpr int kValWalk = 2;

// Validate (validation_manager.go:71-175) for one validation-required node: its pods with the validation-selector bit, in
// list order, up to the first one that is not ready (the chunks of the list, kPodChunks loads in flight, until then).
__device__ __forceinline__ uint32_t validation_summary(const uint16_t* __restrict__ pod_flags, const unsigned char* bytes,
                                                       long long total_bytes, int p0, int p1, uint32_t fl, bool walk) {
  bool not_ready = false, ready_before = false;
  const int len = p1 - p0;
  if (walk && len > 0) {
    const long long c0 = (2LL * p0) & ~15LL;
    const int nchunks = (int)((2LL * p1 - c0 + 15) >> 4);
    if (c0 + 16LL * nchunks <= total_bytes) {
      const uint4* src = reinterpret_cast<const uint4*>(bytes + c0);
      int rel = (int)((c0 >> 1) - p0);
      for (int cb = 0; cb < nchunks && !not_ready; cb += kPodChunks) {
        uint4 x[kPodChunks];
#pragma unroll
        for (int u = 0; u < kPodChunks; u++) x[u] = cb + u < nchunks ? __ldcs(src + cb + u) : make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
        for (int u = 0; u < kPodChunks; u++) {
          const uint32_t wv[4] = {x[u].x, x[u].y, x[u].z, x[u].w};
#pragma unroll
          for (int e = 0; e < 8; e++) {
            const uint32_t f = (e & 1) ? wv[e >> 1] >> 16 : wv[e >> 1];
            if (!not_ready && (f & UST_POD_MATCH_VALIDATION_SELECTOR) && (unsigned)(rel + e) < (unsigned)len) {
              if (f & UST_POD_READY) ready_before = true;
              else not_ready = true;
            }
          }
          rel += 8;
        }
      }
    } else {  // the list ends within the last 16 bytes of the whole array: plain 2-byte loads
      for (int p = p0; p < p1 && !not_ready; p++) {
        const uint32_t f = __ldg(pod_flags + p);
        if (f & UST_POD_MATCH_VALIDATION_SELECTOR) {
          if (f & UST_POD_READY) ready_before = true;
          else not_ready = true;
        }
      }
    }
  }
  return ust_validation_byte(not_ready, ready_before, walk, fl);
}

// VALIDATION: the call has UST_EVAL_VALIDATION (`validation` != 0); the other instantiation is the kernel without it
template <bool VALIDATION>
__global__ void __launch_bounds__(kThreads, 6) ust_pod_summary_kernel(long long n, int active, const uint8_t* __restrict__ hot,
                                                                      const int32_t* __restrict__ pod_off,
                                                                      const uint16_t* __restrict__ pod_flags, long long n_pods,
                                                                      const uint8_t* __restrict__ podlut, uint8_t* __restrict__ podsum,
                                                                      const uint32_t* __restrict__ flags, int validation,
                                                                      unsigned long long* __restrict__ errinv) {
  __shared__ __align__(16) uint8_t lut[256];   // what a pod raises, by its own eight bits (ust_lut.h: ust_build_pod_lut256)
  __shared__ __align__(16) uint8_t res[kPodBlock];   // summary byte per node of the block (bits 6-7: state - 3 while in work)
  __shared__ unsigned short list[kPodBlock];         // block-local indices of the nodes whose list is read
  __shared__ int cnt;
  const int t = threadIdx.x, lane = t & 31;
  if (t < 64) reinterpret_cast<uint32_t*>(lut)[t] = __ldg(reinterpret_cast<const uint32_t*>(podlut) + t);
  const unsigned char* bytes = reinterpret_cast<const unsigned char*>(pod_flags);
  const long long total_bytes = 2 * n_pods;
  // hot bytes of this thread's 16 nodes of a block ("excluded" past the end of the array)
  auto load_hot = [&](long long base) -> uint4 {
    const long long i0 = base + 16 * t;
    uint32_t w[4] = {0x0E0E0E0Eu, 0x0E0E0E0Eu, 0x0E0E0E0Eu, 0x0E0E0E0Eu};
    if (i0 + 16 <= n) return __ldg(reinterpret_cast<const uint4*>(hot + i0));  // base, 16t: multiples of 16
    for (int k = 0; k < 16; k++)
      if (i0 + k < n) w[k >> 2] = (w[k >> 2] & ~(0xFFu << (8 * (k & 3)))) | ((uint32_t)hot[i0 + k] << (8 * (k & 3)));
    return make_uint4(w[0], w[1], w[2], w[3]);
  };
  for (long long base = (long long)blockIdx.x * kPodBlock; base < n; base += (long long)gridDim.x * kPodBlock) {
    if (t == 0) cnt = 0;
    __syncthreads();
    // ---- scan the block's hot bytes, compact the nodes that need their pods
    const long long i0 = base + 16 * t;
    const uint4 hv = load_hot(base);
    const uint32_t w[4] = {hv.x, hv.y, hv.z, hv.w};
    unsigned needbits = 0;
    uint32_t init[4];
#pragma unroll
    for (int k = 0; k < 16; k++) {
      const unsigned s = (w[k >> 2] >> (8 * (k & 3))) & 15u;
      const bool val = VALIDATION && s == UST_STATE_VALIDATION_REQUIRED;  // tag 3 (bits 6-7)
      const bool need = active && ((s >= UST_STATE_WAIT_FOR_JOBS_REQUIRED && s <= UST_STATE_DRAIN_REQUIRED) || val);
      // wait-for-jobs: the list overrides the pre-evaluated bit (0x10) even when it is empty
      const uint32_t b = need ? (val ? 0xC0u : (((s - UST_STATE_WAIT_FOR_JOBS_REQUIRED) << 6) | (s == UST_STATE_WAIT_FOR_JOBS_REQUIRED ? 0x10u : 0u))) : 0u;
      if ((k & 3) == 0) init[k >> 2] = 0;
      init[k >> 2] |= b << (8 * (k & 3));
      needbits |= (need ? 1u : 0u) << k;
    }
    *reinterpret_cast<uint4*>(res + 16 * t) = make_uint4(init[0], init[1], init[2], init[3]);
    const int mine_cnt = __popc(needbits);
    int incl = mine_cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(kFull, incl, o);
      if (lane >= o) incl += v;
    }
    int wbase = 0;
    if (lane == 31) wbase = atomicAdd(&cnt, incl);   // warps land in arrival order: the list is node-ordered within a warp
    wbase = __shfl_sync(kFull, wbase, 31);
    int slot = wbase + incl - mine_cnt;
    while (needbits) {
      const int k = __ffs(needbits) - 1;
      needbits &= needbits - 1;
      list[slot++] = (unsigned short)(16 * t + k);
    }
    __syncthreads();
    // ---- one thread per listed node
    const int total = cnt;
    for (int q = t; q < total; q += kThreads) {
      const int li = list[q];
      const long long i = base + li;
      const int p0 = __ldg(pod_off + i), p1 = __ldg(pod_off + i + 1);
      const int len = p1 - p0;
      unsigned r = 0;
      // the node's actuator only asks about pods that match ITS selector: wait-for-completion (bit 9), the deletion
      // filter (bit 8) or the drain selector (bit 10) - the others are not even looked up
      const unsigned tag = res[li];
      if (VALIDATION && tag == 0xC0u) {  // validation-required (validation mode): the byte of ust_lut.h, and the abort Validate causes
        const uint32_t v = validation_summary(pod_flags, bytes, total_bytes, p0, p1, __ldg(flags + i), validation == kValWalk);
        // ~key of pass 10 at this node (shard-local index, like the streaming pass's revision-hash keys)
        if (((v >> UST_VALSUM_OUTCOME_SHIFT) & 7u) == UST_VAL_ERROR) atomicMax(errinv, ~UST_KEY(10, (unsigned long long)i + 1ull));
        res[li] = (uint8_t)v;
        continue;
      }
      const unsigned s = UST_STATE_WAIT_FOR_JOBS_REQUIRED + (tag >> 6);
      const uint32_t sel = s == UST_STATE_WAIT_FOR_JOBS_REQUIRED ? (uint32_t)UST_POD_MATCH_WAIT_SELECTOR
                         : (s == UST_STATE_POD_DELETION_REQUIRED ? (uint32_t)UST_POD_MATCH_DELETION_FILTER : (uint32_t)UST_POD_MATCH_DRAIN_SELECTOR);
      // ... and once every bit the node's state reads is set, the rest of the list cannot change the answer
      const unsigned sat = s == UST_STATE_WAIT_FOR_JOBS_REQUIRED ? UST_PODSUM_WAIT_RUNNING
                         : (s == UST_STATE_POD_DELETION_REQUIRED ? (UST_PODSUM_TO_DELETE | UST_PODSUM_CANNOT_DELETE) : UST_PODSUM_DRAIN_ERROR);
      // 16-byte chunks covering the list; the last one may reach past the list but, when `safe`, not past the array
      const long long c0 = (2LL * p0) & ~15LL;
      const int nchunks = len > 0 ? (int)((2LL * p1 - c0 + 15) >> 4) : 0;
      const bool safe = c0 + 16LL * nchunks <= total_bytes;
      if (safe) {
        const uint4* src = reinterpret_cast<const uint4*>(bytes + c0);
        int rel = (int)((c0 >> 1) - p0);  // pod index of the chunk's element 0, relative to the list (<= 0 for chunk 0)
        for (int cb = 0; cb < nchunks; cb += kPodChunks) {
          uint4 x[kPodChunks];
#pragma unroll
          for (int u = 0; u < kPodChunks; u++) x[u] = cb + u < nchunks ? __ldcs(src + cb + u) : make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
          for (int u = 0; u < kPodChunks; u++) {
            if (cb + u < nchunks && (r & sat) != sat) {
              const uint32_t wv[4] = {x[u].x, x[u].y, x[u].z, x[u].w};
#pragma unroll
              for (int e = 0; e < 8; e++) {
                const uint32_t f = (e & 1) ? wv[e >> 1] >> 16 : wv[e >> 1];
                if ((f & sel) && (unsigned)(rel + e) < (unsigned)len) r |= lut[f & 255u];
              }
            }
            rel += 8;
          }
        }
      } else {  // the list ends within the last 16 bytes of the whole array: plain 2-byte loads
        for (int p = p0; p < p1; p++) {
          const uint32_t f = __ldg(pod_flags + p);
          if (f & sel) r |= lut[f & 255u];
        }
      }
      unsigned ps;
      if (s == UST_STATE_WAIT_FOR_JOBS_REQUIRED) ps = 0x10u | (r & UST_PODSUM_WAIT_RUNNING);
      else if (s == UST_STATE_POD_DELETION_REQUIRED) ps = r & (UST_PODSUM_TO_DELETE | UST_PODSUM_CANNOT_DELETE);
      else ps = r & UST_PODSUM_DRAIN_ERROR;
      res[li] = (uint8_t)ps;
    }
    __syncthreads();
    // ---- coalesced write of the block's bytes
    if (i0 + 16 <= n) {
      *reinterpret_cast<uint4*>(podsum + i0) = *reinterpret_cast<const uint4*>(res + 16 * t);
    } else {
      for (int k = 0; k < 16; k++)
        if (i0 + k < n) podsum[i0 + k] = res[16 * t + k];
    }
  }
}

// BuildState at wire level (SURVEY 8f.4): the owner join itself. One entry per driver pod with the 128-bit UID of
// OwnerReferences[0] ((0, 0) = no owner reference: an orphaned pod, common_manager.go:225-227); the driver
// DaemonSets' UIDs arrive sorted with their original indices. A pod whose owner is none of them is dropped
// (GetPodsOwnedbyDs skips it, GetOrphanedPods does not take it: common_manager.go:190-222) - it gets ds_idx -2 and
// counts as "not in snapshot". 17 B read + 4 B written per pod. The DaemonSet map (common_manager.go:181-185, keyed
// by UID) is an open-addressing hash table built by the host at load factor <= 1/4 (ust_uid_hash, linear probing,
// (0, 0) = empty slot) and copied to shared memory: one 16-byte lookup per pod in the common case. Counting is
// byte-sliced as in the streaming pass; per-DaemonSet counts are packed byte counters (<= 8 DaemonSets) or
// warp-aggregated atomics. ust_build_state_uid_kernel and ust_build_state_delta_kernel share these pieces and differ in
// their loops only.
constexpr int kUidTabSmem = 2048;  // hash slots held in shared memory (DaemonSets <= 512); larger tables stay in global memory
constexpr int kBuildU = 4;         // pods per thread and iteration: four 16-byte loads in flight
constexpr int kBuildSpill = 240;   // pods a thread counts between spills (a byte lane holds 255)

// The pieces of a BuildState pass. The kernel declares the shared arrays - tab / ord (the hash table, UID only),
// cnt_ds[kUidTabSmem / 4] (owned pods per DaemonSet), inc[256] (hot byte -> hot_increments) and cnt[16] (the counted
// fields) - and keeps a thread's counts in registers: nibble sums lo / hi and byte lanes B (ust_common.cuh), `pending`
// pods since the last spill, `excluded` pods in no bucket, and with n_ds <= 8 `dsl`, its owned-pod count per DaemonSet,
// one byte each.
//
// Prologue, whole CTA, before a barrier: the hash table staged (UID, when it fits), the counters cleared, the increment
// table filled. Returns in_smem: the table (UID) or the per-DaemonSet counters (index form) are in shared memory.
template <bool UID>
__device__ __forceinline__ bool build_prologue(ulonglong2* tab, int* ord, unsigned int* cnt_ds, unsigned long long* inc,
                                               unsigned int* cnt, int n_ds, const ulonglong2* __restrict__ ds_tab,
                                               const int32_t* __restrict__ ds_tab_idx, int tab_slots) {
  const int t = threadIdx.x;
  const bool in_smem = UID ? tab_slots <= kUidTabSmem : n_ds <= kUidTabSmem / 4;  // UID: then n_ds <= kUidTabSmem / 4 too
  if (in_smem) {
    if (UID)
      for (int i = t; i < tab_slots; i += kThreads) { tab[i] = ds_tab[i]; ord[i] = ds_tab_idx[i]; }
    for (int i = t; i < n_ds; i += kThreads) cnt_ds[i] = 0;
  }
  inc[t] = hot_increments(t);
  if (t < 16) cnt[t] = 0;
  return in_smem;
}

// The owner join of one pod with owner UID u: -1 = orphaned (IsOrphanedPod), -2 = owned by none of the driver DaemonSets
// (dropped), else the DaemonSet's index. Linear probing; the table is at most a quarter full.
__device__ __forceinline__ int build_join(const ulonglong2& u, const ulonglong2* table, const int* order, unsigned slot_mask) {
  int d = -2;
  if ((u.x | u.y) == 0ull) {
    d = -1;  // IsOrphanedPod
  } else {
    unsigned slot = ust_uid_hash(u.x, u.y) & slot_mask;
    for (;;) {
      const ulonglong2 e = table[slot];
      if (e.x == u.x && e.y == u.y) { d = order[slot]; break; }
      if ((e.x | e.y) == 0ull) break;  // empty slot: not a driver DaemonSet's pod
      slot = (slot + 1u) & slot_mask;
    }
  }
  return d;
}

// The counts of one existing pod with hot byte hb; `owned` = not dropped by the join. In the snapshot unless dropped or
// marked pending-unscheduled by the host (code 14).
__device__ __forceinline__ void build_count(unsigned hb, bool owned, const unsigned long long* inc, uint32_t (&B)[4], uint32_t& lo,
                                            uint32_t& hi, int& pending, long long& excluded) {
  if (owned && (hb & 15u) < 14u) {
    const unsigned long long v = inc[hb];
    lo += (uint32_t)v;
    hi += (uint32_t)(v >> 32);
  } else {
    excluded++;
  }
  if ((++pending & 7) == 0) widen(lo, hi, B);
}

// Per-DaemonSet owned-pod counts (before the pending-skip, upgrade_state.go:128), whole warp; d < 0 counts for none. A
// handful of DaemonSets (the usual case): eight byte counters packed in a register, flushed with the other counters;
// otherwise one atomic per distinct DaemonSet per warp.
__device__ __forceinline__ void build_count_ds(int d, unsigned long long& dsl, unsigned int* cnt_ds, unsigned long long* ds_count,
                                               int n_ds, bool in_smem) {
  if (n_ds <= 8) {
    if (d >= 0) dsl += 1ull << (8 * d);
  } else {
    const unsigned act = __ballot_sync(kFull, d >= 0);
    if (d >= 0) {
      const unsigned peers = __match_any_sync(act, d);
      if ((threadIdx.x & 31) == __ffs(peers) - 1) {
        if (in_smem) atomicAdd(&cnt_ds[d], (unsigned)__popc(peers));
        else atomicAdd(&ds_count[d], (unsigned long long)__popc(peers));
      }
    }
  }
}

// A thread's byte lanes and packed DaemonSet counts into shared memory; due every kBuildSpill pods and at the end.
__device__ __forceinline__ void build_spill(uint32_t (&B)[4], uint32_t& lo, uint32_t& hi, int& pending, unsigned long long& dsl,
                                            unsigned int* cnt, unsigned int* cnt_ds) {
  widen(lo, hi, B);
#pragma unroll
  for (int f = 0; f < 16; f++) {
    const unsigned v = field_of(B, f);
    if (v) atomicAdd(&cnt[f], v);
  }
  if (dsl) {
#pragma unroll
    for (int q = 0; q < 8; q++) {
      const unsigned v = (unsigned)(dsl >> (8 * q)) & 0xFFu;
      if (v) atomicAdd(&cnt_ds[q], v);
    }
    dsl = 0;
  }
  B[0] = B[1] = B[2] = B[3] = 0;
  pending = 0;
}

// Epilogue, whole CTA, after the last spill and a barrier: fields 0..13 per state code, 14 unavailable, 15 candidates ->
// ws->bs_acc[0..13], [16], [17]; the pods in no bucket -> ws->bs_acc[UST_STATE_EXCLUDED]; the per-DaemonSet counts ->
// ds_count.
__device__ __forceinline__ void build_finish(int t, long long excluded, const unsigned int* cnt, const unsigned int* cnt_ds,
                                             unsigned long long* ds_count, int n_ds, bool in_smem, UstWorkspace* ws) {
  for (int o = 16; o > 0; o >>= 1) excluded += __shfl_xor_sync(kFull, excluded, o);
  if ((t & 31) == 0 && excluded) atomicAdd(&ws->bs_acc[UST_STATE_EXCLUDED], (unsigned long long)excluded);
  if (t < 14) { if (cnt[t]) atomicAdd(&ws->bs_acc[t], (unsigned long long)cnt[t]); }
  else if (t == 14) { if (cnt[14]) atomicAdd(&ws->bs_acc[16], (unsigned long long)cnt[14]); }
  else if (t == 15) { if (cnt[15]) atomicAdd(&ws->bs_acc[17], (unsigned long long)cnt[15]); }
  if (in_smem)
    for (int i = t; i < n_ds; i += kThreads)
      if (cnt_ds[i]) atomicAdd(&ds_count[i], (unsigned long long)cnt_ds[i]);
}

// The sum over a CTA of every thread's count c: warp reduction, then one shared-memory atomic per warp into `tot`, which
// the caller zeroed before a barrier. Whole CTA; `tot` holds the sum after the helper's barrier. The caller reads it on
// one thread, which may also reset it for the next sum: the next barrier orders that reset before any new atomic.
__device__ __forceinline__ void cta_sum(unsigned c, unsigned int& tot) {
  c = __reduce_add_sync(kFull, c);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(&tot, c);
  __syncthreads();
}

// The first output position of this thread's c outputs when the CTA writes its outputs in thread order from
// cta_off[blockIdx.x] on (the scanned CTA counts, ust_diff_scan_kernel): warp shuffle-up scan, per-warp totals in shared
// memory, sum of the earlier warps. Whole CTA.
__device__ __forceinline__ long long cta_first_pos(unsigned c, const unsigned int* __restrict__ cta_off) {
  __shared__ unsigned int wtot[kWarps];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  unsigned incl = c;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned u = __shfl_up_sync(kFull, incl, o);
    if (lane >= o) incl += u;
  }
  if (lane == 31) wtot[warp] = incl;
  __syncthreads();
  unsigned before = 0;
  for (int w = 0; w < warp; w++) before += wtot[w];
  return (long long)cta_off[blockIdx.x] + before + incl - c;
}

// UID = false is the index form (ust_build_state: the host has already resolved the owner, ds_idx_in holds it; an index
// outside [0, n_ds) counts for no DaemonSet): same counting, no join, nothing dropped. A grid-stride loop over chunks of
// kThreads * kBuildU pods.
template <bool UID>
__global__ void __launch_bounds__(kThreads) ust_build_state_uid_kernel(long long n, const uint8_t* __restrict__ hot,
                                                                       const ulonglong2* __restrict__ owner,
                                                                       const int32_t* __restrict__ ds_idx_in, int n_ds,
                                                                       const ulonglong2* __restrict__ ds_tab,
                                                                       const int32_t* __restrict__ ds_tab_idx, int tab_slots,
                                                                       int32_t* __restrict__ ds_idx_out,
                                                                       unsigned long long* ds_count, UstWorkspace* ws) {
  __shared__ ulonglong2 tab[kUidTabSmem];
  __shared__ int ord[kUidTabSmem];
  __shared__ unsigned int cnt_ds[kUidTabSmem / 4];
  __shared__ unsigned long long inc[256];
  __shared__ unsigned int cnt[16];
  const int t = threadIdx.x;
  const bool in_smem = build_prologue<UID>(tab, ord, cnt_ds, inc, cnt, n_ds, ds_tab, ds_tab_idx, tab_slots);
  __syncthreads();
  const ulonglong2* table = in_smem ? tab : ds_tab;
  const int* order = in_smem ? ord : ds_tab_idx;
  const unsigned slot_mask = (unsigned)tab_slots - 1u;  // tab_slots is a power of two
  uint32_t B[4] = {0, 0, 0, 0}, lo = 0, hi = 0;
  int pending = 0;
  long long excluded = 0;
  unsigned long long dsl = 0;
  const long long stride = (long long)gridDim.x * kThreads * kBuildU;
  for (long long i0 = (long long)blockIdx.x * kThreads * kBuildU; i0 < n; i0 += stride) {  // warp-uniform trip count
    ulonglong2 u[kBuildU];
    int dk[kBuildU];
    unsigned hb[kBuildU];
#pragma unroll
    for (int k = 0; k < kBuildU; k++) {
      const long long i = i0 + (long long)k * kThreads + t;
      u[k] = make_ulonglong2(0ull, 0ull);
      dk[k] = -1;
      hb[k] = UST_STATE_EXCLUDED;
      if (i < n) {
        if (UID) u[k] = __ldcs(owner + i); else dk[k] = __ldcs(ds_idx_in + i);
        hb[k] = __ldg(hot + i);
      }
    }
#pragma unroll
    for (int k = 0; k < kBuildU; k++) {
      const long long i = i0 + (long long)k * kThreads + t;
      int d = -2;
      if (i < n) {
        d = UID ? build_join(u[k], table, order, slot_mask) : ((dk[k] >= 0 && dk[k] < n_ds) ? dk[k] : -1);
        if (UID) __stcs(ds_idx_out + i, d);
        build_count(hb[k], d != -2, inc, B, lo, hi, pending, excluded);
      }
      build_count_ds(d, dsl, cnt_ds, ds_count, n_ds, in_smem);
    }
    if (pending >= kBuildSpill) build_spill(B, lo, hi, pending, dsl, cnt, cnt_ds);
  }
  build_spill(B, lo, hi, pending, dsl, cnt, cnt_ds);
  __syncthreads();
  build_finish(t, excluded, cnt, cnt_ds, ds_count, n_ds, in_smem, ws);
}

__global__ void ust_build_state_finish_kernel(int n_ds, const int32_t* ds_desired, unsigned long long* ds_count,
                                              UstWorkspace* ws, ust_counters* out) {
  ust_counters c;
  for (int i = 0; i < 16; i++) c.hist[i] = (long long)ws->bs_acc[i];
  c.unavailable = (long long)ws->bs_acc[16];
  c.candidates = (long long)ws->bs_acc[17];
  c.total_managed = c.hist[0] + c.hist[1] + c.hist[2] + c.hist[3] + c.hist[4] + c.hist[5] + c.hist[8] + c.hist[9] +
                    c.hist[10] + c.hist[11] + c.hist[12];
  c.in_progress = c.total_managed - c.hist[0] - c.hist[11] - c.hist[1];
  c.max_unavailable = 0;
  c.upgrades_available = 0;
  c.error_code = UST_OK;
  c.error_index = -1;
  c.error_pass = -1;
  for (int d = 0; d < n_ds; d++)
    if ((unsigned long long)(long long)ds_desired[d] != ds_count[d]) {  // upgrade_state.go:128-131
      c.error_code = UST_ERR_DS_UNSCHEDULED;
      c.error_index = d;
      break;
    }
  for (int i = 0; i < 7; i++) c.reserved[i] = 0;
  *out = c;
  for (int i = 0; i < 18; i++) ws->bs_acc[i] = 0;
  for (int d = 0; d < n_ds; d++) ds_count[d] = 0;
}

// The resident driver-pod list of ust_build_state_delta: the join and the counts of the BuildState pieces above (same
// finish kernel); the pass also compares each pod's owner index with the previous call's and works in fixed tiles of
// kBuildTile pods, so that the changed count of every tile comes out of it (cta_sum): the scan of ust_diff_scan_kernel
// and ust_build_state_write_kernel then compact the changed pods in index order. 21 B read + 4 B written per pod here,
// 8 B read per pod by the write pass.
constexpr int kBuildTile = 4096;  // pods per tile: 16 per thread

__global__ void __launch_bounds__(kThreads) ust_build_state_delta_kernel(long long n, const uint8_t* __restrict__ hot,
                                                                         const ulonglong2* __restrict__ owner, int n_ds,
                                                                         const ulonglong2* __restrict__ ds_tab,
                                                                         const int32_t* __restrict__ ds_tab_idx, int tab_slots,
                                                                         const int32_t* __restrict__ prev, int32_t* __restrict__ cur,
                                                                         unsigned int* __restrict__ tile_count,
                                                                         unsigned long long* ds_count, UstWorkspace* ws) {
  __shared__ ulonglong2 tab[kUidTabSmem];
  __shared__ int ord[kUidTabSmem];
  __shared__ unsigned int cnt_ds[kUidTabSmem / 4];
  __shared__ unsigned long long inc[256];
  __shared__ unsigned int cnt[16];
  __shared__ unsigned int tile_changed;
  const int t = threadIdx.x;
  const bool in_smem = build_prologue<true>(tab, ord, cnt_ds, inc, cnt, n_ds, ds_tab, ds_tab_idx, tab_slots);
  if (t == 0) tile_changed = 0;
  __syncthreads();
  const ulonglong2* table = in_smem ? tab : ds_tab;
  const int* order = in_smem ? ord : ds_tab_idx;
  const unsigned slot_mask = (unsigned)tab_slots - 1u;
  uint32_t B[4] = {0, 0, 0, 0}, lo = 0, hi = 0;
  int pending = 0;
  long long excluded = 0;
  unsigned long long dsl = 0;
  const long long tiles = (n + kBuildTile - 1) / kBuildTile;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {  // CTA-uniform trip counts
    unsigned changed = 0;
    for (int j = 0; j < kBuildTile; j += kThreads * kBuildU) {
      const long long i0 = tile * kBuildTile + j;
      ulonglong2 u[kBuildU];
      unsigned hb[kBuildU];
      int pv[kBuildU];
#pragma unroll
      for (int k = 0; k < kBuildU; k++) {
        const long long i = i0 + (long long)k * kThreads + t;
        u[k] = make_ulonglong2(0ull, 0ull);
        hb[k] = UST_STATE_EXCLUDED;
        pv[k] = 0;
        if (i < n) { u[k] = __ldcs(owner + i); hb[k] = __ldg(hot + i); pv[k] = __ldcs(prev + i); }
      }
#pragma unroll
      for (int k = 0; k < kBuildU; k++) {
        const long long i = i0 + (long long)k * kThreads + t;
        int d = -2;
        if (i < n) {
          d = build_join(u[k], table, order, slot_mask);
          __stcs(cur + i, d);
          changed += d != pv[k] ? 1u : 0u;
          build_count(hb[k], d != -2, inc, B, lo, hi, pending, excluded);
        }
        build_count_ds(d, dsl, cnt_ds, ds_count, n_ds, in_smem);
      }
      if (pending >= kBuildSpill) build_spill(B, lo, hi, pending, dsl, cnt, cnt_ds);
    }
    cta_sum(changed, tile_changed);
    if (t == 0) { tile_count[tile] = tile_changed; tile_changed = 0; }
    __syncthreads();
  }
  build_spill(B, lo, hi, pending, dsl, cnt, cnt_ds);
  __syncthreads();
  build_finish(t, excluded, cnt, cnt_ds, ds_count, n_ds, in_smem, ws);
}

// The ordered write of ust_build_state_delta's sparse outputs: tile b's changed pods go to positions tile_off[b] .. (the
// scanned tile counts), in index order; those at or beyond `cap` are not written.
__global__ void __launch_bounds__(kThreads) ust_build_state_write_kernel(long long n, const int32_t* __restrict__ cur,
                                                                         const int32_t* __restrict__ prev,
                                                                         const unsigned int* __restrict__ tile_off, long long cap,
                                                                         long long* __restrict__ out_idx, int32_t* __restrict__ out_ds) {
  const int t = threadIdx.x;
  const long long i0 = (long long)blockIdx.x * kBuildTile + 16 * t;
  int c16[16];
  unsigned m = 0;
  if (i0 + 16 <= n) {  // cur and prev are 16-byte aligned (device allocations), i0 a multiple of 16
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const int4 a = __ldcs(reinterpret_cast<const int4*>(cur + i0) + q), b = __ldcs(reinterpret_cast<const int4*>(prev + i0) + q);
      c16[4 * q] = a.x; c16[4 * q + 1] = a.y; c16[4 * q + 2] = a.z; c16[4 * q + 3] = a.w;
      m |= (unsigned)(a.x != b.x) << (4 * q) | (unsigned)(a.y != b.y) << (4 * q + 1) | (unsigned)(a.z != b.z) << (4 * q + 2) |
           (unsigned)(a.w != b.w) << (4 * q + 3);
    }
  } else {
#pragma unroll
    for (int k = 0; k < 16; k++) {
      c16[k] = 0;
      if (i0 + k < n) { c16[k] = cur[i0 + k]; m |= (unsigned)(c16[k] != prev[i0 + k]) << k; }
    }
  }
  long long pos = cta_first_pos(__popc(m), tile_off);
#pragma unroll
  for (int k = 0; k < 16; k++) {
    if (!((m >> k) & 1u)) continue;
    if (pos < cap) { out_idx[pos] = i0 + k; out_ds[pos] = c16[k]; }
    pos++;
  }
}

// The n_changed overwrites of ust_build_state_delta: state byte and owner UID of the pods at idx (new indices).
__global__ void __launch_bounds__(kThreads) ust_build_state_patch_kernel(long long m, const long long* __restrict__ idx,
                                                                         const uint8_t* __restrict__ state,
                                                                         const ulonglong2* __restrict__ uid, uint8_t* hot_out,
                                                                         ulonglong2* uid_out) {
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long k = (long long)blockIdx.x * kThreads + threadIdx.x; k < m; k += stride) {
    const long long i = __ldg(idx + k);
    hot_out[i] = __ldg(state + k);
    uid_out[i] = __ldg(uid + k);
  }
}

// Delta update of the resident snapshot (SURVEY 8f.2): scatter the re-encoded nodes into the SoA arrays. CLOCK (clocked
// pod-list deltas): their start times too.
template <bool CLOCK>
__global__ void __launch_bounds__(kThreads) ust_patch_kernel(long long m, const long long* __restrict__ idx,
                                                             const uint8_t* __restrict__ state, const uint32_t* __restrict__ flags,
                                                             const int32_t* __restrict__ pod_rev, const int32_t* __restrict__ ds_idx,
                                                             uint8_t* hot_out, uint32_t* flags_out, int32_t* rev_out, int32_t* ds_out,
                                                             const long long* __restrict__ start, long long* start_out) {
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long k = (long long)blockIdx.x * kThreads + threadIdx.x; k < m; k += stride) {
    const long long i = __ldg(idx + k);
    hot_out[i] = __ldg(state + k);
    flags_out[i] = __ldg(flags + k);
    rev_out[i] = __ldg(pod_rev + k);
    ds_out[i] = __ldg(ds_idx + k);
    if (CLOCK) start_out[i] = __ldg(start + k);
  }
}

// Membership splice of the resident snapshot (ust_apply_state_delta_splice): one pass over the old columns and the previous
// call's outputs that writes every surviving node at its new index in a second buffer set, and the inserted nodes beside
// them (previous output next_state = 0xFF, which no state code equals, so the diff reports them). A CTA owns
// kSpliceTile old positions [b0, b1) of 0..n (position n holds no node, only the inserts at the end). It finds the
// parts of the two sorted lists that fall in its range once, by binary search, and turns them into per-position new
// indices in shared memory:
//   old node i          -> i - #removed < i + #inserts with insert_before <= i
//   insert k at pos p   -> p - #removed < p + k
// 16 B read + 16 B written per surviving node.
constexpr int kSpliceTile = 2048;
constexpr int kSplicePer = kSpliceTile / kThreads;  // contiguous positions per thread in the scan
static_assert(kSplicePer * kThreads == kSpliceTile, "splice tile");

__device__ __forceinline__ long long splice_lower_bound(const long long* __restrict__ a, long long len, long long v) {
  long long lo = 0, hi = len;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (__ldg(a + mid) < v) lo = mid + 1; else hi = mid;
  }
  return lo;
}
// The last index r in [0, len) with a[r] <= v over a sorted array in global memory (0 when there is none; every caller
// searches a v >= a[0]). Run and segment starts: long long for node positions, int32_t for pod positions.
template <class T>
__device__ __forceinline__ long long last_le(const T* __restrict__ a, long long len, T v) {
  long long lo = 0, hi = len;
  while (hi - lo > 1) {
    const long long mid = (lo + hi) >> 1;
    if (__ldg(a + mid) <= v) lo = mid; else hi = mid;
  }
  return lo;
}
// ... and over a staged slice a[0, len), from a hint r with a[r] <= v (0, or the answer for a smaller v)
template <class T>
__device__ __forceinline__ int last_le_from(const T* a, int r, int len, T v) {
  int hi = len;
  while (hi - r > 1) {
    const int mid = (r + hi) >> 1;
    if (a[mid] <= v) r = mid; else hi = mid;
  }
  return r;
}

__global__ void __launch_bounds__(kThreads) ust_splice_kernel(long long n, long long n_rm, const long long* __restrict__ rm,
                                                              long long n_ins, const long long* __restrict__ ib,
                                                              const uint8_t* __restrict__ ins_hot, const uint32_t* __restrict__ ins_flags,
                                                              const int32_t* __restrict__ ins_rev, const int32_t* __restrict__ ins_ds,
                                                              const uint8_t* __restrict__ hot, const uint32_t* __restrict__ flags,
                                                              const int32_t* __restrict__ rev, const int32_t* __restrict__ ds,
                                                              const uint8_t* __restrict__ next, const uint16_t* __restrict__ act,
                                                              uint8_t* __restrict__ o_hot, uint32_t* __restrict__ o_flags,
                                                              int32_t* __restrict__ o_rev, int32_t* __restrict__ o_ds,
                                                              uint8_t* __restrict__ o_next, uint16_t* __restrict__ o_act) {
  __shared__ long long s_dst[kSpliceTile];   // inserts at or before the position (range-relative), then old node's new index
  __shared__ long long s_base[kSpliceTile];  // position - removed before it: insert k at the position goes to s_base + k
  __shared__ uint8_t s_rm[kSpliceTile];
  __shared__ long long s_bounds[4];
  __shared__ long long s_wmax[kWarps];
  __shared__ int s_wsum[kWarps];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const long long b0 = (long long)blockIdx.x * kSpliceTile;
  const long long b1 = b0 + kSpliceTile < n + 1 ? b0 + kSpliceTile : n + 1;
  const int len = (int)(b1 - b0);
  if (t < 4) s_bounds[t] = t < 2 ? splice_lower_bound(rm, n_rm, t ? b1 : b0) : splice_lower_bound(ib, n_ins, t == 3 ? b1 : b0);
  for (int j = t; j < kSpliceTile; j += kThreads) { s_dst[j] = 0; s_rm[j] = 0; }
  __syncthreads();
  const long long r0 = s_bounds[0], r1 = s_bounds[1], q0 = s_bounds[2], q1 = s_bounds[3];
  for (long long k = r0 + t; k < r1; k += kThreads) s_rm[__ldg(rm + k) - b0] = 1;
  for (long long k = q0 + t; k < q1; k += kThreads) {
    const long long p = __ldg(ib + k);
    if (k + 1 == q1 || __ldg(ib + k + 1) != p) s_dst[p - b0] = k + 1 - q0;  // last insert at p: inserts at or before p
  }
  __syncthreads();
  // running max of the insert counts (they only grow with the position), exclusive running sum of the removals
  long long vi[kSplicePer];
  int vr[kSplicePer];
  long long mx = 0;
  int sm = 0;
#pragma unroll
  for (int e = 0; e < kSplicePer; e++) {
    const int j = t * kSplicePer + e;
    mx = s_dst[j] > mx ? s_dst[j] : mx;
    vi[e] = mx;
    vr[e] = sm;
    sm += s_rm[j];
  }
  long long wmx = mx;
  int wsm = sm;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const long long u = __shfl_up_sync(kFull, wmx, o);
    const int v = __shfl_up_sync(kFull, wsm, o);
    if (lane >= o) { wmx = u > wmx ? u : wmx; wsm += v; }
  }
  if (lane == 31) { s_wmax[warp] = wmx; s_wsum[warp] = wsm; }
  long long pmx = __shfl_up_sync(kFull, wmx, 1);
  int psm = __shfl_up_sync(kFull, wsm, 1);
  if (lane == 0) { pmx = 0; psm = 0; }
  __syncthreads();
  for (int w = 0; w < warp; w++) { pmx = s_wmax[w] > pmx ? s_wmax[w] : pmx; psm += s_wsum[w]; }
#pragma unroll
  for (int e = 0; e < kSplicePer; e++) {
    const int j = t * kSplicePer + e;
    const long long base = b0 + j - (r0 + psm + vr[e]);
    s_base[j] = base;
    s_dst[j] = base + q0 + (vi[e] > pmx ? vi[e] : pmx);
  }
  __syncthreads();
  const int old_len = b1 <= n ? len : len - 1;  // position n is no node
#pragma unroll 4
  for (int j = t; j < old_len; j += kThreads) {
    const long long i = b0 + j;
    const uint8_t h = __ldcs(hot + i);
    const uint32_t f = __ldcs(flags + i);
    const int32_t r = __ldcs(rev + i);
    const int32_t d = __ldcs(ds + i);
    const uint8_t x = __ldcs(next + i);
    const uint16_t a = __ldcs(act + i);
    if (s_rm[j]) continue;
    const long long o = s_dst[j];
    o_hot[o] = h; o_flags[o] = f; o_rev[o] = r; o_ds[o] = d; o_next[o] = x; o_act[o] = a;
  }
  for (long long k = q0 + t; k < q1; k += kThreads) {
    const long long o = s_base[__ldg(ib + k) - b0] + k;
    o_hot[o] = __ldg(ins_hot + k); o_flags[o] = __ldg(ins_flags + k); o_rev[o] = __ldg(ins_rev + k); o_ds[o] = __ldg(ins_ds + k);
    o_next[o] = 0xFF;
    o_act[o] = 0;
  }
}

// New node order of the resident snapshot (ust_apply_state_delta_reorder): one pass that writes every node of the new
// snapshot at its new index in a second buffer set. The new order is a list of runs: run r covers new positions [run_off[r], run_off[r + 1]) and reads them from old nodes
// run_src[r], run_src[r] + 1, ... (run_src >= 0), or from inserted nodes -1 - run_src, ... (run_src < 0), whose previous
// output next_state is 0xFF (no state code equals it, so the diff reports them). A CTA owns kGatherTile new positions;
// it finds the runs that cover them once, by binary search, and stages their offsets and sources in shared memory
// (every run is at least one position long, so at most kGatherTile of them meet a tile). Each thread then finds its
// positions' runs in that range, walking forward from the run of its previous position.
// 16 B read + 16 B written per node, 16 B per run; a run is read contiguously. OUTCOME (ust_apply_state_delta_pods_reorder):
// the previous actuator_outcome travels too (1 B more each way; 0xFF for inserted nodes). CLOCK
// (ust_apply_state_delta_pods_clocked): the start time too (8 B more each way; inserted nodes bring theirs).
constexpr int kGatherTile = 2048;

// The run lookup of the gather kernels (ust_reorder_kernel, ust_build_state_reorder_kernel): copy(p, src, k) for every new
// position p of this CTA's tile, with the source of p's run (old start, or -1 - offset into the inserted entries) and p's
// offset k in that run.
template <class Copy>
__device__ __forceinline__ void gather_runs(long long n, long long n_runs, const long long* __restrict__ run_off,
                                            const long long* __restrict__ run_src, Copy copy) {
  __shared__ long long s_off[kGatherTile];
  __shared__ long long s_src[kGatherTile];
  __shared__ long long s_runs[2];
  const int t = threadIdx.x;
  const long long b0 = (long long)blockIdx.x * kGatherTile;
  if (b0 >= n) return;  // n == 0: the one CTA of the launch has nothing to do
  const long long b1 = b0 + kGatherTile < n ? b0 + kGatherTile : n;
  if (t < 2) s_runs[t] = last_le(run_off, n_runs, t ? b1 - 1 : b0);  // the last run that starts at or before b0 / b1 - 1
  __syncthreads();
  const long long r0 = s_runs[0];
  const int nr = (int)(s_runs[1] - r0 + 1);
  for (int j = t; j < nr; j += kThreads) { s_off[j] = __ldg(run_off + r0 + j); s_src[j] = __ldg(run_src + r0 + j); }
  __syncthreads();
  const int len = (int)(b1 - b0);
  int r = 0;
#pragma unroll 4
  for (int j = t; j < len; j += kThreads) {
    const long long p = b0 + j;
    r = last_le_from(s_off, r, nr, p);
    copy(p, s_src[r], p - s_off[r]);
  }
}

template <bool OUTCOME, bool CLOCK>
__global__ void __launch_bounds__(kThreads) ust_reorder_kernel(long long n, long long n_runs, const long long* __restrict__ run_off,
                                                               const long long* __restrict__ run_src,
                                                               const uint8_t* __restrict__ ins_hot, const uint32_t* __restrict__ ins_flags,
                                                               const int32_t* __restrict__ ins_rev, const int32_t* __restrict__ ins_ds,
                                                               const uint8_t* __restrict__ hot, const uint32_t* __restrict__ flags,
                                                               const int32_t* __restrict__ rev, const int32_t* __restrict__ ds,
                                                               const uint8_t* __restrict__ next, const uint16_t* __restrict__ act,
                                                               const uint8_t* __restrict__ oc,
                                                               uint8_t* __restrict__ o_hot, uint32_t* __restrict__ o_flags,
                                                               int32_t* __restrict__ o_rev, int32_t* __restrict__ o_ds,
                                                               uint8_t* __restrict__ o_next, uint16_t* __restrict__ o_act,
                                                               uint8_t* __restrict__ o_oc, const long long* __restrict__ ins_start,
                                                               const long long* __restrict__ start, long long* __restrict__ o_start) {
  gather_runs(n, n_runs, run_off, run_src, [=](long long p, long long src, long long k) {
    if (src >= 0) {
      const long long i = src + k;
      o_hot[p] = __ldcs(hot + i); o_flags[p] = __ldcs(flags + i); o_rev[p] = __ldcs(rev + i); o_ds[p] = __ldcs(ds + i);
      o_next[p] = __ldcs(next + i); o_act[p] = __ldcs(act + i);
      if (OUTCOME) o_oc[p] = __ldcs(oc + i);
      if (CLOCK) o_start[p] = __ldcs(start + i);
    } else {
      const long long i = -1 - src + k;
      o_hot[p] = __ldg(ins_hot + i); o_flags[p] = __ldg(ins_flags + i); o_rev[p] = __ldg(ins_rev + i); o_ds[p] = __ldg(ins_ds + i);
      o_next[p] = 0xFF; o_act[p] = 0;
      if (OUTCOME) o_oc[p] = 0xFF;
      if (CLOCK) o_start[p] = __ldg(ins_start + i);
    }
  });
}

// Clocked pod-list calls (ust_apply_state_clocked, ust_apply_state_delta_pods_clocked): bits 18 and 27 of the resident flags,
// derived from the resident start column and the call's clock just before the evaluation reads them (include/ust.h,
// ust_clock). A thread reads 16 hot bytes in one load; only wait-for-jobs-required and validation-required nodes read their
// flags word - and, with a valid start annotation, their start - and write the word back when it changes. 1 B per node,
// plus up to 12 B read and 4 B written per such node. (A variant that issued the flags loads of all 16 nodes first, then
// their start loads, measured slower at C4: 67 against 53 us, DESIGN.md.)
// On the way the kernel lists the candidates of the call's next deadline (include/ust.h, ust_next_deadline): the nodes whose
// bit is clear now and turns on at some later time, d + 1 with d = start + timeout wrapped and now <= d < INT64_MAX. CTA b
// appends them to its own `region` slots of `cand` (a warp scan, one shared-memory atomic per warp) and leaves their count
// in cand_count[b]; ust_deadline_kernel reads that list and nothing else. A node is stored as its 32-bit offset among the
// CTA's own nodes, in the order the CTA visits them (cand_node() below). CTA 0 resets the call's deadline.
__global__ void __launch_bounds__(kThreads) ust_clock_kernel(long long n, const uint8_t* __restrict__ hot, uint32_t* __restrict__ flags,
                                                             const long long* __restrict__ start, long long now, long long wait_timeout,
                                                             uint32_t* __restrict__ cand, unsigned int* __restrict__ cand_count,
                                                             long long region, unsigned long long* __restrict__ deadline) {
  __shared__ unsigned int n_cand;
  const int t = threadIdx.x, lane = t & 31;
  if (t == 0) {
    n_cand = 0;
    if (blockIdx.x == 0) *deadline = ~0ull;
  }
  __syncthreads();
  uint32_t* mine = cand + (long long)blockIdx.x * region;
  const long long chunks = (n + 15) / 16;  // the hot column carries 16 bytes of padding
  const long long stride = (long long)gridDim.x * kThreads;
  uint32_t it16 = 0;  // 16 * kThreads * the iteration: the offset of this iteration's first node among the CTA's
  for (long long c0 = (long long)blockIdx.x * kThreads; c0 < chunks; c0 += stride, it16 += 16 * kThreads) {  // warp-uniform trip count
    const long long c = c0 + t;
    unsigned cbits = 0;  // this chunk's candidates
    if (c < chunks) {
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(hot) + c);
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int j = 0; j < 16; j++) {
        const unsigned s = (w[j >> 2] >> (8 * (j & 3))) & UST_HOT_STATE_MASK;
        const long long i = c * 16 + j;
        if ((s != UST_STATE_WAIT_FOR_JOBS_REQUIRED && s != UST_STATE_VALIDATION_REQUIRED) || i >= n) continue;
        const bool wait = s == UST_STATE_WAIT_FOR_JOBS_REQUIRED;
        const uint32_t anno = wait ? UST_F_WAIT_START_ANNO : UST_F_VALIDATION_START_ANNO;
        const uint32_t invalid = wait ? UST_F_WAIT_START_INVALID : UST_F_VALIDATION_START_INVALID;
        const uint32_t f = flags[i];
        const bool valid = (f & (anno | invalid)) == anno;
        const long long d = valid ? ust_deadline(__ldg(start + i), wait ? wait_timeout : (long long)UST_VALIDATION_TIMEOUT_SECONDS) : 0;
        const bool timed_out = valid && now > d;
        if (valid && !timed_out && d != LLONG_MAX) cbits |= 1u << j;
        const uint32_t g = (f & ~(UST_F_WAIT_TIMED_OUT | UST_F_VALIDATION_TIMED_OUT)) |
                           (timed_out ? (wait ? UST_F_WAIT_TIMED_OUT : UST_F_VALIDATION_TIMED_OUT) : 0u);
        if (g != f) flags[i] = g;
      }
    }
    const unsigned k = __popc(cbits);
    if (__any_sync(kFull, k != 0)) {
      unsigned incl = k;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned u = __shfl_up_sync(kFull, incl, o);
        if (lane >= o) incl += u;
      }
      unsigned base = 0;
      if (lane == 31) base = atomicAdd(&n_cand, incl);
      unsigned pos = __shfl_sync(kFull, base, 31) + incl - k;
      while (cbits) {
        const int j = __ffs(cbits) - 1;
        cbits &= cbits - 1;
        mine[pos++] = it16 + 16u * (uint32_t)t + (uint32_t)j;
      }
    }
  }
  __syncthreads();
  if (t == 0) cand_count[blockIdx.x] = n_cand;
}

// The next deadline of a clocked call (include/ust.h, ust_next_deadline), behind its verification kernel: every candidate
// the clock kernel listed is evaluated twice with the functions of the verification kernel - node_entry on the summary byte
// the call used, apply_abort with the call's abort point (from the counters it wrote) - once as the call saw it and once
// with its timed-out bit set. A validation-required node in validation mode asks validation_summary again for its byte,
// with the bit set (its pods walked again up to the first one that is not ready). The smallest d of the nodes whose entry
// differs: warp reduction, one shared-memory atomic per warp, one global atomic per CTA. CTA b reads the list of the clock
// kernel's CTA b. `validation`: as for ust_pod_summary_kernel.
// node index of a candidate offset of CTA b (ust_clock_kernel's iteration order, the same grid)
__device__ __forceinline__ long long cand_node(uint32_t off, long long b) {
  const long long it = off / (16 * kThreads), rem = off % (16 * kThreads);
  return ((long long)b * kThreads + it * (long long)gridDim.x * kThreads) * 16 + rem;
}

__global__ void __launch_bounds__(kThreads) ust_deadline_kernel(const __grid_constant__ UstParams P, const uint32_t* __restrict__ cand,
                                                                const unsigned int* __restrict__ cand_count, long long region,
                                                                const long long* __restrict__ start, long long wait_timeout,
                                                                int validation, long long n_pods, unsigned long long* __restrict__ deadline) {
  __shared__ Shared S;
  __shared__ unsigned long long cta_min;
  const int t = threadIdx.x;
  const unsigned cnt = __ldg(cand_count + blockIdx.x);
  if (cnt == 0) return;  // (CTA-uniform)
  for (int k = t; k < (int)UST_LUT_WORDS; k += kThreads) S.lut[k] = __ldg(P.lut + k);  // the table, then the meta pairs behind it
  if (t == 0) {
    const long long pass = P.out->error_pass;  // the call's abort, as the verification kernel reported it (one GPU: node offset 0,
                                               // ust_next_deadline refuses more than one rank)
    S.abort_key = pass >= 0 ? UST_KEY(pass, (unsigned long long)(P.out->error_index + 1)) : ~0ull;
    cta_min = ~0ull;
  }
  __syncthreads();
  const uint32_t* mine = cand + (long long)blockIdx.x * region;
  const unsigned char* bytes = reinterpret_cast<const unsigned char*>(P.pod_flags);
  // a node's entry as the evaluation forms it from its flags word and summary byte (general_step; neither state reads the grant)
  auto entry = [&](uint32_t hb, uint32_t f, uint32_t ps, int rev, uint32_t di, long long i) {
    uint32_t extra = 0u;
    fold_podsum(ps, f, extra);
    return apply_abort(S, node_entry(P, S, false, hb, f, rev, di, extra), hb, i);
  };
  unsigned long long best = ~0ull;  // the smallest d, with its sign bit flipped (unsigned order = signed order)
  for (unsigned q = t; q < cnt; q += kThreads) {
    const long long i = cand_node(__ldg(mine + q), blockIdx.x);
    const uint32_t hb = __ldg(P.hot + i), f = __ldg(P.flags + i), di = (uint32_t)__ldg(P.ds_idx + i);
    const int rev = __ldg(P.pod_rev + i);
    const uint32_t ps = P.podsum ? __ldg(P.podsum + i) : 0u;
    const bool wait = (hb & UST_HOT_STATE_MASK) == UST_STATE_WAIT_FOR_JOBS_REQUIRED;
    const long long d = ust_deadline(__ldg(start + i), wait ? wait_timeout : (long long)UST_VALIDATION_TIMEOUT_SECONDS);
    const uint32_t f1 = f | (wait ? UST_F_WAIT_TIMED_OUT : UST_F_VALIDATION_TIMED_OUT);
    uint32_t ps1 = ps;
    if (!wait && P.podsum && validation)
      ps1 = validation_summary(P.pod_flags, bytes, 2 * n_pods, __ldg(P.pod_off + i), __ldg(P.pod_off + i + 1), f1, validation == kValWalk);
    if (entry(hb, f, ps, rev, di, i) != entry(hb, f1, ps1, rev, di, i)) {
      const unsigned long long key = (unsigned long long)d ^ (1ull << 63);
      best = key < best ? key : best;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long u = __shfl_xor_sync(kFull, best, o);
    best = u < best ? u : best;
  }
  if ((t & 31) == 0 && best != ~0ull) atomicMin(&cta_min, best);
  __syncthreads();
  if (t == 0 && cta_min != ~0ull) atomicMin(deadline, cta_min);
}

// The resident driver-pod list of ust_build_state_delta in a new order: state byte, owner UID and previous owner index of
// every pod that stays, from its old position; a joined pod takes its inserted values and previous owner index INT32_MIN,
// which no owner index equals, so the diff reports it. 21 B read + 21 B written per pod.
__global__ void __launch_bounds__(kThreads) ust_build_state_reorder_kernel(long long n, long long n_runs, const long long* __restrict__ run_off,
                                                                           const long long* __restrict__ run_src,
                                                                           const uint8_t* __restrict__ ins_hot, const ulonglong2* __restrict__ ins_uid,
                                                                           const uint8_t* __restrict__ hot, const ulonglong2* __restrict__ uid,
                                                                           const int32_t* __restrict__ prev, uint8_t* __restrict__ o_hot,
                                                                           ulonglong2* __restrict__ o_uid, int32_t* __restrict__ o_prev) {
  gather_runs(n, n_runs, run_off, run_src, [=](long long p, long long src, long long k) {
    if (src >= 0) {
      const long long i = src + k;
      o_hot[p] = __ldcs(hot + i); o_uid[p] = __ldcs(uid + i); o_prev[p] = __ldcs(prev + i);
    } else {
      const long long i = -1 - src + k;
      o_hot[p] = __ldg(ins_hot + i); o_uid[p] = __ldg(ins_uid + i); o_prev[p] = INT32_MIN;
    }
  });
}

// Replacement pod lists of the resident pod-list snapshot (ust_apply_state_delta_pods). The host has checked the lists
// (node_idx strictly increasing, offsets well formed) and knows every replaced list's old length, so it picks the path:
//   every list keeps its length: ust_pods_scatter_kernel copies each new list over the old one, in place;
//   some length changes: ust_pods_runs_kernel builds the run table of the new CSR, ust_pods_relayout_kernel writes the
//   new offsets and pod_flags into the second CSR pair in one pass.
// shift[k] (host-computed, n_lists + 1 entries) = sum over j < k of (new length - old length) of list j: node i's new
// offset is off[i] + shift[#{k : node_idx[k] < i}].
constexpr int kRelayTile = 8192;                   // new pod positions per CTA: 32 per thread, four 16-byte stores
constexpr int kRelayRuns = 2048;                   // runs a CTA stages in shared memory (more: it searches them in global memory)
constexpr int kOffTile = 2048;                     // offsets per CTA

// One warp per list: 2 B read and written per pod of the replaced lists, 12 B per list.
__global__ void __launch_bounds__(kThreads) ust_pods_scatter_kernel(long long n_lists, const long long* __restrict__ node_idx,
                                                                    const int32_t* __restrict__ new_off,
                                                                    const uint16_t* __restrict__ new_flags,
                                                                    const int32_t* __restrict__ off, uint16_t* __restrict__ flags) {
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * kWarps;
  for (long long k = (long long)blockIdx.x * kWarps + (threadIdx.x >> 5); k < n_lists; k += warps) {
    const int s0 = __ldg(new_off + k), s1 = __ldg(new_off + k + 1);
    const int d = __ldg(off + __ldg(node_idx + k)) - s0;
    for (int p = s0 + lane; p < s1; p += 32) flags[d + p] = __ldg(new_flags + p);
  }
}

// The new CSR as 2 n_lists + 1 runs of new pod positions [run_start[r], run_start[r + 1]) (run_start[2 n_lists + 1] =
// new_total), in the encoding of gather_pods: run 2k, the unchanged nodes between list k - 1 and list k, old pods from
// run_src[2k] on; run 2k + 1, new list k, run_src[2k + 1] = -1 - new_off[k]. Runs may be empty.
__global__ void __launch_bounds__(kThreads) ust_pods_runs_kernel(long long n_lists, const long long* __restrict__ node_idx,
                                                                 const int32_t* __restrict__ new_off, const int32_t* __restrict__ shift,
                                                                 const int32_t* __restrict__ off, int new_total,
                                                                 int32_t* __restrict__ run_start, int32_t* __restrict__ run_src) {
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long k = (long long)blockIdx.x * kThreads + threadIdx.x; k <= n_lists; k += stride) {
    const int prev_end = k ? __ldg(off + __ldg(node_idx + k - 1) + 1) : 0;  // old end of list k - 1
    const int d = __ldg(shift + k);
    run_start[2 * k] = prev_end + d;
    run_src[2 * k] = prev_end;
    if (k < n_lists) {
      run_start[2 * k + 1] = __ldg(off + __ldg(node_idx + k)) + d;
      run_src[2 * k + 1] = -1 - __ldg(new_off + k);
    } else {
      run_start[2 * k + 1] = new_total;
    }
  }
}

// Eight pods from src[s], s any position: two aligned 16-byte loads, shifted by s & 7 pods (the buffers hold 8 pods
// of padding past their last pod, so the second load stays inside them).
__device__ __forceinline__ uint4 pods8_at(const uint16_t* __restrict__ src, int s) {
  const uint4* a = reinterpret_cast<const uint4*>(src + (s & ~7));
  const uint4 lo = __ldg(a), hi = __ldg(a + 1);
  uint32_t v0 = lo.x, v1 = lo.y, v2 = lo.z, v3 = lo.w, v4 = hi.x, v5 = hi.y, v6 = hi.z, v7 = hi.w;
  const int w = (s & 7) >> 1;  // whole words
  if (w & 2) { v0 = v2; v1 = v3; v2 = v4; v3 = v5; v4 = v6; v5 = v7; }
  if (w & 1) { v0 = v1; v1 = v2; v2 = v3; v3 = v4; v4 = v5; }
  const unsigned sh = (s & 1) * 16u;
  return make_uint4(__funnelshift_r(v0, v1, sh), __funnelshift_r(v1, v2, sh), __funnelshift_r(v2, v3, sh), __funnelshift_r(v3, v4, sh));
}

// The runs of a pod tile, staged in shared memory by gather_pods
struct PodRunsSmem {
  int32_t start[kRelayRuns + 1];
  int32_t src[kRelayRuns];
};

// The pod half of ust_pods_relayout_kernel and ust_pods_reorder_kernel: new pod_flags [q0, q1), tile blockIdx.x of
// kRelayTile positions, from n_runs runs. Run r covers new positions [run_start[r], run_start[r + 1]) and reads old pods
// run_src[r], run_src[r] + 1, ... (run_src >= 0) or new-list pods -1 - run_src[r], ... (run_src < 0). The CTA finds its
// tile's runs once, by binary search, and stages them in shared memory (a tile that meets more than kRelayRuns of them,
// empty ones included, searches them in global memory instead). A chunk of 8 pods inside one run is one shifted 16-byte
// copy (pods8_at), a chunk across runs goes pod by pod; 16-byte stores.
__device__ __forceinline__ void gather_pods(long long n_runs, const int32_t* __restrict__ run_start, const int32_t* __restrict__ run_src,
                                            const uint16_t* __restrict__ flags, const uint16_t* __restrict__ new_flags,
                                            uint16_t* __restrict__ o_flags, int new_total, PodRunsSmem& sm, long long (&bounds)[2]) {
  const int t = threadIdx.x;
  const int q0 = blockIdx.x * kRelayTile;
  const int q1 = q0 + kRelayTile < new_total ? q0 + kRelayTile : new_total;
  if (t < 2) bounds[t] = last_le(run_start, n_runs, t ? q1 - 1 : q0);  // the last run that starts at or before q0 / q1 - 1
  __syncthreads();
  const long long r0 = bounds[0];
  const int nr = (int)(bounds[1] - r0 + 1);
  const bool staged = nr <= kRelayRuns;  // empty runs are not bounded by the tile
  if (staged) {
    for (int j = t; j <= nr; j += kThreads) sm.start[j] = __ldg(run_start + r0 + j);
    for (int j = t; j < nr; j += kThreads) sm.src[j] = __ldg(run_src + r0 + j);
  }
  __syncthreads();
  const int32_t* S = staged ? sm.start : run_start + r0;
  const int32_t* R = staged ? sm.src : run_src + r0;
  const int chunks = (q1 - q0 + 7) >> 3;
#pragma unroll 2
  for (int c = t; c < chunks; c += kThreads) {
    const int q = q0 + 8 * c;
    int r = last_le_from(S, 0, nr, q);  // the run that holds q
    uint4 v;
    if (q + 8 <= S[r + 1] && q + 8 <= new_total) {  // the chunk lies in one run: one shifted 16-byte copy
      const int src = R[r];
      v = pods8_at(src >= 0 ? flags : new_flags, (src >= 0 ? src : -1 - src) + (q - S[r]));
    } else {  // it straddles runs (or the end of the array): pod by pod
      uint32_t w[4] = {0u, 0u, 0u, 0u};
#pragma unroll
      for (int e = 0; e < 8; e++) {
        const int p = q + e;
        if (p >= new_total) break;
        while (S[r + 1] <= p) r++;
        const int src = R[r];
        const uint16_t x = __ldg((src >= 0 ? flags : new_flags) + (src >= 0 ? src : -1 - src) + (p - S[r]));
        w[e >> 1] |= (uint32_t)x << (16 * (e & 1));
      }
      v = make_uint4(w[0], w[1], w[2], w[3]);
    }
    *reinterpret_cast<uint4*>(o_flags + q) = v;
  }
}

union RelayoutSmem {
  PodRunsSmem pods;
  struct { long long idx[kOffTile]; int32_t shift[kOffTile + 1]; } offs;
};

// CTAs [0, pod_ctas) gather the new pod_flags by tiles of kRelayTile new positions; the CTAs after them write the n + 1
// new offsets by tiles of kOffTile nodes. Both search their tile's runs once and stage them in shared memory.
// 2 B read + 2 B written per pod, 8 B per node, each new list once.
__global__ void __launch_bounds__(kThreads) ust_pods_relayout_kernel(long long n, long long n_lists, const long long* __restrict__ node_idx,
                                                                     const int32_t* __restrict__ shift, const int32_t* __restrict__ off,
                                                                     int32_t* __restrict__ o_off, const int32_t* __restrict__ run_start,
                                                                     const int32_t* __restrict__ run_src, const uint16_t* __restrict__ flags,
                                                                     const uint16_t* __restrict__ new_flags, uint16_t* __restrict__ o_flags,
                                                                     int new_total, int pod_ctas) {
  __shared__ __align__(16) RelayoutSmem sm;
  __shared__ long long s_bounds[2];
  const int t = threadIdx.x;
  if ((int)blockIdx.x >= pod_ctas) {
    // ---- offsets: node i takes shift[c], c = #{k : node_idx[k] < i}
    const long long b0 = (long long)(blockIdx.x - pod_ctas) * kOffTile;
    const long long b1 = b0 + kOffTile < n + 1 ? b0 + kOffTile : n + 1;
    if (t < 2) s_bounds[t] = splice_lower_bound(node_idx, n_lists, t ? b1 : b0);
    __syncthreads();
    const long long c0 = s_bounds[0];
    const int nc = (int)(s_bounds[1] - c0);  // node_idx is strictly increasing: at most kOffTile of them fall in [b0, b1)
    for (int j = t; j < nc; j += kThreads) sm.offs.idx[j] = __ldg(node_idx + c0 + j);
    for (int j = t; j <= nc; j += kThreads) sm.offs.shift[j] = __ldg(shift + c0 + j);
    __syncthreads();
    for (int j = t; j < (int)(b1 - b0); j += kThreads) {
      const long long i = b0 + j;
      int lo = 0, hi = nc;  // first staged k with node_idx[k] >= i
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (sm.offs.idx[mid] < i) lo = mid + 1; else hi = mid;
      }
      o_off[i] = __ldcs(off + i) + sm.offs.shift[lo];
    }
    return;
  }
  // ---- pods
  gather_pods(2 * n_lists + 1, run_start, run_src, flags, new_flags, o_flags, new_total, sm.pods, s_bounds);
}

// The pod-list CSR of the resident pod-list snapshot in a new node order, with replaced and inserted lists
// (ust_apply_state_delta_pods_reorder). The host cuts the new snapshot into S segments, each a stretch of consecutive
// old nodes or one new list: segment s covers new nodes [seg_node[s], seg_node[s + 1]) and new pods [pod_start[s],
// pod_start[s + 1]) (seg_node[S] = n, pod_start[S] = new_total), read from old nodes seg_src[s], seg_src[s] + 1, ...
// (seg_src >= 0) or from new list -1 - seg_src[s]. ust_pods_reorder_runs_kernel finds each segment's first source pod
// (pod_src: old pod off[seg_src], or -1 - new_off[k] for list k); ust_pods_reorder_kernel then writes the n + 1 new offsets
// and the new pod_flags into the second CSR pair in one pass, as ust_pods_relayout_kernel does.
constexpr int kReorderOffTile = 1024;  // offsets per CTA: a full shuffle puts one segment on every node

__global__ void __launch_bounds__(kThreads) ust_pods_reorder_runs_kernel(long long n_segs, const long long* __restrict__ seg_src,
                                                                         const int32_t* __restrict__ off,
                                                                         const int32_t* __restrict__ new_off,
                                                                         int32_t* __restrict__ pod_src) {
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long s = (long long)blockIdx.x * kThreads + threadIdx.x; s < n_segs; s += stride) {
    const long long src = __ldg(seg_src + s);
    pod_src[s] = src >= 0 ? __ldg(off + src) : -1 - __ldg(new_off + (-1 - src));
  }
}

union PodsReorderSmem {
  PodRunsSmem pods;
  struct { long long node[kReorderOffTile]; long long src[kReorderOffTile]; int32_t start[kReorderOffTile]; int32_t psrc[kReorderOffTile]; } offs;
};

// CTAs [0, pod_ctas) gather the new pod_flags by tiles of kRelayTile new positions; the CTAs after them write the n + 1
// new offsets by tiles of kReorderOffTile nodes. Both search their tile's segments once and stage them in shared memory.
// 2 B read + 2 B written per pod, 8 B per node, a few dozen bytes per segment.
__global__ void __launch_bounds__(kThreads) ust_pods_reorder_kernel(long long n, long long n_segs, const long long* __restrict__ seg_node,
                                                                    const long long* __restrict__ seg_src,
                                                                    const int32_t* __restrict__ pod_start,
                                                                    const int32_t* __restrict__ pod_src, const int32_t* __restrict__ off,
                                                                    const uint16_t* __restrict__ flags, const uint16_t* __restrict__ new_flags,
                                                                    int32_t* __restrict__ o_off, uint16_t* __restrict__ o_flags,
                                                                    int new_total, int pod_ctas) {
  __shared__ __align__(16) PodsReorderSmem sm;
  __shared__ long long s_bounds[2];
  const int t = threadIdx.x;
  if ((int)blockIdx.x >= pod_ctas) {
    // ---- offsets: node i of segment s takes pod_start[s] + off[seg_src[s] + i - seg_node[s]] - pod_src[s] (old nodes) or
    // pod_start[s] (a new list); node n takes new_total
    const long long b0 = (long long)(blockIdx.x - pod_ctas) * kReorderOffTile;
    const long long b1 = b0 + kReorderOffTile < n ? b0 + kReorderOffTile : n;  // nodes [b0, b1) of [0, n)
    if (b1 > b0) {
      if (t < 2) s_bounds[t] = last_le(seg_node, n_segs, t ? b1 - 1 : b0);  // the last segment that starts at or before b0 / b1 - 1
      __syncthreads();
      const long long s0 = s_bounds[0];
      const int ns = (int)(s_bounds[1] - s0 + 1);  // every segment holds a node: at most kReorderOffTile of them
      for (int j = t; j < ns; j += kThreads) {
        sm.offs.node[j] = __ldg(seg_node + s0 + j);
        sm.offs.src[j] = __ldg(seg_src + s0 + j);
        sm.offs.start[j] = __ldg(pod_start + s0 + j);
        sm.offs.psrc[j] = __ldg(pod_src + s0 + j);
      }
      __syncthreads();
      int r = 0;
      for (int j = t; j < (int)(b1 - b0); j += kThreads) {
        const long long i = b0 + j;
        r = last_le_from(sm.offs.node, r, ns, i);
        const long long src = sm.offs.src[r];
        o_off[i] = src >= 0 ? sm.offs.start[r] + (__ldcs(off + src + (i - sm.offs.node[r])) - sm.offs.psrc[r]) : sm.offs.start[r];
      }
    }
    if (b0 <= n && n < b0 + kReorderOffTile && t == 0) o_off[n] = new_total;
    return;
  }
  // ---- pods: the segments are the runs of gather_pods
  gather_pods(n_segs, pod_start, pod_src, flags, new_flags, o_flags, new_total, sm.pods, s_bounds);
}

// Rollout simulation (SURVEY 8f.3): the state feedback between two reconciles. Untimed (sp.timed == 0): "ideal actuators" - every call
// the reference makes through its providers takes effect, every asynchronous actuator succeeds, and whatever a node
// is waiting for (jobs, pod readiness, validation) has happened by the next reconcile. One streaming pass, in place:
// 13 B read + up to 9 B written per node.
//   state   <- actuator_outcome when the pass scheduled an asynchronous actuator (pod_manager.go:393-403,
//              drain_manager.go:111-139), else next_state (NodeUpgradeStateProvider.ChangeNodeUpgradeState)
//   annotations per action bit (ChangeNodeUpgradeAnnotation, upgrade_suit_test.go:121-130)
//   CORDON / UNCORDON -> Spec.Unschedulable (cordon_manager.go:40-47)
//   RESTART_DRIVER_POD -> the DaemonSet controller recreates the pod at the current revision and it becomes ready;
//              an orphaned pod is not recreated: the node leaves the snapshot (no driver pod to list)
//   still waiting after the pass: wait-for-jobs with running pods -> the jobs finish; pod-restart with a synced pod
//              that is not ready -> it becomes ready; validation-required -> the validation pod becomes ready
__global__ void __launch_bounds__(kThreads) ust_feedback_kernel(long long n, uint8_t* hot, uint32_t* flags, int32_t* pod_rev,
                                                                const int32_t* __restrict__ ds_idx, int n_ds,
                                                                const int32_t* __restrict__ ds_rev,
                                                                const uint8_t* __restrict__ next, const uint16_t* __restrict__ actions,
                                                                const uint8_t* __restrict__ outcome, const ust_counters* step,
                                                                const UstSimParams sp, int32_t* entered, int32_t* wait_start,
                                                                int32_t* valid_start) {
  if (step->error_code != UST_OK) return;  // the reconcile returned an error: nothing it decided is fed back
  const long long stride = (long long)gridDim.x * kThreads;
  const long long now = sp.now, now_next = sp.now + sp.dt;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += stride) {
    unsigned b = hot[i];
    const unsigned s = b & 15u;
    if (s >= UST_STATE_OTHER) continue;  // other label values / not in the snapshot: never processed
    uint32_t f = flags[i];
    const unsigned a = actions[i];
    const unsigned oc = outcome[i];
    unsigned ns = next[i];
    if ((a & (UST_A_SCHEDULE_WAIT_CHECK | UST_A_SCHEDULE_POD_EVICTION | UST_A_SCHEDULE_DRAIN)) && oc != UST_OUTCOME_NONE) ns = oc;
    if (a & UST_A_CLEAR_UPGRADE_REQUESTED) f &= ~UST_F_UPGRADE_REQUESTED;
    if (a & UST_A_SET_INITIAL_STATE_ANNO) f |= UST_F_INITIAL_STATE_ANNO;
    if (a & UST_A_CLEAR_INITIAL_STATE_ANNO) f &= ~UST_F_INITIAL_STATE_ANNO;
    if (a & UST_A_CORDON) b |= UST_HOT_UNSCHEDULABLE;
    if (a & UST_A_UNCORDON) b &= ~UST_HOT_UNSCHEDULABLE;
    if (a & UST_A_UNBLOCK_SAFE_LOAD) f &= ~UST_F_SAFE_LOAD;
    if (a & UST_A_SET_WAIT_START) f |= UST_F_WAIT_START_ANNO;
    if (a & UST_A_CLEAR_WAIT_START) f &= ~(UST_F_WAIT_START_ANNO | UST_F_WAIT_TIMED_OUT | UST_F_WAIT_START_INVALID);
    // requestor mode (upgrade_requestor.go:277-319, :454-488): the annotation and the NodeMaintenance object
    if (a & UST_A_REQUESTOR_ANNO_CHANGE) f = s == UST_STATE_UPGRADE_REQUIRED ? (f | UST_F_REQUESTOR_MODE) : (f & ~UST_F_REQUESTOR_MODE);
    if (a & UST_A_NM_CREATE_OR_DELETE) {
      if (s == UST_STATE_UPGRADE_REQUIRED) {
        f |= UST_F_NM_PRESENT;
      } else {  // the object goes, and with it the maintenance operator's cordon
        f &= ~(UST_F_NM_PRESENT | UST_F_NM_READY);
        b &= ~UST_HOT_UNSCHEDULABLE;
      }
    }
    int rev = pod_rev[i];
    if (a & UST_A_RESTART_DRIVER_POD) {
      const int d = ds_idx[i];
      if ((f & UST_F_POD_ORPHANED) || d < 0 || d >= n_ds) {
        ns = UST_STATE_EXCLUDED;
      } else {
        rev = ds_rev[d];
        f = (f | UST_F_POD_READY) & ~(UST_F_POD_FAILING | UST_F_POD_TERMINATING);
      }
    }
    int ent = 0, ws = 0, vs = 0;
    if (sp.timed) {
      ent = entered[i]; ws = wait_start[i]; vs = valid_start[i];
      if (a & UST_A_SET_WAIT_START) ws = (int)now;                 // annotation = currentTime (pod_manager.go:339)
      if (a & UST_A_CLEAR_WAIT_START) ws = kSimNone;
      // Validate() of a node whose validation pod is not ready runs handleTimeout (validation_manager.go:139-175)
      if (s == UST_STATE_VALIDATION_REQUIRED && ns == UST_STATE_VALIDATION_REQUIRED && !(f & UST_F_VALIDATION_DONE)) {
        if (vs == kSimNone) vs = (int)now;
        else if (ust_timed_out(now, vs, sp.validation_timeout)) { ns = UST_STATE_FAILED; vs = kSimNone; }
      }
      if (ns != UST_STATE_VALIDATION_REQUIRED) vs = kSimNone;      // the annotation is removed once the pod is ready (:104-110)
      if (ns != s) ent = (int)now;
    }
    if (ns == UST_STATE_WAIT_FOR_JOBS_REQUIRED) {
      if (!sp.timed) f &= ~UST_F_WAIT_PODS_RUNNING;
      else {
        if (ns != s) f = sp.job_seconds > 0 ? (f | UST_F_WAIT_PODS_RUNNING) : (f & ~UST_F_WAIT_PODS_RUNNING);
        if (now_next >= (long long)ent + sp.job_seconds) f &= ~UST_F_WAIT_PODS_RUNNING;
        const bool timed_out = ws != kSimNone && ust_timed_out(now_next, ws, sp.wait_timeout);
        f = timed_out ? (f | UST_F_WAIT_TIMED_OUT) : (f & ~UST_F_WAIT_TIMED_OUT);
      }
    }
    if (ns == UST_STATE_POD_RESTART_REQUIRED) {
      f &= ~UST_F_POD_TERMINATING;
      if (!(f & UST_F_POD_FAILING)) f |= UST_F_POD_READY;
    }
    if (ns == UST_STATE_VALIDATION_REQUIRED) {
      if (!sp.timed) f |= UST_F_VALIDATION_DONE;
      else {
        const bool ready = sp.validation_seconds >= 0 && now_next >= (long long)ent + sp.validation_seconds;
        f = ready ? (f | UST_F_VALIDATION_DONE) : (f & ~UST_F_VALIDATION_DONE);
      }
    }
    if (ns == UST_STATE_NODE_MAINTENANCE_REQUIRED && (f & UST_F_NM_PRESENT)) {
      // the maintenance operator: cordon + drain, then Ready (maintenance_seconds after the object was created)
      const bool ready = !sp.timed || now_next >= (long long)ent + sp.maintenance_seconds;
      if (ready) { f |= UST_F_NM_READY; b |= UST_HOT_UNSCHEDULABLE; }
    }
    hot[i] = (uint8_t)((b & 0xF0u) | (ns & 15u));
    flags[i] = f;
    pod_rev[i] = rev;
    if (sp.timed) { entered[i] = ent; wait_start[i] = ws; valid_start[i] = vs; }
  }
}

// the per-node clocks of a timed simulation at time 0: every node "entered" its state then; a wait-start annotation that
// is already there started then, or - when the snapshot says it has timed out - long ago
__global__ void __launch_bounds__(kThreads) ust_sim_init_kernel(long long n, const uint32_t* __restrict__ flags, int32_t* entered,
                                                                int32_t* wait_start, int32_t* valid_start) {
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += stride) {
    const uint32_t f = flags[i];
    entered[i] = 0;
    wait_start[i] = !(f & UST_F_WAIT_START_ANNO) ? kSimNone : ((f & UST_F_WAIT_TIMED_OUT) ? kSimLongAgo : 0);
    valid_start[i] = kSimNone;
  }
}

// Packed host format (ust_apply_state_packed): the interned pod revision travels as uint16 and the DaemonSet index
// as int8 over PCIe; this widens a range of them into the int32 arrays the streaming pass reads. 3 B read + 8 B
// written per node, once per upload segment.
__global__ void __launch_bounds__(kThreads) ust_widen_kernel(long long n, const uint16_t* __restrict__ rev16,
                                                             const int8_t* __restrict__ ds8, int32_t* __restrict__ rev_out,
                                                             int32_t* __restrict__ ds_out) {
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += stride) {
    rev_out[i] = (int32_t)__ldcs(rev16 + i);
    ds_out[i] = (int32_t)__ldcs(ds8 + i);
  }
}
// Sparse outputs of a delta call (SURVEY 8f.2): the nodes whose (next_state, actions) differ from the previous call's,
// compacted in node order. Three launches: per-block counts, a one-CTA scan of the block counts, the ordered write.
// 6 B/node read twice; the alternative is 3 B/node over PCIe. OUTCOME (ust_apply_state_delta_pods): actuator_outcome
// is compared and returned too, 8 B/node read twice.
constexpr int kDiffBlock = 4096;  // nodes per CTA: 16 per thread
template <bool OUTCOME>
__device__ __forceinline__ unsigned diff_mask16(const uint8_t* next, const uint16_t* act, const uint8_t* oc, const uint8_t* pnext,
                                                const uint16_t* pact, const uint8_t* poc, long long i0, long long n) {
  unsigned m = 0;
  if (i0 + 16 <= n) {
    const uint4 a = __ldcs(reinterpret_cast<const uint4*>(next + i0)), b = __ldcs(reinterpret_cast<const uint4*>(pnext + i0));
    const uint4 c0 = __ldcs(reinterpret_cast<const uint4*>(act + i0)), c1 = __ldcs(reinterpret_cast<const uint4*>(act + i0 + 8));
    const uint4 d0 = __ldcs(reinterpret_cast<const uint4*>(pact + i0)), d1 = __ldcs(reinterpret_cast<const uint4*>(pact + i0 + 8));
    uint32_t x[4] = {a.x ^ b.x, a.y ^ b.y, a.z ^ b.z, a.w ^ b.w};
    if constexpr (OUTCOME) {  // an outcome byte that differs counts like a next_state byte that differs
      const uint4 e = __ldcs(reinterpret_cast<const uint4*>(oc + i0)), f = __ldcs(reinterpret_cast<const uint4*>(poc + i0));
      x[0] |= e.x ^ f.x; x[1] |= e.y ^ f.y; x[2] |= e.z ^ f.z; x[3] |= e.w ^ f.w;
    }
    const uint32_t y[8] = {c0.x ^ d0.x, c0.y ^ d0.y, c0.z ^ d0.z, c0.w ^ d0.w, c1.x ^ d1.x, c1.y ^ d1.y, c1.z ^ d1.z, c1.w ^ d1.w};
#pragma unroll
    for (int k = 0; k < 16; k++) {
      const bool dn = ((x[k >> 2] >> (8 * (k & 3))) & 0xFFu) != 0;
      const bool da = ((y[k >> 1] >> (16 * (k & 1))) & 0xFFFFu) != 0;
      m |= (dn || da ? 1u : 0u) << k;
    }
  } else {
    for (int k = 0; k < 16; k++)
      if (i0 + k < n && (next[i0 + k] != pnext[i0 + k] || act[i0 + k] != pact[i0 + k] || (OUTCOME && oc[i0 + k] != poc[i0 + k])))
        m |= 1u << k;
  }
  return m;
}
template <bool OUTCOME>
__global__ void __launch_bounds__(kThreads) ust_diff_count_kernel(long long n, const uint8_t* __restrict__ next, const uint16_t* __restrict__ act,
                                                                  const uint8_t* __restrict__ oc, const uint8_t* __restrict__ pnext,
                                                                  const uint16_t* __restrict__ pact, const uint8_t* __restrict__ poc,
                                                                  unsigned int* __restrict__ block_count) {
  __shared__ unsigned int tot;
  if (threadIdx.x == 0) tot = 0;
  __syncthreads();
  const long long i0 = (long long)blockIdx.x * kDiffBlock + 16 * threadIdx.x;
  const unsigned c = i0 < n ? __popc(diff_mask16<OUTCOME>(next, act, oc, pnext, pact, poc, i0, n)) : 0u;
  cta_sum(c, tot);
  if (threadIdx.x == 0) block_count[blockIdx.x] = tot;
}
// exclusive scan of the block counts in place (one CTA); total -> *n_out
__global__ void __launch_bounds__(1024) ust_diff_scan_kernel(int blocks, unsigned int* block_count, long long* n_out) {
  __shared__ unsigned long long part[32];
  __shared__ unsigned long long carry;
  const int t = threadIdx.x;
  if (t == 0) carry = 0;
  __syncthreads();
  for (int b0 = 0; b0 < blocks; b0 += 1024) {
    const int b = b0 + t;
    const unsigned long long v = b < blocks ? block_count[b] : 0ull;
    unsigned long long incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long u = __shfl_up_sync(kFull, incl, o);
      if ((t & 31) >= o) incl += u;
    }
    if ((t & 31) == 31) part[t >> 5] = incl;
    __syncthreads();
    unsigned long long before = carry, tot = 0;
    for (int w = 0; w < 32; w++) { if (w < (t >> 5)) before += part[w]; tot += part[w]; }
    // offsets fit 32 bits per launch range: the API caps a sparse call at 2^31 changed outputs
    if (b < blocks) block_count[b] = (unsigned int)(before + incl - v);
    __syncthreads();
    if (t == 0) carry += tot;
    __syncthreads();
  }
  if (t == 0) *n_out = (long long)carry;
}
template <bool OUTCOME>
__global__ void __launch_bounds__(kThreads) ust_diff_write_kernel(long long n, const uint8_t* __restrict__ next, const uint16_t* __restrict__ act,
                                                                  const uint8_t* __restrict__ oc, const uint8_t* __restrict__ pnext,
                                                                  const uint16_t* __restrict__ pact, const uint8_t* __restrict__ poc,
                                                                  const unsigned int* __restrict__ block_off, long long cap,
                                                                  long long* __restrict__ out_idx, uint8_t* __restrict__ out_next,
                                                                  uint16_t* __restrict__ out_act, uint8_t* __restrict__ out_oc) {
  const int t = threadIdx.x;
  const long long i0 = (long long)blockIdx.x * kDiffBlock + 16 * t;
  const unsigned m = i0 < n ? diff_mask16<OUTCOME>(next, act, oc, pnext, pact, poc, i0, n) : 0u;
  long long pos = cta_first_pos(__popc(m), block_off);
  unsigned mm = m;
  while (mm) {
    const int k = __ffs(mm) - 1;
    mm &= mm - 1;
    if (pos < cap) {
      out_idx[pos] = i0 + k;
      out_next[pos] = next[i0 + k];
      out_act[pos] = act[i0 + k];
      if constexpr (OUTCOME) out_oc[pos] = oc[i0 + k];
    }
    pos++;
  }
}

}  // namespace

int ust_launch_verify(const UstParams& p, int grid, void* stream, int pdl) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3(kVThreads);
  cfg.dynamicSmemBytes = 0;
  cfg.stream = (cudaStream_t)stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  return (int)cudaLaunchKernelEx(&cfg, ust_verify_kernel, p);
}
int ust_launch_pod_summary(long long n, int active, const uint8_t* hot, const int32_t* pod_off, const uint16_t* pod_flags,
                           long long n_pods, const uint8_t* podlut, uint8_t* podsum, const uint32_t* flags, int validation,
                           unsigned long long* errinv, int grid, void* stream) {
  if (n <= 0) return 0;
  const long long blocks = (n + kPodBlock - 1) / kPodBlock;
  if (grid > blocks) grid = (int)blocks;
  if (validation)
    ust_pod_summary_kernel<true><<<grid, kThreads, 0, (cudaStream_t)stream>>>(n, active, hot, pod_off, pod_flags, n_pods, podlut,
                                                                            podsum, flags, validation, errinv);
  else
    ust_pod_summary_kernel<false><<<grid, kThreads, 0, (cudaStream_t)stream>>>(n, active, hot, pod_off, pod_flags, n_pods, podlut,
                                                                             podsum, flags, validation, errinv);
  return (int)cudaGetLastError();
}
int ust_launch_build_state(long long n, const uint8_t* hot, const int32_t* ds_idx, int n_ds, const int32_t* ds_desired,
                           unsigned long long* ds_count, UstWorkspace* ws, ust_counters* out, int grid, void* stream) {
  ust_build_state_uid_kernel<false><<<grid, kThreads, 0, (cudaStream_t)stream>>>(n, hot, nullptr, ds_idx, n_ds, nullptr, nullptr, 8,
                                                                                 nullptr, ds_count, ws);
  ust_build_state_finish_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(n_ds, ds_desired, ds_count, ws, out);
  return (int)cudaGetLastError();
}
int ust_launch_widen(long long n, const uint16_t* rev16, const int8_t* ds8, int32_t* rev_out, int32_t* ds_out, int grid,
                     void* stream) {
  if (n <= 0) return 0;
  const long long want = (n + kThreads - 1) / kThreads;
  ust_widen_kernel<<<(unsigned)(want < grid ? want : grid), kThreads, 0, (cudaStream_t)stream>>>(n, rev16, ds8, rev_out, ds_out);
  return (int)cudaGetLastError();
}
int ust_launch_patch(long long m, const long long* idx, const uint8_t* state, const uint32_t* flags, const int32_t* pod_rev,
                     const int32_t* ds_idx, uint8_t* hot_out, uint32_t* flags_out, int32_t* rev_out, int32_t* ds_out, void* stream,
                     const long long* start, long long* start_out) {
  if (m <= 0) return 0;
  const long long grid = (m + kThreads - 1) / kThreads;
  const unsigned g = (unsigned)(grid > 65535 * 16 ? 65535 * 16 : grid);
  if (start_out)
    ust_patch_kernel<true><<<g, kThreads, 0, (cudaStream_t)stream>>>(m, idx, state, flags, pod_rev, ds_idx, hot_out, flags_out, rev_out,
                                                                    ds_out, start, start_out);
  else
    ust_patch_kernel<false><<<g, kThreads, 0, (cudaStream_t)stream>>>(m, idx, state, flags, pod_rev, ds_idx, hot_out, flags_out, rev_out,
                                                                     ds_out, nullptr, nullptr);
  return (int)cudaGetLastError();
}
UstClockGrid ust_clock_grid(long long n, int grid) {
  const long long chunks = (n + 15) / 16;
  const long long want = (chunks + kThreads - 1) / kThreads;
  UstClockGrid g;
  // enough CTAs that a CTA's candidate offsets fit 32 bits (only past ~2^31 nodes per CTA of `grid`)
  const long long least = ((chunks * 16) >> 31) + 1;
  const long long ctas = want < grid ? want : (grid > least ? grid : least);
  g.ctas = n <= 0 ? 0 : (int)ctas;
  g.region = g.ctas ? (chunks + (long long)g.ctas * kThreads - 1) / ((long long)g.ctas * kThreads) * kThreads * 16 : 0;
  return g;
}
int ust_launch_clock(long long n, const uint8_t* hot, uint32_t* flags, const long long* start, long long now, long long wait_timeout,
                     const UstClockGrid& g, uint32_t* cand, unsigned int* cand_count, unsigned long long* deadline, void* stream) {
  if (g.ctas == 0) return (int)cudaMemsetAsync(deadline, 0xFF, sizeof(unsigned long long), (cudaStream_t)stream);
  ust_clock_kernel<<<(unsigned)g.ctas, kThreads, 0, (cudaStream_t)stream>>>(n, hot, flags, start, now, wait_timeout, cand, cand_count,
                                                                           g.region, deadline);
  return (int)cudaGetLastError();
}
int ust_launch_deadline(const UstParams& p, const UstClockGrid& g, const uint32_t* cand, const unsigned int* cand_count,
                        const long long* start, long long wait_timeout, int validation, long long n_pods, unsigned long long* deadline,
                        void* stream) {
  if (g.ctas == 0) return 0;
  ust_deadline_kernel<<<(unsigned)g.ctas, kThreads, 0, (cudaStream_t)stream>>>(p, cand, cand_count, g.region, start, wait_timeout,
                                                                              validation, n_pods, deadline);
  return (int)cudaGetLastError();
}
int ust_launch_splice(long long n, long long n_rm, const long long* rm, long long n_ins, const long long* ib, const uint8_t* ins_hot,
                      const uint32_t* ins_flags, const int32_t* ins_rev, const int32_t* ins_ds, const uint8_t* hot, const uint32_t* flags,
                      const int32_t* rev, const int32_t* ds, const uint8_t* next, const uint16_t* act, uint8_t* o_hot, uint32_t* o_flags,
                      int32_t* o_rev, int32_t* o_ds, uint8_t* o_next, uint16_t* o_act, void* stream) {
  const long long grid = n / kSpliceTile + 1;  // positions 0..n
  ust_splice_kernel<<<(unsigned)grid, kThreads, 0, (cudaStream_t)stream>>>(n, n_rm, rm, n_ins, ib, ins_hot, ins_flags, ins_rev, ins_ds, hot,
                                                                           flags, rev, ds, next, act, o_hot, o_flags, o_rev, o_ds, o_next, o_act);
  return (int)cudaGetLastError();
}
int ust_launch_reorder(long long n, long long n_runs, const long long* run_off, const long long* run_src, const uint8_t* ins_hot,
                       const uint32_t* ins_flags, const int32_t* ins_rev, const int32_t* ins_ds, const uint8_t* hot, const uint32_t* flags,
                       const int32_t* rev, const int32_t* ds, const uint8_t* next, const uint16_t* act, const uint8_t* oc, uint8_t* o_hot,
                       uint32_t* o_flags, int32_t* o_rev, int32_t* o_ds, uint8_t* o_next, uint16_t* o_act, uint8_t* o_oc, void* stream,
                       const long long* ins_start, const long long* start, long long* o_start) {
  const long long grid = n > 0 ? (n + kGatherTile - 1) / kGatherTile : 1;  // one launch also for the empty snapshot
  if (oc && o_start)
    ust_reorder_kernel<true, true><<<(unsigned)grid, kThreads, 0, (cudaStream_t)stream>>>(
        n, n_runs, run_off, run_src, ins_hot, ins_flags, ins_rev, ins_ds, hot, flags, rev, ds, next, act, oc, o_hot, o_flags, o_rev, o_ds,
        o_next, o_act, o_oc, ins_start, start, o_start);
  else if (oc)
    ust_reorder_kernel<true, false><<<(unsigned)grid, kThreads, 0, (cudaStream_t)stream>>>(n, n_runs, run_off, run_src, ins_hot, ins_flags, ins_rev,
                                                                                  ins_ds, hot, flags, rev, ds, next, act, oc, o_hot, o_flags,
                                                                                  o_rev, o_ds, o_next, o_act, o_oc, nullptr, nullptr, nullptr);
  else
    ust_reorder_kernel<false, false><<<(unsigned)grid, kThreads, 0, (cudaStream_t)stream>>>(n, n_runs, run_off, run_src, ins_hot, ins_flags, ins_rev,
                                                                                   ins_ds, hot, flags, rev, ds, next, act, nullptr, o_hot,
                                                                                   o_flags, o_rev, o_ds, o_next, o_act, nullptr, nullptr, nullptr,
                                                                                   nullptr);
  return (int)cudaGetLastError();
}
int ust_launch_pods_scatter(long long n_lists, const long long* node_idx, const int32_t* new_off, const uint16_t* new_flags,
                            const int32_t* off, uint16_t* flags, int grid, void* stream) {
  const long long want = (n_lists + kWarps - 1) / kWarps;
  const int g = want < 1 ? 1 : (want < grid ? (int)want : grid);
  ust_pods_scatter_kernel<<<g, kThreads, 0, (cudaStream_t)stream>>>(n_lists, node_idx, new_off, new_flags, off, flags);
  return (int)cudaGetLastError();
}
int ust_launch_pods_relayout(long long n, long long n_lists, const long long* node_idx, const int32_t* new_off, const int32_t* shift,
                             const int32_t* off, const uint16_t* flags, const uint16_t* new_flags, int new_total, int32_t* runs,
                             int32_t* o_off, uint16_t* o_flags, int grid, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  int32_t* run_start = runs;                      // 2 n_lists + 2 entries
  int32_t* run_src = runs + 2 * n_lists + 2;      // 2 n_lists + 1 entries
  const long long want = (n_lists + 1 + kThreads - 1) / kThreads;
  ust_pods_runs_kernel<<<(unsigned)(want < grid ? want : grid), kThreads, 0, st>>>(n_lists, node_idx, new_off, shift, off, new_total,
                                                                                 run_start, run_src);
  const int pod_ctas = (new_total + kRelayTile - 1) / kRelayTile;
  const long long off_ctas = n / kOffTile + 1;    // offsets 0..n
  ust_pods_relayout_kernel<<<(unsigned)(pod_ctas + off_ctas), kThreads, 0, st>>>(n, n_lists, node_idx, shift, off, o_off, run_start, run_src,
                                                                                 flags, new_flags, o_flags, new_total, pod_ctas);
  return (int)cudaGetLastError();
}
int ust_launch_pods_reorder(long long n, long long n_segs, const long long* segs, int32_t* seg_pods, const int32_t* off,
                            const uint16_t* flags, const int32_t* new_off, const uint16_t* new_flags, int new_total, int32_t* o_off,
                            uint16_t* o_flags, int grid, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const long long* seg_node = segs;                // n_segs + 1 entries
  const long long* seg_src = segs + n_segs + 1;    // n_segs entries
  const int32_t* pod_start = seg_pods;             // n_segs + 1 entries
  int32_t* pod_src = seg_pods + n_segs + 1;        // n_segs entries
  const long long want = (n_segs + kThreads - 1) / kThreads;
  ust_pods_reorder_runs_kernel<<<(unsigned)(want < 1 ? 1 : (want < grid ? want : grid)), kThreads, 0, st>>>(n_segs, seg_src, off, new_off,
                                                                                                          pod_src);
  const int pod_ctas = (new_total + kRelayTile - 1) / kRelayTile;
  const long long off_ctas = n / kReorderOffTile + 1;  // offsets 0..n
  ust_pods_reorder_kernel<<<(unsigned)(pod_ctas + off_ctas), kThreads, 0, st>>>(n, n_segs, seg_node, seg_src, pod_start, pod_src, off, flags,
                                                                                new_flags, o_off, o_flags, new_total, pod_ctas);
  return (int)cudaGetLastError();
}
int ust_launch_feedback(long long n, uint8_t* hot, uint32_t* flags, int32_t* pod_rev, const int32_t* ds_idx, int n_ds,
                        const int32_t* ds_rev, const uint8_t* next, const uint16_t* actions, const uint8_t* outcome,
                        const ust_counters* step, const UstSimParams& sp, int32_t* entered, int32_t* wait_start,
                        int32_t* valid_start, int grid, void* stream) {
  if (n <= 0) return 0;
  ust_feedback_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(n, hot, flags, pod_rev, ds_idx, n_ds, ds_rev, next, actions, outcome, step,
                                                                   sp, entered, wait_start, valid_start);
  return (int)cudaGetLastError();
}
int ust_launch_sim_init(long long n, const uint32_t* flags, int32_t* entered, int32_t* wait_start, int32_t* valid_start, int grid,
                        void* stream) {
  if (n <= 0) return 0;
  ust_sim_init_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(n, flags, entered, wait_start, valid_start);
  return (int)cudaGetLastError();
}
int ust_launch_build_state_uids(long long n, const uint8_t* hot, const void* owner_uid, int n_ds, const void* ds_tab,
                                const int32_t* ds_tab_idx, int tab_slots, const int32_t* ds_desired, int32_t* ds_idx_out,
                                unsigned long long* ds_count, UstWorkspace* ws, ust_counters* out, int grid, void* stream) {
  ust_build_state_uid_kernel<true><<<grid, kThreads, 0, (cudaStream_t)stream>>>(
      n, hot, reinterpret_cast<const ulonglong2*>(owner_uid), nullptr, n_ds, reinterpret_cast<const ulonglong2*>(ds_tab), ds_tab_idx,
      tab_slots, ds_idx_out, ds_count, ws);
  ust_build_state_finish_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(n_ds, ds_desired, ds_count, ws, out);
  return (int)cudaGetLastError();
}
int ust_launch_diff(long long n, const uint8_t* next, const uint16_t* actions, const uint8_t* outcome, const uint8_t* prev_next,
                    const uint16_t* prev_actions, const uint8_t* prev_outcome, unsigned int* block_count, long long* n_out, long long cap,
                    long long* out_idx, uint8_t* out_next, uint16_t* out_actions, uint8_t* out_outcome, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const long long blocks = (n + kDiffBlock - 1) / kDiffBlock;
  if (blocks > 0) {
    if (outcome)
      ust_diff_count_kernel<true><<<(unsigned)blocks, kThreads, 0, st>>>(n, next, actions, outcome, prev_next, prev_actions, prev_outcome,
                                                                           block_count);
    else
      ust_diff_count_kernel<false><<<(unsigned)blocks, kThreads, 0, st>>>(n, next, actions, nullptr, prev_next, prev_actions, nullptr,
                                                                            block_count);
  }
  ust_diff_scan_kernel<<<1, 1024, 0, st>>>((int)blocks, block_count, n_out);
  if (blocks > 0) {
    if (outcome)
      ust_diff_write_kernel<true><<<(unsigned)blocks, kThreads, 0, st>>>(n, next, actions, outcome, prev_next, prev_actions, prev_outcome,
                                                                           block_count, cap, out_idx, out_next, out_actions, out_outcome);
    else
      ust_diff_write_kernel<false><<<(unsigned)blocks, kThreads, 0, st>>>(n, next, actions, nullptr, prev_next, prev_actions, nullptr,
                                                                            block_count, cap, out_idx, out_next, out_actions, nullptr);
  }
  return (int)cudaGetLastError();
}
int ust_diff_blocks(long long n) { return (int)((n + kDiffBlock - 1) / kDiffBlock); }
int ust_build_state_tiles(long long n) { return (int)((n + kBuildTile - 1) / kBuildTile); }
int ust_launch_build_state_delta(long long n, const uint8_t* hot, const void* owner_uid, int n_ds, const void* ds_tab,
                                 const int32_t* ds_tab_idx, int tab_slots, const int32_t* ds_desired, const int32_t* prev,
                                 int32_t* cur, unsigned int* tile_count, unsigned long long* ds_count, UstWorkspace* ws,
                                 ust_counters* out, int grid, void* stream) {
  const long long tiles = ust_build_state_tiles(n);
  if (grid > tiles) grid = tiles < 1 ? 1 : (int)tiles;
  ust_build_state_delta_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(
      n, hot, reinterpret_cast<const ulonglong2*>(owner_uid), n_ds, reinterpret_cast<const ulonglong2*>(ds_tab), ds_tab_idx, tab_slots,
      prev, cur, tile_count, ds_count, ws);
  ust_build_state_finish_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(n_ds, ds_desired, ds_count, ws, out);
  return (int)cudaGetLastError();
}
int ust_launch_build_state_write(long long n, const int32_t* cur, const int32_t* prev, unsigned int* tile_count, long long* n_out,
                                 long long cap, long long* out_idx, int32_t* out_ds, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const long long tiles = ust_build_state_tiles(n);
  ust_diff_scan_kernel<<<1, 1024, 0, st>>>((int)tiles, tile_count, n_out);
  if (tiles > 0)
    ust_build_state_write_kernel<<<(unsigned)tiles, kThreads, 0, st>>>(n, cur, prev, tile_count, cap, out_idx, out_ds);
  return (int)cudaGetLastError();
}
int ust_launch_build_state_reorder(long long n, long long n_runs, const long long* run_off, const long long* run_src,
                                   const uint8_t* ins_hot, const void* ins_uid, const uint8_t* hot, const void* uid,
                                   const int32_t* prev, uint8_t* o_hot, void* o_uid, int32_t* o_prev, void* stream) {
  const long long grid = n > 0 ? (n + kGatherTile - 1) / kGatherTile : 1;
  ust_build_state_reorder_kernel<<<(unsigned)grid, kThreads, 0, (cudaStream_t)stream>>>(
      n, n_runs, run_off, run_src, ins_hot, reinterpret_cast<const ulonglong2*>(ins_uid), hot, reinterpret_cast<const ulonglong2*>(uid),
      prev, o_hot, reinterpret_cast<ulonglong2*>(o_uid), o_prev);
  return (int)cudaGetLastError();
}
int ust_launch_build_state_patch(long long m, const long long* idx, const uint8_t* state, const void* uid, uint8_t* hot_out,
                                 void* uid_out, void* stream) {
  if (m <= 0) return 0;
  const long long grid = (m + kThreads - 1) / kThreads;
  ust_build_state_patch_kernel<<<(unsigned)(grid > 65535 * 16 ? 65535 * 16 : grid), kThreads, 0, (cudaStream_t)stream>>>(
      m, idx, state, reinterpret_cast<const ulonglong2*>(uid), hot_out, reinterpret_cast<ulonglong2*>(uid_out));
  return (int)cudaGetLastError();
}
