// ust_stream.cu — the streaming kernel of ApplyState for sm_90a (H100).
//
// What replaces what: one launch of ust_stream_kernel computes, for every node of the snapshot, what the
// reference's ClusterUpgradeStateManagerImpl.ApplyState (pkg/upgrade/upgrade_state.go:171-281) computes with its
// twelve sequential Process* loops: next state label and actuator-call bitmask per node, plus the cluster counters of
// common_manager.go:715-788. HBM-bound byte/integer streaming, no tensor-core work.
//
// Shape:
//   * one persistent CTA per SM, warp-specialised: warp 0 is the PRODUCER, the other warps are CONSUMERS;
//   * the snapshot is cut into tiles of UST_TILE_NODES nodes (tile order == slice order of the upgrade-required
//     bucket, upgrade_inplace.go:71). The producer's elected lane claims tiles (a strided static part, then an atomic
//     ticket so that every SM runs dry at the same moment) and moves each tile's four input columns - state (1 B),
//     flags (4), pod_rev (4), ds_idx (4) per node - into one stage of a shared-memory ring with TMA bulk copies
//     (cp.async.bulk, UBLKCP in SASS) that complete on the stage's "full" mbarrier (L2 evict-first only when the
//     inputs fit in L2). Bytes in flight are bounded by
//     the ring (UST_STAGES x 39 KiB per SM), not by registers;
//   * the per-policy transition table (4.4 KiB, built by the host: ust_lut.h) arrives the same way, once per CTA;
//   * consumer warps wait on "full", evaluate 128-node groups straight out of shared memory - one 16-byte lookup
//     indexed by the node's hot byte (table window + byte-sliced counter increments; the table is replicated per bank
//     group, so the lookup never conflicts), one lookup in the transition table - write next_state (1 B) + actions
//     (2 B) with full-width coalesced stores, and arrive on the stage's "empty" mbarrier: 16 algorithmic bytes per
//     node, each touched once;
//   * the upgrade-slot grant - the only cluster-wide dependency - is SPECULATED per tile (from the policy, or from
//     where the previous call's budget cut). No grid barrier, no fence, nobody waits: a CTA that runs out of tiles
//     adds its counters to the workspace (fire-and-forget reductions) and leaves;
//   * ust_verify_kernel (ust_kernels.cu), launched behind this kernel with programmatic dependent launch and already
//     resident when it ends, derives the slot budget (GetUpgradesAvailable, common_manager.go:748-776), checks the
//     speculation in O(1), writes the counters, and re-evaluates the tiles of a wrong speculation - in the common
//     case there are none and it returns at once.
#include "ust_common.cuh"

using namespace ustd;

namespace {

constexpr int kTile = UST_TILE_NODES;
constexpr int kStages = UST_STAGES;
constexpr int kCW = UST_CONSUMER_WARPS;
constexpr int kThreads = UST_STREAM_THREADS;
constexpr int kGroups = kTile / 128;              // 128-node groups per full tile: one per warp instruction (4 nodes per lane)
constexpr int kGPW = (kGroups + kCW - 1) / kCW;   // groups per consumer warp per full tile
static_assert(kGroups % kCW == 0 || kCW > kGroups, "consumer warps must divide the groups of a tile");
#ifndef UST_HOT_REP
#define UST_HOT_REP 8
#endif
constexpr int kHotRep = UST_HOT_REP;              // replicas of the hot-byte table: 8 = one per 16-byte bank group (16 KiB)
static_assert(kHotRep == 1 || kHotRep == 8, "hot-byte table: plain or one replica per bank group");
constexpr int kHotShift = kHotRep == 8 ? 7 : 4;   // byte offset of entry b (replica 0) = b << kHotShift
constexpr uint32_t kHotMask = 0x7Fu << kHotShift;
constexpr uint32_t kLutBytes = UST_LUT_WORDS * sizeof(uint32_t);  // table + 16 {x, y} meta pairs
static_assert(kLutBytes % 16 == 0, "bulk copies move multiples of 16 bytes");

template <bool PODS>
struct Stage {            // one tile's input columns as the TMA engine lays them down
  uint32_t flags[kTile];
  int32_t rev[kTile];
  int32_t ds[kTile];
  uint8_t hot[kTile];
  uint8_t ps[PODS ? kTile : 16];   // pod-list summary byte per node (PODS variants only)
};

template <bool PODS>
struct __align__(128) SS {
  uint32_t lut[UST_LUT_ENTRIES];   // + meta directly behind it: filled by ONE bulk copy
  uint2 meta[16];
  uint4 hotent[128 * kHotRep];     // per hot byte (bit 7 ignored): {window shift - 2 | index mask << 16, table base, sixteen 4-bit one-hot count increments}
  Stage<PODS> st[kStages];
  int dsrev[UST_DS_SMEM_MAX + 1];
  unsigned long long full[kStages], empty[kStages], lutbar;
  int tile_of[kStages];            // tile held by the stage; -1 = end of stream
  unsigned int stage_acc[kStages]; // (consumer warps done << 16) | upgrade candidates of the tile so far
  unsigned int cnt[16];
  unsigned int spec_before;
  unsigned long long errinv;
  int spec_cut;
  int last;
  long long V[UST_V_LEN];          // split mode: the vector the last CTA publishes
};

// Residency on an H100 SM (228 KiB shared memory, 1 KiB of it reserved per CTA; 65536 registers, 16384 per
// sub-partition, a CTA's warp w on sub-partition w % 4): UST_STREAM_CTAS_PER_SM streaming CTAs and one verification CTA
// at the same time. With two, the CTA of call k+1 is resident and filling its ring while call k's still streams, so the
// SM's memory pipe does not drain between calls (DESIGN.md §3.1, §3.3). Losing this is a silent slow-down, hence here.
constexpr int kSmemPerSM = 228 * 1024, kSmemReservedPerCTA = 1024, kRegsPerSM = 65536, kRegsPerSubPartition = 16384;
constexpr int kStreamWarps = kThreads / 32, kVerifyWarps = UST_VERIFY_THREADS / 32;
static_assert(UST_STREAM_CTAS_PER_SM * (sizeof(SS<true>) + kSmemReservedPerCTA) + UST_VERIFY_SMEM_MAX + kSmemReservedPerCTA <= kSmemPerSM,
              "shared memory: the streaming CTAs (pod-list variant) and a verification CTA must fit on one SM");
static_assert(UST_STREAM_CTAS_PER_SM * kStreamWarps * 32 * UST_STREAM_MAXREG + kVerifyWarps * 32 * UST_VERIFY_MAXREG <= kRegsPerSM,
              "registers: the streaming CTAs and a verification CTA must fit on one SM");
static_assert(UST_STREAM_CTAS_PER_SM * ((kStreamWarps + 3) / 4) * 32 * UST_STREAM_MAXREG +
                      ((kVerifyWarps + 3) / 4) * 32 * UST_VERIFY_MAXREG <= kRegsPerSubPartition,
              "registers: the streaming CTAs and a verification CTA must fit on one SM sub-partition");

// Byte-sliced SIMD-in-register counting (hot_increments, ust_common.cuh). The hot-byte table holds a hot byte's 64-bit
// increment word next to the node's table window; a thread sums the entries of its nodes of two groups (no field can
// exceed 8), widens the nibbles to byte lanes, and keeps going. No atomics until the byte lanes fill up or the CTA runs
// out of tiles.
__device__ __forceinline__ uint4 hot_entry(unsigned b) {
  const unsigned code = b & 15u;
  const unsigned long long v = hot_increments(b);
  uint32_t x = 0, y = 0;  // the state's lookup constants (ust_lut.h): 16 compile-time pairs
#pragma unroll
  for (int s = 0; s < 16; s++)
    if (code == (unsigned)s) { x = ust_meta_x(s); y = ust_meta_y(s); }
  return make_uint4(x, y, (uint32_t)v, (uint32_t)(v >> 32));
}

template <bool PODS>
__device__ __forceinline__ void flush_counts(SS<PODS>& S, uint32_t (&B)[4]) {  // whole warp, converged
#pragma unroll
  for (int f = 0; f < 16; f++) {
    const unsigned v = __reduce_add_sync(kFull, field_of(B, f));
    if ((threadIdx.x & 31) == 0 && v) atomicAdd(&S.cnt[f], v);
  }
  B[0] = B[1] = B[2] = B[3] = 0;
}

// revision-hash error seen while streaming (pod_manager.go:84-89, :108-110; abort sites common_manager.go:234-238,
// :463-467, :533-538): remember the earliest one in pass order
template <bool PODS>
__device__ __forceinline__ void note_error_byte(const UstParams& P, SS<PODS>& S, unsigned b, uint32_t fl, long long i) {
  const unsigned code = b & 15u;
  if (!(b & UST_HOT_REVISION_HASH_ERROR) || !P.active) return;
  if (!(code == UST_STATE_UNKNOWN || code == UST_STATE_DONE || code == UST_STATE_POD_RESTART_REQUIRED || code == UST_STATE_FAILED)) return;
  if (fl & UST_F_POD_ORPHANED) return;
  atomicMax(&S.errinv, ~UST_KEY(pass_of_state(code), (unsigned long long)i + 1ull));
}

// One node: `hoff` = byte offset of its hot-byte table entry (this lane's replica), `wbits` = its SKIP /
// UNSCHEDULABLE bits already at w positions 2, 3, `fl` = the input bits of its flags word (+ pod-list bits).
template <bool DS_SMEM, bool PODS>
__device__ __forceinline__ uint32_t eval_node(const UstParams& P, const SS<PODS>& S, uint32_t hoff, uint32_t wbits, uint32_t fl,
                                              int rev, uint32_t di, uint32_t grant, uint32_t& lo, uint32_t& hi) {
  const uint4 m = *reinterpret_cast<const uint4*>(reinterpret_cast<const char*>(S.hotent) + hoff);
  lo += m.z;
  hi += m.w;
  uint32_t w = fl | wbits | grant;
  // podRevisionHash == daemonsetRevisionHash (common_manager.go:318); a missing DaemonSet never matches
  bool synced;
  if (DS_SMEM) synced = (di < (uint32_t)P.n_ds) && (rev == S.dsrev[min(di, (uint32_t)P.n_ds)]);
  else synced = di < (uint32_t)P.n_ds && rev == __ldg(P.ds_rev + di);
  if (synced) w |= UST_W_SYNCED;
  const uint32_t off = (__funnelshift_r(w, 0u, m.x) & (m.x >> 16)) | m.y;
  return *reinterpret_cast<const uint32_t*>(reinterpret_cast<const char*>(S.lut) + off);
}

// One 128-node group of a tile (lane l owns nodes 4l .. 4l+3 of the group): evaluate, count, store.
// FULL: the whole tile is inside the shard (no validity checks).
template <bool FULL, bool DS_SMEM, bool OUTCOME, bool PODS>
__device__ __forceinline__ void eval_group(const UstParams& P, SS<PODS>& S, const Stage<PODS>& st, int g, long long base, int valid,
                                           uint32_t grant, uint32_t& lo, uint32_t& hi, unsigned& mycand) {
  const int lane = threadIdx.x & 31;
  const uint32_t rep_off = kHotRep == 8 ? (uint32_t)(lane & 7) << 4 : 0u;
  const int q = g * 32 + lane;  // 4-node unit within the tile
  int nv = 4;
  if (!FULL) {
    nv = valid - 4 * q;
    nv = nv < 0 ? 0 : (nv > 4 ? 4 : nv);
    if (nv == 0) return;
  }
  uint32_t x = reinterpret_cast<const uint32_t*>(st.hot)[q];
  const uint4 f = reinterpret_cast<const uint4*>(st.flags)[q];
  const uint4 r = reinterpret_cast<const uint4*>(st.rev)[q];
  const uint4 d = reinterpret_cast<const uint4*>(st.ds)[q];
  uint32_t ps = 0;
  if (PODS) ps = reinterpret_cast<const uint32_t*>(st.ps)[q];
  if (!FULL && nv < 4) {  // nodes past the end of the shard: "not in snapshot", never stored
    const uint32_t keep = (1u << (8 * nv)) - 1u;
    x = (x & keep) | (0x0E0E0E0Eu & ~keep);
  }
  if (x & 0x80808080u) {  // rare
    const long long i = base + 4 * q;
    note_error_byte(P, S, x & 0xFFu, f.x, i);
    note_error_byte(P, S, (x >> 8) & 0xFFu, f.y, i + 1);
    note_error_byte(P, S, (x >> 16) & 0xFFu, f.z, i + 2);
    note_error_byte(P, S, x >> 24, f.w, i + 3);
  }
  mycand += __popc(cand_mask4(x));
  constexpr uint32_t kW = UST_W_SKIP | UST_W_UNSCHEDULABLE;
  // without pod lists the derived pod bits of w are never set: mask them out of the flags word
  constexpr uint32_t kIn = UST_F_INPUT_MASK;
  uint32_t fl[4] = {f.x & kIn, f.y & kIn, f.z & kIn, f.w & kIn};
  if (PODS) {
    fl[0] = pods_apply(fl[0], ps & 0xFFu);
    fl[1] = pods_apply(fl[1], (ps >> 8) & 0xFFu);
    fl[2] = pods_apply(fl[2], (ps >> 16) & 0xFFu);
    fl[3] = pods_apply(fl[3], ps >> 24);
  }
  uint32_t e[4];
  e[0] = eval_node<DS_SMEM>(P, S, ((x << kHotShift) & kHotMask) | rep_off, (x >> 3) & kW, fl[0], (int)r.x, d.x, grant, lo, hi);
  e[1] = eval_node<DS_SMEM>(P, S, ((kHotShift >= 8 ? x << (kHotShift - 8) : x >> (8 - kHotShift)) & kHotMask) | rep_off, (x >> 11) & kW,
                            fl[1], (int)r.y, d.y, grant, lo, hi);
  e[2] = eval_node<DS_SMEM>(P, S, ((x >> (16 - kHotShift)) & kHotMask) | rep_off, (x >> 19) & kW, fl[2], (int)r.z, d.z, grant, lo, hi);
  e[3] = eval_node<DS_SMEM>(P, S, ((x >> (24 - kHotShift)) & kHotMask) | rep_off, (x >> 27) & kW, fl[3], (int)r.w, d.w, grant, lo, hi);
  uint32_t next4, out4;
  uint2 act4;
  pack4(e, next4, act4, out4);
  if (FULL || nv == 4) {
    __stcs(reinterpret_cast<uint32_t*>(P.next + base) + q, next4);
    __stcs(reinterpret_cast<uint2*>(P.actions + base) + q, act4);
    if (OUTCOME) __stcs(reinterpret_cast<uint32_t*>(P.outcome + base) + q, out4);
  } else {
    for (int k = 0; k < nv; k++) {
      P.next[base + 4 * q + k] = (uint8_t)(e[k] >> 16);
      P.actions[base + 4 * q + k] = (uint16_t)e[k];
      if (OUTCOME) P.outcome[base + 4 * q + k] = (uint8_t)(e[k] >> 24);
    }
  }
}

// ---- producer: warp 0 ---------------------------------------------------------------------------------------------
// Tiles of [tile_begin, tile_end): `static_rounds` rounds in stride order (tile = begin + cta + round * grid), the
// rest by atomic ticket, two claims in flight so that the ticket's L2 round trip never stalls the ring. Contains the
// CTA's one start-up __syncthreads (after the first ring-full of copies is on its way).
template <bool PODS>
__device__ void produce(const UstParams& P, SS<PODS>& S) {
  const int lane = threadIdx.x;
  const int tn = P.tile_nodes, G = (int)gridDim.x, R = P.static_rounds;
  const int t_end = P.tile_end;
  const int dyn_base = P.tile_begin + R * G;
  // L2 priority of the input columns (UstParams::evict_first_inputs)
  const uint64_t pol = P.evict_first_inputs ? policy_evict_first() : policy_evict_normal();
  unsigned int* ticket = &P.ws->ticket[P.parity][P.seg];
  int pA = 0x7FFFFFFF, pB = 0x7FFFFFFF;
  if (lane == 0) {
    if (R == 0) { pA = dyn_base + (int)atomicAdd(ticket, 1u); pB = dyn_base + (int)atomicAdd(ticket, 1u); }
    else if (R == 1) pA = dyn_base + (int)atomicAdd(ticket, 1u);
  }
  bool synced = false;
  uint32_t it = 0;
  for (;; it++) {
    int tile = 0;
    if (lane == 0) {
      const int i = (int)it;
      if (i < R) tile = P.tile_begin + (int)blockIdx.x + i * G;
      else tile = ((i - R) & 1) ? pB : pA;
      if (i + 2 >= R) {  // the claim used two iterations from now
        const int c = dyn_base + (int)atomicAdd(ticket, 1u);
        if ((i + 2 - R) & 1) pB = c; else pA = c;
      }
    }
    tile = __shfl_sync(kFull, tile, 0);
    if (tile >= t_end) break;
    if (it == (uint32_t)kStages && !synced) { __syncthreads(); synced = true; }
    const int s = (int)(it % kStages);
    const uint32_t ph = (it / kStages) & 1u;
    mbar_wait(&S.empty[s], ph ^ 1u);
    Stage<PODS>& st = S.st[s];
    const long long base = (long long)tile * tn;
    const long long rem = P.n - base;
    const int valid = rem < tn ? (int)rem : tn;
    const int v16 = valid & ~15;
    if (valid != v16) {  // ragged end of the shard: the last < 16 nodes by hand (bulk copies move multiples of 16 bytes)
      const int k = v16 + lane;
      if (k < valid) {
        st.hot[k] = P.hot[base + k];
        st.flags[k] = P.flags[base + k];
        st.rev[k] = P.pod_rev[base + k];
        st.ds[k] = P.ds_idx[base + k];
        if (PODS) st.ps[k] = P.podsum[base + k];
      }
    }
    __syncwarp();
    if (lane == 0) {
      S.tile_of[s] = tile;
      mbar_arrive_expect_tx(&S.full[s], (uint32_t)v16 * (PODS ? 14u : 13u));
      if (v16) {
        bulk_g2s_stream(st.flags, P.flags + base, (uint32_t)v16 * 4u, &S.full[s], pol);
        bulk_g2s_stream(st.rev, P.pod_rev + base, (uint32_t)v16 * 4u, &S.full[s], pol);
        bulk_g2s_stream(st.ds, P.ds_idx + base, (uint32_t)v16 * 4u, &S.full[s], pol);
        bulk_g2s_stream(st.hot, P.hot + base, (uint32_t)v16, &S.full[s], pol);
        if (PODS) bulk_g2s_stream(st.ps, P.podsum + base, (uint32_t)v16, &S.full[s], pol);
      }
    }
  }
  if (!synced) __syncthreads();
  // end of stream: a stage that holds no tile
  const int s = (int)(it % kStages);
  const uint32_t ph = (it / kStages) & 1u;
  mbar_wait(&S.empty[s], ph ^ 1u);
  if (lane == 0) {
    S.tile_of[s] = -1;
    mbar_arrive(&S.full[s]);
  }
}

// ---- consumers: warps 1 .. kCW --------------------------------------------------------------------------------------
template <bool DS_SMEM, bool OUTCOME, bool PODS>
__device__ void consume(const UstParams& P, SS<PODS>& S, int cw) {
  const int lane = threadIdx.x & 31;
  const int tn = P.tile_nodes, groups = tn >> 7;
  const int spec_cut = S.spec_cut;
  uint32_t B[4] = {0, 0, 0, 0};
  int pending = 0;  // upper bound of any byte lane of B
  unsigned spec_before = 0;  // this thread's upgrade candidates in tiles before the speculative cut
  for (uint32_t it = 0;; it++) {
    const int s = (int)(it % kStages);
    const uint32_t ph = (it / kStages) & 1u;
    mbar_wait(&S.full[s], ph);
    const int tile = *reinterpret_cast<volatile int*>(&S.tile_of[s]);
    if (tile < 0) break;
    if (P.stamps && it == 0 && cw == 0 && lane == 0) P.ws->dbg[P.parity][blockIdx.x][1] = now_ns();
    const Stage<PODS>& st = S.st[s];
    const long long base = (long long)tile * tn;
    const long long rem = P.n - base;
    const int valid = rem < tn ? (int)rem : tn;
    // the speculation: tiles before the cut assume every upgrade candidate gets a slot, the others that none does
    const uint32_t grant = tile < spec_cut ? UST_W_GRANTED : 0u;
    uint32_t lo = 0, hi = 0;
    unsigned mycand = 0;
    if (valid == kTile) {
#pragma unroll
      for (int j = 0; j < kGPW; j++) {
        if (cw + j * kCW < kGroups) eval_group<true, DS_SMEM, OUTCOME, PODS>(P, S, st, cw + j * kCW, base, valid, grant, lo, hi, mycand);
        if ((j & 1) && j + 1 < kGPW) widen(lo, hi, B);  // a nibble counter holds the 8 nodes of two groups
      }
    } else {
      int j = 0;
      for (int g = cw; g < groups; g += kCW, j++) {
        eval_group<false, DS_SMEM, OUTCOME, PODS>(P, S, st, g, base, valid, grant, lo, hi, mycand);
        if (j & 1) widen(lo, hi, B);
      }
    }
    widen(lo, hi, B);
    if (tile < spec_cut) spec_before += mycand;
    // the tile's upgrade candidates (for the ordered slot allocation): the last warp to finish the stage publishes
    const unsigned wc = __reduce_add_sync(kFull, mycand);
    if (lane == 0) {
      const unsigned old = atomicAdd(&S.stage_acc[s], (1u << 16) | wc);
      if ((old >> 16) == (unsigned)(kCW - 1)) {
        P.cand_tile[tile] = (old & 0xFFFFu) + wc;
        S.stage_acc[s] = 0;
      }
      mbar_arrive(&S.empty[s]);  // this warp is done with the stage
    }
    __syncwarp();
    pending += 4 * kGPW;
    if (pending > 255 - 4 * kGPW) { flush_counts(S, B); pending = 0; }
  }
  flush_counts(S, B);
  // candidates before the speculative cut: with them the verification kernel finds a cut that stayed in (or near) the
  // tile of the previous call's without scanning the per-tile counts
  spec_before = __reduce_add_sync(kFull, spec_before);
  if (lane == 0 && spec_before) atomicAdd(&S.spec_before, spec_before);
}

template <bool DS_SMEM, bool OUTCOME, bool PODS>
__global__ void __maxnreg__(UST_STREAM_MAXREG) ust_stream_kernel(const __grid_constant__ UstParams P) {
  extern __shared__ __align__(128) unsigned char ust_smem[];
  SS<PODS>& S = *reinterpret_cast<SS<PODS>*>(ust_smem);
  const int t = threadIdx.x, warp = t >> 5;
  UstWorkspace* ws = P.ws;
  // the next kernel of the stream (the verification kernel) may be made resident now: it waits for this grid itself
  griddep_launch_dependents();
  if (P.stamps && t == 0) {
    ws->dbg[P.parity][blockIdx.x][0] = now_ns();
    unsigned sm;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(sm));
    ws->dbg_sm[P.parity][blockIdx.x] = sm;
  }
  if (warp == 0) {
    if (t == 0) {
      for (int s = 0; s < kStages; s++) { mbar_init(&S.full[s], 1); mbar_init(&S.empty[s], kCW); }
      mbar_init(&S.lutbar, 1);
      mbar_fence_init();
      // the per-policy transition table (DriverUpgradePolicySpec + manager options, compiled to 4.4 KiB by ust_lut.h):
      // one bulk copy; it was uploaded by a copy, not by a kernel, so it does not have to wait for the previous grid
      mbar_arrive_expect_tx(&S.lutbar, kLutBytes);
      bulk_g2s(S.lut, P.lut, kLutBytes, &S.lutbar);
    }
    __syncwarp();
    // everything before this line overlapped the tail of the previous kernel of the stream. A call that does not depend
    // on the previous one (P.relaxed: the host has checked that no buffer of this call is written by it) streams on at
    // once and waits at its end, before it touches the workspace.
    if (!P.relaxed) griddep_wait();
    produce<PODS>(P, S);
  } else {
    const int ct = t - 32, cn = kThreads - 32;
    for (int i = ct; i < 128 * kHotRep; i += cn) S.hotent[i] = hot_entry((unsigned)(kHotRep == 8 ? i >> 3 : i));
    if (ct < 16) S.cnt[ct] = 0;
    if (ct >= 32 && ct < 32 + kStages) S.stage_acc[ct - 32] = 0;
    if (!P.relaxed) griddep_wait();
    if (DS_SMEM)
      for (int i = ct; i <= P.n_ds; i += cn) S.dsrev[i] = i < P.n_ds ? __ldg(P.ds_rev + i) : 0;
    if (ct == 0) {
      if (UST_STREAM_CTAS_PER_SM > 1 && P.relaxed) {
        // This call shares its parity's set (hint slot, spec_used, cand_tile) with the call before the previous one,
        // whose verification kernel may still read it: wait until that kernel - and every one before it - has left.
        // Nothing is spent here in practice (the previous call's whole streaming pass ran in between), and nothing
        // waited for can be starved: those CTAs were all resident before this grid could launch.
        while ((unsigned long long)ld_acquire_gpu(reinterpret_cast<const long long*>(&ws->verify_done)) < P.verify_before)
          __nanosleep(64);
      }
      S.errinv = 0;
      S.spec_before = 0;
      // speculative cut: the previous call's, when it was made under the same signature; else the policy default
      const bool slotted = P.active && !P.requestor;
      const int hs = P.relaxed ? P.parity : P.parity ^ 1;  // a slot no running kernel writes (ust_dev.h)
      const bool hinted = P.spec_sig != 0 && __ldcg(&ws->hint_sig[hs]) == P.spec_sig;
      const int cut = !slotted ? 0 : (hinted ? __ldcg(&ws->hint_cut[hs]) : P.spec_cut_tile);
      S.spec_cut = cut;
      if (blockIdx.x == 0) ws->spec_used[P.parity] = cut;  // the verification kernel judges the speculation that was made
    }
    __syncthreads();
    mbar_wait(&S.lutbar, 0);
    if (PODS && S.meta[UST_STATE_VALIDATION_REQUIRED].x != ust_meta_x(UST_STATE_VALIDATION_REQUIRED)) {
      // validation mode moves state 9's window (ust_lut.h): then state 9's lookup pair is the table's, not the compile-time
      // one of hot_entry. Consumer warps only (named barrier 1; the condition is the same for all of them), once per CTA.
      if (ct < 8 * kHotRep) {
        uint4& e = S.hotent[(UST_STATE_VALIDATION_REQUIRED + 16 * (ct / kHotRep)) * kHotRep + ct % kHotRep];
        e.x = S.meta[UST_STATE_VALIDATION_REQUIRED].x;
        e.y = S.meta[UST_STATE_VALIDATION_REQUIRED].y;
      }
      asm volatile("bar.sync 1, %0;" ::"n"(kThreads - 32) : "memory");
    }
    consume<DS_SMEM, OUTCOME, PODS>(P, S, warp - 1);
  }
  // this CTA has run out of tiles: add its counts to the shard's (reductions, nobody waits for them) and leave.
  // The previous call's verification kernel must be through with the workspace first (it is, unless this call started
  // early: then this is where it waits).
  __syncthreads();
  if (P.stamps && t == 0) ws->dbg[P.parity][blockIdx.x][2] = now_ns();
  griddep_wait();
  unsigned long long* acc = ws->acc[P.parity];
  if (blockIdx.x == 0 && P.seg == 0 && t >= 64 && t < 64 + 18 + 1 + UST_MAX_SEGMENTS) {
    // clear the previous call's accumulator set (the next call's): its only reader has completed
    const int o = t - 64, q = P.parity ^ 1;
    if (o < 18) ws->acc[q][o] = 0;
    else if (o == 18) ws->errinv[q] = 0;
    else ws->ticket[q][o - 19] = 0;
  }
  if (t < 14) { if (S.cnt[t]) atomicAdd(&acc[t], (unsigned long long)S.cnt[t]); }
  else if (t == 14) { if (S.cnt[14]) atomicAdd(&acc[UST_V_UNAVAILABLE], (unsigned long long)S.cnt[14]); }
  else if (t == 15) { if (S.cnt[15]) atomicAdd(&acc[UST_V_CANDIDATES], (unsigned long long)S.cnt[15]); }
  else if (t == 32) { if (S.errinv) atomicMax(&ws->errinv[P.parity], S.errinv); }
  else if (t == 33) { if (S.spec_before) atomicAdd(&acc[UST_STATE_EXCLUDED], (unsigned long long)S.spec_before); }  // lane 14 is free: "not in snapshot" is derived
  if (P.stamps && t == 0) ws->dbg[P.parity][blockIdx.x][3] = now_ns();
  if (!(P.split && P.publish)) return;
  // ---- split mode (a host-launched collective follows): the last CTA of the call's last streaming launch publishes
  // this shard's lanes of the exchange vector
  __threadfence();
  __syncthreads();
  if (t == 0) S.last = atomicAdd(&ws->arrive, 1u) == gridDim.x - 1u;
  __syncthreads();
  if (!S.last) return;
  __threadfence();
  if (t == 0) ws->arrive = 0;
  if (t < UST_V_LEN) {
    long long v = 0;
    if (t < 14 || t == UST_V_UNAVAILABLE || t == UST_V_CANDIDATES) v = (long long)__ldcg(&acc[t]);
    else if (t == UST_V_RANK_CAND + P.rank) v = (long long)__ldcg(&acc[UST_V_CANDIDATES]);
    else if (t == UST_V_RANK_NODES + P.rank) v = P.n;
    else if (t == UST_V_RANK_ERRINV + P.rank) v = (long long)__ldcg(&ws->errinv[P.parity]);
    S.V[t] = v;
  }
  __syncthreads();
  if (t < UST_V_LEN) {
    long long v = S.V[t];
    if (t == UST_STATE_EXCLUDED) {  // everything that is in no bucket
      long long in = 0;
      for (int f = 0; f < 14; f++) in += S.V[f];
      v = P.n - in;
    }
    P.xchg[t] = v;
  }
}

template <bool DS_SMEM, bool OUTCOME, bool PODS>
cudaError_t launch_variant(const UstParams& p, int grid, cudaStream_t st, int pdl) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = sizeof(SS<PODS>);
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, ust_stream_kernel<DS_SMEM, OUTCOME, PODS>, p);
}

template <bool DS_SMEM, bool OUTCOME, bool PODS>
cudaError_t config_variant(int* ctas_per_sm) {
  // the whole 228 KiB as shared memory: the streaming CTAs and the verification kernel's CTA (5.6 KiB, ptxas sm_90a) must
  // fit together, or the next call's CTA cannot become resident before this one has left the SM
  cudaError_t e = cudaFuncSetAttribute(ust_stream_kernel<DS_SMEM, OUTCOME, PODS>, cudaFuncAttributePreferredSharedMemoryCarveout,
                                       (int)cudaSharedmemCarveoutMaxShared);
  if (e != cudaSuccess) return e;
  e = cudaFuncSetAttribute(ust_stream_kernel<DS_SMEM, OUTCOME, PODS>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           (int)sizeof(SS<PODS>));
  if (e != cudaSuccess) return e;
  int blocks = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks, ust_stream_kernel<DS_SMEM, OUTCOME, PODS>, kThreads, sizeof(SS<PODS>));
  if (e == cudaSuccess && blocks < *ctas_per_sm) *ctas_per_sm = blocks;
  return e;
}

}  // namespace

int ust_launch_stream(const UstParams& p, int grid, void* stream, int pdl) {
  cudaStream_t st = (cudaStream_t)stream;
  const int variant = (p.n_ds <= UST_DS_SMEM_MAX ? 4 : 0) | (p.outcome ? 2 : 0) | (p.podsum ? 1 : 0);
  switch (variant) {
    case 7: return (int)launch_variant<true, true, true>(p, grid, st, pdl);
    case 6: return (int)launch_variant<true, true, false>(p, grid, st, pdl);
    case 5: return (int)launch_variant<true, false, true>(p, grid, st, pdl);
    case 4: return (int)launch_variant<true, false, false>(p, grid, st, pdl);
    case 3: return (int)launch_variant<false, true, true>(p, grid, st, pdl);
    case 2: return (int)launch_variant<false, true, false>(p, grid, st, pdl);
    case 1: return (int)launch_variant<false, false, true>(p, grid, st, pdl);
    default: return (int)launch_variant<false, false, false>(p, grid, st, pdl);
  }
}

int ust_stream_config(int device, int* num_sms, size_t* smem_bytes, int* ctas_per_sm) {
  cudaError_t e;
  int c = 1 << 30;
  if ((e = config_variant<true, true, true>(&c)) != cudaSuccess) return (int)e;
  if ((e = config_variant<true, true, false>(&c)) != cudaSuccess) return (int)e;
  if ((e = config_variant<true, false, true>(&c)) != cudaSuccess) return (int)e;
  if ((e = config_variant<true, false, false>(&c)) != cudaSuccess) return (int)e;
  if ((e = config_variant<false, true, true>(&c)) != cudaSuccess) return (int)e;
  if ((e = config_variant<false, true, false>(&c)) != cudaSuccess) return (int)e;
  if ((e = config_variant<false, false, true>(&c)) != cudaSuccess) return (int)e;
  if ((e = config_variant<false, false, false>(&c)) != cudaSuccess) return (int)e;
  *ctas_per_sm = c;
  int sms = 0;
  if ((e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device)) != cudaSuccess) return (int)e;
  *num_sms = sms;
  *smem_bytes = sizeof(SS<true>);
  return 0;
}
