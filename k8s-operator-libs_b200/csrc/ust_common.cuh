// ust_common.cuh — device code shared by the streaming kernel (ust_stream.cu) and the kernels of ust_kernels.cu: PTX
// wrappers (mbarrier, TMA bulk copy, programmatic dependent launch, system-scope accesses), the byte-sliced counters of
// the streaming and BuildState passes, the cluster-wide arithmetic between the streaming and the verification kernel
// (GetUpgradesAvailable and friends), and the decision a call's last CTA makes about the slot speculation.
#pragma once
#include <cuda_runtime.h>

#include "ust_dev.h"

namespace ustd {

constexpr unsigned kFull = 0xFFFFFFFFu;

// ---- PTX wrappers ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, uint32_t parity) {
  uint32_t done = 0;
  while (!done) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  }
}
// one 1-D TMA bulk copy global -> shared, completing `bytes` on the mbarrier (bytes: multiple of 16, both ends
// 16-byte aligned); streamed data carries an evict-first L2 policy
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void bulk_g2s_stream(void* dst, const void* src, uint32_t bytes, unsigned long long* bar, uint64_t pol) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(pol) : "memory");
}
__device__ __forceinline__ uint64_t policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t policy_evict_normal() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p));
  return p;
}
// programmatic dependent launch: let the next kernel of the stream start its prologue / wait for the previous one
__device__ __forceinline__ void griddep_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

__device__ __forceinline__ unsigned long long now_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void st_relaxed_sys(long long* p, long long v) { asm volatile("st.relaxed.sys.global.s64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }
__device__ __forceinline__ void st_release_sys(long long* p, long long v) { asm volatile("st.release.sys.global.s64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }
__device__ __forceinline__ long long ld_acquire_sys(const long long* p) {
  long long v;
  asm volatile("ld.acquire.sys.global.s64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_gpu(long long* p, long long v) { asm volatile("st.release.gpu.global.s64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }
__device__ __forceinline__ long long ld_acquire_gpu(const long long* p) {
  long long v;
  asm volatile("ld.acquire.gpu.global.s64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ long long ld_relaxed_sys(const long long* p) {
  long long v;
  asm volatile("ld.relaxed.sys.global.s64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
constexpr unsigned long long kCommTimeoutNs = 4000000000ull;  // give up on a missing peer after 4 s

// (pass + 1) of each state code, one nibble per code: position of its Process* pass in ApplyState
// (upgrade_state.go:205-274), 0 = never processed. Same content as ust_pass_of_state[] in ust_lut.h.
__device__ __forceinline__ int pass_of_state(unsigned code) {
  constexpr unsigned long long kPassPlus1 =
      (1ull << 0) | (3ull << 4) | (4ull << 8) | (5ull << 12) | (6ull << 16) | (7ull << 20) | (8ull << 24) | (0ull << 28) |
      (9ull << 32) | (11ull << 36) | (12ull << 40) | (2ull << 44) | (10ull << 48);
  return (int)((kPassPlus1 >> (4 * code)) & 15ull) - 1;
}

// candidate bytes of a hot word: bit 7 of byte k set iff node k is upgrade-required and not marked skip
// (upgrade_inplace.go:82)
__device__ __forceinline__ uint32_t cand_mask4(uint32_t x) {
  const uint32_t y = (x & 0x2F2F2F2Fu) ^ 0x01010101u;  // zero byte <=> code == 1 && !SKIP
  return ~(((y & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | y) & 0x80808080u;
}

// ---- byte-sliced SIMD-in-register counting (the streaming pass and the BuildState passes) -------------------------
// A hot byte increments sixteen 4-bit one-hot fields packed in 64 bits: fields 0-13 count the state codes, field 14 the
// unavailable nodes, field 15 the upgrade candidates; codes 14 and 15 count nothing. GetCurrentUnavailableNodes
// (common_manager.go:146-165) counts every snapshot entry that is cordoned or not ready; an upgrade candidate is
// upgrade-required and not marked skip (upgrade_inplace.go:82). A thread sums the increments of up to 8 nodes in two
// registers (lo = fields 0-7, hi = fields 8-15), widens the nibbles into four byte-lane words and keeps going.
__device__ __forceinline__ unsigned long long hot_increments(unsigned b) {
  const unsigned code = b & 15u;
  unsigned long long v = 0;
  if (code < 14) {
    v = 1ull << (4 * code);
    if (b & (UST_HOT_UNSCHEDULABLE | UST_HOT_NOT_READY)) v |= 1ull << 56;
    if (code == UST_STATE_UPGRADE_REQUIRED && !(b & UST_HOT_SKIP)) v |= 1ull << 60;
  }
  return v;
}
// byte lanes: B[0] = fields 0,2,4,6  B[1] = fields 1,3,5,7  B[2] = fields 8,10,12,14  B[3] = fields 9,11,13,15
__device__ __forceinline__ unsigned field_of(const uint32_t (&B)[4], int f) {
  return (B[(f >> 3) * 2 + (f & 1)] >> (8 * ((f & 7) >> 1))) & 0xFFu;
}
__device__ __forceinline__ void widen(uint32_t& lo, uint32_t& hi, uint32_t (&B)[4]) {
  B[0] += lo & 0x0F0F0F0Fu;
  B[1] += (lo >> 4) & 0x0F0F0F0Fu;
  B[2] += hi & 0x0F0F0F0Fu;
  B[3] += (hi >> 4) & 0x0F0F0F0Fu;
  lo = hi = 0;
}

// four table entries (actions | next << 16 | outcome << 24) -> the three output words of a 4-node group
__device__ __forceinline__ void pack4(const uint32_t e[4], uint32_t& next4, uint2& act4, uint32_t& out4) {
  act4.x = __byte_perm(e[0], e[1], 0x5410);
  act4.y = __byte_perm(e[2], e[3], 0x5410);
  const uint32_t hi01 = __byte_perm(e[0], e[1], 0x7632);  // [e0.b2 e0.b3 e1.b2 e1.b3]
  const uint32_t hi23 = __byte_perm(e[2], e[3], 0x7632);
  next4 = __byte_perm(hi01, hi23, 0x6420);
  out4 = __byte_perm(hi01, hi23, 0x7531);
}

// pod-list summary byte -> the w bits it stands for (ust_pod_summary_kernel): bit 0 = a wait-selector pod is
// running, bits 1..3 = UST_W_PD_HAS / UST_W_PD_MISMATCH / UST_W_DRAIN_ERROR, bit 4 = the list overrides the
// pre-evaluated UST_F_WAIT_PODS_RUNNING of the flags word. A validation-required node in validation mode uses bits 1-3
// and 5-7 (ust_lut.h, UST_VALSUM_*): they land at w bits 22-24 and 26-28, state 9's window in that mode. Every other
// node's bits 5-7 are clear, and no other state reads w bits 25-28.
__device__ __forceinline__ uint32_t pods_apply(uint32_t fl, uint32_t ps) {
  return (fl & ~((ps & 0x10u) << 12)) | ((ps & 1u) << 16) | ((ps & 0xEEu) << 21);
}
static_assert(UST_F_WAIT_PODS_RUNNING == (1u << 16) && UST_W_PD_HAS == (UST_PODSUM_TO_DELETE << 21) &&
              UST_W_PD_MISMATCH == (UST_PODSUM_CANNOT_DELETE << 21) && UST_W_DRAIN_ERROR == (UST_PODSUM_DRAIN_ERROR << 21) &&
              UST_PODSUM_WAIT_RUNNING == 1u && UST_VAL_SHIFT == UST_VALSUM_OUTCOME_SHIFT + 21 && (UST_F_INPUT_MASK & 0x1FC00000u) == 0,
              "pod summary byte layout");

// ---- the decision between streaming and verification ------------------------------------------------------------
struct DecideShared {
  long long V[UST_V_LEN];        // cluster-wide exchange vector
  unsigned long long abort_key;  // ~0 = none
  long long budget;              // max(upgradesAvailable, 0)
  long long avail;
  long long max_unav;
  long long node_offset;         // global index of this shard's node 0
  long long cand_before;         // upgrade candidates on lower ranks
  long long total, in_progress;
  long long slots_left;
  long long part[32];
  long long run_before;
  long long spec_before;         // this shard's candidates in the tiles before the speculative cut (counted while streaming)
  int run0, run1;                // cut search: the run of tiles that contains the crossing
  int found;
  int spec_cut;                  // effective speculative cut of this call (hint or policy default), in tiles
  int redo, cut, lo, hi, scan;
};

// this shard's lanes of the exchange vector from the workspace accumulators of the call (one load per thread)
__device__ __forceinline__ void load_local_vector(const UstParams& P, DecideShared& D) {
  const int t = threadIdx.x;
  const unsigned long long* acc = P.ws->acc[P.parity];
  if (t < UST_V_LEN) {
    long long v = 0;
    if (t < 14 || t == UST_V_UNAVAILABLE || t == UST_V_CANDIDATES) v = (long long)__ldcg(&acc[t]);
    else if (t == UST_V_RANK_CAND + P.rank) v = (long long)__ldcg(&acc[UST_V_CANDIDATES]);
    else if (t == UST_V_RANK_NODES + P.rank) v = P.n;
    else if (t == UST_V_RANK_ERRINV + P.rank) v = (long long)__ldcg(&P.ws->errinv[P.parity]);
    D.V[t] = v;
  } else if (t == UST_V_LEN) {
    D.spec_before = (long long)__ldcg(&acc[UST_STATE_EXCLUDED]);  // lane 14 of the accumulators: see ust_stream.cu
  }
}
// ... lane 14 of the LOCAL vector: everything that is in no bucket - "not in snapshot" (upgrade_state.go:149-152) and
// code 15. One thread of warp 0, after a __syncwarp() (lanes 0..13 are written by warp 0), before any exchange.
__device__ __forceinline__ void fix_excluded_lane(const UstParams& P, DecideShared& D) {
  long long in = 0;
#pragma unroll
  for (int f = 0; f < 14; f++) in += D.V[f];
  D.V[UST_STATE_EXCLUDED] = P.n - in;
}

// Cluster-wide scalars from the exchange vector. Every calling thread computes all of them (same instructions, same
// values: no broadcast needed afterwards).
struct Scalars {
  unsigned long long abort_key;
  long long total, in_progress, budget, avail, max_unav, node_offset, cand_before;
};
__device__ inline Scalars derive_scalars(const UstParams& P, const long long* V) {
  Scalars s;
  const long long h0 = V[0], h1 = V[1], h2 = V[2], h4 = V[4], h11 = V[11];
  // GetTotalManagedNodes (common_manager.go:715-730): 11 buckets — not 6, 7, other
  const long long total = h0 + h1 + h2 + V[3] + h4 + V[5] + V[8] + V[9] + V[10] + h11 + V[12];
  const long long in_progress = total - h0 - h11 - h1;  // GetUpgradesInProgress (:733-739)
  unsigned long long abort_key = ~0ull;
  long long off = 0, my_off = 0, cand_before = 0;
  for (int r = 0; r < P.world; r++) {
    if (r == P.rank) my_off = off;
    if (r < P.rank) cand_before += V[UST_V_RANK_CAND + r];
    const unsigned long long e = (unsigned long long)V[UST_V_RANK_ERRINV + r];
    if (e) {
      const unsigned long long k = ~e;
      const unsigned long long gk = (k & 0xFF00000000000000ull) | ((k & 0x00FFFFFFFFFFFFFFull) + (unsigned long long)off);
      if (gk < abort_key) abort_key = gk;
    }
    off += V[UST_V_RANK_NODES + r];
  }
  long long max_unav = 0, avail = 0;
  const bool slots = P.active && !P.requestor;
  if (slots) {
    // upgrade_inplace.go:49-62 + intstr.GetScaledValueFromIntOrPercent(v, total, roundUp=true)
    if (P.max_unav_kind == UST_MAXUNAVAIL_INVALID && UST_KEY(2, 0) < abort_key) abort_key = UST_KEY(2, 0);
    max_unav = total;
    if (P.max_unav_kind == UST_MAXUNAVAIL_INT) max_unav = P.max_unav_value;
    else if (P.max_unav_kind == UST_MAXUNAVAIL_PERCENT) {
      // int(math.Ceil(float64(v) * float64(total) / 100)). While |v * total| < 2^52 the product is exact in float64 and
      // the correctly rounded quotient is closer than 2^-7 to the true one, which is an integer or at least 1/100 away
      // from one: the ceiling is the integer one. Beyond that, float64 as the reference computes it.
      const long long v = P.max_unav_value;
      if (v > -(1LL << 20) && v < (1LL << 20) && total < (1LL << 31)) {
        const long long x = v * total, q = x / 100;
        max_unav = q + ((x % 100) > 0 ? 1 : 0);
      } else {
        max_unav = (long long)ceil(__ddiv_rn(__dmul_rn((double)v, (double)total), 100.0));
      }
    }
    // GetUpgradesAvailable (common_manager.go:748-776)
    avail = (P.max_parallel == 0) ? h1 : P.max_parallel - in_progress;
    const long long cur_unav = V[UST_V_UNAVAILABLE] + h2;
    if (avail > max_unav) avail = max_unav;
    if (cur_unav >= max_unav) avail = 0;
    else if (max_unav < total && cur_unav + avail > max_unav) avail = max_unav - cur_unav;
  }
  // SchedulePodEviction with a nil DeletionSpec (pod_manager.go:125-134)
  if (P.active && P.pd_enabled && !P.pd_spec_present && h4 > 0 && UST_KEY(5, 0) < abort_key) abort_key = UST_KEY(5, 0);
  s.abort_key = abort_key;
  s.total = total;
  s.in_progress = in_progress;
  s.avail = avail;
  s.max_unav = max_unav;
  s.budget = avail > 0 ? avail : 0;
  s.node_offset = my_off;
  s.cand_before = cand_before;
  return s;
}

// ust_counters, one field per lane of a warp (31 int64 fields)
__device__ inline void write_counters(const UstParams& P, const long long* V, const Scalars& s, long long redone_tiles, bool comm_failed) {
  const int lane = threadIdx.x & 31;
  long long code = UST_OK, index = -1, pass = -1;
  if (s.abort_key != ~0ull) {
    pass = (long long)(s.abort_key >> 56);
    const long long idx1 = (long long)(s.abort_key & 0x00FFFFFFFFFFFFFFull);
    index = idx1 - 1;
    // node aborts: pass 10 (validation-required) can only be Validate's; the others are revision-hash lookups
    code = idx1 ? (pass == 10 ? UST_ERR_VALIDATION : UST_ERR_REVISION_HASH)
                : (pass == 2 ? UST_ERR_MAX_UNAVAILABLE : UST_ERR_POD_DELETION_SPEC);
  }
  const bool slots = P.active && !P.requestor && !(code && pass < 2) && code != UST_ERR_MAX_UNAVAILABLE;
  if (comm_failed) { code = UST_ERR_COMM; index = -1; pass = -1; }
  // one field per lane, picked with selects (a branchy pick would run its ten arms one after the other)
  long long v = V[lane < 18 ? lane : 0];   // hist[0..15], unavailable, candidates: lanes 0..17 of the vector
  v = lane == 18 ? s.total : v;
  v = lane == 19 ? s.in_progress : v;
  v = lane == 20 ? (slots ? s.max_unav : 0) : v;
  v = lane == 21 ? (slots ? s.avail : 0) : v;
  v = lane == 22 ? code : v;
  v = lane == 23 ? index : v;
  v = lane == 24 ? pass : v;
  v = lane == 25 ? redone_tiles : v;  // reserved[0]: tiles the verification kernel re-evaluates (diagnostic; the pipelined host path re-downloads when != 0)
  v = lane > 25 ? 0 : v;
  static_assert(UST_V_UNAVAILABLE == 16 && UST_V_CANDIDATES == 17, "counter fields 16, 17 mirror the vector");
  static_assert(sizeof(ust_counters) == 32 * 8, "one field per lane");
  reinterpret_cast<long long*>(P.out)[lane] = v;
}

// The decision, made by every CTA of the verification kernel for itself once the cluster-wide vector is in D.V (it is
// a few hundred instructions on 42 numbers): warp 0 derives the slot budget and checks the speculation in O(1)
// (rank-local: "nobody gets a slot" only fails if this shard has a budget, "everybody" only if the budget is smaller
// than its candidates); only when that cannot tell - or the call aborts - the CTA searches the per-tile candidate
// counts for the tile where the budget cuts (two block-wide passes, every load in flight at once). Tiles before the
// cut are fully granted, tiles behind it get nothing, the cut tile hands out `slots_left` in slice order
// (upgrade_inplace.go:71-109). `write_global`: this CTA also publishes the counters and the next call's speculation
// hint. `comm_failed`: a peer never showed up - the call fails, nothing is re-evaluated.
__device__ inline void decide(const UstParams& P, DecideShared& D, bool write_global, bool comm_failed) {
  const int t = threadIdx.x, nt = blockDim.x, nT = P.n_tiles;
  const bool slotted = P.active && !P.requestor;
  if (t < 32) {
    if (P.stamps && write_global && t == 0) P.ws->dbg2[4] = now_ns();
    const Scalars s = derive_scalars(P, D.V);
    if (P.stamps && write_global && t == 0) P.ws->dbg2[5] = now_ns() + (s.total & 1);
    const bool aborting = s.abort_key != ~0ull;
    const long long lc = D.V[UST_V_RANK_CAND + P.rank];   // this shard's candidates
    const long long lb = s.budget - s.cand_before;         // slots left when slice order reaches this shard
    const int sc = D.spec_cut < 0 ? 0 : (D.spec_cut > nT ? nT : D.spec_cut);
    bool need = false;
    if (slotted && lc > 0) need = sc <= 0 ? lb > 0 : (sc >= nT ? lb < lc : true);
    int cut = nT, scan = 0;
    if (slotted && lc > 0 && (need || aborting) && !comm_failed) {
      if (lb <= 0) cut = 0;
      else if (lb < lc) scan = 1;   // the cut lies inside this shard: find it
    }
    const int redo = comm_failed ? 0 : (aborting ? 2 : (need ? 1 : 0));  // need: final once the cut is known
    if (t == 0) {
      D.abort_key = s.abort_key; D.budget = s.budget; D.avail = s.avail; D.max_unav = s.max_unav;
      D.node_offset = s.node_offset; D.cand_before = s.cand_before; D.total = s.total; D.in_progress = s.in_progress;
      D.cut = cut; D.slots_left = 0; D.scan = scan; D.redo = redo; D.lo = 1; D.hi = 0;
      D.run0 = D.run1 = 0; D.run_before = 0; D.found = 0;
    }
    if (write_global && !scan && !(redo == 1)) {  // the common case ends here: counters out, no tile is redone
      write_counters(P, D.V, s, redo == 2 ? (long long)nT : 0, comm_failed);
      if (t == 0 && P.spec_sig != 0 && slotted && !aborting && !comm_failed) {
        P.ws->hint_cut[P.parity] = D.spec_cut;  // the all-or-nothing guess held
        P.ws->hint_sig[P.parity] = P.spec_sig;
      }
    }
    if (P.stamps && write_global && t == 0) P.ws->dbg2[6] = now_ns();
  }
  __syncthreads();
  if (P.stamps && write_global && t == 0) P.ws->dbg2[7] = now_ns();
  if (D.redo != 1 && !D.scan) return;
  const long long lb = D.budget - D.cand_before;
  const int sc_mid = D.spec_cut;
  if (D.scan && sc_mid > 0 && sc_mid < nT && !P.split) {
    // The speculation came from the previous call's cut, and the streaming pass has counted this shard's candidates in
    // the tiles before it: the budget most likely cuts in that tile again or next to it. One window of per-tile counts
    // around it (one load per thread, one round trip) settles that without looking at the other tiles.
    constexpr int kHalf = 64;
    const int c = sc_mid - kHalf + t;
    const bool in = t < 2 * kHalf && c >= 0 && c < nT;
    const long long cand = in ? (long long)__ldcg(&P.cand_tile[c]) : 0;
    long long incl = cand;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long v = __shfl_up_sync(kFull, incl, o);
      if ((t & 31) >= o) incl += v;
    }
    if ((t & 31) == 31) D.part[t >> 5] = incl;
    __syncthreads();
    long long pre = incl - cand, before_sc = 0;   // pre: candidates of the window before tile c
    for (int w = 0; w < (nt >> 5); w++) {
      const long long v = D.part[w];
      if (w < (t >> 5)) pre += v;
      if (w < kHalf / 32) before_sc += v;         // the window's tiles before the speculative cut
    }
    const long long prefix = D.spec_before - before_sc + pre;  // this shard's candidates before tile c
    if (in && prefix <= lb && lb < prefix + cand) { D.cut = c; D.slots_left = lb - prefix; D.found = 1; }
    __syncthreads();
  }
  if (D.scan && !D.found) {
    // pass 1: thread t sums the tiles [c0, c1); block-wide exclusive scan; the run that contains the crossing is
    // published. pass 2: the whole CTA loads that run (<= per tiles) and scans again.
    const int per = (nT + nt - 1) / nt;
    const int c0 = t * per < nT ? t * per : nT, c1 = c0 + per < nT ? c0 + per : nT;
    long long mine = 0;
    for (int cb = c0; cb < c1; cb += 16) {   // 16 loads in flight
      unsigned v[16];
#pragma unroll
      for (int k = 0; k < 16; k++) v[k] = cb + k < c1 ? __ldcg(&P.cand_tile[cb + k]) : 0u;
#pragma unroll
      for (int k = 0; k < 16; k++) mine += v[k];
    }
    long long incl = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long v = __shfl_up_sync(kFull, incl, o);
      if ((t & 31) >= o) incl += v;
    }
    __syncthreads();
    if ((t & 31) == 31) D.part[t >> 5] = incl;
    __syncthreads();
    long long before = incl - mine;
    for (int w = 0; w < (t >> 5); w++) before += D.part[w];
    if (before <= lb && lb < before + mine) { D.run0 = c0; D.run1 = c1; D.run_before = before; }
    __syncthreads();
    const int r0 = D.run0, r1 = D.run1;
    long long run_before = D.run_before;
    for (int b = r0; b < r1; b += nt) {   // one round unless a thread owns more than nt tiles
      const int c = b + t;
      const long long cand = c < r1 ? (long long)__ldcg(&P.cand_tile[c]) : 0;
      long long inc2 = cand;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const long long v = __shfl_up_sync(kFull, inc2, o);
        if ((t & 31) >= o) inc2 += v;
      }
      __syncthreads();
      if ((t & 31) == 31) D.part[t >> 5] = inc2;
      __syncthreads();
      long long pre = run_before + inc2 - cand, tot = 0;
      for (int w = 0; w < (nt >> 5); w++) { const long long v = D.part[w]; if (w < (t >> 5)) pre += v; tot += v; }
      if (c < r1 && pre <= lb && lb < pre + cand) { D.cut = c; D.slots_left = lb - pre; }
      run_before += tot;
    }
    __syncthreads();
  }
  if (t < 32) {
    const bool aborting = D.abort_key != ~0ull;
    const int cut = D.cut;
    const int sc = D.spec_cut < 0 ? 0 : (D.spec_cut > nT ? nT : D.spec_cut);
    int lo = 1, hi = 0;
    if (!aborting) {
      if (sc <= cut) { lo = sc; hi = (cut < nT && D.slots_left > 0) ? cut : cut - 1; }
      else { lo = cut; hi = sc - 1; }
    }
    const int redo = aborting ? 2 : (lo <= hi ? 1 : 0);
    if (t == 0) { D.redo = redo; D.lo = lo; D.hi = hi; }
    if (write_global) {
      Scalars s;
      s.abort_key = D.abort_key; s.total = D.total; s.in_progress = D.in_progress; s.budget = D.budget; s.avail = D.avail;
      s.max_unav = D.max_unav; s.node_offset = D.node_offset; s.cand_before = D.cand_before;
      write_counters(P, D.V, s, redo == 2 ? (long long)nT : (redo == 1 ? (long long)(hi - lo + 1) : 0), false);
      if (t == 0 && P.spec_sig != 0 && slotted && !aborting) {
        P.ws->hint_cut[P.parity] = cut;  // where the budget really cut this time = next call's speculation
        P.ws->hint_sig[P.parity] = P.spec_sig;
      }
    }
  }
  __syncthreads();
}

// Cluster-wide vector for world > 1 without a host-launched collective (verification kernel, every CTA): CTA 0 pushes
// this shard's lanes into every rank's mailbox over NVLink - one 8-byte store per half lane and peer, all of them in
// flight at once, each word tagged with the call number, so nothing has to be fenced or flagged; every CTA polls the
// words of every rank in the OWN mailbox (local memory) until they carry this call's number, and sums for itself - no
// intra-GPU broadcast, no CTA waits for another CTA of its grid. One-hot per-rank lanes make the sum an all-gather.
// Returns false when a peer did not show up in time.
__device__ __forceinline__ void st_mbox(unsigned long long* p, unsigned long long v) {
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_mbox(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ inline bool exchange_vector(const UstParams& P, DecideShared& D, bool pusher) {
  const int t = threadIdx.x, nt = blockDim.x;
  const int par = (int)(P.epoch & 1);
  const unsigned long long tag = (unsigned long long)(unsigned)P.epoch << 32;
  if (pusher && t >= 64) {
    // warps 0 and 1 push nothing: they publish the sum to the other CTAs of this grid afterwards (ust_verify_kernel), and
    // their release must not have to wait for this CTA's NVLink stores to be acknowledged by the peers
    for (int i = t - 64; i < P.world * UST_MBOX_WORDS; i += nt - 64) {
      const int r = i / UST_MBOX_WORDS, w = i - r * UST_MBOX_WORDS;
      const unsigned long long lane = (unsigned long long)D.V[w >> 1];
      const unsigned long long half = (w & 1) ? (lane >> 32) : (lane & 0xFFFFFFFFull);
      st_mbox(&P.mbox[r]->slot[par][P.rank][w], tag | half);
    }
  }
  __syncthreads();  // D.V is about to be overwritten with the sum
  // word w of rank r: thread (r * WORDS + w) when the block is wide enough, else a strided loop
  int ok = 1;
  const unsigned long long t0 = now_ns();
  long long mine[(UST_MAX_WORLD * UST_MBOX_WORDS + 255) / 256];   // the kernel runs at least 256 threads
  int k = 0;
  for (int i = t; i < P.world * UST_MBOX_WORDS; i += nt, k++) {
    const int r = i / UST_MBOX_WORDS, w = i - r * UST_MBOX_WORDS;
    const unsigned long long* src = &P.mbox[P.rank]->slot[par][r][w];
    unsigned long long v = ld_mbox(src);
    while ((v >> 32) != (tag >> 32)) {
      if (now_ns() - t0 > kCommTimeoutNs) { ok = 0; break; }
      __nanosleep(20);
      v = ld_mbox(src);
    }
    mine[k] = (long long)(v & 0xFFFFFFFFull);
  }
  if (t < UST_V_LEN) D.V[t] = 0;
  ok = __syncthreads_and(ok);
  // sum the halves into the lanes (shared-memory atomics: 84 x world adds)
  k = 0;
  for (int i = t; i < P.world * UST_MBOX_WORDS; i += nt, k++) {
    const int w = i % UST_MBOX_WORDS;
    atomicAdd(reinterpret_cast<unsigned long long*>(&D.V[w >> 1]), (unsigned long long)mine[k] << (32 * (w & 1)));
  }
  __syncthreads();
  return ok != 0;
}

}  // namespace ustd
