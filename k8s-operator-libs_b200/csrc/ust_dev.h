// ust_dev.h — structures shared by the host side of libust.so (ust_api.cu) and its kernels.
#pragma once
#include <stdint.h>

#include "../../include/ust.h"
#include "ust_lut.h"

#define UST_THREADS 256          /* auxiliary kernels */
#ifndef UST_VERIFY_THREADS
#define UST_VERIFY_THREADS 384   /* verification kernel */
#endif
#define UST_MAX_CTAS 1024        /* per-CTA diagnostic stamps */
#define UST_MAX_WORLD 8
#define UST_DS_SMEM_MAX 1024

// Streaming kernel geometry (ust_stream.cu): a tile is the unit a CTA claims, the TMA engine copies into one ring
// stage, and the slot speculation is made for. Tiles of fewer nodes (a multiple of 128) are used for small
// snapshots so that every SM gets work; the ring stages are sized for the largest.
#ifndef UST_TILE_NODES
#define UST_TILE_NODES 3072
#endif
#ifndef UST_STAGES
#define UST_STAGES 4
#endif
#ifndef UST_CONSUMER_WARPS
#define UST_CONSUMER_WARPS 12
#endif
#define UST_STREAM_THREADS (32 * (1 + UST_CONSUMER_WARPS))
// Streaming CTAs that must fit on one SM together with one verification CTA (checked at compile time, ust_stream.cu).
// 2 (a build variant, scripts/build_variants.py): the next call's CTA is resident and filling its ring while this
// call's CTA still streams (DESIGN.md §3.1, §3.3)
#ifndef UST_STREAM_CTAS_PER_SM
#define UST_STREAM_CTAS_PER_SM 1
#endif
// CTAs a streaming launch has per SM (1: co-residency serves the next call; 2: one call fills both slots)
#ifndef UST_STREAM_GRID_PER_SM
#define UST_STREAM_GRID_PER_SM 1
#endif
#define UST_STREAM_MAXREG 64     /* __maxnreg__ of the streaming kernel */
#ifndef UST_VERIFY_MAXREG
#define UST_VERIFY_MAXREG 80     /* __maxnreg__ of the verification kernel */
#endif
#define UST_VERIFY_SMEM_MAX 6144 /* static shared memory of the verification kernel (asserted in ust_kernels.cu) */

// Exchange vector (int64 lanes): what one shard contributes to / learns from the cluster-wide
// constraint arithmetic (upgrade_inplace.go:49-62). Summed across shards; per-rank slots are one-hot,
// so the sum doubles as an all-gather.
#define UST_V_HIST 0                         /* 16 lanes: nodes per state code */
#define UST_V_UNAVAILABLE 16
#define UST_V_CANDIDATES 17
#define UST_V_RANK_CAND (18)                 /* UST_MAX_WORLD lanes */
#define UST_V_RANK_NODES (18 + UST_MAX_WORLD)
#define UST_V_RANK_ERRINV (18 + 2 * UST_MAX_WORLD) /* ~abort key of the rank, 0 = none */
#define UST_V_LEN (18 + 3 * UST_MAX_WORLD)

// Peer mailboxes of the fused multi-GPU exchange: rank s writes its lanes into slot[epoch & 1][s] of EVERY rank's
// mailbox over NVLink (CUDA IPC mapping). Every 8-byte word carries half a lane and the call number
// ({data:32, epoch:32}, one 8-byte store each - delivered whole), so the data is its own flag: no fence, no separate
// flag store, the reader polls the words it needs.
#define UST_MBOX_WORDS (2 * UST_V_LEN)   /* 84 words = 672 B per slot */
struct UstMailbox {
  unsigned long long slot[2][UST_MAX_WORLD][UST_MBOX_WORDS + 12];
};

// Device workspace owned by a handle. The per-call accumulators exist twice: call k uses set (k & 1); the streaming
// kernel of call k+1 clears the set of call k (the verification kernel of call k, the only reader, has completed by
// then - stream order), so nobody ever waits for a reset. Invariant between calls: the set of the NEXT call is zero.
#define UST_MAX_SEGMENTS 16   /* streaming launches per call (pipelined uploads): one ticket each */
struct UstWorkspace {
  unsigned long long acc[2][18];  // hist[0..13], -, -, unavailable, candidates (this shard)
  unsigned long long errinv[2];   // ~min abort key seen while streaming, 0 = none
  unsigned int ticket[2][UST_MAX_SEGMENTS];  // dynamic tile claiming, one counter per streaming launch of the call
  int spec_used[2];               // the speculative cut the streaming kernel ran with
  unsigned long long bs_acc[18];  // BuildState kernels (zero between calls: their finish kernel clears it)
  unsigned int arrive;            // split mode: CTAs of the publishing streaming launch that have finished
  unsigned int comm_timeout;      // set when a peer did not show up (kernel gives up instead of hanging)
  // fused exchange: CTA 0 of the verification kernel talks to the peers; it leaves the summed vector here for the
  // other CTAs of its grid and then sets xflag = (epoch << 32) | ok (by epoch parity, like the mailboxes)
  long long xsum[2][UST_V_LEN];
  unsigned long long xflag[2];
  // Speculation hint carried from call to call (results never depend on it, only how many tiles are redone):
  // an earlier call's cut tile, valid for calls with the same signature (size, tiling, slot policy). One slot per
  // call parity: the verification kernel writes its own call's slot; a streaming kernel reads the previous call's slot
  // - or, when it runs beside the previous call's verification kernel (UstParams::relaxed), the slot of the call
  // before that, which nobody is writing.
  unsigned long long hint_sig[2];
  int hint_cut[2];
  // verification CTAs that have exited, ever (since the workspace was last cleared): a relaxed streaming kernel waits
  // until every verification kernel before the previous call's has finished before it touches its parity's set
  unsigned long long verify_done;
  // %globaltimer stamps per streaming CTA, by call parity: entry, first tile landed, stream end (all warps), exit;
  // and the SM it ran on
  unsigned long long dbg[2][UST_MAX_CTAS][4];
  unsigned int dbg_sm[2][UST_MAX_CTAS];
  unsigned long long dbg2[16];              // verification kernel, CTA 0: woken, vector loaded, decided, done; 4..: inside the decision
};

// abort key: (pass << 56) | (global node index + 1); policy-level aborts use index part 0
#define UST_KEY(pass, gidx_plus1) ((((unsigned long long)(pass)) << 56) | (unsigned long long)(gidx_plus1))

struct UstParams {
  long long n;  // nodes in this shard
  const uint8_t* hot;
  const uint32_t* flags;
  const int32_t* pod_rev;
  const int32_t* ds_idx;
  const int32_t* ds_rev;
  int n_ds;
  const int32_t* pod_off;     // nullable
  const uint16_t* pod_flags;  // nullable
  uint8_t* next;
  uint16_t* actions;
  uint8_t* outcome;  // nullable
  const uint32_t* lut;    // UST_LUT_ENTRIES words, then 16 uint2 lookup constants (ust_lut.h)
  const uint8_t* podlut;  // UST_PODLUT_ENTRIES bytes
  uint8_t* podsum;        // per-node pod-list summary (written by the pod-summary kernel, read by the streaming pass); null = no pod lists
  UstWorkspace* ws;
  unsigned int* cand_tile;  // upgrade candidates per tile (streaming pass writes, the decision reads)
  long long* xchg;        // UST_V_LEN lanes (split mode: the streaming kernel writes, the verification kernel reads the reduced copy)
  ust_counters* out;      // device
  // policy (flattened; see include/ust.h)
  long long max_parallel;
  long long max_unav_value;
  int max_unav_kind;
  int active;             // policy != nil && AutoUpgrade (upgrade_state.go:179-182); 0 => every node is a no-op
  int requestor;
  int pd_enabled;
  int pd_spec_present;
  int eval_pods;          // pod lists present and evaluate_actuators
  int spec_cut_tile;      // speculation: tiles before this index assume every upgrade candidate gets a slot
  unsigned long long spec_sig;  // signature under which a device-resident hint from the previous call applies (0 = none)
  // sharding
  int rank;
  int world;
  // tiling
  int tile_nodes;         // nodes per tile (a multiple of 128, 128 .. UST_TILE_NODES)
  int n_tiles;            // tiles of the shard
  int tile_begin;         // streaming sub-range launches (pipelined uploads): tiles [tile_begin, tile_end)
  int tile_end;
  int static_rounds;      // rounds of the range a CTA takes in stride order before it claims tiles by ticket
  int parity;             // which accumulator set of the workspace this call uses (call number & 1)
  int seg;                // index of this streaming launch within the call (its ticket counter)
  int publish;            // split mode: this streaming launch is the last one of the call, its last CTA publishes P.xchg
  int split;              // split mode: a host-launched collective reduces P.xchg between the two kernels
  int relaxed;            // the call does not depend on the previous call of the handle (see apply_device): its streaming kernel
                          // starts without waiting for that call's verification kernel and overlaps its tail
  unsigned long long verify_before;  // relaxed: UstWorkspace::verify_done once every verification kernel before the previous call's has finished
  int evict_first_inputs; // the input columns are read with L2 evict-first priority (the call's inputs fit in L2), else evict-normal
  int stamps;             // diagnostics: write %globaltimer stamps
  // fused multi-GPU exchange (world > 1): mailboxes of all ranks as mapped into this process, call number
  int fused_exchange;
  long long epoch;
  UstMailbox* mbox[UST_MAX_WORLD];
};

// kernel launchers; all return cudaError_t as int. `pdl` = launch with programmatic stream serialization.
int ust_launch_stream(const UstParams& p, int grid, void* stream, int pdl);   // ust_stream.cu
int ust_launch_verify(const UstParams& p, int grid, void* stream, int pdl);   // ust_kernels.cu
// also raises the dynamic shared-memory limit; `ctas_per_sm` = streaming CTAs an SM holds (occupancy API, fewest over the variants)
int ust_stream_config(int device, int* num_sms, size_t* smem_bytes, int* ctas_per_sm);
// `validation`: 0 = UST_EVAL_VALIDATION off; 1 = on, empty selector; 2 = on, walk the validation pods. An annotation that
// does not parse publishes its abort key into `errinv` (the call's UstWorkspace::errinv slot)
int ust_launch_pod_summary(long long n, int active, const uint8_t* hot, const int32_t* pod_off, const uint16_t* pod_flags,
                           long long n_pods, const uint8_t* podlut, uint8_t* podsum, const uint32_t* flags, int validation,
                           unsigned long long* errinv, int grid, void* stream);
int ust_launch_build_state(long long n, const uint8_t* hot, const int32_t* ds_idx, int n_ds, const int32_t* ds_desired,
                           unsigned long long* ds_count, UstWorkspace* ws, ust_counters* out, int grid, void* stream);
// slot of a 128-bit UID in the DaemonSet hash table (before masking to the table size); host build and device lookup
#ifdef __CUDACC__
__host__ __device__
#endif
static inline unsigned ust_uid_hash(unsigned long long x, unsigned long long y) {
  unsigned h = (unsigned)x * 0x9E3779B9u + (unsigned)(x >> 32) * 0x85EBCA6Bu + (unsigned)y * 0xC2B2AE35u + (unsigned)(y >> 32) * 0x27D4EB2Fu;
  return h ^ (h >> 15);
}
int ust_launch_build_state_uids(long long n, const uint8_t* hot, const void* owner_uid, int n_ds, const void* ds_tab,
                                const int32_t* ds_tab_idx, int tab_slots, const int32_t* ds_desired, int32_t* ds_idx_out,
                                unsigned long long* ds_count, UstWorkspace* ws, ust_counters* out, int grid, void* stream);
// resident driver-pod list (ust_build_state_delta): the join + count + diff pass and the finish kernel (`prev` holds each
// pod's previous owner index, `cur` receives the new one, tile_count one changed count per kBuildTile pods), then the scan
// of the tile counts and the ordered write of the changed (index, owner index) pairs, at most `cap` of them (four launches)
int ust_launch_build_state_delta(long long n, const uint8_t* hot, const void* owner_uid, int n_ds, const void* ds_tab,
                                 const int32_t* ds_tab_idx, int tab_slots, const int32_t* ds_desired, const int32_t* prev,
                                 int32_t* cur, unsigned int* tile_count, unsigned long long* ds_count, UstWorkspace* ws,
                                 ust_counters* out, int grid, void* stream);
int ust_launch_build_state_write(long long n, const int32_t* cur, const int32_t* prev, unsigned int* tile_count, long long* n_out,
                                 long long cap, long long* out_idx, int32_t* out_ds, void* stream);
int ust_build_state_tiles(long long n);
// the driver-pod list in a new order (runs as for ust_launch_reorder), inserted pods with previous owner index INT32_MIN
int ust_launch_build_state_reorder(long long n, long long n_runs, const long long* run_off, const long long* run_src,
                                   const uint8_t* ins_hot, const void* ins_uid, const uint8_t* hot, const void* uid,
                                   const int32_t* prev, uint8_t* o_hot, void* o_uid, int32_t* o_prev, void* stream);
int ust_launch_build_state_patch(long long m, const long long* idx, const uint8_t* state, const void* uid, uint8_t* hot_out,
                                 void* uid_out, void* stream);
// with start_out non-null (clocked pod-list deltas) the changed nodes' start times are scattered as well
int ust_launch_patch(long long m, const long long* idx, const uint8_t* state, const uint32_t* flags, const int32_t* pod_rev,
                     const int32_t* ds_idx, uint8_t* hot_out, uint32_t* flags_out, int32_t* rev_out, int32_t* ds_out, void* stream,
                     const long long* start = nullptr, long long* start_out = nullptr);
// clocked pod-list calls: bits 18 and 27 of the wait-for-jobs-required and validation-required nodes' flags, derived in place
// from their start times (include/ust.h, ust_clock); hot carries 16 bytes of padding. The same launch lists the candidates
// of the call's next deadline (ust_next_deadline): CTA b of the launch writes up to `region` candidates into cand
// [b * region, (b + 1) * region) (32-bit offsets among the CTA's own nodes) and their count into cand_count[b], and resets *deadline (n == 0: a memset does). The
// deadline launch behind the verification kernel (`p`: the call's parameters) evaluates them and min-reduces into *deadline:
// the smallest d = start + timeout (wrapped) whose flip changes the node's entry, with its sign bit flipped; ~0 = none.
// `validation` as for ust_launch_pod_summary.
struct UstClockGrid {
  int ctas;            // CTAs of both launches (0 when n == 0)
  long long region;    // candidate slots per CTA: cand holds ctas * region entries
};
UstClockGrid ust_clock_grid(long long n, int grid);
int ust_launch_clock(long long n, const uint8_t* hot, uint32_t* flags, const long long* start, long long now, long long wait_timeout,
                     const UstClockGrid& g, uint32_t* cand, unsigned int* cand_count, unsigned long long* deadline, void* stream);
int ust_launch_deadline(const UstParams& p, const UstClockGrid& g, const uint32_t* cand, const unsigned int* cand_count,
                        const long long* start, long long wait_timeout, int validation, long long n_pods, unsigned long long* deadline,
                        void* stream);
// membership splice (ust_apply_state_delta_splice): the resident columns and the previous outputs, rewritten in the new node
// order into the o_* arrays (n - n_rm + n_ins entries); rm / ib sorted and checked by the caller
int ust_launch_splice(long long n, long long n_rm, const long long* rm, long long n_ins, const long long* ib, const uint8_t* ins_hot,
                      const uint32_t* ins_flags, const int32_t* ins_rev, const int32_t* ins_ds, const uint8_t* hot, const uint32_t* flags,
                      const int32_t* rev, const int32_t* ds, const uint8_t* next, const uint16_t* act, uint8_t* o_hot, uint32_t* o_flags,
                      int32_t* o_rev, int32_t* o_ds, uint8_t* o_next, uint16_t* o_act, void* stream);
// new node order of the resident snapshot (ust_apply_state_delta_reorder): the resident columns and the previous
// outputs, gathered into the o_* arrays (n entries). Run r covers new positions [run_off[r], run_off[r + 1]) and reads old
// nodes from run_src[r] on, or inserted nodes from -1 - run_src[r] on (run_src[r] < 0); checked by the caller. With `oc`
// non-null (ust_apply_state_delta_pods_reorder) the previous actuator_outcome is gathered into o_oc as well, and with o_start
// non-null as well (clocked) the start times into o_start (inserted nodes from ins_start)
int ust_launch_reorder(long long n, long long n_runs, const long long* run_off, const long long* run_src, const uint8_t* ins_hot,
                       const uint32_t* ins_flags, const int32_t* ins_rev, const int32_t* ins_ds, const uint8_t* hot, const uint32_t* flags,
                       const int32_t* rev, const int32_t* ds, const uint8_t* next, const uint16_t* act, const uint8_t* oc, uint8_t* o_hot,
                       uint32_t* o_flags, int32_t* o_rev, int32_t* o_ds, uint8_t* o_next, uint16_t* o_act, uint8_t* o_oc, void* stream,
                       const long long* ins_start = nullptr, const long long* start = nullptr, long long* o_start = nullptr);
// rollout simulation: the clock of the feedback between two reconciles (include/ust.h, ust_sim_options)
struct UstSimParams {
  int timed;            // 0: whatever a node waits for has happened by the next reconcile
  long long now, dt;    // time of the reconcile that was just evaluated, seconds to the next one
  long long wait_timeout, job_seconds, validation_seconds, validation_timeout, maintenance_seconds;
};
int ust_launch_feedback(long long n, uint8_t* hot, uint32_t* flags, int32_t* pod_rev, const int32_t* ds_idx, int n_ds,
                        const int32_t* ds_rev, const uint8_t* next, const uint16_t* actions, const uint8_t* outcome,
                        const ust_counters* step, const UstSimParams& sp, int32_t* entered, int32_t* wait_start,
                        int32_t* valid_start, int grid, void* stream);
int ust_launch_sim_init(long long n, const uint32_t* flags, int32_t* entered, int32_t* wait_start, int32_t* valid_start, int grid,
                        void* stream);
int ust_launch_widen(long long n, const uint16_t* rev16, const int8_t* ds8, int32_t* rev_out, int32_t* ds_out, int grid,
                     void* stream);
// sparse outputs of a delta call: nodes whose (next_state, actions) differ from the previous call's, in node order; with
// `outcome` non-null (pod-list deltas) also those whose actuator_outcome differs, which is then written to out_outcome
int ust_launch_diff(long long n, const uint8_t* next, const uint16_t* actions, const uint8_t* outcome, const uint8_t* prev_next,
                    const uint16_t* prev_actions, const uint8_t* prev_outcome, unsigned int* block_count, long long* n_out, long long cap,
                    long long* out_idx, uint8_t* out_next, uint16_t* out_actions, uint8_t* out_outcome, void* stream);
int ust_diff_blocks(long long n);
// replacement pod lists of the resident pod-list snapshot (ust_apply_state_delta_pods), checked by the caller: list k
// (new_flags[new_off[k] .. new_off[k + 1])) replaces the list of node node_idx[k]. Same lengths: copied in place into
// flags at the offsets in off (one launch). Otherwise: new offsets into o_off (n + 1) and the new CSR into o_flags
// (new_total pods + 16 of padding), with shift[k] = sum over j < k of the length change of list j and `runs` holding
// 4 n_lists + 3 entries (two launches)
int ust_launch_pods_scatter(long long n_lists, const long long* node_idx, const int32_t* new_off, const uint16_t* new_flags,
                            const int32_t* off, uint16_t* flags, int grid, void* stream);
int ust_launch_pods_relayout(long long n, long long n_lists, const long long* node_idx, const int32_t* new_off, const int32_t* shift,
                             const int32_t* off, const uint16_t* flags, const uint16_t* new_flags, int new_total, int32_t* runs,
                             int32_t* o_off, uint16_t* o_flags, int grid, void* stream);
// the pod-list CSR of the resident pod-list snapshot in a new node order (ust_apply_state_delta_pods_reorder), checked by
// the caller: n_segs segments of the new snapshot, each a stretch of consecutive old nodes or one new list. segs holds
// seg_node (n_segs + 1 entries: first new node of each segment, then n) and seg_src (n_segs: first old node, or -1 - k for
// list k of new_off / new_flags); seg_pods holds pod_start (n_segs + 1: first new pod of each segment, then new_total) and
// room for n_segs more entries that the first launch fills. New offsets into o_off (n + 1), the new CSR into o_flags
// (new_total pods + 16 of padding); two launches
int ust_launch_pods_reorder(long long n, long long n_segs, const long long* segs, int32_t* seg_pods, const int32_t* off,
                            const uint16_t* flags, const int32_t* new_off, const uint16_t* new_flags, int new_total, int32_t* o_off,
                            uint16_t* o_flags, int grid, void* stream);
