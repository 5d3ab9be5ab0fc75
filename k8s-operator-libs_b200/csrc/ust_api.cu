// ust_api.cu — host side of libust.so: the C ABI of include/ust.h over the kernels of ust_kernels.cu.
// No node is ever evaluated on the CPU here; without an sm_90 device every computing call fails.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>  // types only; the library is resolved with dlopen when ust_comm_init is called

#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <chrono>
#include <mutex>
#include <string>
#include <vector>

#include "ust_dev.h"

namespace {

thread_local std::string g_create_error;

struct NcclApi {
  void* lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  bool load(std::string* err) {
    if (lib) return true;
    // prefer a copy already mapped into the process (e.g. the one PyTorch ships), then the system one
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* n : names) {
      lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL | RTLD_NOLOAD);
      if (lib) break;
    }
    for (const char* n : names) {
      if (lib) break;
      lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
    }
    if (!lib) { *err = std::string("cannot load libnccl: ") + dlerror(); return false; }
    GetUniqueId = (decltype(GetUniqueId))dlsym(lib, "ncclGetUniqueId");
    CommInitRank = (decltype(CommInitRank))dlsym(lib, "ncclCommInitRank");
    AllReduce = (decltype(AllReduce))dlsym(lib, "ncclAllReduce");
    AllGather = (decltype(AllGather))dlsym(lib, "ncclAllGather");
    CommDestroy = (decltype(CommDestroy))dlsym(lib, "ncclCommDestroy");
    GetErrorString = (decltype(GetErrorString))dlsym(lib, "ncclGetErrorString");
    if (!GetUniqueId || !CommInitRank || !AllReduce || !CommDestroy) { *err = "libnccl lacks required symbols"; return false; }
    return true;
  }
};
NcclApi g_nccl;
std::mutex g_nccl_mu;

// A growable device buffer that owns its memory. Move-only: std::swap hands the allocations over, a copy would free
// them twice.
template <class T>
struct DevBuf {
  T* p = nullptr;
  size_t cap = 0;  // elements
  DevBuf() = default;
  DevBuf(DevBuf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
  DevBuf& operator=(DevBuf&& o) noexcept { std::swap(p, o.p); std::swap(cap, o.cap); return *this; }
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { if (p) cudaFree(p); }
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    size_t want = cap ? cap : 1024;
    while (want < n) want += want / 2 + 1024;  // geometric growth
    T* q = nullptr;
    cudaError_t e = cudaMalloc(&q, want * sizeof(T));
    if (e != cudaSuccess) return e;
    if (p) cudaFree(p);
    p = q;
    cap = want;
    return cudaSuccess;
  }
};

// The four input columns of a set of nodes. The padding lets the kernels' 16-byte loads run past the last node.
struct Columns {
  DevBuf<uint8_t> hot;
  DevBuf<uint32_t> flags;
  DevBuf<int32_t> rev, ds;
  cudaError_t reserve(size_t n) {
    cudaError_t e = hot.reserve(n + 16);
    if (e == cudaSuccess) e = flags.reserve(n + 4);
    if (e == cudaSuccess) e = rev.reserve(n + 4);
    if (e == cudaSuccess) e = ds.reserve(n + 4);
    return e;
  }
  // nodes [first, first + count) of the host columns; null rev / ds are not copied (packed format: widened on the device)
  cudaError_t upload(const uint8_t* state, const uint32_t* f, const int32_t* r, const int32_t* d, size_t first, size_t count,
                     cudaStream_t st) {
    if (!count) return cudaSuccess;
    cudaError_t e = cudaMemcpyAsync(hot.p + first, state + first, count, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(flags.p + first, f + first, count * 4, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess && r) e = cudaMemcpyAsync(rev.p + first, r + first, count * 4, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess && d) e = cudaMemcpyAsync(ds.p + first, d + first, count * 4, cudaMemcpyHostToDevice, st);
    return e;
  }
};

// Nodes given by index: the re-encoded nodes of a delta call, the inserted nodes of a splice.
struct IndexedColumns {
  DevBuf<long long> idx;
  Columns cols;
};

// The outputs of one evaluation.
struct Outputs {
  DevBuf<uint8_t> next;
  DevBuf<uint16_t> actions;
  cudaError_t reserve(size_t n) {
    cudaError_t e = next.reserve(n + 16);
    return e == cudaSuccess ? actions.reserve(n + 8) : e;
  }
};

}  // namespace

struct ust_handle {
  int device = -1;
  cudaStream_t stream = nullptr;
  cudaStream_t stream_d2h = nullptr;   // pipelined host path: downloads, kernels and uploads on three streams
  cudaStream_t stream_h2d = nullptr;
  cudaEvent_t seg_done[16] = {};
  cudaEvent_t seg_up[16] = {};
  cudaEvent_t d2h_done = nullptr;
  std::mutex mu;
  std::string err;
  int64_t launches = 0;
  int num_sms = 0;
  size_t stream_smem = 0;   // dynamic shared memory of the streaming kernel (largest variant)
  size_t l2_bytes = 0;      // L2 cache of the device
  int stream_ctas_per_sm = 0;   // streaming CTAs an SM holds (occupancy API, fewest over the variants)
  unsigned long long verify_ctas = 0;  // verification CTAs launched since the workspace was cleared (UstWorkspace::verify_done)
  bool ws_dirty = false;
  bool pdl = true;          // launch the kernels of a call with programmatic dependent launch (UST_PDL=0 turns it off: tuning)
  bool stamps = false;      // UST_STAMPS: per-CTA %globaltimer stamps (diagnostics)
  int static_pct = 75;      // share of a launch's tile rounds taken in stride order before the ticket (UST_STATIC_PCT: tuning)
  unsigned call_seq = 0;    // calls whose kernels were launched: call k uses accumulator set k & 1 of the workspace
  // the previous call's buffers, when its kernels are the last thing enqueued on the handle's own stream (else n = -1):
  // a call that touches none of them does not wait for it (UstParams::relaxed)
  struct Span { const char* p; size_t len; };
  Span prev_in[4] = {}, prev_out[3] = {};
  int64_t prev_n = -1;
  bool chain_entry = false;     // set by ust_apply_state_device for the apply_device call it makes
  int64_t relaxed_calls = 0;   // diagnostics
  bool overlap_calls = true;  // UST_OVERLAP=0 turns the overlap of independent back-to-back calls off (tuning)
  cudaStream_t last_stream = nullptr;  // stream of the previous device-resident call (calls on another stream are ordered behind it)
  // set by adopt_resident / drop_resident only
  int64_t resident_n = -1;  // nodes of the snapshot the last ust_apply_state left in the staging arrays (-1 = none)
  int32_t resident_n_ds = 0;  // ... and the size of its DaemonSet table
  bool outputs_resident = false;  // `outs` holds the outputs of the last call on the resident snapshot
  // the resident pod-list snapshot (ust_apply_state_delta_pods): nodes in `staged`, pod lists in s_podoff / s_podflags,
  // outputs in `outs` and s_outcome. Only the pod-list entry points see it.
  int64_t pods_n = -1;      // its nodes (-1 = none)
  int64_t pods_total = 0;   // its pods
  bool pods_clocked = false;  // it was left by a clocked call: its start times are in s_start (ust_apply_state_clocked)
  DevBuf<ust_counters> sim_hist;  // rollout simulation: one ust_counters per simulated reconcile
  int segments = 6;      // upload / compute / download pipeline depth of the host path (UST_SEGMENTS, tuning)
  bool no_hint = false;  // UST_NO_HINT=1 (tuning): every call speculates from the policy default, never from the previous call

  UstWorkspace* ws = nullptr;
  uint32_t* lut_dev = nullptr;      // UST_LUT_WORDS words
  uint8_t* podlut_dev = nullptr;
  uint32_t* lut_host = nullptr;     // pinned staging copy
  uint8_t* podlut_host = nullptr;   // pinned
  ust_policy lut_policy;            // policy the device tables were built for
  bool lut_valid = false;
  ust_counters* counters_dev = nullptr;
  ust_counters* counters_host = nullptr;  // pinned
  long long* xchg_dev = nullptr;
  DevBuf<unsigned long long> ds_count;  // BuildState: pods per DaemonSet (zero between calls)

  // staging for the host-pointer API; `staged` and `outs` hold the resident snapshot and its outputs
  Columns staged;
  Outputs outs;
  DevBuf<uint8_t> s_outcome, s_outcome_prev;  // actuator_outcome; the previous call's (pod-list deltas: swapped like outs / outs_prev)
  DevBuf<int32_t> s_dsrev, s_podoff, s_dsdesired;
  DevBuf<uint16_t> s_rev16;          // packed host format: interned pod revisions / DaemonSet indices as uploaded
  DevBuf<int8_t> s_ds8;
  DevBuf<uint16_t> s_podflags;
  DevBuf<uint8_t> s_podsum;
  DevBuf<unsigned int> s_candtile[2];   // upgrade candidates per tile of the current call (by call parity: the previous
                                        // call's verification kernel may still be reading its own)
  // sparse delta outputs: the previous call's outputs, block counts, compacted entries
  Outputs outs_prev, outs_sparse;
  DevBuf<unsigned int> sp_blocks;
  DevBuf<long long> sp_idx;
  long long* sp_count_dev = nullptr;
  long long* sp_count_host = nullptr;  // pinned
  DevBuf<uint64_t> s_uid, s_dsuid;   // BuildState owner join: pod owner UIDs, DaemonSet UID hash table (+ s_dsorder: slot -> index)
  DevBuf<int32_t> s_dsorder;
  IndexedColumns changed;            // delta updates: indices and values of the changed nodes
  // pod-list deltas: the replaced lists as uploaded (node indices, offsets, pods, length-change prefix), the run table of a
  // relayout, the second CSR pair a relayout writes (swapped with s_podoff / s_podflags; allocated on the first relayout),
  // the sparse outcomes; on the host the list length of every node of the pod-list snapshot, and the lengths the
  // checks of a pod-list ust_apply_state fill (swapped in when that call leaves its snapshot resident)
  DevBuf<long long> pl_idx;
  DevBuf<int32_t> pl_off, pl_shift, pl_runs, s_podoff2;
  DevBuf<uint16_t> pl_flags, s_podflags2;
  DevBuf<uint8_t> sp_outcome;
  std::vector<int32_t> pod_len, pod_len_next, pl_shift_host;
  // new node order (splice, reorder): the second set the splice / gather kernel writes (swapped with the resident columns
  // and the previous outputs afterwards; allocated on the first such call), the removal list, the reorder's runs
  // (run_off, then run_src: see add_run) and the inserted nodes with their positions (splice); run_seen: one bit per old
  // node while a reorder is checked, all zero between calls
  Columns splice_cols;
  Outputs splice_outs;
  DevBuf<long long> removed, runs;
  IndexedColumns inserted;
  std::vector<long long> run_off, run_src;
  std::vector<uint64_t> run_seen;
  // a reorder of the pod-list snapshot: the previous outcome in the new order (swapped with s_outcome), the segments of
  // the new pod CSR (seg_node, seg_src / pod_start, pod_src: see ust_launch_pods_reorder) and their host copies
  DevBuf<uint8_t> splice_outcome;
  DevBuf<long long> pr_segs;
  DevBuf<int32_t> pr_pods;
  std::vector<long long> seg_node, seg_src;
  std::vector<int32_t> seg_pod;
  long long pod_pass_ns = 0;  // diagnostics: host time of the last pods_reorder_segments
  DevBuf<int32_t> sim_entered, sim_wait, sim_valid;  // timed rollout simulation: per-node clocks
  // clocked pod-list calls: the start time of every node of the pod-list snapshot, the gather target of a reorder (swapped
  // with it afterwards), the starts of the changed and of the inserted nodes as uploaded. Only clocked calls allocate them.
  DevBuf<long long> s_start, s_start2, chg_start, ins_start;
  // the next deadline of a clocked call (ust_next_deadline): the clock launch's geometry, its candidate list and per-CTA
  // counts, the reduced value; deadline_ready: the last ApplyState, BuildState or simulation call on the handle was a clocked
  // call that left its snapshot resident (set by adopt_resident, cleared by every such entry point)
  UstClockGrid clk_grid = {0, 0};
  DevBuf<uint32_t> clk_cand;
  DevBuf<unsigned int> clk_count;
  DevBuf<unsigned long long> clk_deadline;
  bool deadline_ready = false;
  // the resident driver-pod list of ust_build_state_delta (bs_n pods, 0 until the first call; nothing else reads or drops
  // it): state bytes, owner UIDs and the owner indices of the last call in `bs`. `bs2` is the gather target of a reorder
  // (hot / uid allocated on the first reorder; swapped with `bs` afterwards); bs2.owner receives a call's owner indices
  // (swapped with bs.owner afterwards). The joined and the overwritten pods as uploaded; the sparse owner indices.
  struct PodList {
    DevBuf<uint8_t> hot;
    DevBuf<uint64_t> uid;
    DevBuf<int32_t> owner;
  };
  PodList bs, bs2;
  int64_t bs_n = 0;
  DevBuf<uint8_t> bs_ins_hot, bs_chg_hot;
  DevBuf<uint64_t> bs_ins_uid, bs_chg_uid;
  DevBuf<int32_t> bs_out_ds;

  // multi-GPU
  int rank = 0, world = 1, comm_mode = 0;
  ncclComm_t comm = nullptr;
  // fused exchange: own mailbox + the peers' mailboxes mapped through CUDA IPC
  UstMailbox* mbox_own = nullptr;
  UstMailbox* mbox[UST_MAX_WORLD] = {};
  bool mbox_ready = false;
  long long epoch = 0;

  int fail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    err = buf;
    return code;
  }
};

#define UST_CUDA(h, call)                                                                                   \
  do {                                                                                                      \
    cudaError_t e_ = (call);                                                                                \
    if (e_ != cudaSuccess) return (h)->fail(UST_ERR_CUDA, "%s failed: %s", #call, cudaGetErrorString(e_)); \
  } while (0)

// after a call that failed half-way: the workspace starts over (with it the count of finished verification CTAs)
static cudaError_t clear_workspace(ust_handle* h, cudaStream_t st) {
  h->verify_ctas = 0;
  return cudaMemsetAsync(h->ws, 0, sizeof(UstWorkspace), st);
}

static bool policy_active(const ust_policy* p) { return p != nullptr && p->auto_upgrade != 0; }

// tables depend on these fields only
static ust_policy table_key(const ust_policy* p) {
  ust_policy k;
  memset(&k, 0, sizeof(k));
  if (!policy_active(p)) return k;  // all-noop tables
  k = *p;
  k.max_parallel_upgrades = 0;
  k.max_unavailable_kind = 0;
  k.max_unavailable_value = 0;
  return k;
}

static int ensure_tables(ust_handle* h, const ust_policy* p, cudaStream_t st) {
  const ust_policy key = table_key(p);
  if (h->lut_valid && memcmp(&key, &h->lut_policy, sizeof(key)) == 0) return UST_OK;
  UST_CUDA(h, cudaStreamSynchronize(st));  // the pinned staging copy may still be in flight
  if (policy_active(p)) {
    ust_build_lut(&key, h->lut_host);
    ust_build_pod_lut256(&key, h->podlut_host);
  } else {
    ust_build_lut(nullptr, h->lut_host);
    memset(h->podlut_host, 0, UST_PODLUT_ENTRIES);
  }
  UST_CUDA(h, cudaMemcpyAsync(h->lut_dev, h->lut_host, UST_LUT_WORDS * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
  UST_CUDA(h, cudaMemcpyAsync(h->podlut_dev, h->podlut_host, UST_PODLUT_ENTRIES, cudaMemcpyHostToDevice, st));
  h->lut_policy = key;
  h->lut_valid = true;
  return UST_OK;
}

// Tiling of a shard: tiles of UST_TILE_NODES nodes; smaller tiles (halved, multiples of 128) when the snapshot is so small that
// full-size tiles would leave CTAs without work. UST_STREAM_GRID_PER_SM persistent CTAs per SM, never more CTAs than tiles.
static int max_grid(const ust_handle* h) { return h->num_sms * UST_STREAM_GRID_PER_SM; }
static int pick_tile_nodes(const ust_handle* h, int64_t n) {
  int tn = UST_TILE_NODES;
  // at least one tile per CTA; a CTA keeps up to UST_STAGES tiles in flight at once, so a small snapshot is one load
  // round trip whatever its tile size - and larger tiles mean larger (more efficient) bulk copies
  while (tn > 128 && n / tn < (int64_t)max_grid(h)) { tn = (tn / 2) & ~127; if (tn < 128) tn = 128; }  // multiples of 128 nodes
  return tn;
}
static int pick_grid(const ust_handle* h, int tiles) {
  const int g = tiles < max_grid(h) ? tiles : max_grid(h);
  return g < 1 ? 1 : g;
}
// rounds of a launch's tile range that a CTA takes in stride order before it starts claiming tiles by ticket
static int pick_static_rounds(const ust_handle* h, int tiles, int grid) {
  const int rounds = tiles / grid;
  int r = (int)((int64_t)rounds * h->static_pct / 100);
  if (rounds - r < 2) r = rounds - 2;
  if (r < 1 && rounds >= 1) r = 1;  // the first round never waits for a ticket
  return r < 0 ? 0 : r;
}

// UST_EVAL_VALIDATION answers Validate from the pod lists: it needs them, and the actuator evaluation it is part of
static int check_eval_mode(ust_handle* h, const ust_policy* p, bool pods) {
  if (!p || !(p->evaluate_actuators & UST_EVAL_VALIDATION)) return UST_OK;
  if (!(p->evaluate_actuators & UST_EVAL_ACTUATORS))
    return h->fail(UST_ERR_INVALID_ARGUMENT, "evaluate_actuators: UST_EVAL_VALIDATION requires UST_EVAL_ACTUATORS");
  if (!pods) return h->fail(UST_ERR_INVALID_ARGUMENT, "evaluate_actuators: UST_EVAL_VALIDATION requires pod lists, which this call has not");
  return UST_OK;
}

static int check_aligned(ust_handle* h, const void* p, const char* what) {
  if (((uintptr_t)p & 15u) != 0) return h->fail(UST_ERR_INVALID_ARGUMENT, "%s must be 16-byte aligned", what);
  return UST_OK;
}

// The start of every evaluation enqueued on `st` (apply_device, apply_pipelined): orders it behind the previous call,
// builds the tables and the launch parameters, and takes the call's exchange epoch and workspace parity.
static int begin_call(ust_handle* h, const ust_policy* policy, int64_t n, const uint8_t* state, const uint32_t* flags,
                      const int32_t* pod_rev, const int32_t* ds_idx, int32_t n_ds, const int32_t* ds_rev,
                      const int32_t* pod_off, const uint16_t* pod_flags, uint8_t* next_state, uint16_t* actions,
                      uint8_t* outcome, ust_counters* out_dev, cudaStream_t st, UstParams* out, int* grid_out) {
  // a handle's workspace, tables and counters serve one call at a time: a call on another stream than the previous
  // one is ordered behind it (calls on the same stream are ordered by the stream)
  if (h->last_stream && h->last_stream != st) UST_CUDA(h, cudaStreamSynchronize(h->last_stream));
  h->last_stream = st;
  if (h->ws_dirty) {
    UST_CUDA(h, clear_workspace(h, st));
    h->ws_dirty = false;
  }
  int rc = ensure_tables(h, policy, st);
  if (rc) return rc;
  const bool active = policy_active(policy);
  UstParams P;
  memset(&P, 0, sizeof(P));
  P.n = n;
  P.hot = state; P.flags = flags; P.pod_rev = pod_rev; P.ds_idx = ds_idx;
  P.ds_rev = ds_rev; P.n_ds = n_ds;
  P.pod_off = pod_off; P.pod_flags = pod_flags;
  P.next = next_state; P.actions = actions; P.outcome = outcome;
  P.lut = h->lut_dev; P.podlut = h->podlut_dev;
  P.ws = h->ws; P.xchg = h->xchg_dev;
  P.out = out_dev ? out_dev : h->counters_dev;
  P.active = active ? 1 : 0;
  if (active) {
    P.max_parallel = policy->max_parallel_upgrades;
    P.max_unav_value = policy->max_unavailable_value;
    P.max_unav_kind = policy->max_unavailable_kind;
    P.requestor = policy->use_maintenance_operator != 0;
    P.pd_enabled = policy->pod_deletion_enabled != 0;
    P.pd_spec_present = policy->pod_deletion_spec_present != 0;
    // pod lists given (even empty ones: "no pods" is an answer, not "unknown") and actuator evaluation asked for
    P.eval_pods = (policy->evaluate_actuators != 0 && pod_off) ? 1 : 0;
  }
  P.rank = h->rank;
  P.world = h->world;
  if (h->world > 1 && h->comm_mode == 1 && h->mbox_ready) {
    P.fused_exchange = 1;
    for (int r = 0; r < h->world; r++) P.mbox[r] = h->mbox[r];
  }
  P.split = (h->world > 1 && !P.fused_exchange) ? 1 : 0;
  // Speculative slot grant (verified by the call's last CTA, so only speed depends on it):
  // with no MaxParallelUpgrades / MaxUnavailable limit every candidate gets a slot (upgrade_inplace.go:49-62);
  // with limits the budget is normally tiny next to the number of candidates.
  P.spec_cut_tile = (active && policy->max_parallel_upgrades == 0 && policy->max_unavailable_kind == UST_MAXUNAVAIL_NIL) ? 0x7FFFFFFF : 0;
  const int tn = pick_tile_nodes(h, n);
  const int64_t tiles64 = (n + tn - 1) / tn;
  const int tiles = (int)tiles64;
  const int grid = pick_grid(h, tiles);
  if (active && !P.requestor && !h->no_hint) {
    // signature of everything the cut position depends on besides the data itself (FNV-1a)
    unsigned long long sig = 1469598103934665603ull;
    const long long parts[6] = {n, tn, policy->max_parallel_upgrades, policy->max_unavailable_kind, policy->max_unavailable_value, h->world * 64 + h->rank};
    for (long long v : parts) { sig ^= (unsigned long long)v; sig *= 1099511628211ull; }
    P.spec_sig = sig ? sig : 1;
  }
  P.tile_nodes = tn;
  P.n_tiles = tiles;
  P.tile_begin = 0;
  P.tile_end = tiles;
  P.static_rounds = pick_static_rounds(h, tiles, grid);
  P.publish = 1;
  P.stamps = (h->stamps && grid <= UST_MAX_CTAS) ? 1 : 0;
  // L2 priority of the streamed inputs. Inputs larger than the L2 (C3: 130 MB against 50 MB on an H100) are read with
  // normal priority: evict-first made a 10 M-node call 2.7 % slower (DESIGN.md §3.1). Inputs that fit keep evict-first,
  // which measured faster there (1 M nodes).
  P.evict_first_inputs = (size_t)n * 13u <= h->l2_bytes ? 1 : 0;
  for (auto& b : h->s_candtile) {
    // growing a buffer frees the old one: nothing of an earlier call may still be using it
    if ((size_t)tiles + 1 > b.cap && h->last_stream) cudaStreamSynchronize(h->last_stream);
    cudaError_t ce = b.reserve((size_t)tiles + 1);
    if (ce != cudaSuccess) return h->fail(UST_ERR_CUDA, "cudaMalloc failed: %s", cudaGetErrorString(ce));
  }
  if (P.fused_exchange) P.epoch = ++h->epoch;  // collective call number: identical on every rank
  P.parity = (int)(h->call_seq++ & 1u);
  P.cand_tile = h->s_candtile[P.parity].p;
  h->prev_n = -1;
  h->ws_dirty = true;  // cleared again once every launch of this call has been enqueued successfully
  *out = P;
  *grid_out = grid;
  return UST_OK;
}

// the verification kernel behind the streaming launches of a call (+ the collective, split mode)
static int launch_verify(ust_handle* h, UstParams& P, cudaStream_t st, bool pdl) {
  if (P.split) {
    ncclResult_t r = g_nccl.AllReduce(h->xchg_dev, h->xchg_dev, UST_V_LEN, ncclInt64, ncclSum, h->comm, st);
    if (r != ncclSuccess) return h->fail(UST_ERR_COMM, "ncclAllReduce failed: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?");
  }
  int e = ust_launch_verify(P, h->num_sms, st, (pdl && !P.split) ? 1 : 0);
  if (e) return h->fail(UST_ERR_CUDA, "verification kernel launch failed: %s", cudaGetErrorString((cudaError_t)e));
  h->launches += 1;
  h->verify_ctas += (unsigned long long)h->num_sms;
  return UST_OK;
}

// The pod CSR must be well-formed before a kernel walks it: pod_off[0] == 0, non-decreasing, pod_off[n] == n_pods.
// `lens` (nullable, n entries) receives the list lengths on the way.
static int check_pod_offsets_host(ust_handle* h, int64_t n, const int32_t* pod_off, int64_t n_pods, int32_t* lens = nullptr) {
  if (n == 0) return UST_OK;
  if (pod_off[0] != 0) return h->fail(UST_ERR_INVALID_ARGUMENT, "pod_off[0] must be 0");
  for (int64_t i = 0; i < n; i++) {
    if (pod_off[i + 1] < pod_off[i]) return h->fail(UST_ERR_INVALID_ARGUMENT, "pod_off must not decrease (node %lld)", (long long)i);
    if (lens) lens[i] = pod_off[i + 1] - pod_off[i];
  }
  if ((int64_t)pod_off[n] != n_pods) return h->fail(UST_ERR_INVALID_ARGUMENT, "pod_off[n_nodes] must equal n_pods");
  return UST_OK;
}

static int launch_deadline(ust_handle* h, const UstParams& P, const ust_clock* clock, int validation, int64_t n_pods, cudaStream_t st);

// core: everything device-resident, enqueue on `st`. `clock` (clocked calls, whose clock kernel has run): the call's next
// deadline is evaluated behind the verification kernel.
static int apply_device(ust_handle* h, const ust_policy* policy, int64_t n, const uint8_t* state, const uint32_t* flags,
                        const int32_t* pod_rev, const int32_t* ds_idx, int32_t n_ds, const int32_t* ds_rev,
                        const int32_t* pod_off, const uint16_t* pod_flags, int64_t n_pods, uint8_t* next_state,
                        uint16_t* actions, uint8_t* outcome, ust_counters* out_dev, cudaStream_t st,
                        const ust_clock* clock = nullptr) {
  const bool chain = h->chain_entry;  // called by ust_apply_state_device itself: the call may overlap the previous one
  h->chain_entry = false;
  if (!chain) h->prev_n = -1;
  if (n < 0) return h->fail(UST_ERR_NIL_STATE, "currentState should not be empty");
  if (n > 0 && (!state || !flags || !pod_rev || !ds_idx || !next_state || !actions))
    return h->fail(UST_ERR_NIL_STATE, "currentState should not be empty");
  if (n_ds < 0 || (n_ds > 0 && !ds_rev)) return h->fail(UST_ERR_INVALID_ARGUMENT, "bad DaemonSet table");
  if (n >= (1LL << 40)) return h->fail(UST_ERR_INVALID_ARGUMENT, "too many nodes");
  const void* ptrs[] = {state, flags, pod_rev, ds_idx, next_state, actions, outcome};
  const char* names[] = {"state", "flags", "pod_rev", "ds_idx", "next_state", "actions", "actuator_outcome"};
  for (int i = 0; i < 7; i++)
    if (ptrs[i]) { int rc = check_aligned(h, ptrs[i], names[i]); if (rc) return rc; }
  if (pod_off && pod_flags) { int rc = check_aligned(h, pod_flags, "pod_flags"); if (rc) return rc; }
  UST_CUDA(h, cudaSetDevice(h->device));
  const bool prev_known = h->prev_n >= 0;  // the previous call's buffers (begin_call forgets them)
  UstParams P;
  int grid = 0;
  int rc = begin_call(h, policy, n, state, flags, pod_rev, ds_idx, n_ds, ds_rev, pod_off, pod_flags, next_state, actions,
                      outcome, out_dev, st, &P, &grid);
  if (rc) return rc;

  // UST_EVAL_VALIDATION: the validation-required nodes get their byte too (ust_lut.h); an empty selector reads no pod
  const int validation = !P.eval_pods || !ust_validation_mode(policy) ? 0 : (policy->validation_enabled ? 2 : 1);
  if (P.eval_pods) {
    // pod lists: one byte per node first (only the nodes whose actuator looks at its pods are read),
    // then the ordinary streaming pass with that byte as a fifth input stream
    UST_CUDA(h, h->s_podsum.reserve((size_t)n + 16));
    P.podsum = h->s_podsum.p;
    P.evict_first_inputs = 1;  // the pod-list pass was not measured faster with evict-normal inputs
    int e = ust_launch_pod_summary(n, P.active, P.hot, P.pod_off, P.pod_flags, n_pods, P.podlut, P.podsum, P.flags, validation,
                                   &P.ws->errinv[P.parity], h->num_sms * 6, st);
    if (e) return h->fail(UST_ERR_CUDA, "pod-summary kernel launch failed: %s", cudaGetErrorString((cudaError_t)e));
    h->launches += 1;
  }
  // Independent back-to-back calls overlap: when the last thing enqueued on the handle's own stream is the previous
  // call's verification kernel and this call reads nothing that call writes and writes nothing that call reads or
  // writes, its streaming kernel does not wait for it (programmatic dependent launch without the initial wait: the
  // CTAs of this call take over the SMs as the CTAs of that one run out of tiles, and that call's decision and exchange
  // run beside them). Everything else - another stream, pod lists, shared output arrays - keeps the strict order.
  ust_handle::Span in[4] = {{(const char*)state, (size_t)n}, {(const char*)flags, (size_t)n * 4}, {(const char*)pod_rev, (size_t)n * 4},
                            {(const char*)ds_idx, (size_t)n * 4}};
  ust_handle::Span outs[3] = {{(const char*)next_state, (size_t)n}, {(const char*)actions, (size_t)n * 2},
                             {(const char*)outcome, outcome ? (size_t)n : 0}};
  auto overlaps = [](const ust_handle::Span& a, const ust_handle::Span& b) {
    return a.len && b.len && a.p < b.p + b.len && b.p < a.p + a.len;
  };
  bool relaxed = chain && h->pdl && h->overlap_calls && st == h->stream && prev_known && !P.eval_pods && !P.split;
  for (int i = 0; relaxed && i < 3; i++) {
    for (int j = 0; j < 3; j++) relaxed = relaxed && !overlaps(outs[i], h->prev_out[j]);   // write / write
    for (int j = 0; j < 4; j++) relaxed = relaxed && !overlaps(outs[i], h->prev_in[j]);    // write / read (that call's redo)
  }
  for (int i = 0; relaxed && i < 4; i++)
    for (int j = 0; j < 3; j++) relaxed = relaxed && !overlaps(in[i], h->prev_out[j]);     // read / write
  P.relaxed = relaxed ? 1 : 0;
  h->relaxed_calls += relaxed ? 1 : 0;
  if (relaxed) {
    P.static_rounds = P.n_tiles / grid + 3;  // no tickets: a CTA's tiles are fixed, the next call fills the tail
    // the last verification kernel enqueued is the previous call's; every one before it must have finished before this
    // call touches its parity's set (DESIGN.md §3.3)
    P.verify_before = h->verify_ctas - (unsigned long long)h->num_sms;
  }
  int e = ust_launch_stream(P, grid, st, h->pdl ? 1 : 0);
  if (e) return h->fail(UST_ERR_CUDA, "streaming kernel launch failed: %s", cudaGetErrorString((cudaError_t)e));
  h->launches += 1;
  rc = launch_verify(h, P, st, h->pdl);
  if (rc) return rc;
  h->ws_dirty = false;
  if (clock) {
    rc = launch_deadline(h, P, clock, validation, n_pods, st);
    if (rc) return rc;
  }
  if (chain && st == h->stream && !P.eval_pods) {
    for (int i = 0; i < 4; i++) h->prev_in[i] = in[i];
    for (int i = 0; i < 3; i++) h->prev_out[i] = outs[i];
    h->prev_n = n;
  }
  return UST_OK;
}

static int finish_with_counters(ust_handle* h, cudaStream_t st, ust_counters* out, bool fetched = false) {
  if (!fetched) UST_CUDA(h, cudaMemcpyAsync(h->counters_host, h->counters_dev, sizeof(ust_counters), cudaMemcpyDeviceToHost, st));
  cudaError_t e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) {
    h->ws_dirty = true;
    return h->fail(UST_ERR_CUDA, "kernel execution failed: %s", cudaGetErrorString(e));
  }
  if (out) *out = *h->counters_host;
  const int code = (int)h->counters_host->error_code;
  if (code != UST_OK) {
    switch (code) {
      case UST_ERR_REVISION_HASH:
        return h->fail(code, "failed to get daemonset template/pod revision hash (node index %lld, pass %lld)",
                       (long long)h->counters_host->error_index, (long long)h->counters_host->error_pass);
      case UST_ERR_MAX_UNAVAILABLE: return h->fail(code, "failed to compute maxUnavailable from the current total nodes");
      case UST_ERR_POD_DELETION_SPEC: return h->fail(code, "pod deletion spec should not be empty");
      case UST_ERR_DS_UNSCHEDULED: return h->fail(code, "driver DaemonSet should not have Unscheduled pods");
      case UST_ERR_COMM: return h->fail(code, "multi-GPU exchange timed out: a peer rank did not take part in the call");
      default: return h->fail(code, "ApplyState aborted with code %d", code);
    }
  }
  return UST_OK;
}

// Host-pointer entry points hand caller-owned buffers to asynchronous copies: whatever way such a call ends, nothing
// of it may still be in flight when it returns (the caller may free or reuse the buffers).
struct StreamDrain {
  ust_handle* h;
  bool armed = true;
  explicit StreamDrain(ust_handle* hh) : h(hh) {}
  ~StreamDrain() {
    if (!armed) return;
    if (h->stream_h2d) cudaStreamSynchronize(h->stream_h2d);
    if (h->stream) cudaStreamSynchronize(h->stream);
    if (h->stream_d2h) cudaStreamSynchronize(h->stream_d2h);
  }
};

#pragma GCC visibility push(default)

// Host columns of ust_apply_state (wide), or of ust_apply_state_packed: uint16 pod revisions and int8 DaemonSet
// indices, 3 instead of 8 bytes per node over PCIe, widened on the device (rev and ds are then null).
struct HostNodes {
  const uint8_t* state;
  const uint32_t* flags;
  const int32_t* rev;
  const int32_t* ds;
  const uint16_t* rev16;
  const int8_t* ds8;
};

static int upload_nodes(ust_handle* h, const HostNodes& in, size_t first, size_t count, cudaStream_t st) {
  UST_CUDA(h, h->staged.upload(in.state, in.flags, in.rev, in.ds, first, count, st));
  if (in.rev16 && count) {
    UST_CUDA(h, cudaMemcpyAsync(h->s_rev16.p + first, in.rev16 + first, count * 2, cudaMemcpyHostToDevice, st));
    UST_CUDA(h, cudaMemcpyAsync(h->s_ds8.p + first, in.ds8 + first, count, cudaMemcpyHostToDevice, st));
  }
  return UST_OK;
}

static int widen_nodes(ust_handle* h, size_t first, size_t count, cudaStream_t st) {
  int we = ust_launch_widen((long long)count, h->s_rev16.p + first, h->s_ds8.p + first, h->staged.rev.p + first,
                            h->staged.ds.p + first, 4 * h->num_sms, st);
  if (we) return h->fail(UST_ERR_CUDA, "widen kernel launch failed: %s", cudaGetErrorString((cudaError_t)we));
  h->launches += 1;
  return UST_OK;
}

static void drop_resident(ust_handle* h) {
  h->resident_n = -1;
  h->outputs_resident = false;
  h->pods_n = -1;
}

// The snapshot in `staged` stays resident after a call that produced counters (a reference-level abort and
// UST_ERR_TRUNCATED included), with the call's outputs unless `outputs` is false. A call that failed keeps nothing.
// n_pods >= 0: the call evaluated pod lists of that many pods and their actuator outcomes; its snapshot is the pod-list
// snapshot, which only ust_apply_state_delta_pods and ust_fetch_outputs_pods use (`clocked`: with its start times, which
// only the clocked pod-list calls use).
static int adopt_resident(ust_handle* h, int rc, int64_t n, int32_t n_ds, bool outputs = true, int64_t n_pods = -1,
                          bool clocked = false) {
  if (rc != UST_ERR_CUDA && rc != UST_ERR_INVALID_ARGUMENT && rc != UST_ERR_COMM && rc != UST_ERR_NIL_STATE) {
    if (n_pods >= 0) {
      h->pods_n = n;
      h->pods_total = n_pods;
      h->pods_clocked = clocked;
      h->deadline_ready = clocked;
      return rc;
    }
    h->resident_n = n;
    h->resident_n_ds = n_ds;
    h->outputs_resident = outputs;
  }
  return rc;
}

// Pipelined host path: the snapshot is cut into segments of whole tiles; segment s+1 uploads while segment
// s streams through the kernel and segment s-1's results download (PCIe is full duplex). The streaming pass
// is speculative, so a segment's outputs are final unless the end-of-call verification had to redo tiles —
// then (rare) the outputs are downloaded again.
static int apply_pipelined(ust_handle* h, const ust_policy* policy, int64_t n, const HostNodes& in, int32_t n_ds,
                           uint8_t* next_state, uint16_t* actions, uint8_t* outcome, ust_counters* out) {
  cudaStream_t up = h->stream, down = h->stream_d2h, h2d = h->stream_h2d;  // up = compute stream of the call
  UstParams P;
  int grid = 0;
  int rc = begin_call(h, policy, n, h->staged.hot.p, h->staged.flags.p, h->staged.rev.p, h->staged.ds.p, n_ds, h->s_dsrev.p,
                      nullptr, nullptr, h->outs.next.p, h->outs.actions.p, outcome ? h->s_outcome.p : nullptr, nullptr, up,
                      &P, &grid);
  if (rc) return rc;
  const int tiles = P.n_tiles;
  // Segments: the uploads are the critical path (PCIe), every segment adds copy-engine turnarounds, and what follows
  // the last upload - its kernels and the download of its outputs - is exposed. So: few segments, and a last one of
  // 1/16 of the tiles.
  const int kSegments = h->segments;  // <= UST_MAX_SEGMENTS: one ticket counter and one event pair per streaming launch
  const int last_tiles = (kSegments > 1 && tiles >= 64) ? tiles / 16 : 0;
  const int per = last_tiles ? (tiles - last_tiles + kSegments - 2) / (kSegments - 1) : (tiles + kSegments - 1) / kSegments;
  // uploads start once the compute stream has reached this call (tables, DaemonSet table, previous call's reads)
  UST_CUDA(h, cudaEventRecord(h->d2h_done, up));
  UST_CUDA(h, cudaStreamWaitEvent(h2d, h->d2h_done, 0));
  int seg = 0;
  for (int c0 = 0, c1 = 0; c0 < tiles; c0 = c1, seg++) {
    c1 = c0 + per < tiles - last_tiles ? c0 + per : (c0 < tiles - last_tiles ? tiles - last_tiles : tiles);
    const int64_t n0 = (int64_t)c0 * P.tile_nodes, n1 = c1 == tiles ? n : (int64_t)c1 * P.tile_nodes;
    const size_t len = (size_t)(n1 - n0);
    rc = upload_nodes(h, in, (size_t)n0, len, h2d);
    if (rc) return rc;
    UST_CUDA(h, cudaEventRecord(h->seg_up[seg], h2d));
    UST_CUDA(h, cudaStreamWaitEvent(up, h->seg_up[seg], 0));
    if (in.rev16 && len) {
      rc = widen_nodes(h, (size_t)n0, len, up);
      if (rc) return rc;
    }
    UstParams Ps = P;
    Ps.tile_begin = c0;
    Ps.tile_end = c1;
    Ps.publish = c1 == tiles;
    Ps.seg = seg;
    const int g = pick_grid(h, c1 - c0);
    Ps.static_rounds = pick_static_rounds(h, c1 - c0, g);
    Ps.stamps = 0;
    int e = ust_launch_stream(Ps, g, up, 0);
    if (e) return h->fail(UST_ERR_CUDA, "streaming kernel launch failed: %s", cudaGetErrorString((cudaError_t)e));
    h->launches += 1;
    UST_CUDA(h, cudaEventRecord(h->seg_done[seg], up));
    UST_CUDA(h, cudaStreamWaitEvent(down, h->seg_done[seg], 0));
    if (len) {
      UST_CUDA(h, cudaMemcpyAsync(next_state + n0, h->outs.next.p + n0, len, cudaMemcpyDeviceToHost, down));
      UST_CUDA(h, cudaMemcpyAsync(actions + n0, h->outs.actions.p + n0, len * 2, cudaMemcpyDeviceToHost, down));
      if (outcome) UST_CUDA(h, cudaMemcpyAsync(outcome + n0, h->s_outcome.p + n0, len, cudaMemcpyDeviceToHost, down));
    }
  }
  rc = launch_verify(h, P, up, false);
  if (rc) return rc;
  h->ws_dirty = false;
  UST_CUDA(h, cudaMemcpyAsync(h->counters_host, h->counters_dev, sizeof(ust_counters), cudaMemcpyDeviceToHost, up));
  // the call ends when the segments' downloads have ended too
  UST_CUDA(h, cudaEventRecord(h->d2h_done, down));
  UST_CUDA(h, cudaStreamWaitEvent(up, h->d2h_done, 0));
  rc = finish_with_counters(h, up, out, true);
  if (rc != UST_ERR_CUDA && h->counters_host->reserved[0] != 0) {  // the verification redid tiles: fetch the final outputs
    UST_CUDA(h, cudaMemcpyAsync(next_state, h->outs.next.p, (size_t)n, cudaMemcpyDeviceToHost, up));
    UST_CUDA(h, cudaMemcpyAsync(actions, h->outs.actions.p, (size_t)n * 2, cudaMemcpyDeviceToHost, up));
    if (outcome) UST_CUDA(h, cudaMemcpyAsync(outcome, h->s_outcome.p, (size_t)n, cudaMemcpyDeviceToHost, up));
    UST_CUDA(h, cudaStreamSynchronize(up));
  }
  return rc;
}

// Clocked pod-list calls: the clock must come with the start times of the nodes the call carries, and agree with the policy
// about whether the wait has a timeout at all.
static int check_clock(ust_handle* h, const ust_policy* policy, const ust_clock* clock, bool carried) {
  if (!clock) return h->fail(UST_ERR_INVALID_ARGUMENT, "clock: required");
  if (carried && !clock->start) return h->fail(UST_ERR_INVALID_ARGUMENT, "clock: start is NULL while the call carries nodes");
  if (policy && (policy->wait_timeout_nonzero != 0) != (clock->wait_timeout_seconds != 0))
    return h->fail(UST_ERR_INVALID_ARGUMENT, "policy.wait_timeout_nonzero must say whether clock.wait_timeout_seconds != 0");
  return UST_OK;
}

// Clocked calls: bits 18 and 27 of the staged flags from the resident start column, just before the evaluation reads them,
// and the candidates of the call's next deadline (evaluated by launch_deadline behind the verification kernel)
static int launch_clock(ust_handle* h, const ust_clock* clock, int64_t n, cudaStream_t st) {
  const UstClockGrid g = ust_clock_grid((long long)n, 8 * h->num_sms);
  UST_CUDA(h, h->clk_cand.reserve((size_t)g.ctas * (size_t)g.region + 1));
  UST_CUDA(h, h->clk_count.reserve((size_t)g.ctas + 1));
  UST_CUDA(h, h->clk_deadline.reserve(1));
  h->clk_grid = g;
  int e = ust_launch_clock((long long)n, h->staged.hot.p, h->staged.flags.p, h->s_start.p, (long long)clock->now,
                           (long long)clock->wait_timeout_seconds, g, h->clk_cand.p, h->clk_count.p, h->clk_deadline.p, st);
  if (e) return h->fail(UST_ERR_CUDA, "clock kernel launch failed: %s", cudaGetErrorString((cudaError_t)e));
  h->launches += n > 0 ? 1 : 0;
  return UST_OK;
}

// The candidates of launch_clock evaluated a second time, behind the call's verification kernel (`P`: its parameters)
static int launch_deadline(ust_handle* h, const UstParams& P, const ust_clock* clock, int validation, int64_t n_pods, cudaStream_t st) {
  int e = ust_launch_deadline(P, h->clk_grid, h->clk_cand.p, h->clk_count.p, h->s_start.p, (long long)clock->wait_timeout_seconds,
                              validation, (long long)n_pods, h->clk_deadline.p, st);
  if (e) return h->fail(UST_ERR_CUDA, "deadline kernel launch failed: %s", cudaGetErrorString((cudaError_t)e));
  h->launches += h->clk_grid.ctas > 0 ? 1 : 0;
  return UST_OK;
}

// ust_apply_state, ust_apply_state_clocked and ust_apply_state_packed after their argument checks: upload, evaluate,
// download. Snapshots of 2^19 nodes or more take the pipelined path unless they come with pod lists. A call with pod lists
// and actuator_outcome leaves the pod-list snapshot (its list lengths are in h->pod_len_next, filled by the offset check);
// one with pod lists but no outcome leaves nothing resident. `clock` (nullable; pod lists and outcome given): the start
// times are uploaded beside the snapshot and the two timeouts derived from them.
static int apply_host(ust_handle* h, const ust_policy* policy, int64_t n, const HostNodes& in, int32_t n_ds,
                      const int32_t* ds_rev, const ust_pods* pods, uint8_t* next_state, uint16_t* actions,
                      uint8_t* outcome, ust_counters* out, const ust_clock* clock = nullptr) {
  drop_resident(h);  // the staging arrays are overwritten from here on
  UST_CUDA(h, cudaSetDevice(h->device));
  StreamDrain drain(h);
  cudaStream_t st = h->stream;
  const size_t N = (size_t)n;
  UST_CUDA(h, h->staged.reserve(N));
  if (in.rev16) {
    UST_CUDA(h, h->s_rev16.reserve(N + 8));
    UST_CUDA(h, h->s_ds8.reserve(N + 16));
  }
  UST_CUDA(h, h->outs.reserve(N));
  UST_CUDA(h, h->s_dsrev.reserve((size_t)n_ds + 1));
  if (outcome) UST_CUDA(h, h->s_outcome.reserve(N + 16));
  if (pods) {
    UST_CUDA(h, h->s_podoff.reserve(N + 1));
    UST_CUDA(h, h->s_podflags.reserve((size_t)pods->n_pods + 8));
  }
  if (n_ds) UST_CUDA(h, cudaMemcpyAsync(h->s_dsrev.p, ds_rev, (size_t)n_ds * 4, cudaMemcpyHostToDevice, st));
  if (!pods && n >= (1 << 19))
    return adopt_resident(h, apply_pipelined(h, policy, n, in, n_ds, next_state, actions, outcome, out), n, n_ds);
  int rc = upload_nodes(h, in, 0, N, st);
  if (rc) return rc;
  if (in.rev16 && N) {
    rc = widen_nodes(h, 0, N, st);
    if (rc) return rc;
  }
  if (pods) {
    UST_CUDA(h, cudaMemcpyAsync(h->s_podoff.p, pods->pod_off, (N + 1) * 4, cudaMemcpyHostToDevice, st));
    if (pods->n_pods) UST_CUDA(h, cudaMemcpyAsync(h->s_podflags.p, pods->pod_flags, (size_t)pods->n_pods * 2, cudaMemcpyHostToDevice, st));
  }
  if (clock) {
    UST_CUDA(h, h->s_start.reserve(N + 1));
    if (N) UST_CUDA(h, cudaMemcpyAsync(h->s_start.p, clock->start, N * 8, cudaMemcpyHostToDevice, st));
    rc = launch_clock(h, clock, n, st);
    if (rc) return rc;
  }
  rc = apply_device(h, policy, n, h->staged.hot.p, h->staged.flags.p, h->staged.rev.p, h->staged.ds.p, n_ds, h->s_dsrev.p,
                    pods ? h->s_podoff.p : nullptr, pods ? h->s_podflags.p : nullptr, pods ? pods->n_pods : 0, h->outs.next.p,
                    h->outs.actions.p, outcome ? h->s_outcome.p : nullptr, nullptr, st, clock);
  if (rc) return rc;
  if (N) {
    UST_CUDA(h, cudaMemcpyAsync(next_state, h->outs.next.p, N, cudaMemcpyDeviceToHost, st));
    UST_CUDA(h, cudaMemcpyAsync(actions, h->outs.actions.p, N * 2, cudaMemcpyDeviceToHost, st));
    if (outcome) UST_CUDA(h, cudaMemcpyAsync(outcome, h->s_outcome.p, N, cudaMemcpyDeviceToHost, st));
  }
  rc = finish_with_counters(h, st, out);
  if (!pods) return adopt_resident(h, rc, n, n_ds);
  if (!outcome) return rc;
  std::swap(h->pod_len, h->pod_len_next);
  return adopt_resident(h, rc, n, n_ds, true, pods->n_pods, clock != nullptr);
}

// The launch of ust_build_state / _uids once their inputs are enqueued: `launch(grid)` starts the counting kernel and
// the finish kernel behind it.
template <class Launch>
static int build_state_launch(ust_handle* h, int64_t n_pods, int32_t n_ds, cudaStream_t st, Launch launch) {
  if ((size_t)n_ds + 1 > h->ds_count.cap) {  // between calls only the finish kernel clears the counts
    UST_CUDA(h, h->ds_count.reserve((size_t)n_ds + 1));
    UST_CUDA(h, cudaMemsetAsync(h->ds_count.p, 0, h->ds_count.cap * sizeof(unsigned long long), st));
  }
  if (h->ws_dirty) { UST_CUDA(h, clear_workspace(h, st)); h->ws_dirty = false; }
  int64_t grid = (n_pods + 1023) / 1024;  // 256 threads x 4 pods per iteration
  if (grid < 1) grid = 1;
  if (grid > 8 * h->num_sms) grid = 8 * h->num_sms;
  h->ws_dirty = true;
  int e = launch((int)grid);
  if (e) return h->fail(UST_ERR_CUDA, "build-state kernel launch failed: %s", cudaGetErrorString((cudaError_t)e));
  h->ws_dirty = false;
  h->launches += 2;
  return UST_OK;
}

// The DaemonSet map of BuildState's owner join, keyed by UID (common_manager.go:181-185): an open-addressing table at load
// factor <= 1/4 (ust_uid_hash, linear probing, (0, 0) = empty slot) and the DaemonSet index of every slot. The UIDs must be
// non-empty and distinct.
struct DsTable {
  size_t slots = 8;
  std::vector<uint64_t> tab;
  std::vector<int32_t> idx;
};
static int ds_table(ust_handle* h, int32_t n_ds, const uint64_t* ds_uid, DsTable* t) {
  size_t& slots = t->slots;
  while (slots < 4 * (size_t)n_ds) slots <<= 1;
  t->tab.assign(2 * slots, 0);
  t->idx.assign(slots, -2);
  uint64_t* tab = t->tab.data();
  for (int32_t d = 0; d < n_ds; d++) {
    const uint64_t x = ds_uid[2 * (size_t)d], y = ds_uid[2 * (size_t)d + 1];
    if ((x | y) == 0) return h->fail(UST_ERR_INVALID_ARGUMENT, "DaemonSet %d has an empty UID", (int)d);
    size_t s = ust_uid_hash(x, y) & (slots - 1);
    while ((tab[2 * s] | tab[2 * s + 1]) != 0) {
      if (tab[2 * s] == x && tab[2 * s + 1] == y)
        return h->fail(UST_ERR_INVALID_ARGUMENT, "DaemonSets %d and %d share a UID", (int)t->idx[s], (int)d);
      s = (s + 1) & (slots - 1);
    }
    tab[2 * s] = x; tab[2 * s + 1] = y; t->idx[s] = d;
  }
  return UST_OK;
}
// the table and DesiredNumberScheduled per DaemonSet, enqueued on `st` (the caller synchronises before `t` goes)
static int upload_ds_table(ust_handle* h, const DsTable& t, int32_t n_ds, const int32_t* ds_desired, cudaStream_t st) {
  UST_CUDA(h, h->s_dsuid.reserve(2 * t.slots));
  UST_CUDA(h, h->s_dsorder.reserve(t.slots));
  UST_CUDA(h, h->s_dsdesired.reserve((size_t)n_ds + 1));
  UST_CUDA(h, cudaMemcpyAsync(h->s_dsuid.p, t.tab.data(), t.slots * 16, cudaMemcpyHostToDevice, st));
  UST_CUDA(h, cudaMemcpyAsync(h->s_dsorder.p, t.idx.data(), t.slots * 4, cudaMemcpyHostToDevice, st));
  if (n_ds) UST_CUDA(h, cudaMemcpyAsync(h->s_dsdesired.p, ds_desired, (size_t)n_ds * 4, cudaMemcpyHostToDevice, st));
  return UST_OK;
}

extern "C" {

int ust_abi_version(void) { return UST_ABI_VERSION; }
const char* ust_create_error(void) { return g_create_error.c_str(); }
const char* ust_last_error(const ust_handle* h) { return h ? h->err.c_str() : "null handle"; }
int64_t ust_launch_count(const ust_handle* h) { return h ? h->launches : 0; }

int ust_create(ust_handle** out, int device) {
  if (!out) return UST_ERR_INVALID_ARGUMENT;
  *out = nullptr;
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0) {
    g_create_error = std::string("no CUDA device: ") + cudaGetErrorString(e);
    return UST_ERR_CUDA;
  }
  if (device < 0 || device >= count) { g_create_error = "device index out of range"; return UST_ERR_INVALID_ARGUMENT; }
  cudaDeviceProp prop;
  if ((e = cudaGetDeviceProperties(&prop, device)) != cudaSuccess) { g_create_error = cudaGetErrorString(e); return UST_ERR_CUDA; }
  if (prop.major != 9 || prop.minor != 0) {  // sm_90a code runs on compute capability 9.0 only
    g_create_error = "libust.so carries sm_90a code only; device is sm_" + std::to_string(prop.major) + std::to_string(prop.minor);
    return UST_ERR_CUDA;
  }
  ust_handle* h = new ust_handle();
  h->device = device;
  h->no_hint = getenv("UST_NO_HINT") != nullptr;
  if (const char* sg = getenv("UST_SEGMENTS")) { int v = atoi(sg); if (v >= 1 && v <= UST_MAX_SEGMENTS) h->segments = v; }
  auto bail = [&](const char* what, cudaError_t err) {
    g_create_error = std::string(what) + ": " + cudaGetErrorString(err);
    ust_destroy(h);
    return UST_ERR_CUDA;
  };
  if ((e = cudaSetDevice(device)) != cudaSuccess) return bail("cudaSetDevice", e);
  if ((e = cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking)) != cudaSuccess) return bail("cudaStreamCreate", e);
  if ((e = cudaStreamCreateWithFlags(&h->stream_d2h, cudaStreamNonBlocking)) != cudaSuccess) return bail("cudaStreamCreate", e);
  if ((e = cudaStreamCreateWithFlags(&h->stream_h2d, cudaStreamNonBlocking)) != cudaSuccess) return bail("cudaStreamCreate", e);
  for (auto& ev : h->seg_up)
    if ((e = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming)) != cudaSuccess) return bail("cudaEventCreate", e);
  for (auto& ev : h->seg_done)
    if ((e = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming)) != cudaSuccess) return bail("cudaEventCreate", e);
  if ((e = cudaEventCreateWithFlags(&h->d2h_done, cudaEventDisableTiming)) != cudaSuccess) return bail("cudaEventCreate", e);
  if ((e = cudaMalloc(&h->ws, sizeof(UstWorkspace))) != cudaSuccess) return bail("cudaMalloc", e);
  if ((e = cudaMemset(h->ws, 0, sizeof(UstWorkspace))) != cudaSuccess) return bail("cudaMemset", e);
  if ((e = cudaMalloc(&h->lut_dev, UST_LUT_WORDS * sizeof(uint32_t))) != cudaSuccess) return bail("cudaMalloc", e);
  if ((e = cudaMalloc(&h->podlut_dev, UST_PODLUT_ENTRIES)) != cudaSuccess) return bail("cudaMalloc", e);
  if ((e = cudaMallocHost(&h->lut_host, UST_LUT_WORDS * sizeof(uint32_t))) != cudaSuccess) return bail("cudaMallocHost", e);
  if ((e = cudaMallocHost(&h->podlut_host, UST_PODLUT_ENTRIES)) != cudaSuccess) return bail("cudaMallocHost", e);
  if ((e = cudaMalloc(&h->counters_dev, sizeof(ust_counters))) != cudaSuccess) return bail("cudaMalloc", e);
  if ((e = cudaMallocHost(&h->counters_host, sizeof(ust_counters))) != cudaSuccess) return bail("cudaMallocHost", e);
  if ((e = cudaMalloc(&h->xchg_dev, UST_V_LEN * sizeof(long long))) != cudaSuccess) return bail("cudaMalloc", e);
  if ((e = cudaMalloc(&h->sp_count_dev, sizeof(long long))) != cudaSuccess) return bail("cudaMalloc", e);
  if ((e = cudaMallocHost(&h->sp_count_host, sizeof(long long))) != cudaSuccess) return bail("cudaMallocHost", e);
  if ((e = cudaMemset(h->xchg_dev, 0, UST_V_LEN * sizeof(long long))) != cudaSuccess) return bail("cudaMemset", e);
  if (const char* v = getenv("UST_PDL")) h->pdl = atoi(v) != 0;
  if (const char* v = getenv("UST_STATIC_PCT")) { h->static_pct = atoi(v); if (h->static_pct < 0) h->static_pct = 0; if (h->static_pct > 100) h->static_pct = 100; }
  h->stamps = getenv("UST_STAMPS") != nullptr;
  if (const char* v = getenv("UST_OVERLAP")) h->overlap_calls = atoi(v) != 0;
  {
    int l2 = 0;
    if ((e = cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, device)) != cudaSuccess) return bail("cudaDeviceGetAttribute", e);
    h->l2_bytes = (size_t)l2;
  }
  int rc = ust_stream_config(device, &h->num_sms, &h->stream_smem, &h->stream_ctas_per_sm);
  if (rc != 0 || h->num_sms < 1) {
    g_create_error = std::string("no sm_90a kernel image usable on this device: ") + cudaGetErrorString((cudaError_t)rc);
    ust_destroy(h);
    return UST_ERR_CUDA;
  }
  *out = h;
  return UST_OK;
}

void ust_destroy(ust_handle* h) {
  if (!h) return;
  if (h->device >= 0) cudaSetDevice(h->device);
  if (h->stream_h2d) cudaStreamSynchronize(h->stream_h2d);
  if (h->stream) cudaStreamSynchronize(h->stream);
  if (h->stream_d2h) cudaStreamSynchronize(h->stream_d2h);
  if (h->last_stream) cudaStreamSynchronize(h->last_stream);
  for (int r = 0; r < UST_MAX_WORLD; r++)
    if (h->mbox[r] && h->mbox[r] != h->mbox_own) cudaIpcCloseMemHandle(h->mbox[r]);
  if (h->mbox_own) cudaFree(h->mbox_own);
  if (h->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(h->comm);
  if (h->ws) cudaFree(h->ws);
  if (h->lut_dev) cudaFree(h->lut_dev);
  if (h->podlut_dev) cudaFree(h->podlut_dev);
  if (h->lut_host) cudaFreeHost(h->lut_host);
  if (h->podlut_host) cudaFreeHost(h->podlut_host);
  if (h->counters_dev) cudaFree(h->counters_dev);
  if (h->counters_host) cudaFreeHost(h->counters_host);
  if (h->xchg_dev) cudaFree(h->xchg_dev);
  if (h->sp_count_dev) cudaFree(h->sp_count_dev);
  if (h->sp_count_host) cudaFreeHost(h->sp_count_host);
  for (auto& ev : h->seg_done) if (ev) cudaEventDestroy(ev);
  for (auto& ev : h->seg_up) if (ev) cudaEventDestroy(ev);
  if (h->stream_h2d) cudaStreamDestroy(h->stream_h2d);
  if (h->d2h_done) cudaEventDestroy(h->d2h_done);
  if (h->stream_d2h) cudaStreamDestroy(h->stream_d2h);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;  // frees the DevBufs, on the device set above
}

void* ust_host_alloc(size_t bytes) {
  void* p = nullptr;
  if (cudaMallocHost(&p, bytes ? bytes : 1) != cudaSuccess) return nullptr;
  return p;
}
void ust_host_free(void* p) { if (p) cudaFreeHost(p); }

void* ust_stream(ust_handle* h) { return h ? (void*)h->stream : nullptr; }

int ust_sync(ust_handle* h) {
  if (!h) return UST_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> g(h->mu);
  h->prev_n = -1;  // whatever this entry point enqueues sits between two device calls: they keep the strict order
  UST_CUDA(h, cudaSetDevice(h->device));
  cudaError_t e = cudaStreamSynchronize(h->stream);
  if (e == cudaSuccess && h->last_stream && h->last_stream != h->stream) e = cudaStreamSynchronize(h->last_stream);
  if (e != cudaSuccess) { h->ws_dirty = true; return h->fail(UST_ERR_CUDA, "stream sync failed: %s", cudaGetErrorString(e)); }
  return UST_OK;
}

int ust_apply_state_device(ust_handle* h, const ust_policy* policy, int64_t n_nodes, const uint8_t* state,
                           const uint32_t* flags, const int32_t* pod_rev, const int32_t* ds_idx, int32_t n_ds,
                           const int32_t* ds_rev, const ust_pods* pods, uint8_t* next_state, uint16_t* actions,
                           uint8_t* actuator_outcome, ust_counters* out_device, void* stream) {
  if (!h) return UST_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> g(h->mu);
  h->deadline_ready = false;
  h->chain_entry = true;  // the one entry point whose calls may overlap the previous call's tail (apply_device)
  cudaStream_t st = stream ? (cudaStream_t)stream : h->stream;
  if (pods && (!pods->pod_off || pods->n_pods < 0 || (pods->n_pods > 0 && !pods->pod_flags)))
    return h->fail(UST_ERR_INVALID_ARGUMENT, "bad pod lists");
  if (int rc = check_eval_mode(h, policy, pods != nullptr)) return rc;
  return apply_device(h, policy, n_nodes, state, flags, pod_rev, ds_idx, n_ds, ds_rev, pods ? pods->pod_off : nullptr,
                      pods ? pods->pod_flags : nullptr, pods ? pods->n_pods : 0, next_state, actions, actuator_outcome,
                      out_device, st);
}

// ust_apply_state and ust_apply_state_clocked (`clock` non-null: pod lists and actuator_outcome required)
static int apply_state_common(ust_handle* h, const ust_policy* policy, const ust_clock* clock, int64_t n, const uint8_t* state,
                              const uint32_t* flags, const int32_t* pod_rev, const int32_t* ds_idx, int32_t n_ds,
                              const int32_t* ds_rev, const ust_pods* pods, uint8_t* next_state, uint16_t* actions,
                              uint8_t* actuator_outcome, ust_counters* out) {
  h->prev_n = -1;  // whatever this entry point enqueues sits between two device calls: they keep the strict order
  h->deadline_ready = false;
  if (n < 0 || (n > 0 && (!state || !flags || !pod_rev || !ds_idx || !next_state || !actions)))
    return h->fail(UST_ERR_NIL_STATE, "currentState should not be empty");
  if (n_ds < 0 || (n_ds > 0 && !ds_rev)) return h->fail(UST_ERR_INVALID_ARGUMENT, "bad DaemonSet table");
  if (pods && (!pods->pod_off || pods->n_pods < 0 || (pods->n_pods > 0 && !pods->pod_flags)))
    return h->fail(UST_ERR_INVALID_ARGUMENT, "bad pod lists");
  if (int rc = check_eval_mode(h, policy, pods != nullptr)) return rc;
  if (clock) {  // (ust_apply_state_clocked has checked that it was given one)
    if (!pods || !actuator_outcome)
      return h->fail(UST_ERR_INVALID_ARGUMENT, "ust_apply_state_clocked: pod lists and actuator_outcome are required");
    if (int rc = check_clock(h, policy, clock, n > 0)) return rc;
  }
  if (pods) {
    // a call that may leave the pod-list snapshot notes its list lengths for the checks of ust_apply_state_delta_pods
    int32_t* lens = nullptr;
    if (actuator_outcome) {
      h->pod_len_next.resize((size_t)n);
      lens = h->pod_len_next.data();
    }
    int prc = check_pod_offsets_host(h, n, pods->pod_off, pods->n_pods, lens);
    if (prc) return prc;
  }
  return apply_host(h, policy, n, HostNodes{state, flags, pod_rev, ds_idx, nullptr, nullptr}, n_ds, ds_rev, pods, next_state,
                    actions, actuator_outcome, out, clock);
}

int ust_apply_state(ust_handle* h, const ust_policy* policy, int64_t n, const uint8_t* state, const uint32_t* flags,
                    const int32_t* pod_rev, const int32_t* ds_idx, int32_t n_ds, const int32_t* ds_rev,
                    const ust_pods* pods, uint8_t* next_state, uint16_t* actions, uint8_t* actuator_outcome,
                    ust_counters* out) {
  if (!h) return UST_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> g(h->mu);
  return apply_state_common(h, policy, nullptr, n, state, flags, pod_rev, ds_idx, n_ds, ds_rev, pods, next_state, actions,
                            actuator_outcome, out);
}

int ust_apply_state_clocked(ust_handle* h, const ust_policy* policy, const ust_clock* clock, int64_t n, const uint8_t* state,
                            const uint32_t* flags, const int32_t* pod_rev, const int32_t* ds_idx, int32_t n_ds,
                            const int32_t* ds_rev, const ust_pods* pods, uint8_t* next_state, uint16_t* actions,
                            uint8_t* actuator_outcome, ust_counters* out) {
  if (!h) return UST_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> g(h->mu);
  h->prev_n = -1;
  h->deadline_ready = false;  // (also cleared by apply_state_common: a call refused here counts as well)
  if (!clock) return h->fail(UST_ERR_INVALID_ARGUMENT, "clock: required");
  return apply_state_common(h, policy, clock, n, state, flags, pod_rev, ds_idx, n_ds, ds_rev, pods, next_state, actions,
                            actuator_outcome, out);
}

// The runs of a reorder as the gather kernel reads them (ust_launch_reorder): h->run_off holds the exclusive prefix of
// the run lengths (one entry more than there are runs), h->run_src per run the old start, or -1 - offset into the
// inserted nodes. Adjacent runs that continue each other are merged.
static void clear_runs(ust_handle* h) {
  h->run_off.assign(1, 0);
  h->run_src.clear();
}
static void add_run(ust_handle* h, long long src, long long len) {
  if (!h->run_src.empty()) {
    const long long last = h->run_src.back(), last_len = h->run_off.back() - h->run_off[h->run_off.size() - 2];
    if ((last >= 0) == (src >= 0) && (src >= 0 ? last + last_len == src : last - last_len == src)) {
      h->run_off.back() += len;
      return;
    }
  }
  h->run_src.push_back(src);
  h->run_off.push_back(h->run_off.back() + len);
}

// Bits [a, a + len) of the bitmap: set (false when one of them was set already) or cleared.
static bool mark_bits(uint64_t* w, long long a, long long len, bool set) {
  const long long e = a + len;
  for (long long i = a >> 6; i <= (e - 1) >> 6; i++) {
    const long long lo = std::max(a, i << 6), hi = std::min(e, (i + 1) << 6);
    const uint64_t m = hi - lo == 64 ? ~0ull : ((1ull << (hi - lo)) - 1) << (lo & 63);
    if (!set) { w[i] &= ~m; continue; }
    if (w[i] & m) return false;
    w[i] |= m;
  }
  return true;
}

// A reorder (n_runs runs run_src / run_len over n_old old entries, n_insert inserted ones) checked in full and turned into
// runs, O(n + n_runs): a bitmap over the old snapshot finds old nodes that two runs name. Sets *n_new to the new size.
static int reorder_runs(ust_handle* h, int64_t n_runs, const int64_t* run_src, const int64_t* run_len, int64_t n_insert, int64_t n_old,
                        int64_t* n_new) {
  if (n_runs < 0 || n_insert < 0 || (n_runs > 0 && (!run_src || !run_len))) return h->fail(UST_ERR_INVALID_ARGUMENT, "bad reorder");
  const size_t words = ((size_t)n_old + 63) / 64;
  if (h->run_seen.size() < words) h->run_seen.resize(words, 0);
  clear_runs(h);
  int rc = UST_OK;
  int64_t marked = 0, ins = 0;  // runs whose old nodes are marked; inserted nodes taken
  for (int64_t r = 0; r < n_runs && rc == UST_OK; r++) {
    const long long src = run_src[r], len = run_len[r];
    if (len < 1 || src < -1)
      rc = h->fail(UST_ERR_INVALID_ARGUMENT, "reorder: run %lld has source %lld and length %lld", (long long)r, src, len);
    else if (len >= (1LL << 40) - h->run_off.back())
      rc = h->fail(UST_ERR_INVALID_ARGUMENT, "too many nodes");
    else if (src < 0 && len > n_insert - ins)
      rc = h->fail(UST_ERR_INVALID_ARGUMENT, "reorder: the inserted runs take more than the %lld inserted nodes", (long long)n_insert);
    else if (src >= 0 && (src >= n_old || len > n_old - src))
      rc = h->fail(UST_ERR_INVALID_ARGUMENT, "reorder: run %lld (old nodes %lld + %lld) leaves the snapshot of %lld nodes", (long long)r, src,
                   len, (long long)n_old);
    else if (src >= 0 && (marked = r + 1, !mark_bits(h->run_seen.data(), src, len, true)))
      rc = h->fail(UST_ERR_INVALID_ARGUMENT, "reorder: run %lld names an old node that an earlier run names", (long long)r);
    else if (src < 0) {
      add_run(h, -1 - ins, len);
      ins += len;
    } else {
      add_run(h, src, len);
    }
  }
  for (int64_t r = 0; r < marked; r++)  // the bitmap is all zero again
    if (run_src[r] >= 0) mark_bits(h->run_seen.data(), run_src[r], run_len[r], false);
  if (rc == UST_OK && ins != n_insert)
    rc = h->fail(UST_ERR_INVALID_ARGUMENT, "reorder: the inserted runs take %lld of the %lld inserted nodes", (long long)ins, (long long)n_insert);
  *n_new = h->run_off.back();
  return rc;
}

// The pod lists of a reorder of the pod-list snapshot of n_new nodes, after reorder_runs: the runs and the replaced lists
// (node_idx: new indices, checked) walked together. Fills h->pod_len_next with every new node's list length (moved run by
// run from h->pod_len, the lengths of replaced and inserted lists written over it) and cuts the new snapshot into the
// segments of ust_launch_pods_reorder, with their pod starts. Fails when an inserted node has no list or the new pod total
// reaches 2^31. Linear in n_new (4 B read and written per node), otherwise O(n_runs + n_lists); h->pod_len is untouched.
static int pods_reorder_segments(ust_handle* h, const ust_pod_lists* pl, int64_t L, int64_t n_new, int64_t* new_total) {
  h->pod_len_next.resize((size_t)n_new);
  int32_t* len = h->pod_len_next.data();
  const int32_t* old = h->pod_len.data();
  const size_t NR = h->run_src.size();
  h->seg_node.clear();
  h->seg_src.clear();
  h->seg_pod.clear();
  h->seg_node.reserve(NR + 2 * (size_t)L + 1);
  h->seg_src.reserve(NR + 2 * (size_t)L);
  h->seg_pod.reserve(NR + 2 * (size_t)L + 1);
  int64_t k = 0, total = 0;  // next list; pods ahead of the segment being cut (int32 once the total is checked)
  for (size_t r = 0; r < NR; r++) {
    const long long o = h->run_off[r], e = h->run_off[r + 1], src = h->run_src[r];
    for (long long p = o; p < e;) {
      h->seg_node.push_back(p);
      h->seg_pod.push_back((int32_t)total);
      if (k < L && pl->node_idx[k] == p) {  // a replaced or inserted list: a segment of its own
        len[p] = pl->pod_off[k + 1] - pl->pod_off[k];
        h->seg_src.push_back(-1 - k);
        total += len[p];
        k++;
        p++;
      } else if (src < 0) {
        return h->fail(UST_ERR_INVALID_ARGUMENT, "pod lists: inserted node %lld has no list: every inserted node needs one", p);
      } else {  // old nodes up to the next replaced list
        const long long q = k < L && pl->node_idx[k] < e ? pl->node_idx[k] : e;
        const int32_t* from = old + src + (p - o);
        int64_t pods = 0;
        for (long long j = 0; j < q - p; j++) {
          len[p + j] = from[j];
          pods += from[j];
        }
        h->seg_src.push_back(src + (p - o));
        total += pods;
        p = q;
      }
    }
  }
  if (total >= (1LL << 31)) return h->fail(UST_ERR_INVALID_ARGUMENT, "pod lists: %lld pods in all, pod_off is int32", (long long)total);
  h->seg_node.push_back(n_new);
  h->seg_pod.push_back((int32_t)total);
  *new_total = total;
  return UST_OK;
}

// One call of ust_apply_state_delta, _delta_sparse, _delta_splice, _delta_reorder, _delta_pods, _delta_pods_reorder or
// _delta_pods_clocked. The constructors take the arguments every dense or sparse entry point has, in ABI order
// (actuator_outcome: pod-list calls only among the sparse ones); an entry point then sets the fields of its own structs.
struct DeltaCall {
  const ust_policy* policy;
  int64_t n_changed;                     // the re-encoded nodes: their indices and (wide) columns
  const int64_t* idx;
  HostNodes changed;
  int32_t n_ds;
  const int32_t* ds_rev;
  uint8_t* next_state;                   // outputs: n entries each (dense) or max_out entries each and their count (sparse)
  uint16_t* actions;
  uint8_t* actuator_outcome;
  ust_counters* out;
  bool sparse = false;
  int64_t max_out = 0;
  int64_t* out_idx = nullptr;
  int64_t* n_out = nullptr;
  const ust_splice* splice = nullptr;    // the new node order: at most one of the two
  const ust_reorder* reorder = nullptr;
  bool pods = false;                     // the call is on the pod-list snapshot, `lists` (nullable) replaces some of its lists
  const ust_pod_lists* lists = nullptr;
  bool clocked = false;                  // the entry point takes a clock, which must be given
  const ust_clock* clock = nullptr;
  DeltaCall(const ust_policy* policy_, int64_t n_changed_, const int64_t* idx_, const uint8_t* state, const uint32_t* flags,
            const int32_t* pod_rev, const int32_t* ds_idx, int32_t n_ds_, const int32_t* ds_rev_, uint8_t* next_state_,
            uint16_t* actions_, uint8_t* actuator_outcome_, ust_counters* out_)
      : policy(policy_), n_changed(n_changed_), idx(idx_), changed{state, flags, pod_rev, ds_idx, nullptr, nullptr}, n_ds(n_ds_),
        ds_rev(ds_rev_), next_state(next_state_), actions(actions_), actuator_outcome(actuator_outcome_), out(out_) {}
  DeltaCall(const ust_policy* policy_, int64_t n_changed_, const int64_t* idx_, const uint8_t* state, const uint32_t* flags,
            const int32_t* pod_rev, const int32_t* ds_idx, int32_t n_ds_, const int32_t* ds_rev_, int64_t max_out_, int64_t* out_idx_,
            uint8_t* next_state_, uint16_t* actions_, uint8_t* actuator_outcome_, int64_t* n_out_, ust_counters* out_)
      : DeltaCall(policy_, n_changed_, idx_, state, flags, pod_rev, ds_idx, n_ds_, ds_rev_, next_state_, actions_, actuator_outcome_, out_) {
    sparse = true; max_out = max_out_; out_idx = out_idx_; n_out = n_out_;
  }
};

// What the checks of a delta call derive from it. The host scratch they fill besides (the reorder's runs, the pod-list
// segments, h->pod_len_next, h->pl_shift_host) is overwritten by the next call's checks; nothing resident changes.
struct DeltaPlan {
  int64_t n_old = 0, n = 0;            // snapshot size before and after the new node order
  int64_t n_remove = 0, n_insert = 0;  // nodes removed (splice) and inserted (splice or reorder) ...
  HostNodes ins = {};                  // ... and the inserted nodes' columns
  bool gather = false;                 // the node order changes: columns and previous outputs move into the second set
  int64_t new_total = 0;               // pods of the new pod-list snapshot
  bool same_len = true;                // every replaced list keeps its length: copied in place
  bool pods_gather = false;            // a reorder of the pod-list snapshot: its CSR is gathered anew
};

// Every check of a delta call, before any device work: a call that fails here leaves the resident snapshot as it was.
static int plan_delta(ust_handle* h, const DeltaCall& c, DeltaPlan* p) {
  if (c.clocked && !c.clock) return h->fail(UST_ERR_INVALID_ARGUMENT, "clock: required");
  if (int rc = check_eval_mode(h, c.policy, c.pods)) return rc;
  const int64_t n_old = c.pods ? h->pods_n : h->resident_n;
  if (n_old < 0 && c.pods)
    return h->fail(UST_ERR_INVALID_ARGUMENT, "no resident pod-list snapshot: call ust_apply_state with pod lists and actuator_outcome first");
  if (n_old < 0) return h->fail(UST_ERR_INVALID_ARGUMENT, "no resident snapshot: call ust_apply_state (without pod lists) first");
  if (c.pods && h->pods_clocked != (c.clock != nullptr))
    return h->fail(UST_ERR_INVALID_ARGUMENT, c.clock ? "the resident pod-list snapshot has no start times: it was left by an unclocked call"
                                                     : "the resident pod-list snapshot was left by a clocked call: use ust_apply_state_delta_pods_clocked");
  if (c.clock) {
    if (int rc = check_clock(h, c.policy, c.clock, c.n_changed > 0)) return rc;
    if (c.reorder && c.reorder->n_insert > 0 && !c.clock->insert_start)
      return h->fail(UST_ERR_INVALID_ARGUMENT, "clock: insert_start is NULL while the reorder inserts nodes");
  }
  if (c.sparse && !c.pods && !h->outputs_resident)
    return h->fail(UST_ERR_INVALID_ARGUMENT, "no resident outputs to compare with: the previous call must be an ApplyState on this snapshot");
  // the new node order, checked in full before anything is touched
  p->n_old = p->n = n_old;
  if (const ust_reorder* ro = c.reorder) {
    if (ro->n_insert > 0 && (!ro->state || !ro->flags || !ro->pod_rev || !ro->ds_idx)) return h->fail(UST_ERR_INVALID_ARGUMENT, "bad reorder");
    if (int rc = reorder_runs(h, ro->n_runs, ro->run_src, ro->run_len, ro->n_insert, n_old, &p->n)) return rc;
    p->gather = true;
    p->n_insert = ro->n_insert;
    p->ins = HostNodes{ro->state, ro->flags, ro->pod_rev, ro->ds_idx, nullptr, nullptr};
  } else if (const ust_splice* sp = c.splice) {
    const int64_t n_rm = sp->n_remove, n_ins = sp->n_insert;
    if (n_rm < 0 || n_ins < 0 || n_rm > n_old || (n_rm > 0 && !sp->remove_idx) ||
        (n_ins > 0 && (!sp->insert_before || !sp->state || !sp->flags || !sp->pod_rev || !sp->ds_idx)))
      return h->fail(UST_ERR_INVALID_ARGUMENT, "bad splice");
    for (int64_t k = 0; k < n_rm; k++)
      if (sp->remove_idx[k] < (k ? sp->remove_idx[k - 1] + 1 : 0) || sp->remove_idx[k] >= n_old)
        return h->fail(UST_ERR_INVALID_ARGUMENT, "splice: remove_idx[%lld] = %lld is not strictly increasing in [0, %lld)", (long long)k,
                       (long long)sp->remove_idx[k], (long long)n_old);
    for (int64_t k = 0; k < n_ins; k++)
      if (sp->insert_before[k] < (k ? sp->insert_before[k - 1] : 0) || sp->insert_before[k] > n_old)
        return h->fail(UST_ERR_INVALID_ARGUMENT, "splice: insert_before[%lld] = %lld is not non-decreasing in [0, %lld]", (long long)k,
                       (long long)sp->insert_before[k], (long long)n_old);
    p->n = n_old - n_rm + n_ins;
    p->gather = n_rm || n_ins;
    p->n_remove = n_rm; p->n_insert = n_ins;
    p->ins = HostNodes{sp->state, sp->flags, sp->pod_rev, sp->ds_idx, nullptr, nullptr};
  }
  const int64_t n = p->n;
  if (n >= (1LL << 40)) return h->fail(UST_ERR_INVALID_ARGUMENT, "too many nodes");
  if (c.n_changed < 0 || (c.n_changed > 0 && (!c.idx || !c.changed.state || !c.changed.flags || !c.changed.rev || !c.changed.ds)))
    return h->fail(UST_ERR_INVALID_ARGUMENT, "bad arguments");
  if (!c.sparse && n > 0 && (!c.next_state || !c.actions)) return h->fail(UST_ERR_INVALID_ARGUMENT, "bad arguments");
  if (c.sparse && (c.max_out < 0 || !c.n_out || (c.max_out > 0 && (!c.out_idx || !c.next_state || !c.actions || (c.pods && !c.actuator_outcome)))))
    return h->fail(UST_ERR_INVALID_ARGUMENT, "bad arguments");
  if (c.n_ds < 0 || (c.n_ds > 0 && !c.ds_rev)) return h->fail(UST_ERR_INVALID_ARGUMENT, "bad DaemonSet table");
  for (int64_t k = 0; k < c.n_changed; k++)
    if (c.idx[k] < 0 || c.idx[k] >= n) return h->fail(UST_ERR_INVALID_ARGUMENT, "changed node %lld has index %lld outside the snapshot of %lld nodes", (long long)k, (long long)c.idx[k], (long long)n);
  // replacement pod lists, checked in O(n_lists + n_pods) against the host copy of the resident list lengths; with every
  // length kept they are copied in place, otherwise the CSR is laid out anew (pl_shift_host: prefix of the length changes).
  // Under a reorder the CSR is always gathered anew, from the segments that pods_reorder_segments cuts.
  const ust_pod_lists* pl = c.lists;
  const int64_t L = c.pods && pl ? pl->n_lists : 0;
  p->new_total = c.pods ? h->pods_total : 0;
  if (L != 0) {
    if (L < 0 || !pl->node_idx || !pl->pod_off || pl->n_pods < 0 || (pl->n_pods > 0 && !pl->pod_flags))
      return h->fail(UST_ERR_INVALID_ARGUMENT, "bad pod lists");
    for (int64_t k = 0; k < L; k++)
      if (pl->node_idx[k] < (k ? pl->node_idx[k - 1] + 1 : 0) || pl->node_idx[k] >= n)
        return h->fail(UST_ERR_INVALID_ARGUMENT, "pod lists: node_idx[%lld] = %lld is not strictly increasing in [0, %lld)", (long long)k,
                       (long long)pl->node_idx[k], (long long)n);
    if (int rc = check_pod_offsets_host(h, L, pl->pod_off, pl->n_pods)) return rc;
  }
  p->pods_gather = c.pods && c.reorder;
  if (p->pods_gather) {
    const auto t0 = std::chrono::steady_clock::now();
    if (int rc = pods_reorder_segments(h, pl, L, n, &p->new_total)) return rc;
    h->pod_pass_ns = std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count();
  } else if (L != 0) {
    h->pl_shift_host.resize((size_t)L + 1);
    int64_t d = 0;
    for (int64_t k = 0; k < L; k++) {
      h->pl_shift_host[(size_t)k] = (int32_t)d;  // |d| stays below 2^31 when the new total does (checked below)
      const int32_t len = pl->pod_off[k + 1] - pl->pod_off[k];
      p->same_len = p->same_len && len == h->pod_len[(size_t)pl->node_idx[k]];
      d += (int64_t)len - h->pod_len[(size_t)pl->node_idx[k]];
    }
    h->pl_shift_host[(size_t)L] = (int32_t)d;
    p->new_total += d;
    if (p->new_total >= (1LL << 31)) return h->fail(UST_ERR_INVALID_ARGUMENT, "pod lists: %lld pods in all, pod_off is int32", (long long)p->new_total);
  }
  return UST_OK;
}

// The device work of a delta call once plan_delta has passed: the new node order (the previous outputs move with the nodes;
// on the pod-list snapshot their lists, previous outcome and start times too), the replaced lists, the re-encoded nodes,
// the two timeouts (clocked), the evaluation, then all outputs (dense) or those that differ from the previous call's
// (sparse), and the new snapshot becomes the resident one.
static int run_delta(ust_handle* h, const DeltaCall& c, const DeltaPlan& p) {
  UST_CUDA(h, cudaSetDevice(h->device));
  StreamDrain drain(h);
  cudaStream_t st = h->stream;
  const int64_t L = c.pods && c.lists ? c.lists->n_lists : 0;
  const size_t N = (size_t)p.n, M = (size_t)c.n_changed, I = (size_t)p.n_insert, NR = h->run_src.size(), R = (size_t)p.n_remove;
  if (p.gather) {  // the previous outputs travel with the snapshot
    UST_CUDA(h, h->splice_cols.reserve(N));
    UST_CUDA(h, h->splice_outs.reserve(N));
    if (c.reorder) UST_CUDA(h, h->runs.reserve(2 * NR + 2));
    else UST_CUDA(h, h->removed.reserve(R + 1));
    if (!c.reorder) UST_CUDA(h, h->inserted.idx.reserve(I + 1));
    UST_CUDA(h, h->inserted.cols.reserve(I));
  }
  UST_CUDA(h, h->s_dsrev.reserve((size_t)c.n_ds + 1));
  // (under a reorder s_outcome holds the previous outcome at the old size, which the gather reads: it is not resized)
  if (c.pods ? !c.reorder : c.actuator_outcome != nullptr) UST_CUDA(h, h->s_outcome.reserve(N + 16));
  if (c.pods && c.sparse) {
    UST_CUDA(h, h->s_outcome_prev.reserve(N + 16));
    UST_CUDA(h, h->sp_outcome.reserve((size_t)c.max_out + 1));
  }
  const size_t S = p.pods_gather ? h->seg_src.size() : 0;
  if (p.pods_gather) {
    UST_CUDA(h, h->splice_outcome.reserve(N + 16));
    UST_CUDA(h, h->pr_segs.reserve(2 * S + 1));
    UST_CUDA(h, h->pr_pods.reserve(2 * S + 1));
    UST_CUDA(h, h->s_podoff2.reserve(N + 1));
    UST_CUDA(h, h->s_podflags2.reserve((size_t)p.new_total + 16));
  }
  if (L) {  // the new lists carry 8 pods of padding for the relayout's 16-byte loads, the new CSR too
    UST_CUDA(h, h->pl_idx.reserve((size_t)L));
    UST_CUDA(h, h->pl_off.reserve((size_t)L + 1));
    UST_CUDA(h, h->pl_flags.reserve((size_t)c.lists->n_pods + 16));
    if (!p.same_len) {
      UST_CUDA(h, h->pl_shift.reserve((size_t)L + 1));
      UST_CUDA(h, h->pl_runs.reserve(4 * (size_t)L + 3));
      UST_CUDA(h, h->s_podoff2.reserve(N + 1));
      UST_CUDA(h, h->s_podflags2.reserve((size_t)p.new_total + 16));
    }
  }
  UST_CUDA(h, h->changed.idx.reserve(M + 1));
  UST_CUDA(h, h->changed.cols.reserve(M));
  if (c.clock) {
    UST_CUDA(h, h->chg_start.reserve(M + 1));
    if (c.reorder) {
      UST_CUDA(h, h->s_start2.reserve(N + 1));
      UST_CUDA(h, h->ins_start.reserve(I + 1));
    }
  }
  if (c.sparse) {  // the pair this call writes holds the new size as well
    UST_CUDA(h, h->outs_prev.reserve(N));
    UST_CUDA(h, h->sp_blocks.reserve((size_t)ust_diff_blocks(p.n) + 1));
    UST_CUDA(h, h->sp_idx.reserve((size_t)c.max_out + 1));
    UST_CUDA(h, h->outs_sparse.reserve((size_t)c.max_out));
  }
  drop_resident(h);  // until the patched snapshot has been evaluated
  if (p.pods_gather) std::swap(h->pod_len, h->pod_len_next);
  else for (int64_t k = 0; k < L; k++) h->pod_len[(size_t)c.lists->node_idx[k]] = c.lists->pod_off[k + 1] - c.lists->pod_off[k];
  if (c.n_ds) UST_CUDA(h, cudaMemcpyAsync(h->s_dsrev.p, c.ds_rev, (size_t)c.n_ds * 4, cudaMemcpyHostToDevice, st));
  if (L) {
    if (!p.pods_gather) UST_CUDA(h, cudaMemcpyAsync(h->pl_idx.p, c.lists->node_idx, (size_t)L * 8, cudaMemcpyHostToDevice, st));
    UST_CUDA(h, cudaMemcpyAsync(h->pl_off.p, c.lists->pod_off, ((size_t)L + 1) * 4, cudaMemcpyHostToDevice, st));
    if (c.lists->n_pods) UST_CUDA(h, cudaMemcpyAsync(h->pl_flags.p, c.lists->pod_flags, (size_t)c.lists->n_pods * 2, cudaMemcpyHostToDevice, st));
  }
  if (p.pods_gather) {  // the run table and the gather of the new CSR, into the second pair
    long long* segs = h->pr_segs.p;
    UST_CUDA(h, cudaMemcpyAsync(segs, h->seg_node.data(), (S + 1) * 8, cudaMemcpyHostToDevice, st));
    if (S) UST_CUDA(h, cudaMemcpyAsync(segs + S + 1, h->seg_src.data(), S * 8, cudaMemcpyHostToDevice, st));
    UST_CUDA(h, cudaMemcpyAsync(h->pr_pods.p, h->seg_pod.data(), (S + 1) * 4, cudaMemcpyHostToDevice, st));
    int e = ust_launch_pods_reorder((long long)p.n, (long long)S, segs, h->pr_pods.p, h->s_podoff.p, h->s_podflags.p, h->pl_off.p,
                                    h->pl_flags.p, (int)p.new_total, h->s_podoff2.p, h->s_podflags2.p, 8 * h->num_sms, st);
    if (e) return h->fail(UST_ERR_CUDA, "pod-list reorder kernel launch failed: %s", cudaGetErrorString((cudaError_t)e));
    h->launches += 2;
    std::swap(h->s_podoff, h->s_podoff2);
    std::swap(h->s_podflags, h->s_podflags2);
  } else if (L) {
    int e;
    if (p.same_len) {
      e = ust_launch_pods_scatter((long long)L, h->pl_idx.p, h->pl_off.p, h->pl_flags.p, h->s_podoff.p, h->s_podflags.p, 8 * h->num_sms, st);
      h->launches += 1;
    } else {
      UST_CUDA(h, cudaMemcpyAsync(h->pl_shift.p, h->pl_shift_host.data(), ((size_t)L + 1) * 4, cudaMemcpyHostToDevice, st));
      e = ust_launch_pods_relayout((long long)p.n, (long long)L, h->pl_idx.p, h->pl_off.p, h->pl_shift.p, h->s_podoff.p, h->s_podflags.p,
                                   h->pl_flags.p, (int)p.new_total, h->pl_runs.p, h->s_podoff2.p, h->s_podflags2.p, 8 * h->num_sms, st);
      h->launches += 2;
      std::swap(h->s_podoff, h->s_podoff2);
      std::swap(h->s_podflags, h->s_podflags2);
    }
    if (e) return h->fail(UST_ERR_CUDA, "pod-list kernel launch failed: %s", cudaGetErrorString((cudaError_t)e));
  }
  if (p.gather) {
    UST_CUDA(h, h->inserted.cols.upload(p.ins.state, p.ins.flags, p.ins.rev, p.ins.ds, 0, I, st));
    const Columns &in = h->inserted.cols, &s = h->staged, &x = h->splice_cols;
    int e;
    if (c.reorder) {
      long long* off = h->runs.p;
      long long* src = h->runs.p + NR + 1;
      UST_CUDA(h, cudaMemcpyAsync(off, h->run_off.data(), (NR + 1) * 8, cudaMemcpyHostToDevice, st));
      if (NR) UST_CUDA(h, cudaMemcpyAsync(src, h->run_src.data(), NR * 8, cudaMemcpyHostToDevice, st));
      if (c.clock && I) UST_CUDA(h, cudaMemcpyAsync(h->ins_start.p, c.clock->insert_start, I * 8, cudaMemcpyHostToDevice, st));
      e = ust_launch_reorder((long long)p.n, (long long)NR, off, src, in.hot.p, in.flags.p, in.rev.p, in.ds.p, s.hot.p, s.flags.p, s.rev.p,
                             s.ds.p, h->outs.next.p, h->outs.actions.p, c.pods ? h->s_outcome.p : nullptr, x.hot.p, x.flags.p, x.rev.p,
                             x.ds.p, h->splice_outs.next.p, h->splice_outs.actions.p, c.pods ? h->splice_outcome.p : nullptr, st,
                             c.clock ? h->ins_start.p : nullptr, c.clock ? h->s_start.p : nullptr, c.clock ? h->s_start2.p : nullptr);
      if (e) return h->fail(UST_ERR_CUDA, "reorder kernel launch failed: %s", cudaGetErrorString((cudaError_t)e));
      if (c.pods) std::swap(h->s_outcome, h->splice_outcome);  // the previous outcome in the new order
      if (c.clock) std::swap(h->s_start, h->s_start2);          // the start times in the new order
    } else {
      // a splice keeps its own kernel: the gather kernel measured slower on splices (DESIGN.md §3.4)
      if (R) UST_CUDA(h, cudaMemcpyAsync(h->removed.p, c.splice->remove_idx, R * 8, cudaMemcpyHostToDevice, st));
      if (I) UST_CUDA(h, cudaMemcpyAsync(h->inserted.idx.p, c.splice->insert_before, I * 8, cudaMemcpyHostToDevice, st));
      e = ust_launch_splice((long long)p.n_old, (long long)R, h->removed.p, (long long)p.n_insert, h->inserted.idx.p, in.hot.p, in.flags.p,
                            in.rev.p, in.ds.p, s.hot.p, s.flags.p, s.rev.p, s.ds.p, h->outs.next.p, h->outs.actions.p,
                            x.hot.p, x.flags.p, x.rev.p, x.ds.p, h->splice_outs.next.p, h->splice_outs.actions.p, st);
      if (e) return h->fail(UST_ERR_CUDA, "splice kernel launch failed: %s", cudaGetErrorString((cudaError_t)e));
    }
    h->launches += 1;
    // the new set becomes the resident one (the previous outputs in `outs`, as after any call)
    std::swap(h->staged, h->splice_cols);
    std::swap(h->outs, h->splice_outs);
  }
  if (M) {
    static_assert(sizeof(long long) == sizeof(int64_t), "index width");
    UST_CUDA(h, cudaMemcpyAsync(h->changed.idx.p, c.idx, M * 8, cudaMemcpyHostToDevice, st));
    UST_CUDA(h, h->changed.cols.upload(c.changed.state, c.changed.flags, c.changed.rev, c.changed.ds, 0, M, st));
    if (c.clock) UST_CUDA(h, cudaMemcpyAsync(h->chg_start.p, c.clock->start, M * 8, cudaMemcpyHostToDevice, st));
    const Columns &d = h->changed.cols, &s = h->staged;
    int e = ust_launch_patch((long long)c.n_changed, h->changed.idx.p, d.hot.p, d.flags.p, d.rev.p, d.ds.p, s.hot.p, s.flags.p,
                             s.rev.p, s.ds.p, st, c.clock ? h->chg_start.p : nullptr, c.clock ? h->s_start.p : nullptr);
    if (e) return h->fail(UST_ERR_CUDA, "patch kernel launch failed: %s", cudaGetErrorString((cudaError_t)e));
    h->launches += 1;
  }
  if (c.clock) {
    int rc = launch_clock(h, c.clock, p.n, st);
    if (rc) return rc;
  }
  if (c.sparse) std::swap(h->outs, h->outs_prev);  // the previous call's outputs step aside; this call writes the other pair
  if (c.sparse && c.pods) std::swap(h->s_outcome, h->s_outcome_prev);
  int rc = apply_device(h, c.policy, p.n, h->staged.hot.p, h->staged.flags.p, h->staged.rev.p, h->staged.ds.p, c.n_ds, h->s_dsrev.p,
                        c.pods ? h->s_podoff.p : nullptr, c.pods ? h->s_podflags.p : nullptr, c.pods ? p.new_total : 0, h->outs.next.p,
                        h->outs.actions.p, c.actuator_outcome || c.pods ? h->s_outcome.p : nullptr, nullptr, st, c.clock);
  if (rc) return rc;
  if (!c.sparse) {
    if (N) {
      UST_CUDA(h, cudaMemcpyAsync(c.next_state, h->outs.next.p, N, cudaMemcpyDeviceToHost, st));
      UST_CUDA(h, cudaMemcpyAsync(c.actions, h->outs.actions.p, N * 2, cudaMemcpyDeviceToHost, st));
      if (c.actuator_outcome) UST_CUDA(h, cudaMemcpyAsync(c.actuator_outcome, h->s_outcome.p, N, cudaMemcpyDeviceToHost, st));
    }
  } else {
    int e = ust_launch_diff((long long)p.n, h->outs.next.p, h->outs.actions.p, c.pods ? h->s_outcome.p : nullptr, h->outs_prev.next.p,
                            h->outs_prev.actions.p, c.pods ? h->s_outcome_prev.p : nullptr, h->sp_blocks.p, h->sp_count_dev,
                            (long long)c.max_out, h->sp_idx.p, h->outs_sparse.next.p, h->outs_sparse.actions.p,
                            c.pods ? h->sp_outcome.p : nullptr, st);
    if (e) return h->fail(UST_ERR_CUDA, "diff kernel launch failed: %s", cudaGetErrorString((cudaError_t)e));
    h->launches += 3;
    UST_CUDA(h, cudaMemcpyAsync(h->sp_count_host, h->sp_count_dev, sizeof(long long), cudaMemcpyDeviceToHost, st));
    UST_CUDA(h, cudaStreamSynchronize(st));
    const int64_t cnt = *h->sp_count_host;
    *c.n_out = cnt;
    if (cnt <= c.max_out && cnt > 0) {
      UST_CUDA(h, cudaMemcpyAsync(c.out_idx, h->sp_idx.p, (size_t)cnt * 8, cudaMemcpyDeviceToHost, st));
      UST_CUDA(h, cudaMemcpyAsync(c.next_state, h->outs_sparse.next.p, (size_t)cnt, cudaMemcpyDeviceToHost, st));
      UST_CUDA(h, cudaMemcpyAsync(c.actions, h->outs_sparse.actions.p, (size_t)cnt * 2, cudaMemcpyDeviceToHost, st));
      if (c.pods) UST_CUDA(h, cudaMemcpyAsync(c.actuator_outcome, h->sp_outcome.p, (size_t)cnt, cudaMemcpyDeviceToHost, st));
    }
  }
  rc = adopt_resident(h, finish_with_counters(h, st, c.out), p.n, c.n_ds, true, c.pods ? p.new_total : -1, c.clock != nullptr);
  if (c.sparse && (rc == UST_OK) && *c.n_out > c.max_out)
    return h->fail(UST_ERR_TRUNCATED, "%lld outputs changed, the caller's arrays hold %lld: fetch them with %s", (long long)*c.n_out,
                   (long long)c.max_out, c.pods ? "ust_fetch_outputs_pods" : "ust_fetch_outputs");
  return rc;
}

// The entry of every delta call. `one_gpu`: the name of an entry point that refuses more than one rank (ust_comm_init): a
// shard's node indices and pod lists are its own, so a new order or new lists would have to reach every rank.
static int delta_entry(ust_handle* h, const char* one_gpu, const DeltaCall& c) {
  if (!h) return UST_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> g(h->mu);
  h->prev_n = -1;  // whatever this entry point enqueues sits between two device calls: they keep the strict order
  h->deadline_ready = false;
  if (one_gpu && h->world > 1) return h->fail(UST_ERR_INVALID_ARGUMENT, "%s runs on one GPU", one_gpu);
  DeltaPlan p;
  const int rc = plan_delta(h, c, &p);
  return rc ? rc : run_delta(h, c, p);
}

int ust_apply_state_delta(ust_handle* h, const ust_policy* policy, int64_t n_changed, const int64_t* idx, const uint8_t* state,
                          const uint32_t* flags, const int32_t* pod_rev, const int32_t* ds_idx, int32_t n_ds,
                          const int32_t* ds_rev, uint8_t* next_state, uint16_t* actions, uint8_t* actuator_outcome,
                          ust_counters* out) {
  return delta_entry(h, nullptr, DeltaCall(policy, n_changed, idx, state, flags, pod_rev, ds_idx, n_ds, ds_rev, next_state, actions,
                                           actuator_outcome, out));
}

int ust_apply_state_delta_sparse(ust_handle* h, const ust_policy* policy, int64_t n_changed, const int64_t* idx,
                                 const uint8_t* state, const uint32_t* flags, const int32_t* pod_rev, const int32_t* ds_idx,
                                 int32_t n_ds, const int32_t* ds_rev, int64_t max_out, int64_t* out_idx,
                                 uint8_t* out_next_state, uint16_t* out_actions, int64_t* n_out, ust_counters* out) {
  return delta_entry(h, nullptr, DeltaCall(policy, n_changed, idx, state, flags, pod_rev, ds_idx, n_ds, ds_rev, max_out, out_idx,
                                           out_next_state, out_actions, nullptr, n_out, out));
}

int ust_apply_state_delta_splice(ust_handle* h, const ust_policy* policy, const ust_splice* splice, int64_t n_changed,
                                 const int64_t* idx, const uint8_t* state, const uint32_t* flags, const int32_t* pod_rev,
                                 const int32_t* ds_idx, int32_t n_ds, const int32_t* ds_rev, int64_t max_out, int64_t* out_idx,
                                 uint8_t* out_next_state, uint16_t* out_actions, int64_t* n_out, ust_counters* out) {
  DeltaCall c(policy, n_changed, idx, state, flags, pod_rev, ds_idx, n_ds, ds_rev, max_out, out_idx, out_next_state, out_actions,
              nullptr, n_out, out);
  c.splice = splice;
  return delta_entry(h, "ust_apply_state_delta_splice", c);
}

int ust_apply_state_delta_reorder(ust_handle* h, const ust_policy* policy, const ust_reorder* reorder, int64_t n_changed,
                                  const int64_t* idx, const uint8_t* state, const uint32_t* flags, const int32_t* pod_rev,
                                  const int32_t* ds_idx, int32_t n_ds, const int32_t* ds_rev, int64_t max_out, int64_t* out_idx,
                                  uint8_t* out_next_state, uint16_t* out_actions, int64_t* n_out, ust_counters* out) {
  DeltaCall c(policy, n_changed, idx, state, flags, pod_rev, ds_idx, n_ds, ds_rev, max_out, out_idx, out_next_state, out_actions,
              nullptr, n_out, out);
  c.reorder = reorder;
  return delta_entry(h, "ust_apply_state_delta_reorder", c);
}

int ust_apply_state_delta_pods(ust_handle* h, const ust_policy* policy, const ust_pod_lists* lists, int64_t n_changed,
                               const int64_t* idx, const uint8_t* state, const uint32_t* flags, const int32_t* pod_rev,
                               const int32_t* ds_idx, int32_t n_ds, const int32_t* ds_rev, int64_t max_out, int64_t* out_idx,
                               uint8_t* out_next_state, uint16_t* out_actions, uint8_t* out_outcome, int64_t* n_out, ust_counters* out) {
  DeltaCall c(policy, n_changed, idx, state, flags, pod_rev, ds_idx, n_ds, ds_rev, max_out, out_idx, out_next_state, out_actions,
              out_outcome, n_out, out);
  c.pods = true; c.lists = lists;
  return delta_entry(h, "ust_apply_state_delta_pods", c);
}

int ust_apply_state_delta_pods_reorder(ust_handle* h, const ust_policy* policy, const ust_reorder* reorder, const ust_pod_lists* lists,
                                       int64_t n_changed, const int64_t* idx, const uint8_t* state, const uint32_t* flags,
                                       const int32_t* pod_rev, const int32_t* ds_idx, int32_t n_ds, const int32_t* ds_rev, int64_t max_out,
                                       int64_t* out_idx, uint8_t* out_next_state, uint16_t* out_actions, uint8_t* out_outcome,
                                       int64_t* n_out, ust_counters* out) {
  DeltaCall c(policy, n_changed, idx, state, flags, pod_rev, ds_idx, n_ds, ds_rev, max_out, out_idx, out_next_state, out_actions,
              out_outcome, n_out, out);
  c.reorder = reorder; c.pods = true; c.lists = lists;
  return delta_entry(h, "ust_apply_state_delta_pods_reorder", c);
}

int ust_apply_state_delta_pods_clocked(ust_handle* h, const ust_policy* policy, const ust_clock* clock, const ust_reorder* reorder,
                                       const ust_pod_lists* lists, int64_t n_changed, const int64_t* idx, const uint8_t* state,
                                       const uint32_t* flags, const int32_t* pod_rev, const int32_t* ds_idx, int32_t n_ds,
                                       const int32_t* ds_rev, int64_t max_out, int64_t* out_idx, uint8_t* out_next_state,
                                       uint16_t* out_actions, uint8_t* out_outcome, int64_t* n_out, ust_counters* out) {
  DeltaCall c(policy, n_changed, idx, state, flags, pod_rev, ds_idx, n_ds, ds_rev, max_out, out_idx, out_next_state, out_actions,
              out_outcome, n_out, out);
  c.reorder = reorder; c.pods = true; c.lists = lists; c.clocked = true; c.clock = clock;
  return delta_entry(h, "ust_apply_state_delta_pods_clocked", c);
}

int ust_fetch_outputs_pods(ust_handle* h, uint8_t* next_state, uint16_t* actions, uint8_t* actuator_outcome) {
  if (!h) return UST_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> g(h->mu);
  h->prev_n = -1;  // whatever this entry point enqueues sits between two device calls: they keep the strict order
  if (h->pods_n < 0) return h->fail(UST_ERR_INVALID_ARGUMENT, "no resident pod-list outputs");
  if (h->pods_n > 0 && (!next_state || !actions || !actuator_outcome)) return h->fail(UST_ERR_INVALID_ARGUMENT, "bad arguments");
  UST_CUDA(h, cudaSetDevice(h->device));
  const size_t N = (size_t)h->pods_n;
  if (N) {
    UST_CUDA(h, cudaMemcpyAsync(next_state, h->outs.next.p, N, cudaMemcpyDeviceToHost, h->stream));
    UST_CUDA(h, cudaMemcpyAsync(actions, h->outs.actions.p, N * 2, cudaMemcpyDeviceToHost, h->stream));
    UST_CUDA(h, cudaMemcpyAsync(actuator_outcome, h->s_outcome.p, N, cudaMemcpyDeviceToHost, h->stream));
  }
  UST_CUDA(h, cudaStreamSynchronize(h->stream));
  return UST_OK;
}

int ust_next_deadline(ust_handle* h, int64_t* t) {
  if (!h) return UST_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> g(h->mu);
  h->prev_n = -1;  // whatever this entry point enqueues sits between two device calls: they keep the strict order
  if (!t) return h->fail(UST_ERR_INVALID_ARGUMENT, "t: required");
  if (h->world > 1)  // each rank would know only its shard's candidates, and its abort point only by the global index
    return h->fail(UST_ERR_INVALID_ARGUMENT, "ust_next_deadline runs on one GPU: more than one rank is set up by ust_comm_init");
  if (h->pods_n < 0 || !h->pods_clocked)
    return h->fail(UST_ERR_INVALID_ARGUMENT, "no clocked pod-list snapshot is resident: call ust_apply_state_clocked first");
  if (!h->deadline_ready)
    return h->fail(UST_ERR_INVALID_ARGUMENT, "the last call on the handle was not a clocked call that left its snapshot resident");
  UST_CUDA(h, cudaSetDevice(h->device));
  unsigned long long key = 0;
  UST_CUDA(h, cudaMemcpyAsync(&key, h->clk_deadline.p, sizeof(key), cudaMemcpyDeviceToHost, h->stream));
  UST_CUDA(h, cudaStreamSynchronize(h->stream));
  // key: the smallest deadline d with its sign bit flipped, ~0 = none; the bit turns on at d + 1 (d < INT64_MAX)
  *t = key == ~0ull ? INT64_MIN : (int64_t)(key ^ (1ull << 63)) + 1;
  return UST_OK;
}

int ust_fetch_outputs(ust_handle* h, uint8_t* next_state, uint16_t* actions) {
  if (!h) return UST_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> g(h->mu);
  h->prev_n = -1;  // whatever this entry point enqueues sits between two device calls: they keep the strict order
  if (h->resident_n < 0 || !h->outputs_resident) return h->fail(UST_ERR_INVALID_ARGUMENT, "no resident outputs");
  if (h->resident_n > 0 && (!next_state || !actions)) return h->fail(UST_ERR_INVALID_ARGUMENT, "bad arguments");
  UST_CUDA(h, cudaSetDevice(h->device));
  const size_t N = (size_t)h->resident_n;
  if (N) {
    UST_CUDA(h, cudaMemcpyAsync(next_state, h->outs.next.p, N, cudaMemcpyDeviceToHost, h->stream));
    UST_CUDA(h, cudaMemcpyAsync(actions, h->outs.actions.p, N * 2, cudaMemcpyDeviceToHost, h->stream));
  }
  UST_CUDA(h, cudaStreamSynchronize(h->stream));
  return UST_OK;
}

int ust_apply_state_packed(ust_handle* h, const ust_policy* policy, int64_t n, const uint8_t* state, const uint32_t* flags,
                           const uint16_t* pod_rev16, const int8_t* ds_idx8, int32_t n_ds, const int32_t* ds_rev,
                           uint8_t* next_state, uint16_t* actions, uint8_t* actuator_outcome, ust_counters* out) {
  if (!h) return UST_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> g(h->mu);
  h->deadline_ready = false;
  h->prev_n = -1;  // whatever this entry point enqueues sits between two device calls: they keep the strict order
  if (n < 0 || (n > 0 && (!state || !flags || !pod_rev16 || !ds_idx8 || !next_state || !actions)))
    return h->fail(UST_ERR_NIL_STATE, "currentState should not be empty");
  if (n_ds < 0 || n_ds > 127 || (n_ds > 0 && !ds_rev)) return h->fail(UST_ERR_INVALID_ARGUMENT, "bad DaemonSet table (the packed format holds at most 127 DaemonSets)");
  if (int rc = check_eval_mode(h, policy, false)) return rc;
  return apply_host(h, policy, n, HostNodes{state, flags, nullptr, nullptr, pod_rev16, ds_idx8}, n_ds, ds_rev, nullptr,
                    next_state, actions, actuator_outcome, out);
}

static int simulate_common(ust_handle* h, const ust_policy* policy, const ust_sim_options* opt, int32_t steps, ust_counters* history,
                           uint8_t* final_state, uint32_t* final_flags, int32_t* final_pod_rev, int32_t* steps_done) {
  if (int rc = check_eval_mode(h, policy, false)) return rc;
  const int64_t n = h->resident_n;
  if (n < 0) return h->fail(UST_ERR_INVALID_ARGUMENT, "no resident snapshot: call ust_apply_state (without pod lists) first");
  if (steps < 0 || steps > (1 << 20)) return h->fail(UST_ERR_INVALID_ARGUMENT, "bad step count");
  if (h->world > 1) return h->fail(UST_ERR_INVALID_ARGUMENT, "rollout simulation runs on one GPU");
  if (opt && (opt->seconds_per_reconcile < 0 || opt->wait_timeout_seconds < 0 || opt->job_seconds < 0 || opt->validation_timeout_seconds < 0 ||
              opt->maintenance_seconds < 0 || (int64_t)steps * opt->seconds_per_reconcile >= (1LL << 29)))
    return h->fail(UST_ERR_INVALID_ARGUMENT, "bad simulation options (times are non-negative; the horizon stays below 2^29 seconds)");
  if (opt && policy && (policy->wait_timeout_nonzero != 0) != (opt->wait_timeout_seconds != 0))
    return h->fail(UST_ERR_INVALID_ARGUMENT, "policy.wait_timeout_nonzero must say whether wait_timeout_seconds != 0");
  ust_policy pol;
  if (policy) { pol = *policy; pol.evaluate_actuators = 1; }  // the asynchronous actuators' results are what is fed back
  UST_CUDA(h, cudaSetDevice(h->device));
  StreamDrain drain(h);
  cudaStream_t st = h->stream;
  const size_t N = (size_t)n;
  UST_CUDA(h, h->s_outcome.reserve(N + 16));
  UST_CUDA(h, h->sim_hist.reserve((size_t)steps + 1));
  const int32_t n_ds = h->resident_n_ds;
  drop_resident(h);
  int grid = 8 * h->num_sms;
  UstSimParams sp;
  memset(&sp, 0, sizeof(sp));
  if (opt) {
    sp.timed = 1;
    sp.dt = opt->seconds_per_reconcile;
    sp.wait_timeout = opt->wait_timeout_seconds; sp.job_seconds = opt->job_seconds; sp.validation_seconds = opt->validation_seconds;
    sp.validation_timeout = opt->validation_timeout_seconds; sp.maintenance_seconds = opt->maintenance_seconds;
    UST_CUDA(h, h->sim_entered.reserve(N + 1)); UST_CUDA(h, h->sim_wait.reserve(N + 1)); UST_CUDA(h, h->sim_valid.reserve(N + 1));
    int e = ust_launch_sim_init(n, h->staged.flags.p, h->sim_entered.p, h->sim_wait.p, h->sim_valid.p, grid, st);
    if (e) return h->fail(UST_ERR_CUDA, "simulation init kernel launch failed: %s", cudaGetErrorString((cudaError_t)e));
    h->launches += 1;
  }
  const Columns& s = h->staged;
  for (int32_t k = 0; k < steps; k++) {
    int rc = apply_device(h, policy ? &pol : nullptr, n, s.hot.p, s.flags.p, s.rev.p, s.ds.p, n_ds, h->s_dsrev.p, nullptr, nullptr,
                          0, h->outs.next.p, h->outs.actions.p, h->s_outcome.p, h->sim_hist.p + k, st);
    if (rc) return rc;
    sp.now = (long long)k * sp.dt;
    int e = ust_launch_feedback(n, s.hot.p, s.flags.p, s.rev.p, s.ds.p, n_ds, h->s_dsrev.p, h->outs.next.p, h->outs.actions.p,
                                h->s_outcome.p, h->sim_hist.p + k, sp, h->sim_entered.p, h->sim_wait.p, h->sim_valid.p, grid, st);
    if (e) return h->fail(UST_ERR_CUDA, "feedback kernel launch failed: %s", cudaGetErrorString((cudaError_t)e));
    h->launches += 1;
  }
  std::vector<ust_counters> hist((size_t)steps);
  if (steps) UST_CUDA(h, cudaMemcpyAsync(hist.data(), h->sim_hist.p, (size_t)steps * sizeof(ust_counters), cudaMemcpyDeviceToHost, st));
  if (N && final_state) UST_CUDA(h, cudaMemcpyAsync(final_state, s.hot.p, N, cudaMemcpyDeviceToHost, st));
  if (N && final_flags) UST_CUDA(h, cudaMemcpyAsync(final_flags, s.flags.p, N * 4, cudaMemcpyDeviceToHost, st));
  if (N && final_pod_rev) UST_CUDA(h, cudaMemcpyAsync(final_pod_rev, s.rev.p, N * 4, cudaMemcpyDeviceToHost, st));
  cudaError_t ce = cudaStreamSynchronize(st);
  if (ce != cudaSuccess) { h->ws_dirty = true; return h->fail(UST_ERR_CUDA, "kernel execution failed: %s", cudaGetErrorString(ce)); }
  adopt_resident(h, UST_OK, n, n_ds, false);  // the snapshot now holds the simulated state
  int32_t done = steps;
  int rc = UST_OK;
  for (int32_t k = 0; k < steps; k++)
    if (hist[(size_t)k].error_code != UST_OK) { done = k; rc = (int)hist[(size_t)k].error_code; break; }
  if (history) memcpy(history, hist.data(), (size_t)steps * sizeof(ust_counters));
  if (steps_done) *steps_done = done;
  if (rc) return h->fail(rc, "the simulated reconcile %d returned an error (code %d); the state before it is kept", (int)done, rc);
  return UST_OK;
}

int ust_simulate_rollout(ust_handle* h, const ust_policy* policy, int32_t steps, ust_counters* history, uint8_t* final_state,
                         uint32_t* final_flags, int32_t* final_pod_rev, int32_t* steps_done) {
  if (!h) return UST_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> g(h->mu);
  h->deadline_ready = false;
  h->prev_n = -1;  // whatever this entry point enqueues sits between two device calls: they keep the strict order
  return simulate_common(h, policy, nullptr, steps, history, final_state, final_flags, final_pod_rev, steps_done);
}

int ust_simulate_rollout_timed(ust_handle* h, const ust_policy* policy, const ust_sim_options* options, int32_t steps,
                               ust_counters* history, uint8_t* final_state, uint32_t* final_flags, int32_t* final_pod_rev,
                               int32_t* steps_done) {
  if (!h) return UST_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> g(h->mu);
  h->deadline_ready = false;
  if (!options) return UST_ERR_INVALID_ARGUMENT;
  h->prev_n = -1;  // whatever this entry point enqueues sits between two device calls: they keep the strict order
  return simulate_common(h, policy, options, steps, history, final_state, final_flags, final_pod_rev, steps_done);
}

int ust_build_state(ust_handle* h, int64_t n_pods, const uint8_t* state, const int32_t* ds_idx, int32_t n_ds,
                    const int32_t* ds_desired, ust_counters* out) {
  if (!h) return UST_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> g(h->mu);
  h->deadline_ready = false;
  h->prev_n = -1;  // whatever this entry point enqueues sits between two device calls: they keep the strict order
  if (n_pods < 0 || (n_pods > 0 && (!state || !ds_idx)) || n_ds < 0 || (n_ds > 0 && !ds_desired))
    return h->fail(UST_ERR_INVALID_ARGUMENT, "bad arguments");
  drop_resident(h);  // shares the staging arrays
  UST_CUDA(h, cudaSetDevice(h->device));
  StreamDrain drain(h);
  cudaStream_t st = h->stream;
  const size_t N = (size_t)n_pods;
  UST_CUDA(h, h->staged.hot.reserve(N + 16));
  UST_CUDA(h, h->staged.ds.reserve(N + 4));
  UST_CUDA(h, h->s_dsdesired.reserve((size_t)n_ds + 1));
  if (N) {
    UST_CUDA(h, cudaMemcpyAsync(h->staged.hot.p, state, N, cudaMemcpyHostToDevice, st));
    UST_CUDA(h, cudaMemcpyAsync(h->staged.ds.p, ds_idx, N * 4, cudaMemcpyHostToDevice, st));
  }
  if (n_ds) UST_CUDA(h, cudaMemcpyAsync(h->s_dsdesired.p, ds_desired, (size_t)n_ds * 4, cudaMemcpyHostToDevice, st));
  int rc = build_state_launch(h, n_pods, n_ds, st, [&](int grid) {
    return ust_launch_build_state(n_pods, h->staged.hot.p, h->staged.ds.p, n_ds, h->s_dsdesired.p, h->ds_count.p, h->ws,
                                  h->counters_dev, grid, st);
  });
  if (rc) return rc;
  return finish_with_counters(h, st, out);
}

int ust_build_state_uids(ust_handle* h, int64_t n_pods, const uint8_t* state, const uint64_t* owner_uid, int32_t n_ds,
                         const uint64_t* ds_uid, const int32_t* ds_desired, int32_t* ds_idx_out, ust_counters* out) {
  if (!h) return UST_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> g(h->mu);
  h->deadline_ready = false;
  h->prev_n = -1;  // whatever this entry point enqueues sits between two device calls: they keep the strict order
  if (n_pods < 0 || (n_pods > 0 && (!state || !owner_uid || !ds_idx_out)) || n_ds < 0 || (n_ds > 0 && (!ds_uid || !ds_desired)))
    return h->fail(UST_ERR_INVALID_ARGUMENT, "bad arguments");
  DsTable tab;
  if (int rc = ds_table(h, n_ds, ds_uid, &tab)) return rc;
  drop_resident(h);  // shares the staging arrays
  UST_CUDA(h, cudaSetDevice(h->device));
  StreamDrain drain(h);
  cudaStream_t st = h->stream;
  const size_t N = (size_t)n_pods;
  UST_CUDA(h, h->staged.hot.reserve(N + 16));
  UST_CUDA(h, h->staged.ds.reserve(N + 4));
  UST_CUDA(h, h->s_uid.reserve(2 * N + 2));
  if (N) {
    UST_CUDA(h, cudaMemcpyAsync(h->staged.hot.p, state, N, cudaMemcpyHostToDevice, st));
    UST_CUDA(h, cudaMemcpyAsync(h->s_uid.p, owner_uid, N * 16, cudaMemcpyHostToDevice, st));
  }
  if (int rc = upload_ds_table(h, tab, n_ds, ds_desired, st)) return rc;
  int rc = build_state_launch(h, n_pods, n_ds, st, [&](int grid) {
    return ust_launch_build_state_uids(n_pods, h->staged.hot.p, h->s_uid.p, n_ds, h->s_dsuid.p, h->s_dsorder.p, (int)tab.slots,
                                       h->s_dsdesired.p, h->staged.ds.p, h->ds_count.p, h->ws, h->counters_dev, grid, st);
  });
  if (rc) return rc;
  if (N) UST_CUDA(h, cudaMemcpyAsync(ds_idx_out, h->staged.ds.p, N * 4, cudaMemcpyDeviceToHost, st));
  return finish_with_counters(h, st, out);  // synchronises the stream: the table outlives its copies
}

int ust_build_state_delta(ust_handle* h, const ust_driver_pod_reorder* reorder, int64_t n_changed, const int64_t* idx,
                          const uint8_t* state, const uint64_t* owner_uid, int32_t n_ds, const uint64_t* ds_uid,
                          const int32_t* ds_desired, int64_t max_out, int64_t* out_idx, int32_t* out_ds_idx, int64_t* n_out,
                          ust_counters* out) {
  if (!h) return UST_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> g(h->mu);
  h->deadline_ready = false;
  h->prev_n = -1;  // whatever this entry point enqueues sits between two device calls: they keep the strict order
  // the new order and every argument, checked in full before anything is touched
  const int64_t n_old = h->bs_n;
  int64_t n = n_old;
  if (reorder) {
    if (reorder->n_insert > 0 && (!reorder->state || !reorder->owner_uid)) return h->fail(UST_ERR_INVALID_ARGUMENT, "bad reorder");
    if (int rc = reorder_runs(h, reorder->n_runs, reorder->run_src, reorder->run_len, reorder->n_insert, n_old, &n)) return rc;
  }
  // the tile offsets of the sparse outputs are 32-bit
  if (n >= (1LL << 31)) return h->fail(UST_ERR_INVALID_ARGUMENT, "too many pods: the driver-pod list holds fewer than 2^31");
  if (n_changed < 0 || (n_changed > 0 && (!idx || !state || !owner_uid)) || max_out < 0 || !n_out ||
      (max_out > 0 && (!out_idx || !out_ds_idx)))
    return h->fail(UST_ERR_INVALID_ARGUMENT, "bad arguments");
  if (n_ds < 0 || (n_ds > 0 && (!ds_uid || !ds_desired))) return h->fail(UST_ERR_INVALID_ARGUMENT, "bad DaemonSet table");
  {  // idx: distinct indices into the new list (the reorder's bitmap, all zero again afterwards)
    const size_t words = ((size_t)n + 63) / 64;
    if (h->run_seen.size() < words) h->run_seen.resize(words, 0);
    int64_t k = 0;
    int rc = UST_OK;
    for (; k < n_changed; k++) {
      if (idx[k] < 0 || idx[k] >= n) {
        rc = h->fail(UST_ERR_INVALID_ARGUMENT, "changed pod %lld has index %lld outside the list of %lld pods", (long long)k, (long long)idx[k], (long long)n);
        break;
      }
      if (!mark_bits(h->run_seen.data(), idx[k], 1, true)) {
        rc = h->fail(UST_ERR_INVALID_ARGUMENT, "changed pod %lld: index %lld is named twice", (long long)k, (long long)idx[k]);
        break;
      }
    }
    for (int64_t j = 0; j < k; j++) mark_bits(h->run_seen.data(), idx[j], 1, false);
    if (rc) return rc;
  }
  DsTable tab;
  if (int rc = ds_table(h, n_ds, ds_uid, &tab)) return rc;
  h->bs_n = 0;  // empty until the call has produced counters
  UST_CUDA(h, cudaSetDevice(h->device));
  StreamDrain drain(h);
  cudaStream_t st = h->stream;
  const size_t N = (size_t)n, M = (size_t)n_changed, NR = h->run_src.size();
  const size_t I = reorder ? (size_t)reorder->n_insert : 0;
  if (reorder) {  // the new order, gathered into the second set, which becomes the resident one
    UST_CUDA(h, h->bs2.hot.reserve(N + 16));
    UST_CUDA(h, h->bs2.uid.reserve(2 * N + 2));
    UST_CUDA(h, h->bs2.owner.reserve(N + 4));
    UST_CUDA(h, h->runs.reserve(2 * NR + 2));
    UST_CUDA(h, h->bs_ins_hot.reserve(I + 1));
    UST_CUDA(h, h->bs_ins_uid.reserve(2 * I + 2));
    long long* off = h->runs.p;
    long long* src = h->runs.p + NR + 1;
    UST_CUDA(h, cudaMemcpyAsync(off, h->run_off.data(), (NR + 1) * 8, cudaMemcpyHostToDevice, st));
    if (NR) UST_CUDA(h, cudaMemcpyAsync(src, h->run_src.data(), NR * 8, cudaMemcpyHostToDevice, st));
    if (I) {
      UST_CUDA(h, cudaMemcpyAsync(h->bs_ins_hot.p, reorder->state, I, cudaMemcpyHostToDevice, st));
      UST_CUDA(h, cudaMemcpyAsync(h->bs_ins_uid.p, reorder->owner_uid, I * 16, cudaMemcpyHostToDevice, st));
    }
    int e = ust_launch_build_state_reorder((long long)n, (long long)NR, off, src, h->bs_ins_hot.p, h->bs_ins_uid.p, h->bs.hot.p,
                                           h->bs.uid.p, h->bs.owner.p, h->bs2.hot.p, h->bs2.uid.p, h->bs2.owner.p, st);
    if (e) return h->fail(UST_ERR_CUDA, "driver-pod reorder kernel launch failed: %s", cudaGetErrorString((cudaError_t)e));
    h->launches += 1;
    std::swap(h->bs, h->bs2);
  } else {  // same size as before: no-ops once the list holds pods
    UST_CUDA(h, h->bs.hot.reserve(N + 16));
    UST_CUDA(h, h->bs.uid.reserve(2 * N + 2));
    UST_CUDA(h, h->bs.owner.reserve(N + 4));
  }
  UST_CUDA(h, h->bs2.owner.reserve(N + 4));  // this call's owner indices
  if (M) {
    UST_CUDA(h, h->changed.idx.reserve(M + 1));
    UST_CUDA(h, h->bs_chg_hot.reserve(M + 1));
    UST_CUDA(h, h->bs_chg_uid.reserve(2 * M + 2));
    static_assert(sizeof(long long) == sizeof(int64_t), "index width");
    UST_CUDA(h, cudaMemcpyAsync(h->changed.idx.p, idx, M * 8, cudaMemcpyHostToDevice, st));
    UST_CUDA(h, cudaMemcpyAsync(h->bs_chg_hot.p, state, M, cudaMemcpyHostToDevice, st));
    UST_CUDA(h, cudaMemcpyAsync(h->bs_chg_uid.p, owner_uid, M * 16, cudaMemcpyHostToDevice, st));
    int e = ust_launch_build_state_patch((long long)M, h->changed.idx.p, h->bs_chg_hot.p, h->bs_chg_uid.p, h->bs.hot.p, h->bs.uid.p, st);
    if (e) return h->fail(UST_ERR_CUDA, "driver-pod patch kernel launch failed: %s", cudaGetErrorString((cudaError_t)e));
    h->launches += 1;
  }
  const int tiles = ust_build_state_tiles((long long)n);
  UST_CUDA(h, h->sp_blocks.reserve((size_t)tiles + 1));
  UST_CUDA(h, h->sp_idx.reserve((size_t)max_out + 1));
  UST_CUDA(h, h->bs_out_ds.reserve((size_t)max_out + 1));
  if (int rc = upload_ds_table(h, tab, n_ds, ds_desired, st)) return rc;
  int rc = build_state_launch(h, n, n_ds, st, [&](int grid) {
    return ust_launch_build_state_delta((long long)n, h->bs.hot.p, h->bs.uid.p, n_ds, h->s_dsuid.p, h->s_dsorder.p, (int)tab.slots,
                                        h->s_dsdesired.p, h->bs.owner.p, h->bs2.owner.p, h->sp_blocks.p, h->ds_count.p, h->ws,
                                        h->counters_dev, grid, st);
  });
  if (rc) return rc;
  int e = ust_launch_build_state_write((long long)n, h->bs2.owner.p, h->bs.owner.p, h->sp_blocks.p, h->sp_count_dev, (long long)max_out,
                                       h->sp_idx.p, h->bs_out_ds.p, st);
  if (e) return h->fail(UST_ERR_CUDA, "driver-pod diff kernel launch failed: %s", cudaGetErrorString((cudaError_t)e));
  h->launches += tiles > 0 ? 2 : 1;
  UST_CUDA(h, cudaMemcpyAsync(h->sp_count_host, h->sp_count_dev, sizeof(long long), cudaMemcpyDeviceToHost, st));
  UST_CUDA(h, cudaStreamSynchronize(st));
  const int64_t cnt = *h->sp_count_host;
  *n_out = cnt;
  if (cnt <= max_out && cnt > 0) {
    UST_CUDA(h, cudaMemcpyAsync(out_idx, h->sp_idx.p, (size_t)cnt * 8, cudaMemcpyDeviceToHost, st));
    UST_CUDA(h, cudaMemcpyAsync(out_ds_idx, h->bs_out_ds.p, (size_t)cnt * 4, cudaMemcpyDeviceToHost, st));
  }
  rc = finish_with_counters(h, st, out);
  if (rc == UST_ERR_CUDA) return rc;
  std::swap(h->bs.owner, h->bs2.owner);  // this call's owner indices are the previous ones of the next call
  h->bs_n = n;
  if (rc == UST_OK && cnt > max_out)
    return h->fail(UST_ERR_TRUNCATED, "%lld owner indices changed, the caller's arrays hold %lld: fetch them with ust_fetch_build_state",
                   (long long)cnt, (long long)max_out);
  return rc;
}

int ust_fetch_build_state(ust_handle* h, int64_t n_pods, int32_t* ds_idx) {
  if (!h) return UST_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> g(h->mu);
  h->prev_n = -1;  // whatever this entry point enqueues sits between two device calls: they keep the strict order
  if (n_pods != h->bs_n) return h->fail(UST_ERR_INVALID_ARGUMENT, "the resident driver-pod list holds %lld pods, not %lld", (long long)h->bs_n, (long long)n_pods);
  if (n_pods > 0 && !ds_idx) return h->fail(UST_ERR_INVALID_ARGUMENT, "bad arguments");
  UST_CUDA(h, cudaSetDevice(h->device));
  if (n_pods) UST_CUDA(h, cudaMemcpyAsync(ds_idx, h->bs.owner.p, (size_t)n_pods * 4, cudaMemcpyDeviceToHost, h->stream));
  UST_CUDA(h, cudaStreamSynchronize(h->stream));
  return UST_OK;
}

uint32_t ust_table_entry(const ust_policy* policy, unsigned state_code, uint32_t w) {
  // the very table the kernels stage and the very lookup they make (ust_lut.h), built for `policy` (cached per thread)
  static thread_local std::vector<uint32_t> lut;
  static thread_local ust_policy cached;
  static thread_local bool have = false;
  state_code &= 15u;
  const ust_policy key = table_key(policy);
  if (!have || memcmp(&key, &cached, sizeof(key)) != 0) {
    lut.assign(UST_LUT_WORDS, 0u);
    ust_build_lut(policy_active(policy) ? &key : nullptr, lut.data());
    cached = key;
    have = true;
  }
  return ust_lut_lookup(lut.data(), state_code, w);
}
int ust_table_window_shift(unsigned state_code) { return ust_window_shift[state_code & 15u]; }
int ust_table_window(const ust_policy* policy, unsigned state_code, int* width) {
  const ust_policy key = table_key(policy);  // the policy the table is built for (an inactive one: the plain layout)
  const ust_policy* p = policy_active(policy) ? &key : nullptr;
  if (width) *width = ust_policy_bits_of(p, (int)(state_code & 15u));
  return ust_policy_shift_of(p, (int)(state_code & 15u));
}

// audit: entries of the 2048-entry pod table (ust_build_pod_lut) that T[pf & 255] & gate(pf) disagrees with
int ust_debug_podlut_mismatches(const ust_policy* p) {
  if (!p) return -1;
  uint8_t full[UST_PODLUT_ENTRIES], T[256];
  ust_build_pod_lut(p, full);
  ust_build_pod_lut256(p, T);
  int bad = 0;
  for (unsigned pf = 0; pf < UST_PODLUT_ENTRIES; pf++) bad += (T[pf & 255u] & ust_pod_gate(pf)) != full[pf];
  return bad;
}

long long ust_debug_relaxed_calls(ust_handle* h) { return h ? (long long)h->relaxed_calls : -1; }

// diagnostics: host nanoseconds of the last list-length pass (pods_reorder_segments) of ust_apply_state_delta_pods_reorder
long long ust_debug_pod_pass_ns(ust_handle* h) { return h ? h->pod_pass_ns : -1; }

// diagnostics (not in include/ust.h): %globaltimer stamps taken by CTA 0 of the last fused launch
int ust_debug_stamps(ust_handle* h, unsigned long long* out, int n_ctas) {
  if (!h || !out || n_ctas < 1 || n_ctas > UST_MAX_CTAS) return UST_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> g(h->mu);
  h->prev_n = -1;  // whatever this entry point enqueues sits between two device calls: they keep the strict order
  UST_CUDA(h, cudaSetDevice(h->device));
  UST_CUDA(h, cudaDeviceSynchronize());
  const unsigned last = (h->call_seq - 1u) & 1u;
  UST_CUDA(h, cudaMemcpy(out, h->ws->dbg[last], (size_t)n_ctas * 4 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  UST_CUDA(h, cudaMemcpy(out + (size_t)n_ctas * 4, h->ws->dbg2, 16 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));  // verification kernel
  return UST_OK;
}

// diagnostics: the streaming CTAs' stamps of the last two calls (UST_STAMPS). out[c][i][0..4] for c = 0 (the call before
// the last one) and 1 (the last call), CTA i < n_ctas: entry, first tile landed, stream end, exit (%globaltimer ns), SM id
int ust_debug_stamps_pair(ust_handle* h, unsigned long long* out, int n_ctas) {
  if (!h || !out || n_ctas < 1 || n_ctas > UST_MAX_CTAS) return UST_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> g(h->mu);
  h->prev_n = -1;
  UST_CUDA(h, cudaSetDevice(h->device));
  UST_CUDA(h, cudaDeviceSynchronize());
  std::vector<unsigned long long> st((size_t)2 * UST_MAX_CTAS * 4);
  std::vector<unsigned int> sm((size_t)2 * UST_MAX_CTAS);
  UST_CUDA(h, cudaMemcpy(st.data(), h->ws->dbg, st.size() * sizeof(st[0]), cudaMemcpyDeviceToHost));
  UST_CUDA(h, cudaMemcpy(sm.data(), h->ws->dbg_sm, sm.size() * sizeof(sm[0]), cudaMemcpyDeviceToHost));
  const unsigned last = (h->call_seq - 1u) & 1u;
  for (int c = 0; c < 2; c++) {
    const unsigned par = c == 1 ? last : last ^ 1u;
    for (int i = 0; i < n_ctas; i++) {
      unsigned long long* o = out + ((size_t)c * n_ctas + i) * 5;
      for (int k = 0; k < 4; k++) o[k] = st[((size_t)par * UST_MAX_CTAS + i) * 4 + k];
      o[4] = sm[(size_t)par * UST_MAX_CTAS + i];
    }
  }
  return UST_OK;
}

// diagnostics: streaming CTAs one SM holds (cudaOccupancyMaxActiveBlocksPerMultiprocessor, fewest over the kernel's variants)
int ust_debug_stream_ctas_per_sm(ust_handle* h) { return h ? h->stream_ctas_per_sm : -1; }

int ust_get_unique_id(void* out_bytes) {
  if (!out_bytes) return UST_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> g(g_nccl_mu);
  std::string err;
  if (!g_nccl.load(&err)) { g_create_error = err; return UST_ERR_COMM; }
  ncclUniqueId id;
  static_assert(sizeof(ncclUniqueId) == UST_UNIQUE_ID_BYTES, "ncclUniqueId size");
  if (g_nccl.GetUniqueId(&id) != ncclSuccess) { g_create_error = "ncclGetUniqueId failed"; return UST_ERR_COMM; }
  memcpy(out_bytes, &id, sizeof(id));
  return UST_OK;
}

int ust_comm_init(ust_handle* h, int rank, int world_size, const void* unique_id_bytes) {
  if (!h) return UST_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> g(h->mu);
  h->deadline_ready = false;
  h->prev_n = -1;  // whatever this entry point enqueues sits between two device calls: they keep the strict order
  if (world_size < 1 || world_size > UST_MAX_WORLD || rank < 0 || rank >= world_size)
    return h->fail(UST_ERR_INVALID_ARGUMENT, "world size must be 1..%d", UST_MAX_WORLD);
  if (world_size == 1) { h->rank = 0; h->world = 1; return UST_OK; }
  if (!unique_id_bytes) return h->fail(UST_ERR_INVALID_ARGUMENT, "unique id required");
  {
    std::lock_guard<std::mutex> g2(g_nccl_mu);
    std::string err;
    if (!g_nccl.load(&err)) return h->fail(UST_ERR_COMM, "%s", err.c_str());
  }
  UST_CUDA(h, cudaSetDevice(h->device));
  ncclUniqueId id;
  memcpy(&id, unique_id_bytes, sizeof(id));
  ncclResult_t r = g_nccl.CommInitRank(&h->comm, world_size, id, rank);
  if (r != ncclSuccess) return h->fail(UST_ERR_COMM, "ncclCommInitRank failed: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?");
  h->rank = rank;
  h->world = world_size;
  // Mailboxes for the fused exchange: allocate, all-gather the CUDA IPC handles over the new communicator, map the
  // peers' buffers. Any failure leaves the NCCL exchange (mode 0) as the only mode.
  h->mbox_ready = false;
  do {
    if (!g_nccl.AllGather) break;
    if (cudaMalloc(&h->mbox_own, sizeof(UstMailbox)) != cudaSuccess) break;
    if (cudaMemset(h->mbox_own, 0, sizeof(UstMailbox)) != cudaSuccess) break;
    cudaIpcMemHandle_t mine;
    if (cudaIpcGetMemHandle(&mine, h->mbox_own) != cudaSuccess) { cudaGetLastError(); break; }
    cudaIpcMemHandle_t* dev = nullptr;
    if (cudaMalloc(&dev, sizeof(cudaIpcMemHandle_t) * (size_t)(world_size + 1)) != cudaSuccess) break;
    cudaMemcpy(dev + world_size, &mine, sizeof(mine), cudaMemcpyHostToDevice);
    ncclResult_t g = g_nccl.AllGather(dev + world_size, dev, sizeof(mine), ncclChar, h->comm, h->stream);
    cudaError_t ce = cudaStreamSynchronize(h->stream);
    std::vector<cudaIpcMemHandle_t> all((size_t)world_size);
    if (g == ncclSuccess && ce == cudaSuccess) cudaMemcpy(all.data(), dev, sizeof(mine) * (size_t)world_size, cudaMemcpyDeviceToHost);
    cudaFree(dev);
    if (g != ncclSuccess || ce != cudaSuccess) break;
    bool ok = true;
    for (int r = 0; r < world_size && ok; r++) {
      if (r == rank) { h->mbox[r] = h->mbox_own; continue; }
      void* p = nullptr;
      if (cudaIpcOpenMemHandle(&p, all[(size_t)r], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); ok = false; break; }
      h->mbox[r] = (UstMailbox*)p;
    }
    h->mbox_ready = ok;
  } while (0);
  h->epoch = 0;
  return UST_OK;
}

int ust_comm_set_mode(ust_handle* h, int mode) {
  if (!h) return UST_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> g(h->mu);
  h->prev_n = -1;  // whatever this entry point enqueues sits between two device calls: they keep the strict order
  if (mode != 0 && mode != 1) return h->fail(UST_ERR_INVALID_ARGUMENT, "unknown exchange mode %d", mode);
  if (mode == 1 && !(h->world > 1 && h->mbox_ready))
    return h->fail(UST_ERR_COMM, "fused exchange unavailable: peer mailboxes could not be mapped (CUDA IPC)");
  h->comm_mode = mode;
  return UST_OK;
}

}  // extern "C"
#pragma GCC visibility pop
