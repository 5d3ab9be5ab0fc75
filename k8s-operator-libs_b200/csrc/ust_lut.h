// ust_lut.h — per-policy transition tables consumed by the sm_90a kernels (ust_kernels.cu).
//
// The kernel never branches on a node's state. For every node it forms a 32-bit predicate word
//   w = (flags & UST_F_INPUT_MASK) | skip/unschedulable from the hot byte | derived bits
// and looks the result up in a table indexed by (state code, the window of w that state reads: up to 9 bits). Which
// window a state reads is fixed by the bit layout in include/ust.h; WHAT each (state, window) maps to depends on the
// policy and the manager options, so the table is rebuilt whenever those change (1105 entries packed widest window
// first, built on the host in microseconds, cached in the handle, 4.4 KiB in shared memory per CTA).
//
// Entry layout:  bits 0-15 actions (UST_A_*), bits 16-23 next state, bits 24-31 actuator outcome
// (UST_OUTCOME_NONE = no actuator ran) — byte-aligned so the kernel packs four nodes with PRMT.
#pragma once
#include <stdint.h>

#include "../../include/ust.h"

#ifdef __CUDACC__
#define UST_HD __host__ __device__
#else
#define UST_HD
#endif

// bits of w that the kernel derives (never taken from the caller's flags word)
#define UST_W_SKIP (1u << 2)
#define UST_W_UNSCHEDULABLE (1u << 3)
#define UST_W_GRANTED (1u << 4)     /* upgrade slot available for this candidate (upgrade_inplace.go:87-99) */
#define UST_W_SYNCED (1u << 9)      /* pod revision hash == DaemonSet revision hash (common_manager.go:318) */
#define UST_W_PD_HAS (1u << 22)     /* numPodsToDelete != 0                    pod_manager.go:184 */
#define UST_W_PD_MISMATCH (1u << 23) /* numPodsCanDelete != numPodsToDelete    pod_manager.go:194 */
#define UST_W_DRAIN_ERROR (1u << 24) /* drain helper reports an error pod      drain_manager.go:121-128 */

// The window of w each state's transition reads: first bit (always >= 2: the kernel shifts by sh-2 so the table index
// comes out pre-multiplied by 4) and width. Only these bits can change what ust_transition() returns for the state -
// tests/test_abi_cpu.py::test_transition_table_matches_oracle checks that against the oracle for every 9-bit key.
UST_HD constexpr int ust_shift_of(int s) {
  switch (s) {
    case 0: case 11: return 3;   // unknown / upgrade-done: UNSCHED, UPG_REQ, SAFE_LOAD, ORPHANED, SYNCED
    case 1: return 2;            // upgrade-required: SKIP, UNSCHED, GRANTED, UPG_REQ
    case 3: return 16;           // wait-for-jobs: WAIT_*
    case 4: return 22;           // pod-deletion: PD_HAS, PD_MISMATCH
    case 5: return 24;           // drain-required: DRAIN_ERROR
    case 6: return 20;           // node-maintenance: NM_PRESENT, NM_READY
    case 8: return 7;            // pod-restart: SAFE_LOAD, ORPHANED, SYNCED, POD_READY, INITIAL, REQUESTOR, TERMINATING, FAILING
    case 9: return 6;            // validation: VALIDATION_DONE, SAFE_LOAD, INITIAL, REQUESTOR
    case 10: return 13;          // uncordon: REQUESTOR
    case 12: return 8;           // upgrade-failed: ORPHANED, SYNCED, POD_READY, INITIAL
    default: return 2;           // cordon-required, post-maintenance, other, excluded, reserved: read nothing
  }
}
UST_HD constexpr int ust_bits_of(int s) {
  switch (s) {
    case 0: case 11: return 7;   // bits 3..9
    case 1: return 4;            // bits 2..5
    case 3: return 4;            // bits 16..19
    case 4: return 2;            // bits 22..23
    case 5: return 1;            // bit 24
    case 6: return 2;            // bits 20..21
    case 8: return 9;            // bits 7..15
    case 9: return 8;            // bits 6..13
    case 10: return 1;           // bit 13
    case 12: return 5;           // bits 8..12
    default: return 0;
  }
}
#define UST_LUT_WINDOW_BITS 9    /* the widest window */
#define UST_LUT_WINDOW (1u << UST_LUT_WINDOW_BITS)
// Compact layout: the windows are packed widest first, so every window starts at a multiple of its own size and the
// kernel can OR the index into the base. 1105 entries instead of 16 x 512.
UST_HD constexpr int ust_base_of(int s) {
  int b = 0;
  for (int q = 0; q < 16; q++)
    if (ust_bits_of(q) > ust_bits_of(s) || (ust_bits_of(q) == ust_bits_of(s) && q < s)) b += 1 << ust_bits_of(q);
  return b;
}
UST_HD constexpr int ust_lut_used() {
  int b = 0;
  for (int q = 0; q < 16; q++) b += 1 << ust_bits_of(q);
  return b;
}
#define UST_LUT_ENTRIES ((unsigned)((ust_lut_used() + 3) & ~3))   /* 1108 words; + 16 {x, y} meta pairs behind it */
#define UST_LUT_WORDS (UST_LUT_ENTRIES + 32u)
// per-state lookup constants: byte offset of a node's entry = (funnelshift_r(w, 0, x) & (x >> 16)) | y
UST_HD constexpr uint32_t ust_meta_x(int s) { return (uint32_t)(ust_shift_of(s) - 2) | ((((1u << ust_bits_of(s)) - 1u) << 2) << 16); }
UST_HD constexpr uint32_t ust_meta_y(int s) { return (uint32_t)ust_base_of(s) * 4u; }

// Validation mode (UST_EVAL_ACTUATORS | UST_EVAL_VALIDATION): the pod-summary kernel answers Validate for a
// validation-required node and writes everything that node's transition reads into its summary byte, bits 1-3 and 5-7
// (UST_VALSUM_*), which pods_apply() puts at w bits 22-24 and 26-28. State 9 then reads the 7-bit window 22..28 of its
// table slot instead of bits 6..13; no other state's window moves.
#define UST_VAL_SHIFT 22
#define UST_VAL_BITS 7
static inline bool ust_validation_mode(const ust_policy* p) {
  return p && (p->evaluate_actuators & (UST_EVAL_ACTUATORS | UST_EVAL_VALIDATION)) == (UST_EVAL_ACTUATORS | UST_EVAL_VALIDATION);
}
static inline int ust_policy_shift_of(const ust_policy* p, int s) {
  return (s == UST_STATE_VALIDATION_REQUIRED && ust_validation_mode(p)) ? UST_VAL_SHIFT : ust_shift_of(s);
}
static inline int ust_policy_bits_of(const ust_policy* p, int s) {
  return (s == UST_STATE_VALIDATION_REQUIRED && ust_validation_mode(p)) ? UST_VAL_BITS : ust_bits_of(s);
}
static inline uint32_t ust_policy_meta_x(const ust_policy* p, int s) {
  return (uint32_t)(ust_policy_shift_of(p, s) - 2) | ((((1u << ust_policy_bits_of(p, s)) - 1u) << 2) << 16);
}

static constexpr int ust_window_shift[16] = {ust_shift_of(0), ust_shift_of(1), ust_shift_of(2), ust_shift_of(3), ust_shift_of(4), ust_shift_of(5),
                                             ust_shift_of(6), ust_shift_of(7), ust_shift_of(8), ust_shift_of(9), ust_shift_of(10), ust_shift_of(11),
                                             ust_shift_of(12), ust_shift_of(13), ust_shift_of(14), ust_shift_of(15)};

// position of each state's Process* pass in ApplyState's call order (upgrade_state.go:205-274);
// -1 = the state is never processed
static const int ust_pass_of_state[16] = {0, 2, 3, 4, 5, 6, 7, -1, 8, 10, 11, 1, 9, -1, -1, -1};

static inline uint32_t ust_lut_pack(unsigned state, unsigned next, unsigned actions, unsigned outcome) {
  if (next != state) actions |= UST_A_SET_STATE;
  return (actions & 0xFFFFu) | ((next & 0xFFu) << 16) | ((outcome & 0xFFu) << 24);
}

// updateNodeToUncordonOrDoneState (common_manager.go:673-708)
static inline void ust_uncordon_or_done(uint32_t w, unsigned* next, unsigned* actions) {
  bool requestor = (w & UST_F_REQUESTOR_MODE) != 0;
  *next = UST_STATE_UNCORDON_REQUIRED;
  if ((w & UST_F_INITIAL_STATE_ANNO) && !requestor) *next = UST_STATE_DONE;
  if (*next == UST_STATE_DONE || requestor) *actions |= UST_A_CLEAR_INITIAL_STATE_ANNO;
}

// Go's `now > start + timeout` on int64 (pod_manager.go:354, validation_manager.go:161): the sum wraps in two's complement,
// so a start near INT64_MAX counts as timed out. Computed in uint64: signed overflow is undefined in C++.
UST_HD inline bool ust_timed_out(int64_t now, int64_t start, int64_t timeout) {
  return now > (int64_t)((uint64_t)start + (uint64_t)timeout);
}

// Pod-list summary byte of a validation-required node in validation mode (ust_pod_summary_kernel): bits 1-3 the outcome
// of Validate (validation_manager.go:71-175) for the node's validation pods in list order and its start-time annotation,
// bits 5-7 the flag bits ProcessValidationRequiredNodes reads (common_manager.go:573-604). Bits 0 and 4 stay clear.
#define UST_VALSUM_OUTCOME_SHIFT 1
#define UST_VALSUM_SAFE_LOAD 0x20u
#define UST_VALSUM_INITIAL_STATE_ANNO 0x40u
#define UST_VALSUM_REQUESTOR_MODE 0x80u
enum {
  UST_VAL_WAIT = 0,         // not done, no annotation call: no matching pod, or the first one is not ready and the
                            // annotation is present, valid and not timed out
  UST_VAL_SET_START = 1,    // the first matching pod is not ready and there is no annotation: set it to now (:140-150)
  UST_VAL_RESTART = 2,      // a ready pod before the first not-ready one: delete (:106-113), then set (:140-150)
  UST_VAL_DONE = 3,         // every matching pod ready: done, annotation deleted
  UST_VAL_TIMED_OUT = 4,    // now > start + 600: upgrade-failed, annotation deleted (:161-169)
  UST_VAL_ERROR = 5         // the annotation does not parse: Validate returns an error (:155-160), ApplyState aborts
};
// the byte from the walk's findings and the node's flags word (device and host)
UST_HD inline uint32_t ust_validation_byte(bool any_not_ready, bool ready_before, bool walked, uint32_t fl) {
  unsigned o = UST_VAL_WAIT;
  if (walked) {
    if (!any_not_ready) o = ready_before ? UST_VAL_DONE : UST_VAL_WAIT;
    else if (ready_before) o = UST_VAL_RESTART;
    else if (!(fl & UST_F_VALIDATION_START_ANNO)) o = UST_VAL_SET_START;
    else if (fl & UST_F_VALIDATION_START_INVALID) o = UST_VAL_ERROR;
    else if (fl & UST_F_VALIDATION_TIMED_OUT) o = UST_VAL_TIMED_OUT;
  }
  return (o << UST_VALSUM_OUTCOME_SHIFT) | ((fl & UST_F_SAFE_LOAD) ? UST_VALSUM_SAFE_LOAD : 0u) |
         ((fl & UST_F_INITIAL_STATE_ANNO) ? UST_VALSUM_INITIAL_STATE_ANNO : 0u) | ((fl & UST_F_REQUESTOR_MODE) ? UST_VALSUM_REQUESTOR_MODE : 0u);
}

// validation-required in validation mode: the summary byte sits at w bits 21.. (bits 0 and 4 of it are never set)
static inline void ust_validation_transition(uint32_t w, const ust_policy* p, unsigned* next, unsigned* a) {
  const uint32_t b = (w >> (UST_VAL_SHIFT - 1)) & 0xEEu;
  if (b & UST_VALSUM_SAFE_LOAD) *a |= UST_A_UNBLOCK_SAFE_LOAD;  // UnblockLoading runs before Validate
  const uint32_t wf = ((b & UST_VALSUM_INITIAL_STATE_ANNO) ? UST_F_INITIAL_STATE_ANNO : 0u) |
                      ((b & UST_VALSUM_REQUESTOR_MODE) ? UST_F_REQUESTOR_MODE : 0u);
  if (!p->validation_enabled) {  // empty podSelector: Validate is true without any list (validation_manager.go:72-74)
    ust_uncordon_or_done(wf, next, a);
    return;
  }
  switch ((b >> UST_VALSUM_OUTCOME_SHIFT) & 7u) {
    case UST_VAL_SET_START: *a |= UST_A_SET_WAIT_START; break;
    case UST_VAL_RESTART: *a |= UST_A_CLEAR_WAIT_START | UST_A_SET_WAIT_START; break;
    case UST_VAL_DONE: *a |= UST_A_CLEAR_WAIT_START; ust_uncordon_or_done(wf, next, a); break;
    case UST_VAL_TIMED_OUT: *a |= UST_A_CLEAR_WAIT_START; *next = UST_STATE_FAILED; break;
    default: break;  // UST_VAL_WAIT; UST_VAL_ERROR: the abort (published by the pod-summary kernel) decides the node
  }
}

// One node's transition as a function of its state code, predicate word and the policy.
static inline uint32_t ust_transition(unsigned s, uint32_t w, const ust_policy* p) {
  unsigned next = s, a = 0, outcome = UST_OUTCOME_NONE;
  const bool orphan = (w & UST_F_POD_ORPHANED) != 0;
  const bool synced = !orphan && (w & UST_W_SYNCED);
  switch (s) {
    case UST_STATE_UNKNOWN:
    case UST_STATE_DONE:  // ProcessDoneOrUnknownNodes  common_manager.go:229-291
      if ((!synced && !orphan) || (w & UST_F_SAFE_LOAD) || (w & UST_F_UPGRADE_REQUESTED)) {
        if (w & UST_W_UNSCHEDULABLE) a |= UST_A_SET_INITIAL_STATE_ANNO;
        next = UST_STATE_UPGRADE_REQUIRED;
      } else if (s == UST_STATE_UNKNOWN) {
        next = UST_STATE_DONE;
      }
      break;
    case UST_STATE_UPGRADE_REQUIRED:
      if (w & UST_F_UPGRADE_REQUESTED) a |= UST_A_CLEAR_UPGRADE_REQUESTED;
      if (w & UST_W_SKIP) break;
      if (p->use_maintenance_operator) {  // upgrade_requestor.go:277-319
        a |= UST_A_NM_CREATE_OR_DELETE | UST_A_REQUESTOR_ANNO_CHANGE;
        next = UST_STATE_NODE_MAINTENANCE_REQUIRED;
      } else if ((w & UST_W_GRANTED) || (w & UST_W_UNSCHEDULABLE)) {  // upgrade_inplace.go:87-101
        next = UST_STATE_CORDON_REQUIRED;
      }
      break;
    case UST_STATE_CORDON_REQUIRED:  // common_manager.go:361-380
      a |= UST_A_CORDON;
      next = UST_STATE_WAIT_FOR_JOBS_REQUIRED;
      break;
    case UST_STATE_WAIT_FOR_JOBS_REQUIRED:  // common_manager.go:384-419
      if (!p->wait_selector_set) {
        next = p->pod_deletion_enabled ? UST_STATE_POD_DELETION_REQUIRED : UST_STATE_DRAIN_REQUIRED;
      } else {
        a |= UST_A_SCHEDULE_WAIT_CHECK;
        if (p->evaluate_actuators) {  // pod_manager.go:256-317, :331-368
          outcome = UST_STATE_WAIT_FOR_JOBS_REQUIRED;
          if (w & UST_F_WAIT_PODS_RUNNING) {
            if (p->wait_timeout_nonzero) {
              if (!(w & UST_F_WAIT_START_ANNO)) a |= UST_A_SET_WAIT_START;
              else if (w & UST_F_WAIT_START_INVALID) {}
              else if (w & UST_F_WAIT_TIMED_OUT) { outcome = UST_STATE_POD_DELETION_REQUIRED; a |= UST_A_CLEAR_WAIT_START; }
            }
          } else {
            a |= UST_A_CLEAR_WAIT_START;
            outcome = UST_STATE_POD_DELETION_REQUIRED;
          }
        }
      }
      break;
    case UST_STATE_POD_DELETION_REQUIRED:  // common_manager.go:424-453
      if (!p->pod_deletion_enabled) {
        next = UST_STATE_DRAIN_REQUIRED;
      } else {
        a |= UST_A_SCHEDULE_POD_EVICTION;
        if (p->evaluate_actuators) {  // pod_manager.go:176-220, :393-403
          if (!(w & UST_W_PD_HAS)) outcome = UST_STATE_POD_RESTART_REQUIRED;
          else if (w & UST_W_PD_MISMATCH) outcome = p->drain_enabled ? UST_STATE_DRAIN_REQUIRED : UST_STATE_FAILED;
          else outcome = UST_STATE_POD_RESTART_REQUIRED;
        }
      }
      break;
    case UST_STATE_DRAIN_REQUIRED:  // common_manager.go:329-357
      if (!p->drain_enabled) {
        next = UST_STATE_POD_RESTART_REQUIRED;
      } else {
        a |= UST_A_SCHEDULE_DRAIN;
        if (p->evaluate_actuators)  // drain_manager.go:106-131
          outcome = (w & UST_W_DRAIN_ERROR) ? UST_STATE_FAILED : UST_STATE_POD_RESTART_REQUIRED;
      }
      break;
    case UST_STATE_NODE_MAINTENANCE_REQUIRED:  // upgrade_requestor.go:416-452; in-place mode never touches it
      if (p->use_maintenance_operator) {
        if (!(w & UST_F_NM_PRESENT)) next = UST_STATE_UPGRADE_REQUIRED;
        else if (w & UST_F_NM_READY) next = UST_STATE_POD_RESTART_REQUIRED;
      }
      break;
    case UST_STATE_POD_RESTART_REQUIRED:  // common_manager.go:457-524
      if (!synced || orphan) {
        if (!(w & UST_F_POD_TERMINATING)) a |= UST_A_RESTART_DRIVER_POD;
      } else {
        if (w & UST_F_SAFE_LOAD) a |= UST_A_UNBLOCK_SAFE_LOAD;
        if (w & UST_F_POD_READY) {
          if (!p->validation_enabled) ust_uncordon_or_done(w, &next, &a);
          else next = UST_STATE_VALIDATION_REQUIRED;
        } else if (w & UST_F_POD_FAILING) {
          next = UST_STATE_FAILED;
        }
      }
      break;
    case UST_STATE_FAILED:  // common_manager.go:528-570 (no requestor-mode check here)
      if (synced && (w & UST_F_POD_READY)) {
        if (w & UST_F_INITIAL_STATE_ANNO) { next = UST_STATE_DONE; a |= UST_A_CLEAR_INITIAL_STATE_ANNO; }
        else next = UST_STATE_UNCORDON_REQUIRED;
      }
      break;
    case UST_STATE_VALIDATION_REQUIRED:  // common_manager.go:573-604
      if (ust_validation_mode(p)) { ust_validation_transition(w, p, &next, &a); break; }
      if (w & UST_F_SAFE_LOAD) a |= UST_A_UNBLOCK_SAFE_LOAD;
      if (w & UST_F_VALIDATION_DONE) ust_uncordon_or_done(w, &next, &a);
      break;
    case UST_STATE_UNCORDON_REQUIRED:  // upgrade_inplace.go:124-147, upgrade_requestor.go:454-488
      if (!(w & UST_F_REQUESTOR_MODE)) { a |= UST_A_UNCORDON; next = UST_STATE_DONE; }
      else if (p->use_maintenance_operator) { next = UST_STATE_DONE; a |= UST_A_REQUESTOR_ANNO_CHANGE | UST_A_NM_CREATE_OR_DELETE; }
      break;
    default: break;  // post-maintenance-required, other, excluded: never processed
  }
  return ust_lut_pack(s, next, a, outcome);
}

// lut[ust_base_of(s) + key] for key = (w >> ust_shift_of(s)) & (2^ust_bits_of(s) - 1); then the 16 {x, y} meta pairs.
// `p` == NULL: the table of an inactive policy (every node is a no-op).
static inline void ust_build_lut(const ust_policy* p, uint32_t* lut) {
  for (unsigned i = 0; i < UST_LUT_WORDS; i++) lut[i] = 0;
  for (int s = 0; s < 16; s++) {
    // a policy's window fits its state's slot: validation mode gives state 9 7 of the 8 bits it has
    const int sh = ust_policy_shift_of(p, s), base = ust_base_of(s);
    for (uint32_t key = 0; key < (1u << ust_policy_bits_of(p, s)); key++) {
      const uint32_t w = (uint32_t)(((uint64_t)key << sh) & 0xFFFFFFFFull);
      lut[base + (int)key] = p ? ust_transition((unsigned)s, w, p) : ust_lut_pack((unsigned)s, (unsigned)s, 0, 0xFF);
    }
    lut[UST_LUT_ENTRIES + 2 * s] = ust_policy_meta_x(p, s);
    lut[UST_LUT_ENTRIES + 2 * s + 1] = ust_meta_y(s);
  }
}
// the lookup the kernels make, on the host (audit / tests)
static inline uint32_t ust_lut_lookup(const uint32_t* lut, unsigned s, uint32_t w) {
  const uint32_t x = lut[UST_LUT_ENTRIES + 2 * s], y = lut[UST_LUT_ENTRIES + 2 * s + 1];
  const uint32_t sh = x & 31u;
  const uint32_t fs = (uint32_t)(((uint64_t)w << 32) >> (32 + sh));  // __funnelshift_r(w, 0, sh)
  return lut[((fs & (x >> 16)) | y) >> 2];
}

// Pod-list table: for one workload pod, which actuator conditions it raises (index = pod_flags & 0x7FF).
// kubectl drain filter chain, k8s.io/kubectl v0.35.1 pkg/drain/filters.go (see oracle for the restatement).
#define UST_PODLUT_ENTRIES 2048u
#define UST_PODSUM_WAIT_RUNNING 0x01u
#define UST_PODSUM_TO_DELETE 0x02u    /* matches the deletion filter */
#define UST_PODSUM_CANNOT_DELETE 0x04u /* ... but the base filter chain keeps it */
#define UST_PODSUM_DRAIN_ERROR 0x08u

// Which filter of the chain stopped a pod (ust_pod_chain_keeps's `stop`): none, or the filter and whether it is an error.
#define UST_CHAIN_NONE 0u
#define UST_CHAIN_DAEMONSET 1u      /* daemonSetFilter: skipped with a warning (IgnoreAllDaemonSets) */
#define UST_CHAIN_DS_MISSING 2u     /* daemonSetFilter: an error, its DaemonSet is NotFound and there is no force */
#define UST_CHAIN_MIRROR 3u         /* mirrorPodFilter: skipped */
#define UST_CHAIN_LOCAL_STORAGE 4u  /* localStorageFilter: an error */
#define UST_CHAIN_UNREPLICATED 5u   /* unreplicatedFilter: an error */

static inline bool ust_pod_chain_keeps(unsigned pf, bool force, bool delete_emptydir, bool* is_error, unsigned* stop = nullptr) {
  const unsigned phase = pf & UST_POD_PHASE_MASK;
  const bool finished = phase == UST_PHASE_SUCCEEDED || phase == UST_PHASE_FAILED;
  unsigned s = UST_CHAIN_NONE;
  if ((pf & UST_POD_HAS_CONTROLLER) && (pf & UST_POD_CONTROLLED_BY_DS) && !finished) {
    if (pf & UST_POD_DS_MISSING) { if (!force) s = UST_CHAIN_DS_MISSING; }
    else s = UST_CHAIN_DAEMONSET;
  }
  if (s == UST_CHAIN_NONE) {
    if (pf & UST_POD_MIRROR) s = UST_CHAIN_MIRROR;
    else if ((pf & UST_POD_HAS_EMPTYDIR) && !finished && !delete_emptydir) s = UST_CHAIN_LOCAL_STORAGE;
    else if (!finished && !(pf & UST_POD_HAS_CONTROLLER) && !force) s = UST_CHAIN_UNREPLICATED;
  }
  *is_error = s == UST_CHAIN_DS_MISSING || s == UST_CHAIN_LOCAL_STORAGE || s == UST_CHAIN_UNREPLICATED;
  if (stop) *stop = s;
  return s != UST_CHAIN_NONE;
}

static inline void ust_build_pod_lut(const ust_policy* p, uint8_t* podlut) {
  for (unsigned pf = 0; pf < UST_PODLUT_ENTRIES; pf++) {
    unsigned r = 0;
    const unsigned phase = pf & UST_POD_PHASE_MASK;
    if ((pf & UST_POD_MATCH_WAIT_SELECTOR) && (phase == UST_PHASE_RUNNING || phase == UST_PHASE_PENDING)) r |= UST_PODSUM_WAIT_RUNNING;
    bool err;
    if (pf & UST_POD_MATCH_DELETION_FILTER) {
      r |= UST_PODSUM_TO_DELETE;
      if (ust_pod_chain_keeps(pf, p->pod_deletion_force != 0, p->pod_deletion_delete_emptydir != 0, &err)) r |= UST_PODSUM_CANNOT_DELETE;
    }
    if (pf & UST_POD_MATCH_DRAIN_SELECTOR) {
      ust_pod_chain_keeps(pf, p->drain_force != 0, p->drain_delete_emptydir != 0, &err);
      if (err) r |= UST_PODSUM_DRAIN_ERROR;
    }
    podlut[pf] = (uint8_t)r;
  }
}

// The form the pod-summary kernel uses. The three selector-match bits (8-10) only gate output bits - wait-running needs
// bit 9, to-delete / cannot-delete bit 8, drain-error bit 10 - and everything else is a function of the pod's own eight
// bits (phase + 5 flags):   podlut[pf] == T[pf & 255] & ust_pod_gate(pf).
// A node's actuator reads only the output bits of ITS selector (pod_manager.go:263 / :139,179 / drain_manager.go:86), so
// the kernel skips pods that lack that bit and ORs T[pf & 255] of the others: no gate arithmetic, half the lookups,
// and a 256-byte table (two words per shared-memory bank) instead of 2 KiB (sixteen).
static inline unsigned ust_pod_gate(unsigned pf) { return ((pf >> 9) & 1u) | ((pf >> 7) & 0xAu) | ((pf >> 6) & 4u); }
static inline void ust_build_pod_lut256(const ust_policy* p, uint8_t* T) {
  uint8_t full[UST_PODLUT_ENTRIES];
  ust_build_pod_lut(p, full);
  for (unsigned low = 0; low < 256; low++) T[low] = (uint8_t)(full[low | 0x700u] & 15u);
}
