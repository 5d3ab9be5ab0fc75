// upgrade.cpp — see upgrade.hpp. Encode -> ust_apply_state (H100) -> Replay.
#include "upgrade.hpp"

#include <algorithm>
#include <climits>
#include <thread>
#include <unordered_map>
#include <unordered_set>
#include <cstring>

#include "../csrc/ust_lut.h"  // ust_pod_chain_keeps: the pods a drain evicts

namespace upgrade {

const char* const UpgradeStateUnknown = "";
const char* const UpgradeStateUpgradeRequired = "upgrade-required";
const char* const UpgradeStateCordonRequired = "cordon-required";
const char* const UpgradeStateWaitForJobsRequired = "wait-for-jobs-required";
const char* const UpgradeStatePodDeletionRequired = "pod-deletion-required";
const char* const UpgradeStateDrainRequired = "drain-required";
const char* const UpgradeStateNodeMaintenanceRequired = "node-maintenance-required";
const char* const UpgradeStatePostMaintenanceRequired = "post-maintenance-required";
const char* const UpgradeStatePodRestartRequired = "pod-restart-required";
const char* const UpgradeStateValidationRequired = "validation-required";
const char* const UpgradeStateUncordonRequired = "uncordon-required";
const char* const UpgradeStateDone = "upgrade-done";
const char* const UpgradeStateFailed = "upgrade-failed";
const char* const PodControllerRevisionHashLabelKey = "controller-revision-hash";

static const char* const kNullString = "null";  // consts.go:90
static const char* const kTrueString = "true";  // consts.go:92
static const char* const kDrainInsteadMessage = "Pod deletion failed but drain is enabled in spec. Will attempt a node drain";  // pod_manager.go:396-399
static std::string g_driver_name;                 // util.go:91-99

// The eight keys are functions of the driver name only (util.go:101-133). The reference formats them on every use; an
// encoder that walks a million nodes cannot (six formatted strings per node were a third of Encode's time), so they are
// built once per SetDriverName.
struct DriverKeys {
  bool valid = false;
  std::string state, skip, safeLoad, requested, requestorMode, initialState, waitStart, validationStart;
};
static DriverKeys g_keys;
static std::string key(const char* tail) { return "nvidia.com/" + g_driver_name + tail; }
static const DriverKeys& keys() {
  if (!g_keys.valid) {
    g_keys.state = key("-driver-upgrade-state");
    g_keys.skip = key("-driver-upgrade.skip");
    g_keys.safeLoad = key("-driver-upgrade.driver-wait-for-safe-load");
    g_keys.requested = key("-driver-upgrade-requested");
    g_keys.requestorMode = key("-driver-upgrade-requestor-mode");
    g_keys.initialState = key("-driver-upgrade.node-initial-state.unschedulable");
    g_keys.waitStart = key("-driver-upgrade-wait-for-pod-completion-start-time");
    g_keys.validationStart = key("-driver-upgrade-validation-start-time");
    g_keys.valid = true;
  }
  return g_keys;
}
void SetDriverName(const std::string& driver) { g_driver_name = driver; g_keys.valid = false; }
std::string GetUpgradeStateLabelKey() { return keys().state; }
std::string GetUpgradeSkipNodeLabelKey() { return keys().skip; }
std::string GetUpgradeDriverWaitForSafeLoadAnnotationKey() { return keys().safeLoad; }
std::string GetUpgradeRequestedAnnotationKey() { return keys().requested; }
std::string GetUpgradeRequestorModeAnnotationKey() { return keys().requestorMode; }
std::string GetUpgradeInitialStateAnnotationKey() { return keys().initialState; }
std::string GetWaitForPodCompletionStartTimeAnnotationKey() { return keys().waitStart; }
std::string GetValidationStartTimeAnnotationKey() { return keys().validationStart; }
std::string GetEventReason() {
  std::string s = g_driver_name;
  for (char& c : s)
    if (c >= 'a' && c <= 'z') c = (char)(c - 'a' + 'A');
  return s + "DriverUpgrade";
}

const char* const EventTypeNormal = "Normal";
const char* const EventTypeWarning = "Warning";

bool IsOrphanedPod(const Pod& pod) { return pod.OwnerReferences.empty(); }
bool IsNodeInRequestorMode(const Node& node) { return node.Annotations.count(keys().requestorMode) != 0; }
ClusterUpgradeState NewClusterUpgradeState() { return ClusterUpgradeState(); }

static const char* const kStateNames[13] = {
    UpgradeStateUnknown, UpgradeStateUpgradeRequired, UpgradeStateCordonRequired, UpgradeStateWaitForJobsRequired,
    UpgradeStatePodDeletionRequired, UpgradeStateDrainRequired, UpgradeStateNodeMaintenanceRequired,
    UpgradeStatePostMaintenanceRequired, UpgradeStatePodRestartRequired, UpgradeStateValidationRequired,
    UpgradeStateUncordonRequired, UpgradeStateDone, UpgradeStateFailed};
const char* StateNameOfCode(unsigned code) { return code < 13 ? kStateNames[code] : nullptr; }
int StateCodeOfLabel(const std::string& label) {
  for (int i = 0; i < 13; i++)
    if (label == kStateNames[i]) return i;
  return UST_STATE_OTHER;
}

// buckets in the order ApplyState walks them (upgrade_state.go:205-274)
static const int kPassOrder[12] = {UST_STATE_UNKNOWN, UST_STATE_DONE, UST_STATE_UPGRADE_REQUIRED, UST_STATE_CORDON_REQUIRED,
                                   UST_STATE_WAIT_FOR_JOBS_REQUIRED, UST_STATE_POD_DELETION_REQUIRED, UST_STATE_DRAIN_REQUIRED,
                                   UST_STATE_NODE_MAINTENANCE_REQUIRED, UST_STATE_POD_RESTART_REQUIRED, UST_STATE_FAILED,
                                   UST_STATE_VALIDATION_REQUIRED, UST_STATE_UNCORDON_REQUIRED};

static size_t len(const ClusterUpgradeState& s, const char* name) {
  auto it = s.NodeStates.find(name);
  return it == s.NodeStates.end() ? 0 : it->second.size();
}

// ---- construction -------------------------------------------------------------------------------------------
Error ClusterUpgradeStateManagerImpl::New(int device, StateOptions opts, std::unique_ptr<ClusterUpgradeStateManagerImpl>* out) {
  std::unique_ptr<ClusterUpgradeStateManagerImpl> m(new ClusterUpgradeStateManagerImpl());
  m->opts_ = opts;
  if (ust_create(&m->handle_, device) != UST_OK)
    return Errorf(std::string("failed to create upgrade state manager: ") + ust_create_error());
  *out = std::move(m);
  return std::nullopt;
}
std::unique_ptr<ClusterUpgradeStateManagerImpl> ClusterUpgradeStateManagerImpl::NewDetached(StateOptions opts) {
  std::unique_ptr<ClusterUpgradeStateManagerImpl> m(new ClusterUpgradeStateManagerImpl());
  m->opts_ = opts;
  return m;
}
ClusterUpgradeStateManagerImpl::~ClusterUpgradeStateManagerImpl() {
  {
    std::unique_lock<std::mutex> l(actMu_);
    actCv_.wait(l, [&] { return actQueue_.empty() && actRunning_ == 0; });
    actStop_ = true;
  }
  actCv_.notify_all();
  for (auto& t : actThreads_) t.join();
  if (handle_) ust_destroy(handle_);
}

// ---- the PodEvictor's workers (StateOptions::EvictionOnDevice) ---------------------------------------------------
void ClusterUpgradeStateManagerImpl::handOff(std::set<std::string>* dedupe, const std::string& name, std::function<void()> job) {
  std::lock_guard<std::mutex> l(actMu_);
  dedupe->insert(name);
  actQueue_.push_back([this, dedupe, name, job = std::move(job)] {
    job();
    std::lock_guard<std::mutex> g(actMu_);
    dedupe->erase(name);  // defer m.nodesInProgress.Remove / m.drainingNodes.Remove (pod_manager.go:165, drain_manager.go:110)
  });
  if (actIdle_ < actQueue_.size() && actThreads_.size() < kActuatorWorkers) {
    actThreads_.emplace_back([this] {
      std::unique_lock<std::mutex> l(actMu_);
      for (;;) {
        actIdle_++;
        actCv_.wait(l, [&] { return actStop_ || !actQueue_.empty(); });
        actIdle_--;
        if (actQueue_.empty()) return;  // stopping
        std::function<void()> f = std::move(actQueue_.front());
        actQueue_.pop_front();
        actRunning_++;
        l.unlock();
        f();
        l.lock();
        actRunning_--;
        actCv_.notify_all();
      }
    });
  }
  actCv_.notify_all();
}
void ClusterUpgradeStateManagerImpl::WaitForActuators() {
  std::unique_lock<std::mutex> l(actMu_);
  actCv_.wait(l, [&] { return actQueue_.empty() && actRunning_ == 0; });
}

ClusterUpgradeStateManager& ClusterUpgradeStateManagerImpl::WithPodDeletionEnabled(PodDeletionFilter filter) {
  if (!filter) return *this;  // "Cannot enable PodDeletion state as PodDeletionFilter is nil"  upgrade_state.go:330-333
  filter_ = std::move(filter);
  podDeletionStateEnabled_ = true;
  return *this;
}
ClusterUpgradeStateManager& ClusterUpgradeStateManagerImpl::WithValidationEnabled(const std::string& podSelector) {
  if (podSelector.empty()) return *this;  // upgrade_state.go:342-345
  validationSelector_ = podSelector;
  validationStateEnabled_ = true;
  return *this;
}

// ---- predicates ---------------------------------------------------------------------------------------------
bool ClusterUpgradeStateManagerImpl::IsUpgradeRequested(const Node& n) const {
  auto it = n.Annotations.find(keys().requested);
  return it != n.Annotations.end() && it->second == kTrueString;
}
bool ClusterUpgradeStateManagerImpl::IsNodeUnschedulable(const Node& n) const { return n.Unschedulable; }
bool ClusterUpgradeStateManagerImpl::isNodeConditionReady(const Node& n) const {
  for (const auto& c : n.Conditions)
    if (c.Type == "Ready" && c.Status != "True") return false;
  return true;
}
bool ClusterUpgradeStateManagerImpl::SkipNodeUpgrade(const Node& n) const {
  auto it = n.Labels.find(keys().skip);
  return it != n.Labels.end() && it->second == kTrueString;
}
bool ClusterUpgradeStateManagerImpl::isDriverPodFailing(const Pod& p) const {
  for (const auto& st : p.InitContainerStatuses)
    if (!st.Ready && st.RestartCount > 10) return true;
  for (const auto& st : p.ContainerStatuses)
    if (!st.Ready && st.RestartCount > 10) return true;
  return false;
}

// ---- counters (common_manager.go:146-165, :715-788) ---------------------------------------------------------
int ClusterUpgradeStateManagerImpl::GetTotalManagedNodes(const ClusterUpgradeState& s) const {
  return (int)(len(s, UpgradeStateUnknown) + len(s, UpgradeStateDone) + len(s, UpgradeStateUpgradeRequired) +
               len(s, UpgradeStateCordonRequired) + len(s, UpgradeStateWaitForJobsRequired) +
               len(s, UpgradeStatePodDeletionRequired) + len(s, UpgradeStateFailed) + len(s, UpgradeStateDrainRequired) +
               len(s, UpgradeStatePodRestartRequired) + len(s, UpgradeStateUncordonRequired) +
               len(s, UpgradeStateValidationRequired));
}
int ClusterUpgradeStateManagerImpl::GetUpgradesInProgress(const ClusterUpgradeState& s) const {
  return GetTotalManagedNodes(s) - (int)(len(s, UpgradeStateUnknown) + len(s, UpgradeStateDone) + len(s, UpgradeStateUpgradeRequired));
}
int ClusterUpgradeStateManagerImpl::GetUpgradesDone(const ClusterUpgradeState& s) const { return (int)len(s, UpgradeStateDone); }
int ClusterUpgradeStateManagerImpl::GetUpgradesFailed(const ClusterUpgradeState& s) const { return (int)len(s, UpgradeStateFailed); }
int ClusterUpgradeStateManagerImpl::GetUpgradesPending(const ClusterUpgradeState& s) const { return (int)len(s, UpgradeStateUpgradeRequired); }
int ClusterUpgradeStateManagerImpl::GetCurrentUnavailableNodes(const ClusterUpgradeState& s) const {
  int unavailable = 0;
  for (const auto& kv : s.NodeStates)
    for (const NodeUpgradeState* ns : kv.second) {
      if (IsNodeUnschedulable(*ns->Node)) { unavailable++; continue; }
      if (!isNodeConditionReady(*ns->Node)) unavailable++;
    }
  return unavailable;
}
int ClusterUpgradeStateManagerImpl::GetUpgradesAvailable(const ClusterUpgradeState& s, int maxParallelUpgrades, int maxUnavailable) const {
  const int inProgress = GetUpgradesInProgress(s), total = GetTotalManagedNodes(s);
  int available = maxParallelUpgrades == 0 ? (int)len(s, UpgradeStateUpgradeRequired) : maxParallelUpgrades - inProgress;
  const int currentUnavailable = GetCurrentUnavailableNodes(s) + (int)len(s, UpgradeStateCordonRequired);
  if (available > maxUnavailable) available = maxUnavailable;
  if (currentUnavailable >= maxUnavailable) available = 0;
  else if (maxUnavailable < total && currentUnavailable + available > maxUnavailable) available = maxUnavailable - currentUnavailable;
  return available;
}

// A Kubernetes UID (UUID string) as the two uint64 the ABI joins on: 32 hex digits are taken literally, anything else
// is hashed (FNV-1a) into the same space; (0, 0) is reserved for "no owner reference". Same rule as the Go shim.
struct Uid128 { uint64_t hi, lo; };
static Uid128 uid128(const std::string& uid) {
  Uid128 u{0, 0};
  int n = 0;
  for (char ch : uid) {
    if (ch == '-') continue;
    int v = (ch >= '0' && ch <= '9') ? ch - '0' : (ch >= 'a' && ch <= 'f') ? ch - 'a' + 10 : (ch >= 'A' && ch <= 'F') ? ch - 'A' + 10 : -1;
    if (v < 0 || n >= 32) { n = -1; break; }
    if (n < 16) u.hi = (u.hi << 4) | (uint64_t)v; else u.lo = (u.lo << 4) | (uint64_t)v;
    n++;
  }
  if (n != 32) {
    u.hi = 14695981039346656037ull; u.lo = 1099511628211ull;
    for (unsigned char ch : uid) { u.hi = (u.hi ^ ch) * 1099511628211ull; u.lo = (u.lo ^ u.hi) * 14029467366897019727ull; }
  }
  if ((u.hi | u.lo) == 0) u.lo = 1;
  return u;
}

// ---- BuildState (upgrade_state.go:99-164) --------------------------------------------------------------------
// What BuildState lists (upgrade_state.go:105-119): the DaemonSets keyed by UID (common_manager.go:180-186) and, in the map's
// order, their 128-bit UIDs and DesiredNumberScheduled (padded by one entry: never pass empty vectors' data()); the pods.
struct Listed {
  std::map<std::string, DaemonSet*> daemonSets;
  std::vector<DaemonSet*> dsByIndex;
  std::vector<uint64_t> dsUid;
  std::vector<int32_t> desired;
  std::vector<Pod*> podList;
};
static Error list(K8sClient* client, const std::string& ns, const StringMap& driverLabels, Listed* l) {
  std::vector<DaemonSet*> dsList;
  if (Error e = client->ListDaemonSets(ns, driverLabels, &dsList)) return Errorf("error getting DaemonSet list: " + *e);
  for (DaemonSet* ds : dsList) l->daemonSets[ds->UID] = ds;
  if (Error e = client->ListPods(ns, driverLabels, &l->podList)) return e;
  for (const auto& kv : l->daemonSets) {
    const Uid128 u = uid128(kv.first);
    l->dsByIndex.push_back(kv.second);
    l->dsUid.push_back(u.hi); l->dsUid.push_back(u.lo);
    l->desired.push_back(kv.second->DesiredNumberScheduled);
  }
  l->dsUid.resize(l->dsUid.size() + 2); l->desired.push_back(0);
  return std::nullopt;
}

// A driver pod's state byte and the 128-bit UID of its OwnerReferences[0] ((0, 0) = none), as the owner join takes them.
static void derivePod(const Pod& pod, uint8_t* state, uint64_t* owner) {
  // upgrade_state.go:149-152: a pod not yet scheduled to a node is skipped - after the count check
  *state = (pod.NodeName.empty() && pod.Phase == "Pending") ? UST_STATE_EXCLUDED : UST_STATE_OTHER;
  owner[0] = owner[1] = 0;
  if (!IsOrphanedPod(pod)) {
    const Uid128 u = uid128(pod.OwnerReferences[0].UID);
    owner[0] = u.hi; owner[1] = u.lo;
  }
}

int ClusterUpgradeStateManagerImpl::BuildStateDevice(int64_t n, const uint8_t* state, const uint64_t* owner, int32_t n_ds,
                                                     const uint64_t* ds_uid, const int32_t* desired, int32_t* owner_idx, ust_counters* c) {
  if (handle_ == nullptr) return UST_ERR_CUDA;
  return ust_build_state_uids(handle_, n, state, owner, n_ds, ds_uid, desired, owner_idx, c);
}

static const char* const kNoDeviceBuildState = "no H100 device bound to this manager: BuildState has no CPU path";

Error ClusterUpgradeStateManagerImpl::BuildState(const std::string& ns, const StringMap& driverLabels,
                                                 std::unique_ptr<ClusterUpgradeState>* out) {
  Listed l;
  if (Error e = list(K8sClient, ns, driverLabels, &l)) return e;

  // The owner join runs on the GPU (ust_build_state_uids): every listed pod goes in with the 128-bit form of its
  // OwnerReferences[0].UID, the DaemonSets with theirs; back comes, per pod, the owning DaemonSet's index, -1 for an
  // orphaned pod, -2 for a pod owned by something else (dropped: GetPodsOwnedbyDs skips it, GetOrphanedPods does
  // not take it - common_manager.go:190-222), after the per-DaemonSet count check of upgrade_state.go:128-131.
  const size_t np = l.podList.size();
  std::vector<uint8_t> podState(np + 1);
  std::vector<uint64_t> owner(2 * np + 2, 0);
  std::vector<int32_t> owner_idx(np + 1, -2);
  for (size_t i = 0; i < np; i++) derivePod(*l.podList[i], &podState[i], &owner[2 * i]);
  ust_counters c;
  int rc = BuildStateDevice((int64_t)np, podState.data(), owner.data(), (int32_t)l.dsByIndex.size(), l.dsUid.data(), l.desired.data(),
                            owner_idx.data(), &c);
  if (rc == UST_ERR_DS_UNSCHEDULED) return Errorf("driver DaemonSet should not have Unscheduled pods");  // upgrade_state.go:128-131
  if (rc != UST_OK) return Errorf(handle_ ? ust_last_error(handle_) : kNoDeviceBuildState);
  return assembleState(l.podList, podState.data(), owner_idx.data(), l.daemonSets, out);
}

// BuildState after the owner join: the snapshot from the pods' state bytes and owner indices.
Error ClusterUpgradeStateManagerImpl::assembleState(const std::vector<Pod*>& podList, const uint8_t* podState, const int32_t* owner_idx,
                                                    std::map<std::string, DaemonSet*>& daemonSets,
                                                    std::unique_ptr<ClusterUpgradeState>* out) {
  const size_t np = podList.size();
  const size_t nds = daemonSets.size();
  // filteredPodList in the reference's order: DaemonSet by DaemonSet (map order), then the orphans (:126-136)
  std::vector<Pod*> filtered;
  std::vector<uint8_t> state;
  std::vector<std::vector<size_t>> byOwner(nds + 1);  // last bucket: orphans
  for (size_t i = 0; i < np; i++) {
    if (owner_idx[i] >= 0) byOwner[(size_t)owner_idx[i]].push_back(i);
    else if (owner_idx[i] == -1) byOwner.back().push_back(i);
  }
  for (const auto& bucket : byOwner)
    for (size_t i : bucket) { filtered.push_back(podList[i]); state.push_back(podState[i]); }

  auto st = std::make_unique<ClusterUpgradeState>();
  const std::string labelKey = GetUpgradeStateLabelKey();
  for (size_t i = 0; i < filtered.size(); i++) {
    Pod* pod = filtered[i];
    if (state[i] == UST_STATE_EXCLUDED) continue;
    Node* node = nullptr;
    if (Error e = NodeUpgradeStateProvider->GetNode(pod->NodeName, &node)) return Errorf("unable to get node " + pod->NodeName + ": " + *e);
    auto nus = std::make_unique<NodeUpgradeState>();
    nus->Node = node;
    nus->DriverPod = pod;
    nus->ListIndex = (int64_t)i;
    nus->DriverDaemonSet = IsOrphanedPod(*pod) ? nullptr : daemonSets[pod->OwnerReferences[0].UID];
    if (opts_.Requestor.UseMaintenanceOperator)
      if (Error e = K8sClient->GetNodeMaintenance(node->Name, &nus->NodeMaintenance)) return Errorf("failed while trying to fetch nodeMaintennace obj: " + *e);
    auto it = node->Labels.find(labelKey);
    st->NodeStates[it == node->Labels.end() ? "" : it->second].push_back(nus.get());
    st->owned.push_back(std::move(nus));
  }
  *out = std::move(st);
  return std::nullopt;
}

// A new order given per position as the old index it takes (-1: an entry that joins), as the maximal runs of ust_reorder /
// ust_driver_pod_reorder: consecutive old entries, joined entries.
static void orderRuns(const std::vector<int64_t>& from, std::vector<int64_t>* run_src, std::vector<int64_t>* run_len) {
  for (size_t p = 0; p < from.size(); p++) {
    const bool cont = p > 0 && ((from[p] < 0 && from[p - 1] < 0) || (from[p] >= 0 && from[p - 1] >= 0 && from[p] == from[p - 1] + 1));
    if (cont) { run_len->back()++; continue; }
    run_src->push_back(from[p] < 0 ? -1 : from[p]);
    run_len->push_back(1);
  }
}

// ---- incremental BuildState (upgrade.hpp) ------------------------------------------------------------------------------
void ClusterUpgradeStateManagerImpl::ResetBuildIncremental() { podCache_ = PodCache(); }

int ClusterUpgradeStateManagerImpl::BuildStateCached(int32_t n_ds, const uint64_t* ds_uid, const int32_t* desired, PodCache* cache,
                                                     ust_counters* c) {
  PodCache& k = *cache;
  if (handle_ == nullptr) return UST_ERR_CUDA;
  const size_t n = k.state.size(), m = k.changed.size(), ni = k.insert_at.size();
  // the joined and the overwritten pods' values (never pass NULL for empty arrays)
  std::vector<uint8_t> ist(ni + 1), cst(m + 1);
  std::vector<uint64_t> iuid(2 * ni + 2), cuid(2 * m + 2);
  for (size_t j = 0; j < ni; j++) {
    const size_t i = (size_t)k.insert_at[j];
    ist[j] = k.state[i]; iuid[2 * j] = k.owner[2 * i]; iuid[2 * j + 1] = k.owner[2 * i + 1];
  }
  std::vector<int64_t> ix(k.changed);
  ix.push_back(0);
  for (size_t j = 0; j < m; j++) {
    const size_t i = (size_t)k.changed[j];
    cst[j] = k.state[i]; cuid[2 * j] = k.owner[2 * i]; cuid[2 * j + 1] = k.owner[2 * i + 1];
  }
  const ust_driver_pod_reorder ro = {(int64_t)k.run_src.size(), k.run_src.data(), k.run_len.data(), (int64_t)ni, ist.data(), iuid.data()};
  const int64_t cap = (int64_t)(n / 4 + 1024);
  std::vector<int64_t> oi((size_t)cap + 1);
  std::vector<int32_t> od((size_t)cap + 1);
  int64_t n_out = 0;
  const int rc = ust_build_state_delta(handle_, k.reorder ? &ro : nullptr, (int64_t)m, ix.data(), cst.data(), cuid.data(), n_ds, ds_uid,
                                       desired, cap, oi.data(), od.data(), &n_out, c);
  if (rc == UST_ERR_CUDA || rc == UST_ERR_INVALID_ARGUMENT) return rc;
  if (n_out > cap) {  // nothing was written to the arrays (UST_ERR_TRUNCATED, or UST_ERR_DS_UNSCHEDULED with its own code)
    buildStats_.outputs_received += (int64_t)n;
    const int frc = ust_fetch_build_state(handle_, (int64_t)n, k.ownerIdx.data());
    if (frc != UST_OK) return frc;
    return rc == UST_ERR_TRUNCATED ? UST_OK : rc;
  }
  for (int64_t j = 0; j < n_out; j++) k.ownerIdx[(size_t)oi[(size_t)j]] = od[(size_t)j];
  buildStats_.outputs_received += n_out;
  return rc;
}

Error ClusterUpgradeStateManagerImpl::BuildStateIncremental(const std::string& ns, const StringMap& driverLabels,
                                                            std::unique_ptr<ClusterUpgradeState>* out) {
  Listed l;
  if (Error e = list(K8sClient, ns, driverLabels, &l)) return e;
  PodCache& k = podCache_;
  buildStats_.reconciles++;
  const bool full = !k.valid;
  const size_t nOld = full ? 0 : k.state.size(), np = l.podList.size();
  // the list in this reconcile's order: per position the cached pod it continues (-1: a pod that joins)
  PodCache nk;
  nk.posOf.reserve(np);
  nk.rv.resize(np);
  nk.state.resize(np);
  nk.owner.resize(2 * np);
  nk.ownerIdx.resize(np);
  std::vector<int64_t> from(np, -1);
  std::vector<char> present(nOld, 0);
  bool moved = false;
  int64_t last = -1, removed = (int64_t)nOld;
  for (size_t i = 0; i < np; i++) {
    const Pod& pod = *l.podList[i];
    const std::string key = pod.Namespace + "/" + pod.Name;
    if (!nk.posOf.emplace(key, i).second) {
      ResetBuildIncremental();
      return Errorf("pod " + key + " is listed twice");
    }
    nk.rv[i] = pod.ResourceVersion;
    auto it = full ? k.posOf.end() : k.posOf.find(key);
    if (it == k.posOf.end()) {  // joins
      derivePod(pod, &nk.state[i], &nk.owner[2 * i]);
      buildStats_.rederived++;
      nk.insert_at.push_back((int64_t)i);
      nk.ownerIdx[i] = INT32_MIN;  // comes back from the device: every joined pod is reported
      continue;
    }
    const size_t q = it->second;
    present[q] = 1;
    removed--;
    moved = moved || (int64_t)q < last;
    last = (int64_t)q;
    from[i] = (int64_t)q;
    nk.ownerIdx[i] = k.ownerIdx[q];
    if (!pod.ResourceVersion.empty() && pod.ResourceVersion == k.rv[q]) {
      nk.state[i] = k.state[q]; nk.owner[2 * i] = k.owner[2 * q]; nk.owner[2 * i + 1] = k.owner[2 * q + 1];
      buildStats_.reused++;
      continue;
    }
    derivePod(pod, &nk.state[i], &nk.owner[2 * i]);
    buildStats_.rederived++;
    if (nk.state[i] != k.state[q] || nk.owner[2 * i] != k.owner[2 * q] || nk.owner[2 * i + 1] != k.owner[2 * q + 1])
      nk.changed.push_back((int64_t)i);
  }
  // joins, leaves and moves travel as one reorder (after a reset: the whole list as one inserted run)
  nk.reorder = full || moved || removed > 0 || !nk.insert_at.empty();
  if (nk.reorder) orderRuns(from, &nk.run_src, &nk.run_len);
  if (full) {
    buildStats_.full_uploads++;
  } else {
    buildStats_.inserted += (int64_t)nk.insert_at.size();
    buildStats_.removed += removed;
    buildStats_.reorders += nk.reorder ? 1 : 0;
  }
  k = std::move(nk);
  ust_counters c;
  const int rc = BuildStateCached((int32_t)l.dsByIndex.size(), l.dsUid.data(), l.desired.data(), &k, &c);
  if (rc != UST_OK && rc != UST_ERR_DS_UNSCHEDULED) {  // the device list is not what the cache holds: start over
    ResetBuildIncremental();
    return Errorf(handle_ ? ust_last_error(handle_) : kNoDeviceBuildState);
  }
  k.valid = true;
  if (rc == UST_ERR_DS_UNSCHEDULED) return Errorf("driver DaemonSet should not have Unscheduled pods");  // upgrade_state.go:128-131
  return assembleState(l.podList, k.state.data(), k.ownerIdx.data(), l.daemonSets, out);
}

// ---- ApplyState = Encode -> kernel -> Replay -------------------------------------------------------------------
static void flatten_policy(const DriverUpgradePolicySpec& p, bool podDeletionEnabled, bool validationEnabled, bool useMaintenanceOperator,
                           ust_policy* c) {
  std::memset(c, 0, sizeof(*c));
  c->auto_upgrade = p.AutoUpgrade;
  c->max_parallel_upgrades = p.MaxParallelUpgrades;
  if (p.MaxUnavailable) {
    // intstr.GetScaledValueFromIntOrPercent: Int => IntVal; String must be "<int>%"; anything else is an error
    if (p.MaxUnavailable->Type == IntOrString::Int) {
      c->max_unavailable_kind = UST_MAXUNAVAIL_INT;
      c->max_unavailable_value = p.MaxUnavailable->IntVal;
    } else {
      const std::string& s = p.MaxUnavailable->StrVal;
      bool ok = s.size() >= 2 && s.back() == '%';
      size_t i = ok && (s[0] == '-' || s[0] == '+') ? 1 : 0;
      ok = ok && i < s.size() - 1;
      for (size_t k = i; ok && k + 1 < s.size(); k++) ok = s[k] >= '0' && s[k] <= '9';
      if (ok) {
        c->max_unavailable_kind = UST_MAXUNAVAIL_PERCENT;
        c->max_unavailable_value = std::stoll(s.substr(0, s.size() - 1));
      } else {
        c->max_unavailable_kind = UST_MAXUNAVAIL_INVALID;
      }
    }
  }
  c->pod_deletion_enabled = podDeletionEnabled;
  c->validation_enabled = validationEnabled;
  // a nil PodDeletionSpec is the PodManager's error to raise (pod_manager.go:132-134): the actuator gets the nil
  c->pod_deletion_spec_present = 1;
  if (p.PodDeletion) { c->pod_deletion_force = p.PodDeletion->Force; c->pod_deletion_delete_emptydir = p.PodDeletion->DeleteEmptyDir; }
  if (p.DrainSpec) { c->drain_enabled = p.DrainSpec->Enable; c->drain_force = p.DrainSpec->Force; c->drain_delete_emptydir = p.DrainSpec->DeleteEmptyDir; }
  if (p.WaitForCompletion) { c->wait_selector_set = !p.WaitForCompletion->PodSelector.empty(); c->wait_timeout_nonzero = p.WaitForCompletion->TimeoutSecond != 0; }
  c->use_maintenance_operator = useMaintenanceOperator;
}

// strconv.ParseInt(s, 10, 64) (Go 1.x): an optional sign, then decimal digits only; the error text is Go's. The input is
// quoted as strconv.Quote does: \", \\, \a \b \f \n \r \t \v, other ASCII controls and bytes that are not valid UTF-8
// as \xhh, C1 controls (U+0080-U+009F) as \u00hh. Other runes are copied: Go also escapes the non-printable ones among
// them (format characters such as U+200B, unassigned code points), which this does not.
static void goQuoteTo(const std::string& s, std::string* q) {
  static const char* hex = "0123456789abcdef";
  auto esc = [&](const char* pfx, unsigned v) { *q += pfx; *q += hex[(v >> 4) & 15]; *q += hex[v & 15]; };
  *q += '"';
  for (size_t i = 0; i < s.size();) {
    const unsigned char ch = (unsigned char)s[i];
    if (ch < 0x80) {
      switch (ch) {
        case '"': *q += "\\\""; break;
        case '\\': *q += "\\\\"; break;
        case '\a': *q += "\\a"; break;
        case '\b': *q += "\\b"; break;
        case '\f': *q += "\\f"; break;
        case '\n': *q += "\\n"; break;
        case '\r': *q += "\\r"; break;
        case '\t': *q += "\\t"; break;
        case '\v': *q += "\\v"; break;
        default:
          if (ch < 0x20 || ch == 0x7f) esc("\\x", ch); else *q += (char)ch;
      }
      i++;
      continue;
    }
    // one UTF-8 sequence: its length and code point, or an invalid byte (overlong forms, surrogates and > U+10FFFF too)
    const size_t len = ch >= 0xF0 ? 4 : ch >= 0xE0 ? 3 : ch >= 0xC0 ? 2 : 0;
    uint32_t cp = len == 4 ? ch & 7u : len == 3 ? ch & 15u : ch & 31u;
    bool ok = len > 0 && i + len <= s.size();
    for (size_t k = 1; ok && k < len; k++) {
      const unsigned char c = (unsigned char)s[i + k];
      ok = (c & 0xC0) == 0x80;
      cp = (cp << 6) | (c & 0x3Fu);
    }
    ok = ok && !(len == 2 && cp < 0x80) && !(len == 3 && cp < 0x800) && !(len == 4 && (cp < 0x10000 || cp > 0x10FFFF)) &&
         !(cp >= 0xD800 && cp <= 0xDFFF);
    if (!ok) { esc("\\x", ch); i++; continue; }
    if (cp <= 0x9F) esc("\\u00", cp); else q->append(s, i, len);
    i += len;
  }
  *q += '"';
}
static bool parseInt64(const std::string& s, int64_t* out, std::string* err) {
  auto fail = [&](const char* what) {
    *err = "strconv.ParseInt: parsing ";
    goQuoteTo(s, err);
    *err += ": ";
    *err += what;
    return false;
  };
  size_t i = 0;
  bool neg = false;
  if (!s.empty() && (s[0] == '+' || s[0] == '-')) { neg = s[0] == '-'; i = 1; }
  if (i == s.size()) return fail("invalid syntax");
  uint64_t u = 0;
  for (; i < s.size(); i++) {
    if (s[i] < '0' || s[i] > '9') return fail("invalid syntax");
    const uint64_t d = (uint64_t)(s[i] - '0');
    if (u > (UINT64_MAX - d) / 10) return fail("value out of range");  // ParseUint stops at the first overflow
    u = u * 10 + d;
  }
  if (u > (neg ? (uint64_t)INT64_MAX + 1 : (uint64_t)INT64_MAX)) return fail("value out of range");
  *out = neg ? (int64_t)(0 - u) : (int64_t)u;
  return true;
}

// A validation pod as Validate sees it (validation_manager.go:95-136): it matched the selector, and it is ready when it
// is Running, has container statuses and all of them are Ready.
static uint16_t validationPodFlags(const Pod& p) {
  bool ready = p.Phase == "Running" && !p.ContainerStatuses.empty();
  for (const auto& cs : p.ContainerStatuses) ready = ready && cs.Ready;
  return (uint16_t)(UST_POD_MATCH_VALIDATION_SELECTOR | (ready ? UST_POD_READY : 0));
}

// A wait-selector pod as ScheduleCheckOnPodCompletion sees it (pod_manager.go:263, :371-391): it matched the selector,
// and only its phase matters; a phase IsPodRunningOrPending does not name counts as not running.
// a pod phase as UST_PHASE_*; a phase IsPodRunningOrPending does not name is UST_PHASE_OTHER
static uint16_t phaseBits(const Pod& p) {
  return (uint16_t)(p.Phase == "Running" ? UST_PHASE_RUNNING : p.Phase == "Pending" ? UST_PHASE_PENDING
                    : p.Phase == "Succeeded" ? UST_PHASE_SUCCEEDED : p.Phase == "Failed" ? UST_PHASE_FAILED : UST_PHASE_OTHER);
}
static uint16_t waitPodFlags(const Pod& p) { return (uint16_t)(UST_POD_MATCH_WAIT_SELECTOR | phaseBits(p)); }
// "any wait pod Running or Pending" (pod_manager.go:278-284) over a node's list as handed to the device
static bool anyWaitRunning(const uint16_t* b, const uint16_t* e) {
  for (; b != e; b++) {
    const unsigned phase = *b & UST_POD_PHASE_MASK;
    if ((*b & UST_POD_MATCH_WAIT_SELECTOR) && (phase == UST_PHASE_RUNNING || phase == UST_PHASE_PENDING)) return true;
  }
  return false;
}

// A workload pod as the kubectl drain filter chain sees it (k8s.io/kubectl pkg/drain/filters.go; ust_pod_chain_keeps):
// phase, metav1.GetControllerOf (the first owner reference with Controller set) and whether that controller is a
// DaemonSet the DaemonSet List does not hold (daemonSetFilter's Get by namespace and name, NotFound), the mirror-pod
// annotation, an emptyDir volume; and whether the pod-deletion filter and the drain's PodSelector select it. kubectl's
// skipDeletedFilter never skips a pod here: both helpers leave SkipWaitForDeleteTimeoutSeconds at 0 (pod_manager.go:146-157,
// drain_manager.go:76-96), and shouldSkipPod requires it to be > 0 (filters.go).
static const OwnerReference* controllerOf(const Pod& p) {
  for (const auto& o : p.OwnerReferences)
    if (o.Controller) return &o;
  return nullptr;
}
static const char* const kMirrorPodAnnotationKey = "kubernetes.io/config.mirror";  // corev1.MirrorPodAnnotationKey

// The text of kubectl's drain errors: the filters' fatal messages (k8s.io/kubectl v0.35.1 pkg/drain/filters.go:
// localStorageFatal, unmanagedFatal; daemonSetFilter returns the Get's error, the API's NotFound text), PodDeleteList.errors
// (drain.go: "cannot delete <message>: <ns/name, ...>" per distinct message) and utilerrors.NewAggregate's Error
// (k8s.io/apimachinery pkg/util/errors: one error prints itself, several print "[a, b]"). Restated from upstream, not
// pinned by the reference's tests. Upstream groups the pods in a Go map, so its message order varies from run to run;
// here the messages come in the order of their first pod in the List, and each message's pods in List order.
Error DrainFilterError(const std::vector<const Pod*>& pods, const std::vector<uint16_t>& bits, const DrainSpec& spec) {
  std::vector<std::pair<std::string, std::string>> failed;  // message, its pods
  for (size_t j = 0; j < pods.size() && j < bits.size(); j++) {
    bool isError = false;
    unsigned stop = UST_CHAIN_NONE;
    if (!(bits[j] & UST_POD_MATCH_DRAIN_SELECTOR)) continue;
    ust_pod_chain_keeps(bits[j], spec.Force, spec.DeleteEmptyDir, &isError, &stop);
    if (!isError) continue;
    const Pod& p = *pods[j];
    std::string msg;
    if (stop == UST_CHAIN_DS_MISSING) msg = "daemonsets.apps \"" + controllerOf(p)->Name + "\" not found";
    else if (stop == UST_CHAIN_LOCAL_STORAGE) msg = "Pods with local storage (use --delete-emptydir-data to override)";
    else msg = "Pods declare no controller (use --force to override)";
    auto it = std::find_if(failed.begin(), failed.end(), [&](const auto& f) { return f.first == msg; });
    if (it == failed.end()) it = failed.insert(failed.end(), {msg, ""});
    else it->second += ", ";
    it->second += p.Namespace + "/" + p.Name;
  }
  if (failed.empty()) return std::nullopt;
  std::string s;
  for (const auto& f : failed) s += (s.empty() ? "" : ", ") + ("cannot delete " + f.first + ": " + f.second);
  return Errorf(failed.size() == 1 ? s : "[" + s + "]");
}
// What the workload entries of one reconcile are derived from: every pod by node (ListPodsBySelector("", "")), the pods
// the drain's PodSelector matches (a second List, only for a non-empty selector: the mirror matches no label selector
// itself) and every DaemonSet (ListDaemonSets), keyed by Namespace/Name.
struct WorkloadLists {
  std::unordered_map<std::string, std::vector<const Pod*>> byNode;
  bool drainAll = true;
  std::unordered_set<std::string> drainSelected, daemonSets;
  const PodDeletionFilter* filter = nullptr;  // nullptr: the pod-deletion pass is not answered on the device
  bool drain = false;                         // the drain pass is
  Error podsError, selectorError, dsError;
};
static void listWorkload(K8sClient* client, const DriverUpgradePolicySpec& policy, const PodDeletionFilter* filter, bool drain,
                         WorkloadLists* w) {
  w->filter = filter;
  w->drain = drain;
  if (client == nullptr) { w->podsError = Errorf("no K8sClient to list the workload pods with"); return; }
  std::vector<Pod*> pods;
  if ((w->podsError = client->ListPodsBySelector("", "", &pods))) return;
  for (const Pod* p : pods)
    if (!p->NodeName.empty()) w->byNode[p->NodeName].push_back(p);
  if (drain && !policy.DrainSpec->PodSelector.empty()) {
    w->drainAll = false;
    std::vector<Pod*> sel;
    if (!(w->selectorError = client->ListPodsBySelector(policy.DrainSpec->PodSelector, "", &sel)))
      for (const Pod* p : sel) w->drainSelected.insert(p->Namespace + "/" + p->Name);
  }
  std::vector<DaemonSet*> dss;
  if (!(w->dsError = client->ListDaemonSets("", {}, &dss)))
    for (const DaemonSet* d : dss) w->daemonSets.insert(d->Namespace + "/" + d->Name);
}
static uint16_t workloadPodFlags(const Pod& p, const WorkloadLists& w) {
  uint16_t f = phaseBits(p);
  if (const OwnerReference* c = controllerOf(p)) {
    f |= UST_POD_HAS_CONTROLLER;
    if (c->Kind == "DaemonSet") {
      f |= UST_POD_CONTROLLED_BY_DS;
      if (!w.daemonSets.count(p.Namespace + "/" + c->Name)) f |= UST_POD_DS_MISSING;
    }
  }
  if (p.Annotations.count(kMirrorPodAnnotationKey)) f |= UST_POD_MIRROR;
  if (p.HasEmptyDirVolume) f |= UST_POD_HAS_EMPTYDIR;
  if (w.filter && (*w.filter)(p)) f |= UST_POD_MATCH_DELETION_FILTER;
  if (w.drain && (w.drainAll || w.drainSelected.count(p.Namespace + "/" + p.Name))) f |= UST_POD_MATCH_DRAIN_SELECTOR;
  return f;
}

// The one List per selector of a ValidateOnDevice / WaitForCompletionOnDevice reconcile, grouped by node. The reference
// lists per node, with the selector and the field selector spec.nodeName=<node> (validation_manager.go:77-79,
// pod_manager.go:320-329); this takes one cluster-wide List and keeps its order within each node. That rests on one
// assumption: the API server returns a node's pods in the same relative order in both Lists (it sorts a List by
// namespace and name). Validate's answer depends on that order: a ready pod listed before a not-ready one resets the
// start time (INTEGRATION.md, "Encoding the validation pods"); the wait-for-completion check does not ("any pod Running
// or Pending").
using PodsByNode = std::unordered_map<std::string, std::vector<const Pod*>>;
static Error listPodsBySelector(K8sClient* client, const std::string& selector, const char* what, PodsByNode* byNode) {
  if (client == nullptr) return Errorf(std::string("no K8sClient to list the ") + what + " pods with");
  std::vector<Pod*> pods;
  if (Error e = client->ListPodsBySelector(selector, "", &pods)) return e;
  for (const Pod* p : pods)
    if (!p->NodeName.empty()) (*byNode)[p->NodeName].push_back(p);
  return std::nullopt;
}
// A node's pods in one List, in the List's order; nullptr: none.
static const std::vector<const Pod*>* podsOf(const PodsByNode& byNode, const std::string& node) {
  auto it = byNode.find(node);
  return it == byNode.end() ? nullptr : &it->second;
}

// One snapshot entry -> its four SoA values. `ds` / `dsErr`: index of its DaemonSet in the table (-1 = orphaned) and
// whether that DaemonSet's revision-hash lookup failed; `deferred` receives an error the reference would raise when
// its pass reaches the node; `start` (the clocked calls only, else nullptr) the node's start time: the parsed validation
// start time with `validation` (ValidateOnDevice), replaced on a wait-for-jobs-required node by the parsed wait start
// time with `wait` (WaitForCompletionOnDevice), 0 otherwise. The device reads it only in those two states.
Error ClusterUpgradeStateManagerImpl::encodeOne(const NodeUpgradeState* ns, int code, int32_t ds, bool dsErr,
                                                std::map<std::string, int32_t>* intern, const std::vector<int32_t>& ds_rev,
                                                uint8_t* hot_out, uint32_t* flags_out, int32_t* rev_out, std::string* deferred,
                                                int64_t* start, bool validation, bool wait) {
  auto internHash = [&](const std::string& h) {  // find first: emplace would build (and throw away) a map node per node
    auto it = intern->find(h);
    return it != intern->end() ? it->second : intern->emplace(h, (int32_t)intern->size() + 1).first->second;
  };
  const Node& n = *ns->Node;
  uint8_t hot = (uint8_t)code;
  uint32_t f = 0;
  if (IsNodeUnschedulable(n)) hot |= UST_HOT_UNSCHEDULABLE;
  if (!isNodeConditionReady(n)) hot |= UST_HOT_NOT_READY;
  if (SkipNodeUpgrade(n)) hot |= UST_HOT_SKIP;
  if (IsUpgradeRequested(n)) f |= UST_F_UPGRADE_REQUESTED;
  if (n.Annotations.count(keys().initialState)) f |= UST_F_INITIAL_STATE_ANNO;
  if (IsNodeInRequestorMode(n)) f |= UST_F_REQUESTOR_MODE;
  // ValidationManager.Validate is an actuator with side effects: Replay calls it, at the reference's point in
  // the pass order, and drops the transition when it reports "not done" (common_manager.go:587-596)
  f |= UST_F_VALIDATION_DONE;
  int32_t rev = 0;
  bool synced = false;
  if (ns->IsOrphanedPod()) {
    f |= UST_F_POD_ORPHANED;
  } else {
    std::string podHash;
    if (ns->DriverPod == nullptr || PodManager->GetPodControllerRevisionHash(ns->DriverPod, &podHash) || dsErr)
      hot |= UST_HOT_REVISION_HASH_ERROR;  // pod_manager.go:84-89, :108-110
    else {
      rev = internHash(podHash);
      synced = rev == ds_rev[(size_t)ds];
    }
  }
  // IsWaitingForSafeDriverLoad: the reference consults it in the unknown / upgrade-done passes only
  // (common_manager.go:240) and returns its error there; the pod-restart and validation passes call UnblockLoading
  // unconditionally (:477, :581), a no-op unless the node is waiting - there the predicate only selects whether the
  // call is replayed, and an error from it selects "replay".
  if (code == UST_STATE_UNKNOWN || code == UST_STATE_DONE) {
    bool waiting = false;
    if (Error err = SafeDriverLoadManager->IsWaitingForSafeDriverLoad(&n, &waiting)) {
      if (!(hot & UST_HOT_REVISION_HASH_ERROR)) {  // podInSyncWithDS fails first (:234-238)
        *deferred = *err;
        hot |= UST_HOT_REVISION_HASH_ERROR;         // same abort point: before any action on the node
      }
    } else if (waiting) {
      f |= UST_F_SAFE_LOAD;
    }
  } else if (code == UST_STATE_VALIDATION_REQUIRED || (code == UST_STATE_POD_RESTART_REQUIRED && synced)) {
    bool waiting = false;
    if (SafeDriverLoadManager->IsWaitingForSafeDriverLoad(&n, &waiting) || waiting) f |= UST_F_SAFE_LOAD;
  }
  if (const Pod* p = ns->DriverPod) {
    bool ready = p->Phase == "Running" && !p->ContainerStatuses.empty();  // common_manager.go:617-630
    for (const auto& cs : p->ContainerStatuses) ready = ready && cs.Ready;
    if (ready) f |= UST_F_POD_READY;
    if (isDriverPodFailing(*p)) f |= UST_F_POD_FAILING;
    if (p->DeletionTimestampSet) f |= UST_F_POD_TERMINATING;
  }
  if (ns->NodeMaintenance) {
    f |= UST_F_NM_PRESENT;
    if (ns->NodeMaintenance->ReadyConditionWithReasonReady) f |= UST_F_NM_READY;
  }
  if (start) *start = 0;
  if (start && validation) {  // StateOptions::ValidateOnDevice: the start-time annotation handleTimeout reads (validation_manager.go:142-160)
    auto it = n.Annotations.find(keys().validationStart);
    if (it != n.Annotations.end()) {
      f |= UST_F_VALIDATION_START_ANNO;
      std::string err;
      if (!parseInt64(it->second, start, &err)) {
        f |= UST_F_VALIDATION_START_INVALID;
        *start = 0;
        // Validate's error when it reaches the node (:97-101); the device returns UST_ERR_VALIDATION there
        if (code == UST_STATE_VALIDATION_REQUIRED) *deferred = "unable to handle timeout for validation state: " + err;
      }
    }
  }
  if (start && wait) {  // StateOptions::WaitForCompletionOnDevice: the start-time annotation HandleTimeoutOnPodCompletions
                        // reads (pod_manager.go:336-353); a value that does not parse is an error the check swallows
    auto it = n.Annotations.find(keys().waitStart);
    int64_t v = 0;
    if (it != n.Annotations.end()) {
      f |= UST_F_WAIT_START_ANNO;
      std::string err;
      if (!parseInt64(it->second, &v, &err)) { f |= UST_F_WAIT_START_INVALID; v = 0; }
    }
    if (code == UST_STATE_WAIT_FOR_JOBS_REQUIRED) *start = v;
  }
  *hot_out = hot;
  *flags_out = f;
  *rev_out = rev;
  return std::nullopt;
}

Error ClusterUpgradeStateManagerImpl::Encode(const ClusterUpgradeState& s, const DriverUpgradePolicySpec& policy, EncodedSnapshot* out) {
  EncodedSnapshot& e = *out;
  e = EncodedSnapshot();
  (void)keys();  // built before any worker thread reads them
  flatten_policy(policy, podDeletionStateEnabled_, validationStateEnabled_, opts_.Requestor.UseMaintenanceOperator, &e.policy);
  // 1. the entries, buckets in pass order: SoA index order == replay order, and the upgrade-required bucket keeps its
  //    slice order
  std::vector<int8_t> codes;
  auto take = [&](const std::vector<NodeUpgradeState*>& bucket, int code) {
    e.entries.insert(e.entries.end(), bucket.begin(), bucket.end());
    codes.insert(codes.end(), bucket.size(), (int8_t)code);
  };
  for (int code : kPassOrder) {
    auto it = s.NodeStates.find(kStateNames[code]);
    if (it != s.NodeStates.end()) take(it->second, code);
  }
  // every other bucket still counts towards GetCurrentUnavailableNodes (common_manager.go:149)
  for (const auto& kv : s.NodeStates) {
    const int code = StateCodeOfLabel(kv.first);
    if (code == UST_STATE_OTHER || code == UST_STATE_POST_MAINTENANCE_REQUIRED) take(kv.second, code);
  }
  const size_t n = e.entries.size();
  // 2. the DaemonSet table: one revision lookup per DaemonSet (pod_manager.go:92-118), in first-use order
  std::map<std::string, int32_t> intern;
  std::map<const DaemonSet*, int32_t> dsIndex;
  std::vector<char> dsHashError;
  e.ds_idx.assign(n, -1);
  for (size_t i = 0; i < n; i++) {
    const NodeUpgradeState* ns = e.entries[i];
    if (ns->IsOrphanedPod()) continue;
    auto it = dsIndex.find(ns->DriverDaemonSet);
    if (it == dsIndex.end()) {
      std::string dsHash;
      const bool bad = (bool)PodManager->GetDaemonsetControllerRevisionHash(ns->DriverDaemonSet, &dsHash);
      it = dsIndex.emplace(ns->DriverDaemonSet, (int32_t)e.ds_rev.size()).first;
      e.ds_rev.push_back(bad ? 0 : intern.emplace(dsHash, (int32_t)intern.size() + 1).first->second);
      dsHashError.push_back(bad ? 1 : 0);
    }
    e.ds_idx[i] = it->second;
  }
  // 3. the nodes, independent of one another. A worker interns the revision hashes it meets in a copy of the table above
  //    (so "pod hash == DaemonSet hash" is an id comparison everywhere); hashes no DaemonSet has get provisional ids that
  //    are made global afterwards.
  e.state.assign(n, 0);
  e.flags.assign(n, 0);
  e.pod_rev.assign(n, 0);
  e.validateOnDevice = validateOnDevice();
  e.waitOnDevice = waitOnDevice(policy);
  e.evictOnDevice = evictOnDevice(policy);
  const bool clocked = e.validateOnDevice || e.waitOnDevice || e.evictOnDevice;
  if (clocked) e.start.assign(n, 0);
  const int32_t base = (int32_t)intern.size();
  const size_t workers = (size_t)std::max(1, std::min(opts_.EncodeThreads, (int)(n / 4096 + 1)));
  struct Part { std::map<std::string, int32_t> intern; std::vector<std::pair<size_t, std::string>> deferred; Error err; size_t errAt = 0; };
  std::vector<Part> parts(workers);
  auto work = [&](size_t w) {
    Part& p = parts[w];
    p.intern = intern;
    const size_t i0 = n * w / workers, i1 = n * (w + 1) / workers;
    for (size_t i = i0; i < i1; i++) {
      const int32_t ds = e.ds_idx[i];
      uint8_t hot; uint32_t f; int32_t rev; std::string deferred;
      if (Error err = encodeOne(e.entries[i], codes[i], ds, ds >= 0 && dsHashError[(size_t)ds], &p.intern, e.ds_rev, &hot, &f, &rev, &deferred,
                                clocked ? &e.start[i] : nullptr, e.validateOnDevice, e.waitOnDevice)) {
        p.err = err; p.errAt = i;
        return;
      }
      if (!deferred.empty()) p.deferred.emplace_back(i, deferred);
      e.state[i] = hot; e.flags[i] = f; e.pod_rev[i] = rev;
    }
  };
  if (workers == 1) {
    work(0);
  } else {
    std::vector<std::thread> pool;
    for (size_t w = 1; w < workers; w++) pool.emplace_back(work, w);
    work(0);
    for (auto& t : pool) t.join();
  }
  for (size_t w = 0; w < workers; w++) {   // first error in index order, like the sequential walk
    if (parts[w].err) return parts[w].err;
    for (auto& d : parts[w].deferred) e.deferred[d.first] = d.second;
  }
  if (workers > 1) {  // provisional ids (> base, per worker) -> global ids
    for (size_t w = 0; w < workers; w++) {
      std::vector<int32_t> remap(parts[w].intern.size() + 1, 0);
      bool moved = false;
      for (const auto& kv : parts[w].intern) {
        if (kv.second <= base) continue;
        const int32_t g = intern.emplace(kv.first, (int32_t)intern.size() + 1).first->second;
        remap[(size_t)kv.second] = g;
        moved = moved || g != kv.second;
      }
      if (!moved) continue;
      const size_t i0 = n * w / workers, i1 = n * (w + 1) / workers;
      for (size_t i = i0; i < i1; i++)
        if (e.pod_rev[i] > base) e.pod_rev[i] = remap[(size_t)e.pod_rev[i]];
    }
  }
  // 4. ValidateOnDevice / WaitForCompletionOnDevice / EvictionOnDevice: every entry's list (an empty one when it has no
  //    pod), from one List per selector: its validation pods, then its wait-selector pods, then (pod-deletion-required and
  //    drain-required entries only) every pod on its node. A pod several Lists hold is in the list once per List, each
  //    entry with its own role's bits: each pass reads only the entries that carry its own selector bit.
  if (clocked) {
    e.policy.evaluate_actuators = UST_EVAL_ACTUATORS | (e.validateOnDevice ? UST_EVAL_VALIDATION : 0);
    e.now = opts_.Now();
    PodsByNode vpods, wpods;
    if (e.validateOnDevice) e.listError = listPodsBySelector(K8sClient, validationSelector_, "validation", &vpods);
    if (e.waitOnDevice) {
      e.waitListError = listPodsBySelector(K8sClient, policy.WaitForCompletion->PodSelector, "wait-for-completion", &wpods);
      e.waitRunning.assign(n, 0);
    }
    WorkloadLists wl;
    if (e.evictOnDevice) {
      listWorkload(K8sClient, policy, evictPodDeletion(policy) ? &filter_ : nullptr, evictDrain(policy), &wl);
      e.evictListError = wl.podsError ? wl.podsError : wl.dsError;
      e.drainListError = e.evictListError ? e.evictListError : wl.selectorError;
    }
    e.pod_off.assign(n + 1, 0);
    for (size_t i = 0; i < n; i++) {
      const std::string& name = e.entries[i]->Node->Name;
      if (const auto* v = e.listError ? nullptr : podsOf(vpods, name))
        for (const Pod* p : *v) e.pod_flags.push_back(validationPodFlags(*p));
      const size_t w0 = e.pod_flags.size();
      if (const auto* w = e.waitListError ? nullptr : podsOf(wpods, name))
        for (const Pod* p : *w) e.pod_flags.push_back(waitPodFlags(*p));
      if (e.waitOnDevice) e.waitRunning[i] = anyWaitRunning(e.pod_flags.data() + w0, e.pod_flags.data() + e.pod_flags.size());
      const int code = codes[i];
      if (e.evictOnDevice && !e.evictListError && (code == UST_STATE_POD_DELETION_REQUIRED || code == UST_STATE_DRAIN_REQUIRED))
        if (const auto* a = podsOf(wl.byNode, name)) {
          EncodedSnapshot::Workload& wk = e.workload[i];
          for (const Pod* p : *a) {
            wk.pods.push_back(p);
            wk.bits.push_back(workloadPodFlags(*p, wl));
          }
          e.pod_flags.insert(e.pod_flags.end(), wk.bits.begin(), wk.bits.end());
        }
      e.pod_off[i + 1] = (int32_t)e.pod_flags.size();
    }
  }
  return std::nullopt;
}

Error ClusterUpgradeStateManagerImpl::Replay(const EncodedSnapshot& enc, const DriverUpgradePolicySpec& policy,
                                             const uint8_t* next_state, const uint16_t* actions, int abi_rc,
                                             const ust_counters& counters, const uint8_t* actuator_outcome) {
  const size_t n = enc.entries.size();
  const bool drainEnabled = policy.DrainSpec && policy.DrainSpec->Enable;
  const bool waitSelector = policy.WaitForCompletion && !policy.WaitForCompletion->PodSelector.empty();
  const bool requestor = opts_.Requestor.UseMaintenanceOperator;
  auto setState = [&](size_t i) { return NodeUpgradeStateProvider->ChangeNodeUpgradeState(enc.entries[i]->Node, StateNameOfCode(next_state[i])); };
  auto anno = [&](size_t i, const std::string& k, const char* v) { return NodeUpgradeStateProvider->ChangeNodeUpgradeAnnotation(enc.entries[i]->Node, k, v); };
  auto validationError = [](const Error& e) { return Errorf("unable to handle timeout for validation state: " + *e); };  // :97-101
  // The events of the managers an option replaces (logEvent / logEventf, util.go:162-176). Workers take `recorder` and
  // `reason` by value.
  upgrade::EventRecorder* const recorder = EventRecorder;
  const std::string reason = recorder ? GetEventReason() : std::string();
  auto event = [recorder, reason](const Node& n, const char* type, const std::string& message) {
    if (recorder) recorder->Event(n, type, reason, message);
  };
  // validation_manager.go:97-101 passes err.Error() to a format without a verb: Go appends it as %!(EXTRA string=...)
  auto validationEvent = [&](const Node& n, const std::string& err) {
    event(n, EventTypeWarning, "Failed to handle timeout for validation state%!(EXTRA string=" + err + ")");
  };
  auto abortError = [&](long long idx = -1) -> Error {
    if (idx >= 0) { auto it = enc.deferred.find((size_t)idx); if (it != enc.deferred.end()) return Errorf(it->second); }
    return Errorf(ust_last_error(handle_));
  };

  size_t i = 0;
  for (int pass = 0; pass < 12; pass++) {
    const int code = kPassOrder[pass];
    // policy-level abort raised at the start of a pass (intstr parse error, upgrade_inplace.go:54-60)
    if (abi_rc != UST_OK && counters.error_index < 0 && counters.error_pass == pass) return abortError();
    if (code == UST_STATE_NODE_MAINTENANCE_REQUIRED && !requestor) {  // upgrade_state.go:299-309
      while (i < n && (int)(enc.state[i] & UST_HOT_STATE_MASK) == code) i++;
      continue;
    }
    const size_t begin = i;
    std::vector<Node*> batchNodes;
    std::vector<Pod*> restartPods;
    for (; i < n && (int)(enc.state[i] & UST_HOT_STATE_MASK) == code; i++) {
      if (code == UST_STATE_UNCORDON_REQUIRED) continue;  // two sub-passes below
      const unsigned a = actions[i];
      Node* node = enc.entries[i]->Node;
      const bool onDevice = code == UST_STATE_VALIDATION_REQUIRED && enc.validateOnDevice;
      if ((a & UST_A_ERROR) && !onDevice) return abortError((long long)i);
      if (a & UST_A_CLEAR_UPGRADE_REQUESTED)
        if (Error e = anno(i, GetUpgradeRequestedAnnotationKey(), kNullString)) return e;
      if (a & UST_A_SET_INITIAL_STATE_ANNO)
        if (Error e = anno(i, GetUpgradeInitialStateAnnotationKey(), kTrueString)) return e;
      if (a & UST_A_CORDON)
        if (Error e = CordonManager->Cordon(node)) return e;
      if (a & UST_A_UNBLOCK_SAFE_LOAD)
        if (Error e = SafeDriverLoadManager->UnblockLoading(node)) return e;
      if (onDevice) {
        // the calls Validate makes (validation_manager.go:71-175), as the device answered it
        if (enc.listError) return enc.listError;  // its List failed (:79-83)
        const std::string& key = GetValidationStartTimeAnnotationKey();
        if (a & UST_A_ERROR) {  // the start time does not parse (:155-160)
          auto it = node->Annotations.find(key);
          int64_t start = 0;
          std::string err;
          if (it != node->Annotations.end() && !parseInt64(it->second, &start, &err)) validationEvent(*node, err);
          return abortError((long long)i);
        }
        if (next_state[i] == UST_STATE_FAILED) {  // handleTimeout: timed out (:161-172)
          (void)NodeUpgradeStateProvider->ChangeNodeUpgradeState(node, UpgradeStateFailed);  // error ignored (:163)
          if (Error e = anno(i, key, kNullString)) { validationEvent(*node, *e); return validationError(e); }
          continue;
        }
        if (a & UST_A_CLEAR_WAIT_START)  // a ready pod (:106-113)
          if (Error e = anno(i, key, kNullString)) return e;
        if (a & UST_A_SET_WAIT_START)    // handleTimeout: no start time yet (:143-152)
          if (Error e = anno(i, key, std::to_string(enc.now).c_str())) { validationEvent(*node, *e); return validationError(e); }
        if (!(a & UST_A_SET_STATE)) continue;  // "Validations not complete on the node"
      } else if (code == UST_STATE_VALIDATION_REQUIRED) {
        bool done = false;
        if (Error e = ValidationManager->Validate(node, &done)) return e;
        if (!done) continue;  // "Validations not complete on the node"
      }
      if ((a & UST_A_NM_CREATE_OR_DELETE) && code == UST_STATE_UPGRADE_REQUIRED)  // upgrade_requestor.go:296
        if (K8sClient != nullptr)
          if (Error e = K8sClient->CreateOrUpdateNodeMaintenance(enc.entries[i])) return e;
      if ((a & UST_A_REQUESTOR_ANNO_CHANGE) && code == UST_STATE_UPGRADE_REQUIRED)
        if (Error e = anno(i, GetUpgradeRequestorModeAnnotationKey(), kTrueString)) return Errorf("failed annotate node for 'upgrade-requestor-mode'. " + *e);
      if (a & UST_A_SET_STATE) {
        Error e = setState(i);
        // common_manager.go:399, :432 deliberately ignore this error in the wait-for-jobs / pod-deletion passes
        if (e && code != UST_STATE_WAIT_FOR_JOBS_REQUIRED && code != UST_STATE_POD_DELETION_REQUIRED) return e;
      }
      if (a & UST_A_CLEAR_INITIAL_STATE_ANNO)
        if (Error e = anno(i, GetUpgradeInitialStateAnnotationKey(), kNullString)) return e;
      if (a & (UST_A_SCHEDULE_WAIT_CHECK | UST_A_SCHEDULE_POD_EVICTION | UST_A_SCHEDULE_DRAIN)) batchNodes.push_back(node);
      if (a & UST_A_RESTART_DRIVER_POD) restartPods.push_back(enc.entries[i]->DriverPod);
    }
    const bool cut = abi_rc != UST_OK && counters.error_pass == pass;  // the kernel stopped inside this pass
    switch (code) {
      case UST_STATE_WAIT_FOR_JOBS_REQUIRED:
        if (enc.waitOnDevice && i > begin) {
          // the calls ScheduleCheckOnPodCompletion makes (pod_manager.go:256-317), as the device answered it. Its per-node
          // List came first: a failed one returns before any node's check has started.
          if (enc.waitListError) return enc.waitListError;
          if (actuator_outcome == nullptr) return Errorf("Replay: the wait-for-jobs pass on the device needs actuator_outcome");
          const std::string& key = GetWaitForPodCompletionStartTimeAnnotationKey();
          for (size_t k = begin; k < i; k++) {
            if (!(actions[k] & UST_A_SCHEDULE_WAIT_CHECK)) continue;
            // The reference checks each node in a goroutine that took the node by value (go func(node corev1.Node), :275):
            // its calls get a copy, so that they do not write to the caller's snapshot object. Every error is recorded as an
            // event and dropped there (:290-312).
            Node node = *enc.entries[k]->Node;
            auto timeoutEvent = [&](const std::string& err) {  // :290-296
              event(node, EventTypeWarning, "Failed to handle timeout for job completions, " + err);
            };
            if (actuator_outcome[k] == UST_STATE_POD_DELETION_REQUIRED) {
              if (!enc.waitRunning[k]) {  // no wait pod Running or Pending: delete the start time, then the state (:300-309)
                if (Error e = NodeUpgradeStateProvider->ChangeNodeUpgradeAnnotation(&node, key, kNullString))
                  event(node, EventTypeWarning, "Failed to remove annotation used to track job completions: " + *e);
                else
                  (void)NodeUpgradeStateProvider->ChangeNodeUpgradeState(&node, UpgradeStatePodDeletionRequired);
              } else {  // still running, timed out: the state, then the start time (HandleTimeoutOnPodCompletions :354-365)
                (void)NodeUpgradeStateProvider->ChangeNodeUpgradeState(&node, UpgradeStatePodDeletionRequired);
                if (Error e = NodeUpgradeStateProvider->ChangeNodeUpgradeAnnotation(&node, key, kNullString)) timeoutEvent(*e);
              }
            } else if (actions[k] & UST_A_SET_WAIT_START) {  // running, no start time yet (:336-345)
              if (Error e = NodeUpgradeStateProvider->ChangeNodeUpgradeAnnotation(&node, key, std::to_string(enc.now))) timeoutEvent(*e);
            } else if (enc.waitRunning[k] && waitSelector && policy.WaitForCompletion->TimeoutSecond != 0) {
              // still waiting, or the start time does not parse (:348-353): only the latter has an event
              auto it = node.Annotations.find(key);
              int64_t start = 0;
              std::string err;
              if (it != node.Annotations.end() && !parseInt64(it->second, &start, &err)) timeoutEvent(err);
            }
            // otherwise no timeout: no call
          }
        } else if (waitSelector && !batchNodes.empty()) {  // common_manager.go:404-418
          PodManagerConfig cfg;
          cfg.WaitForCompletionSpec = &*policy.WaitForCompletion;
          cfg.Nodes = batchNodes;
          if (Error e = PodManager->ScheduleCheckOnPodCompletion(cfg)) return e;
        }
        break;
      case UST_STATE_POD_DELETION_REQUIRED:
        if (enc.evictOnDevice && evictPodDeletion(policy)) {
          if (i == begin) break;
          // the goroutines of SchedulePodEviction (pod_manager.go:159-227), as the device answered them. The List they
          // were answered from came first: a failed one returns before any node is touched.
          if (enc.evictListError) return enc.evictListError;
          if (actuator_outcome == nullptr) return Errorf("Replay: the pod-deletion pass on the device needs actuator_outcome");
          const PodDeletionSpec& spec = *policy.PodDeletion;
          for (size_t k = begin; k < i; k++) {
            if (!(actions[k] & UST_A_SCHEDULE_POD_EVICTION)) continue;
            const std::string& name = enc.entries[k]->Node->Name;
            {
              std::lock_guard<std::mutex> l(actMu_);
              if (nodesInProgress_.count(name)) continue;  // "Node is already getting pods deleted, skipping" (:224-226)
            }
            Node node = *enc.entries[k]->Node;  // go func(node corev1.Node) (:164, :223): the calls act on a copy
            const auto w = enc.workload.find(k);
            // toDelete: the pods the filter selects (:176-182). GetPodsForDeletion(node).Pods() holds a pod only when every
            // filter says "delete", and the deletion filter says "skip" for any other pod (:138-144), so Pods() is a subset
            // of toDelete; with numPodsCanDelete == numPodsToDelete (:193-201) the two sets are equal, in the List's order.
            std::vector<Pod> toDelete;
            if (w != enc.workload.end())
              for (size_t j = 0; j < w->second.pods.size(); j++)
                if (w->second.bits[j] & UST_POD_MATCH_DELETION_FILTER) toDelete.push_back(*w->second.pods[j]);
            const uint8_t out = actuator_outcome[k];
            if (out == UST_STATE_DRAIN_REQUIRED || out == UST_STATE_FAILED) {  // updateNodeToDrainOrFailed (:194-201, :393-403)
              if (drainEnabled) event(node, EventTypeWarning, kDrainInsteadMessage);
              (void)NodeUpgradeStateProvider->ChangeNodeUpgradeState(&node, StateNameOfCode(out));
            } else if (out != UST_STATE_POD_RESTART_REQUIRED) {
              return Errorf("Replay: no pod-deletion outcome for node " + name);
            } else if (toDelete.empty()) {  // "No pods require deletion" (:184-188)
              (void)NodeUpgradeStateProvider->ChangeNodeUpgradeState(&node, UpgradeStatePodRestartRequired);
            } else {  // DeleteOrEvictPods, then the state (:210-222)
              EvictionOptions o;
              o.Force = spec.Force; o.DeleteEmptyDir = spec.DeleteEmptyDir; o.TimeoutSecond = spec.TimeoutSecond;
              upgrade::NodeUpgradeStateProvider* provider = NodeUpgradeStateProvider;
              upgrade::PodEvictor* evictor = PodEvictor;
              stats_.actuator_handoffs++;
              handOff(&nodesInProgress_, name, [provider, evictor, node, pods = std::move(toDelete), o, drainEnabled, event]() mutable {
                std::vector<Pod*> ptrs;
                for (Pod& p : pods) ptrs.push_back(&p);
                const Error err = evictor ? evictor->DeleteOrEvictPods(node, ptrs, o) : Errorf("no PodEvictor");
                if (err) {
                  event(node, EventTypeWarning, "Failed to delete workload pods on the node for the driver upgrade, " + *err);
                  if (drainEnabled) event(node, EventTypeWarning, kDrainInsteadMessage);
                  (void)provider->ChangeNodeUpgradeState(&node, drainEnabled ? UpgradeStateDrainRequired : UpgradeStateFailed);
                } else {
                  (void)provider->ChangeNodeUpgradeState(&node, UpgradeStatePodRestartRequired);
                  event(node, EventTypeNormal, "Deleted workload pods on the node for the driver upgrade");
                }
              });
            }
          }
        } else if (podDeletionStateEnabled_ && !batchNodes.empty()) {  // common_manager.go:437-452
          PodManagerConfig cfg;
          cfg.DeletionSpec = policy.PodDeletion ? &*policy.PodDeletion : nullptr;
          cfg.DrainEnabled = drainEnabled;
          cfg.Nodes = batchNodes;
          if (Error e = PodManager->SchedulePodEviction(cfg)) return e;
        }
        break;
      case UST_STATE_DRAIN_REQUIRED:
        if (enc.evictOnDevice && drainEnabled) {
          if (i == begin) break;
          // the goroutines of ScheduleNodesDrain (drain_manager.go:98-137), as the device answered RunNodeDrain's filter
          // chain; the cordon, the eviction and the state change after them run on a worker
          if (enc.drainListError) return enc.drainListError;
          if (actuator_outcome == nullptr) return Errorf("Replay: the drain pass on the device needs actuator_outcome");
          const upgrade::DrainSpec& spec = *policy.DrainSpec;
          for (size_t k = begin; k < i; k++) {
            if (!(actions[k] & UST_A_SCHEDULE_DRAIN)) continue;
            const std::string& name = enc.entries[k]->Node->Name;
            {
              std::lock_guard<std::mutex> l(actMu_);
              if (drainingNodes_.count(name)) continue;  // "Node is already being drained, skipping" (:134-136)
            }
            const uint8_t out = actuator_outcome[k];
            if (out != UST_STATE_FAILED && out != UST_STATE_POD_RESTART_REQUIRED) return Errorf("Replay: no drain outcome for node " + name);
            // list.Pods() of GetPodsForDeletion: the selected pods the chain does not keep, in the List's order
            std::vector<Pod> toEvict;
            const auto w = enc.workload.find(k);
            if (out == UST_STATE_POD_RESTART_REQUIRED && w != enc.workload.end())
              for (size_t j = 0; j < w->second.pods.size(); j++) {
                bool isError = false;
                const uint16_t b = w->second.bits[j];
                if ((b & UST_POD_MATCH_DRAIN_SELECTOR) && !ust_pod_chain_keeps(b, spec.Force, spec.DeleteEmptyDir, &isError))
                  toEvict.push_back(*w->second.pods[j]);
              }
            // GetPodsForDeletion's errors (:121-128), as RunNodeDrain returns them
            Error filterError;
            if (out == UST_STATE_FAILED) {
              if (w != enc.workload.end()) filterError = DrainFilterError(w->second.pods, w->second.bits, spec);
              if (!filterError) filterError = Errorf("the drain filter chain reports an error");
            }
            EvictionOptions o;
            o.Force = spec.Force; o.DeleteEmptyDir = spec.DeleteEmptyDir; o.TimeoutSecond = spec.TimeoutSecond;
            upgrade::NodeUpgradeStateProvider* provider = NodeUpgradeStateProvider;
            upgrade::CordonManager* cordon = CordonManager;
            upgrade::PodEvictor* evictor = PodEvictor;
            stats_.actuator_handoffs++;
            event(*enc.entries[k]->Node, EventTypeNormal, "Scheduling drain of the node");  // :104-107
            Node node = *enc.entries[k]->Node;  // the worker's copy: it outlives this call
            handOff(&drainingNodes_, name, [provider, cordon, evictor, node, pods = std::move(toEvict), o, filterError, event]() mutable {
              if (Error e = cordon->Cordon(&node)) {  // drain.RunCordonOrUncordon (:111-118)
                (void)provider->ChangeNodeUpgradeState(&node, UpgradeStateFailed);
                event(node, EventTypeWarning, "Failed to cordon the node, " + *e);
                return;
              }
              Error err = filterError;
              if (!err && !pods.empty()) {  // DeleteOrEvictPods returns at once for no pods
                std::vector<Pod*> ptrs;
                for (Pod& p : pods) ptrs.push_back(&p);
                err = evictor ? evictor->DeleteOrEvictPods(node, ptrs, o) : Errorf("no PodEvictor");
              }
              if (err) {  // :121-127
                (void)provider->ChangeNodeUpgradeState(&node, UpgradeStateFailed);
                event(node, EventTypeWarning, "Failed to drain the node, " + *err);
              } else {    // :129-132
                event(node, EventTypeNormal, "Successfully drained the node");
                (void)provider->ChangeNodeUpgradeState(&node, UpgradeStatePodRestartRequired);
              }
            });
          }
        } else if (drainEnabled) {  // common_manager.go:346-356 (called even with an empty node list)
          DrainConfiguration cfg;
          cfg.Spec = &*policy.DrainSpec;
          cfg.Nodes = batchNodes;
          if (Error e = DrainManager->ScheduleNodesDrain(cfg)) return e;
        }
        break;
      case UST_STATE_POD_RESTART_REQUIRED:
        if (!cut)  // an abort inside the pass returns before SchedulePodsRestart (common_manager.go:462-523)
          if (Error e = PodManager->SchedulePodsRestart(restartPods)) return e;
        break;
      case UST_STATE_UNCORDON_REQUIRED: {
        // in-place flow first, then the requestor flow (upgrade_state.go:311-325)
        for (size_t k = begin; k < i; k++) {
          if (actions[k] & UST_A_UNCORDON) {
            if (Error e = CordonManager->Uncordon(enc.entries[k]->Node)) return e;
            if (Error e = setState(k)) return e;
          }
        }
        for (size_t k = begin; k < i; k++) {
          if ((actions[k] & UST_A_REQUESTOR_ANNO_CHANGE) && !(actions[k] & UST_A_UNCORDON)) {
            if (Error e = setState(k)) return e;
            if (Error e = anno(k, GetUpgradeRequestorModeAnnotationKey(), kNullString))
              return Errorf("failed to remove '" + GetUpgradeRequestorModeAnnotationKey() + "' annotation . " + *e);
            if (K8sClient != nullptr)
              if (Error e = K8sClient->DeleteOrUpdateNodeMaintenance(enc.entries[k])) return e;  // upgrade_requestor.go:482
          }
        }
      } break;
      default: break;
    }
  }
  if (abi_rc != UST_OK) return abortError(counters.error_index);
  return std::nullopt;
}

// The next deadline of the clocked call the handle just made (ust_next_deadline); nullopt when none is pending or the handle
// has none to give (the call failed).
static std::optional<int64_t> next_deadline(ust_handle* h) {
  int64_t t = INT64_MIN;
  if (ust_next_deadline(h, &t) != UST_OK || t == INT64_MIN) return std::nullopt;
  return t;
}

Error ClusterUpgradeStateManagerImpl::ApplyState(ClusterUpgradeState* currentState, const DriverUpgradePolicySpec* upgradePolicy) {
  nextTimeout_.reset();
  if (currentState == nullptr) return Errorf("currentState should not be empty");  // upgrade_state.go:175-177
  if (upgradePolicy == nullptr || !upgradePolicy->AutoUpgrade) return std::nullopt;  // upgrade_state.go:179-182
  if (handle_ == nullptr) return Errorf("no H100 device bound to this manager: ApplyState has no CPU path");
  EncodedSnapshot enc;
  if (Error e = Encode(*currentState, *upgradePolicy, &enc)) return e;
  const size_t n = enc.entries.size();
  std::vector<uint8_t> next(n + 1);
  std::vector<uint16_t> actions(n + 1);
  enc.state.push_back(0); enc.flags.push_back(0); enc.pod_rev.push_back(0); enc.ds_idx.push_back(0);  // never pass NULL for n == 0
  enc.ds_rev.push_back(0);
  int rc;
  std::vector<uint8_t> outcome(n + 1, UST_OUTCOME_NONE);
  if (enc.validateOnDevice || enc.waitOnDevice || enc.evictOnDevice) {  // Validate / the wait check / the eviction and drain
                                                                       // decisions on the device: the pods, the start times
                                                                       // and `now` go with the call
    enc.pod_flags.push_back(0); enc.start.push_back(0);
    const ust_pods pods = {enc.pod_off.data(), enc.pod_flags.data(), (int64_t)enc.pod_flags.size() - 1};
    const ust_clock clock = {enc.now, upgradePolicy->WaitForCompletion ? upgradePolicy->WaitForCompletion->TimeoutSecond : 0, enc.start.data(), nullptr};
    rc = ust_apply_state_clocked(handle_, &enc.policy, &clock, (int64_t)n, enc.state.data(), enc.flags.data(), enc.pod_rev.data(),
                                 enc.ds_idx.data(), (int32_t)enc.ds_rev.size() - 1, enc.ds_rev.data(), &pods, next.data(), actions.data(),
                                 outcome.data(), &last_);
    if (enc.validateOnDevice || enc.waitOnDevice) nextTimeout_ = next_deadline(handle_);
  } else {
    rc = ust_apply_state(handle_, &enc.policy, (int64_t)n, enc.state.data(), enc.flags.data(), enc.pod_rev.data(), enc.ds_idx.data(),
                         (int32_t)enc.ds_rev.size() - 1, enc.ds_rev.data(), nullptr, next.data(), actions.data(), nullptr, &last_);
  }
  if (rc == UST_ERR_CUDA || rc == UST_ERR_INVALID_ARGUMENT || rc == UST_ERR_NIL_STATE) return Errorf(ust_last_error(handle_));
  return Replay(enc, *upgradePolicy, next.data(), actions.data(), rc, last_, outcome.data());
}

// ---- incremental ApplyState: the resourceVersion-keyed encode cache (upgrade.hpp) --------------------------------------
void ClusterUpgradeStateManagerImpl::ResetIncremental() { cache_ = Cache(); }

int ClusterUpgradeStateManagerImpl::EvaluateCached(const ust_policy& policy, bool full, const std::vector<int64_t>& changed,
                                                   Cache* cache, ust_counters* c) {
  Cache& k = *cache;
  const size_t n = k.slots.size();
  if (handle_ == nullptr) return UST_ERR_CUDA;
  // never pass NULL for empty arrays
  std::vector<int32_t> dsrev = k.ds_rev;
  dsrev.push_back(0);
  if (full) {
    k.next.assign(n + 1, 0);
    k.actions.assign(n + 1, 0);
    std::vector<uint8_t> st = k.state; st.push_back(0);
    std::vector<uint32_t> fl = k.flags; fl.push_back(0);
    std::vector<int32_t> rv = k.pod_rev; rv.push_back(0);
    std::vector<int32_t> di = k.ds_idx; di.push_back(0);
    return ust_apply_state(handle_, &policy, (int64_t)n, st.data(), fl.data(), rv.data(), di.data(), (int32_t)k.ds_rev.size(),
                           dsrev.data(), nullptr, k.next.data(), k.actions.data(), nullptr, c);
  }
  const size_t m = changed.size();
  std::vector<uint8_t> st(m + 1);
  std::vector<uint32_t> fl(m + 1);
  std::vector<int32_t> rv(m + 1), di(m + 1);
  std::vector<int64_t> ix(changed);
  ix.push_back(0);
  for (size_t j = 0; j < m; j++) {
    const size_t i = (size_t)changed[j];
    st[j] = k.state[i]; fl[j] = k.flags[i]; rv[j] = k.pod_rev[i]; di[j] = k.ds_idx[i];
  }
  // nodes that joined: their columns from the cache, at the positions the splice / reorder gives them
  const Cache::Splice& ps = k.pending;
  const size_t ni = ps.insert_at.size();
  std::vector<uint8_t> ist(ni + 1);
  std::vector<uint32_t> ifl(ni + 1);
  std::vector<int32_t> irv(ni + 1), idi(ni + 1);
  for (size_t j = 0; j < ni; j++) {
    const size_t i = (size_t)ps.insert_at[j];
    ist[j] = k.state[i]; ifl[j] = k.flags[i]; irv[j] = k.pod_rev[i]; idi[j] = k.ds_idx[i];
  }
  const ust_splice splice = {(int64_t)ps.remove_idx.size(), ps.remove_idx.data(), (int64_t)ni, ps.insert_before.data(),
                             ist.data(), ifl.data(), irv.data(), idi.data()};
  const ust_reorder reorder = {(int64_t)ps.run_src.size(), ps.run_src.data(), ps.run_len.data(), (int64_t)ni,
                               ist.data(), ifl.data(), irv.data(), idi.data()};
  const int64_t cap = (int64_t)(n / 4 + 1024);
  std::vector<int64_t> oi((size_t)cap + 1);
  std::vector<uint8_t> on((size_t)cap + 1);
  std::vector<uint16_t> oa((size_t)cap + 1);
  int64_t n_out = 0;
  int rc = ps.run_src.empty()
               ? ust_apply_state_delta_splice(handle_, &policy, ps.empty() ? nullptr : &splice, (int64_t)m, ix.data(), st.data(), fl.data(),
                                              rv.data(), di.data(), (int32_t)k.ds_rev.size(), dsrev.data(), cap, oi.data(), on.data(),
                                              oa.data(), &n_out, c)
               : ust_apply_state_delta_reorder(handle_, &policy, &reorder, (int64_t)m, ix.data(), st.data(), fl.data(), rv.data(),
                                               di.data(), (int32_t)k.ds_rev.size(), dsrev.data(), cap, oi.data(), on.data(), oa.data(),
                                               &n_out, c);
  if (rc == UST_ERR_CUDA || rc == UST_ERR_INVALID_ARGUMENT || rc == UST_ERR_COMM) return rc;
  if (n_out > cap) {
    // More changed outputs than the arrays hold: nothing was written to them. That is UST_ERR_TRUNCATED, or a
    // reference-level abort, which keeps its own code. Either way the call's full outputs are resident: fetch them all.
    stats_.outputs_received += (int64_t)n;
    const int frc = ust_fetch_outputs(handle_, k.next.data(), k.actions.data());
    if (frc != UST_OK) return frc;
    return rc == UST_ERR_TRUNCATED ? UST_OK : rc;
  }
  for (int64_t j = 0; j < n_out; j++) { k.next[(size_t)oi[(size_t)j]] = on[(size_t)j]; k.actions[(size_t)oi[(size_t)j]] = oa[(size_t)j]; }
  stats_.outputs_received += n_out;
  return rc;
}

int ClusterUpgradeStateManagerImpl::EvaluateCachedPods(const ust_policy& policy, int64_t now, int64_t waitTimeout, bool full,
                                                       const std::vector<int64_t>& changed, Cache* cache, ust_counters* c) {
  Cache& k = *cache;
  const size_t n = k.slots.size();
  cachedDeadline_.reset();
  if (handle_ == nullptr) return UST_ERR_CUDA;
  // never pass NULL for empty arrays
  std::vector<int32_t> dsrev = k.ds_rev;
  dsrev.push_back(0);
  std::vector<int32_t> off;
  std::vector<uint16_t> pf;
  auto csr = [&](size_t m, const int64_t* rows) {  // the lists of `rows` (nullptr: every slot) as one CSR
    off.assign(m + 1, 0);
    for (size_t j = 0; j < m; j++) {
      const auto& l = k.lists[rows ? (size_t)rows[j] : j];
      pf.insert(pf.end(), l.begin(), l.end());
      off[j + 1] = (int32_t)pf.size();
    }
    pf.push_back(0);
  };
  if (full) {
    k.next.assign(n + 1, 0);
    k.actions.assign(n + 1, 0);
    k.outcome.assign(n + 1, UST_OUTCOME_NONE);
    std::vector<uint8_t> st = k.state; st.push_back(0);
    std::vector<uint32_t> fl = k.flags; fl.push_back(0);
    std::vector<int32_t> rv = k.pod_rev; rv.push_back(0);
    std::vector<int32_t> di = k.ds_idx; di.push_back(0);
    std::vector<int64_t> sv = k.start; sv.push_back(0);
    csr(n, nullptr);
    const ust_pods pods = {off.data(), pf.data(), (int64_t)pf.size() - 1};
    const ust_clock clock = {now, waitTimeout, sv.data(), nullptr};
    const int rc = ust_apply_state_clocked(handle_, &policy, &clock, (int64_t)n, st.data(), fl.data(), rv.data(), di.data(),
                                           (int32_t)k.ds_rev.size(), dsrev.data(), &pods, k.next.data(), k.actions.data(),
                                           k.outcome.data(), c);
    cachedDeadline_ = next_deadline(handle_);
    return rc;
  }
  const size_t m = changed.size();
  std::vector<uint8_t> st(m + 1);
  std::vector<uint32_t> fl(m + 1);
  std::vector<int32_t> rv(m + 1), di(m + 1);
  std::vector<int64_t> sv(m + 1), ix(changed);
  ix.push_back(0);
  for (size_t j = 0; j < m; j++) {
    const size_t i = (size_t)changed[j];
    st[j] = k.state[i]; fl[j] = k.flags[i]; rv[j] = k.pod_rev[i]; di[j] = k.ds_idx[i]; sv[j] = k.start[i];
  }
  // nodes that joined: their columns and start times from the cache, at the positions the runs give them
  const Cache::Splice& ps = k.pending;
  const size_t ni = ps.insert_at.size();
  std::vector<uint8_t> ist(ni + 1);
  std::vector<uint32_t> ifl(ni + 1);
  std::vector<int32_t> irv(ni + 1), idi(ni + 1);
  std::vector<int64_t> isv(ni + 1);
  for (size_t j = 0; j < ni; j++) {
    const size_t i = (size_t)ps.insert_at[j];
    ist[j] = k.state[i]; ifl[j] = k.flags[i]; irv[j] = k.pod_rev[i]; idi[j] = k.ds_idx[i]; isv[j] = k.start[i];
  }
  const ust_reorder reorder = {(int64_t)ps.run_src.size(), ps.run_src.data(), ps.run_len.data(), (int64_t)ni,
                               ist.data(), ifl.data(), irv.data(), idi.data()};
  std::vector<int64_t> li(k.listChanged);
  li.push_back(0);
  csr(k.listChanged.size(), k.listChanged.data());
  const ust_pod_lists lists = {(int64_t)k.listChanged.size(), li.data(), off.data(), pf.data(), (int64_t)pf.size() - 1};
  const ust_clock clock = {now, waitTimeout, sv.data(), isv.data()};
  const int64_t cap = (int64_t)(n / 4 + 1024);
  std::vector<int64_t> oi((size_t)cap + 1);
  std::vector<uint8_t> on((size_t)cap + 1), oo((size_t)cap + 1);
  std::vector<uint16_t> oa((size_t)cap + 1);
  int64_t n_out = 0;
  const int rc = ust_apply_state_delta_pods_clocked(handle_, &policy, &clock, ps.empty() ? nullptr : &reorder,
                                                    k.listChanged.empty() ? nullptr : &lists, (int64_t)m, ix.data(), st.data(), fl.data(),
                                                    rv.data(), di.data(), (int32_t)k.ds_rev.size(), dsrev.data(), cap, oi.data(), on.data(),
                                                    oa.data(), oo.data(), &n_out, c);
  if (rc == UST_ERR_CUDA || rc == UST_ERR_INVALID_ARGUMENT || rc == UST_ERR_COMM) return rc;
  cachedDeadline_ = next_deadline(handle_);
  if (n_out > cap) {  // UST_ERR_TRUNCATED or a reference-level abort with more outputs than the arrays hold: fetch them all
    stats_.outputs_received += (int64_t)n;
    k.next.resize(n + 1);
    k.actions.resize(n + 1);
    k.outcome.resize(n + 1, UST_OUTCOME_NONE);
    const int frc = ust_fetch_outputs_pods(handle_, k.next.data(), k.actions.data(), k.outcome.data());
    if (frc != UST_OK) return frc;
    return rc == UST_ERR_TRUNCATED ? UST_OK : rc;
  }
  for (int64_t j = 0; j < n_out; j++) {
    const size_t i = (size_t)oi[(size_t)j];
    k.next[i] = on[(size_t)j]; k.actions[i] = oa[(size_t)j]; k.outcome[i] = oo[(size_t)j];
  }
  stats_.outputs_received += n_out;
  return rc;
}

Error ClusterUpgradeStateManagerImpl::ApplyStateIncremental(ClusterUpgradeState* currentState, const DriverUpgradePolicySpec* upgradePolicy) {
  nextTimeout_.reset();
  if (currentState == nullptr) return Errorf("currentState should not be empty");  // upgrade_state.go:175-177
  if (upgradePolicy == nullptr || !upgradePolicy->AutoUpgrade) return std::nullopt;  // upgrade_state.go:179-182
  ust_policy pol;
  flatten_policy(*upgradePolicy, podDeletionStateEnabled_, validationStateEnabled_, opts_.Requestor.UseMaintenanceOperator, &pol);
  Cache& k = cache_;
  stats_.reconciles++;
  // ValidateOnDevice / WaitForCompletionOnDevice: the cache holds the clocked pod-list snapshot; a change of mode starts
  // it over
  const bool val = validateOnDevice(), wait = waitOnDevice(*upgradePolicy), evict = evictOnDevice(*upgradePolicy);
  const bool dev = val || wait || evict;
  if (k.valid && (k.validation != val || k.wait != wait || k.evict != evict)) ResetIncremental();
  k.pods = dev; k.validation = val; k.wait = wait; k.evict = evict;
  int64_t now = 0;
  PodsByNode byNode, waitByNode;
  Error listErr, waitListErr, evictListErr;
  WorkloadLists wl;
  std::string workPolicy;  // what the workload bits depend on besides the pods: which passes, the drain's selector
  if (evict) {
    listWorkload(K8sClient, *upgradePolicy, evictPodDeletion(*upgradePolicy) ? &filter_ : nullptr, evictDrain(*upgradePolicy), &wl);
    evictListErr = wl.podsError ? wl.podsError : wl.dsError;
    workPolicy = std::string(wl.filter ? "F" : "-") + (wl.drain ? "D" + upgradePolicy->DrainSpec->PodSelector : "-") + "|";
  }
  if (dev) {
    pol.evaluate_actuators = UST_EVAL_ACTUATORS | (val ? UST_EVAL_VALIDATION : 0);
    now = opts_.Now();
    if (val) listErr = listPodsBySelector(K8sClient, validationSelector_, "validation", &byNode);
    if (wait) waitListErr = listPodsBySelector(K8sClient, upgradePolicy->WaitForCompletion->PodSelector, "wait-for-completion", &waitByNode);
  }
  const bool full = !k.valid;
  for (auto& sl : k.slots) sl.seen = false;
  // the DaemonSet table: identities are cached by UID, revision hashes are looked up once per DaemonSet per reconcile
  std::map<const DaemonSet*, int32_t> dsOf;
  auto dsIndexOf = [&](const DaemonSet* d) -> int32_t {
    auto it = dsOf.find(d);
    if (it != dsOf.end()) return it->second;
    auto ins = k.dsIndexByUID.emplace(d->UID, (int32_t)k.dsIndexByUID.size());
    const int32_t idx = ins.first->second;
    if ((size_t)idx >= k.ds_rev.size()) { k.ds_rev.resize((size_t)idx + 1, 0); k.dsHashError.resize((size_t)idx + 1, false); }
    std::string dsHash;
    const bool bad = (bool)PodManager->GetDaemonsetControllerRevisionHash(d, &dsHash);
    k.ds_rev[(size_t)idx] = bad ? 0 : k.intern.emplace(dsHash, (int32_t)k.intern.size() + 1).first->second;
    k.dsHashError[(size_t)idx] = bad;
    dsOf.emplace(d, idx);
    return idx;
  };
  std::vector<int64_t> changed;
  // Slots follow BuildState's list order (NodeUpgradeState::ListIndex), of which every bucket's slice order is a
  // subsequence; entries without a ListIndex take their position in the bucket walk instead. The slots move to this
  // reconcile's order: a node the cache has not seen joins at its position, a cached slot no entry names has left, and a
  // cached node that changed its position moves with its slot (a driver pod re-created under a new name moves its node
  // in a list sorted by name).
  std::vector<const NodeUpgradeState*> order;
  {
    std::vector<std::pair<int64_t, const NodeUpgradeState*>> listed;
    bool haveIndex = true;
    auto collect = [&](const std::vector<NodeUpgradeState*>& v) {
      for (const NodeUpgradeState* ns : v) { haveIndex = haveIndex && ns->ListIndex >= 0; listed.emplace_back(ns->ListIndex, ns); }
    };
    for (int code : kPassOrder) {
      auto it = currentState->NodeStates.find(kStateNames[code]);
      if (it != currentState->NodeStates.end()) collect(it->second);
    }
    for (const auto& kv : currentState->NodeStates) {
      const int code = StateCodeOfLabel(kv.first);
      if (code == UST_STATE_OTHER || code == UST_STATE_POST_MAINTENANCE_REQUIRED) collect(kv.second);
    }
    if (haveIndex) std::stable_sort(listed.begin(), listed.end(), [](const auto& x, const auto& y) { return x.first < y.first; });
    order.reserve(listed.size());
    for (const auto& l : listed) order.push_back(l.second);
  }
  // The new slot order: per position the old slot it takes, or -1 for a node that joins. The same change is kept for the
  // device (Cache::pending): a splice while the surviving slots keep their relative order, else runs of a reorder.
  const size_t nOld = k.slots.size();
  std::vector<int64_t> from;
  from.reserve(order.size());
  std::vector<char> present(nOld, 0);
  Cache::Splice sp;
  bool moved = false;
  long long lastSlot = -1;
  for (const NodeUpgradeState* ns : order) {
    auto it = k.idOf.find(ns->Node->Name);
    if (it == k.idOf.end()) {  // joins right after the last cached slot before it
      sp.insert_before.push_back(lastSlot + 1);
      sp.insert_at.push_back((int64_t)from.size());
      from.push_back(-1);
      continue;
    }
    const size_t slot = k.slotOfId[it->second];
    if (present[slot]) { ResetIncremental(); return Errorf("node " + ns->Node->Name + " appears twice in the snapshot"); }
    present[slot] = 1;
    moved = moved || (long long)slot < lastSlot;
    lastSlot = (long long)slot;
    from.push_back((int64_t)slot);
  }
  for (size_t i = 0; i < nOld; i++)
    if (!present[i]) sp.remove_idx.push_back((int64_t)i);
  if (moved || (dev && !sp.empty())) {  // maximal runs of consecutive old slots, joins as inserted runs (the pod-list calls
                                        // take no splice)
    sp.insert_before.clear();
    orderRuns(from, &sp.run_src, &sp.run_len);
  }
  // The host arrays move to the new order (linear). Joined slots start empty and are encoded by the walk below.
  std::vector<char> joined;
  if (!sp.empty()) {
    for (int64_t i : sp.remove_idx) {  // the node left: its name and id go, its entries are not carried over
      k.idOf.erase(k.slots[(size_t)i].name);
      k.freeIds.push_back(k.slots[(size_t)i].id);
    }
    const size_t nNew = from.size();
    Cache nk;
    nk.slots.reserve(nNew); nk.state.reserve(nNew); nk.flags.reserve(nNew); nk.pod_rev.reserve(nNew); nk.ds_idx.reserve(nNew);
    nk.next.reserve(nNew); nk.actions.reserve(nNew); nk.deferredMsg.reserve(nNew);
    if (dev) nk.outcome.reserve(nNew);
    joined.assign(nNew, 0);
    for (size_t p = 0; p < nNew; p++) {
      if (from[p] < 0) {
        const std::string& name = order[p]->Node->Name;
        size_t id = k.slotOfId.size();
        if (!k.freeIds.empty()) { id = k.freeIds.back(); k.freeIds.pop_back(); } else k.slotOfId.push_back(0);
        if (!k.idOf.emplace(name, id).second) { ResetIncremental(); return Errorf("node " + name + " appears twice in the snapshot"); }
        joined[p] = 1;
        nk.slots.emplace_back();
        nk.slots.back().name = name;
        nk.slots.back().id = id;
        nk.state.push_back(UST_STATE_EXCLUDED); nk.flags.push_back(0); nk.pod_rev.push_back(0); nk.ds_idx.push_back(-1);
        nk.next.push_back(0); nk.actions.push_back(0); nk.deferredMsg.emplace_back();
        if (dev) {
          nk.lists.emplace_back(); nk.listSig.emplace_back("\x01"); nk.start.push_back(0);
          nk.nval.push_back(0); nk.waitSig.emplace_back("\x01"); nk.outcome.push_back(UST_OUTCOME_NONE);
          nk.nwork.push_back(0); nk.workSig.emplace_back("\x01");
        }
        continue;
      }
      const size_t q = (size_t)from[p];
      nk.slots.push_back(std::move(k.slots[q]));
      nk.state.push_back(k.state[q]); nk.flags.push_back(k.flags[q]); nk.pod_rev.push_back(k.pod_rev[q]); nk.ds_idx.push_back(k.ds_idx[q]);
      nk.next.push_back(q < k.next.size() ? k.next[q] : 0); nk.actions.push_back(q < k.actions.size() ? k.actions[q] : 0);
      nk.deferredMsg.push_back(std::move(k.deferredMsg[q]));
      if (dev) {
        nk.lists.push_back(std::move(k.lists[q])); nk.listSig.push_back(std::move(k.listSig[q])); nk.start.push_back(k.start[q]);
        nk.nval.push_back(k.nval[q]); nk.waitSig.push_back(std::move(k.waitSig[q]));
        nk.nwork.push_back(k.nwork[q]); nk.workSig.push_back(std::move(k.workSig[q]));
        nk.outcome.push_back(q < k.outcome.size() ? k.outcome[q] : UST_OUTCOME_NONE);
      }
    }
    k.slots.swap(nk.slots); k.state.swap(nk.state); k.flags.swap(nk.flags); k.pod_rev.swap(nk.pod_rev); k.ds_idx.swap(nk.ds_idx);
    k.next.swap(nk.next); k.actions.swap(nk.actions); k.deferredMsg.swap(nk.deferredMsg);
    k.lists.swap(nk.lists); k.listSig.swap(nk.listSig); k.start.swap(nk.start);
    k.nval.swap(nk.nval); k.waitSig.swap(nk.waitSig); k.outcome.swap(nk.outcome);
    k.nwork.swap(nk.nwork); k.workSig.swap(nk.workSig);
    for (size_t i = 0; i < k.slots.size(); i++) k.slotOfId[k.slots[i].id] = i;
  }
  if (!full) {
    stats_.inserted += (int64_t)sp.insert_at.size();
    stats_.removed += (int64_t)sp.remove_idx.size();
    stats_.reorders += moved ? 1 : 0;
  }
  k.pending = full ? Cache::Splice() : std::move(sp);
  stats_.slots = (int64_t)k.slots.size();
  // this reconcile's view in pass order (what Replay walks): entry, its slot
  EncodedSnapshot view;
  view.policy = pol;
  view.validateOnDevice = val;
  view.waitOnDevice = wait;
  view.now = now;
  view.listError = listErr;
  view.waitListError = waitListErr;
  view.evictOnDevice = evict;
  view.evictListError = evictListErr;
  view.drainListError = evictListErr ? evictListErr : wl.selectorError;
  std::vector<char> sendList(dev ? k.slots.size() : 0, 0);
  std::vector<size_t> slotOfView;
  bool orderBroken = false;
  auto visit = [&](NodeUpgradeState* ns, int code) -> Error {
    const Node& n = *ns->Node;
    const size_t i = k.slotOfId[k.idOf.at(n.Name)];
    Cache::Slot& sl = k.slots[i];
    if (sl.seen) return Errorf("node " + n.Name + " appears twice in the snapshot");
    sl.seen = true;
    int32_t ds = -1;
    bool dsErr = false;
    if (!ns->IsOrphanedPod()) { ds = dsIndexOf(ns->DriverDaemonSet); dsErr = k.dsHashError[(size_t)ds]; }
    // everything the encoding of the entry depends on
    const bool versioned = !n.ResourceVersion.empty() && (ns->DriverPod == nullptr || !ns->DriverPod->ResourceVersion.empty());
    std::string sig = std::to_string(code) + "|" + n.ResourceVersion + "|" + (ns->DriverPod ? ns->DriverPod->ResourceVersion : "-") + "|" +
                      std::to_string(ds) + (dsErr ? "!" : "") + "|" + std::to_string(ds >= 0 ? k.ds_rev[(size_t)ds] : 0) + "|" +
                      (ns->NodeMaintenance ? (ns->NodeMaintenance->ReadyConditionWithReasonReady ? "R" : "P") : "-");
    if (!versioned || sig != sl.sig || sl.code != code) {
      uint8_t hot; uint32_t f; int32_t rev; std::string deferred;
      int64_t start = 0;
      if (Error err = encodeOne(ns, code, ds, dsErr, &k.intern, k.ds_rev, &hot, &f, &rev, &deferred, dev ? &start : nullptr, val, wait))
        return err;
      stats_.encoded++;
      if (hot != k.state[i] || f != k.flags[i] || rev != k.pod_rev[i] || ds != k.ds_idx[i] || (dev && start != k.start[i])) {
        k.state[i] = hot; k.flags[i] = f; k.pod_rev[i] = rev; k.ds_idx[i] = ds;
        if (dev) k.start[i] = start;
        if (joined.empty() || !joined[i]) changed.push_back((int64_t)i);  // a joined node travels with the splice / reorder
      }
      k.deferredMsg[i] = deferred;
      sl.sig = versioned ? sig : std::string();
      sl.code = code;
    } else {
      stats_.reused++;
    }
    if (dev) {
      // the node's list, validation pods first, then wait-selector pods, then workload pods: each part is rebuilt when its
      // (pod, resourceVersion) sequence changed, and the list is sent when its bits did (or the node joined: an inserted
      // node brings its list). After a failed List that part stays as it is.
      const bool joinedNode = !joined.empty() && joined[i];
      auto refresh = [&](const PodsByNode& by, std::string* sigStore, uint16_t (*flagsOf)(const Pod&), std::vector<uint16_t>* half) {
        const std::vector<const Pod*>* pods = podsOf(by, n.Name);
        std::string lsig;
        bool lversioned = true;
        if (pods)
          for (const Pod* p : *pods) {
            lversioned = lversioned && !p->ResourceVersion.empty();
            lsig += p->Namespace + "/" + p->Name + "@" + p->ResourceVersion + ";";
          }
        if (lversioned && lsig == *sigStore) return false;
        half->clear();
        if (pods)
          for (const Pod* p : *pods) half->push_back(flagsOf(*p));
        *sigStore = lversioned ? lsig : std::string("\x01");
        return true;
      };
      std::vector<uint16_t>& list = k.lists[i];
      std::vector<uint16_t> vhalf, whalf, ahalf;
      const bool newV = val && !listErr && refresh(byNode, &k.listSig[i], validationPodFlags, &vhalf);
      const bool newW = wait && !waitListErr && refresh(waitByNode, &k.waitSig[i], waitPodFlags, &whalf);
      // the workload part: every pod of a pod-deletion-required or drain-required node, nothing for any other node. Its
      // bits also depend on whether the DaemonSet each pod's controller names exists, and on the policy; after a failed
      // drain-selector List the part is rebuilt (its drain bits unknown: that pass returns the error) and again next time.
      const bool workNode = evict && (code == UST_STATE_POD_DELETION_REQUIRED || code == UST_STATE_DRAIN_REQUIRED);
      const std::vector<const Pod*>* work = workNode && !evictListErr ? podsOf(wl.byNode, n.Name) : nullptr;
      bool newA = false;
      if (evict && !evictListErr) {
        std::string asig = workNode ? workPolicy : std::string();
        bool aversioned = !wl.selectorError;
        if (work)
          for (const Pod* p : *work) {
            aversioned = aversioned && !p->ResourceVersion.empty();
            const OwnerReference* c = controllerOf(*p);
            const bool dsMissing = c && c->Kind == "DaemonSet" && !wl.daemonSets.count(p->Namespace + "/" + c->Name);
            asig += p->Namespace + "/" + p->Name + "@" + p->ResourceVersion + (dsMissing ? "!;" : ";");
          }
        if (!aversioned || asig != k.workSig[i]) {
          newA = true;
          if (work)
            for (const Pod* p : *work) ahalf.push_back(workloadPodFlags(*p, wl));
          k.workSig[i] = aversioned ? asig : std::string("\x01");
        }
      }
      if (newV || newW || newA) {
        const size_t nv0 = (size_t)k.nval[i], na0 = (size_t)k.nwork[i];
        if (!newV) vhalf.assign(list.begin(), list.begin() + nv0);
        if (!newW) whalf.assign(list.begin() + nv0, list.end() - na0);
        if (!newA) ahalf.assign(list.end() - na0, list.end());
        const int32_t nv = (int32_t)vhalf.size(), na = (int32_t)ahalf.size();
        vhalf.insert(vhalf.end(), whalf.begin(), whalf.end());
        vhalf.insert(vhalf.end(), ahalf.begin(), ahalf.end());
        if (vhalf != list) { list.swap(vhalf); sendList[i] = 1; }
        k.nval[i] = nv;
        k.nwork[i] = na;
      }
      if (joinedNode) sendList[i] = 1;
      if (val && code == UST_STATE_VALIDATION_REQUIRED) stats_.validate_avoided++;
      if (wait && code == UST_STATE_WAIT_FOR_JOBS_REQUIRED) stats_.wait_avoided++;
      if ((code == UST_STATE_POD_DELETION_REQUIRED && evictPodDeletion(*upgradePolicy)) ||
          (code == UST_STATE_DRAIN_REQUIRED && evictDrain(*upgradePolicy)))
        stats_.evict_lists_avoided++;
      // Replay reads the node's workload pods beside the bits the device holds for them: the same sequence of pods
      if (work && work->size() == (size_t)k.nwork[i]) {
        EncodedSnapshot::Workload& wk = view.workload[view.entries.size()];
        wk.pods = *work;
        wk.bits.assign(list.end() - k.nwork[i], list.end());
      }
    }
    if (!slotOfView.empty() && (int)(view.state.back() & UST_HOT_STATE_MASK) == code && slotOfView.back() > i)
      orderBroken = true;  // within a bucket, slot order must be the slice order: slots are handed out in it
                           // (upgrade_inplace.go:71) and the first error in it ends the pass
    view.entries.push_back(ns);
    view.state.push_back(k.state[i]);
    slotOfView.push_back(i);
    return std::nullopt;
  };
  Error walkErr;
  for (int code : kPassOrder) {
    auto it = currentState->NodeStates.find(kStateNames[code]);
    if (it == currentState->NodeStates.end()) continue;
    for (NodeUpgradeState* ns : it->second)
      if ((walkErr = visit(ns, code))) break;
    if (walkErr) break;
  }
  if (!walkErr)
    for (const auto& kv : currentState->NodeStates) {
      const int code = StateCodeOfLabel(kv.first);
      if (code != UST_STATE_OTHER && code != UST_STATE_POST_MAINTENANCE_REQUIRED) continue;
      for (NodeUpgradeState* ns : kv.second)
        if ((walkErr = visit(ns, code))) break;
      if (walkErr) break;
    }
  if (walkErr) { ResetIncremental(); return walkErr; }
  if (orderBroken) {  // the slots follow the list order: a bucket whose slice order contradicts it is inconsistent input
    ResetIncremental();
    return Errorf("incremental ApplyState: a bucket's slice order contradicts the list order");
  }
  std::sort(changed.begin(), changed.end());
  if (full) stats_.full_uploads++;
  int rc;
  if (dev) {
    k.listChanged.clear();
    for (size_t i = 0; i < sendList.size(); i++)
      if (full || sendList[i]) k.listChanged.push_back((int64_t)i);
    stats_.lists_sent += (int64_t)k.listChanged.size();
    stats_.lists_reused += (int64_t)(k.slots.size() - k.listChanged.size());
    if (!full && changed.empty() && k.listChanged.empty() && k.pending.empty()) stats_.time_only++;
    cachedDeadline_.reset();
    rc = EvaluateCachedPods(pol, now, upgradePolicy->WaitForCompletion ? upgradePolicy->WaitForCompletion->TimeoutSecond : 0, full, changed,
                            &k, &last_);
    if (val || wait) nextTimeout_ = cachedDeadline_;
  } else {
    rc = EvaluateCached(pol, full, changed, &k, &last_);
  }
  if (rc == UST_ERR_CUDA || rc == UST_ERR_INVALID_ARGUMENT || rc == UST_ERR_NIL_STATE || rc == UST_ERR_COMM) {
    ResetIncremental();
    return Errorf(handle_ ? ust_last_error(handle_) : "no H100 device bound to this manager: ApplyState has no CPU path");
  }
  k.valid = true;
  // Replay walks this reconcile's view: gather its outputs, translate the abort position
  const size_t nv = view.entries.size();
  std::vector<uint8_t> next(nv + 1), outcome(nv + 1, UST_OUTCOME_NONE);
  std::vector<uint16_t> actions(nv + 1);
  if (wait) view.waitRunning.assign(nv, 0);
  ust_counters c = last_;
  for (size_t v = 0; v < nv; v++) {
    const size_t i = slotOfView[v];
    next[v] = k.next[i];
    actions[v] = k.actions[i];
    if (dev) outcome[v] = k.outcome[i];
    if (wait && (view.state[v] & UST_HOT_STATE_MASK) == UST_STATE_WAIT_FOR_JOBS_REQUIRED) {
      const std::vector<uint16_t>& l = k.lists[i];  // the list the device holds for the node
      view.waitRunning[v] = anyWaitRunning(l.data() + k.nval[i], l.data() + l.size() - k.nwork[i]);
    }
    if (!k.deferredMsg[i].empty()) view.deferred[v] = k.deferredMsg[i];
    if (last_.error_index == (int64_t)i) c.error_index = (int64_t)v;
  }
  return Replay(view, *upgradePolicy, next.data(), actions.data(), rc, c, outcome.data());
}

}  // namespace upgrade
