// upgrade.hpp — host-side mirror of github.com/NVIDIA/k8s-operator-libs/pkg/upgrade for the ApplyState /
// BuildState path, written in C++ because the build image has no Go toolchain (DESIGN.md §1). Names, argument
// meaning and error behaviour follow the reference so that callers (and tests) read like the Go:
//
//   ClusterUpgradeStateManager      pkg/upgrade/upgrade_state.go:35-53
//   CommonUpgradeStateManager       pkg/upgrade/common_manager.go:23-41
//   NodeUpgradeState / ClusterUpgradeState   common_manager.go:58-80
//   UpgradeState* constants, key getters     consts.go:19-93, util.go:91-155
//   DriverUpgradePolicySpec & sub-specs      api/upgrade/v1alpha1/upgrade_spec.go:27-110
//   actuator interfaces: NodeUpgradeStateProvider (node_upgrade_state_provider.go:33-37), CordonManager
//   (cordon_manager.go:33-36), DrainManager (drain_manager.go:48-50), PodManager (pod_manager.go:53-60),
//   ValidationManager (validation_manager.go:48-50), SafeDriverLoadManager (safe_driver_load_manager.go:74-79)
//
// Decisions are NOT made here: ApplyState encodes the snapshot into the struct-of-arrays of include/ust.h, calls
// ust_apply_state (H100 kernel) and replays the returned per-node action bitmasks through the actuator interfaces
// in the reference's pass order. Without libust.so / a H100 every ApplyState returns an error.
#pragma once
#include <condition_variable>
#include <cstdint>
#include <ctime>
#include <deque>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <optional>
#include <set>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../../include/ust.h"

namespace upgrade {

// ---- errors: Go's `error` ---------------------------------------------------------------------------
using Error = std::optional<std::string>;  // nullopt == nil
inline Error Errorf(std::string s) { return Error(std::move(s)); }

// ---- consts.go:49-82 ----------------------------------------------------------------------------------
extern const char* const UpgradeStateUnknown;
extern const char* const UpgradeStateUpgradeRequired;
extern const char* const UpgradeStateCordonRequired;
extern const char* const UpgradeStateWaitForJobsRequired;
extern const char* const UpgradeStatePodDeletionRequired;
extern const char* const UpgradeStateDrainRequired;
extern const char* const UpgradeStateNodeMaintenanceRequired;
extern const char* const UpgradeStatePostMaintenanceRequired;
extern const char* const UpgradeStatePodRestartRequired;
extern const char* const UpgradeStateValidationRequired;
extern const char* const UpgradeStateUncordonRequired;
extern const char* const UpgradeStateDone;
extern const char* const UpgradeStateFailed;
extern const char* const PodControllerRevisionHashLabelKey;  // pod_manager.go:72

// util.go:91-155
void SetDriverName(const std::string& driver);
std::string GetUpgradeStateLabelKey();
std::string GetUpgradeSkipNodeLabelKey();
std::string GetUpgradeDriverWaitForSafeLoadAnnotationKey();
std::string GetUpgradeRequestedAnnotationKey();
std::string GetUpgradeRequestorModeAnnotationKey();
std::string GetUpgradeInitialStateAnnotationKey();
std::string GetWaitForPodCompletionStartTimeAnnotationKey();
std::string GetValidationStartTimeAnnotationKey();
// util.go:158-160: strings.ToUpper(DriverName) + "DriverUpgrade", the reason of every event the managers record. Driver
// names are ASCII (they are label-key prefixes), so ASCII upper-casing is Go's ToUpper here.
std::string GetEventReason();

// ---- the slice of corev1 / appsv1 the path reads --------------------------------------------------------
using StringMap = std::map<std::string, std::string>;
struct NodeCondition { std::string Type, Status; };
struct Node {
  std::string Name;
  std::string ResourceVersion;           // metadata.resourceVersion ("" = unknown: the object is re-encoded every reconcile)
  StringMap Labels, Annotations;
  bool Unschedulable = false;            // Spec.Unschedulable
  std::vector<NodeCondition> Conditions;  // Status.Conditions
};
struct ContainerStatus { bool Ready = false; int RestartCount = 0; };
struct OwnerReference { std::string Kind, Name, UID; bool Controller = false; };  // Controller: *Controller == true
struct Pod {
  std::string Name, Namespace, NodeName;  // Spec.NodeName
  std::string ResourceVersion;
  StringMap Labels;
  std::vector<OwnerReference> OwnerReferences;
  std::string Phase;                      // Status.Phase
  std::vector<ContainerStatus> ContainerStatuses, InitContainerStatuses;
  bool DeletionTimestampSet = false;      // !DeletionTimestamp.IsZero()
  StringMap Annotations;
  bool HasEmptyDirVolume = false;         // a Spec.Volumes entry with EmptyDir != nil
};
struct DaemonSet {
  std::string Name, Namespace, UID;
  std::string ResourceVersion;
  int DesiredNumberScheduled = 0;         // Status.DesiredNumberScheduled
};
struct NodeMaintenance {                   // maintenance-operator api v0.3.0, the fields the path reads
  std::string Name;
  bool ReadyConditionWithReasonReady = false;  // upgrade_requestor.go:437-439
};
bool IsOrphanedPod(const Pod& pod);        // common_manager.go:223-225
bool IsNodeInRequestorMode(const Node& node);  // util.go:135-138

// ---- api/upgrade/v1alpha1 --------------------------------------------------------------------------------
struct IntOrString {
  enum Kind { Int, String } Type = Int;
  int64_t IntVal = 0;
  std::string StrVal;
  static IntOrString FromInt(int64_t v) { IntOrString x; x.Type = Int; x.IntVal = v; return x; }
  static IntOrString FromString(std::string s) { IntOrString x; x.Type = String; x.StrVal = std::move(s); return x; }
};
struct WaitForCompletionSpec { std::string PodSelector; int TimeoutSecond = 0; };
struct PodDeletionSpec { bool Force = false; int TimeoutSecond = 300; bool DeleteEmptyDir = false; };
struct DrainSpec { bool Enable = false, Force = false; std::string PodSelector; int TimeoutSecond = 300; bool DeleteEmptyDir = false; };
struct DriverUpgradePolicySpec {
  bool AutoUpgrade = false;
  int64_t MaxParallelUpgrades = 0;
  std::optional<IntOrString> MaxUnavailable;
  std::optional<PodDeletionSpec> PodDeletion;
  std::optional<WaitForCompletionSpec> WaitForCompletion;
  std::optional<upgrade::DrainSpec> DrainSpec;
};

// ---- common_manager.go:58-80 ------------------------------------------------------------------------------
struct NodeUpgradeState {
  upgrade::Node* Node = nullptr;
  Pod* DriverPod = nullptr;
  DaemonSet* DriverDaemonSet = nullptr;
  upgrade::NodeMaintenance* NodeMaintenance = nullptr;
  // Position of the entry's driver pod in BuildState's filteredPodList (upgrade_state.go:126-136), -1 = unknown. Not in
  // the reference's struct: ApplyStateIncremental uses it as the one node order every bucket's slice order is a
  // subsequence of, so that cached entries keep their place when a node changes bucket.
  int64_t ListIndex = -1;
  bool IsOrphanedPod() const { return DriverDaemonSet == nullptr; }
};
struct ClusterUpgradeState {
  std::map<std::string, std::vector<NodeUpgradeState*>> NodeStates;
  std::vector<std::unique_ptr<NodeUpgradeState>> owned;  // BuildState keeps its entries alive here
};
ClusterUpgradeState NewClusterUpgradeState();

// ---- actuator interfaces (stay host-side; driven by the kernel's action bits) --------------------------
struct NodeUpgradeStateProvider {
  virtual ~NodeUpgradeStateProvider() = default;
  virtual Error GetNode(const std::string& nodeName, Node** out) = 0;
  virtual Error ChangeNodeUpgradeState(Node* node, const std::string& newNodeState) = 0;
  virtual Error ChangeNodeUpgradeAnnotation(Node* node, const std::string& key, const std::string& value) = 0;  // "null" deletes
};
struct CordonManager {
  virtual ~CordonManager() = default;
  virtual Error Cordon(Node* node) = 0;
  virtual Error Uncordon(Node* node) = 0;
};
struct DrainConfiguration { const upgrade::DrainSpec* Spec = nullptr; std::vector<Node*> Nodes; };
struct DrainManager {
  virtual ~DrainManager() = default;
  virtual Error ScheduleNodesDrain(const DrainConfiguration& drainConfig) = 0;
};
using PodDeletionFilter = std::function<bool(const Pod&)>;
struct PodManagerConfig {
  std::vector<Node*> Nodes;
  const PodDeletionSpec* DeletionSpec = nullptr;
  const upgrade::WaitForCompletionSpec* WaitForCompletionSpec = nullptr;
  bool DrainEnabled = false;
};
struct PodManager {
  virtual ~PodManager() = default;
  virtual Error ScheduleCheckOnPodCompletion(const PodManagerConfig& config) = 0;
  virtual Error SchedulePodsRestart(const std::vector<Pod*>& pods) = 0;
  virtual Error SchedulePodEviction(const PodManagerConfig& config) = 0;
  virtual PodDeletionFilter GetPodDeletionFilter() = 0;
  virtual Error GetPodControllerRevisionHash(const Pod* pod, std::string* hash) = 0;
  virtual Error GetDaemonsetControllerRevisionHash(const DaemonSet* daemonset, std::string* hash) = 0;
};
// The options of the kubectl drain.Helper that deletes or evicts a node's pods (pod_manager.go:146-157,
// drain_manager.go:76-96): Force, DeleteEmptyDirData, Timeout and GracePeriodSeconds.
struct EvictionOptions { bool Force = false, DeleteEmptyDir = false; int TimeoutSecond = 0; int GracePeriodSeconds = -1; };
// Not in the reference: the side effect of a pod-deletion or drain goroutine, drain.Helper.DeleteOrEvictPods(pods), which
// StateOptions::EvictionOnDevice calls on a mirror-owned worker thread. `node` is the worker's copy of the node; `pods` are
// copies of the pods to delete, in the List's order. Called concurrently for different nodes.
struct PodEvictor {
  virtual ~PodEvictor() = default;
  virtual Error DeleteOrEvictPods(const Node& node, const std::vector<Pod*>& pods, const EvictionOptions& o) = 0;
};
// record.EventRecorder (k8s.io/client-go/tools/record), the slice the managers use: Event(object, eventtype, reason,
// message) on a node. `message` is the final text, as fmt.Sprintf made it in the reference. The three on-device options
// call it from the reconcile's thread and from the mirror's worker threads at once (as the reference's goroutines call
// theirs): it must be safe to call concurrently.
extern const char* const EventTypeNormal;   // corev1.EventTypeNormal
extern const char* const EventTypeWarning;  // corev1.EventTypeWarning
struct EventRecorder {
  virtual ~EventRecorder() = default;
  virtual void Event(const Node& object, const std::string& eventType, const std::string& reason, const std::string& message) = 0;
};
// The error kubectl's drain.RunNodeDrain returns before it evicts anything: utilerrors.NewAggregate over the errors of
// GetPodsForDeletion, for a node's pods (the List's objects, in its order) with their UST_POD_* bits as Encode made them,
// under `spec`'s Force and DeleteEmptyDir. Only pods with UST_POD_MATCH_DRAIN_SELECTOR take part. nullopt: no pod stops
// the drain.
Error DrainFilterError(const std::vector<const Pod*>& pods, const std::vector<uint16_t>& bits, const DrainSpec& spec);
struct ValidationManager {
  virtual ~ValidationManager() = default;
  virtual Error Validate(Node* node, bool* done) = 0;
};
struct SafeDriverLoadManager {
  virtual ~SafeDriverLoadManager() = default;
  virtual Error IsWaitingForSafeDriverLoad(const Node* node, bool* waiting) = 0;
  virtual Error UnblockLoading(Node* node) = 0;
};
// what BuildState lists (controller-runtime client in the reference, upgrade_state.go:105-119)
struct K8sClient {
  virtual ~K8sClient() = default;
  virtual Error ListDaemonSets(const std::string& ns, const StringMap& labels, std::vector<DaemonSet*>* out) = 0;
  virtual Error ListPods(const std::string& ns, const StringMap& labels, std::vector<Pod*>* out) = 0;
  virtual Error GetNodeMaintenance(const std::string& nodeName, NodeMaintenance** out) { *out = nullptr; return std::nullopt; }
  // requestor mode: createOrUpdateNodeMaintenance (upgrade_requestor.go:320-368) / deleteOrUpdateNodeMaintenance
  // (:370-414), the NodeMaintenance CRUD of the upgrade-required and uncordon-required passes
  virtual Error CreateOrUpdateNodeMaintenance(NodeUpgradeState* nodeState) { (void)nodeState; return std::nullopt; }
  virtual Error DeleteOrUpdateNodeMaintenance(NodeUpgradeState* nodeState) { (void)nodeState; return std::nullopt; }
  // The ValidationManager's List (validation_manager.go:77-79) and the PodManager's (pod_manager.go:320-329): the pods of
  // every namespace that match the label selector `selector` ("k=v[,k=v]") and run on node `nodeName` ("" = on any node),
  // in the order the API returns them. Used by StateOptions::ValidateOnDevice and WaitForCompletionOnDevice, which make
  // one such List per reconcile each, with nodeName "".
  virtual Error ListPodsBySelector(const std::string& selector, const std::string& nodeName, std::vector<Pod*>* out) {
    (void)selector; (void)nodeName; (void)out;
    return Errorf("this K8sClient cannot list pods by label selector");
  }
};

struct RequestorOptions { bool UseMaintenanceOperator = false; };  // upgrade_requestor.go:527-546 (the switch only)
struct StateOptions {                                                 // upgrade_state.go:94-96
  RequestorOptions Requestor;
  // Not in the reference: host threads Encode may use (<= 1: the calling thread only). Encoding is the host-side cost of a
  // call (object walking, string-keyed map lookups: ~1 us per node) and is independent per node; with more than one thread
  // the injected PodManager::GetPodControllerRevisionHash and SafeDriverLoadManager::IsWaitingForSafeDriverLoad are called
  // concurrently (they are read-only in the reference: pod_manager.go:84-89, safe_driver_load_manager.go:51-57).
  int EncodeThreads = 1;
  // Not in the reference: answer ValidationManager::Validate on the device (UST_EVAL_VALIDATION) instead of calling it.
  // With a non-empty WithValidationEnabled selector, ApplyState and ApplyStateIncremental make one
  // K8sClient::ListPodsBySelector per reconcile, hand every node its validation pods and its parsed validation start-time
  // annotation to the clocked pod-list calls, and replay the annotation and state calls Validate would have made; the
  // injected ValidationManager is never called. ApplyStateIncremental then keeps the lists and start times resident too.
  bool ValidateOnDevice = false;
  // Not in the reference: answer PodManager::ScheduleCheckOnPodCompletion on the device (UST_EVAL_ACTUATORS) instead of
  // calling it. With a policy whose WaitForCompletion has a non-empty PodSelector, ApplyState and ApplyStateIncremental
  // make one K8sClient::ListPodsBySelector per reconcile for that selector, hand every node its wait-selector pods (after
  // its validation pods when ValidateOnDevice is on too) and its parsed wait-for-pod-completion start-time annotation to
  // the clocked pod-list calls, and replay the annotation and state calls the check would have made; the injected
  // PodManager is never asked to check. Eviction and drain go to the injected managers unless EvictionOnDevice is on too;
  // pod restarts always do. Without a selector the wait-for-jobs pass moves its nodes on by itself and the option changes
  // nothing.
  bool WaitForCompletionOnDevice = false;
  // Not in the reference: decide PodManager::SchedulePodEviction (with WithPodDeletionEnabled and policy.PodDeletion) and
  // DrainManager::ScheduleNodesDrain (with policy.DrainSpec->Enable) on the device (UST_EVAL_ACTUATORS) instead of calling
  // them. ApplyState and ApplyStateIncremental make one K8sClient::ListPodsBySelector("", "") per reconcile (a second one
  // for a non-empty DrainSpec.PodSelector) and one ListDaemonSets, hand every pod-deletion-required and drain-required node
  // its pods with the kubectl filter chain's inputs (after its validation and wait pods), and replay the state changes the
  // goroutines would make from the device's actuator_outcome. Deleting or evicting pods, and the drain's cordon, run on
  // mirror-owned worker threads through the injected PodEvictor and CordonManager; a node being worked on is skipped as the
  // reference skips it. The injected PodManager then only restarts driver pods and looks up revision hashes. The workers
  // call the PodEvictor, the CordonManager and the NodeUpgradeStateProvider while the reconcile (and the next ones) make
  // their own calls, as the reference's goroutines do: those three must be safe to call concurrently.
  bool EvictionOnDevice = false;
  // The reconcile's time.Now().Unix(): read once per ApplyState call; the device derives the validation and
  // wait-for-completion timeouts from it, and a new start-time annotation of either kind is set to it.
  std::function<int64_t()> Now = [] { return (int64_t)time(nullptr); };
};

// ---- the encoded snapshot (include/ust.h layout) and its replay ------------------------------------------
struct EncodedSnapshot {
  std::vector<NodeUpgradeState*> entries;  // SoA index -> snapshot entry, buckets in ApplyState's pass order
  std::vector<uint8_t> state;
  std::vector<uint32_t> flags;
  std::vector<int32_t> pod_rev, ds_idx, ds_rev;
  std::map<size_t, std::string> deferred;  // an error the reference raises when it reaches the node (IsWaitingForSafeDriverLoad)
  ust_policy policy{};
  // StateOptions::ValidateOnDevice (with a validation selector): per entry its validation pods (CSR, UST_POD_* bits in the
  // List's order) and its parsed validation start-time annotation; the reconcile's `now`; and the List's error, which
  // Replay returns at the first validation-required node, after its UnblockLoading, as Validate would.
  bool validateOnDevice = false;
  std::vector<int32_t> pod_off;
  std::vector<uint16_t> pod_flags;
  std::vector<int64_t> start;
  int64_t now = 0;
  Error listError;
  // StateOptions::WaitForCompletionOnDevice (with a wait selector): the wait-selector pods follow each entry's validation
  // pods in pod_off / pod_flags (UST_POD_MATCH_WAIT_SELECTOR + phase), a wait-for-jobs-required entry's start is its parsed
  // wait start-time annotation; per entry whether one of its wait pods is Running or Pending (Replay tells the two
  // pod-deletion-required call orders apart with it); and the wait List's error, which Replay returns at the
  // wait-for-jobs pass when that pass has nodes.
  bool waitOnDevice = false;
  std::vector<char> waitRunning;
  Error waitListError;
  // StateOptions::EvictionOnDevice: a pod-deletion-required or drain-required entry's workload pods follow its wait pods in
  // pod_off / pod_flags; here, by entry index, the same pods (the List's objects) beside their bits, which Replay reads to
  // tell "nothing to delete" apart and to pick the pods to evict. The error of the pod or DaemonSet List, returned at the
  // pod-deletion pass when it has nodes; and that error or the drain-selector List's, returned at the drain pass.
  struct Workload { std::vector<const Pod*> pods; std::vector<uint16_t> bits; };
  bool evictOnDevice = false;
  std::unordered_map<size_t, Workload> workload;
  Error evictListError, drainListError;
};

// ---- common_manager.go:23-41 --------------------------------------------------------------------------------
class CommonUpgradeStateManager {
 public:
  virtual ~CommonUpgradeStateManager() = default;
  virtual int GetTotalManagedNodes(const ClusterUpgradeState& s) const = 0;
  virtual int GetUpgradesInProgress(const ClusterUpgradeState& s) const = 0;
  virtual int GetUpgradesDone(const ClusterUpgradeState& s) const = 0;
  virtual int GetUpgradesAvailable(const ClusterUpgradeState& s, int maxParallelUpgrades, int maxUnavailable) const = 0;
  virtual int GetUpgradesFailed(const ClusterUpgradeState& s) const = 0;
  virtual int GetUpgradesPending(const ClusterUpgradeState& s) const = 0;
  virtual bool IsPodDeletionEnabled() const = 0;
  virtual bool IsValidationEnabled() const = 0;
};

// ---- upgrade_state.go:35-53 -----------------------------------------------------------------------------------
class ClusterUpgradeStateManager : public CommonUpgradeStateManager {
 public:
  virtual ClusterUpgradeStateManager& WithPodDeletionEnabled(PodDeletionFilter filter) = 0;
  virtual ClusterUpgradeStateManager& WithValidationEnabled(const std::string& podSelector) = 0;
  virtual Error BuildState(const std::string& ns, const StringMap& driverLabels, std::unique_ptr<ClusterUpgradeState>* out) = 0;
  virtual Error ApplyState(ClusterUpgradeState* currentState, const DriverUpgradePolicySpec* upgradePolicy) = 0;
};

class ClusterUpgradeStateManagerImpl : public ClusterUpgradeStateManager {
 public:
  // exported fields operators and tests overwrite (common_manager.go:84-100)
  upgrade::K8sClient* K8sClient = nullptr;
  upgrade::DrainManager* DrainManager = nullptr;
  upgrade::PodManager* PodManager = nullptr;
  upgrade::CordonManager* CordonManager = nullptr;
  upgrade::NodeUpgradeStateProvider* NodeUpgradeStateProvider = nullptr;
  upgrade::ValidationManager* ValidationManager = nullptr;
  upgrade::SafeDriverLoadManager* SafeDriverLoadManager = nullptr;
  upgrade::PodEvictor* PodEvictor = nullptr;  // StateOptions::EvictionOnDevice only
  // The manager's EventRecorder (common_manager.go:84-100, upgrade_state.go:65-92). The mirror records only the events of
  // the managers an on-device option replaces (ValidateOnDevice, WaitForCompletionOnDevice, EvictionOnDevice), at the
  // reference's points; the injected managers record their own. nullptr records nothing (util.go:162-176).
  upgrade::EventRecorder* EventRecorder = nullptr;

  // NewClusterUpgradeStateManager (upgrade_state.go:65-92): binds CUDA device `device` through ust_create
  static Error New(int device, StateOptions opts, std::unique_ptr<ClusterUpgradeStateManagerImpl>* out);
  // A manager without a device: Encode / Replay work (recording, auditing), ApplyState and BuildState fail loudly.
  static std::unique_ptr<ClusterUpgradeStateManagerImpl> NewDetached(StateOptions opts);
  ~ClusterUpgradeStateManagerImpl() override;

  ClusterUpgradeStateManager& WithPodDeletionEnabled(PodDeletionFilter filter) override;  // upgrade_state.go:329-337
  ClusterUpgradeStateManager& WithValidationEnabled(const std::string& podSelector) override;  // :341-350
  Error BuildState(const std::string& ns, const StringMap& driverLabels, std::unique_ptr<ClusterUpgradeState>* out) override;
  Error ApplyState(ClusterUpgradeState* currentState, const DriverUpgradePolicySpec* upgradePolicy) override;

  int GetTotalManagedNodes(const ClusterUpgradeState& s) const override;
  int GetUpgradesInProgress(const ClusterUpgradeState& s) const override;
  int GetUpgradesDone(const ClusterUpgradeState& s) const override;
  int GetUpgradesAvailable(const ClusterUpgradeState& s, int maxParallelUpgrades, int maxUnavailable) const override;
  int GetUpgradesFailed(const ClusterUpgradeState& s) const override;
  int GetUpgradesPending(const ClusterUpgradeState& s) const override;
  int GetCurrentUnavailableNodes(const ClusterUpgradeState& s) const;
  bool IsPodDeletionEnabled() const override { return podDeletionStateEnabled_; }
  bool IsValidationEnabled() const override { return validationStateEnabled_; }

  // predicates (same names as the Go methods)
  bool IsUpgradeRequested(const Node& n) const;     // common_manager.go:323-325
  bool IsNodeUnschedulable(const Node& n) const;    // :651-653
  bool isNodeConditionReady(const Node& n) const;   // :656-663
  bool SkipNodeUpgrade(const Node& n) const;        // :666-668
  bool isDriverPodFailing(const Pod& p) const;      // :636-648

  // The two halves of ApplyState around the kernel call. Public so that they can be audited separately:
  // Encode evaluates every reference predicate once and fills the struct-of-arrays; Replay performs the calls
  // named by the action bits, in the reference's pass order, stopping at the first error. `actuator_outcome` is read
  // only for the wait-for-jobs pass of an enc.waitOnDevice snapshot and the pod-deletion and drain passes of an
  // enc.evictOnDevice one, which need it.
  Error Encode(const ClusterUpgradeState& s, const DriverUpgradePolicySpec& policy, EncodedSnapshot* out);
  Error Replay(const EncodedSnapshot& enc, const DriverUpgradePolicySpec& policy, const uint8_t* next_state,
               const uint16_t* actions, int abi_rc, const ust_counters& counters, const uint8_t* actuator_outcome = nullptr);

  const ust_counters& LastCounters() const { return last_; }

  // Not in the reference: when the next reconcile in which only time passes will do something. Nothing changes in the API
  // when a wait-for-completion or validation deadline passes, so no watch event triggers that reconcile; a loop can sleep
  // until this time instead of polling. The value is the device's ust_next_deadline (include/ust.h) of the last ApplyState
  // or ApplyStateIncremental that made a clocked call with ValidateOnDevice or WaitForCompletionOnDevice in effect: the
  // smallest t > that reconcile's `now` at which a reconcile with the same objects makes a call this one did not make (a
  // node times out, or its outcome changes). nullopt when the last ApplyState / ApplyStateIncremental made no such call,
  // when the call failed, or when no deadline is pending.
  // What it does not cover, because each is an object change whose watch event triggers a reconcile of its own, and that
  // reconcile's call includes the deadline it brings: a start-time annotation that Replay sets in this reconcile
  // (UST_A_SET_WAIT_START, for either timeout), and evictions or drains that finish on the workers. A clock that moves
  // backwards is not covered either.
  std::optional<int64_t> NextTimeout() const { return nextTimeout_; }

  // ---- incremental ApplyState (SURVEY 8f.2): the resourceVersion-keyed encode cache -------------------------------
  // The same contract as ApplyState for a reconcile loop that calls it again and again with fresh BuildState
  // snapshots. The manager keeps the encoded snapshot (host and device) from call to call, in a node order that does
  // not move when a node changes bucket (first-seen order = BuildState's pod-list order); an entry is re-encoded only
  // when the resourceVersion of its node, its driver pod or its DaemonSet changed (or is unknown), only the re-encoded
  // entries are uploaded (ust_apply_state_delta_sparse) and only the outputs that differ from the previous reconcile's
  // come back. The reference re-derives everything from node.Labels / Annotations on every reconcile
  // (upgrade_state.go:140-161, common_manager.go:229-604); the provider calls skipped for an unchanged object are
  // GetPodControllerRevisionHash and IsWaitingForSafeDriverLoad, both pure functions of the object in the reference's
  // own implementations (pod_manager.go:84-89, safe_driver_load_manager.go:51-53).
  // The cached slots follow the list order (slots are handed out in slice order, upgrade_inplace.go:71). Nodes that join
  // the cluster are inserted at their list position and encoded on their own; nodes that leave are removed with their
  // slot; nodes that move in the list (a driver pod re-created under a new name, DaemonSets listed in another order)
  // move with their slot and are not re-encoded. Joins and leaves alone travel to the device as one splice of the
  // resident snapshot (ust_apply_state_delta_splice); with moves, as one reorder (ust_apply_state_delta_reorder). A full
  // encode + upload happens on the first call only.
  Error ApplyStateIncremental(ClusterUpgradeState* currentState, const DriverUpgradePolicySpec* upgradePolicy);
  struct IncrementalStats {
    int64_t reconciles = 0, full_uploads = 0, encoded = 0, reused = 0, outputs_received = 0;
    int64_t inserted = 0, removed = 0;  // nodes that joined / left the cached snapshot by a splice or reorder
    int64_t reorders = 0;               // reconciles that went to the device as a reorder (a surviving node moved)
    int64_t slots = 0;                  // size of the cached snapshot after the last reconcile
    // StateOptions::ValidateOnDevice / WaitForCompletionOnDevice: pod lists sent to the device / left resident (a node has
    // one list, its validation and wait-selector pods together, so both options share these two counters), reconciles
    // that sent no node and no list (only time passed), the ValidationManager::Validate calls (one API List each) not made,
    // and the per-node Lists of PodManager::ScheduleCheckOnPodCompletion not made (one per wait-for-jobs-required node)
    int64_t lists_sent = 0, lists_reused = 0, time_only = 0, validate_avoided = 0, wait_avoided = 0;
    // StateOptions::EvictionOnDevice: the per-node pod Lists not made (one per pod-deletion-required or drain-required node
    // of a pass the option answers), and the nodes handed to the PodEvictor's workers (by Replay, in either ApplyState)
    int64_t evict_lists_avoided = 0, actuator_handoffs = 0;
  };
  const IncrementalStats& Stats() const { return stats_; }
  void ResetIncremental();
  // Switches StateOptions::ValidateOnDevice; the incremental cache starts over on the next call when the mode changes.
  void SetValidateOnDevice(bool on) { opts_.ValidateOnDevice = on; }
  // Switches StateOptions::WaitForCompletionOnDevice, with the same effect on the incremental cache.
  void SetWaitForCompletionOnDevice(bool on) { opts_.WaitForCompletionOnDevice = on; }
  // Switches StateOptions::EvictionOnDevice, with the same effect on the incremental cache.
  void SetEvictionOnDevice(bool on) { opts_.EvictionOnDevice = on; }
  // Blocks until every eviction and drain handed to the workers has ended (their state changes made). The destructor
  // waits too.
  void WaitForActuators();

  // ---- incremental BuildState: the driver-pod list stays on the device (ust_build_state_delta) -----------------------------
  // The same contract, result and errors as BuildState, for a reconcile loop that calls it again and again. The manager keeps
  // the raw ListPods order (keyed by Namespace/Name) with each pod's state byte, owner UID and owner index; a pod's state
  // byte and owner UID are re-derived only when its resourceVersion changed (or is ""), pods that join, leave or move in the
  // list go to the device as runs of one reorder, and only the owner indices that changed come back. With
  // ApplyStateIncremental on the same manager the whole reconcile stays incremental: BuildState's list never leaves the
  // device, and neither does ApplyState's snapshot. The first call (and the first after a reset) sends every pod.
  Error BuildStateIncremental(const std::string& ns, const StringMap& driverLabels, std::unique_ptr<ClusterUpgradeState>* out);
  struct BuildStats {
    int64_t reconciles = 0, full_uploads = 0;
    int64_t rederived = 0, reused = 0;  // pods whose state byte and owner UID were derived anew / taken from the cache
    int64_t inserted = 0, removed = 0;  // pods that joined / left the cached list
    int64_t reorders = 0;               // reconciles whose list moved on the device (a join, a leave or a move)
    int64_t outputs_received = 0;       // owner indices that came back (sparse, or all of them after a truncation)
  };
  const BuildStats& BuildStateStats() const { return buildStats_; }
  void ResetBuildIncremental();

 protected:
  // The cached driver-pod list of BuildStateIncremental, in this reconcile's ListPods order, and what changed since the
  // device last saw it: with `reorder`, the new order as ust_driver_pod_reorder runs (after a reset: the whole list as one
  // inserted run) and the joined pods' positions; the positions whose values were overwritten.
  struct PodCache {
    std::unordered_map<std::string, size_t> posOf;  // Namespace/Name -> position
    std::vector<std::string> rv;                     // resourceVersion the pod's values were derived at
    std::vector<uint8_t> state;
    std::vector<uint64_t> owner;                     // two per pod
    std::vector<int32_t> ownerIdx;                   // owning DaemonSet index / -1 / -2 (INT32_MIN until a joined pod's comes back)
    std::vector<int64_t> run_src, run_len, insert_at, changed;
    bool reorder = false;
    bool valid = false;
  };
  // The device call of BuildState: ust_build_state_uids. Returns the ABI's return code.
  virtual int BuildStateDevice(int64_t n, const uint8_t* state, const uint64_t* owner, int32_t n_ds, const uint64_t* ds_uid,
                               const int32_t* desired, int32_t* owner_idx, ust_counters* c);
  // The device half of BuildStateIncremental: hand cache->run_src / changed to ust_build_state_delta and patch the owner
  // indices that changed into cache->ownerIdx (already in the new order), or fetch them all. Returns the ABI's return code.
  // (Both virtual so that the host-logic test can put the oracle behind them.)
  virtual int BuildStateCached(int32_t n_ds, const uint64_t* ds_uid, const int32_t* desired, PodCache* cache, ust_counters* c);
  // The device half of ApplyStateIncremental: evaluate the cached snapshot. full: upload all of it and fetch all
  // outputs; else apply cache->pending to the resident snapshot, upload the entries `changed` and patch the outputs that
  // differ into cache_.next / cache_.actions (whose entries already follow the splice).
  // Returns the ABI's return code. (Virtual so that the host-logic test can put the oracle behind the same cache.)
  struct Cache {
    struct Slot { std::string name, sig; size_t id = 0; int code = UST_STATE_EXCLUDED; bool seen = false; };
    // Node name -> stable id of its slot, id -> SoA index. A splice moves slots; the ids stay, so only slotOfId is
    // rewritten (one linear pass), and only the names that joined or left touch the hash map.
    std::unordered_map<std::string, size_t> idOf;
    std::vector<size_t> slotOfId;
    std::vector<size_t> freeIds;
    // The change of node order the host arrays went through since the device last saw them (indices into the previous
    // snapshot): remove_idx are the slots that left; insert_at[k] is the new index of inserted node k, whose columns are
    // state[insert_at[k]] etc. While the surviving slots keep their order it is a ust_splice (insert_before); when one
    // of them moved, the new order as ust_reorder runs (run_src / run_len) instead, and insert_before is empty.
    // Empty after a full upload.
    struct Splice {
      std::vector<int64_t> remove_idx, insert_before, insert_at;
      std::vector<int64_t> run_src, run_len;
      bool empty() const { return remove_idx.empty() && insert_before.empty() && run_src.empty(); }
    };
    Splice pending;
    std::vector<Slot> slots;
    std::vector<uint8_t> state, next;
    std::vector<uint32_t> flags;
    std::vector<int32_t> pod_rev, ds_idx, ds_rev;
    std::vector<uint16_t> actions;
    std::vector<std::string> deferredMsg;            // per slot: the error the reference raises when it reaches the node
    std::map<std::string, int32_t> intern;           // revision hash -> id
    std::map<std::string, int32_t> dsIndexByUID;
    std::vector<bool> dsHashError;
    bool valid = false;
    // StateOptions::ValidateOnDevice only (pods == true): per slot its validation pod list, the (pod, resourceVersion)
    // sequence it was built from ("" = no pods, "\x01" = unknown) and its validation start time; and the slots whose list
    // goes down with this call, in slot order (every inserted slot among them). In this mode pending never holds a
    // splice: a change of node order is always run_src / run_len, as the pod-list calls take it.
    bool pods = false;
    std::vector<std::vector<uint16_t>> lists;
    std::vector<std::string> listSig;
    std::vector<int64_t> start;
    std::vector<int64_t> listChanged;
    // Which of the two options filled the lists (a change starts the cache over). With WaitForCompletionOnDevice a slot's
    // list is its validation pods (the first nval entries) followed by its wait-selector pods, whose (pod, resourceVersion)
    // sequence is waitSig; each half is rebuilt from its own List. In either mode, actuator_outcome per slot, patched
    // like next / actions: the replay of a wait-for-jobs-required node reads it on every reconcile.
    bool validation = false, wait = false;
    std::vector<int32_t> nval;
    std::vector<std::string> waitSig;
    std::vector<uint8_t> outcome;
    // With EvictionOnDevice the list ends with the node's workload pods (the last nwork entries; none unless the node is
    // pod-deletion-required or drain-required), built from the (pod, resourceVersion, DaemonSet found) sequence workSig.
    bool evict = false;
    std::vector<int32_t> nwork;
    std::vector<std::string> workSig;
  };
  virtual int EvaluateCached(const ust_policy& policy, bool full, const std::vector<int64_t>& changed, Cache* cache, ust_counters* c);
  // The same on the clocked pod-list snapshot (StateOptions::ValidateOnDevice / WaitForCompletionOnDevice): full:
  // ust_apply_state_clocked with every list and start time; else ust_apply_state_delta_pods_clocked with cache->pending as
  // runs, the lists of cache->listChanged and the start times of `changed` and of the inserted slots, patching
  // cache->outcome too. `now` / `waitTimeout` make the ust_clock.
  // It also leaves the call's next deadline (ust_next_deadline; nullopt for none, or when the call failed) in
  // cachedDeadline_, which ApplyStateIncremental carries out through NextTimeout(); an override sets it as well.
  virtual int EvaluateCachedPods(const ust_policy& policy, int64_t now, int64_t waitTimeout, bool full,
                                 const std::vector<int64_t>& changed, Cache* cache, ust_counters* c);
  std::optional<int64_t> cachedDeadline_;
  ClusterUpgradeStateManagerImpl() = default;
  explicit ClusterUpgradeStateManagerImpl(StateOptions opts) : opts_(std::move(opts)) {}  // a manager without a device

 private:
  Error encodeOne(const NodeUpgradeState* ns, int code, int32_t ds, bool dsErr, std::map<std::string, int32_t>* intern,
                  const std::vector<int32_t>& ds_rev, uint8_t* hot, uint32_t* flags, int32_t* rev, std::string* deferred,
                  int64_t* start, bool validation, bool wait);
  bool validateOnDevice() const { return opts_.ValidateOnDevice && validationStateEnabled_; }
  bool waitOnDevice(const DriverUpgradePolicySpec& p) const {
    return opts_.WaitForCompletionOnDevice && p.WaitForCompletion && !p.WaitForCompletion->PodSelector.empty();
  }
  // StateOptions::EvictionOnDevice: the pod-deletion pass / the drain pass it answers, and whether it answers either
  bool evictPodDeletion(const DriverUpgradePolicySpec& p) const { return opts_.EvictionOnDevice && podDeletionStateEnabled_ && p.PodDeletion; }
  bool evictDrain(const DriverUpgradePolicySpec& p) const { return opts_.EvictionOnDevice && p.DrainSpec && p.DrainSpec->Enable; }
  bool evictOnDevice(const DriverUpgradePolicySpec& p) const { return evictPodDeletion(p) || evictDrain(p); }
  // Runs `job` on a worker thread; `name` stays in `*dedupe` until the job has ended.
  void handOff(std::set<std::string>* dedupe, const std::string& name, std::function<void()> job);
  Error assembleState(const std::vector<Pod*>& podList, const uint8_t* podState, const int32_t* owner_idx,
                      std::map<std::string, DaemonSet*>& daemonSets, std::unique_ptr<ClusterUpgradeState>* out);
  Cache cache_;
  IncrementalStats stats_;
  PodCache podCache_;
  BuildStats buildStats_;
  ust_handle* handle_ = nullptr;
  StateOptions opts_;
  bool podDeletionStateEnabled_ = false, validationStateEnabled_ = false;
  PodDeletionFilter filter_;
  std::string validationSelector_;
  ust_counters last_{};
  std::optional<int64_t> nextTimeout_;  // NextTimeout()
  // The PodEvictor's workers: a queue served by up to kActuatorWorkers threads, and the reference's two dedupe sets
  // (pod_manager.go:160-165, drain_manager.go:104-110), guarded by actMu_.
  static constexpr size_t kActuatorWorkers = 16;
  std::mutex actMu_;
  std::condition_variable actCv_;
  std::deque<std::function<void()>> actQueue_;
  std::vector<std::thread> actThreads_;
  size_t actIdle_ = 0, actRunning_ = 0;
  bool actStop_ = false;
  std::set<std::string> nodesInProgress_, drainingNodes_;
};

const char* StateNameOfCode(unsigned code);  // "" for unknown; nullptr for codes without a label
int StateCodeOfLabel(const std::string& label);

}  // namespace upgrade
