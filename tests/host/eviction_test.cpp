// StateOptions::EvictionOnDevice (eviction_spec.hpp).
//   eviction_test         host halves only: Encode's workload entries and each bit's source, after the validation and wait
//                         pods; what ApplyStateIncremental hands to the device (a stand-in records it); Replay of hand-made
//                         outcomes through passes 5 and 6, the worker's calls, the dedupe sets and the Lists' errors
//   eviction_test --gpu   the reference's SchedulePodEviction and ScheduleNodesDrain specs through ApplyState, the host's
//                         "nothing to delete" against the device's outcome, and a reconcile loop of ApplyStateIncremental
//                         with the option against ApplyState with the restated PodManagerImpl and DrainManagerImpl
#include <atomic>
#include <cstdlib>
#include <cstring>
#include <set>

#include "eviction_spec.hpp"

using namespace upgrade;
using namespace espec;

namespace {

const std::string kGpuLabel = "nvidia.com/gpu";
PodDeletionFilter gpuFilter() { return [](const Pod& p) { return p.Labels.count("nvidia.com/gpu") != 0; }; }

// Nodes with a driver pod each, in list order; workload pods and DaemonSets in the fake store. Everything the mirror's
// workers call is locked.
struct World {
  std::deque<Node> nodes;
  std::vector<int> pos;        // list position of each node (a move swaps two); -1: the node left
  std::deque<Pod> drivers, pods;
  std::vector<char> podAlive;
  std::deque<DaemonSet> dss;
  DaemonSet driverDs;
  ClusterUpgradeState state;
  std::vector<std::unique_ptr<NodeUpgradeState>> owned;
  std::vector<std::string> log;
  LockedProvider provider;
  FailingCordon cordon;
  LockedDrain drain;
  LockedPods podm;
  SafeDriverLoadManagerImpl safeLoad{&provider};
  Store store;
  LogEvictor evictor;
  int64_t version = 10;
  World() {
    provider.log = drain.log = podm.log = cordon.log = evictor.log = &log;
    cordon.mu = evictor.mu = podm.mu = drain.mu = &provider.mu;
    driverDs.Name = "driver"; driverDs.UID = "uid-ds";
  }
  Node& node(const std::string& name, const std::string& label, StringMap annotations = {}) {
    nodes.emplace_back();
    Node& n = nodes.back();
    n.Name = name;
    n.ResourceVersion = std::to_string(version++);
    n.Labels[GetUpgradeStateLabelKey()] = label;
    n.Annotations = std::move(annotations);
    provider.nodes[name] = &n;
    pos.push_back((int)pos.size());
    drivers.emplace_back();
    Pod& d = drivers.back();
    d.Name = "drv-" + name; d.Namespace = "gpu-operator"; d.NodeName = name; d.ResourceVersion = "1";
    d.OwnerReferences.push_back({"DaemonSet", "driver", driverDs.UID});
    d.Labels[PodControllerRevisionHashLabelKey] = "test-hash-12345";
    d.Phase = "Running"; d.ContainerStatuses = {{true, 0}};
    return n;
  }
  Pod& pod(const std::string& name, const std::string& node, const std::string& phase, bool gpu = true) {
    pods.push_back(makeWorkloadPod(name, node, phase, version++));
    podAlive.push_back(1);
    if (gpu) pods.back().Labels[kGpuLabel] = "1";
    return pods.back();
  }
  DaemonSet& ds(const std::string& name) {
    dss.emplace_back();
    dss.back().Name = name; dss.back().Namespace = "apps"; dss.back().UID = "uid-" + name;
    return dss.back();
  }
  void bump(Pod& p) { p.ResourceVersion = std::to_string(version++); }
  void snapshot() {
    state = ClusterUpgradeState();
    owned.clear();
    std::vector<std::pair<int, size_t>> order;
    for (size_t i = 0; i < nodes.size(); i++)
      if (pos[i] >= 0) order.emplace_back(pos[i], i);
    std::sort(order.begin(), order.end());
    for (size_t k = 0; k < order.size(); k++) {
      const size_t i = order[k].second;
      auto e = std::make_unique<NodeUpgradeState>();
      e->Node = &nodes[i]; e->DriverPod = &drivers[i]; e->DriverDaemonSet = &driverDs; e->ListIndex = (int64_t)k;
      state.NodeStates[nodes[i].Labels[GetUpgradeStateLabelKey()]].push_back(e.get());
      owned.push_back(std::move(e));
    }
    store.all.clear();
    for (size_t i = 0; i < pods.size(); i++)
      if (podAlive[i]) store.all.push_back(&pods[i]);
    std::stable_sort(store.all.begin(), store.all.end(), [](const Pod* x, const Pod* y) { return x->Name < y->Name; });
    store.workloadDs.clear();
    for (DaemonSet& d : dss) store.workloadDs.push_back(&d);
  }
  void wire(ClusterUpgradeStateManagerImpl* m) {
    m->NodeUpgradeStateProvider = &provider; m->CordonManager = &cordon; m->DrainManager = &drain; m->PodManager = &podm;
    m->SafeDriverLoadManager = &safeLoad; m->K8sClient = &store; m->PodEvictor = &evictor;
  }
  // the reference's managers over this world
  std::unique_ptr<PodManagerImpl> refPods;
  std::unique_ptr<DrainManagerImpl> refDrain;
  void wireReference(ClusterUpgradeStateManagerImpl* m, const PodDeletionFilter& filter) {
    wire(m);
    refPods.reset(new PodManagerImpl());
    refPods->store = &store; refPods->client = &store; refPods->provider = &provider; refPods->evictor = &evictor;
    refPods->podDeletionFilter = filter; refPods->log = &log; refPods->now = [] { return (int64_t)1700000000; };
    refDrain.reset(new DrainManagerImpl());
    refDrain->store = &store; refDrain->evictor = &evictor; refDrain->cordon = &cordon; refDrain->provider = &provider;
    m->PodManager = refPods.get();
    m->DrainManager = refDrain.get();
  }
  std::vector<std::string> calls() const {  // the log without the pod-restart pass's SchedulePodsRestart, which is always made
    std::vector<std::string> out;
    for (const std::string& l : log)
      if (l != "restart") out.push_back(l);
    return out;
  }
  std::string image() const {
    std::string s;
    for (size_t i = 0; i < nodes.size(); i++) {
      if (pos[i] < 0) continue;
      const Node& n = nodes[i];
      s += n.Name + "{" + n.Labels.at(GetUpgradeStateLabelKey());
      for (const auto& kv : n.Annotations) s += "," + kv.first + "=" + kv.second;
      s += "}";
    }
    return s;
  }
};

DriverUpgradePolicySpec evictPolicy(bool drain, bool force = false, const std::string& selector = "") {
  DriverUpgradePolicySpec p;
  p.AutoUpgrade = true;
  p.PodDeletion = PodDeletionSpec{};
  p.PodDeletion->Force = force;
  p.PodDeletion->TimeoutSecond = 120;
  p.DrainSpec = upgrade::DrainSpec{};
  p.DrainSpec->Enable = drain;
  p.DrainSpec->Force = force;
  p.DrainSpec->PodSelector = selector;
  p.DrainSpec->TimeoutSecond = 60;
  return p;
}

// What ApplyStateIncremental hands to the device, recorded; the outputs are "no transition, no call".
struct StandIn : ClusterUpgradeStateManagerImpl {
  struct Call {
    bool full = false;
    std::vector<int64_t> changed, listed;
    std::vector<std::vector<uint16_t>> lists;
    int32_t evaluate = 0;
  };
  std::vector<Call> calls;
  explicit StandIn(StateOptions o) : ClusterUpgradeStateManagerImpl(std::move(o)) {}
  int EvaluateCached(const ust_policy& policy, bool full, const std::vector<int64_t>& changed, Cache* k, ust_counters* c) override {
    k->outcome.clear();
    return EvaluateCachedPods(policy, 0, 0, full, changed, k, c);
  }
  int EvaluateCachedPods(const ust_policy& policy, int64_t, int64_t, bool full, const std::vector<int64_t>& changed, Cache* k,
                         ust_counters* c) override {
    Call call;
    call.full = full; call.changed = changed; call.listed = k->listChanged; call.evaluate = policy.evaluate_actuators;
    for (int64_t i : k->listChanged) call.lists.push_back(k->lists[(size_t)i]);
    calls.push_back(call);
    const size_t n = k->slots.size();
    k->next.assign(n + 1, 0);
    k->actions.assign(n + 1, 0);
    k->outcome.assign(n + 1, UST_OUTCOME_NONE);
    for (size_t i = 0; i < n; i++) k->next[i] = k->state[i] & UST_HOT_STATE_MASK;
    std::memset(c, 0, sizeof(*c));
    c->error_index = -1;
    return UST_OK;
  }
};

const uint16_t DEL = UST_POD_MATCH_DELETION_FILTER, DRN = UST_POD_MATCH_DRAIN_SELECTOR, RUN = UST_PHASE_RUNNING;
const uint8_t PRR = UST_STATE_POD_RESTART_REQUIRED, DRQ = UST_STATE_DRAIN_REQUIRED, FLD = UST_STATE_FAILED;

std::map<std::string, std::vector<uint16_t>> listsOf(const EncodedSnapshot& e) {
  std::map<std::string, std::vector<uint16_t>> out;
  for (size_t i = 0; i < e.entries.size(); i++)
    out[e.entries[i]->Node->Name] = std::vector<uint16_t>(e.pod_flags.begin() + e.pod_off[i], e.pod_flags.begin() + e.pod_off[i + 1]);
  return out;
}

void cpu_specs(Runner& R) {
  SetDriverName("gpu");

  R.it("Encode: workload entries for pod-deletion-required and drain-required nodes only, each bit from its source", [&] {
    World w;
    w.node("n0", UpgradeStatePodDeletionRequired);
    w.node("n1", UpgradeStateDrainRequired);
    w.node("n2", UpgradeStateDone);
    w.ds("present");
    Pod& a = w.pod("a-ctrl-second", "n0", "Running");  // the controller is the second owner reference
    a.OwnerReferences = {{"ReplicaSet", "rs", "u1", false}, {"ReplicaSet", "rs2", "u2", true}};
    w.pod("b-ds-present", "n0", "Running").OwnerReferences = {{"DaemonSet", "present", "u3", true}};
    w.pod("c-ds-missing", "n0", "Pending").OwnerReferences = {{"DaemonSet", "gone", "u4", true}};
    w.pod("d-ds-not-controller", "n0", "Running").OwnerReferences = {{"DaemonSet", "gone", "u5", false}};
    w.pod("e-mirror", "n0", "Running", false).Annotations["kubernetes.io/config.mirror"] = "x";
    w.pod("f-emptydir", "n0", "Running").HasEmptyDirVolume = true;
    w.pod("g-finished", "n0", "Succeeded");
    w.pod("h-drain", "n1", "Failed", false);
    w.pod("i-elsewhere", "n2", "Running");
    w.pod("j-unscheduled", "", "Pending");
    w.snapshot();
    StateOptions o;
    o.EvictionOnDevice = true;
    auto m = ClusterUpgradeStateManagerImpl::NewDetached(o);
    w.wire(m.get());
    m->WithPodDeletionEnabled(gpuFilter());
    EncodedSnapshot e;
    EXPECT(R, !m->Encode(w.state, evictPolicy(true), &e).has_value());
    EXPECT(R, e.evictOnDevice && !e.waitOnDevice && !e.validateOnDevice && e.policy.evaluate_actuators == (int32_t)UST_EVAL_ACTUATORS);
    EXPECT(R, w.store.allLists == 1 && w.store.lists == 1 && w.store.dsLists == 1);  // an empty drain selector: no second List
    bool zero = true;
    for (int64_t s : e.start) zero = zero && s == 0;
    EXPECT(R, zero && e.start.size() == e.entries.size());
    auto L = listsOf(e);
    const uint16_t C = UST_POD_HAS_CONTROLLER, DS = UST_POD_CONTROLLED_BY_DS, MISS = UST_POD_DS_MISSING;
    EXPECT(R, (L["n0"] == std::vector<uint16_t>{(uint16_t)(RUN | C | DEL | DRN), (uint16_t)(RUN | C | DS | DEL | DRN),
                                                (uint16_t)(UST_PHASE_PENDING | C | DS | MISS | DEL | DRN), (uint16_t)(RUN | DEL | DRN),
                                                (uint16_t)(RUN | UST_POD_MIRROR | DRN), (uint16_t)(RUN | UST_POD_HAS_EMPTYDIR | DEL | DRN),
                                                (uint16_t)(UST_PHASE_SUCCEEDED | DEL | DRN)}));
    EXPECT(R, (L["n1"] == std::vector<uint16_t>{(uint16_t)(UST_PHASE_FAILED | DRN)}));
    EXPECT(R, L["n2"].empty());
    EXPECT(R, e.workload.size() == 2);
    for (const auto& kv : e.workload) EXPECT(R, kv.second.pods.size() == kv.second.bits.size());
    // a drain PodSelector: a second List, whose members alone carry the drain bit; drain off: no drain bits
    World s;
    s.node("n0", UpgradeStateDrainRequired);
    s.pod("a", "n0", "Running").Labels["app"] = "train";
    s.pod("b", "n0", "Running");
    s.snapshot();
    auto m2 = ClusterUpgradeStateManagerImpl::NewDetached(o);
    s.wire(m2.get());
    EncodedSnapshot e2;
    EXPECT(R, !m2->Encode(s.state, evictPolicy(true, false, "app=train"), &e2).has_value());
    EXPECT(R, s.store.lists == 2 && s.store.allLists == 1 && s.store.dsLists == 1);
    EXPECT(R, (listsOf(e2)["n0"] == std::vector<uint16_t>{(uint16_t)(RUN | DRN), RUN}));
    // without the option nothing changes; with it but neither pass enabled, neither
    for (int variant = 0; variant < 2; variant++) {
      StateOptions q;
      q.EvictionOnDevice = variant == 1;
      auto plain = ClusterUpgradeStateManagerImpl::NewDetached(q);
      w.wire(plain.get());
      EncodedSnapshot x;
      DriverUpgradePolicySpec px = evictPolicy(variant == 0);
      EXPECT(R, !plain->Encode(w.state, px, &x).has_value());
      EXPECT(R, !x.evictOnDevice && x.pod_off.empty() && x.workload.empty() && x.policy.evaluate_actuators == 0 && x.flags == e.flags);
    }
  });

  R.it("Encode with ValidateOnDevice and WaitForCompletionOnDevice too: validation pods, then wait pods, then workload pods", [&] {
    World w;
    w.node("n0", UpgradeStatePodDeletionRequired);
    w.pods.push_back(vspec::makeValidationPod("a-val", "n0", true, {true}, 1)); w.podAlive.push_back(1);
    w.pods.push_back(wspec::makeWaitPod("b-job", "n0", "Running", 1)); w.podAlive.push_back(1);
    w.pods.back().Labels["tier"] = "gpu";
    w.pod("c-gpu", "n0", "Running");
    w.snapshot();
    StateOptions o;
    o.EvictionOnDevice = o.ValidateOnDevice = o.WaitForCompletionOnDevice = true;
    auto m = ClusterUpgradeStateManagerImpl::NewDetached(o);
    w.wire(m.get());
    m->WithPodDeletionEnabled(gpuFilter());
    m->WithValidationEnabled("app=validator");
    DriverUpgradePolicySpec p = evictPolicy(false);
    p.WaitForCompletion = WaitForCompletionSpec{"tier=gpu", 30};
    EncodedSnapshot e;
    EXPECT(R, !m->Encode(w.state, p, &e).has_value());
    EXPECT(R, e.policy.evaluate_actuators == (int32_t)(UST_EVAL_ACTUATORS | UST_EVAL_VALIDATION) && w.store.lists == 3);
    const uint16_t V = UST_POD_MATCH_VALIDATION_SELECTOR | UST_POD_READY, W = UST_POD_MATCH_WAIT_SELECTOR;
    // the workload part holds every pod of the node, the validation and wait pods among them, with workload bits only
    EXPECT(R, (listsOf(e)["n0"] == std::vector<uint16_t>{V, (uint16_t)(W | RUN), (uint16_t)(W | RUN), RUN, RUN, (uint16_t)(RUN | DEL)}));
  });

  R.it("ApplyStateIncremental hands down only changed workload parts, nothing for an unchanged node, and drops them on leaving", [&] {
    World w;
    w.node("n0", UpgradeStatePodDeletionRequired);
    w.node("n1", UpgradeStateDrainRequired);
    w.node("n2", UpgradeStateDone);
    w.ds("ds");
    w.pod("p0", "n0", "Running");
    Pod& q = w.pod("p1", "n1", "Running");
    q.OwnerReferences = {{"DaemonSet", "ds", "u", true}};
    w.pod("p2", "n2", "Running");
    StateOptions o;
    o.EvictionOnDevice = true;
    auto* dev = new StandIn(o);
    std::unique_ptr<ClusterUpgradeStateManagerImpl> owner(dev);
    w.wire(dev);
    dev->WithPodDeletionEnabled(gpuFilter());
    const DriverUpgradePolicySpec p = evictPolicy(true);
    auto reconcile = [&] { w.snapshot(); EXPECT(R, !dev->ApplyStateIncremental(&w.state, &p).has_value()); };
    reconcile();
    EXPECT(R, dev->calls.back().full && dev->calls.back().listed.size() == 3 && dev->calls.back().evaluate == (int32_t)UST_EVAL_ACTUATORS);
    reconcile();  // nothing changed
    EXPECT(R, dev->calls.back().listed.empty() && dev->calls.back().changed.empty());
    w.pod("p3", "n0", "Pending").HasEmptyDirVolume = true;  // a pod appears
    w.pods[2].Phase = "Succeeded"; w.bump(w.pods[2]);           // a pod on a node without entries finishes
    reconcile();
    EXPECT(R, (dev->calls.back().listed == std::vector<int64_t>{0}));
    EXPECT(R, (dev->calls.back().lists[0] == std::vector<uint16_t>{(uint16_t)(RUN | DEL | DRN),
                                                                   (uint16_t)(UST_PHASE_PENDING | UST_POD_HAS_EMPTYDIR | DEL | DRN)}));
    w.dss.clear();  // the DaemonSet disappears: its pod's bits change without a new resourceVersion
    reconcile();
    EXPECT(R, (dev->calls.back().listed == std::vector<int64_t>{1}));
    EXPECT(R, (dev->calls.back().lists[0] == std::vector<uint16_t>{(uint16_t)(RUN | UST_POD_HAS_CONTROLLER | UST_POD_CONTROLLED_BY_DS |
                                                                              UST_POD_DS_MISSING | DEL | DRN)}));
    w.nodes[0].Labels[GetUpgradeStateLabelKey()] = UpgradeStatePodRestartRequired; w.nodes[0].ResourceVersion = "99";
    w.nodes[2].Labels[GetUpgradeStateLabelKey()] = UpgradeStateDrainRequired; w.nodes[2].ResourceVersion = "99";
    reconcile();  // n0 leaves the two states (its entries go), n2 enters them (its pods come)
    EXPECT(R, (dev->calls.back().listed == std::vector<int64_t>{0, 2}) && dev->calls.back().lists[0].empty());
    EXPECT(R, (dev->calls.back().lists[1] == std::vector<uint16_t>{(uint16_t)(UST_PHASE_SUCCEEDED | DEL | DRN)}));
    const auto& st = dev->Stats();
    EXPECT(R, st.full_uploads == 1 && st.evict_lists_avoided == 2 * 5 && w.store.allLists == 5 && w.store.dsLists == 5);
    if (R.failed_here)
      std::printf("    %lld avoided, %d Lists, %d DaemonSet Lists\n", (long long)st.evict_lists_avoided, w.store.allLists, w.store.dsLists);
    EXPECT(R, managerCalls(w.log) == 0);
    dev->SetEvictionOnDevice(false);
    reconcile();
    EXPECT(R, dev->Stats().full_uploads == 2 && w.store.allLists == 5);
  });

  // Replay of passes 5 and 6 from hand-made outcomes: one node in `label`.
  struct Case { const char* label; uint8_t outcome; bool drain; std::string failEvict, failCordon, failState; };
  auto replay = [&](const Case& c, std::vector<std::string>* log, int* copies, std::string* image) -> Error {
    World w;
    w.node("n0", c.label);
    w.pod("a", "n0", "Running");
    w.pod("b", "n0", "Running", false);
    w.pod("c", "n0", "Succeeded");
    w.evictor.failNode = c.failEvict;
    w.cordon.failNode = c.failCordon;
    w.provider.match = c.failState;
    w.provider.failAt = 0;
    w.snapshot();
    StateOptions o;
    o.EvictionOnDevice = true;
    auto m = ClusterUpgradeStateManagerImpl::NewDetached(o);
    w.wire(m.get());
    m->WithPodDeletionEnabled(gpuFilter());
    const DriverUpgradePolicySpec p = evictPolicy(c.drain);
    EncodedSnapshot e;
    if (Error err = m->Encode(w.state, p, &e)) return err;
    const int code = StateCodeOfLabel(c.label);
    const uint8_t next = (uint8_t)code;
    const uint16_t actions = code == UST_STATE_DRAIN_REQUIRED ? UST_A_SCHEDULE_DRAIN : UST_A_SCHEDULE_POD_EVICTION;
    ust_counters k{};
    k.error_index = -1; k.error_pass = -1;
    Error err = m->Replay(e, p, &next, &actions, UST_OK, k, &c.outcome);
    m->WaitForActuators();
    *log = w.calls();
    *copies = w.provider.copies;
    *image = w.image();
    EXPECT(R, managerCalls(w.log) == 0);
    return err;
  };
  const std::string evAB = "evict n0 force=0 emptydir=0 timeout=120 grace=-1: a c";
  R.it("Replay, pass 5: nothing to delete, a mismatch with drain on and off, evict OK and evict failure; on a copy, errors dropped", [&] {
    std::vector<std::string> log;
    int copies = 0;
    std::string img;
    EXPECT(R, !replay({UpgradeStatePodDeletionRequired, DRQ, true, "", "", ""}, &log, &copies, &img));
    EXPECT(R, (log == std::vector<std::string>{"state n0=drain-required"}) && copies == 1);
    EXPECT(R, !replay({UpgradeStatePodDeletionRequired, FLD, false, "", "", ""}, &log, &copies, &img));
    EXPECT(R, (log == std::vector<std::string>{"state n0=upgrade-failed"}) && copies == 1);
    EXPECT(R, !replay({UpgradeStatePodDeletionRequired, PRR, false, "", "", ""}, &log, &copies, &img));
    EXPECT(R, (log == std::vector<std::string>{evAB, "state n0=pod-restart-required"}) && copies == 1);
    EXPECT(R, !replay({UpgradeStatePodDeletionRequired, PRR, true, "n0", "", ""}, &log, &copies, &img));
    EXPECT(R, (log == std::vector<std::string>{"FAILED " + evAB, "state n0=drain-required"}));
    EXPECT(R, !replay({UpgradeStatePodDeletionRequired, PRR, false, "n0", "", ""}, &log, &copies, &img));
    EXPECT(R, (log == std::vector<std::string>{"FAILED " + evAB, "state n0=upgrade-failed"}));
    EXPECT(R, !replay({UpgradeStatePodDeletionRequired, PRR, false, "", "", "state n0"}, &log, &copies, &img));
    EXPECT(R, (log == std::vector<std::string>{evAB, "FAILED state n0=pod-restart-required"}));
    // no filter-matching pod: pod-restart-required without an eviction
    World w;
    w.node("n0", UpgradeStatePodDeletionRequired);
    w.pod("x", "n0", "Running", false);
    w.snapshot();
    StateOptions o;
    o.EvictionOnDevice = true;
    auto m = ClusterUpgradeStateManagerImpl::NewDetached(o);
    w.wire(m.get());
    m->WithPodDeletionEnabled(gpuFilter());
    EncodedSnapshot e;
    EXPECT(R, !m->Encode(w.state, evictPolicy(false), &e));
    const uint8_t next = UST_STATE_POD_DELETION_REQUIRED;
    const uint16_t a = UST_A_SCHEDULE_POD_EVICTION;
    ust_counters k{};
    k.error_index = -1; k.error_pass = -1;
    EXPECT(R, !m->Replay(e, evictPolicy(false), &next, &a, UST_OK, k, &PRR));
    m->WaitForActuators();
    EXPECT(R, (w.calls() == std::vector<std::string>{"state n0=pod-restart-required"}) && m->Stats().actuator_handoffs == 0);
    // the snapshot's node object is left alone
    EXPECT(R, w.nodes[0].Labels.at(GetUpgradeStateLabelKey()) == UpgradeStatePodDeletionRequired || w.provider.copies == 1);
  });
  R.it("Replay, pass 6: cordon, then evict, then the state; cordon failure, drain error status and evict failure give upgrade-failed", [&] {
    std::vector<std::string> log;
    int copies = 0;
    std::string img;
    const std::string evAll = "evict n0 force=0 emptydir=0 timeout=60 grace=-1: c";  // a and b are unreplicated: kept without force
    EXPECT(R, !replay({UpgradeStateDrainRequired, PRR, true, "", "", ""}, &log, &copies, &img));
    EXPECT(R, (log == std::vector<std::string>{"cordon n0", evAll, "state n0=pod-restart-required"}) && copies == 1);
    EXPECT(R, !replay({UpgradeStateDrainRequired, PRR, true, "", "n0", ""}, &log, &copies, &img));
    EXPECT(R, (log == std::vector<std::string>{"FAILED cordon n0", "state n0=upgrade-failed"}));
    EXPECT(R, !replay({UpgradeStateDrainRequired, FLD, true, "", "", ""}, &log, &copies, &img));
    EXPECT(R, (log == std::vector<std::string>{"cordon n0", "state n0=upgrade-failed"}));
    EXPECT(R, !replay({UpgradeStateDrainRequired, PRR, true, "n0", "", ""}, &log, &copies, &img));
    EXPECT(R, (log == std::vector<std::string>{"cordon n0", "FAILED " + evAll, "state n0=upgrade-failed"}));
    EXPECT(R, !replay({UpgradeStateDrainRequired, PRR, true, "", "", "state n0"}, &log, &copies, &img));
    EXPECT(R, (log == std::vector<std::string>{"cordon n0", evAll, "FAILED state n0=pod-restart-required"}));
  });

  R.it("Dedupe: a node whose eviction or drain is still running gets no second call and no state change", [&] {
    struct LatchEvictor : PodEvictor {
      std::mutex m;
      std::condition_variable cv;
      bool open = false;
      std::atomic<int> calls{0};
      Error DeleteOrEvictPods(const Node&, const std::vector<Pod*>&, const EvictionOptions&) override {
        calls++;
        std::unique_lock<std::mutex> l(m);
        cv.wait(l, [&] { return open; });
        return std::nullopt;
      }
    } latch;
    World w;
    w.node("n0", UpgradeStatePodDeletionRequired);
    w.node("n1", UpgradeStateDrainRequired);
    w.pod("a", "n0", "Running");
    w.pod("b", "n1", "Running").OwnerReferences = {{"ReplicaSet", "rs", "u", true}};
    StateOptions o;
    o.EvictionOnDevice = true;
    auto m = ClusterUpgradeStateManagerImpl::NewDetached(o);
    w.wire(m.get());
    m->PodEvictor = &latch;
    m->WithPodDeletionEnabled(gpuFilter());
    const DriverUpgradePolicySpec p = evictPolicy(true);
    const uint8_t next[2] = {UST_STATE_POD_DELETION_REQUIRED, UST_STATE_DRAIN_REQUIRED}, outcome[2] = {PRR, PRR};
    const uint16_t actions[2] = {UST_A_SCHEDULE_POD_EVICTION, UST_A_SCHEDULE_DRAIN};
    ust_counters k{};
    k.error_index = -1; k.error_pass = -1;
    for (int rec = 0; rec < 2; rec++) {
      w.snapshot();
      EncodedSnapshot e;
      EXPECT(R, !m->Encode(w.state, p, &e));
      EXPECT(R, !m->Replay(e, p, next, actions, UST_OK, k, outcome));
      if (rec == 0)
        while (latch.calls < 2) std::this_thread::yield();
    }
    {
      std::lock_guard<std::mutex> l(w.provider.mu);
      EXPECT(R, latch.calls == 2 && (w.calls() == std::vector<std::string>{"cordon n1"}) && m->Stats().actuator_handoffs == 2);
    }
    { std::lock_guard<std::mutex> l(latch.m); latch.open = true; }
    latch.cv.notify_all();
    m->WaitForActuators();
    EXPECT(R, latch.calls == 2 && w.calls().size() == 3 && w.image() == "n0{pod-restart-required}n1{pod-restart-required}");
    // once the workers ended, the nodes are taken again
    w.nodes[0].Labels[GetUpgradeStateLabelKey()] = UpgradeStatePodDeletionRequired;
    w.nodes[1].Labels[GetUpgradeStateLabelKey()] = UpgradeStateDrainRequired;
    w.snapshot();
    EncodedSnapshot e;
    EXPECT(R, !m->Encode(w.state, p, &e));
    EXPECT(R, !m->Replay(e, p, next, actions, UST_OK, k, outcome));
    m->WaitForActuators();
    EXPECT(R, latch.calls == 4);
  });

  R.it("Replay: a failed pod or DaemonSet List returns at the pass it serves, only when that pass has nodes", [&] {
    // which List fails x which passes have nodes
    for (int which = 0; which < 3; which++)
      for (int nodes = 0; nodes < 3; nodes++) {
        World w;
        w.node("n0", UpgradeStateCordonRequired);
        if (nodes == 0) w.node("n1", UpgradeStatePodDeletionRequired);
        if (nodes == 1) w.node("n2", UpgradeStateDrainRequired);
        w.node("n3", UpgradeStateUncordonRequired);
        const Error boom = Errorf("etcdserver: request timed out");
        if (which == 0) w.store.listError = boom;  // both kinds of pod List
        if (which == 1) w.store.dsError = boom;
        w.snapshot();
        StateOptions o;
        o.EvictionOnDevice = true;
        auto m = ClusterUpgradeStateManagerImpl::NewDetached(o);
        w.wire(m.get());
        m->WithPodDeletionEnabled(gpuFilter());
        const DriverUpgradePolicySpec p = evictPolicy(true, false, which == 2 ? "app=x" : "");
        if (which == 2) w.store.selectorError = boom;  // the drain-selector List only
        EncodedSnapshot e;
        EXPECT(R, !m->Encode(w.state, p, &e));
        std::vector<uint8_t> next, outcome;
        std::vector<uint16_t> actions;
        for (size_t i = 0; i < e.entries.size(); i++) {
          const int code = e.state[i] & UST_HOT_STATE_MASK;
          next.push_back(code == UST_STATE_CORDON_REQUIRED ? (uint8_t)UST_STATE_WAIT_FOR_JOBS_REQUIRED : (uint8_t)code);
          actions.push_back(code == UST_STATE_CORDON_REQUIRED ? (uint16_t)(UST_A_CORDON | UST_A_SET_STATE)
                            : code == UST_STATE_POD_DELETION_REQUIRED ? (uint16_t)UST_A_SCHEDULE_POD_EVICTION
                            : code == UST_STATE_DRAIN_REQUIRED ? (uint16_t)UST_A_SCHEDULE_DRAIN : (uint16_t)UST_A_UNCORDON);
          outcome.push_back(PRR);
        }
        ust_counters k{};
        k.error_index = -1; k.error_pass = -1;
        const Error err = m->Replay(e, p, next.data(), actions.data(), UST_OK, k, outcome.data());
        m->WaitForActuators();
        // the selector List serves the drain pass only
        const bool expectErr = nodes == 1 || (nodes == 0 && which != 2);
        EXPECT(R, expectErr ? (err && *err == *boom) : !err);
        EXPECT(R, w.log.size() >= 2 && w.log[0] == "cordon n0");
        const bool reachedUncordon = std::find(w.log.begin(), w.log.end(), "uncordon n3") != w.log.end();
        EXPECT(R, reachedUncordon == !expectErr);
        if (R.failed_here) std::printf("    which %d nodes %d: %s\n", which, nodes, err ? err->c_str() : "ok");
      }
  });
}

// ---- on the H100 ---------------------------------------------------------------------------------------------------
std::unique_ptr<ClusterUpgradeStateManagerImpl> device(StateOptions o, bool* ok) {
  std::unique_ptr<ClusterUpgradeStateManagerImpl> m;
  if (auto e = ClusterUpgradeStateManagerImpl::New(0, o, &m)) {
    std::printf("cannot create manager: %s\n", e->c_str());
    *ok = false;
    return ClusterUpgradeStateManagerImpl::NewDetached(o);
  }
  return m;
}

void gpu_specs(Runner& R, bool* ok) {
  SetDriverName("gpu");
  // One cluster through ApplyState with the restated managers, and through ApplyState and ApplyStateIncremental with
  // EvictionOnDevice: the same calls per node, the same nodes afterwards, the same error.
  using Setup = std::function<void(World&)>;
  auto both = [&](const char* name, const DriverUpgradePolicySpec& p, const Setup& setup, const std::function<void(const World&)>& expect) {
    R.it(name, [&] {
      World a, b, c;
      for (World* w : {&a, &b, &c}) { setup(*w); w->snapshot(); }
      StateOptions o;
      auto ma = device(o, ok);
      a.wireReference(ma.get(), gpuFilter());
      ma->WithPodDeletionEnabled(gpuFilter());
      o.EvictionOnDevice = true;
      auto mb = device(o, ok), mc = device(o, ok);
      b.wire(mb.get()); c.wire(mc.get());
      mb->WithPodDeletionEnabled(gpuFilter()); mc->WithPodDeletionEnabled(gpuFilter());
      const Error ea = ma->ApplyState(&a.state, &p), eb = mb->ApplyState(&b.state, &p), ec = mc->ApplyStateIncremental(&c.state, &p);
      mb->WaitForActuators(); mc->WaitForActuators();
      EXPECT(R, ea == eb && ea == ec);
      EXPECT(R, perNode(a.log) == perNode(b.log) && perNode(b.log) == perNode(c.log));
      EXPECT(R, a.image() == b.image() && b.image() == c.image());
      EXPECT(R, managerCalls(b.log) == 0 && managerCalls(c.log) == 0);
      if (R.failed_here) {
        for (auto& s : a.log) std::printf("    ref: %s\n", s.c_str());
        for (auto& s : b.log) std::printf("    dev: %s\n", s.c_str());
      }
      expect(b);
    });
  };
  auto label = [](const World& w, size_t i = 0) { return w.nodes[i].Labels.at(GetUpgradeStateLabelKey()); };
  // pod_manager_test.go:226-430: a CPU pod, standalone GPU pods (no controller) and a GPU pod with an emptyDir
  auto gpuPods = [](bool emptyDirPod, bool allEmptyDir) {
    return [=](World& w) {
      w.node("n0", UpgradeStatePodDeletionRequired);
      w.pod("cpu-pod", "n0", "Running", false);
      w.pod("gpu-pod1", "n0", "Running").HasEmptyDirVolume = allEmptyDir;
      if (!allEmptyDir) w.pod("gpu-pod2", "n0", "Running");
      if (emptyDirPod) w.pod("test-gpu-pod", "n0", "Running").HasEmptyDirVolume = true;
    };
  };
  auto withSpec = [](bool drain, bool force, bool emptyDir) {
    DriverUpgradePolicySpec p = evictPolicy(drain, force);
    p.PodDeletion->DeleteEmptyDir = emptyDir;
    return p;
  };
  both("standalone gpu pods with force are deleted: pod-restart-required (pod_manager_test.go:236)", withSpec(false, true, false),
       gpuPods(false, false), [&](const World& w) { EXPECT(R, label(w) == UpgradeStatePodRestartRequired && w.calls().size() == 2); });
  both("without force, drain disabled: upgrade-failed, nothing deleted (:267)", withSpec(false, false, false), gpuPods(false, false),
       [&](const World& w) { EXPECT(R, label(w) == UpgradeStateFailed && w.calls().size() == 1); });
  both("without force, drain enabled: drain-required (:300)", withSpec(true, false, false), gpuPods(false, false),
       [&](const World& w) { EXPECT(R, label(w) == UpgradeStateDrainRequired); });
  both("with emptyDir, force and deleteEmptyDir: deleted (:332)", withSpec(false, true, true), gpuPods(true, false),
       [&](const World& w) { EXPECT(R, label(w) == UpgradeStatePodRestartRequired); });
  both("with emptyDir, force, no deleteEmptyDir, drain disabled: upgrade-failed (:366)", withSpec(false, true, false), gpuPods(false, true),
       [&](const World& w) { EXPECT(R, label(w) == UpgradeStateFailed); });
  both("with emptyDir, force, no deleteEmptyDir, drain enabled: drain-required (:399)", withSpec(true, true, false), gpuPods(false, true),
       [&](const World& w) { EXPECT(R, label(w) == UpgradeStateDrainRequired); });
  // drain_manager_test.go:33-161
  both("DrainManager should drain nodes (drain_manager_test.go:33)", evictPolicy(true, true), [](World& w) {
    w.node("n0", UpgradeStateDrainRequired);
    w.pod("p", "n0", "Running", false);
  }, [&](const World& w) { EXPECT(R, label(w) == UpgradeStatePodRestartRequired && w.calls().size() == 3); });
  both("DrainManager should drain all nodes it receives (:55)", evictPolicy(true, true), [](World& w) {
    for (int i = 0; i < 3; i++) w.node("n" + std::to_string(i), UpgradeStateDrainRequired);
  }, [&](const World& w) { EXPECT(R, label(w, 0) == UpgradeStatePodRestartRequired && label(w, 2) == UpgradeStatePodRestartRequired); });
  both("DrainManager should not fail on an empty node list (:91)", evictPolicy(true), [](World& w) {
    w.node("n0", UpgradeStateDone);
  }, [&](const World& w) { EXPECT(R, w.calls().empty()); });
  both("DrainManager should skip drain if drain is disabled in the spec (:143)", evictPolicy(false), [](World& w) {
    w.node("n0", UpgradeStateDrainRequired);
  }, [&](const World& w) { EXPECT(R, label(w) == UpgradeStatePodRestartRequired && w.calls().size() == 1); });
  both("a drain selector evicts only the pods it selects; an error pod it selects fails the drain", evictPolicy(true, false, "app=train"),
       [](World& w) {
         w.node("n0", UpgradeStateDrainRequired);
         w.node("n1", UpgradeStateDrainRequired);
         Pod& a = w.pod("a", "n0", "Running"); a.Labels["app"] = "train"; a.OwnerReferences = {{"Job", "j", "u", true}};
         w.pod("b", "n0", "Running");  // unreplicated but not selected
         w.pod("c", "n1", "Running").Labels["app"] = "train";  // unreplicated and selected: an error
       }, [&](const World& w) { EXPECT(R, label(w, 0) == UpgradeStatePodRestartRequired && label(w, 1) == UpgradeStateFailed); });
  both("a DaemonSet pod: skipped while its DaemonSet exists, an error once it is gone (without force)", evictPolicy(true), [](World& w) {
    w.ds("present");
    w.node("n0", UpgradeStateDrainRequired);
    w.node("n1", UpgradeStateDrainRequired);
    w.pod("a", "n0", "Running").OwnerReferences = {{"DaemonSet", "present", "u", true}};
    w.pod("b", "n1", "Running").OwnerReferences = {{"DaemonSet", "gone", "u", true}};
  }, [&](const World& w) { EXPECT(R, label(w, 0) == UpgradeStatePodRestartRequired && label(w, 1) == UpgradeStateFailed); });

  R.it("on a C4-like snapshot the host's 'nothing to delete' agrees with the device on every pod-deletion-required node", [&] {
    spec::BLcg r{2024};
    ust_handle* h = nullptr;
    if (ust_create(&h, 0) != UST_OK) { *ok = false; EXPECT(R, false); return; }
    int none = 0, mismatch = 0, evict = 0;
    for (int force = 0; force < 2; force++) {
      World w;
      w.ds("present");
      const char* phases[] = {"Running", "Pending", "Succeeded", "Failed", "Unknown"};
      for (int i = 0; i < 4000; i++) {
        const std::string n = "n" + std::to_string(i);
        w.node(n, UpgradeStatePodDeletionRequired);
        for (int j = (int)(r.next() % 5); j > 0; j--) {
          Pod& p = w.pod("p" + std::to_string(j) + "-" + n, n, phases[r.next() % 5], r.chance(50));
          const int kind = (int)(r.next() % 5);
          if (kind == 1) p.OwnerReferences = {{"ReplicaSet", "rs", "u", true}};
          if (kind == 2) p.OwnerReferences = {{"DaemonSet", r.chance(50) ? "present" : "gone", "u", true}};
          if (kind == 3) p.OwnerReferences = {{"ReplicaSet", "rs", "u", false}};
          if (r.chance(5)) p.Annotations["kubernetes.io/config.mirror"] = "m";
          p.HasEmptyDirVolume = r.chance(15);
        }
      }
      w.snapshot();
      StateOptions o;
      o.EvictionOnDevice = true;
      auto m = ClusterUpgradeStateManagerImpl::NewDetached(o);
      w.wire(m.get());
      m->WithPodDeletionEnabled(gpuFilter());
      const DriverUpgradePolicySpec p = evictPolicy(false, force == 1);
      EncodedSnapshot e;
      EXPECT(R, !m->Encode(w.state, p, &e));
      const size_t n = e.entries.size();
      std::vector<uint8_t> next(n + 1), outcome(n + 1);
      std::vector<uint16_t> actions(n + 1);
      e.state.push_back(0); e.flags.push_back(0); e.pod_rev.push_back(0); e.ds_idx.push_back(0); e.ds_rev.push_back(0);
      e.pod_flags.push_back(0); e.start.push_back(0);
      const ust_pods pods = {e.pod_off.data(), e.pod_flags.data(), (int64_t)e.pod_flags.size() - 1};
      const ust_clock clock = {1700000000, 0, e.start.data(), nullptr};
      ust_counters c;
      EXPECT(R, ust_apply_state_clocked(h, &e.policy, &clock, (int64_t)n, e.state.data(), e.flags.data(), e.pod_rev.data(), e.ds_idx.data(),
                                        (int32_t)e.ds_rev.size() - 1, e.ds_rev.data(), &pods, next.data(), actions.data(), outcome.data(),
                                        &c) == UST_OK);
      // the restated helper decides every node on its own
      DrainHelper helper;
      helper.client = &w.store; helper.Force = force == 1; helper.additional = gpuFilter();
      for (size_t i = 0; i < n; i++) {
        const std::string& name = e.entries[i]->Node->Name;
        bool nothing = true;
        const auto it = e.workload.find(i);
        if (it != e.workload.end())
          for (uint16_t b : it->second.bits) nothing = nothing && !(b & UST_POD_MATCH_DELETION_FILTER);
        std::vector<Pod*> listed, deletable;
        w.store.ListPodsBySelector("", name, &listed);
        int toDelete = 0;
        for (const Pod* q : listed) toDelete += gpuFilter()(*q) ? 1 : 0;
        helper.GetPodsForDeletion(name, &deletable);
        const uint8_t want = toDelete == 0 ? PRR : (int)deletable.size() != toDelete ? FLD : PRR;
        const bool good = (actions[i] & UST_A_SCHEDULE_POD_EVICTION) && outcome[i] == want && nothing == (toDelete == 0);
        EXPECT(R, good);
        if (!good) { std::printf("    node %s: outcome %u want %u toDelete %d nothing %d\n", name.c_str(), outcome[i], want, toDelete, nothing); break; }
        none += toDelete == 0; mismatch += want == FLD; evict += toDelete != 0 && want == PRR;
      }
    }
    ust_destroy(h);
    std::printf("    %d nothing to delete, %d mismatched, %d evicted\n", none, mismatch, evict);
    EXPECT(R, none > 0 && mismatch > 0 && evict > 0);
  });
}

// The reconcile loop: nodes in every state, workload pods that appear, finish and gain emptyDirs, DaemonSets that
// disappear, evictions and cordons that fail, nodes that join, leave and move.
void evolve(World& w, spec::BLcg r, int rec) {
  const char* states[] = {UpgradeStatePodDeletionRequired, UpgradeStateDrainRequired, UpgradeStateDone, UpgradeStateCordonRequired,
                          UpgradeStateWaitForJobsRequired, UpgradeStatePodRestartRequired, UpgradeStateUpgradeRequired};
  for (size_t i = 0; i < w.nodes.size(); i++) {
    if (w.pos[i] < 0) continue;
    Node& n = w.nodes[i];
    const std::string st = n.Labels[GetUpgradeStateLabelKey()];
    if (st != UpgradeStatePodDeletionRequired && st != UpgradeStateDrainRequired && r.chance(15)) {  // back into the two states
      n.Labels[GetUpgradeStateLabelKey()] = states[r.next() % 2];
      spec::LogProvider::bump(&n);
    }
    if (r.chance(1)) w.pos[i] = -1;  // leaves
  }
  for (size_t i = 0; i < w.pods.size(); i++) {
    if (!w.podAlive[i]) continue;
    Pod& p = w.pods[i];
    if (r.chance(4)) { p.Phase = r.chance(50) ? "Succeeded" : "Failed"; w.bump(p); }
    else if (r.chance(2)) { p.HasEmptyDirVolume = true; w.bump(p); }
    else if (r.chance(2)) w.podAlive[i] = 0;
  }
  for (size_t i = 0; i < w.nodes.size(); i++)
    if (w.pos[i] >= 0 && r.chance(6)) {
      const std::string n = w.nodes[i].Name;
      Pod& p = w.pod("p" + std::to_string(rec) + "-" + n, n, r.chance(80) ? "Running" : "Pending", r.chance(70));
      const int kind = (int)(r.next() % 4);
      if (kind == 1) p.OwnerReferences = {{"ReplicaSet", "rs", "u", true}};
      if (kind == 2) p.OwnerReferences = {{"DaemonSet", "ds" + std::to_string(r.next() % 3), "u", true}};
      if (r.chance(30)) p.Labels["app"] = "train";
    }
  if (rec % 50 == 10 && !w.dss.empty()) w.dss.pop_back();  // a DaemonSet disappears
  if (rec % 50 == 30) w.ds("ds" + std::to_string(w.dss.size()));
  for (int j = (int)(r.next() % 3); j > 0; j--) {  // joins
    w.node("j" + std::to_string(rec) + "-" + std::to_string(j), states[r.next() % 7]);
    w.pos.back() = (int)(r.next() % (w.pos.size() + 1)) * 2 + 1;
  }
  int k = 0;  // re-number the list; now and then two nodes trade places
  std::vector<std::pair<int, size_t>> order;
  for (size_t i = 0; i < w.nodes.size(); i++)
    if (w.pos[i] >= 0) order.emplace_back(w.pos[i] * 2, i);
  std::sort(order.begin(), order.end());
  for (auto& o : order) w.pos[o.second] = k++;
  if (order.size() > 4 && r.chance(30)) std::swap(w.pos[order[1].second], w.pos[order[order.size() - 2].second]);
}

void loop(Runner& R, bool requestor, bool others, int n_nodes, int rounds, bool* ok) {
  SetDriverName("gpu");
  const std::string name = std::string("ApplyStateIncremental with EvictionOnDevice == ApplyState with PodManagerImpl and DrainManagerImpl "
                                       "over a reconcile loop (") + (requestor ? "requestor" : "in-place") + " mode, the other two options " +
                           (others ? "on" : "off") + ")";
  R.it(name.c_str(), [&] {
    World a, b;
    spec::BLcg seed{99};
    for (World* w : {&a, &b}) {
      spec::BLcg r = seed;
      w->ds("ds0"); w->ds("ds1"); w->ds("ds2");
      for (int i = 0; i < n_nodes; i++) {
        const char* states[] = {UpgradeStatePodDeletionRequired, UpgradeStateDrainRequired, UpgradeStateDone, UpgradeStateCordonRequired};
        const std::string n = "n" + std::to_string(i);
        w->node(n, states[r.next() % 4]);
        for (int j = (int)(r.next() % 4); j > 0; j--) w->pod("p" + std::to_string(j) + "-" + n, n, "Running", r.chance(60));
      }
    }
    StateOptions o;
    o.Requestor.UseMaintenanceOperator = requestor;
    o.Now = [] { return (int64_t)1700000000; };
    StateOptions od = o;
    od.EvictionOnDevice = true;
    od.ValidateOnDevice = od.WaitForCompletionOnDevice = others;
    auto mb = device(od, ok);
    b.wire(mb.get());
    mb->WithPodDeletionEnabled(gpuFilter());
    if (others) mb->WithValidationEnabled("app=validator");
    DriverUpgradePolicySpec p = evictPolicy(true, false, "");
    p.MaxParallelUpgrades = 0;
    if (others) p.WaitForCompletion = WaitForCompletionSpec{"tier=gpu", 300};
    int handoffs = 0, evictFails = 0, cordonFails = 0, refEvictions = 0, refDrains = 0, badLists = 0, replaced = 0;
    vspec::ValidationManagerImpl vref;
    vref.client = &a.store; vref.provider = &a.provider; vref.podSelector = "app=validator"; vref.now = o.Now;
    std::set<std::string> seen;
    for (int rec = 0; rec < rounds; rec++) {
      p.DrainSpec->PodSelector = (rec / 60) % 2 ? "app=train" : "";
      p.PodDeletion->Force = p.DrainSpec->Force = rec % 7 == 3;
      p.PodDeletion->DeleteEmptyDir = p.DrainSpec->DeleteEmptyDir = rec % 5 == 1;
      auto ma = device(o, ok);  // the reference's way: a fresh manager every reconcile
      a.wireReference(ma.get(), gpuFilter());
      ma->WithPodDeletionEnabled(gpuFilter());
      if (others) { ma->WithValidationEnabled("app=validator"); ma->ValidationManager = &vref; }
      a.snapshot(); b.snapshot();
      a.log.clear(); b.log.clear();
      // now and then the eviction of the first pod-deletion-required node, or the cordon of the first drain-required one,
      // fails. (A failed List is not in the loop: the reference's goroutines drop it, the option returns it; the CPU
      // cases cover that rule.)
      auto first = [&](const char* label) {
        auto it = a.state.NodeStates.find(label);
        return it == a.state.NodeStates.end() || it->second.empty() ? std::string() : it->second[0]->Node->Name;
      };
      for (World* w : {&a, &b}) {
        w->evictor.failNode = rec % 3 == 1 ? first(UpgradeStatePodDeletionRequired) : "";
        w->cordon.failNode = rec % 5 == 2 ? first(UpgradeStateDrainRequired) : "";
      }
      const int listsBefore = b.store.allLists, dsBefore = b.store.dsLists, podListsBefore = b.store.lists;
      const int evBefore = a.refPods->evictions;
      const Error ea = ma->ApplyState(&a.state, &p);
      const Error eb = mb->ApplyStateIncremental(&b.state, &p);
      mb->WaitForActuators();
      refEvictions += a.refPods->evictions - evBefore;
      replaced += managerCalls(b.log);
      refDrains += a.refDrain->calls;
      badLists += b.store.allLists - listsBefore > 1 || b.store.dsLists - dsBefore > 1 ||
                  b.store.lists - podListsBefore > 2 + (others ? 2 : 0);
      EXPECT(R, ea == eb);
      EXPECT(R, perNode(a.log) == perNode(b.log));
      EXPECT(R, a.image() == b.image());
      for (const std::string& s : b.log) {
        evictFails += s.rfind("FAILED evict", 0) == 0;
        cordonFails += s.rfind("FAILED cordon", 0) == 0;
      }
      if (R.failed_here) {
        std::printf("    (reconcile %d: %s / %s)\n", rec, ea ? ea->c_str() : "ok", eb ? eb->c_str() : "ok");
        const auto pa = perNode(a.log), pb = perNode(b.log);
        for (const auto& kv : pa)
          if (!pb.count(kv.first) || pb.at(kv.first) != kv.second)
            for (const auto& s : kv.second) std::printf("    ref %s: %s\n", kv.first.c_str(), s.c_str());
        for (const auto& kv : pb)
          if (!pa.count(kv.first) || pa.at(kv.first) != kv.second)
            for (const auto& s : kv.second) std::printf("    dev %s: %s\n", kv.first.c_str(), s.c_str());
        break;
      }
      a.podm.restarted.clear(); b.podm.restarted.clear();
      evolve(a, spec::BLcg{7000u + (uint64_t)rec}, rec); evolve(b, spec::BLcg{7000u + (uint64_t)rec}, rec);
    }
    const auto& st = mb->Stats();
    handoffs = (int)st.actuator_handoffs;
    std::printf("    %lld reconciles, %lld full uploads, %lld reorders, %lld lists sent, %lld reused, %lld per-node Lists avoided, "
                "%d hand-offs, %d failed evictions, %d failed cordons; reference: %d SchedulePodEviction, %d ScheduleNodesDrain\n",
                (long long)st.reconciles, (long long)st.full_uploads, (long long)st.reorders, (long long)st.lists_sent,
                (long long)st.lists_reused, (long long)st.evict_lists_avoided, handoffs, evictFails, cordonFails, refEvictions, refDrains);
    EXPECT(R, replaced == 0 && badLists == 0 && refEvictions > 0 && refDrains > 0);
    EXPECT(R, st.full_uploads == 1 && handoffs > 0 && evictFails > 0 && cordonFails > 0 && st.evict_lists_avoided > 0);
  });
}

}  // namespace

int main(int argc, char** argv) {
  const bool gpu = argc > 1 && std::strcmp(argv[1], "--gpu") == 0;
  Runner R;
  bool ok = true;
  if (gpu) {
    gpu_specs(R, &ok);
    for (bool others : {false, true}) {
      loop(R, false, others, 120, 300, &ok);
      loop(R, true, others, 120, 300, &ok);
    }
  } else {
    cpu_specs(R);
  }
  std::printf("# %d passed, %d failed\n", R.passed, R.failed);
  return (R.failed == 0 && ok) ? 0 : 1;
}
