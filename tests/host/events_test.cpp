// The events of the managers the three on-device options replace (events_spec.hpp).
//   events_test         host halves only: GetEventReason, the drain's aggregate error, and Replay of hand-made outputs for
//                       every row of the events table: type, reason, message and place among the node's calls; a null
//                       recorder leaves the calls as they were, and with the options off the mirror records nothing
//   events_test --gpu   the reference's eviction, drain, wait and validation cases with a recorder against the restated
//                       managers, and reconcile loops with injected failures, each option alone and all three together
#include <cstdlib>
#include <cstring>

#include "events_spec.hpp"

using namespace upgrade;
using namespace espec;

namespace {

const std::string kGpuLabel = "nvidia.com/gpu";
PodDeletionFilter gpuFilter() { return [](const Pod& p) { return p.Labels.count("nvidia.com/gpu") != 0; }; }
const int64_t kNow = 1700000000;

// The restated PodManagerImpl, whose SchedulePodsRestart writes the shared log under the lock the workers take.
struct Pods : evspec::PodManagerImpl {
  std::mutex* mu = nullptr;
  Error SchedulePodsRestart(const std::vector<Pod*>& pods) override {
    std::lock_guard<std::mutex> l(*mu);
    return evspec::PodManagerImpl::SchedulePodsRestart(pods);
  }
};

// Nodes with a driver pod each, in list order; workload, wait and validation pods and DaemonSets in the fake store; the
// restated managers with events, recording into the world's log. Everything the mirror's workers call is locked.
struct World {
  std::deque<Node> nodes;
  std::vector<int> pos;
  std::deque<Pod> drivers, pods;
  std::vector<char> podAlive;
  std::deque<DaemonSet> dss;
  DaemonSet driverDs;
  ClusterUpgradeState state;
  std::vector<std::unique_ptr<NodeUpgradeState>> owned;
  std::vector<std::string> log;
  LockedProvider provider;
  FailingCordon cordon;
  SafeDriverLoadManagerImpl safeLoad{&provider};
  Store store;
  LogEvictor evictor;
  evspec::LogRecorder recorder;
  Pods podm;
  evspec::DrainManagerImpl drain;
  evspec::ValidationManagerImpl val;
  int64_t version = 10, now = kNow;
  World() {
    provider.log = cordon.log = evictor.log = podm.log = recorder.log = &log;
    cordon.mu = evictor.mu = recorder.mu = podm.mu = &provider.mu;
    driverDs.Name = "driver"; driverDs.UID = "uid-ds";
    podm.store = &store; podm.client = &store; podm.provider = &provider; podm.evictor = &evictor;
    podm.podDeletionFilter = gpuFilter(); podm.now = [this] { return now; }; podm.recorder = &recorder;
    drain.store = &store; drain.evictor = &evictor; drain.cordon = &cordon; drain.provider = &provider; drain.recorder = &recorder;
    val.client = &store; val.provider = &provider; val.podSelector = "app=validator"; val.now = [this] { return now; };
    val.recorder = &recorder;
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
  Pod& add(Pod p) {
    p.ResourceVersion = std::to_string(version++);
    pods.push_back(std::move(p));
    podAlive.push_back(1);
    return pods.back();
  }
  Pod& pod(const std::string& name, const std::string& node, const std::string& phase, bool gpu = true) {
    Pod& p = add(makeWorkloadPod(name, node, phase, 0));
    if (gpu) p.Labels[kGpuLabel] = "1";
    return p;
  }
  Pod& waitPod(const std::string& name, const std::string& node, const std::string& phase) {
    return add(wspec::makeWaitPod(name, node, phase, 0));
  }
  Pod& valPod(const std::string& name, const std::string& node, bool ready) {
    return add(vspec::makeValidationPod(name, node, true, {ready}, 0));
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
  // the restated managers for every pass the options leave to them, and the recorder (when `record`)
  void wire(ClusterUpgradeStateManagerImpl* m, bool record = true) {
    m->NodeUpgradeStateProvider = &provider; m->CordonManager = &cordon; m->DrainManager = &drain; m->PodManager = &podm;
    m->ValidationManager = &val; m->SafeDriverLoadManager = &safeLoad; m->K8sClient = &store; m->PodEvictor = &evictor;
    m->EventRecorder = record ? &recorder : nullptr;
    m->WithPodDeletionEnabled(gpuFilter());
    m->WithValidationEnabled("app=validator");
  }
  std::string image() const {
    std::string s;
    for (size_t i = 0; i < nodes.size(); i++) {
      if (pos[i] < 0) continue;
      s += nodes[i].Name + "{" + nodes[i].Labels.at(GetUpgradeStateLabelKey());
      for (const auto& kv : nodes[i].Annotations) s += "," + kv.first + "=" + kv.second;
      s += "}";
    }
    return s;
  }
};

// Each node's calls and events in order (Validate's runs of one delete collapsed, as validation_spec.hpp explains).
std::map<std::string, std::vector<std::string>> byNode(const std::vector<std::string>& log) {
  auto m = perNode(log);
  for (auto& kv : m) kv.second = vspec::collapse(kv.second);
  return m;
}
std::vector<std::string> withoutEvents(const std::vector<std::string>& log) {
  std::vector<std::string> out;
  for (const std::string& s : log)
    if (s.rfind("event ", 0) != 0) out.push_back(s);
  return out;
}

DriverUpgradePolicySpec policy(bool drain, bool force = false, int waitTimeout = 300) {
  DriverUpgradePolicySpec p;
  p.AutoUpgrade = true;
  p.PodDeletion = PodDeletionSpec{};
  p.PodDeletion->Force = force;
  p.PodDeletion->TimeoutSecond = 120;
  p.DrainSpec = upgrade::DrainSpec{};
  p.DrainSpec->Enable = drain;
  p.DrainSpec->Force = force;
  p.DrainSpec->TimeoutSecond = 60;
  p.WaitForCompletion = WaitForCompletionSpec{"app=my-app", waitTimeout};  // wspec::makeWaitPod's label
  return p;
}
StateOptions allOn() {
  StateOptions o;
  o.ValidateOnDevice = o.WaitForCompletionOnDevice = o.EvictionOnDevice = true;
  o.Now = [] { return kNow; };
  return o;
}

// Replay of one node with hand-made outputs on a detached manager; the log afterwards (workers ended).
Error replayOne(World& w, const StateOptions& o, const DriverUpgradePolicySpec& p, uint8_t next, uint16_t actions, uint8_t outcome,
                bool record = true) {
  w.snapshot();
  auto m = ClusterUpgradeStateManagerImpl::NewDetached(o);
  w.wire(m.get(), record);
  EncodedSnapshot e;
  if (Error err = m->Encode(w.state, p, &e)) return err;
  ust_counters k{};
  k.error_index = -1; k.error_pass = -1;
  Error err = m->Replay(e, p, &next, &actions, UST_OK, k, &outcome);
  m->WaitForActuators();
  // the pod-restart pass's SchedulePodsRestart is always made
  w.log.erase(std::remove_if(w.log.begin(), w.log.end(), [](const std::string& l) { return l.rfind("restart", 0) == 0; }), w.log.end());
  return err;
}

const std::string R = "GPUDriverUpgrade";
std::string ev(const char* node, const char* type, const std::string& msg) { return std::string("event ") + node + " " + type + " " + R + ": " + msg; }

void cpu_specs(Runner& T) {
  T.it("GetEventReason is the upper-cased driver name + DriverUpgrade", [&] {
    SetDriverName("ofed");
    EXPECT(T, GetEventReason() == "OFEDDriverUpgrade");
    SetDriverName("gpu");
    EXPECT(T, GetEventReason() == "GPUDriverUpgrade");
  });

  T.it("the drain's aggregate error: one message, several messages in first-pod order, a missing DaemonSet", [&] {
    World w;
    w.ds("present");
    w.node("n0", UpgradeStateDrainRequired);
    w.pod("a-bare", "n0", "Running");
    w.pod("b-emptydir", "n0", "Running").OwnerReferences = {{"ReplicaSet", "rs", "u", true}};
    w.pods.back().HasEmptyDirVolume = true;
    w.pod("c-bare", "n0", "Pending");
    w.pod("d-gone", "n0", "Running").OwnerReferences = {{"DaemonSet", "gone", "u", true}};
    w.pod("e-present", "n0", "Running").OwnerReferences = {{"DaemonSet", "present", "u", true}};
    w.pod("f-finished", "n0", "Succeeded");
    w.snapshot();
    StateOptions o = allOn();
    auto m = ClusterUpgradeStateManagerImpl::NewDetached(o);
    w.wire(m.get());
    // the mirror's helper over Encode's bits and the restated chain over the store agree, for every Force / DeleteEmptyDir
    for (int force = 0; force < 2; force++)
      for (int emptyDir = 0; emptyDir < 2; emptyDir++) {
        DriverUpgradePolicySpec p = policy(true, force == 1);
        p.DrainSpec->DeleteEmptyDir = emptyDir == 1;
        EncodedSnapshot e;
        EXPECT(T, !m->Encode(w.state, p, &e));
        const auto& wk = e.workload.at(0);
        const Error mine = DrainFilterError(wk.pods, wk.bits, *p.DrainSpec);
        evspec::DrainHelper h;
        h.client = &w.store; h.Force = force == 1; h.DeleteEmptyDirData = emptyDir == 1;
        std::vector<Pod*> del;
        const Error theirs = h.GetPodsForDeletion("n0", &del);
        EXPECT(T, mine == theirs);
        if (T.failed_here) std::printf("    force %d emptyDir %d: %s / %s\n", force, emptyDir, mine ? mine->c_str() : "nil", theirs ? theirs->c_str() : "nil");
      }
    auto err = [&](bool force, bool emptyDir, std::vector<const Pod*> pods) {
      std::vector<uint16_t> bits;
      for (const Pod* p : pods) {
        uint16_t b = UST_POD_MATCH_DRAIN_SELECTOR | (p->Phase == "Running" ? UST_PHASE_RUNNING : p->Phase == "Pending" ? UST_PHASE_PENDING : UST_PHASE_SUCCEEDED);
        for (const auto& r : p->OwnerReferences)
          if (r.Controller) b |= UST_POD_HAS_CONTROLLER | (r.Kind == "DaemonSet" ? UST_POD_CONTROLLED_BY_DS : 0) | (r.Name == "gone" ? UST_POD_DS_MISSING : 0);
        if (p->HasEmptyDirVolume) b |= UST_POD_HAS_EMPTYDIR;
        bits.push_back(b);
      }
      upgrade::DrainSpec s;
      s.Force = force; s.DeleteEmptyDir = emptyDir;
      return DrainFilterError(pods, bits, s);
    };
    const Pod *a = &w.pods[0], *b = &w.pods[1], *c = &w.pods[2], *d = &w.pods[3], *f = &w.pods[5];
    EXPECT(T, err(false, false, {a, c, f}) == Error("cannot delete Pods declare no controller (use --force to override): apps/a-bare, apps/c-bare"));
    EXPECT(T, err(false, false, {d}) == Error("cannot delete daemonsets.apps \"gone\" not found: apps/d-gone"));
    EXPECT(T, err(false, false, {b, a, d, c}) ==
                  Error("[cannot delete Pods with local storage (use --delete-emptydir-data to override): apps/b-emptydir, "
                        "cannot delete Pods declare no controller (use --force to override): apps/a-bare, apps/c-bare, "
                        "cannot delete daemonsets.apps \"gone\" not found: apps/d-gone]"));
    EXPECT(T, err(true, false, {b, a, d, c}) == Error("cannot delete Pods with local storage (use --delete-emptydir-data to override): apps/b-emptydir"));
    EXPECT(T, !err(true, true, {b, a, d, c, f}));
  });

  const std::string vkey = (SetDriverName("gpu"), GetValidationStartTimeAnnotationKey()), wkey = GetWaitForPodCompletionStartTimeAnnotationKey();
  const uint8_t NONE = UST_OUTCOME_NONE, PDR = UST_STATE_POD_DELETION_REQUIRED, PRR = UST_STATE_POD_RESTART_REQUIRED,
                DRQ = UST_STATE_DRAIN_REQUIRED, FLD = UST_STATE_FAILED, VAL = UST_STATE_VALIDATION_REQUIRED, WFJ = UST_STATE_WAIT_FOR_JOBS_REQUIRED;
  // Every row of the table: a world, the outputs, the error and the log expected.
  struct Row {
    std::string name;
    std::function<void(World&)> setup;
    DriverUpgradePolicySpec p;
    uint8_t next; uint16_t actions; uint8_t outcome;
    Error err;
    std::vector<std::string> log;
  };
  const std::string evict = "evict n0 force=0 emptydir=0 timeout=120 grace=-1: a";
  const std::string drainEvict = "evict n0 force=0 emptydir=0 timeout=60 grace=-1: a";
  const std::string setV = "annotation n0 " + vkey + "=" + std::to_string(kNow), setW = "annotation n0 " + wkey + "=" + std::to_string(kNow);
  const std::string parseErr = "strconv.ParseInt: parsing \"soon\": invalid syntax";
  auto failing = [](const std::string& match) { return [match](World& w) { w.provider.match = match; w.provider.failAt = 0; }; };
  auto notReady = [](World& w, StringMap anno) { w.node("n0", UpgradeStateValidationRequired, std::move(anno)); w.valPod("v", "n0", false); };
  auto waiting = [](World& w, StringMap anno, const char* phase) { w.node("n0", UpgradeStateWaitForJobsRequired, std::move(anno)); w.waitPod("j", "n0", phase); };
  auto deletion = [](World& w) { w.node("n0", UpgradeStatePodDeletionRequired); w.pod("a", "n0", "Running").OwnerReferences = {{"Job", "j", "u", true}}; };
  auto draining = [](World& w) { w.node("n0", UpgradeStateDrainRequired); w.pod("a", "n0", "Running").OwnerReferences = {{"Job", "j", "u", true}}; };
  std::vector<Row> rows = {
      {"validation: the start time does not parse", [&](World& w) { notReady(w, {{vkey, "soon"}}); }, policy(false), VAL, UST_A_ERROR, NONE,
       Errorf("unable to handle timeout for validation state: " + parseErr),
       {ev("n0", "Warning", "Failed to handle timeout for validation state%!(EXTRA string=" + parseErr + ")")}},
      {"validation: setting the start time fails", [&](World& w) { notReady(w, {}); failing("annotation n0 " + vkey)(w); }, policy(false), VAL,
       UST_A_SET_WAIT_START, NONE, Errorf("unable to handle timeout for validation state: provider error on " + setV),
       {"FAILED " + setV, ev("n0", "Warning", "Failed to handle timeout for validation state%!(EXTRA string=provider error on " + setV + ")")}},
      {"validation: timed out, deleting the start time fails", [&](World& w) { notReady(w, {{vkey, "1"}}); failing("annotation n0 " + vkey)(w); },
       policy(false), FLD, UST_A_SET_STATE, NONE,
       Errorf("unable to handle timeout for validation state: provider error on annotation n0 " + vkey + "=null"),
       {"state n0=upgrade-failed", "FAILED annotation n0 " + vkey + "=null",
        ev("n0", "Warning", "Failed to handle timeout for validation state%!(EXTRA string=provider error on annotation n0 " + vkey + "=null)")}},
      {"wait: setting the start time fails", [&](World& w) { waiting(w, {}, "Running"); failing("annotation n0 " + wkey)(w); }, policy(false), WFJ,
       UST_A_SCHEDULE_WAIT_CHECK | UST_A_SET_WAIT_START, NONE, std::nullopt,
       {"FAILED " + setW, ev("n0", "Warning", "Failed to handle timeout for job completions, provider error on " + setW)}},
      {"wait: the start time does not parse", [&](World& w) { waiting(w, {{wkey, "soon"}}, "Pending"); }, policy(false), WFJ,
       UST_A_SCHEDULE_WAIT_CHECK, NONE, std::nullopt, {ev("n0", "Warning", "Failed to handle timeout for job completions, " + parseErr)}},
      {"wait: the start time does not parse, but no timeout is set: no event", [&](World& w) { waiting(w, {{wkey, "soon"}}, "Running"); },
       policy(false, false, 0), WFJ, UST_A_SCHEDULE_WAIT_CHECK, NONE, std::nullopt, {}},
      {"wait: timed out, deleting the start time fails", [&](World& w) { waiting(w, {{wkey, "1"}}, "Running"); failing("annotation n0 " + wkey)(w); },
       policy(false), WFJ, UST_A_SCHEDULE_WAIT_CHECK, PDR, std::nullopt,
       {"state n0=pod-deletion-required", "FAILED annotation n0 " + wkey + "=null",
        ev("n0", "Warning", "Failed to handle timeout for job completions, provider error on annotation n0 " + wkey + "=null")}},
      {"wait: jobs done, deleting the start time fails: no state change", [&](World& w) { waiting(w, {{wkey, "1"}}, "Succeeded"); failing("annotation n0 " + wkey)(w); },
       policy(false), WFJ, UST_A_SCHEDULE_WAIT_CHECK, PDR, std::nullopt,
       {"FAILED annotation n0 " + wkey + "=null",
        ev("n0", "Warning", "Failed to remove annotation used to track job completions: provider error on annotation n0 " + wkey + "=null")}},
      {"pod deletion: evicted", deletion, policy(false), PDR, UST_A_SCHEDULE_POD_EVICTION, PRR, std::nullopt,
       {evict, "state n0=pod-restart-required", ev("n0", "Normal", "Deleted workload pods on the node for the driver upgrade")}},
      {"pod deletion: eviction fails, drain on", [&](World& w) { deletion(w); w.evictor.failNode = "n0"; }, policy(true), PDR,
       UST_A_SCHEDULE_POD_EVICTION, PRR, std::nullopt,
       {"FAILED " + evict, ev("n0", "Warning", "Failed to delete workload pods on the node for the driver upgrade, eviction failed"),
        ev("n0", "Warning", "Pod deletion failed but drain is enabled in spec. Will attempt a node drain"), "state n0=drain-required"}},
      {"pod deletion: eviction fails, drain off", [&](World& w) { deletion(w); w.evictor.failNode = "n0"; }, policy(false), PDR,
       UST_A_SCHEDULE_POD_EVICTION, PRR, std::nullopt,
       {"FAILED " + evict, ev("n0", "Warning", "Failed to delete workload pods on the node for the driver upgrade, eviction failed"),
        "state n0=upgrade-failed"}},
      {"pod deletion: a count mismatch, drain on", deletion, policy(true), PDR, UST_A_SCHEDULE_POD_EVICTION, DRQ, std::nullopt,
       {ev("n0", "Warning", "Pod deletion failed but drain is enabled in spec. Will attempt a node drain"), "state n0=drain-required"}},
      {"pod deletion: a count mismatch, drain off: no event", deletion, policy(false), PDR, UST_A_SCHEDULE_POD_EVICTION, FLD, std::nullopt,
       {"state n0=upgrade-failed"}},
      {"drain: drained", draining, policy(true), DRQ, UST_A_SCHEDULE_DRAIN, PRR, std::nullopt,
       {ev("n0", "Normal", "Scheduling drain of the node"), "cordon n0", drainEvict, ev("n0", "Normal", "Successfully drained the node"),
        "state n0=pod-restart-required"}},
      {"drain: the cordon fails", [&](World& w) { draining(w); w.cordon.failNode = "n0"; }, policy(true), DRQ, UST_A_SCHEDULE_DRAIN, PRR,
       std::nullopt,
       {ev("n0", "Normal", "Scheduling drain of the node"), "FAILED cordon n0", "state n0=upgrade-failed",
        ev("n0", "Warning", "Failed to cordon the node, cordon failed")}},
      {"drain: the eviction fails", [&](World& w) { draining(w); w.evictor.failNode = "n0"; }, policy(true), DRQ, UST_A_SCHEDULE_DRAIN, PRR,
       std::nullopt,
       {ev("n0", "Normal", "Scheduling drain of the node"), "cordon n0", "FAILED " + drainEvict, "state n0=upgrade-failed",
        ev("n0", "Warning", "Failed to drain the node, eviction failed")}},
      {"drain: error pods", [&](World& w) { draining(w); w.pod("b", "n0", "Running"); w.pod("c", "n0", "Running").OwnerReferences = {{"DaemonSet", "gone", "u", true}}; },
       policy(true), DRQ, UST_A_SCHEDULE_DRAIN, FLD, std::nullopt,
       {ev("n0", "Normal", "Scheduling drain of the node"), "cordon n0", "state n0=upgrade-failed",
        ev("n0", "Warning", "Failed to drain the node, [cannot delete Pods declare no controller (use --force to override): apps/b, "
                            "cannot delete daemonsets.apps \"gone\" not found: apps/c]")}},
  };
  T.it("Replay: every row of the events table, its type, reason, message and place among the node's calls", [&] {
    for (const Row& r : rows) {
      World w;
      r.setup(w);
      const Error err = replayOne(w, allOn(), r.p, r.next, r.actions, r.outcome);
      const bool good = err == r.err && w.log == r.log;
      EXPECT(T, good);
      if (!good) {
        std::printf("    %s: %s\n", r.name.c_str(), err ? err->c_str() : "nil");
        for (const auto& s : w.log) std::printf("      got:  %s\n", s.c_str());
        for (const auto& s : r.log) std::printf("      want: %s\n", s.c_str());
      }
    }
  });
  T.it("a null recorder leaves every call as it was; with the options off the mirror records nothing", [&] {
    for (const Row& r : rows) {
      World w;
      r.setup(w);
      const Error err = replayOne(w, allOn(), r.p, r.next, r.actions, r.outcome, false);
      EXPECT(T, err == r.err && w.log == withoutEvents(r.log));
      // options off: the same outputs go to the restated managers, whose recorder is a different one
      World x;
      r.setup(x);
      evspec::LogRecorder mirror;
      std::vector<std::string> mlog;
      mirror.log = &mlog;
      x.snapshot();
      StateOptions off;
      off.Now = [] { return kNow; };
      auto m = ClusterUpgradeStateManagerImpl::NewDetached(off);
      x.wire(m.get());
      m->EventRecorder = &mirror;
      EncodedSnapshot e;
      EXPECT(T, !m->Encode(x.state, r.p, &e));
      ust_counters k{};
      k.error_index = -1; k.error_pass = -1;
      const uint16_t a = r.actions & ~(uint16_t)UST_A_ERROR;
      (void)m->Replay(e, r.p, &r.next, &a, UST_OK, k, &r.outcome);
      m->WaitForActuators();
      EXPECT(T, mirror.events == 0);
      if (T.failed_here) std::printf("    %s\n", r.name.c_str());
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

void printDiff(const std::vector<std::string>& a, const std::vector<std::string>& b) {
  const auto pa = byNode(a), pb = byNode(b);
  for (const auto& kv : pa)
    if (!pb.count(kv.first) || pb.at(kv.first) != kv.second)
      for (const auto& s : kv.second) std::printf("    ref %s: %s\n", kv.first.c_str(), s.c_str());
  for (const auto& kv : pb)
    if (!pa.count(kv.first) || pa.at(kv.first) != kv.second)
      for (const auto& s : kv.second) std::printf("    dev %s: %s\n", kv.first.c_str(), s.c_str());
}

void gpu_specs(Runner& T, bool* ok) {
  SetDriverName("gpu");
  // One cluster through ApplyState with the restated managers and their events, and through ApplyState and
  // ApplyStateIncremental with all three options and the mirror's events: the same calls and events per node.
  using Setup = std::function<void(World&)>;
  auto both = [&](const char* name, const DriverUpgradePolicySpec& p, const Setup& setup) {
    T.it(name, [&] {
      World a, b, c;
      for (World* w : {&a, &b, &c}) { setup(*w); w->snapshot(); }
      StateOptions off;
      off.Now = [] { return kNow; };
      auto ma = device(off, ok), mb = device(allOn(), ok), mc = device(allOn(), ok);
      a.wire(ma.get()); b.wire(mb.get()); c.wire(mc.get());
      const Error ea = ma->ApplyState(&a.state, &p), eb = mb->ApplyState(&b.state, &p), ec = mc->ApplyStateIncremental(&c.state, &p);
      mb->WaitForActuators(); mc->WaitForActuators();
      EXPECT(T, ea == eb && ea == ec);
      EXPECT(T, byNode(a.log) == byNode(b.log) && byNode(b.log) == byNode(c.log));
      EXPECT(T, a.image() == b.image() && b.image() == c.image());
      EXPECT(T, a.recorder.events > 0 && b.recorder.events == a.recorder.events);
      if (T.failed_here) printDiff(a.log, b.log);
    });
  };
  const std::string vkey = GetValidationStartTimeAnnotationKey(), wkey = GetWaitForPodCompletionStartTimeAnnotationKey();
  // pod_manager_test.go:226-430
  auto gpuPods = [](bool allEmptyDir) {
    return [=](World& w) {
      w.node("n0", UpgradeStatePodDeletionRequired);
      w.pod("cpu-pod", "n0", "Running", false);
      w.pod("gpu-pod1", "n0", "Running").HasEmptyDirVolume = allEmptyDir;
      if (!allEmptyDir) w.pod("gpu-pod2", "n0", "Running");
    };
  };
  auto withSpec = [](bool drain, bool force, bool emptyDir) {
    DriverUpgradePolicySpec p = policy(drain, force);
    p.PodDeletion->DeleteEmptyDir = emptyDir;
    return p;
  };
  both("events: standalone gpu pods with force are deleted (pod_manager_test.go:236)", withSpec(false, true, false), gpuPods(false));
  both("events: without force, drain enabled: drain-required (:300)", withSpec(true, false, false), gpuPods(false));
  both("events: emptyDir, force, no deleteEmptyDir, drain enabled (:399)", withSpec(true, true, false), gpuPods(true));
  both("events: an eviction that fails, drain on and off", policy(true), [](World& w) {
    w.node("n0", UpgradeStatePodDeletionRequired); w.pod("a", "n0", "Running").OwnerReferences = {{"Job", "j", "u", true}};
    w.evictor.failNode = "n0";
  });
  // drain_manager_test.go:33-161
  both("events: DrainManager should drain nodes (drain_manager_test.go:33)", policy(true, true), [](World& w) {
    w.node("n0", UpgradeStateDrainRequired); w.pod("p", "n0", "Running", false);
  });
  both("events: DrainManager should drain all nodes it receives (:55)", policy(true, true), [](World& w) {
    for (int i = 0; i < 3; i++) w.node("n" + std::to_string(i), UpgradeStateDrainRequired);
  });
  both("events: a drain with error pods of each kind, a failed cordon and a failed eviction", policy(true), [](World& w) {
    w.node("n0", UpgradeStateDrainRequired);
    w.pod("a", "n0", "Running");
    w.pod("b", "n0", "Running").OwnerReferences = {{"DaemonSet", "gone", "u", true}};
    w.pod("c", "n0", "Running").OwnerReferences = {{"ReplicaSet", "rs", "u", true}};
    w.pods.back().HasEmptyDirVolume = true;
    w.node("n1", UpgradeStateDrainRequired);
    w.node("n2", UpgradeStateDrainRequired);
    w.pod("d", "n2", "Running").OwnerReferences = {{"Job", "j", "u", true}};
    w.cordon.failNode = "n1";
    w.evictor.failNode = "n2";
  });
  // pod_manager_test.go ScheduleCheckOnPodCompletion, validation_manager_test.go, with the failures that record events
  both("events: wait checks: start set, timed out, done, unparsable, failing writes", policy(false), [wkey](World& w) {
    w.node("n0", UpgradeStateWaitForJobsRequired); w.waitPod("j0", "n0", "Running");
    w.node("n1", UpgradeStateWaitForJobsRequired, {{wkey, "1"}}); w.waitPod("j1", "n1", "Running");
    w.node("n2", UpgradeStateWaitForJobsRequired, {{wkey, "1"}}); w.waitPod("j2", "n2", "Succeeded");
    w.node("n3", UpgradeStateWaitForJobsRequired, {{wkey, "later"}}); w.waitPod("j3", "n3", "Pending");
    w.node("n4", UpgradeStateWaitForJobsRequired); w.waitPod("j4", "n4", "Running");
    w.node("n5", UpgradeStateWaitForJobsRequired, {{wkey, "1"}}); w.waitPod("j5", "n5", "Failed");
    w.provider.match = "annotation n4 " + wkey; w.provider.failAt = 0;
  });
  both("events: wait checks: a timed-out node whose start-time delete fails", policy(false), [wkey](World& w) {
    w.node("n1", UpgradeStateWaitForJobsRequired, {{wkey, "1"}}); w.waitPod("j1", "n1", "Running");
    w.node("n2", UpgradeStateWaitForJobsRequired, {{wkey, "1"}}); w.waitPod("j2", "n2", "Succeeded");
    w.provider.match = wkey + "=null"; w.provider.failAt = 0;
  });
  both("events: validation: the start time does not parse", policy(false), [vkey](World& w) {
    w.node("n0", UpgradeStateValidationRequired, {{vkey, "later"}}); w.valPod("v", "n0", false);
  });
  both("events: validation: timed out, the start-time delete fails", policy(false), [vkey](World& w) {
    w.node("n0", UpgradeStateValidationRequired, {{vkey, "1"}}); w.valPod("v", "n0", false);
    w.provider.match = "annotation n0 " + vkey; w.provider.failAt = 0;
  });
}

// The reconcile loop: nodes that come back into the four states, wait and validation pods that start, finish and turn
// ready, workload pods of every filter kind, start times that do not parse, writes, cordons and evictions that fail,
// DaemonSets that disappear, nodes that join, leave and move; the clock moves two minutes per reconcile.
void evolve(World& w, spec::BLcg r, int rec) {
  const std::string vkey = GetValidationStartTimeAnnotationKey(), wkey = GetWaitForPodCompletionStartTimeAnnotationKey();
  const char* states[] = {UpgradeStatePodDeletionRequired, UpgradeStateDrainRequired, UpgradeStateWaitForJobsRequired,
                          UpgradeStateValidationRequired, UpgradeStateDone, UpgradeStateCordonRequired, UpgradeStateUpgradeRequired};
  w.now += 120;
  for (size_t i = 0; i < w.nodes.size(); i++) {
    if (w.pos[i] < 0) continue;
    Node& n = w.nodes[i];
    for (const std::string& k : {vkey, wkey}) {
      auto it = n.Annotations.find(k);
      if (it != n.Annotations.end() && it->second == "garbage") { n.Annotations.erase(it); spec::LogProvider::bump(&n); }
    }
    const std::string st = n.Labels[GetUpgradeStateLabelKey()];
    const bool busy = st == UpgradeStatePodDeletionRequired || st == UpgradeStateDrainRequired || st == UpgradeStateWaitForJobsRequired ||
                      st == UpgradeStateValidationRequired;
    if (!busy && r.chance(20)) { n.Labels[GetUpgradeStateLabelKey()] = states[r.next() % 4]; spec::LogProvider::bump(&n); }
    if (r.chance(4)) { n.Annotations[r.chance(50) ? vkey : wkey] = "garbage"; spec::LogProvider::bump(&n); }
    if (r.chance(1)) w.pos[i] = -1;
  }
  for (size_t i = 0; i < w.pods.size(); i++) {
    if (!w.podAlive[i]) continue;
    Pod& p = w.pods[i];
    if (p.Labels.count("app") && p.Labels.at("app") == "validator") {
      if (r.chance(20)) { p.ContainerStatuses = {{r.chance(50), 0}}; w.bump(p); }
    } else if (r.chance(5)) { p.Phase = r.chance(50) ? "Succeeded" : "Failed"; w.bump(p); }
    else if (r.chance(2)) { p.HasEmptyDirVolume = true; w.bump(p); }
    else if (r.chance(2)) w.podAlive[i] = 0;
  }
  for (size_t i = 0; i < w.nodes.size(); i++) {
    if (w.pos[i] < 0) continue;
    const std::string n = w.nodes[i].Name, tag = std::to_string(rec) + "-" + n;
    if (r.chance(6)) {
      Pod& p = w.pod("p" + tag, n, r.chance(80) ? "Running" : "Pending", r.chance(70));
      const int kind = (int)(r.next() % 5);
      if (kind == 1) p.OwnerReferences = {{"ReplicaSet", "rs", "u", true}};
      if (kind == 2) p.OwnerReferences = {{"DaemonSet", "ds" + std::to_string(r.next() % 3), "u", true}};
      if (kind == 3) p.Annotations["kubernetes.io/config.mirror"] = "m";
      p.HasEmptyDirVolume = r.chance(10);
    }
    if (r.chance(4)) w.waitPod("w" + tag, n, r.chance(70) ? "Running" : "Succeeded");
    if (r.chance(4)) w.valPod("v" + tag, n, r.chance(50));
  }
  if (rec % 50 == 10 && !w.dss.empty()) w.dss.pop_back();
  if (rec % 50 == 30) w.ds("ds" + std::to_string(w.dss.size()));
  for (int j = (int)(r.next() % 3); j > 0; j--) {
    w.node("j" + std::to_string(rec) + "-" + std::to_string(j), states[r.next() % 7]);
    w.pos.back() = (int)(r.next() % (w.pos.size() + 1)) * 2 + 1;
  }
  int k = 0;
  std::vector<std::pair<int, size_t>> order;
  for (size_t i = 0; i < w.nodes.size(); i++)
    if (w.pos[i] >= 0) order.emplace_back(w.pos[i] * 2, i);
  std::sort(order.begin(), order.end());
  for (auto& o : order) w.pos[o.second] = k++;
  if (order.size() > 4 && r.chance(30)) std::swap(w.pos[order[1].second], w.pos[order[order.size() - 2].second]);
}

void loop(Runner& T, bool requestor, bool val, bool wait, bool evict, int n_nodes, int rounds, std::vector<int>* fired, bool* ok) {
  SetDriverName("gpu");
  const std::string vkey = GetValidationStartTimeAnnotationKey(), wkey = GetWaitForPodCompletionStartTimeAnnotationKey();
  const std::string opts = val && wait && evict ? "all three options" : val ? "ValidateOnDevice alone" : wait ? "WaitForCompletionOnDevice alone"
                                                                                                            : "EvictionOnDevice alone";
  const std::string name = "ApplyStateIncremental with " + opts + " records the events ApplyState with the restated managers records (" +
                           (requestor ? "requestor" : "in-place") + " mode)";
  T.it(name.c_str(), [&] {
    World a, b;
    spec::BLcg seed{4242};
    for (World* w : {&a, &b}) {
      spec::BLcg r = seed;
      w->ds("ds0"); w->ds("ds1"); w->ds("ds2");
      for (int i = 0; i < n_nodes; i++) {
        const char* states[] = {UpgradeStatePodDeletionRequired, UpgradeStateDrainRequired, UpgradeStateWaitForJobsRequired,
                                UpgradeStateValidationRequired, UpgradeStateDone};
        const std::string n = "n" + std::to_string(i);
        w->node(n, states[r.next() % 5]);
        for (int j = (int)(r.next() % 3); j > 0; j--) w->pod("p" + std::to_string(j) + "-" + n, n, "Running", r.chance(60));
        if (r.chance(50)) w->waitPod("w-" + n, n, "Running");
        if (r.chance(50)) w->valPod("v-" + n, n, r.chance(50));
      }
    }
    StateOptions o;
    o.Requestor.UseMaintenanceOperator = requestor;
    o.Now = [&a] { return a.now; };
    StateOptions od = o;
    od.Now = [&b] { return b.now; };
    od.ValidateOnDevice = val; od.WaitForCompletionOnDevice = wait; od.EvictionOnDevice = evict;
    auto ma = device(o, ok), mb = device(od, ok);
    a.wire(ma.get()); b.wire(mb.get());
    DriverUpgradePolicySpec p = policy(true);
    std::vector<int> here(evspec::rows().size(), 0);
    for (int rec = 0; rec < rounds; rec++) {
      p.DrainSpec->PodSelector = (rec / 60) % 2 ? "app=train" : "";
      p.PodDeletion->Force = p.DrainSpec->Force = rec % 7 == 3;
      p.PodDeletion->DeleteEmptyDir = p.DrainSpec->DeleteEmptyDir = rec % 5 == 1;
      p.DrainSpec->Enable = rec % 11 != 4;
      a.snapshot(); b.snapshot();
      a.log.clear(); b.log.clear();
      auto first = [&](const char* label) {
        auto it = a.state.NodeStates.find(label);
        return it == a.state.NodeStates.end() || it->second.empty() ? std::string() : it->second[0]->Node->Name;
      };
      for (World* w : {&a, &b}) {
        w->evictor.failNode = rec % 3 == 1 ? first(UpgradeStatePodDeletionRequired) : "";
        w->cordon.failNode = rec % 5 == 2 ? first(UpgradeStateDrainRequired) : "";
        const std::string wn = first(UpgradeStateWaitForJobsRequired), vn = first(UpgradeStateValidationRequired);
        w->provider.match = rec % 4 == 0 && !wn.empty() ? "annotation " + wn + " " + wkey : rec % 4 == 2 && !vn.empty() ? "annotation " + vn + " " + vkey : "";
        w->provider.failAt = 0; w->provider.seen = 0;
      }
      const Error ea = ma->ApplyState(&a.state, &p);
      const Error eb = mb->ApplyStateIncremental(&b.state, &p);
      mb->WaitForActuators();
      EXPECT(T, ea == eb);
      EXPECT(T, byNode(a.log) == byNode(b.log));
      EXPECT(T, a.image() == b.image());
      for (const std::string& s : b.log) {  // the mirror's own events: the rows of the options that are on
        const int row = evspec::rowOf(s);
        if (row >= 0 && (row == 0 ? val : row <= 2 ? wait : evict)) here[(size_t)row]++;
      }
      if (T.failed_here) {
        std::printf("    (reconcile %d: %s / %s)\n", rec, ea ? ea->c_str() : "ok", eb ? eb->c_str() : "ok");
        printDiff(a.log, b.log);
        break;
      }
      evolve(a, spec::BLcg{9000u + (uint64_t)rec}, rec); evolve(b, spec::BLcg{9000u + (uint64_t)rec}, rec);
    }
    std::printf("    events by row:");
    for (size_t i = 0; i < here.size(); i++) { std::printf(" %d", here[i]); (*fired)[i] += here[i]; }
    std::printf("\n");
    // each option records its own rows
    const bool vRows = here[0] > 0, wRows = here[1] > 0 && here[2] > 0;
    bool eRows = true;
    for (size_t i = 3; i < here.size(); i++) eRows = eRows && here[i] > 0;
    EXPECT(T, (!val || vRows) && (!wait || wRows) && (!evict || eRows));
  });
}

}  // namespace

int main(int argc, char** argv) {
  const bool gpu = argc > 1 && std::strcmp(argv[1], "--gpu") == 0;
  Runner R;
  bool ok = true;
  if (gpu) {
    gpu_specs(R, &ok);
    std::vector<int> fired(evspec::rows().size(), 0);
    for (bool requestor : {false, true}) {
      loop(R, requestor, true, true, true, 80, 300, &fired, &ok);
      loop(R, requestor, true, false, false, 80, 300, &fired, &ok);
      loop(R, requestor, false, true, false, 80, 300, &fired, &ok);
      loop(R, requestor, false, false, true, 80, 300, &fired, &ok);
    }
    R.it("every row of the events table fired in the loops", [&] {
      for (size_t i = 0; i < fired.size(); i++) {
        EXPECT(R, fired[i] > 0);
        if (fired[i] == 0) std::printf("    never: %s\n", evspec::rows()[i].c_str());
      }
    });
  } else {
    cpu_specs(R);
  }
  std::printf("# %d passed, %d failed\n", R.passed, R.failed);
  return (R.failed == 0 && ok) ? 0 : 1;
}
