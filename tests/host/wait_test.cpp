// StateOptions::WaitForCompletionOnDevice (wait_spec.hpp).
//   wait_test         host halves only: Encode's wait pods, phases, start column and WAIT_START bits, alone and after the
//                     validation pods; what ApplyStateIncremental hands to the device (a stand-in records it): replaced
//                     lists and nodes, nothing for a time-only reconcile; Replay of hand-made outputs through pass 4, both
//                     pod-deletion-required call orders, swallowed provider errors and the List's error
//   wait_test --gpu   the reference's wait-for-completion specs through ApplyState, the host's running bit against the
//                     device's outcome, a time-only reconcile, and a reconcile loop of BuildStateIncremental +
//                     ApplyStateIncremental with the option against BuildState + ApplyState with the restated PodManagerImpl
#include <cstdlib>
#include <cstring>
#include <set>

#include "wait_spec.hpp"

using namespace upgrade;
using namespace wspec;

namespace {

const char* kWait = "app=my-app";
const char* kValidation = "app=validator,tier=gpu";

// A one-bucket-per-label cluster built by hand: nodes with a driver pod each, in ListIndex order.
struct Small {
  std::deque<Node> nodes;
  std::deque<Pod> drivers, pods;
  DaemonSet ds;
  ClusterUpgradeState state;
  std::vector<std::unique_ptr<NodeUpgradeState>> owned;
  std::vector<std::string> log;
  ApiProvider provider;
  spec::LogCordon cordon;
  spec::LogDrain drain;
  CountingPods podm;
  SafeDriverLoadManagerImpl safeLoad{&provider};
  vspec::SelectorClient client;
  Small() { provider.log = cordon.log = drain.log = podm.log = &log; ds.Name = "driver"; ds.UID = "uid-ds"; }
  Node& node(const std::string& name, const std::string& label, StringMap annotations = {}) {
    nodes.emplace_back();
    Node& n = nodes.back();
    n.Name = name;
    n.ResourceVersion = "1";
    n.Labels[GetUpgradeStateLabelKey()] = label;
    n.Annotations = std::move(annotations);
    provider.nodes[name] = &n;
    drivers.emplace_back();
    Pod& d = drivers.back();
    d.Name = "drv-" + name; d.Namespace = "gpu-operator"; d.NodeName = name; d.ResourceVersion = "1";
    d.OwnerReferences.push_back({"DaemonSet", "driver", ds.UID});
    d.Labels[PodControllerRevisionHashLabelKey] = "test-hash-12345";
    d.Phase = "Running"; d.ContainerStatuses = {{true, 0}};
    return n;
  }
  Pod& wpod(const std::string& name, const std::string& node, const std::string& phase, int64_t rv = 1) {
    pods.push_back(makeWaitPod(name, node, phase, rv));
    return pods.back();
  }
  void snapshot() {
    state = ClusterUpgradeState();
    owned.clear();
    for (size_t i = 0; i < nodes.size(); i++) {
      auto e = std::make_unique<NodeUpgradeState>();
      e->Node = &nodes[i]; e->DriverPod = &drivers[i]; e->DriverDaemonSet = &ds; e->ListIndex = (int64_t)i;
      state.NodeStates[nodes[i].Labels[GetUpgradeStateLabelKey()]].push_back(e.get());
      owned.push_back(std::move(e));
    }
    client.all.clear();
    for (Pod& p : pods) client.all.push_back(&p);
    std::stable_sort(client.all.begin(), client.all.end(), [](const Pod* x, const Pod* y) { return x->Name < y->Name; });
  }
  void wire(ClusterUpgradeStateManagerImpl* m) {
    m->NodeUpgradeStateProvider = &provider; m->CordonManager = &cordon; m->DrainManager = &drain; m->PodManager = &podm;
    m->SafeDriverLoadManager = &safeLoad; m->K8sClient = &client;
  }
  std::string image() const {
    std::string s;
    for (const Node& n : nodes) {
      s += n.Name + "{" + n.Labels.at(GetUpgradeStateLabelKey()) + (n.Unschedulable ? ",U" : "");
      for (const auto& kv : n.Annotations) s += "," + kv.first + "=" + kv.second;
      s += "}";
    }
    return s;
  }
  std::vector<std::string> calls() const {  // the log without the pod-restart pass's SchedulePodsRestart, which is always made
    std::vector<std::string> out;
    for (const std::string& l : log)
      if (l != "restart") out.push_back(l);
    return out;
  }
};

DriverUpgradePolicySpec waitPolicy(int timeout, const std::string& selector = kWait) {
  DriverUpgradePolicySpec p;
  p.AutoUpgrade = true;
  p.WaitForCompletion = WaitForCompletionSpec{selector, timeout};
  return p;
}

// What ApplyStateIncremental hands to the device, recorded; the outputs are "no transition, no call".
struct StandIn : ClusterUpgradeStateManagerImpl {
  struct Call {
    bool full = false;
    int64_t now = 0, waitTimeout = 0;
    std::vector<int64_t> changed, startOfChanged, listed, run_src, insertStart;
    std::vector<std::vector<uint16_t>> lists;
    int32_t evaluate = 0;
  };
  std::vector<Call> calls;
  explicit StandIn(StateOptions o) : ClusterUpgradeStateManagerImpl(std::move(o)) {}
  static void quiet(Cache* k) {
    const size_t n = k->slots.size();
    k->next.assign(n + 1, 0);
    k->actions.assign(n + 1, 0);
    k->outcome.assign(n + 1, UST_OUTCOME_NONE);
    for (size_t i = 0; i < n; i++) k->next[i] = k->state[i] & UST_HOT_STATE_MASK;
  }
  int EvaluateCached(const ust_policy& policy, bool full, const std::vector<int64_t>& changed, Cache* k, ust_counters* c) override {
    Call call;
    call.full = full; call.changed = changed; call.evaluate = policy.evaluate_actuators;
    calls.push_back(call);
    quiet(k);
    std::memset(c, 0, sizeof(*c));
    c->error_index = -1;
    return UST_OK;
  }
  int EvaluateCachedPods(const ust_policy& policy, int64_t now, int64_t waitTimeout, bool full, const std::vector<int64_t>& changed,
                         Cache* k, ust_counters* c) override {
    Call call;
    call.full = full; call.now = now; call.waitTimeout = waitTimeout; call.changed = changed; call.listed = k->listChanged;
    call.run_src = k->pending.run_src; call.evaluate = policy.evaluate_actuators;
    for (int64_t i : changed) call.startOfChanged.push_back(k->start[(size_t)i]);
    for (int64_t i : k->pending.insert_at) call.insertStart.push_back(k->start[(size_t)i]);
    for (int64_t i : k->listChanged) call.lists.push_back(k->lists[(size_t)i]);
    calls.push_back(call);
    quiet(k);
    std::memset(c, 0, sizeof(*c));
    c->error_index = -1;
    return UST_OK;
  }
};

const uint16_t W = UST_POD_MATCH_WAIT_SELECTOR, V = UST_POD_MATCH_VALIDATION_SELECTOR, RDY = UST_POD_READY;

void cpu_specs(Runner& R) {
  SetDriverName("gpu");
  const std::string wkey = GetWaitForPodCompletionStartTimeAnnotationKey();

  R.it("Encode: one wait List, every node's wait pods with their phases, the start column and the WAIT_START bits", [&] {
    Small w;
    w.node("n0", UpgradeStateWaitForJobsRequired);
    w.node("n1", UpgradeStateWaitForJobsRequired, {{wkey, "1700000000"}});
    w.node("n2", UpgradeStateWaitForJobsRequired, {{wkey, "12x"}});
    w.node("n3", UpgradeStateWaitForJobsRequired, {{wkey, "9223372036854775807"}});
    w.node("n4", UpgradeStateWaitForJobsRequired, {{wkey, "9223372036854775808"}});
    w.node("n5", UpgradeStateDone, {{wkey, "55"}});
    w.node("n6", UpgradeStateWaitForJobsRequired, {{wkey, ""}});
    w.wpod("a-run", "n0", "Running");
    w.wpod("b-pend", "n0", "Pending");
    w.wpod("c-ok", "n0", "Succeeded");
    w.wpod("d-fail", "n0", "Failed");
    w.wpod("e-unknown", "n0", "Unknown");
    w.wpod("f-empty", "n0", "");
    w.wpod("g-done", "n1", "Succeeded");
    w.wpod("h-elsewhere", "n5", "Running");
    w.wpod("i-unscheduled", "", "Pending");
    w.wpod("j-other-app", "n1", "Running").Labels["app"] = "something-else";
    w.snapshot();
    StateOptions o;
    o.WaitForCompletionOnDevice = true;
    o.Now = [] { return (int64_t)1700000123; };
    auto m = ClusterUpgradeStateManagerImpl::NewDetached(o);
    w.wire(m.get());
    const DriverUpgradePolicySpec p = waitPolicy(30);
    EncodedSnapshot e;
    EXPECT(R, !m->Encode(w.state, p, &e).has_value());
    EXPECT(R, w.client.lists == 1);
    EXPECT(R, e.waitOnDevice && !e.validateOnDevice && e.now == 1700000123 && !e.waitListError && !e.listError);
    EXPECT(R, e.policy.evaluate_actuators == (int32_t)UST_EVAL_ACTUATORS && e.policy.wait_timeout_nonzero == 1);
    EXPECT(R, e.pod_off.size() == e.entries.size() + 1 && e.start.size() == e.entries.size() && e.waitRunning.size() == e.entries.size());
    std::map<std::string, std::vector<uint16_t>> lists;
    std::map<std::string, std::pair<uint32_t, int64_t>> bits;
    std::map<std::string, bool> running;
    for (size_t i = 0; i < e.entries.size(); i++) {
      const std::string& n = e.entries[i]->Node->Name;
      lists[n] = std::vector<uint16_t>(e.pod_flags.begin() + e.pod_off[i], e.pod_flags.begin() + e.pod_off[i + 1]);
      bits[n] = {e.flags[i] & (UST_F_WAIT_START_ANNO | UST_F_WAIT_START_INVALID | UST_F_WAIT_TIMED_OUT | UST_F_WAIT_PODS_RUNNING), e.start[i]};
      running[n] = e.waitRunning[i] != 0;
    }
    EXPECT(R, (lists["n0"] == std::vector<uint16_t>{(uint16_t)(W | UST_PHASE_RUNNING), (uint16_t)(W | UST_PHASE_PENDING),
                                                    (uint16_t)(W | UST_PHASE_SUCCEEDED), (uint16_t)(W | UST_PHASE_FAILED),
                                                    (uint16_t)(W | UST_PHASE_OTHER), (uint16_t)(W | UST_PHASE_OTHER)}));
    EXPECT(R, (lists["n1"] == std::vector<uint16_t>{(uint16_t)(W | UST_PHASE_SUCCEEDED)}));
    EXPECT(R, lists["n2"].empty() && lists["n3"].empty() && lists["n6"].empty());
    EXPECT(R, (lists["n5"] == std::vector<uint16_t>{(uint16_t)(W | UST_PHASE_RUNNING)}));  // every node gets its list
    EXPECT(R, running["n0"] && !running["n1"] && !running["n2"] && running["n5"]);
    const uint32_t A = UST_F_WAIT_START_ANNO, I = UST_F_WAIT_START_INVALID;
    EXPECT(R, bits["n0"] == std::make_pair(0u, (int64_t)0));
    EXPECT(R, bits["n1"] == std::make_pair(A, (int64_t)1700000000));
    EXPECT(R, bits["n2"] == std::make_pair(A | I, (int64_t)0));
    EXPECT(R, bits["n3"] == std::make_pair(A, (int64_t)INT64_MAX));
    EXPECT(R, bits["n4"] == std::make_pair(A | I, (int64_t)0));  // one past INT64_MAX: out of range
    EXPECT(R, bits["n5"] == std::make_pair(A, (int64_t)0));      // the start column is state-dependent
    EXPECT(R, bits["n6"] == std::make_pair(A | I, (int64_t)0));  // present but empty
    EXPECT(R, e.deferred.empty());                               // the check swallows a parse error
    // without the option, and with the option but no selector, nothing changes
    for (int variant = 0; variant < 2; variant++) {
      StateOptions q = o;
      q.WaitForCompletionOnDevice = variant == 1;
      auto plain = ClusterUpgradeStateManagerImpl::NewDetached(q);
      w.wire(plain.get());
      EncodedSnapshot x;
      const DriverUpgradePolicySpec px = variant == 0 ? waitPolicy(30) : waitPolicy(30, "");
      EXPECT(R, !plain->Encode(w.state, px, &x).has_value());
      EXPECT(R, !x.waitOnDevice && x.pod_off.empty() && x.start.empty() && x.waitRunning.empty() && x.policy.evaluate_actuators == 0);
      bool same = x.flags.size() == e.flags.size();
      for (size_t i = 0; same && i < x.flags.size(); i++) same = x.flags[i] == (e.flags[i] & ~(A | I)) && x.state[i] == e.state[i];
      EXPECT(R, same);
    }
    EXPECT(R, w.client.lists == 1);
  });

  R.it("Encode with ValidateOnDevice too: two Lists, validation pods first, a pod both selectors match in the list twice", [&] {
    Small w;
    w.node("n0", UpgradeStateValidationRequired, {{GetValidationStartTimeAnnotationKey(), "600"}, {wkey, "700"}});
    w.node("n1", UpgradeStateWaitForJobsRequired, {{GetValidationStartTimeAnnotationKey(), "600"}, {wkey, "700"}});
    w.node("n2", UpgradeStateDone);
    w.pods.push_back(vspec::makeValidationPod("a-val", "n0", true, {true}, 1));
    w.wpod("b-job", "n0", "Running").Labels["tier"] = "gpu";
    w.pods.push_back(vspec::makeValidationPod("c-both", "n1", true, {false}, 1));  // the validation pods match "tier=gpu" too
    w.wpod("d-job", "n1", "Succeeded").Labels["tier"] = "gpu";
    w.snapshot();
    StateOptions o;
    o.WaitForCompletionOnDevice = true;
    o.ValidateOnDevice = true;
    auto m = ClusterUpgradeStateManagerImpl::NewDetached(o);
    w.wire(m.get());
    m->WithValidationEnabled("tier=gpu,app=validator");
    EncodedSnapshot e;
    EXPECT(R, !m->Encode(w.state, waitPolicy(30, "tier=gpu"), &e).has_value());
    EXPECT(R, w.client.lists == 2 && e.policy.evaluate_actuators == (int32_t)(UST_EVAL_ACTUATORS | UST_EVAL_VALIDATION));
    std::map<std::string, std::vector<uint16_t>> lists;
    std::map<std::string, int64_t> start;
    for (size_t i = 0; i < e.entries.size(); i++) {
      const std::string& n = e.entries[i]->Node->Name;
      lists[n] = std::vector<uint16_t>(e.pod_flags.begin() + e.pod_off[i], e.pod_flags.begin() + e.pod_off[i + 1]);
      start[n] = e.start[i];
    }
    // n0: its validation pod (ready), then the same pod as a wait pod (Running), then the job
    EXPECT(R, (lists["n0"] == std::vector<uint16_t>{(uint16_t)(V | RDY), (uint16_t)(W | UST_PHASE_RUNNING), (uint16_t)(W | UST_PHASE_RUNNING)}));
    EXPECT(R, (lists["n1"] == std::vector<uint16_t>{V, (uint16_t)(W | UST_PHASE_RUNNING), (uint16_t)(W | UST_PHASE_SUCCEEDED)}));
    EXPECT(R, lists["n2"].empty());
    EXPECT(R, start["n0"] == 600 && start["n1"] == 700);  // each state's own start time
  });

  R.it("ApplyStateIncremental hands down only the changed lists and nodes, and nothing on a time-only reconcile", [&] {
    Small w;
    for (int i = 0; i < 6; i++) w.node("n" + std::to_string(i), i % 2 ? UpgradeStateWaitForJobsRequired : UpgradeStateDone);
    w.wpod("j1-a", "n1", "Running");
    w.wpod("j1-b", "n1", "Succeeded");
    w.wpod("j3-a", "n3", "Pending");
    int64_t clock = 5000;
    StateOptions o;
    o.WaitForCompletionOnDevice = true;
    o.Now = [&] { return clock; };
    auto* dev = new StandIn(o);
    std::unique_ptr<ClusterUpgradeStateManagerImpl> owner(dev);
    w.wire(dev);
    const DriverUpgradePolicySpec p = waitPolicy(120);
    auto reconcile = [&] {
      w.snapshot();
      EXPECT(R, !dev->ApplyStateIncremental(&w.state, &p).has_value());
    };
    reconcile();  // 0: full
    EXPECT(R, dev->calls.size() == 1 && dev->calls[0].full && dev->calls[0].listed.size() == 6 && dev->calls[0].waitTimeout == 120);
    EXPECT(R, dev->calls[0].evaluate == (int32_t)UST_EVAL_ACTUATORS);
    EXPECT(R, (dev->calls[0].lists[1] == std::vector<uint16_t>{(uint16_t)(W | UST_PHASE_RUNNING), (uint16_t)(W | UST_PHASE_SUCCEEDED)}));
    clock += 700;
    reconcile();  // 1: only time passed
    const StandIn::Call& t = dev->calls.back();
    EXPECT(R, !t.full && t.changed.empty() && t.listed.empty() && t.run_src.empty() && t.now == clock);
    EXPECT(R, dev->Stats().time_only == 1);
    // 2: a job finishes (list replaced); another pod gets a new resourceVersion with the same phase (kept)
    w.pods[0].Phase = "Succeeded"; w.pods[0].ResourceVersion = "2";
    w.pods[2].ResourceVersion = "2";
    reconcile();
    EXPECT(R, (dev->calls.back().listed == std::vector<int64_t>{1}) && dev->calls.back().changed.empty());
    EXPECT(R, (dev->calls.back().lists[0] == std::vector<uint16_t>{(uint16_t)(W | UST_PHASE_SUCCEEDED), (uint16_t)(W | UST_PHASE_SUCCEEDED)}));
    // 3: a start annotation appears on n3: the node goes down with its start time, its list stays
    w.nodes[3].Annotations[GetWaitForPodCompletionStartTimeAnnotationKey()] = "4321"; w.nodes[3].ResourceVersion = "2";
    reconcile();
    EXPECT(R, (dev->calls.back().changed == std::vector<int64_t>{3}) && (dev->calls.back().startOfChanged == std::vector<int64_t>{4321}));
    EXPECT(R, dev->calls.back().listed.empty());
    // 4: a node joins at the end with a job: runs, the joined node brings its list and its start time
    w.node("n6", UpgradeStateWaitForJobsRequired, {{GetWaitForPodCompletionStartTimeAnnotationKey(), "777"}});
    w.wpod("j6-a", "n6", "Running");
    reconcile();
    const StandIn::Call& s = dev->calls.back();
    EXPECT(R, (s.run_src == std::vector<int64_t>{0, -1}) && (s.listed == std::vector<int64_t>{6}));
    EXPECT(R, (s.lists[0] == std::vector<uint16_t>{(uint16_t)(W | UST_PHASE_RUNNING)}) && (s.insertStart == std::vector<int64_t>{777}));
    // 5: the List fails: no list goes down, and ApplyState returns the List's error at the wait-for-jobs pass
    w.client.listError = Errorf("the server is unavailable");
    w.snapshot();
    const Error le = dev->ApplyStateIncremental(&w.state, &p);
    EXPECT(R, le && *le == "the server is unavailable");
    EXPECT(R, dev->calls.back().listed.empty() && dev->calls.back().changed.empty());
    w.client.listError.reset();
    const auto& st = dev->Stats();
    EXPECT(R, st.full_uploads == 1 && st.lists_sent == 6 + 1 + 1 && st.wait_avoided == 3 * 4 + 4 + 4 && w.podm.waitCalls == 0);
    EXPECT(R, w.client.lists == 6 && st.validate_avoided == 0);
    // 6: ValidateOnDevice joins: the cache starts over; a validation pod's change then resends the list with its wait half
    dev->SetValidateOnDevice(true);
    dev->WithValidationEnabled(kValidation);
    w.pods.push_back(vspec::makeValidationPod("v3", "n3", true, {false}, 1));
    reconcile();
    EXPECT(R, dev->calls.back().full && dev->calls.back().evaluate == (int32_t)(UST_EVAL_ACTUATORS | UST_EVAL_VALIDATION));
    w.pods.back().ContainerStatuses = {{true, 0}}; w.pods.back().ResourceVersion = "2";
    reconcile();
    EXPECT(R, (dev->calls.back().listed == std::vector<int64_t>{3}));
    EXPECT(R, (dev->calls.back().lists[0] == std::vector<uint16_t>{(uint16_t)(V | RDY), (uint16_t)(W | UST_PHASE_PENDING)}));
    // 7: the wait option off: the cache starts over without it
    dev->SetWaitForCompletionOnDevice(false);
    dev->SetValidateOnDevice(false);
    reconcile();
    EXPECT(R, dev->calls.back().full && dev->calls.back().evaluate == 0 && dev->Stats().full_uploads == 3);
  });

  // Replay of pass 4 from hand-made outputs: one wait-for-jobs-required node.
  const std::string del = "annotation n0 " + wkey + "=null", set = "annotation n0 " + wkey + "=1234", pdr = "state n0=pod-deletion-required";
  struct Out { uint8_t outcome; uint16_t actions; bool running; };
  auto replay = [&](const Out& o, const std::string& failOn, Error listError, std::vector<std::string>* log, int* copies = nullptr) -> Error {
    Small w;
    w.node("n0", UpgradeStateWaitForJobsRequired, {{wkey, "100"}});
    w.provider.match = failOn;
    w.provider.failAt = 0;
    w.snapshot();
    auto m = ClusterUpgradeStateManagerImpl::NewDetached({});
    w.wire(m.get());
    EncodedSnapshot e;
    e.entries = {w.owned[0].get()};
    e.state = {UST_STATE_WAIT_FOR_JOBS_REQUIRED};
    e.flags = {0};
    e.waitOnDevice = true;
    e.waitRunning = {o.running};
    e.now = 1234;
    e.waitListError = listError;
    const DriverUpgradePolicySpec p = waitPolicy(30);
    ust_counters c{};
    c.error_index = -1;
    c.error_pass = -1;
    const uint8_t next = UST_STATE_WAIT_FOR_JOBS_REQUIRED;
    const uint16_t actions = (uint16_t)(o.actions | UST_A_SCHEDULE_WAIT_CHECK);
    Error err = m->Replay(e, p, &next, &actions, UST_OK, c, &o.outcome);
    *log = w.calls();
    if (copies) *copies = w.provider.copies;
    EXPECT(R, w.podm.waitCalls == 0);
    return err;
  };
  const uint8_t PDR = UST_STATE_POD_DELETION_REQUIRED, WFJ = UST_STATE_WAIT_FOR_JOBS_REQUIRED;
  const uint16_t CLR = UST_A_CLEAR_WAIT_START, SET = UST_A_SET_WAIT_START;
  R.it("Replay, pass 4: finished = delete, then state; timed out = state, then delete; no start time = set it to now", [&] {
    std::vector<std::string> log;
    int copies = 0;
    EXPECT(R, !replay({PDR, CLR, false}, "", std::nullopt, &log, &copies));
    EXPECT(R, (log == std::vector<std::string>{del, pdr}) && copies == 2);
    EXPECT(R, !replay({PDR, CLR, true}, "", std::nullopt, &log, &copies));
    EXPECT(R, (log == std::vector<std::string>{pdr, del}) && copies == 2);
    EXPECT(R, !replay({WFJ, SET, true}, "", std::nullopt, &log, &copies));
    EXPECT(R, (log == std::vector<std::string>{set}) && copies == 1);
    EXPECT(R, !replay({WFJ, 0, true}, "", std::nullopt, &log));
    EXPECT(R, log.empty());
  });
  R.it("Replay, pass 4: the calls get a copy of the node, and the snapshot's node object is left alone", [&] {
    Small w;
    w.node("n0", UpgradeStateWaitForJobsRequired);
    w.snapshot();
    NodeUpgradeStateProviderMock plain;  // writes into the object it is handed
    auto m = ClusterUpgradeStateManagerImpl::NewDetached({});
    w.wire(m.get());
    m->NodeUpgradeStateProvider = &plain;
    EncodedSnapshot e;
    e.entries = {w.owned[0].get()};
    e.state = {UST_STATE_WAIT_FOR_JOBS_REQUIRED};
    e.flags = {0};
    e.waitOnDevice = true;
    e.waitRunning = {1};
    e.now = 1234;
    ust_counters c{};
    c.error_index = -1; c.error_pass = -1;
    const uint8_t next = WFJ, outcome = WFJ;
    const uint16_t actions = (uint16_t)(SET | UST_A_SCHEDULE_WAIT_CHECK);
    const DriverUpgradePolicySpec p = waitPolicy(30);
    EXPECT(R, !m->Replay(e, p, &next, &actions, UST_OK, c, &outcome));
    EXPECT(R, w.nodes[0].Annotations.empty() && w.nodes[0].Labels.at(GetUpgradeStateLabelKey()) == UpgradeStateWaitForJobsRequired);
  });
  R.it("Replay, pass 4: provider errors are swallowed; a failed delete suppresses the state change on the finished path only", [&] {
    std::vector<std::string> log;
    EXPECT(R, !replay({PDR, CLR, false}, del, std::nullopt, &log));
    EXPECT(R, (log == std::vector<std::string>{"FAILED " + del}));
    EXPECT(R, !replay({PDR, CLR, false}, pdr, std::nullopt, &log));
    EXPECT(R, (log == std::vector<std::string>{del, "FAILED " + pdr}));
    EXPECT(R, !replay({PDR, CLR, true}, pdr, std::nullopt, &log));
    EXPECT(R, (log == std::vector<std::string>{"FAILED " + pdr, del}));
    EXPECT(R, !replay({PDR, CLR, true}, del, std::nullopt, &log));
    EXPECT(R, (log == std::vector<std::string>{pdr, "FAILED " + del}));
    EXPECT(R, !replay({WFJ, SET, true}, set, std::nullopt, &log));
    EXPECT(R, (log == std::vector<std::string>{"FAILED " + set}));
  });
  R.it("Replay: a failed List returns at the wait-for-jobs pass (index 4) when it has nodes, and is no error otherwise", [&] {
    for (int withWait = 0; withWait < 2; withWait++) {
      Small w;
      w.node("n0", UpgradeStateCordonRequired);
      if (withWait) w.node("n1", UpgradeStateWaitForJobsRequired);
      w.node("n2", UpgradeStatePodDeletionRequired);
      w.snapshot();
      auto m = ClusterUpgradeStateManagerImpl::NewDetached({});
      w.wire(m.get());
      m->WithPodDeletionEnabled([](const Pod&) { return false; });
      EncodedSnapshot e;
      for (auto& o : w.owned) e.entries.push_back(o.get());
      std::vector<uint8_t> next, outcome;
      std::vector<uint16_t> actions;
      for (const auto& o : w.owned) {
        const int code = StateCodeOfLabel(o->Node->Labels.at(GetUpgradeStateLabelKey()));
        e.state.push_back((uint8_t)code);
        e.flags.push_back(0);
        e.waitRunning.push_back(0);
        next.push_back(code == UST_STATE_CORDON_REQUIRED ? WFJ : (uint8_t)code);
        actions.push_back(code == UST_STATE_CORDON_REQUIRED ? (uint16_t)(UST_A_CORDON | UST_A_SET_STATE)
                          : code == UST_STATE_WAIT_FOR_JOBS_REQUIRED ? (uint16_t)(UST_A_SCHEDULE_WAIT_CHECK | CLR)
                                                                     : (uint16_t)UST_A_SCHEDULE_POD_EVICTION);
        outcome.push_back(code == UST_STATE_WAIT_FOR_JOBS_REQUIRED ? PDR : UST_OUTCOME_NONE);
      }
      e.waitOnDevice = true;
      e.waitListError = Errorf("etcdserver: request timed out");
      ust_counters c{};
      c.error_index = -1; c.error_pass = -1;
      const DriverUpgradePolicySpec p = waitPolicy(30);
      const Error err = m->Replay(e, p, next.data(), actions.data(), UST_OK, c, outcome.data());
      if (withWait) {
        EXPECT(R, err && *err == "etcdserver: request timed out");
        EXPECT(R, (w.calls() == std::vector<std::string>{"cordon n0", "state n0=wait-for-jobs-required"}));
      } else {
        EXPECT(R, !err && (w.calls() == std::vector<std::string>{"cordon n0", "state n0=wait-for-jobs-required", "evict 1"}));
      }
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
  const std::string wkey = GetWaitForPodCompletionStartTimeAnnotationKey();
  const int64_t now = 1700000000;
  // The cluster through ApplyState three times: with the restated PodManagerImpl, and with WaitForCompletionOnDevice
  // (ApplyState and ApplyStateIncremental). Same calls, same nodes afterwards, same error; one List with the option.
  using Setup = std::function<void(Small&)>;
  auto both = [&](const char* name, const DriverUpgradePolicySpec& p, const Setup& setup,
                  const std::function<void(const Small&, const Error&)>& expect) {
    R.it(name, [&] {
      Small a, b, c;
      for (Small* w : {&a, &b, &c}) { setup(*w); w->snapshot(); }
      StateOptions o;
      o.Now = [&] { return now; };
      auto ma = device(o, ok);
      a.wire(ma.get());
      PodManagerImpl ref;
      ref.client = &a.client; ref.provider = &a.provider; ref.now = o.Now; ref.log = &a.log;
      ma->PodManager = &ref;
      o.WaitForCompletionOnDevice = true;
      auto mb = device(o, ok), mc = device(o, ok);
      b.wire(mb.get()); c.wire(mc.get());
      const Error ea = ma->ApplyState(&a.state, &p), eb = mb->ApplyState(&b.state, &p), ec = mc->ApplyStateIncremental(&c.state, &p);
      EXPECT(R, ea == eb && ea == ec);
      EXPECT(R, a.log == b.log && b.log == c.log);
      EXPECT(R, a.image() == b.image() && b.image() == c.image());
      const bool selector = p.WaitForCompletion && !p.WaitForCompletion->PodSelector.empty();
      EXPECT(R, b.podm.waitCalls == 0 && c.podm.waitCalls == 0);
      EXPECT(R, b.client.lists == (selector ? 1 : 0) && c.client.lists == (selector ? 1 : 0));
      if (R.failed_here) {
        std::printf("    %s | %s | %s\n", ea ? ea->c_str() : "ok", eb ? eb->c_str() : "ok", ec ? ec->c_str() : "ok");
        for (auto& s : a.log) std::printf("    ref: %s\n", s.c_str());
        for (auto& s : b.log) std::printf("    dev: %s\n", s.c_str());
      }
      expect(b, eb);
    });
  };
  auto label = [](const Small& w, size_t i = 0) { return w.nodes[i].Labels.at(GetUpgradeStateLabelKey()); };
  auto hasStart = [&](const Small& w, size_t i = 0) { return w.nodes[i].Annotations.count(wkey) != 0; };
  // pod_manager_test.go:117-224
  both("jobs completed: pod-deletion-required, no start time (pod_manager_test.go:118)", waitPolicy(0), [](Small& w) {
    w.node("n0", UpgradeStateWaitForJobsRequired);
    w.wpod("test-pod", "n0", "Succeeded");
  }, [&](const Small& w, const Error& e) { EXPECT(R, !e && label(w) == UpgradeStatePodDeletionRequired && !hasStart(w)); });
  both("a job running without a timeout: the node waits, no start time (:151)", waitPolicy(0), [](Small& w) {
    w.node("n0", UpgradeStateWaitForJobsRequired);
    w.wpod("test-pod", "n0", "Running");
  }, [&](const Small& w, const Error& e) { EXPECT(R, !e && label(w) == UpgradeStateWaitForJobsRequired && !hasStart(w)); });
  both("a job running with TimeoutSecond 30: the start time is set to now (:179-207)", waitPolicy(30), [](Small& w) {
    w.node("n0", UpgradeStateWaitForJobsRequired);
    w.wpod("test-pod", "n0", "Running");
  }, [&](const Small& w, const Error& e) {
    EXPECT(R, !e && label(w) == UpgradeStateWaitForJobsRequired && w.nodes[0].Annotations.at(wkey) == std::to_string(now));
  });
  both("... and 35 s after the start: pod-deletion-required, start time removed (:209-222)", waitPolicy(30), [&](Small& w) {
    w.node("n0", UpgradeStateWaitForJobsRequired, {{wkey, std::to_string(now - 35)}});
    w.wpod("test-pod", "n0", "Running");
  }, [&](const Small& w, const Error& e) { EXPECT(R, !e && label(w) == UpgradeStatePodDeletionRequired && !hasStart(w)); });
  both("exactly at the deadline the node still waits (now > start + timeout)", waitPolicy(30), [&](Small& w) {
    w.node("n0", UpgradeStateWaitForJobsRequired, {{wkey, std::to_string(now - 30)}});
    w.wpod("test-pod", "n0", "Pending");
  }, [&](const Small& w, const Error& e) { EXPECT(R, !e && label(w) == UpgradeStateWaitForJobsRequired && hasStart(w)); });
  both("no wait pod on the node: pod-deletion-required, the start time deleted", waitPolicy(30), [&](Small& w) {
    w.node("n0", UpgradeStateWaitForJobsRequired, {{wkey, std::to_string(now)}});
    w.wpod("elsewhere", "n9", "Running");
  }, [&](const Small& w, const Error& e) { EXPECT(R, !e && label(w) == UpgradeStatePodDeletionRequired && !hasStart(w)); });
  both("an unparsable start time: the error is an event, the node waits", waitPolicy(30), [&](Small& w) {
    w.node("n0", UpgradeStateWaitForJobsRequired, {{wkey, "soon"}});
    w.node("n1", UpgradeStateWaitForJobsRequired, {{wkey, "99999999999999999999"}});
    w.wpod("p0", "n0", "Running");
    w.wpod("p1", "n1", "Running");
  }, [&](const Small& w, const Error& e) { EXPECT(R, !e && label(w, 0) == UpgradeStateWaitForJobsRequired && w.calls().empty()); });
  both("a start time near INT64_MAX: Go's int64 sum wraps, so the node has timed out", waitPolicy(30), [&](Small& w) {
    w.node("n0", UpgradeStateWaitForJobsRequired, {{wkey, "9223372036854775800"}});
    w.wpod("p0", "n0", "Running");
  }, [&](const Small& w, const Error& e) { EXPECT(R, !e && label(w) == UpgradeStatePodDeletionRequired); });
  both("a failed List returns its error at the wait-for-jobs pass, after the cordon-required pass", waitPolicy(30), [&](Small& w) {
    w.node("n0", UpgradeStateCordonRequired);
    w.node("n1", UpgradeStateWaitForJobsRequired);
    w.node("n2", UpgradeStatePodRestartRequired);
    w.client.listError = Errorf("the server could not find the requested resource");
  }, [&](const Small& w, const Error& e) {
    EXPECT(R, e && *e == "the server could not find the requested resource" && label(w, 0) == UpgradeStateWaitForJobsRequired);
  });
  both("a failed List without a wait-for-jobs-required node is no error", waitPolicy(30), [&](Small& w) {
    w.node("n0", UpgradeStateUncordonRequired);
    w.client.listError = Errorf("the server could not find the requested resource");
  }, [&](const Small& w, const Error& e) { EXPECT(R, !e && label(w) == UpgradeStateDone); });
  both("a failed start-time delete keeps a finished node in wait-for-jobs-required", waitPolicy(30), [&](Small& w) {
    w.node("n0", UpgradeStateWaitForJobsRequired, {{wkey, "5"}});
    w.wpod("p0", "n0", "Failed");
    w.provider.match = wkey;
    w.provider.failAt = 0;
  }, [&](const Small& w, const Error& e) { EXPECT(R, !e && label(w) == UpgradeStateWaitForJobsRequired && hasStart(w)); });
  {
    DriverUpgradePolicySpec none;
    none.AutoUpgrade = true;  // upgrade_state_test.go:615: no WaitForCompletion, no deletion filter
    both("without a selector the pass moves its nodes on by itself (upgrade_state_test.go:615)", none, [](Small& w) {
      for (int i = 0; i < 3; i++) w.node("n" + std::to_string(i), UpgradeStateWaitForJobsRequired);
    }, [&](const Small& w, const Error& e) { EXPECT(R, !e && label(w, 2) == UpgradeStateDrainRequired); });
  }
  both("200 wait-for-jobs-required nodes: one List, not 200", waitPolicy(60), [&](Small& w) {
    for (int i = 0; i < 200; i++) {
      const std::string n = "n" + std::to_string(i);
      w.node(n, UpgradeStateWaitForJobsRequired, i % 3 == 0 ? StringMap{{wkey, std::to_string(now - 10 * i)}} : StringMap{});
      if (i % 4) w.wpod("job-" + n, n, i % 4 == 1 ? "Running" : i % 4 == 2 ? "Pending" : "Succeeded");
    }
  }, [&](const Small& w, const Error& e) { EXPECT(R, !e && w.calls().size() > 200); });

  R.it("the host's running bit agrees with the device's outcome on every wait-for-jobs-required node", [&] {
    // random nodes: pods of every phase, start times absent / valid / unparsable / near the deadline, both timeouts
    spec::BLcg r{4242};
    const char* phases[] = {"Running", "Pending", "Succeeded", "Failed", "Unknown"};
    ust_handle* h = nullptr;
    if (ust_create(&h, 0) != UST_OK) { *ok = false; EXPECT(R, false); return; }
    int pdrRunning = 0, pdrFinished = 0, sets = 0, waits = 0;
    for (int timeout : {0, 45}) {
      Small w;
      for (int i = 0; i < 3000; i++) {
        const std::string n = "n" + std::to_string(i);
        const int kind = (int)(r.next() % 4);
        StringMap anno;
        if (kind == 1) anno[wkey] = std::to_string(now - (int64_t)(r.next() % 100));
        if (kind == 2) anno[wkey] = "x" + std::to_string(i);
        w.node(n, UpgradeStateWaitForJobsRequired, anno);
        for (int j = (int)(r.next() % 4); j > 0; j--) w.wpod("p" + std::to_string(j) + "-" + n, n, phases[r.next() % 5]);
      }
      w.snapshot();
      StateOptions o;
      o.WaitForCompletionOnDevice = true;
      o.Now = [&] { return now; };
      auto m = ClusterUpgradeStateManagerImpl::NewDetached(o);
      w.wire(m.get());
      const DriverUpgradePolicySpec p = waitPolicy(timeout);
      EncodedSnapshot e;
      EXPECT(R, !m->Encode(w.state, p, &e));
      const size_t n = e.entries.size();
      std::vector<uint8_t> next(n + 1), outcome(n + 1);
      std::vector<uint16_t> actions(n + 1);
      e.state.push_back(0); e.flags.push_back(0); e.pod_rev.push_back(0); e.ds_idx.push_back(0); e.ds_rev.push_back(0);
      e.pod_flags.push_back(0); e.start.push_back(0);
      const ust_pods pods = {e.pod_off.data(), e.pod_flags.data(), (int64_t)e.pod_flags.size() - 1};
      const ust_clock clock = {e.now, timeout, e.start.data(), nullptr};
      ust_counters c;
      EXPECT(R, ust_apply_state_clocked(h, &e.policy, &clock, (int64_t)n, e.state.data(), e.flags.data(), e.pod_rev.data(), e.ds_idx.data(),
                                        (int32_t)e.ds_rev.size() - 1, e.ds_rev.data(), &pods, next.data(), actions.data(), outcome.data(),
                                        &c) == UST_OK);
      for (size_t i = 0; i < n; i++) {
        const uint32_t f = e.flags[i];
        const bool pdr = outcome[i] == UST_STATE_POD_DELETION_REQUIRED, running = e.waitRunning[i] != 0;
        const bool timedOut = timeout != 0 && (f & UST_F_WAIT_START_ANNO) && !(f & UST_F_WAIT_START_INVALID) && now > e.start[i] + timeout;
        bool good = (actions[i] & UST_A_SCHEDULE_WAIT_CHECK) && (outcome[i] == UST_STATE_WAIT_FOR_JOBS_REQUIRED || pdr);
        good = good && (!pdr || (actions[i] & UST_A_CLEAR_WAIT_START));  // PDR without the delete is impossible
        good = good && (running || pdr);                                   // nothing running: always PDR
        good = good && (!running || pdr == timedOut);                      // running: PDR exactly when timed out
        good = good && (!(actions[i] & UST_A_SET_WAIT_START) || (running && timeout != 0 && !(f & UST_F_WAIT_START_ANNO)));
        EXPECT(R, good);
        if (!good) { std::printf("    node %zu: outcome %u actions %x running %d flags %x\n", i, outcome[i], actions[i], running, f); break; }
        pdrRunning += pdr && running; pdrFinished += pdr && !running; sets += (actions[i] & UST_A_SET_WAIT_START) != 0; waits += !pdr;
      }
    }
    ust_destroy(h);
    std::printf("    %d timed out while running, %d finished, %d start times set, %d waiting\n", pdrRunning, pdrFinished, sets, waits);
    EXPECT(R, pdrRunning > 0 && pdrFinished > 0 && sets > 0 && waits > 0);
  });

  R.it("a reconcile in which only time passed sends nothing and returns exactly the nodes whose wait deadline passed", [&] {
    Small w;
    for (int i = 0; i < 8; i++) {
      const std::string n = "n" + std::to_string(i);
      w.node(n, UpgradeStateWaitForJobsRequired, {{wkey, std::to_string(now + 100 * i)}});
      w.wpod("job-" + n, n, "Running");
    }
    int64_t t = now;
    StateOptions o;
    o.WaitForCompletionOnDevice = true;
    o.Now = [&] { return t; };
    auto m = device(o, ok);
    w.wire(m.get());
    const DriverUpgradePolicySpec p = waitPolicy(250);
    w.snapshot();
    EXPECT(R, !m->ApplyStateIncremental(&w.state, &p));  // full: nothing timed out yet
    EXPECT(R, w.calls().empty());
    const int64_t sent = m->Stats().lists_sent, received = m->Stats().outputs_received;
    t = now + 420;  // n0 (deadline now + 250) and n1 (now + 350) have passed theirs, n2 (now + 450) has not
    w.snapshot();
    EXPECT(R, !m->ApplyStateIncremental(&w.state, &p));
    EXPECT(R, m->Stats().time_only == 1 && m->Stats().lists_sent == sent && m->Stats().outputs_received - received == 2);
    const std::string d0 = "annotation n0 " + wkey + "=null", d1 = "annotation n1 " + wkey + "=null";
    EXPECT(R, (w.calls() == std::vector<std::string>{"state n0=pod-deletion-required", d0, "state n1=pod-deletion-required", d1}));
    EXPECT(R, label(w, 0) == UpgradeStatePodDeletionRequired && label(w, 1) == UpgradeStatePodDeletionRequired &&
              label(w, 2) == UpgradeStateWaitForJobsRequired && w.podm.waitCalls == 0 && w.client.lists == 2);
  });
}

// The reconcile loop: the world of build_state_spec.hpp plus job pods, validation pods, the clock, List and provider errors.
const char* kLoopWait = "tier=gpu";  // job pods carry it, and so do the validation pods: some pods match both selectors
struct WWorld {
  spec::BWorld w;
  vspec::SelectorClient sel;
  ApiProvider fp;
  std::deque<Pod> extra;  // job and validation pods
  std::vector<char> alive;
  std::set<std::string> seededJobs, seededVal;
  void wire(ClusterUpgradeStateManagerImpl* m) {
    w.wire(m);
    sel.base = &w.client;
    fp.log = &w.log;
    m->K8sClient = &sel;
    m->NodeUpgradeStateProvider = &fp;
  }
  void publish() {
    w.publish();
    fp.nodes = w.provider.nodes;
    sel.all.clear();
    for (size_t i = 0; i < extra.size(); i++)
      if (alive[i]) sel.all.push_back(&extra[i]);
    std::stable_sort(sel.all.begin(), sel.all.end(), [](const Pod* x, const Pod* y) { return x->Name < y->Name; });
  }
  void add(Pod p) { extra.push_back(std::move(p)); alive.push_back(1); }
};

void wevolve(WWorld& v, int rec, spec::BLcg r) {
  spec::bevolve(v.w, rec, spec::BLcg{r.s ^ 0x5555});
  for (size_t i = 0; i < v.extra.size(); i++) {  // the pods of nodes that left go with them
    if (!v.alive[i]) continue;
    if (!v.w.provider.nodes.count(v.extra[i].NodeName)) { v.alive[i] = 0; continue; }
    Pod& p = v.extra[i];
    if (p.Labels.count("never")) continue;
    if (p.Namespace == "jobs" && r.chance(12)) {  // a job finishes, or a pending one starts
      p.Phase = p.Phase == "Pending" ? "Running" : (r.chance(70) ? "Succeeded" : "Failed");
      v.w.bumpPod(p);
    } else if (p.Namespace != "jobs" && r.chance(20)) {  // a validation finishes
      p.Phase = "Running";
      p.ContainerStatuses = {{true, 0}};
      v.w.bumpPod(p);
    }
  }
  for (Node& nd : v.w.nodes) {
    if (nd.Name.empty()) continue;
    auto it = nd.Labels.find(GetUpgradeStateLabelKey());
    const std::string st = it == nd.Labels.end() ? "" : it->second;
    // a node that is cordoned gets 0-3 jobs the first time; some never finish (they run past the timeout)
    if ((st == UpgradeStateCordonRequired || st == UpgradeStateWaitForJobsRequired) && !v.seededJobs.count(nd.Name)) {
      v.seededJobs.insert(nd.Name);
      for (int j = (int)(r.next() % 4); j > 0; j--) {
        const char* phase = r.chance(60) ? "Running" : r.chance(50) ? "Pending" : "Succeeded";
        Pod p = makeWaitPod("job-" + nd.Name + "-" + std::to_string(j), nd.Name, phase, v.w.version++);
        p.Labels["tier"] = "gpu";
        if (r.chance(25)) p.Labels["never"] = "1";
        v.add(p);
      }
    }
    if (st == UpgradeStateValidationRequired && !v.seededVal.count(nd.Name)) {
      v.seededVal.insert(nd.Name);
      for (int j = (int)(r.next() % 3); j > 0; j--) {
        Pod p = vspec::makeValidationPod("val-" + nd.Name + "-" + std::to_string(j), nd.Name, r.chance(50), {false}, v.w.version++);
        if (r.chance(20)) p.Labels["never"] = "1";
        v.add(p);
      }
    }
  }
  // now and then an unparsable wait start time, taken away again three reconciles later
  if (rec % 40 == 13 || rec % 40 == 16) {
    const std::string key = GetWaitForPodCompletionStartTimeAnnotationKey();
    for (Node& nd : v.w.nodes) {
      auto it = nd.Labels.find(GetUpgradeStateLabelKey());
      if (nd.Name.empty() || it == nd.Labels.end() || it->second != UpgradeStateWaitForJobsRequired) continue;
      if (rec % 40 == 13) nd.Annotations[key] = "not-a-number";
      else if (nd.Annotations.count(key) && nd.Annotations[key] == "not-a-number") nd.Annotations.erase(key);
      spec::LogProvider::bump(&nd);
    }
  }
}

void loop(Runner& R, bool requestor, bool validate, int n_nodes, int rounds, bool* ok) {
  SetDriverName("gpu");
  const std::string name = std::string("ApplyStateIncremental with WaitForCompletionOnDevice == ApplyState with PodManagerImpl over a reconcile loop (") +
                           (requestor ? "requestor" : "in-place") + " mode, ValidateOnDevice " + (validate ? "on" : "off") + ")";
  R.it(name.c_str(), [&] {
    WWorld a, b;
    spec::bpopulate(a.w, n_nodes, 53); spec::bpopulate(b.w, n_nodes, 53);
    int64_t clock = 1700000000;
    StateOptions o;
    o.Requestor.UseMaintenanceOperator = requestor;
    o.Now = [&] { return clock; };
    StateOptions od = o;
    od.WaitForCompletionOnDevice = true;
    od.ValidateOnDevice = validate;
    auto mb = device(od, ok);
    b.wire(mb.get());
    CountingPods pb;
    pb.log = &b.w.log;
    mb->PodManager = &pb;
    vspec::CountingValidation vb;
    if (validate) { mb->ValidationManager = &vb; mb->WithValidationEnabled(kValidation); }
    PodManagerImpl ref;
    ref.client = &a.sel; ref.provider = &a.fp; ref.now = o.Now; ref.log = &a.w.log;
    vspec::ValidationManagerImpl vref;
    vref.client = &a.sel; vref.provider = &a.fp; vref.podSelector = kValidation; vref.now = o.Now;
    DriverUpgradePolicySpec p;
    p.AutoUpgrade = true;
    p.MaxParallelUpgrades = 14;
    p.MaxUnavailable = IntOrString::FromString("45%");
    p.DrainSpec = upgrade::DrainSpec{};
    p.DrainSpec->Enable = true;
    p.WaitForCompletion = WaitForCompletionSpec{kLoopWait, 300};
    const int64_t steps[] = {17, 90, 240, 45, 400, 3};
    int listErrors = 0, swallowed = 0, timeouts = 0, finished = 0, starts = 0, errors = 0, badLists = 0;
    for (int rec = 0; rec < rounds; rec++) {
      p.WaitForCompletion->TimeoutSecond = rec < 100 ? 300 : rec < 150 ? 0 : 120;
      auto ma = device(o, ok);  // the reference's way: a fresh manager every reconcile
      a.wire(ma.get());
      ma->PodManager = &ref;
      if (validate) { ma->ValidationManager = &vref; ma->WithValidationEnabled(kValidation); }
      a.publish(); b.publish();
      a.w.log.clear(); b.w.log.clear();
      const bool listFails = rec % 37 == 11, providerFails = rec % 41 == 17 || rec % 41 == 30;
      for (WWorld* v : {&a, &b}) {
        v->sel.listError = listFails ? Errorf("etcdserver: request timed out") : std::nullopt;
        v->fp.match = providerFails ? GetWaitForPodCompletionStartTimeAnnotationKey() : (rec % 41 == 24 ? "=pod-deletion-required" : "");
        v->fp.failAt = 0; v->fp.seen = 0;
      }
      const int listsBefore = b.sel.lists;
      std::unique_ptr<ClusterUpgradeState> sa, sb;
      Error ea = ma->BuildState("gpu-operator", {}, &sa);
      Error eb = mb->BuildStateIncremental("gpu-operator", {}, &sb);
      EXPECT(R, ea == eb);
      if (!ea && !eb) {
        ea = ma->ApplyState(sa.get(), &p);
        eb = mb->ApplyStateIncremental(sb.get(), &p);
        EXPECT(R, ea == eb);
        badLists += b.sel.lists - listsBefore != (validate ? 2 : 1);  // one wait List, whatever the bucket's size
      }
      if (ea) {
        errors++;
        listErrors += *ea == "etcdserver: request timed out";
      }
      const std::string key = GetWaitForPodCompletionStartTimeAnnotationKey();
      for (size_t k = 0; k < a.w.log.size(); k++) {
        const std::string& s = a.w.log[k];
        swallowed += s.rfind("FAILED", 0) == 0;
        if (s.find("=pod-deletion-required") != std::string::npos)
          (k + 1 < a.w.log.size() && a.w.log[k + 1].find(key + "=null") != std::string::npos ? timeouts : finished)++;
        starts += s.find(key + "=1") != std::string::npos;
      }
      EXPECT(R, vspec::collapse(a.w.log) == vspec::collapse(b.w.log));
      EXPECT(R, spec::bimage(a.w) == spec::bimage(b.w));
      if (R.failed_here) {
        std::printf("    (reconcile %d: %s / %s)\n", rec, ea ? ea->c_str() : "ok", eb ? eb->c_str() : "ok");
        const auto la = vspec::collapse(a.w.log), lb = vspec::collapse(b.w.log);
        for (size_t k = 0; k < std::max(la.size(), lb.size()); k++)
          if (k >= la.size() || k >= lb.size() || la[k] != lb[k])
            std::printf("    #%zu ref: %s | dev: %s\n", k, k < la.size() ? la[k].c_str() : "-", k < lb.size() ? lb[k].c_str() : "-");
        break;
      }
      // both PodManagers restarted the same driver pods: the world re-creates them
      a.w.pods.restarted.swap(ref.restarted); b.w.pods.restarted.swap(pb.restarted);
      ref.restarted.clear(); pb.restarted.clear();
      clock += steps[rec % 6];
      wevolve(a, rec, spec::BLcg{8100u + (uint64_t)rec}); wevolve(b, rec, spec::BLcg{8100u + (uint64_t)rec});
    }
    const auto& st = mb->Stats();
    std::printf("    %lld reconciles, %lld full uploads, %lld reorders, %lld lists sent, %lld reused, %lld time-only, %lld wait Lists avoided "
                "(reference: %d Lists in %d checks); errors: %d (List %d); %d provider errors swallowed; %d timed out, %d finished, "
                "%d start times set\n",
                (long long)st.reconciles, (long long)st.full_uploads, (long long)st.reorders, (long long)st.lists_sent,
                (long long)st.lists_reused, (long long)st.time_only, (long long)st.wait_avoided, ref.lists, ref.checks, errors, listErrors,
                swallowed, timeouts, finished, starts);
    EXPECT(R, pb.waitCalls == 0 && ref.checks > 0 && vb.calls == 0 && badLists == 0);
    EXPECT(R, st.full_uploads == 1 && st.reorders > 0 && st.wait_avoided > 0 && st.lists_reused > st.lists_sent);
    EXPECT(R, listErrors > 0 && swallowed > 0 && timeouts > 0 && finished > 0 && starts > 0);
  });
}

}  // namespace

int main(int argc, char** argv) {
  const bool gpu = argc > 1 && std::strcmp(argv[1], "--gpu") == 0;
  Runner R;
  bool ok = true;
  if (gpu) {
    gpu_specs(R, &ok);
    for (bool validate : {false, true}) {
      loop(R, false, validate, 300, 300, &ok);
      loop(R, true, validate, 300, 300, &ok);
    }
  } else {
    cpu_specs(R);
  }
  std::printf("# %d passed, %d failed\n", R.passed, R.failed);
  return (R.failed == 0 && ok) ? 0 : 1;
}
