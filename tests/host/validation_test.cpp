// StateOptions::ValidateOnDevice (validation_spec.hpp).
//   validation_test         host halves only: Encode's validation pods, start times and flag bits; what ApplyStateIncremental
//                           hands to the device (a stand-in records it): replaced lists, start times, runs, nothing for a
//                           time-only reconcile; Replay of hand-made outputs through pass 10, errors at every call
//   validation_test --gpu   the reference's Validate cases and ApplyState validation specs, and a reconcile loop of
//                           BuildStateIncremental + ApplyStateIncremental with ValidateOnDevice against BuildState + ApplyState
//                           with the restated ValidationManagerImpl, on the H100
#include <cerrno>
#include <cstdlib>
#include <cstring>
#include <set>

#include "validation_spec.hpp"

using namespace upgrade;
using namespace vspec;

namespace {

const char* kSelector = "app=validator,tier=gpu";

// A one-bucket cluster built by hand: nodes with a driver pod each, in ListIndex order.
struct Small {
  std::deque<Node> nodes;
  std::deque<Pod> drivers, vpods;
  DaemonSet ds;
  ClusterUpgradeState state;
  std::vector<std::unique_ptr<NodeUpgradeState>> owned;
  std::vector<std::string> log;
  FailingProvider provider;
  spec::LogCordon cordon;
  spec::LogDrain drain;
  spec::LogPods pods;
  SafeDriverLoadManagerImpl safeLoad{&provider};
  SelectorClient client;
  Small() { provider.log = cordon.log = drain.log = pods.log = &log; ds.Name = "driver"; ds.UID = "uid-ds"; }
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
  void vpod(const std::string& name, const std::string& node, bool running, std::vector<bool> ready, int64_t rv = 1) {
    vpods.push_back(makeValidationPod(name, node, running, std::move(ready), rv));
  }
  // the snapshot BuildState would give, and the List's view of the validation pods (sorted by name, as the API does)
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
    for (Pod& p : vpods) client.all.push_back(&p);
    std::stable_sort(client.all.begin(), client.all.end(), [](const Pod* x, const Pod* y) { return x->Name < y->Name; });
  }
  void wire(ClusterUpgradeStateManagerImpl* m) {
    m->NodeUpgradeStateProvider = &provider; m->CordonManager = &cordon; m->DrainManager = &drain; m->PodManager = &pods;
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
};

// What ApplyStateIncremental hands to the device, recorded; the outputs are "no transition, no call".
struct StandIn : ClusterUpgradeStateManagerImpl {
  struct Call {
    bool full = false;
    int64_t now = 0;
    std::vector<int64_t> changed, startOfChanged, listed, run_src, run_len, insertStart;
    std::vector<std::vector<uint16_t>> lists;
    int32_t evaluate = 0;
  };
  std::vector<Call> calls;
  explicit StandIn(StateOptions o) : ClusterUpgradeStateManagerImpl(std::move(o)) {}
  static void quiet(Cache* k) {
    const size_t n = k->slots.size();
    k->next.assign(n + 1, 0);
    k->actions.assign(n + 1, 0);
    for (size_t i = 0; i < n; i++) k->next[i] = k->state[i] & UST_HOT_STATE_MASK;
  }
  int EvaluateCached(const ust_policy& policy, bool full, const std::vector<int64_t>& changed, Cache* k, ust_counters* c) override {
    Call call;
    call.full = full; call.changed = changed; call.run_src = k->pending.run_src; call.run_len = k->pending.run_len;
    call.evaluate = policy.evaluate_actuators;
    calls.push_back(call);
    quiet(k);
    std::memset(c, 0, sizeof(*c));
    c->error_index = -1;
    return UST_OK;
  }
  int EvaluateCachedPods(const ust_policy& policy, int64_t now, int64_t, bool full, const std::vector<int64_t>& changed, Cache* k,
                         ust_counters* c) override {
    Call call;
    call.full = full; call.now = now; call.changed = changed; call.listed = k->listChanged;
    call.run_src = k->pending.run_src; call.run_len = k->pending.run_len; call.evaluate = policy.evaluate_actuators;
    for (int64_t i : changed) call.startOfChanged.push_back(k->start[(size_t)i]);
    for (int64_t i : k->pending.insert_at) call.insertStart.push_back(k->start[(size_t)i]);
    for (int64_t i : k->listChanged) call.lists.push_back(k->lists[(size_t)i]);
    if (!k->pending.insert_before.empty()) call.evaluate = -1;  // a splice: the pod-list path has no such entry
    calls.push_back(call);
    quiet(k);
    std::memset(c, 0, sizeof(*c));
    c->error_index = -1;
    return UST_OK;
  }
};

const uint16_t M = UST_POD_MATCH_VALIDATION_SELECTOR, RDY = UST_POD_READY;

void cpu_specs(Runner& R) {
  SetDriverName("gpu");
  const std::string vkey = GetValidationStartTimeAnnotationKey();

  R.it("GetValidationStartTimeAnnotationKey follows the driver name (util.go:151-155)", [&] {
    EXPECT(R, vkey == "nvidia.com/gpu-driver-upgrade-validation-start-time");
  });

  R.it("Encode: one List, every node's validation pods in List order, start times and the three start bits", [&] {
    Small w;
    w.node("n0", UpgradeStateValidationRequired);
    w.node("n1", UpgradeStateValidationRequired, {{vkey, "1700000000"}});
    w.node("n2", UpgradeStateValidationRequired, {{vkey, "12x"}});
    w.node("n3", UpgradeStateDone, {{vkey, "-42"}});
    w.node("n4", UpgradeStateValidationRequired, {{vkey, "99999999999999999999"}});
    w.node("n5", UpgradeStateValidationRequired, {{vkey, "1\t2\a\x80\xc2\x85\"\xe2\x82\xac"}});
    w.node("n6", UpgradeStateValidationRequired, {{vkey, "99999999999999999999x"}});
    w.vpod("a-ready", "n0", true, {true, true});
    w.vpod("b-notready", "n0", true, {true, false});
    w.vpod("c-pending", "n0", false, {});
    w.vpod("d-nostatus", "n1", true, {});
    w.vpod("e-elsewhere", "n3", true, {true});
    w.vpod("f-unscheduled", "", true, {true});
    Pod other = makeValidationPod("g-other-app", "n1", true, {true}, 1);
    other.Labels["app"] = "something-else";
    w.vpods.push_back(other);
    w.snapshot();
    StateOptions o;
    o.ValidateOnDevice = true;
    o.Now = [] { return (int64_t)1700000123; };
    auto m = ClusterUpgradeStateManagerImpl::NewDetached(o);
    w.wire(m.get());
    m->WithValidationEnabled(kSelector);
    DriverUpgradePolicySpec p;
    p.AutoUpgrade = true;
    EncodedSnapshot e;
    EXPECT(R, !m->Encode(w.state, p, &e).has_value());
    EXPECT(R, w.client.lists == 1);
    EXPECT(R, e.validateOnDevice && e.now == 1700000123 && !e.listError);
    EXPECT(R, e.policy.evaluate_actuators == (int32_t)(UST_EVAL_ACTUATORS | UST_EVAL_VALIDATION));
    std::map<std::string, std::vector<uint16_t>> lists;
    std::map<std::string, std::pair<uint32_t, int64_t>> bits;
    std::map<std::string, std::string> deferred;
    EXPECT(R, e.pod_off.size() == e.entries.size() + 1 && e.start.size() == e.entries.size());
    for (size_t i = 0; i < e.entries.size(); i++) {
      const std::string& n = e.entries[i]->Node->Name;
      lists[n] = std::vector<uint16_t>(e.pod_flags.begin() + e.pod_off[i], e.pod_flags.begin() + e.pod_off[i + 1]);
      bits[n] = {e.flags[i] & (UST_F_VALIDATION_START_ANNO | UST_F_VALIDATION_START_INVALID | UST_F_VALIDATION_TIMED_OUT), e.start[i]};
      if (e.deferred.count(i)) deferred[n] = e.deferred.at(i);
    }
    EXPECT(R, (lists["n0"] == std::vector<uint16_t>{(uint16_t)(M | RDY), M, M}));
    EXPECT(R, (lists["n1"] == std::vector<uint16_t>{M}));
    EXPECT(R, lists["n2"].empty() && lists["n4"].empty());
    EXPECT(R, (lists["n3"] == std::vector<uint16_t>{(uint16_t)(M | RDY)}));  // every node gets its list, whatever its state
    EXPECT(R, bits["n0"] == std::make_pair(0u, (int64_t)0));
    EXPECT(R, bits["n1"] == std::make_pair((uint32_t)UST_F_VALIDATION_START_ANNO, (int64_t)1700000000));
    EXPECT(R, bits["n2"] == std::make_pair((uint32_t)(UST_F_VALIDATION_START_ANNO | UST_F_VALIDATION_START_INVALID), (int64_t)0));
    EXPECT(R, bits["n3"] == std::make_pair((uint32_t)UST_F_VALIDATION_START_ANNO, (int64_t)-42));
    EXPECT(R, bits["n4"] == std::make_pair((uint32_t)(UST_F_VALIDATION_START_ANNO | UST_F_VALIDATION_START_INVALID), (int64_t)0));
    EXPECT(R, deferred.size() == 4);
    // Go: strconv.Quote escapes \t and \a by name, an invalid byte as \x80, the C1 control U+0085 as \u0085, and copies
    // the printable U+20AC; ParseUint reports the overflow before the bad character that follows it
    EXPECT(R, deferred["n5"] == "unable to handle timeout for validation state: strconv.ParseInt: parsing \"1\\t2\\a\\x80\\u0085\\\"\xe2\x82\xac\": invalid syntax");
    EXPECT(R, deferred["n6"] == "unable to handle timeout for validation state: strconv.ParseInt: parsing \"99999999999999999999x\": value out of range");
    int64_t v = 0;
    for (const char* t : {"99999999999999999999x", "12x", "99999999999999999999", "-9223372036854775809", "+", ""})
      EXPECT(R, ValidationManagerImpl::parseInt(t, &v).has_value());
    EXPECT(R, ValidationManagerImpl::parseInt("-9223372036854775808", &v) == std::nullopt && v == INT64_MIN);
    EXPECT(R, *ValidationManagerImpl::parseInt("99999999999999999999x", &v) == deferred["n6"].substr(std::strlen("unable to handle timeout for validation state: ")));
    EXPECT(R, deferred["n2"] == "unable to handle timeout for validation state: strconv.ParseInt: parsing \"12x\": invalid syntax");
    EXPECT(R, deferred["n4"] == "unable to handle timeout for validation state: strconv.ParseInt: parsing \"99999999999999999999\": value out of range");
    // without the option (or without a selector) nothing changes
    auto plain = ClusterUpgradeStateManagerImpl::NewDetached({});
    w.wire(plain.get());
    plain->WithValidationEnabled(kSelector);
    EncodedSnapshot q;
    EXPECT(R, !plain->Encode(w.state, p, &q).has_value());
    EXPECT(R, !q.validateOnDevice && q.pod_off.empty() && q.start.empty() && q.policy.evaluate_actuators == 0 && q.deferred.empty());
    EXPECT(R, q.flags.size() == e.flags.size());
    bool sameOtherwise = true;
    for (size_t i = 0; i < q.flags.size(); i++)
      sameOtherwise = sameOtherwise && q.flags[i] == (e.flags[i] & ~(uint32_t)(UST_F_VALIDATION_START_ANNO | UST_F_VALIDATION_START_INVALID)) &&
                      q.state[i] == e.state[i];
    EXPECT(R, sameOtherwise);
    EXPECT(R, w.client.lists == 1);
  });

  R.it("ApplyStateIncremental hands down only what changed: lists, start times, runs; a time-only reconcile sends nothing", [&] {
    Small w;
    for (int i = 0; i < 6; i++) w.node("n" + std::to_string(i), i % 2 ? UpgradeStateValidationRequired : UpgradeStateDone);
    w.vpod("v1-a", "n1", true, {false});
    w.vpod("v1-b", "n1", true, {true});
    w.vpod("v3-a", "n3", false, {});
    int64_t clock = 5000;
    StateOptions o;
    o.ValidateOnDevice = true;
    o.Now = [&] { return clock; };
    auto* dev = new StandIn(o);
    std::unique_ptr<ClusterUpgradeStateManagerImpl> owner(dev);
    o.ValidateOnDevice = false;
    auto* nodeOnly = new StandIn(o);
    std::unique_ptr<ClusterUpgradeStateManagerImpl> owner2(nodeOnly);
    w.wire(dev); w.wire(nodeOnly);
    CountingValidation vd, vn;
    dev->ValidationManager = &vd; nodeOnly->ValidationManager = &vn;
    dev->WithValidationEnabled(kSelector); nodeOnly->WithValidationEnabled(kSelector);
    DriverUpgradePolicySpec p;
    p.AutoUpgrade = true;
    auto reconcile = [&] {
      w.snapshot();  // ListIndex = the position in w.nodes
      EXPECT(R, !dev->ApplyStateIncremental(&w.state, &p).has_value());
      EXPECT(R, !nodeOnly->ApplyStateIncremental(&w.state, &p).has_value());
    };
    reconcile();  // 0: full
    EXPECT(R, dev->calls.size() == 1 && dev->calls[0].full && dev->calls[0].listed.size() == 6);
    EXPECT(R, dev->calls[0].evaluate == (int32_t)(UST_EVAL_ACTUATORS | UST_EVAL_VALIDATION) && nodeOnly->calls[0].evaluate == 0);
    EXPECT(R, (dev->calls[0].lists[1] == std::vector<uint16_t>{M, (uint16_t)(M | RDY)}) && dev->calls[0].lists[0].empty());
    clock += 700;
    reconcile();  // 1: only time passed
    const StandIn::Call& t = dev->calls.back();
    EXPECT(R, !t.full && t.changed.empty() && t.listed.empty() && t.run_src.empty());
    EXPECT(R, dev->Stats().time_only == 1 && t.now == clock);
    // 2: a pod changes readiness (list replaced); another pod gets a new resourceVersion with the same bits (kept)
    w.vpods[0].ContainerStatuses = {{true, 0}}; w.vpods[0].ResourceVersion = "2";
    w.vpods[2].ResourceVersion = "2";
    reconcile();
    EXPECT(R, (dev->calls.back().listed == std::vector<int64_t>{1}) && dev->calls.back().changed.empty());
    EXPECT(R, (dev->calls.back().lists[0] == std::vector<uint16_t>{(uint16_t)(M | RDY), (uint16_t)(M | RDY)}));
    // 3: a start annotation appears on n3 (the node object changed): the node goes down with its start time
    w.nodes[3].Annotations[GetValidationStartTimeAnnotationKey()] = "4321"; w.nodes[3].ResourceVersion = "2";
    reconcile();
    EXPECT(R, (dev->calls.back().changed == std::vector<int64_t>{3}) && (dev->calls.back().startOfChanged == std::vector<int64_t>{4321}));
    EXPECT(R, dev->calls.back().listed.empty());
    // 4: n2 leaves and a node joins at the end, with a pod: runs (no splice), the joined node brings its list and start
    w.nodes[2].Name = "gone"; w.provider.nodes.erase("n2");
    w.nodes.erase(w.nodes.begin() + 2); w.drivers.erase(w.drivers.begin() + 2);
    for (Node& n : w.nodes) w.provider.nodes[n.Name] = &n;
    w.node("n6", UpgradeStateValidationRequired, {{GetValidationStartTimeAnnotationKey(), "777"}});
    w.vpod("v6-a", "n6", true, {true});
    reconcile();
    const StandIn::Call& s = dev->calls.back();
    EXPECT(R, s.evaluate != -1);
    EXPECT(R, (s.run_src == std::vector<int64_t>{0, 3, -1}) && (s.run_len == std::vector<int64_t>{2, 3, 1}));
    EXPECT(R, (s.listed == std::vector<int64_t>{5}) && (s.lists[0] == std::vector<uint16_t>{(uint16_t)(M | RDY)}));
    EXPECT(R, (s.insertStart == std::vector<int64_t>{777}));
    EXPECT(R, nodeOnly->calls.back().run_src.empty());  // the node-only path took a splice
    // 5: two nodes swap places in the list: the runs are the node-only path's
    std::swap(w.nodes[0], w.nodes[1]); std::swap(w.drivers[0], w.drivers[1]);
    for (Node& n : w.nodes) w.provider.nodes[n.Name] = &n;
    reconcile();
    EXPECT(R, !dev->calls.back().run_src.empty());
    EXPECT(R, dev->calls.back().run_src == nodeOnly->calls.back().run_src && dev->calls.back().run_len == nodeOnly->calls.back().run_len);
    EXPECT(R, dev->calls.back().listed.empty() && dev->calls.back().changed.empty());
    // 6: the List fails: nothing about the lists goes down, and ApplyState returns its error at the first
    // validation-required node (the node-only path calls the injected Validate and is not affected)
    w.client.listError = Errorf("the server is unavailable");
    w.snapshot();
    const Error le = dev->ApplyStateIncremental(&w.state, &p);
    EXPECT(R, le && *le == "the server is unavailable");
    EXPECT(R, !nodeOnly->ApplyStateIncremental(&w.state, &p).has_value());
    EXPECT(R, dev->calls.back().listed.empty() && dev->calls.back().changed.empty());
    w.client.listError.reset();
    const auto& st = dev->Stats();
    EXPECT(R, st.full_uploads == 1 && st.lists_sent == 6 + 1 + 1 && st.validate_avoided > 0 && vd.calls == 0 && vn.calls > 0);
    // switching the option off starts the cache over, on the node-only path
    dev->SetValidateOnDevice(false);
    reconcile();
    EXPECT(R, dev->calls.back().full && dev->calls.back().evaluate == 0 && dev->Stats().full_uploads == 2);
  });

  // Replay of pass 10 from hand-made outputs: one validation-required node, each call order, each call failing.
  struct Out { uint8_t next; uint16_t actions; int rc; };
  auto replay = [&](const Out& o, StringMap annotations, const std::string& failOn, int failAt, Error listError,
                    std::vector<std::string>* log) -> Error {
    Small w;
    Node& n = w.node("n0", UpgradeStateValidationRequired, std::move(annotations));
    n.Annotations[GetUpgradeDriverWaitForSafeLoadAnnotationKey()] = "true";
    w.provider.match = failOn;
    w.provider.failAt = failAt;
    w.snapshot();
    auto m = ClusterUpgradeStateManagerImpl::NewDetached({});
    w.wire(m.get());
    CountingValidation v;
    m->ValidationManager = &v;
    EncodedSnapshot e;
    e.entries = {w.owned[0].get()};
    e.state = {UST_STATE_VALIDATION_REQUIRED};
    e.flags = {0};
    e.validateOnDevice = true;
    e.now = 1234;
    e.listError = listError;
    e.deferred[0] = "unable to handle timeout for validation state: strconv.ParseInt: parsing \"x\": invalid syntax";
    DriverUpgradePolicySpec p;
    p.AutoUpgrade = true;
    ust_counters c{};
    c.error_index = o.rc == UST_OK ? -1 : 0;
    c.error_pass = o.rc == UST_OK ? -1 : 10;
    c.error_code = o.rc;
    Error err = m->Replay(e, p, &o.next, &o.actions, o.rc, c);
    log->clear();
    for (const std::string& l : w.log)
      if (l != "restart") log->push_back(l);  // SchedulePodsRestart with no pod: the pod-restart pass always makes it
    EXPECT(R, v.calls == 0);
    return err;
  };
  const std::string unblock = "annotation n0 " + GetUpgradeDriverWaitForSafeLoadAnnotationKey() + "=null";
  const std::string del = "annotation n0 " + vkey + "=null", set = "annotation n0 " + vkey + "=1234";
  const uint16_t U = UST_A_UNBLOCK_SAFE_LOAD, CLR = UST_A_CLEAR_WAIT_START, SET = UST_A_SET_WAIT_START, ST = UST_A_SET_STATE;
  R.it("Replay, pass 10: timeout = unblock, upgrade-failed, delete; clear-then-set; done = delete, state", [&] {
    std::vector<std::string> log;
    EXPECT(R, !replay({UST_STATE_FAILED, (uint16_t)(U | CLR | ST), UST_OK}, {{vkey, "1"}}, "", -1, std::nullopt, &log));
    EXPECT(R, (log == std::vector<std::string>{unblock, "state n0=upgrade-failed", del}));
    EXPECT(R, !replay({UST_STATE_VALIDATION_REQUIRED, (uint16_t)(U | CLR | SET), UST_OK}, {}, "", -1, std::nullopt, &log));
    EXPECT(R, (log == std::vector<std::string>{unblock, del, set}));
    EXPECT(R, !replay({UST_STATE_VALIDATION_REQUIRED, (uint16_t)(U | SET), UST_OK}, {}, "", -1, std::nullopt, &log));
    EXPECT(R, (log == std::vector<std::string>{unblock, set}));
    EXPECT(R, !replay({UST_STATE_VALIDATION_REQUIRED, U, UST_OK}, {}, "", -1, std::nullopt, &log));
    EXPECT(R, (log == std::vector<std::string>{unblock}));
    EXPECT(R, !replay({UST_STATE_UNCORDON_REQUIRED, (uint16_t)(U | CLR | ST), UST_OK}, {}, "", -1, std::nullopt, &log));
    EXPECT(R, (log == std::vector<std::string>{unblock, del, "state n0=uncordon-required"}));
    EXPECT(R, !replay({UST_STATE_DONE, (uint16_t)(U | CLR | ST | UST_A_CLEAR_INITIAL_STATE_ANNO), UST_OK}, {}, "", -1, std::nullopt, &log));
    EXPECT(R, (log == std::vector<std::string>{unblock, del, "state n0=upgrade-done",
                                               "annotation n0 " + GetUpgradeInitialStateAnnotationKey() + "=null"}));
  });
  R.it("Replay, pass 10: an unparsable start time and a failed List end ApplyState after the node's UnblockLoading", [&] {
    std::vector<std::string> log;
    Error e = replay({UST_STATE_VALIDATION_REQUIRED, (uint16_t)(U | UST_A_ERROR), UST_ERR_VALIDATION}, {}, "", -1, std::nullopt, &log);
    EXPECT(R, e && *e == "unable to handle timeout for validation state: strconv.ParseInt: parsing \"x\": invalid syntax");
    EXPECT(R, (log == std::vector<std::string>{unblock}));
    e = replay({UST_STATE_UNCORDON_REQUIRED, (uint16_t)(U | CLR | ST), UST_OK}, {}, "", -1, Errorf("list failed"), &log);
    EXPECT(R, e && *e == "list failed");
    EXPECT(R, (log == std::vector<std::string>{unblock}));
  });
  R.it("Replay, pass 10: a provider error returns at its call (handleTimeout's wrapped, the state change of a timeout ignored)", [&] {
    std::vector<std::string> log;
    const std::string wrap = "unable to handle timeout for validation state: ";
    Error e = replay({UST_STATE_FAILED, (uint16_t)(CLR | ST), UST_OK}, {{vkey, "1"}}, "state n0=upgrade-failed", 0, std::nullopt, &log);
    EXPECT(R, !e && (log == std::vector<std::string>{"FAILED state n0=upgrade-failed", del}));
    e = replay({UST_STATE_FAILED, (uint16_t)(CLR | ST), UST_OK}, {{vkey, "1"}}, del, 0, std::nullopt, &log);
    EXPECT(R, e && *e == wrap + "provider error on " + del.substr(0));
    EXPECT(R, (log == std::vector<std::string>{"state n0=upgrade-failed", "FAILED " + del}));
    e = replay({UST_STATE_VALIDATION_REQUIRED, (uint16_t)(CLR | SET), UST_OK}, {}, del, 0, std::nullopt, &log);
    EXPECT(R, e && *e == "provider error on " + del && (log == std::vector<std::string>{"FAILED " + del}));
    e = replay({UST_STATE_VALIDATION_REQUIRED, (uint16_t)(CLR | SET), UST_OK}, {}, set, 0, std::nullopt, &log);
    EXPECT(R, e && *e == wrap + "provider error on " + set && (log == std::vector<std::string>{del, "FAILED " + set}));
    e = replay({UST_STATE_UNCORDON_REQUIRED, (uint16_t)(CLR | ST), UST_OK}, {}, "state n0=uncordon-required", 0, std::nullopt, &log);
    EXPECT(R, e && *e == "provider error on state n0=uncordon-required");
    e = replay({UST_STATE_VALIDATION_REQUIRED, (uint16_t)(U | SET), UST_OK}, {}, unblock, 0, std::nullopt, &log);
    EXPECT(R, e && *e == "provider error on " + unblock && (log == std::vector<std::string>{"FAILED " + unblock}));
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
  const std::string vkey = GetValidationStartTimeAnnotationKey();
  const int64_t now = 1700000000;
  // One validation-required node through ApplyState twice: with the restated ValidationManagerImpl, and with
  // ValidateOnDevice (full ApplyState and ApplyStateIncremental). Same calls, same node afterwards, same error.
  using Setup = std::function<void(Small&)>;
  auto both = [&](const char* name, const std::string& selector, const Setup& setup,
                  const std::function<void(const Small&, const Error&)>& expect) {
    R.it(name, [&] {
      Small a, b, c;
      for (Small* w : {&a, &b, &c}) { setup(*w); w->snapshot(); }
      StateOptions o;
      o.Now = [&] { return now; };
      auto ma = device(o, ok);
      a.wire(ma.get());
      ValidationManagerImpl ref;
      ref.client = &a.client; ref.provider = &a.provider; ref.podSelector = selector; ref.now = o.Now;
      ma->ValidationManager = &ref;
      if (!selector.empty()) ma->WithValidationEnabled(selector);
      o.ValidateOnDevice = true;
      auto mb = device(o, ok), mc = device(o, ok);
      CountingValidation vb, vc;
      b.wire(mb.get()); c.wire(mc.get());
      mb->ValidationManager = &vb; mc->ValidationManager = &vc;
      if (!selector.empty()) { mb->WithValidationEnabled(selector); mc->WithValidationEnabled(selector); }
      DriverUpgradePolicySpec p;
      p.AutoUpgrade = true;
      const Error ea = ma->ApplyState(&a.state, &p), eb = mb->ApplyState(&b.state, &p), ec = mc->ApplyStateIncremental(&c.state, &p);
      EXPECT(R, ea == eb && ea == ec);
      EXPECT(R, collapse(a.log) == b.log && b.log == c.log);
      EXPECT(R, a.image() == b.image() && b.image() == c.image());
      EXPECT(R, (selector.empty() ? vb.calls == 1 : vb.calls == 0 && vc.calls == 0));
      if (R.failed_here) {
        std::printf("    %s | %s | %s\n", ea ? ea->c_str() : "ok", eb ? eb->c_str() : "ok", ec ? ec->c_str() : "ok");
        for (auto& s : a.log) std::printf("    ref: %s\n", s.c_str());
        for (auto& s : b.log) std::printf("    dev: %s\n", s.c_str());
      }
      expect(b, eb);
    });
  };
  auto label = [](const Small& w) { return w.nodes[0].Labels.at(GetUpgradeStateLabelKey()); };
  auto calls = [](const Small& w) {  // the log without the pod-restart pass's SchedulePodsRestart, which is always made
    size_t k = 0;
    for (const std::string& l : w.log) k += l != "restart";
    return k;
  };
  // validation_manager_test.go:45-171
  both("Validate with an empty podSelector is true (validation_manager_test.go:45)", "", [](Small& w) {
    w.node("n0", UpgradeStateValidationRequired);
  }, [&](const Small& w, const Error& e) { EXPECT(R, !e && label(w) == UpgradeStateUncordonRequired); });
  both("no validation pod on the node: not done, nothing written (:53)", kSelector, [](Small& w) {
    w.node("n0", UpgradeStateValidationRequired);
    w.vpod("v-other-node", "n9", true, {true});
  }, [&](const Small& w, const Error& e) { EXPECT(R, !e && label(w) == UpgradeStateValidationRequired && calls(w) == 0); });
  both("a Running and Ready validation pod: done (:62)", kSelector, [](Small& w) {
    w.node("n0", UpgradeStateValidationRequired);
    w.vpod("v0", "n0", true, {true});
  }, [&](const Small& w, const Error& e) { EXPECT(R, !e && label(w) == UpgradeStateUncordonRequired); });
  both("Running but not Ready: not done, the start time is set (:74)", kSelector, [](Small& w) {
    w.node("n0", UpgradeStateValidationRequired);
    w.vpod("v0", "n0", true, {false});
  }, [&](const Small& w, const Error& e) {
    EXPECT(R, !e && label(w) == UpgradeStateValidationRequired && w.nodes[0].Annotations.at(GetValidationStartTimeAnnotationKey()) == "1700000000");
  });
  both("not Running: not done (:89)", kSelector, [](Small& w) {
    w.node("n0", UpgradeStateValidationRequired);
    w.vpod("v0", "n0", false, {});
  }, [&](const Small& w, const Error& e) { EXPECT(R, !e && label(w) == UpgradeStateValidationRequired); });
  both("not done before the timeout: upgrade-failed, start time removed (:104)", kSelector, [&](Small& w) {
    w.node("n0", UpgradeStateValidationRequired, {{vkey, std::to_string(now - 601)}});
    w.vpod("v0", "n0", true, {false});
  }, [&](const Small& w, const Error& e) {
    EXPECT(R, !e && label(w) == UpgradeStateFailed && !w.nodes[0].Annotations.count(GetValidationStartTimeAnnotationKey()));
  });
  both("done before the timeout: start time removed (:139)", kSelector, [&](Small& w) {
    w.node("n0", UpgradeStateValidationRequired, {{vkey, std::to_string(now - 599)}});
    w.vpod("v0", "n0", true, {true});
  }, [&](const Small& w, const Error& e) {
    EXPECT(R, !e && label(w) == UpgradeStateUncordonRequired && !w.nodes[0].Annotations.count(GetValidationStartTimeAnnotationKey()));
  });
  // upgrade_state_test.go:1018-1127 and around them
  both("validation done with the initial-state annotation: upgrade-done, annotation removed (upgrade_state_test.go:1089)", kSelector, [&](Small& w) {
    w.node("n0", UpgradeStateValidationRequired, {{GetUpgradeInitialStateAnnotationKey(), "true"}});
    w.vpod("v0", "n0", true, {true, true});
  }, [&](const Small& w, const Error& e) {
    EXPECT(R, !e && label(w) == UpgradeStateDone && !w.nodes[0].Annotations.count(GetUpgradeInitialStateAnnotationKey()));
  });
  both("a ready pod listed before a not-ready one resets the start time: the node never times out", kSelector, [&](Small& w) {
    w.node("n0", UpgradeStateValidationRequired, {{vkey, std::to_string(now - 5000)}});
    w.vpod("v0-ready", "n0", true, {true});
    w.vpod("v1-not", "n0", true, {false});
  }, [&](const Small& w, const Error& e) {
    EXPECT(R, !e && label(w) == UpgradeStateValidationRequired && w.nodes[0].Annotations.at(GetValidationStartTimeAnnotationKey()) == "1700000000");
  });
  both("an unparsable start time: ApplyState returns Validate's error after the node's UnblockLoading", kSelector, [&](Small& w) {
    w.node("n0", UpgradeStateValidationRequired, {{vkey, "soon"}, {GetUpgradeDriverWaitForSafeLoadAnnotationKey(), "true"}});
    w.node("n1", UpgradeStateValidationRequired);
    w.vpod("v0", "n0", true, {false});
    w.vpod("v1", "n1", true, {true});
  }, [&](const Small& w, const Error& e) {
    EXPECT(R, e && *e == "unable to handle timeout for validation state: strconv.ParseInt: parsing \"soon\": invalid syntax");
    EXPECT(R, calls(w) == 1 && w.nodes[1].Labels.at(GetUpgradeStateLabelKey()) == UpgradeStateValidationRequired);
  });
  both("a start time that overflows before a bad character: ParseUint's range error (strconv/atoi.go)", kSelector, [&](Small& w) {
    w.node("n0", UpgradeStateValidationRequired, {{vkey, "99999999999999999999x"}});
    w.vpod("v0", "n0", true, {false});
  }, [&](const Small& w, const Error& e) {
    EXPECT(R, e && *e == "unable to handle timeout for validation state: strconv.ParseInt: parsing \"99999999999999999999x\": value out of range");
  });
  both("a failed List: ApplyState returns its error at the first validation-required node", kSelector, [&](Small& w) {
    w.node("n0", UpgradeStateUncordonRequired);
    w.node("n1", UpgradeStateValidationRequired, {{GetUpgradeDriverWaitForSafeLoadAnnotationKey(), "true"}});
    w.client.listError = Errorf("the server could not find the requested resource");
    w.vpod("v1", "n1", true, {true});
  }, [&](const Small& w, const Error& e) {
    EXPECT(R, e && *e == "the server could not find the requested resource" && calls(w) == 1);
    EXPECT(R, w.nodes[0].Labels.at(GetUpgradeStateLabelKey()) == UpgradeStateUncordonRequired);
  });
  both("a failed List without a validation-required node is no error", kSelector, [&](Small& w) {
    w.node("n0", UpgradeStateUncordonRequired);
    w.client.listError = Errorf("the server could not find the requested resource");
  }, [&](const Small& w, const Error& e) { EXPECT(R, !e && w.nodes[0].Labels.at(GetUpgradeStateLabelKey()) == UpgradeStateDone); });
  both("a failing annotation write returns handleTimeout's error", kSelector, [&](Small& w) {
    w.node("n0", UpgradeStateValidationRequired);
    w.vpod("v0", "n0", true, {false});
    w.provider.match = GetValidationStartTimeAnnotationKey();
    w.provider.failAt = 0;
  }, [&](const Small& w, const Error& e) { EXPECT(R, e && e->rfind("unable to handle timeout for validation state: provider error", 0) == 0); });

  R.it("more changed outputs than the sparse arrays hold: every output is fetched and replayed like the sparse ones", [&] {
    // 6000 validation-required nodes: the delta call's arrays hold n / 4 + 1024 outputs, and on the second reconcile every
    // node's outputs change (its start time was set by the first), on the fourth every not-ready node times out
    const int n = 6000;
    Small a, b;
    for (Small* w : {&a, &b})
      for (int i = 0; i < n; i++) {
        const std::string name = "n" + std::to_string(i);
        w->node(name, UpgradeStateValidationRequired);
        w->vpod("v-" + name, name, true, {i % 3 == 0});
      }
    int64_t t = now;
    StateOptions o;
    o.Now = [&] { return t; };
    auto ma = device(o, ok);
    o.ValidateOnDevice = true;
    auto mb = device(o, ok);
    a.wire(ma.get()); b.wire(mb.get());
    ValidationManagerImpl ref;
    ref.client = &a.client; ref.provider = &a.provider; ref.podSelector = kSelector; ref.now = o.Now;
    CountingValidation vb;
    ma->ValidationManager = &ref; mb->ValidationManager = &vb;
    ma->WithValidationEnabled(kSelector); mb->WithValidationEnabled(kSelector);
    DriverUpgradePolicySpec p;
    p.AutoUpgrade = true;
    for (int rec = 0; rec < 4; rec++) {
      a.log.clear(); b.log.clear();
      a.snapshot(); b.snapshot();
      const Error ea = ma->ApplyState(&a.state, &p), eb = mb->ApplyStateIncremental(&b.state, &p);
      EXPECT(R, ea == eb && !ea);
      EXPECT(R, collapse(a.log) == b.log && (rec == 2 || a.log.size() > 1000));
      EXPECT(R, a.image() == b.image());
      if (R.failed_here) { std::printf("    (reconcile %d)\n", rec); break; }
      t += rec == 2 ? 700 : 10;
    }
    const auto& st = mb->Stats();
    std::printf("    %lld outputs received after the full upload\n", (long long)st.outputs_received);
    EXPECT(R, st.full_uploads == 1 && st.outputs_received >= 2 * n && vb.calls == 0);
    size_t failed = 0;
    for (const Node& nd : b.nodes) failed += nd.Labels.at(GetUpgradeStateLabelKey()) == UpgradeStateFailed;
    EXPECT(R, failed == (size_t)(n - (n + 2) / 3));
  });
  R.it("a reconcile in which only time passed sends nothing, and the device's clock times the node out", [&] {
    Small w;
    w.node("n0", UpgradeStateValidationRequired);
    w.node("n1", UpgradeStateDone);
    w.vpod("v0", "n0", true, {false});
    int64_t t = now;
    StateOptions o;
    o.ValidateOnDevice = true;
    o.Now = [&] { return t; };
    auto m = device(o, ok);
    w.wire(m.get());
    CountingValidation v;
    m->ValidationManager = &v;
    m->WithValidationEnabled(kSelector);
    DriverUpgradePolicySpec p;
    p.AutoUpgrade = true;
    w.snapshot();
    EXPECT(R, !m->ApplyStateIncremental(&w.state, &p));  // sets the start time
    EXPECT(R, w.nodes[0].Annotations.at(GetValidationStartTimeAnnotationKey()) == std::to_string(now));
    w.snapshot();
    t += 10;
    EXPECT(R, !m->ApplyStateIncremental(&w.state, &p));  // the annotation write bumped the node: it goes down once
    const int64_t sent = m->Stats().lists_sent;
    for (int k = 0; k < 3; k++) {
      t += 200;
      w.snapshot();
      EXPECT(R, !m->ApplyStateIncremental(&w.state, &p));
    }
    EXPECT(R, m->Stats().time_only == 3 && m->Stats().lists_sent == sent);
    EXPECT(R, w.nodes[0].Labels.at(GetUpgradeStateLabelKey()) == UpgradeStateFailed);  // 610 s after the start
    EXPECT(R, !w.nodes[0].Annotations.count(GetValidationStartTimeAnnotationKey()) && v.calls == 0);
  });
}

// The reconcile loop: the world of build_state_spec.hpp plus validation pods, the clock, List errors and provider errors.
struct VWorld {
  spec::BWorld w;
  SelectorClient sel;
  FailingProvider fp;
  std::deque<Pod> vpods;
  std::vector<char> valive;
  std::set<std::string> seeded;
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
    for (size_t i = 0; i < vpods.size(); i++)
      if (valive[i]) sel.all.push_back(&vpods[i]);
    std::stable_sort(sel.all.begin(), sel.all.end(), [](const Pod* x, const Pod* y) { return x->Name < y->Name; });
  }
};

// between reconciles, the same on both worlds
void vevolve(VWorld& v, int rec, spec::BLcg r) {
  spec::bevolve(v.w, rec, spec::BLcg{r.s ^ 0x5555});
  for (size_t i = 0; i < v.vpods.size(); i++) {  // validation pods of nodes that left go with them
    if (!v.valive[i]) continue;
    if (!v.w.provider.nodes.count(v.vpods[i].NodeName)) { v.valive[i] = 0; continue; }
    Pod& p = v.vpods[i];
    if (!p.Labels.count("never") && r.chance(20)) {  // the validation finishes
      p.Phase = "Running";
      for (auto& cs : p.ContainerStatuses) cs.Ready = true;
      if (p.ContainerStatuses.empty()) p.ContainerStatuses = {{true, 0}};
      v.w.bumpPod(p);
    }
  }
  for (Node& nd : v.w.nodes) {  // a node that reaches validation-required gets its validation pods (0-3) the first time
    if (nd.Name.empty() || v.seeded.count(nd.Name)) continue;
    auto it = nd.Labels.find(GetUpgradeStateLabelKey());
    if (it == nd.Labels.end() || it->second != UpgradeStateValidationRequired) continue;
    v.seeded.insert(nd.Name);
    const int k = (int)(r.next() % 4), kind = (int)(r.next() % 4);
    for (int j = 0; j < k; j++) {
      // kind 0: they finish some time; 1: the first never does (times out); 2: the first is ready, the second never is
      // (the start time is reset every reconcile: no timeout); 3: a mix
      const bool ready = kind == 2 && j == 0;
      Pod p = makeValidationPod("val-" + nd.Name + "-" + std::to_string(j), nd.Name, ready || r.chance(50), {ready}, v.w.version++);
      if ((kind == 1 && j == 0) || (kind == 2 && j == 1) || (kind == 3 && r.chance(30))) p.Labels["never"] = "1";
      v.vpods.push_back(p);
      v.valive.push_back(1);
    }
  }
  // now and then an unparsable start time on the validation-required nodes, taken away again three reconciles later
  if (rec % 40 == 13 || rec % 40 == 16) {
    for (Node& nd : v.w.nodes) {
      auto it = nd.Labels.find(GetUpgradeStateLabelKey());
      if (nd.Name.empty() || it == nd.Labels.end() || it->second != UpgradeStateValidationRequired) continue;
      if (rec % 40 == 13) nd.Annotations[GetValidationStartTimeAnnotationKey()] = "not-a-number";
      else if (nd.Annotations.count(GetValidationStartTimeAnnotationKey()) && nd.Annotations[GetValidationStartTimeAnnotationKey()] == "not-a-number")
        nd.Annotations.erase(GetValidationStartTimeAnnotationKey());
      spec::LogProvider::bump(&nd);
    }
  }
}

void loop(Runner& R, bool requestor, int n_nodes, int rounds, bool* ok) {
  SetDriverName("gpu");
  const std::string name = std::string("ApplyStateIncremental with ValidateOnDevice == ApplyState with ValidationManagerImpl over a reconcile loop (") +
                           (requestor ? "requestor" : "in-place") + " mode)";
  R.it(name.c_str(), [&] {
    VWorld a, b;
    spec::bpopulate(a.w, n_nodes, 91); spec::bpopulate(b.w, n_nodes, 91);
    int64_t clock = 1700000000;
    StateOptions o;
    o.Requestor.UseMaintenanceOperator = requestor;
    o.Now = [&] { return clock; };
    StateOptions od = o;
    od.ValidateOnDevice = true;
    auto mb = device(od, ok);
    b.wire(mb.get());
    CountingValidation vb;
    mb->ValidationManager = &vb;
    mb->WithValidationEnabled(kSelector);
    ValidationManagerImpl ref;
    ref.client = &a.sel; ref.provider = &a.fp; ref.podSelector = kSelector; ref.now = o.Now;
    DriverUpgradePolicySpec p;
    p.AutoUpgrade = true;
    p.MaxParallelUpgrades = 12;
    p.MaxUnavailable = IntOrString::FromString("40%");
    p.DrainSpec = upgrade::DrainSpec{};
    p.DrainSpec->Enable = true;
    const int64_t steps[] = {17, 90, 240, 45, 400, 3};
    int listErrors = 0, providerErrors = 0, parseErrors = 0, timeouts = 0, resets = 0, errors = 0;
    for (int rec = 0; rec < rounds; rec++) {
      auto ma = device(o, ok);  // the reference's way: a fresh manager every reconcile
      a.wire(ma.get());
      ma->ValidationManager = &ref;
      ma->WithValidationEnabled(kSelector);
      a.publish(); b.publish();
      a.w.log.clear(); b.w.log.clear();
      const bool listFails = rec % 37 == 11, providerFails = rec % 41 == 17;
      for (VWorld* v : {&a, &b}) {
        v->sel.listError = listFails ? Errorf("etcdserver: request timed out") : std::nullopt;
        v->fp.match = providerFails ? GetValidationStartTimeAnnotationKey() : "";
        v->fp.failAt = 0; v->fp.seen = 0;
      }
      std::unique_ptr<ClusterUpgradeState> sa, sb;
      Error ea, eb;
      ea = ma->BuildState("gpu-operator", {}, &sa);
      eb = mb->BuildStateIncremental("gpu-operator", {}, &sb);
      EXPECT(R, ea == eb);
      if (!ea && !eb) {
        ea = ma->ApplyState(sa.get(), &p);
        eb = mb->ApplyStateIncremental(sb.get(), &p);
        EXPECT(R, ea == eb);
      }
      if (ea) {
        errors++;
        listErrors += *ea == "etcdserver: request timed out";
        providerErrors += ea->find("provider error") != std::string::npos;
        parseErrors += ea->find("strconv.ParseInt") != std::string::npos;
      }
      for (const std::string& s : a.w.log) {
        timeouts += s.find("=upgrade-failed") != std::string::npos;
        resets += s.find(GetValidationStartTimeAnnotationKey() + "=null") != std::string::npos;
      }
      EXPECT(R, collapse(a.w.log) == collapse(b.w.log));
      EXPECT(R, spec::bimage(a.w) == spec::bimage(b.w));
      if (R.failed_here) {
        std::printf("    (reconcile %d: %s / %s)\n", rec, ea ? ea->c_str() : "ok", eb ? eb->c_str() : "ok");
        const auto la = collapse(a.w.log), lb = collapse(b.w.log);
        for (size_t k = 0; k < std::max(la.size(), lb.size()); k++)
          if (k >= la.size() || k >= lb.size() || la[k] != lb[k])
            std::printf("    #%zu ref: %s | dev: %s\n", k, k < la.size() ? la[k].c_str() : "-", k < lb.size() ? lb[k].c_str() : "-");
        break;
      }
      clock += steps[rec % 6];
      vevolve(a, rec, spec::BLcg{7000u + (uint64_t)rec}); vevolve(b, rec, spec::BLcg{7000u + (uint64_t)rec});
    }
    const auto& st = mb->Stats();
    std::printf("    %lld reconciles, %lld full uploads, %lld reorders, %lld lists sent, %lld reused, %lld time-only, %lld Validate calls "
                "avoided (reference: %d); errors: %d (List %d, provider %d, parse %d); %d timeouts, %d start-time deletes\n",
                (long long)st.reconciles, (long long)st.full_uploads, (long long)st.reorders, (long long)st.lists_sent,
                (long long)st.lists_reused, (long long)st.time_only, (long long)st.validate_avoided, ref.calls, errors, listErrors,
                providerErrors, parseErrors, timeouts, resets);
    EXPECT(R, vb.calls == 0 && ref.calls > 0);
    EXPECT(R, st.full_uploads == 1 && st.reorders > 0);
    EXPECT(R, st.validate_avoided > 0 && st.lists_reused > st.lists_sent);
    EXPECT(R, listErrors > 0 && providerErrors > 0 && parseErrors > 0 && timeouts > 0 && resets > 0);
  });
}

}  // namespace

int main(int argc, char** argv) {
  const bool gpu = argc > 1 && std::strcmp(argv[1], "--gpu") == 0;
  Runner R;
  bool ok = true;
  if (gpu) {
    gpu_specs(R, &ok);
    loop(R, false, 300, 300, &ok);
    loop(R, true, 300, 300, &ok);
  } else {
    cpu_specs(R);
  }
  std::printf("# %d passed, %d failed\n", R.passed, R.failed);
  return (R.failed == 0 && ok) ? 0 : 1;
}
