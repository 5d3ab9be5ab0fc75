// ClusterUpgradeStateManagerImpl::NextTimeout (upgrade.hpp): the device's next deadline carried out of the clocked calls.
//   deadline_test         host halves only: a stand-in behind EvaluateCachedPods supplies the value; NextTimeout carries
//                         it out of ApplyStateIncremental with WaitForCompletionOnDevice or ValidateOnDevice, and is nullopt
//                         without them, after a failed call and when nothing is pending
//   deadline_test --gpu   300 reconciles of BuildStateIncremental + ApplyStateIncremental with WaitForCompletionOnDevice
//                         (ValidateOnDevice off and on, in-place and requestor mode) against BuildState + ApplyState with
//                         the restated PodManagerImpl and ValidationManagerImpl (wait_spec.hpp, validation_spec.hpp): the
//                         same calls every reconcile. Whenever a reconcile changes no object the clock jumps to
//                         NextTimeout(); the reconcile there changes one, and a twin manager reconciling one second earlier
//                         makes exactly the calls of the reconcile before the jump and changes nothing
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <set>

#include "wait_spec.hpp"

using namespace upgrade;
using namespace wspec;

namespace {

const char* kWait = "app=my-app";

// nodes with a driver pod each, in ListIndex order, and their wait-selector pods
struct Cluster {
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
  Cluster() { provider.log = cordon.log = drain.log = podm.log = &log; ds.Name = "driver"; ds.UID = "uid-ds"; }
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
    pods.push_back(makeWaitPod("job-" + name, name, "Running", 1));
    return n;
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
  }
  void wire(ClusterUpgradeStateManagerImpl* m) {
    m->NodeUpgradeStateProvider = &provider; m->CordonManager = &cordon; m->DrainManager = &drain; m->PodManager = &podm;
    m->SafeDriverLoadManager = &safeLoad; m->K8sClient = &client;
  }
  std::vector<std::string> calls() const {  // the log without the pod-restart pass's SchedulePodsRestart, which is always made
    std::vector<std::string> out;
    for (const std::string& l : log)
      if (l.rfind("restart", 0) != 0) out.push_back(l);
    return out;
  }
};

DriverUpgradePolicySpec waitPolicy(int timeout) {
  DriverUpgradePolicySpec p;
  p.AutoUpgrade = true;
  p.WaitForCompletion = WaitForCompletionSpec{kWait, timeout};
  return p;
}

// Outputs "no transition, no call"; the next deadline is whatever the test puts in `deadline`.
struct StandIn : ClusterUpgradeStateManagerImpl {
  std::optional<int64_t> deadline;
  int pods_calls = 0, node_calls = 0;
  explicit StandIn(StateOptions o) : ClusterUpgradeStateManagerImpl(std::move(o)) {}
  static void quiet(Cache* k, ust_counters* c) {
    const size_t n = k->slots.size();
    k->next.assign(n + 1, 0);
    k->actions.assign(n + 1, 0);
    k->outcome.assign(n + 1, UST_OUTCOME_NONE);
    for (size_t i = 0; i < n; i++) k->next[i] = k->state[i] & UST_HOT_STATE_MASK;
    std::memset(c, 0, sizeof(*c));
    c->error_index = -1;
  }
  int EvaluateCached(const ust_policy&, bool, const std::vector<int64_t>&, Cache* k, ust_counters* c) override {
    node_calls++;
    quiet(k, c);
    return UST_OK;
  }
  int EvaluateCachedPods(const ust_policy&, int64_t, int64_t, bool, const std::vector<int64_t>&, Cache* k, ust_counters* c) override {
    pods_calls++;
    quiet(k, c);
    cachedDeadline_ = deadline;
    return UST_OK;
  }
};

void cpu_specs(Runner& R) {
  SetDriverName("gpu");
  const std::string wkey = GetWaitForPodCompletionStartTimeAnnotationKey();
  R.it("NextTimeout carries EvaluateCachedPods' deadline out of ApplyStateIncremental, and only from a clocked call", [&] {
    Cluster w;
    w.node("n0", UpgradeStateWaitForJobsRequired, {{wkey, "1700000000"}});
    w.node("n1", UpgradeStateDone);
    w.snapshot();
    StateOptions o;
    o.WaitForCompletionOnDevice = true;
    o.Now = [] { return (int64_t)1700000010; };
    StandIn m(o);
    w.wire(&m);
    const DriverUpgradePolicySpec p = waitPolicy(100);
    EXPECT(R, !m.NextTimeout().has_value());
    m.deadline = 1700000101;
    EXPECT(R, !m.ApplyStateIncremental(&w.state, &p).has_value());
    EXPECT(R, m.pods_calls == 1 && m.NextTimeout() == std::optional<int64_t>(1700000101));
    m.deadline.reset();  // nothing pending
    EXPECT(R, !m.ApplyStateIncremental(&w.state, &p).has_value());
    EXPECT(R, m.pods_calls == 2 && !m.NextTimeout().has_value());
    m.deadline = 5;
    EXPECT(R, !m.ApplyStateIncremental(&w.state, &p).has_value() && m.NextTimeout() == std::optional<int64_t>(5));
    EXPECT(R, m.ApplyStateIncremental(nullptr, &p).has_value() && !m.NextTimeout().has_value());  // a failed call
    EXPECT(R, !m.ApplyStateIncremental(&w.state, &p).has_value() && m.NextTimeout() == std::optional<int64_t>(5));
    // without a wait selector the option answers nothing: the node-only call, no deadline
    DriverUpgradePolicySpec q = p;
    q.WaitForCompletion->PodSelector = "";
    EXPECT(R, !m.ApplyStateIncremental(&w.state, &q).has_value());
    EXPECT(R, m.node_calls == 1 && !m.NextTimeout().has_value());
  });
  R.it("NextTimeout is nullopt without WaitForCompletionOnDevice and ValidateOnDevice", [&] {
    Cluster w;
    w.node("n0", UpgradeStateWaitForJobsRequired, {{wkey, "1700000000"}});
    w.snapshot();
    StandIn m(StateOptions{});
    w.wire(&m);
    m.deadline = 77;
    const DriverUpgradePolicySpec p = waitPolicy(100);
    EXPECT(R, !m.ApplyStateIncremental(&w.state, &p).has_value());
    EXPECT(R, m.node_calls == 1 && m.pods_calls == 0 && !m.NextTimeout().has_value());
  });
}

// ---- on the device: a reconcile loop that sleeps until NextTimeout() -------------------------------------------------
// The world of build_state_spec.hpp plus job pods and validation pods (as in wait_test.cpp's loop), without injected errors:
// the loop is about the clock.
const char* kLoopWait = "tier=gpu";  // job pods carry it, and so do the validation pods: some pods match both selectors
const char* kValidation = "app=validator,tier=gpu";

// The selector client with NodeMaintenance objects (requestor mode): created and deleted by the passes, Ready when the
// cluster moves on (wevolve), which touches the node so that a cache keyed by resourceVersion sees it.
struct NMClient : vspec::SelectorClient {
  std::map<std::string, NodeMaintenance> nm;
  Error GetNodeMaintenance(const std::string& name, NodeMaintenance** out) override {
    auto it = nm.find(name);
    *out = it == nm.end() ? nullptr : &it->second;
    return std::nullopt;
  }
  Error CreateOrUpdateNodeMaintenance(NodeUpgradeState* s) override { nm[s->Node->Name].Name = s->Node->Name; return std::nullopt; }
  Error DeleteOrUpdateNodeMaintenance(NodeUpgradeState* s) override { nm.erase(s->Node->Name); return std::nullopt; }
};

struct WWorld {
  spec::BWorld w;
  NMClient sel;
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

// Between two reconciles: the cluster moves on (spec::bevolve), jobs finish or start, validations finish; a node that is
// cordoned gets 0-3 jobs the first time, a validation-required node 0-2 validation pods; some never finish.
void wevolve(WWorld& v, int rec, spec::BLcg r) {
  spec::bevolve(v.w, rec, spec::BLcg{r.s ^ 0x5555});
  for (size_t i = 0; i < v.extra.size(); i++) {
    if (!v.alive[i]) continue;
    if (!v.w.provider.nodes.count(v.extra[i].NodeName)) { v.alive[i] = 0; continue; }
    Pod& p = v.extra[i];
    if (p.Labels.count("never")) continue;
    if (p.Namespace == "jobs" && r.chance(12)) {
      p.Phase = p.Phase == "Pending" ? "Running" : (r.chance(70) ? "Succeeded" : "Failed");
      v.w.bumpPod(p);
    } else if (p.Namespace != "jobs" && r.chance(20)) {
      p.Phase = "Running";
      p.ContainerStatuses = {{true, 0}};
      v.w.bumpPod(p);
    }
  }
  for (auto& kv : v.sel.nm)  // the maintenance operator finishes
    if (!kv.second.ReadyConditionWithReasonReady && r.chance(30)) {
      kv.second.ReadyConditionWithReasonReady = true;
      auto nd = v.w.provider.nodes.find(kv.first);
      if (nd != v.w.provider.nodes.end()) spec::LogProvider::bump(nd->second);
    }
  for (Node& nd : v.w.nodes) {
    if (nd.Name.empty()) continue;
    auto it = nd.Labels.find(GetUpgradeStateLabelKey());
    const std::string st = it == nd.Labels.end() ? "" : it->second;
    if ((st == UpgradeStateCordonRequired || st == UpgradeStateWaitForJobsRequired) && !v.seededJobs.count(nd.Name)) {
      v.seededJobs.insert(nd.Name);
      for (int j = (int)(r.next() % 4); j > 0; j--) {
        const char* phase = r.chance(60) ? "Running" : r.chance(50) ? "Pending" : "Succeeded";
        Pod p = makeWaitPod("job-" + nd.Name + "-" + std::to_string(j), nd.Name, phase, v.w.version++);
        p.Labels["tier"] = "gpu";
        if (r.chance(60)) p.Labels["never"] = "1";  // more than in wait_test.cpp's loop: jobs that run into the timeout
        v.add(p);
      }
    }
    if (st == UpgradeStateValidationRequired && !v.seededVal.count(nd.Name)) {
      v.seededVal.insert(nd.Name);
      for (int j = (int)(r.next() % 3); j > 0; j--) {
        Pod p = vspec::makeValidationPod("val-" + nd.Name + "-" + std::to_string(j), nd.Name, r.chance(50), {false}, v.w.version++);
        if (r.chance(35)) p.Labels["never"] = "1";
        v.add(p);
      }
    }
  }
}

// What the cluster does at once with the last reconcile's calls, and nothing else (the first step of spec::bevolve):
// cordons and uncordons take effect. Restarted driver pods come back when it moves on.
void settle(WWorld& v) {
  spec::BWorld& w = v.w;
  for (Node* n : w.cordon.cordoned) { n->Unschedulable = true; spec::LogProvider::bump(n); }
  for (Node* n : w.cordon.uncordoned) { n->Unschedulable = false; spec::LogProvider::bump(n); }
  w.cordon.cordoned.clear(); w.cordon.uncordoned.clear();
}

std::unique_ptr<ClusterUpgradeStateManagerImpl> device(StateOptions o, bool* ok) {
  std::unique_ptr<ClusterUpgradeStateManagerImpl> m;
  if (auto e = ClusterUpgradeStateManagerImpl::New(0, o, &m)) {
    std::printf("cannot create manager: %s\n", e->c_str());
    *ok = false;
    return ClusterUpgradeStateManagerImpl::NewDetached(o);
  }
  return m;
}

// A call that changes an object: everything but the actuators' schedulers ("wait", "evict", "drain", "restart"), whose
// work this world does when it moves on.
bool changesObjects(const std::vector<std::string>& log) {
  for (const std::string& s : log)
    if (s.rfind("restart", 0) != 0 && s.rfind("wait ", 0) != 0 && s.rfind("evict ", 0) != 0 && s.rfind("drain", 0) != 0) return true;
  return false;
}

void loop(Runner& R, bool requestor, bool validate, int n_nodes, int rounds, bool* ok) {
  SetDriverName("gpu");
  const std::string name = std::string("a reconcile loop that sleeps until NextTimeout() makes the reference's calls, and a twin one "
                                       "second before each deadline changes nothing (") +
                           (requestor ? "requestor" : "in-place") + " mode, ValidateOnDevice " + (validate ? "on" : "off") + ")";
  R.it(name.c_str(), [&] {
    WWorld a, b;
    spec::bpopulate(a.w, n_nodes, 59); spec::bpopulate(b.w, n_nodes, 59);
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
    int jumps = 0, landed = 0, quiet = 0, twins = 0;
    bool jumped = false;
    for (int rec = 0; rec < rounds; rec++) {
      p.WaitForCompletion->TimeoutSecond = rec < 150 ? 300 : rec < 200 ? 0 : 120;
      auto ma = device(o, ok);  // the reference's way: a fresh manager every reconcile
      a.wire(ma.get());
      ma->PodManager = &ref;
      if (validate) { ma->ValidationManager = &vref; ma->WithValidationEnabled(kValidation); }
      a.publish(); b.publish();
      a.w.log.clear(); b.w.log.clear();
      const std::string before = spec::bimage(b.w);
      std::unique_ptr<ClusterUpgradeState> sa, sb;
      Error ea = ma->BuildState("gpu-operator", {}, &sa);
      Error eb = mb->BuildStateIncremental("gpu-operator", {}, &sb);
      EXPECT(R, ea == eb);
      if (!ea && !eb) {
        ea = ma->ApplyState(sa.get(), &p);
        eb = mb->ApplyStateIncremental(sb.get(), &p);
        EXPECT(R, ea == eb);
      }
      EXPECT(R, vspec::collapse(a.w.log) == vspec::collapse(b.w.log));
      EXPECT(R, spec::bimage(a.w) == spec::bimage(b.w));
      const bool changed = changesObjects(b.w.log) || spec::bimage(b.w) != before;
      if (jumped) {  // the reconcile at the reported time: a deadline fired
        EXPECT(R, changed);
        landed += changed;
        jumped = false;
      }
      if (R.failed_here) {
        std::printf("    (reconcile %d at %lld: %s / %s)\n", rec, (long long)clock, ea ? ea->c_str() : "ok", eb ? eb->c_str() : "ok");
        const auto la = vspec::collapse(a.w.log), lb = vspec::collapse(b.w.log);
        for (size_t k = 0; k < std::max(la.size(), lb.size()); k++)
          if (k >= la.size() || k >= lb.size() || la[k] != lb[k])
            std::printf("    #%zu ref: %s | dev: %s\n", k, k < la.size() ? la[k].c_str() : "-", k < lb.size() ? lb[k].c_str() : "-");
        break;
      }
      // both PodManagers restarted the same driver pods: the world re-creates them when it next moves on
      // (once each: a pod is restarted by every reconcile until then)
      for (auto* q : {&ref.restarted, &pb.restarted})
        for (Pod* pod : *q) {
          auto& rs = (q == &ref.restarted ? a : b).w.pods.restarted;
          if (std::find(rs.begin(), rs.end(), pod) == rs.end()) rs.push_back(pod);
        }
      ref.restarted.clear(); pb.restarted.clear();
      const std::optional<int64_t> t = (ea || eb) ? std::nullopt : mb->NextTimeout();
      if (!ea && !eb && !changed) {
        quiet++;
        if (t) {
          EXPECT(R, *t > clock);
          // a twin reconciling the same objects one second before the deadline: the calls of this reconcile, no change
          const std::vector<std::string> calls = vspec::collapse(b.w.log);
          int64_t twinClock = *t - 1;
          StateOptions ot = od;
          ot.Now = [&twinClock] { return twinClock; };
          auto twin = device(ot, ok);
          b.wire(twin.get());
          CountingPods pt;
          pt.log = &b.w.log;
          twin->PodManager = &pt;
          vspec::CountingValidation vt;
          if (validate) { twin->ValidationManager = &vt; twin->WithValidationEnabled(kValidation); }
          b.publish();
          b.w.log.clear();
          std::unique_ptr<ClusterUpgradeState> st;
          EXPECT(R, !twin->BuildState("gpu-operator", {}, &st));
          if (st) EXPECT(R, !twin->ApplyState(st.get(), &p));
          EXPECT(R, vspec::collapse(b.w.log) == calls && spec::bimage(b.w) == before);
          EXPECT(R, twin->NextTimeout() == t && pt.waitCalls == 0 && vt.calls == 0);
          // (the twin's pod restarts are those of the reconcile before it, already recorded: not recorded twice)
          b.wire(mb.get());
          mb->PodManager = &pb;
          if (validate) mb->ValidationManager = &vb;
          twins++;
          clock = *t;  // nothing else happens until then
          jumps++;
          jumped = true;
          continue;
        }
      }
      // The cluster moves on when the reconciles have settled with nothing pending, and every tenth reconcile; otherwise only
      // the last reconcile's actuator calls take effect, and the loop reconciles again a few seconds later.
      if ((!ea && !eb && !changed) || rec % 10 == 9) {
        clock += steps[rec % 6];
        wevolve(a, rec, spec::BLcg{9100u + (uint64_t)rec}); wevolve(b, rec, spec::BLcg{9100u + (uint64_t)rec});
      } else {
        clock += 3;
        settle(a); settle(b);
      }
    }
    std::printf("    %d reconciles changed no object; %d jumps to NextTimeout(), %d of them landed on a change; %d twins\n", quiet,
                jumps, landed, twins);
    EXPECT(R, pb.waitCalls == 0 && vb.calls == 0 && ref.checks > 0);
    EXPECT(R, jumps >= 5 && landed == jumps && twins == jumps);
  });
}

}  // namespace

int main(int argc, char** argv) {
  const bool gpu = argc > 1 && std::strcmp(argv[1], "--gpu") == 0;
  Runner R;
  bool ok = true;
  if (gpu) {
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
