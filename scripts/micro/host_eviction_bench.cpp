// ApplyStateIncremental per reconcile with StateOptions::EvictionOnDevice off and on, through the H100 (one GPU).
// The cluster is C4-like: n nodes in the states of encode_bench.cpp, about 10 % of them pod-deletion-required or
// drain-required with 20-40 workload pods each (some GPU pods the deletion filter selects, some DaemonSet pods, some with
// an emptyDir). Off: the injected PodManager and DrainManager restate the reference's SchedulePodEviction and
// ScheduleNodesDrain (one List per node, the filter chain, the eviction); on: one pod List and one DaemonSet List per
// reconcile, the workload pods resident, the evictions handed to the PodEvictor's workers (waited for inside the timing).
// Three series after one untimed full reconcile each:
//   changed   1 % of the objects change between reconciles (node objects, driver pods, workload pods)
//   time      only the clock moves
//   moved     0.1 % of the nodes move in BuildState's list (pairs swap places)
// The mocks make a List free and the provider calls and evictions no-ops, so this measures what the mirror and the library
// add per reconcile; it does not measure the API server's saving, only counts the Lists.
// Build (from the repository root, after build()) and run on a GPU machine:
//   g++ -O2 -std=c++17 -pthread -I. scripts/micro/host_eviction_bench.cpp -Lk8s-operator-libs_b200 -lust_host -lust
//       -Wl,-rpath,$PWD/k8s-operator-libs_b200 -o /tmp/host_eviction_bench
//   /tmp/host_eviction_bench 1000000 [reconciles per series]
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <random>
#include <unordered_map>

#include "tests/host/mocks.hpp"

using namespace upgrade;
using clk = std::chrono::steady_clock;

namespace {

// Provider calls change nothing: every reconcile of a series sees the objects the series made.
struct NoopProvider : mocks::NodeUpgradeStateProviderMock {
  Error ChangeNodeUpgradeState(Node*, const std::string&) override { return std::nullopt; }
  Error ChangeNodeUpgradeAnnotation(Node*, const std::string&, const std::string&) override { return std::nullopt; }
};
struct NoopCordon : CordonManager {
  Error Cordon(Node*) override { return std::nullopt; }
  Error Uncordon(Node*) override { return std::nullopt; }
};
struct NoopEvictor : PodEvictor {
  Error DeleteOrEvictPods(const Node&, const std::vector<Pod*>&, const EvictionOptions&) override { return std::nullopt; }
};
// The workload pods indexed by node: a per-node List costs a hash lookup.
struct IndexedClient : mocks::K8sClientMock {
  std::vector<Pod*> all;
  std::vector<DaemonSet*> workloadDs;
  std::unordered_map<std::string, std::vector<Pod*>> byNode;
  long long lists = 0;
  Error ListDaemonSets(const std::string& ns, const StringMap& l, std::vector<DaemonSet*>* out) override {
    if (!ns.empty()) return mocks::K8sClientMock::ListDaemonSets(ns, l, out);
    lists++;
    *out = workloadDs;
    return std::nullopt;
  }
  Error ListPodsBySelector(const std::string&, const std::string& node, std::vector<Pod*>* out) override {
    lists++;
    if (node.empty()) { *out = all; return std::nullopt; }
    auto it = byNode.find(node);
    if (it == byNode.end()) out->clear(); else *out = it->second;
    return std::nullopt;
  }
};
bool gpuPod(const Pod& p) { return p.Labels.count("nvidia.com/gpu") != 0; }
// kubectl's filter chain (filters.go) with IgnoreAllDaemonSets, for the reference's managers below: does it delete the pod
bool deletable(const Pod& p, bool force, bool emptyDir, bool* error) {
  const bool finished = p.Phase == "Succeeded" || p.Phase == "Failed";
  const OwnerReference* c = nullptr;
  for (const auto& o : p.OwnerReferences) if (o.Controller) { c = &o; break; }
  *error = false;
  if (c && c->Kind == "DaemonSet" && !finished) return false;  // every DaemonSet exists here
  if (p.Annotations.count("kubernetes.io/config.mirror")) return false;
  if (p.HasEmptyDirVolume && !finished && !emptyDir) { *error = true; return false; }
  if (!finished && !c && !force) { *error = true; return false; }
  return true;
}
// pod_manager.go:122-229 and drain_manager.go:58-139 over the client above, the goroutines run in place
struct RefPods : mocks::PodManagerMock {
  IndexedClient* client;
  NodeUpgradeStateProvider* provider;
  Error SchedulePodsRestart(const std::vector<Pod*>&) override { return std::nullopt; }
  Error SchedulePodEviction(const PodManagerConfig& c) override {
    for (Node* n : c.Nodes) {
      std::vector<Pod*> pods;
      if (client->ListPodsBySelector("", n->Name, &pods)) continue;
      Node node = *n;
      int toDelete = 0, can = 0;
      for (const Pod* p : pods) {
        if (!gpuPod(*p)) continue;
        toDelete++;
        bool err;
        can += deletable(*p, c.DeletionSpec->Force, c.DeletionSpec->DeleteEmptyDir, &err);
      }
      (void)provider->ChangeNodeUpgradeState(&node, toDelete == can ? UpgradeStatePodRestartRequired : UpgradeStateFailed);
    }
    return std::nullopt;
  }
};
struct RefDrain : DrainManager {
  IndexedClient* client;
  NodeUpgradeStateProvider* provider;
  Error ScheduleNodesDrain(const DrainConfiguration& c) override {
    for (Node* n : c.Nodes) {
      std::vector<Pod*> pods;
      if (client->ListPodsBySelector("", n->Name, &pods)) continue;
      Node node = *n;
      bool failed = false;
      for (const Pod* p : pods) { bool err; deletable(*p, c.Spec->Force, c.Spec->DeleteEmptyDir, &err); failed = failed || err; }
      (void)provider->ChangeNodeUpgradeState(&node, failed ? UpgradeStateFailed : UpgradeStatePodRestartRequired);
    }
    return std::nullopt;
  }
};

double median(std::vector<double> v) {
  std::sort(v.begin(), v.end());
  return v.empty() ? 0 : v[v.size() / 2];
}

}  // namespace

int main(int argc, char** argv) {
  const long n = argc > 1 ? atol(argv[1]) : 1000000;
  const int reps = argc > 2 ? atoi(argv[2]) : 5;
  SetDriverName("gpu");
  std::mt19937_64 rng(13);
  std::vector<std::unique_ptr<Node>> nodes;
  std::vector<std::unique_ptr<Pod>> pods, jobs;
  std::vector<DaemonSet> wds(8);
  for (int d = 0; d < 8; d++) { wds[d].Name = "workload-ds-" + std::to_string(d); wds[d].Namespace = "apps"; }
  std::vector<DaemonSet> dss(4);
  for (int d = 0; d < 4; d++) { dss[d].Name = "driver-ds-" + std::to_string(d); dss[d].UID = "uid-" + std::to_string(d); }
  ClusterUpgradeState st = NewClusterUpgradeState();
  const char* states[] = {"", UpgradeStateUpgradeRequired, UpgradeStateCordonRequired, UpgradeStateWaitForJobsRequired,
                          UpgradeStatePodDeletionRequired, UpgradeStateDrainRequired, UpgradeStatePodRestartRequired,
                          UpgradeStateValidationRequired, UpgradeStateUncordonRequired, UpgradeStateDone, UpgradeStateFailed};
  const int weight[] = {5, 35, 5, 5, 5, 5, 10, 2, 5, 20, 3};
  const char* phases[] = {"Running", "Running", "Pending", "Succeeded"};
  NoopProvider provider;
  IndexedClient client;
  int64_t version = 1;
  for (long i = 0; i < n; i++) {
    auto node = std::make_unique<Node>();
    node->Name = "node-" + std::to_string(i);
    node->ResourceVersion = std::to_string(version++);
    int r = (int)(rng() % 100), s = 0;
    while (r >= weight[s]) r -= weight[s++];
    if (*states[s]) node->Labels[GetUpgradeStateLabelKey()] = states[s];
    node->Unschedulable = rng() % 10 == 0;
    node->Conditions.push_back({"Ready", rng() % 50 == 0 ? "False" : "True"});
    if (rng() % 20 == 0) node->Annotations[GetUpgradeInitialStateAnnotationKey()] = "true";
    auto pod = std::make_unique<Pod>();
    pod->Name = "driver-" + std::to_string(i);
    pod->Namespace = "gpu-operator";
    pod->NodeName = node->Name;
    pod->ResourceVersion = std::to_string(version++);
    pod->Phase = rng() % 20 ? "Running" : "Pending";
    pod->Labels[PodControllerRevisionHashLabelKey] = rng() % 2 ? "test-hash-12345" : "old-hash-6789";
    pod->ContainerStatuses.push_back({rng() % 10 != 0, 0});
    const int d = (int)(rng() % 4);
    pod->OwnerReferences.push_back({"DaemonSet", dss[d].Name, dss[d].UID});
    if (s == 4 || s == 5) {  // pod-deletion-required / drain-required: 20-40 workload pods
      const int k = 20 + (int)(rng() % 21);
      for (int j = 0; j < k; j++) {
        auto jp = std::make_unique<Pod>();
        jp->Name = "work-" + std::to_string(i) + "-" + std::to_string(j);
        jp->Namespace = "apps";
        jp->NodeName = node->Name;
        jp->ResourceVersion = std::to_string(version++);
        if (rng() % 4 == 0) jp->Labels["nvidia.com/gpu"] = "1";
        const int kind = (int)(rng() % 8);
        if (kind < 5) jp->OwnerReferences.push_back({"ReplicaSet", "rs", "u", true});
        else if (kind == 5) jp->OwnerReferences.push_back({"DaemonSet", wds[rng() % 8].Name, "u", true});
        jp->HasEmptyDirVolume = rng() % 10 == 0;
        jp->Phase = phases[rng() % 4];
        client.byNode[node->Name].push_back(jp.get());
        client.all.push_back(jp.get());
        jobs.push_back(std::move(jp));
      }
    }
    auto ns = std::make_unique<NodeUpgradeState>();
    ns->Node = node.get(); ns->DriverPod = pod.get(); ns->DriverDaemonSet = &dss[d]; ns->ListIndex = i;
    st.NodeStates[states[s]].push_back(ns.get());
    st.owned.push_back(std::move(ns));
    provider.nodes[node->Name] = node.get();
    nodes.push_back(std::move(node)); pods.push_back(std::move(pod));
  }
  for (DaemonSet& d : wds) client.workloadDs.push_back(&d);
  const size_t nWork = st.NodeStates[UpgradeStatePodDeletionRequired].size() + st.NodeStates[UpgradeStateDrainRequired].size();
  std::printf("cluster: %ld nodes, %zu pod-deletion-required or drain-required, %zu workload pods\n", n, nWork, jobs.size());

  int64_t now = 1700000300;
  NoopCordon cordon; mocks::DrainManagerMock drain; mocks::ValidationManagerMock validation; mocks::SafeDriverLoadManagerImpl safe(&provider);
  RefPods podm;
  podm.client = &client; podm.provider = &provider;
  RefDrain rdrain;
  rdrain.client = &client; rdrain.provider = &provider;
  NoopEvictor evictor;
  std::unique_ptr<ClusterUpgradeStateManagerImpl> m[2];
  for (int on = 0; on < 2; on++) {
    StateOptions so;
    so.EvictionOnDevice = on == 1;
    so.Now = [&] { return now; };
    if (auto e = ClusterUpgradeStateManagerImpl::New(0, so, &m[on])) { std::printf("cannot create manager: %s\n", e->c_str()); return 1; }
    m[on]->NodeUpgradeStateProvider = &provider; m[on]->CordonManager = &cordon; m[on]->DrainManager = &rdrain; m[on]->PodManager = &podm;
    m[on]->ValidationManager = &validation; m[on]->SafeDriverLoadManager = &safe; m[on]->K8sClient = &client;
    m[on]->PodEvictor = &evictor;
    m[on]->WithPodDeletionEnabled(gpuPod);
  }
  DriverUpgradePolicySpec pol; pol.AutoUpgrade = true; pol.MaxParallelUpgrades = 100; pol.MaxUnavailable = IntOrString::FromString("25%");
  pol.PodDeletion = PodDeletionSpec{};
  pol.PodDeletion->Force = true;
  pol.DrainSpec = DrainSpec{};
  pol.DrainSpec->Enable = true;
  auto reconcile = [&](int on, double* seconds) -> bool {
    auto t0 = clk::now();
    Error e = m[on]->ApplyStateIncremental(&st, &pol);
    m[on]->WaitForActuators();
    *seconds = std::chrono::duration<double>(clk::now() - t0).count();
    if (e) std::printf("ApplyStateIncremental (%s): %s\n", on ? "on" : "off", e->c_str());
    return !e;
  };
  double s = 0;
  for (int on = 0; on < 2; on++) {
    if (!reconcile(on, &s)) return 1;
    std::printf("first reconcile (full upload), option %s: %.1f ms\n", on ? "on" : "off", s * 1e3);
  }
  auto bump = [&](std::string* rv) { *rv = std::to_string(version++); };
  const char* series[] = {"changed 1%", "time only", "moved 0.1%"};
  std::printf("(Lists: pod and DaemonSet Lists of the mocks; hand-offs: nodes given to the PodEvictor's workers)\n");
  for (int k = 0; k < 3; k++) {
    std::vector<double> t[2];
    long long lists[2] = {0, 0};
    ClusterUpgradeStateManagerImpl::IncrementalStats before = m[1]->Stats();
    for (int r = 0; r < reps; r++) {
      now += 37;
      if (k == 0) {  // 1 % of the objects: node objects, driver pods and workload pods alike
        const long objects = 2 * n + (long)jobs.size();
        for (long c = 0; c < objects / 100; c++) {  // workload pods change phase or gain an emptyDir
          const long o = (long)(rng() % (uint64_t)objects);
          if (o < n) bump(&nodes[(size_t)o]->ResourceVersion);
          else if (o < 2 * n) bump(&pods[(size_t)(o - n)]->ResourceVersion);
          else {
            Pod& jp = *jobs[(size_t)(o - 2 * n)];
            jp.Phase = phases[rng() % 4];
            jp.HasEmptyDirVolume = jp.HasEmptyDirVolume || rng() % 20 == 0;
            bump(&jp.ResourceVersion);
          }
        }
      } else if (k == 2) {  // 0.1 % of the nodes move: pairs of one bucket swap places in the list and in the bucket
        auto& bucket = st.NodeStates[UpgradeStateUpgradeRequired];
        for (long c = 0; c < n / 2000; c++) {
          const size_t a = rng() % bucket.size(), b = rng() % bucket.size();
          std::swap(bucket[a]->ListIndex, bucket[b]->ListIndex);
          std::swap(bucket[a], bucket[b]);
        }
      }
      for (int on = 0; on < 2; on++) {
        const long long l0 = client.lists;
        if (!reconcile(on, &s)) return 1;
        lists[on] += client.lists - l0;
        t[on].push_back(s);
      }
    }
    const ClusterUpgradeStateManagerImpl::IncrementalStats& a = m[1]->Stats();
    std::printf("%-11s off %8.1f ms  on %8.1f ms per reconcile (median of %d); Lists per reconcile off %.0f, on %.0f (%.0f per-node "
                "Lists avoided); on: %.1f lists sent, %.1f hand-offs, %.1f reorders per reconcile\n",
                series[k], median(t[0]) * 1e3, median(t[1]) * 1e3, reps, (double)lists[0] / reps, (double)lists[1] / reps,
                (double)(a.evict_lists_avoided - before.evict_lists_avoided) / reps, (double)(a.lists_sent - before.lists_sent) / reps,
                (double)(a.actuator_handoffs - before.actuator_handoffs) / reps, (double)(a.reorders - before.reorders) / reps);
  }
  return 0;
}
