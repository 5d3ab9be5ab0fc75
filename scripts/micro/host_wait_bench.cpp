// ApplyStateIncremental per reconcile with StateOptions::WaitForCompletionOnDevice off and on, through the H100 (one GPU).
// The cluster is C4-like: n nodes in the states of encode_bench.cpp, 5 % of them wait-for-jobs-required with 0-3 job pods
// each (Running, Pending or Succeeded), half of those nodes with a wait start time. The policy waits for "app=job" with a
// one-hour timeout. Off: the injected PodManager is a restatement of the reference's ScheduleCheckOnPodCompletion (one List
// per wait-for-jobs-required node per reconcile); on: one List per reconcile, the lists and start times resident. Three
// series after one untimed full reconcile each:
//   changed   1 % of the objects change between reconciles (node objects, driver pods, job pods)
//   time      only the clock moves (the on-mode manager sends no node and no list)
//   moved     0.1 % of the nodes move in BuildState's list (pairs swap places)
// The mocks make a List free and the provider calls no-ops, so this measures what the mirror and the library add per
// reconcile; it does not measure the API server's saving, only counts the Lists.
// Build (from the repository root, after build()) and run on a GPU machine:
//   g++ -O2 -std=c++17 -I. scripts/micro/host_wait_bench.cpp -Lk8s-operator-libs_b200 -lust_host -lust
//       -Wl,-rpath,$PWD/k8s-operator-libs_b200 -o /tmp/host_wait_bench
//   /tmp/host_wait_bench 1000000 [reconciles per series]
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
// The job pods indexed by node: a List costs a hash lookup (every pod matches the selector).
struct IndexedClient : mocks::K8sClientMock {
  std::vector<Pod*> all;
  std::unordered_map<std::string, std::vector<Pod*>> byNode;
  long long lists = 0;
  Error ListPodsBySelector(const std::string&, const std::string& node, std::vector<Pod*>* out) override {
    lists++;
    if (node.empty()) { *out = all; return std::nullopt; }
    auto it = byNode.find(node);
    if (it == byNode.end()) out->clear(); else *out = it->second;
    return std::nullopt;
  }
};
// pod_manager.go:256-368 over the client and the provider above
struct RefPods : mocks::PodManagerMock {
  IndexedClient* client;
  NodeUpgradeStateProvider* provider;
  std::function<int64_t()> now;
  Error SchedulePodsRestart(const std::vector<Pod*>&) override { return std::nullopt; }
  Error ScheduleCheckOnPodCompletion(const PodManagerConfig& c) override {
    const std::string key = GetWaitForPodCompletionStartTimeAnnotationKey();
    for (Node* n : c.Nodes) {
      std::vector<Pod*> pods;
      if (Error e = client->ListPodsBySelector(c.WaitForCompletionSpec->PodSelector, n->Name, &pods)) return e;
      Node node = *n;
      bool running = false;
      for (const Pod* p : pods) running = running || p->Phase == "Running" || p->Phase == "Pending";
      if (!running) {
        if (!provider->ChangeNodeUpgradeAnnotation(&node, key, "null")) (void)provider->ChangeNodeUpgradeState(&node, UpgradeStatePodDeletionRequired);
        continue;
      }
      if (c.WaitForCompletionSpec->TimeoutSecond == 0) continue;
      auto it = node.Annotations.find(key);
      if (it == node.Annotations.end()) { (void)provider->ChangeNodeUpgradeAnnotation(&node, key, std::to_string(now())); continue; }
      if (now() > std::atoll(it->second.c_str()) + c.WaitForCompletionSpec->TimeoutSecond) {
        (void)provider->ChangeNodeUpgradeState(&node, UpgradeStatePodDeletionRequired);
        (void)provider->ChangeNodeUpgradeAnnotation(&node, key, "null");
      }
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
  std::vector<DaemonSet> dss(4);
  for (int d = 0; d < 4; d++) { dss[d].Name = "driver-ds-" + std::to_string(d); dss[d].UID = "uid-" + std::to_string(d); }
  ClusterUpgradeState st = NewClusterUpgradeState();
  const char* states[] = {"", UpgradeStateUpgradeRequired, UpgradeStateCordonRequired, UpgradeStateWaitForJobsRequired,
                          UpgradeStatePodDeletionRequired, UpgradeStateDrainRequired, UpgradeStatePodRestartRequired,
                          UpgradeStateValidationRequired, UpgradeStateUncordonRequired, UpgradeStateDone, UpgradeStateFailed};
  const int weight[] = {5, 35, 5, 5, 5, 5, 10, 2, 5, 20, 3};
  const char* phases[] = {"Running", "Pending", "Succeeded"};
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
    if (s == 3) {  // wait-for-jobs-required: 0-3 job pods, half of the nodes with a start time
      if (rng() % 2) node->Annotations[GetWaitForPodCompletionStartTimeAnnotationKey()] = "1700000000";
      const int k = (int)(rng() % 4);
      for (int j = 0; j < k; j++) {
        auto jp = std::make_unique<Pod>();
        jp->Name = "job-" + std::to_string(i) + "-" + std::to_string(j);
        jp->Namespace = "jobs";
        jp->NodeName = node->Name;
        jp->ResourceVersion = std::to_string(version++);
        jp->Labels["app"] = "job";
        jp->Phase = phases[rng() % 3];
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
  const size_t nWait = st.NodeStates[UpgradeStateWaitForJobsRequired].size();
  std::printf("cluster: %ld nodes, %zu wait-for-jobs-required, %zu job pods\n", n, nWait, jobs.size());

  int64_t now = 1700000300;
  NoopCordon cordon; mocks::DrainManagerMock drain; mocks::ValidationManagerMock validation; mocks::SafeDriverLoadManagerImpl safe(&provider);
  RefPods podm;
  podm.client = &client; podm.provider = &provider; podm.now = [&] { return now; };
  std::unique_ptr<ClusterUpgradeStateManagerImpl> m[2];
  for (int on = 0; on < 2; on++) {
    StateOptions so;
    so.WaitForCompletionOnDevice = on == 1;
    so.Now = [&] { return now; };
    if (auto e = ClusterUpgradeStateManagerImpl::New(0, so, &m[on])) { std::printf("cannot create manager: %s\n", e->c_str()); return 1; }
    m[on]->NodeUpgradeStateProvider = &provider; m[on]->CordonManager = &cordon; m[on]->DrainManager = &drain; m[on]->PodManager = &podm;
    m[on]->ValidationManager = &validation; m[on]->SafeDriverLoadManager = &safe; m[on]->K8sClient = &client;
  }
  DriverUpgradePolicySpec pol; pol.AutoUpgrade = true; pol.MaxParallelUpgrades = 100; pol.MaxUnavailable = IntOrString::FromString("25%");
  pol.WaitForCompletion = WaitForCompletionSpec{"app=job", 3600};
  auto reconcile = [&](int on, double* seconds) -> bool {
    auto t0 = clk::now();
    Error e = m[on]->ApplyStateIncremental(&st, &pol);
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
  for (int k = 0; k < 3; k++) {
    std::vector<double> t[2];
    long long lists[2] = {0, 0};
    ClusterUpgradeStateManagerImpl::IncrementalStats before = m[1]->Stats();
    for (int r = 0; r < reps; r++) {
      now += 37;
      if (k == 0) {  // 1 % of the objects: node objects, driver pods and job pods alike
        const long objects = 2 * n + (long)jobs.size();
        for (long c = 0; c < objects / 100; c++) {
          const long o = (long)(rng() % (uint64_t)objects);
          if (o < n) bump(&nodes[(size_t)o]->ResourceVersion);
          else if (o < 2 * n) bump(&pods[(size_t)(o - n)]->ResourceVersion);
          else {
            Pod& jp = *jobs[(size_t)(o - 2 * n)];
            jp.Phase = phases[rng() % 3];
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
    std::printf("%-11s off %8.1f ms  on %8.1f ms per reconcile (median of %d); Lists per reconcile off %.0f, on %.0f (%.0f avoided); "
                "on: %.1f lists sent, %.1f time-only, %.1f reorders per reconcile\n",
                series[k], median(t[0]) * 1e3, median(t[1]) * 1e3, reps, (double)lists[0] / reps, (double)lists[1] / reps,
                (double)(a.wait_avoided - before.wait_avoided) / reps, (double)(a.lists_sent - before.lists_sent) / reps,
                (double)(a.time_only - before.time_only) / reps, (double)(a.reorders - before.reorders) / reps);
  }
  return 0;
}
