// StateOptions::ValidateOnDevice against the reference's ValidationManagerImpl (validation_manager.go:71-175), restated
// here over the same mocks: one List per node through the client, a delete of the start-time annotation per ready pod,
// handleTimeout with the same clock. The device-mode manager must make the same provider / actuator calls, in the same
// order, and return the same error - except that Validate's per-pod deletes of one annotation come as one
// (include/ust.h, UST_A_CLEAR_WAIT_START), so runs of identical deletes are collapsed before comparing.
#pragma once
#include <cstdio>

#include "build_state_spec.hpp"

namespace vspec {
using namespace upgrade;
using namespace mocks;

// K8sClientMock plus the ValidationManager's List: `k=v[,k=v]` label selectors, an optional node name, API order.
struct SelectorClient : K8sClientMock {
  K8sClientMock* base = nullptr;  // DaemonSets and driver pods come from here when set
  std::vector<Pod*> all;          // every pod the List can see, in API order
  Error listError;                // what the List returns instead, when set
  int lists = 0;
  Error ListDaemonSets(const std::string& ns, const StringMap& l, std::vector<DaemonSet*>* out) override {
    return base ? base->ListDaemonSets(ns, l, out) : K8sClientMock::ListDaemonSets(ns, l, out);
  }
  Error ListPods(const std::string& ns, const StringMap& l, std::vector<Pod*>* out) override {
    return base ? base->ListPods(ns, l, out) : K8sClientMock::ListPods(ns, l, out);
  }
  static bool matches(const std::string& selector, const Pod& p) {
    size_t i = 0;
    while (i <= selector.size()) {
      size_t j = selector.find(',', i);
      if (j == std::string::npos) j = selector.size();
      const std::string term = selector.substr(i, j - i);
      const size_t eq = term.find('=');
      auto it = p.Labels.find(term.substr(0, eq));
      if (eq == std::string::npos || it == p.Labels.end() || it->second != term.substr(eq + 1)) return false;
      i = j + 1;
    }
    return true;
  }
  Error ListPodsBySelector(const std::string& selector, const std::string& nodeName, std::vector<Pod*>* out) override {
    lists++;
    if (listError) return listError;
    out->clear();
    for (Pod* p : all)
      if ((nodeName.empty() || p->NodeName == nodeName) && matches(selector, *p)) out->push_back(p);
    return std::nullopt;
  }
};

// validation_manager.go:71-175
struct ValidationManagerImpl : ValidationManager {
  SelectorClient* client = nullptr;
  NodeUpgradeStateProvider* provider = nullptr;
  std::string podSelector;
  std::function<int64_t()> now;
  int calls = 0;
  static bool isPodReady(const Pod& p) {
    if (p.Phase != "Running" || p.ContainerStatuses.empty()) return false;
    for (const auto& cs : p.ContainerStatuses)
      if (!cs.Ready) return false;
    return true;
  }
  // strconv.ParseInt(s, 10, 64) as Go writes it (strconv/atoi.go): ParseUint's loop returns "value out of range" at the
  // first overflow, before it sees a later bad character; the quoting here covers printable ASCII only.
  static Error parseInt(const std::string& s0, int64_t* out) {
    auto syntax = [&] { return Errorf("strconv.ParseInt: parsing \"" + s0 + "\": invalid syntax"); };
    auto range = [&] { return Errorf("strconv.ParseInt: parsing \"" + s0 + "\": value out of range"); };
    if (s0.empty()) return syntax();
    std::string s = s0;
    bool neg = false;
    if (s[0] == '+') s = s.substr(1);
    else if (s[0] == '-') { neg = true; s = s.substr(1); }
    if (s.empty()) return syntax();
    const uint64_t cutoff = UINT64_MAX / 10 + 1;
    uint64_t n = 0;
    for (char c : s) {
      if (c < '0' || c > '9') return syntax();
      if (n >= cutoff) return range();
      n *= 10;
      const uint64_t n1 = n + (uint64_t)(c - '0');
      if (n1 < n) return range();
      n = n1;
    }
    const uint64_t cut = (uint64_t)1 << 63;
    if (!neg && n >= cut) return range();
    if (neg && n > cut) return range();
    *out = neg ? (int64_t)(0 - n) : (int64_t)n;
    return std::nullopt;
  }
  Error handleTimeout(Node* node, int64_t timeoutSeconds) {
    const std::string key = GetValidationStartTimeAnnotationKey();
    const int64_t currentTime = now();
    auto it = node->Annotations.find(key);
    if (it == node->Annotations.end()) return provider->ChangeNodeUpgradeAnnotation(node, key, std::to_string(currentTime));
    const std::string v = it->second;
    int64_t startTime = 0;
    if (Error e = parseInt(v, &startTime)) return e;
    if (currentTime > startTime + timeoutSeconds) {
      (void)provider->ChangeNodeUpgradeState(node, UpgradeStateFailed);
      return provider->ChangeNodeUpgradeAnnotation(node, key, "null");
    }
    return std::nullopt;
  }
  Error Validate(Node* node, bool* done) override {
    calls++;
    *done = false;
    if (podSelector.empty()) { *done = true; return std::nullopt; }
    std::vector<Pod*> pods;
    if (Error e = client->ListPodsBySelector(podSelector, node->Name, &pods)) return e;
    if (pods.empty()) return std::nullopt;
    bool ok = true;
    for (Pod* p : pods) {
      if (!isPodReady(*p)) {
        if (Error e = handleTimeout(node, 600)) return Errorf("unable to handle timeout for validation state: " + *e);
        ok = false;
        break;
      }
      if (Error e = provider->ChangeNodeUpgradeAnnotation(node, GetValidationStartTimeAnnotationKey(), "null")) { *done = ok; return e; }
    }
    *done = ok;
    return std::nullopt;
  }
};
struct CountingValidation : ValidationManager {
  int calls = 0;
  Error Validate(Node*, bool* done) override { calls++; *done = true; return std::nullopt; }
};

// The logging provider of build_state_spec.hpp that can be told to fail the n-th write whose text contains `match`.
struct FailingProvider : spec::LogProvider {
  std::string match;
  int failAt = -1, seen = 0;
  Error fail(const std::string& what) {
    if (match.empty() || what.find(match) == std::string::npos) return std::nullopt;
    if (seen++ != failAt) return std::nullopt;
    log->push_back("FAILED " + what);
    return Errorf("provider error on " + what);
  }
  Error ChangeNodeUpgradeState(Node* n, const std::string& s) override {
    if (Error e = fail("state " + n->Name + "=" + s)) return e;
    return spec::LogProvider::ChangeNodeUpgradeState(n, s);
  }
  Error ChangeNodeUpgradeAnnotation(Node* n, const std::string& k, const std::string& v) override {
    if (Error e = fail("annotation " + n->Name + " " + k + "=" + v)) return e;
    return spec::LogProvider::ChangeNodeUpgradeAnnotation(n, k, v);
  }
};

// Validate's deletes of the start-time annotation come once per ready pod in the reference and once per node from the
// device: collapse runs of the same delete.
inline std::vector<std::string> collapse(const std::vector<std::string>& log) {
  std::vector<std::string> out;
  const std::string suffix = " " + GetValidationStartTimeAnnotationKey() + "=null";
  for (const std::string& s : log) {
    const bool del = s.size() > suffix.size() && s.compare(s.size() - suffix.size(), suffix.size(), suffix) == 0 && s.rfind("annotation ", 0) == 0;
    if (del && !out.empty() && out.back() == s) continue;
    out.push_back(s);
  }
  return out;
}

inline Pod makeValidationPod(const std::string& name, const std::string& node, bool running, std::vector<bool> ready, int64_t rv) {
  Pod p;
  p.Name = name;
  p.Namespace = "gpu-operator";
  p.NodeName = node;
  p.ResourceVersion = std::to_string(rv);
  p.Labels["app"] = "validator";
  p.Labels["tier"] = "gpu";
  p.Phase = running ? "Running" : "Pending";
  for (bool r : ready) p.ContainerStatuses.push_back({r, 0});
  return p;
}

}  // namespace vspec
