// Membership changes under ApplyStateIncremental (membership_spec.hpp).
//   membership_test         host halves only: the oracle stands in for the kernel, and the cache's evaluation replays the
//                           splice it would hand to the device on its own copy of the previous reconcile's arrays
//   membership_test --gpu   through the C ABI and the H100 kernels (ust_apply_state_delta_splice)
#include <cstring>

#include "membership_spec.hpp"

extern "C" int ust_oracle_apply_state(int variant, const ust_policy* policy, int64_t n, const uint8_t* state,
                                      const uint32_t* flags, const int32_t* pod_rev, const int32_t* ds_idx, int32_t n_ds,
                                      const int32_t* ds_rev, const ust_pods* pods, uint8_t* next_state, uint16_t* actions,
                                      uint8_t* actuator_outcome, ust_counters* out);

namespace {

// The incremental path with the oracle behind the cache. Besides evaluating, it checks what the device would be given:
// the previous reconcile's arrays, spliced by Cache::pending and patched at `changed`, must be the cache's arrays.
struct SpliceCheckingOracle : upgrade::ClusterUpgradeStateManagerImpl {
  std::vector<uint8_t> state, next;
  std::vector<uint32_t> flags;
  std::vector<int32_t> pod_rev, ds_idx;
  std::vector<uint16_t> actions;
  std::string problem;
  static inline int64_t splices = 0;  // non-empty splices checked, over all instances (they end with their world)

  // `a` in the new node order; inserted node j takes (*ins)[insert_at[j]] (its column in the cache), or `fill` without `ins`
  template <class T>
  static std::vector<T> splice(const std::vector<T>& a, const Cache::Splice& sp, const std::vector<T>* ins, T fill = T()) {
    std::vector<T> out;
    size_t r = 0, j = 0;
    for (size_t p = 0; p <= a.size(); p++) {
      for (; j < sp.insert_before.size() && sp.insert_before[j] == (int64_t)p; j++)
        out.push_back(ins ? (*ins)[(size_t)sp.insert_at[j]] : fill);
      if (p == a.size()) break;
      if (r < sp.remove_idx.size() && sp.remove_idx[r] == (int64_t)p) { r++; continue; }
      out.push_back(a[p]);
    }
    return out;
  }

  int EvaluateCached(const ust_policy& policy, bool full, const std::vector<int64_t>& changed, Cache* cache, ust_counters* c) override {
    Cache& k = *cache;
    const size_t n = k.slots.size();
    auto note = [&](const std::string& s) { if (problem.empty()) problem = s; };
    if (!full) {
      const Cache::Splice& sp = k.pending;
      for (size_t q = 1; q < sp.remove_idx.size(); q++) if (sp.remove_idx[q] <= sp.remove_idx[q - 1]) note("remove_idx not strictly increasing");
      for (size_t q = 1; q < sp.insert_before.size(); q++) if (sp.insert_before[q] < sp.insert_before[q - 1]) note("insert_before decreasing");
      for (int64_t x : sp.remove_idx) if (x < 0 || x >= (int64_t)state.size()) note("remove_idx out of range");
      for (int64_t x : sp.insert_before) if (x < 0 || x > (int64_t)state.size()) note("insert_before out of range");
      if (sp.insert_at.size() != sp.insert_before.size()) note("insert_at / insert_before sizes differ");
      if (!problem.empty()) return UST_ERR_INVALID_ARGUMENT;
      splices += sp.empty() ? 0 : 1;
      std::vector<uint8_t> st = splice(state, sp, &k.state);
      std::vector<uint32_t> fl = splice(flags, sp, &k.flags);
      std::vector<int32_t> rv = splice(pod_rev, sp, &k.pod_rev), di = splice(ds_idx, sp, &k.ds_idx);
      std::vector<uint8_t> pn = splice(next, sp, (const std::vector<uint8_t>*)nullptr, (uint8_t)0xFF);
      std::vector<uint16_t> pa = splice(actions, sp, (const std::vector<uint16_t>*)nullptr);
      for (int64_t i : changed) {
        if (i < 0 || (size_t)i >= st.size()) { note("changed index outside the new snapshot"); return UST_ERR_INVALID_ARGUMENT; }
        st[(size_t)i] = k.state[(size_t)i]; fl[(size_t)i] = k.flags[(size_t)i]; rv[(size_t)i] = k.pod_rev[(size_t)i]; di[(size_t)i] = k.ds_idx[(size_t)i];
      }
      if (st != k.state || fl != k.flags || rv != k.pod_rev || di != k.ds_idx) note("the replayed splice + overwrites differ from the cache's arrays");
      // the previous outputs moved with their nodes (joined nodes: whatever the host holds, the device reports them)
      for (size_t i = 0; i < n && i < pn.size(); i++)
        if (pn[i] != 0xFF && (pn[i] != k.next[i] || pa[i] != k.actions[i])) { note("previous outputs did not move with their nodes"); break; }
    }
    k.next.assign(n + 1, 0);
    k.actions.assign(n + 1, 0);
    std::vector<uint8_t> st = k.state; st.push_back(0);
    std::vector<uint32_t> fl = k.flags; fl.push_back(0);
    std::vector<int32_t> rv = k.pod_rev, di = k.ds_idx, dr = k.ds_rev;
    rv.push_back(0); di.push_back(0); dr.push_back(0);
    const int rc = ust_oracle_apply_state(0, &policy, (int64_t)n, st.data(), fl.data(), rv.data(), di.data(), (int32_t)k.ds_rev.size(),
                                          dr.data(), nullptr, k.next.data(), k.actions.data(), nullptr, c);
    k.next.resize(n);
    k.actions.resize(n);
    state = k.state; flags = k.flags; pod_rev = k.pod_rev; ds_idx = k.ds_idx; next = k.next; actions = k.actions;
    return rc;
  }
};

}  // namespace

int main(int argc, char** argv) {
  const bool gpu = argc > 1 && std::strcmp(argv[1], "--gpu") == 0;
  mocks::Runner R;
  spec::MakeFn makeFull, makeIncr;
  spec::WorldApplyFn wfull, wincr = [](spec::World& w, const upgrade::DriverUpgradePolicySpec* p) { return w.m->ApplyStateIncremental(&w.state, p); };
  std::function<std::string()> backendCheck = [] { return std::string(); };
  SpliceCheckingOracle* oracle = nullptr;
  bool device_ok = true;
  if (gpu) {
    makeFull = [&](upgrade::StateOptions o) {
      std::unique_ptr<upgrade::ClusterUpgradeStateManagerImpl> m;
      if (auto e = upgrade::ClusterUpgradeStateManagerImpl::New(0, o, &m)) {
        std::printf("cannot create manager: %s\n", e->c_str());
        device_ok = false;
        return upgrade::ClusterUpgradeStateManagerImpl::NewDetached(o);
      }
      return m;
    };
    makeIncr = makeFull;
    wfull = [](spec::World& w, const upgrade::DriverUpgradePolicySpec* p) { return w.m->ApplyState(&w.state, p); };
  } else {
    makeFull = [](upgrade::StateOptions o) { return upgrade::ClusterUpgradeStateManagerImpl::NewDetached(o); };
    makeIncr = [&](upgrade::StateOptions) {
      oracle = new SpliceCheckingOracle();
      return std::unique_ptr<upgrade::ClusterUpgradeStateManagerImpl>(oracle);
    };
    wfull = [](spec::World& w, const upgrade::DriverUpgradePolicySpec* p) -> upgrade::Error {
      upgrade::EncodedSnapshot enc;
      if (auto err = w.m->Encode(w.state, *p, &enc)) return err;
      const size_t n = enc.entries.size();
      std::vector<uint8_t> next(n + 1);
      std::vector<uint16_t> actions(n + 1);
      enc.state.push_back(0); enc.flags.push_back(0); enc.pod_rev.push_back(0); enc.ds_idx.push_back(0); enc.ds_rev.push_back(0);
      ust_counters c;
      const int rc = ust_oracle_apply_state(0, &enc.policy, (int64_t)n, enc.state.data(), enc.flags.data(), enc.pod_rev.data(),
                                            enc.ds_idx.data(), (int32_t)enc.ds_rev.size() - 1, enc.ds_rev.data(), nullptr,
                                            next.data(), actions.data(), nullptr, &c);
      return w.m->Replay(enc, *p, next.data(), actions.data(), rc, c);
    };
    backendCheck = [&] { return oracle ? oracle->problem : std::string("no oracle-backed manager"); };
  }
  spec::run_membership(R, makeFull, wfull, makeIncr, wincr, backendCheck, gpu ? 3000 : 600);
  if (!gpu) {
    R.it("the oracle-backed evaluation saw the splices it checked", [&] { EXPECT(R, SpliceCheckingOracle::splices >= 10); });
  }
  std::printf("# %d passed, %d failed\n", R.passed, R.failed);
  return (R.failed == 0 && device_ok) ? 0 : 1;
}
