// Nodes that move in BuildState's list under ApplyStateIncremental (reorder_spec.hpp).
//   reorder_test         host halves only: the oracle stands in for the kernel, and the cache's evaluation checks the
//                        splice or the reorder runs it would hand to the device and replays them on its own copy of the
//                        previous reconcile's arrays
//   reorder_test --gpu   through the C ABI and the H100 kernels (ust_apply_state_delta_reorder / _splice)
#include <cstring>

#include "reorder_spec.hpp"

extern "C" int ust_oracle_apply_state(int variant, const ust_policy* policy, int64_t n, const uint8_t* state,
                                      const uint32_t* flags, const int32_t* pod_rev, const int32_t* ds_idx, int32_t n_ds,
                                      const int32_t* ds_rev, const ust_pods* pods, uint8_t* next_state, uint16_t* actions,
                                      uint8_t* actuator_outcome, ust_counters* out);

namespace {

// The incremental path with the oracle behind the cache. Besides evaluating, it checks what the device would be given:
// the previous reconcile's arrays, brought into the new order by Cache::pending and patched at `changed`, must be the
// cache's arrays, and the previous outputs must have moved with their nodes.
struct ReorderCheckingOracle : upgrade::ClusterUpgradeStateManagerImpl {
  std::vector<uint8_t> state, next;
  std::vector<uint32_t> flags;
  std::vector<int32_t> pod_rev, ds_idx;
  std::vector<uint16_t> actions;
  std::string problem;
  static inline int64_t reorders = 0, splices = 0;  // checked, over all instances

  // `a` in the new node order; inserted node j takes (*ins)[insert_at[j]] (its column in the cache), or `fill` without `ins`
  template <class T>
  static std::vector<T> apply(const std::vector<T>& a, const Cache::Splice& sp, const std::vector<T>* ins, T fill = T()) {
    std::vector<T> out;
    size_t j = 0;
    if (!sp.run_src.empty()) {  // ust_reorder: the runs concatenated
      for (size_t r = 0; r < sp.run_src.size(); r++)
        for (int64_t e = 0; e < sp.run_len[r]; e++)
          out.push_back(sp.run_src[r] >= 0 ? a[(size_t)(sp.run_src[r] + e)] : ins ? (*ins)[(size_t)sp.insert_at[j++]] : fill);
      return out;
    }
    size_t r = 0;  // ust_splice
    for (size_t p = 0; p <= a.size(); p++) {
      for (; j < sp.insert_before.size() && sp.insert_before[j] == (int64_t)p; j++)
        out.push_back(ins ? (*ins)[(size_t)sp.insert_at[j]] : fill);
      if (p == a.size()) break;
      if (r < sp.remove_idx.size() && sp.remove_idx[r] == (int64_t)p) { r++; continue; }
      out.push_back(a[p]);
    }
    return out;
  }

  // the contract of ust_reorder (include/ust.h), and maximal runs
  std::string checkRuns(const Cache::Splice& sp, size_t n_old) {
    if (sp.run_len.size() != sp.run_src.size()) return "run_src / run_len sizes differ";
    if (!sp.insert_before.empty()) return "insert_before set together with runs";
    std::vector<char> named(n_old, 0);
    int64_t ins = 0;
    for (size_t r = 0; r < sp.run_src.size(); r++) {
      const int64_t s = sp.run_src[r], l = sp.run_len[r];
      if (l < 1 || s < -1) return "run length below 1 or source below -1";
      if (r > 0 && ((s < 0 && sp.run_src[r - 1] < 0) || (s >= 0 && sp.run_src[r - 1] >= 0 && sp.run_src[r - 1] + sp.run_len[r - 1] == s)))
        return "runs are not maximal";
      if (s < 0) { ins += l; continue; }
      if (s + l > (int64_t)n_old) return "an old run leaves the previous snapshot";
      for (int64_t e = s; e < s + l; e++) {
        if (named[(size_t)e]) return "two runs name one old node";
        named[(size_t)e] = 1;
      }
    }
    if (ins != (int64_t)sp.insert_at.size()) return "the inserted runs do not take every inserted node";
    for (int64_t x : sp.remove_idx)
      if (x < 0 || (size_t)x >= n_old || named[(size_t)x]) return "remove_idx names a node that stays";
    size_t stay = 0;
    for (char c : named) stay += c;
    if (stay + sp.remove_idx.size() != n_old) return "an old node neither stays nor is removed";
    return "";
  }

  int EvaluateCached(const ust_policy& policy, bool full, const std::vector<int64_t>& changed, Cache* cache, ust_counters* c) override {
    Cache& k = *cache;
    const size_t n = k.slots.size();
    auto note = [&](const std::string& s) { if (problem.empty() && !s.empty()) problem = s; };
    if (!full) {
      const Cache::Splice& sp = k.pending;
      if (!sp.run_src.empty()) {
        note(checkRuns(sp, state.size()));
        reorders++;
      } else {
        for (size_t q = 1; q < sp.remove_idx.size(); q++) if (sp.remove_idx[q] <= sp.remove_idx[q - 1]) note("remove_idx not strictly increasing");
        for (size_t q = 1; q < sp.insert_before.size(); q++) if (sp.insert_before[q] < sp.insert_before[q - 1]) note("insert_before decreasing");
        for (int64_t x : sp.insert_before) if (x < 0 || x > (int64_t)state.size()) note("insert_before out of range");
        if (sp.insert_at.size() != sp.insert_before.size()) note("insert_at / insert_before sizes differ");
        splices += sp.empty() ? 0 : 1;
      }
      if (!problem.empty()) return UST_ERR_INVALID_ARGUMENT;
      std::vector<uint8_t> st = apply(state, sp, &k.state);
      std::vector<uint32_t> fl = apply(flags, sp, &k.flags);
      std::vector<int32_t> rv = apply(pod_rev, sp, &k.pod_rev), di = apply(ds_idx, sp, &k.ds_idx);
      std::vector<uint8_t> pn = apply(next, sp, (const std::vector<uint8_t>*)nullptr, (uint8_t)0xFF);
      std::vector<uint16_t> pa = apply(actions, sp, (const std::vector<uint16_t>*)nullptr);
      for (int64_t i : changed) {
        if (i < 0 || (size_t)i >= st.size()) { note("changed index outside the new snapshot"); return UST_ERR_INVALID_ARGUMENT; }
        st[(size_t)i] = k.state[(size_t)i]; fl[(size_t)i] = k.flags[(size_t)i]; rv[(size_t)i] = k.pod_rev[(size_t)i]; di[(size_t)i] = k.ds_idx[(size_t)i];
      }
      if (st != k.state || fl != k.flags || rv != k.pod_rev || di != k.ds_idx) note("the replayed reorder + overwrites differ from the cache's arrays");
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
  ReorderCheckingOracle* oracle = nullptr;
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
      oracle = new ReorderCheckingOracle();
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
  spec::run_reorder(R, makeFull, wfull, makeIncr, wincr, backendCheck, gpu ? 3000 : 600);
  if (!gpu) {
    R.it("the oracle-backed evaluation saw the reorders and splices it checked", [&] {
      EXPECT(R, ReorderCheckingOracle::reorders >= 20 && ReorderCheckingOracle::splices >= 2);
    });
  }
  std::printf("# %d passed, %d failed\n", R.passed, R.failed);
  return (R.failed == 0 && device_ok) ? 0 : 1;
}
