// Prints, for tests/test_metrics_cpu.py, the path-10 plan (rectools_b200/csrc/metrics_plan.h: plan_metrics) of the calls
// read from stdin, one per line of `name=value` words with comma-separated lists: `n_inter`, `n_reco`, `ks` (absent: no
// k; `n_k` overrides the count), `ndcg_offsets` (absent: no table; `n_ndcg` overrides the count), `map` (1: out_map given),
// and `no_inter` / `no_reco` / `no_terms` / `no_out` / `no_tp` / `no_ndcg` / `no_ks` / `no_offsets` (1: that pointer is
// NULL).  Output: one line per call, `error= slots= k_max= n_terms= bytes=` and the message (which has spaces) last.
#include <iostream>
#include <map>
#include <sstream>
#include <string>
#include <vector>

#include "../rectools_b200/csrc/metrics_plan.h"

static std::vector<int64_t> numbers(const std::string& s) {
    std::vector<int64_t> out;
    std::stringstream ss(s);
    for (std::string w; std::getline(ss, w, ',');)
        if (!w.empty()) out.push_back(std::stoll(w));
    return out;
}

int main() {
    std::string line;
    while (std::getline(std::cin, line)) {
        std::map<std::string, std::string> v;
        std::istringstream words(line);
        for (std::string w; words >> w;) {
            const size_t eq = w.find('=');
            v[w.substr(0, eq)] = w.substr(eq + 1);
        }
        auto num = [&](const char* key, int64_t def) { return v.count(key) ? std::stoll(v[key]) : def; };
        auto flag = [&](const char* key) { return num(key, 0) != 0; };
        const std::vector<int64_t> ks = numbers(v["ks"]), offsets = numbers(v["ndcg_offsets"]);
        b200::MetricsArgs a;
        a.n_inter = num("n_inter", 0);
        a.inter = !flag("no_inter");
        a.n_reco = num("n_reco", 0);
        a.reco = !flag("no_reco");
        a.n_k = (int32_t)num("n_k", (int64_t)ks.size());
        a.ks = flag("no_ks") ? nullptr : ks.data();
        a.n_ndcg = (int32_t)num("n_ndcg", offsets.empty() ? 0 : (int64_t)offsets.size() - 1);
        a.ndcg_offsets = flag("no_offsets") ? nullptr : offsets.data();
        a.ndcg_terms = !flag("no_terms");
        a.outputs = !flag("no_out");
        a.out_tp = !flag("no_tp");
        a.out_ndcg = !flag("no_ndcg");
        const b200::MetricsPlan p = b200::plan_metrics(a, flag("map"));
        std::cout << "error=" << p.error << " slots=" << p.slots << " k_max=" << p.k_max << " n_terms=" << p.n_terms
                  << " bytes=" << p.device_bytes << " message=" << p.message << "\n";
    }
    return 0;
}
