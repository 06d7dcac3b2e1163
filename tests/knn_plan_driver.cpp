// Prints, for tests/test_item_knn_cpu.py, the path-9 plan (rectools_b200/csrc/knn_plan.h: plan_knn) of the calls read
// from stdin, one per line of `name=value` words with comma-separated lists: `n_items`, `s_indptr`, `s_indices`,
// `s_data` (default 1 per entry), `u_indptr`, `u_indices`, `u_data` (default 1 per entry), `f_indptr` / `f_indices`
// (absent: no filter), `wl` (absent: no whitelist; `wl=-` an empty one), `k`, `budget` (0: the library's 1 GiB),
// `max_rows`, `no_out` (1: NULL outputs), `nan_s` / `nan_u` (1: the first S value / weight is NaN).  Output: one line per
// call, `error= bounds= bound= slot= dense=` and the message (which has spaces) last.
#include <cmath>
#include <iostream>
#include <map>
#include <sstream>
#include <string>
#include <vector>

#include "../rectools_b200/csrc/knn_plan.h"

template <class T>
static std::vector<T> numbers(const std::string& s) {
    std::vector<T> out;
    std::stringstream ss(s);
    for (std::string w; std::getline(ss, w, ',');)
        if (!w.empty()) out.push_back((T)std::stod(w));
    return out;
}

template <class T>
static std::string join(const std::vector<T>& v) {
    std::string s;
    for (size_t i = 0; i < v.size(); ++i) s += (i ? "," : "") + std::to_string(v[i]);
    return s;
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
        auto num = [&](const char* name) { return v.count(name) ? std::stoll(v[name]) : 0ll; };
        auto s_indptr = numbers<int64_t>(v["s_indptr"]), u_indptr = numbers<int64_t>(v["u_indptr"]);
        auto s_indices = numbers<int32_t>(v["s_indices"]), u_indices = numbers<int32_t>(v["u_indices"]);
        auto s_data = v.count("s_data") ? numbers<double>(v["s_data"]) : std::vector<double>(s_indices.size(), 1.0);
        auto u_data = v.count("u_data") ? numbers<float>(v["u_data"]) : std::vector<float>(u_indices.size(), 1.0f);
        if (num("nan_s") && !s_data.empty()) s_data[0] = NAN;
        if (num("nan_u") && !u_data.empty()) u_data[0] = NAN;
        auto f_indptr = numbers<int64_t>(v["f_indptr"]);
        auto f_indices = numbers<int32_t>(v["f_indices"]);
        const bool has_wl = v.count("wl") > 0;
        auto wl = numbers<int32_t>(v["wl"] == "-" ? "" : v["wl"]);
        b200::KnnArgs a;
        a.n_items = num("n_items");
        a.s_indptr = s_indptr.empty() ? nullptr : s_indptr.data();
        a.s_indices = s_indices.empty() ? nullptr : s_indices.data();
        a.s_data = s_data.empty() ? nullptr : s_data.data();
        a.n_rows = u_indptr.empty() ? 0 : (int64_t)u_indptr.size() - 1;
        a.u_indptr = u_indptr.empty() ? nullptr : u_indptr.data();
        a.u_indices = u_indices.empty() ? nullptr : u_indices.data();
        a.u_data = u_data.empty() ? nullptr : u_data.data();
        a.f_indptr = f_indptr.empty() ? nullptr : f_indptr.data();
        a.f_indices = f_indices.empty() ? nullptr : f_indices.data();
        a.whitelist = wl.empty() ? nullptr : wl.data();
        a.n_whitelist = has_wl ? (int64_t)wl.size() : -1;
        a.k = num("k");
        a.outputs = !num("no_out");
        const int64_t budget = num("budget");
        const b200::KnnPlan p = budget > 0 ? b200::plan_knn(a, num("max_rows"), budget) : b200::plan_knn(a, num("max_rows"));
        std::cout << "error=" << p.error << " bounds=" << join(p.bounds) << " bound=" << join(p.bound) << " slot=" << join(p.slot)
                  << " dense=" << p.max_chunk_dense << " message=" << p.message << "\n";
    }
    return 0;
}
