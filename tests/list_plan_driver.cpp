// Prints, for tests/test_popular_cpu.py, the path-7 plan (rectools_b200/csrc/list_plan.h: plan_list) of the calls read
// from stdin, one per line of `name=value` words: `n_list` (the list is 0, 1, 2, ... unless `list` gives it,
// comma-separated), `k`, `lens` (comma-separated viewed counts per row; the rows' ids are 0, 1, 2, ... unless `ids` lists
// them, comma-separated; `lens=-` passes a NULL csr_indptr), `base` (added to every row pointer), `budget` (bytes of a row
// chunk, 0: the library's 1 GiB), `null_list` / `null_indices` / `null_pos` / `null_counts` (1: pass NULL), and B200_*
// hooks, which are set in the environment for that line only.  Output: one line per call, the message (which has
// spaces) last.
#include <iostream>
#include <map>
#include <sstream>
#include <string>
#include <vector>

#include "../rectools_b200/csrc/list_plan.h"

static std::vector<long long> numbers(const std::string& s) {
    std::vector<long long> out;
    std::stringstream ss(s);
    for (std::string w; std::getline(ss, w, ',');)
        if (!w.empty()) out.push_back(std::stoll(w));
    return out;
}

int main() {
    std::string line;
    while (std::getline(std::cin, line)) {
        std::map<std::string, std::string> v;
        std::vector<std::string> hooks;
        std::istringstream words(line);
        for (std::string w; words >> w;) {
            const size_t eq = w.find('=');
            const std::string name = w.substr(0, eq), value = w.substr(eq + 1);
            if (name.rfind("B200_", 0) == 0) {
                setenv(name.c_str(), value.c_str(), 1);
                hooks.push_back(name);
            } else {
                v[name] = value;
            }
        }
        auto num = [&](const char* name) { return v.count(name) ? std::stoll(v[name]) : 0ll; };
        b200::ListArgs a;
        a.n_list = num("n_list");
        std::vector<int32_t> list;
        if (v.count("list"))
            for (long long id : numbers(v["list"])) list.push_back((int32_t)id);
        else
            for (int64_t i = 0; i < a.n_list && i < (1 << 20); ++i) list.push_back((int32_t)i);
        const bool null_indptr = v["lens"] == "-";
        std::vector<int64_t> indptr(1, num("base"));
        for (long long len : numbers(null_indptr ? "" : v["lens"])) indptr.push_back(indptr.back() + len);
        std::vector<int32_t> ids;
        if (v.count("ids"))
            for (long long id : numbers(v["ids"])) ids.push_back((int32_t)id);
        else
            for (int64_t e = 0; e < indptr.back(); ++e) ids.push_back((int32_t)e);
        a.n_rows = v.count("n_rows") ? num("n_rows") : (int64_t)indptr.size() - 1;
        a.list_ids = num("null_list") || list.empty() ? nullptr : list.data();
        a.indptr = null_indptr ? nullptr : indptr.data();
        a.indices = num("null_indices") || ids.empty() ? nullptr : ids.data();
        a.k = num("k");
        a.out_pos = !num("null_pos");
        a.out_counts = !num("null_counts");
        const int64_t budget = num("budget") > 0 ? num("budget") : b200::LIST_CHUNK_BYTES;
        const b200::ListPlan p = b200::plan_list(a, b200::list_chunk_rows_hook(), budget);
        for (const std::string& h : hooks) unsetenv(h.c_str());
        std::cout << "k_out=" << p.k_out << " n_chunks=" << p.n_chunks() << " max_chunk_rows=" << p.max_chunk_rows
                  << " max_chunk_nnz=" << p.max_chunk_nnz << " error=" << p.error << " bounds=";
        for (size_t i = 0; i < p.bounds.size(); ++i) std::cout << (i ? "," : "") << p.bounds[i];
        std::cout << " message=" << p.message << std::endl;
    }
    return 0;
}
