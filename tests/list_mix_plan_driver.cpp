// Prints, for tests/test_popular_in_category_cpu.py, the path-8 plan (rectools_b200/csrc/list_mix_plan.h: plan_list_mix)
// of the calls read from stdin, one per line of `name=value` words: `lists` (comma-separated list lengths; the ids are
// 0, 1, 2, ... unless `ids` lists them, comma-separated; `offsets` gives the offsets instead), `quota` (comma-separated;
// default 0 per list), `mixing`, `k`, `lens` (comma-separated viewed counts per row, ids 0, 1, 2, ...; `lens=-` passes a
// NULL csr_indptr and then `n_rows` gives the rows), `base` (added to every row pointer), `budget` (bytes of a row chunk,
// 0: the library's 1 GiB), `smem` (the shared-memory cap, 0: the default), `null_offsets` / `null_ids` / `null_quota` /
// `null_indices` / `null_pos` / `null_counts` (1: pass NULL), and B200_* hooks, set in the environment for that line only.
// Output: one line per call, the message (which has spaces) last.
#include <iostream>
#include <map>
#include <sstream>
#include <string>
#include <vector>

#include "../rectools_b200/csrc/list_mix_plan.h"

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
        b200::ListMixArgs a;
        std::vector<int64_t> offsets(1, 0);
        if (v.count("offsets")) {
            offsets.clear();
            for (long long o : numbers(v["offsets"])) offsets.push_back(o);
        } else {
            for (long long len : numbers(v["lists"])) offsets.push_back(offsets.back() + len);
        }
        a.n_lists = v.count("n_lists") ? num("n_lists") : (int64_t)offsets.size() - 1;
        std::vector<int32_t> ids;
        if (v.count("ids"))
            for (long long id : numbers(v["ids"])) ids.push_back((int32_t)id);
        else
            for (int64_t i = 0; i < offsets.back() && i < (1 << 20); ++i) ids.push_back((int32_t)i);
        std::vector<int32_t> quota(std::max<int64_t>(a.n_lists, 0), 0);
        const std::vector<long long> q = numbers(v["quota"]);
        for (size_t c = 0; c < q.size() && c < quota.size(); ++c) quota[c] = (int32_t)q[c];
        const bool null_indptr = v["lens"] == "-";
        std::vector<int64_t> indptr(1, num("base"));
        for (long long len : numbers(null_indptr ? "" : v["lens"])) indptr.push_back(indptr.back() + len);
        std::vector<int32_t> viewed;
        for (int64_t e = 0; e < indptr.back(); ++e) viewed.push_back((int32_t)e);
        a.offsets = num("null_offsets") ? nullptr : offsets.data();
        a.list_ids = num("null_ids") || ids.empty() ? nullptr : ids.data();
        a.quota = num("null_quota") || quota.empty() ? nullptr : quota.data();
        a.mixing = num("mixing");
        a.n_rows = v.count("n_rows") ? num("n_rows") : (int64_t)indptr.size() - 1;
        a.indptr = null_indptr ? nullptr : indptr.data();
        a.indices = num("null_indices") || viewed.empty() ? nullptr : viewed.data();
        a.k = num("k");
        a.out_pos = !num("null_pos");
        a.out_counts = !num("null_counts");
        const int64_t budget = num("budget") > 0 ? num("budget") : b200::LIST_CHUNK_BYTES;
        const b200::ListMixPlan p = b200::plan_list_mix(a, b200::list_chunk_rows_hook(), num("smem"), budget);
        for (const std::string& h : hooks) unsetenv(h.c_str());
        std::cout << "k_out=" << p.k_out << " n_total=" << p.n_total << " n_chunks=" << p.n_chunks()
                  << " max_chunk_rows=" << p.max_chunk_rows << " max_chunk_nnz=" << p.max_chunk_nnz
                  << " row_scratch=" << p.row_scratch << " smem=" << (int)p.smem << " error=" << p.error << " slots=";
        for (size_t i = 0; i < p.slots.size(); ++i) std::cout << (i ? "," : "") << p.slots[i];
        std::cout << " bounds=";
        for (size_t i = 0; i < p.bounds.size(); ++i) std::cout << (i ? "," : "") << p.bounds[i];
        std::cout << " message=" << p.message << std::endl;
    }
    return 0;
}
