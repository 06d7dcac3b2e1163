// Prints, for tests/test_candidate_sets_device_cpu.py, the plan of path-5 calls on device lists
// (rectools_b200/csrc/plan.h: plan_candidates_device) or, with `route=host`, on host lists (plan_candidates), for the calls
// read from stdin, one per line of `name=value` words: the CandShape fields (n_rows n_objects k d flags whitelist sparse
// rows res_device id_offset), `budget` (bytes of a row chunk, 0: the engine's 1 GiB), `lens` (comma-separated raw row
// lengths), `base` (cand_indptr[0]) and B200_* hooks, which are set in the environment for that line only.  `lens=-`
// passes a NULL indptr.  Output: one line per call, the message (which has spaces) last.
#include <iostream>
#include <map>
#include <sstream>
#include <string>
#include <vector>

#include "../rectools_b200/csrc/plan.h"

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
        b200::CandShape s;
        s.n_rows = num("n_rows");
        s.n_objects = num("n_objects");
        s.k = num("k");
        s.d = (int)num("d");
        s.flags = (int32_t)num("flags");
        s.whitelist = num("whitelist") != 0;
        s.sparse = num("sparse") != 0;
        s.rows = num("rows") != 0;
        s.res_device = num("res_device") != 0;
        s.id_offset = num("id_offset") != 0;
        const bool null_indptr = v["lens"] == "-";
        std::vector<int64_t> indptr(1, num("base"));
        for (long long len : numbers(null_indptr ? "" : v["lens"])) indptr.push_back(indptr.back() + len);
        const int64_t budget = num("budget") > 0 ? num("budget") : b200::SELECT_CHUNK_BYTES;
        const int64_t* ip = null_indptr ? nullptr : indptr.data();
        const b200::CandPlan p = v["route"] == "host" ? b200::plan_candidates(s, ip, b200::read_hooks(), budget)
                                                      : b200::plan_candidates_device(s, ip, b200::read_hooks(), budget);
        for (const std::string& h : hooks) unsetenv(h.c_str());
        std::cout << "k_out=" << p.k_out << " n_chunks=" << p.n_chunks() << " max_chunk_cands=" << p.max_chunk_cands
                  << " max_chunk_rows=" << p.max_chunk_rows << " error=" << p.error << " bounds=";
        for (size_t i = 0; i < p.bounds.size(); ++i) std::cout << (i ? "," : "") << p.bounds[i];
        std::cout << " message=" << p.message << std::endl;
    }
    return 0;
}
