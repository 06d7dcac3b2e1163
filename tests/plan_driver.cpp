// Prints the plan of rectools_b200/csrc/plan.h for the calls read from stdin, one per line of `name=value` words:
// the CallShape fields (n_rows n_pos k d d_pad sm_count tc_dtype n_peers flags sparse rows n_objects cosine) and B200_*
// hooks, which are set in the environment for that line only and read through read_hooks().  Built and run by
// tests/test_call_plan_cpu.py and tests/test_call_history_cases_cpu.py.
#include <iostream>
#include <map>
#include <sstream>
#include <string>
#include <vector>

#include "../rectools_b200/csrc/plan.h"

int main() {
    std::string line;
    while (std::getline(std::cin, line)) {
        b200::CallShape s;
        std::map<std::string, long long> v;
        std::vector<std::string> hooks;
        std::istringstream words(line);
        for (std::string w; words >> w;) {
            const size_t eq = w.find('=');
            const std::string name = w.substr(0, eq), value = w.substr(eq + 1);
            if (name.rfind("B200_", 0) == 0) {
                setenv(name.c_str(), value.c_str(), 1);
                hooks.push_back(name);
            } else {
                v[name] = std::stoll(value);
            }
        }
        s.n_rows = v["n_rows"];
        s.n_pos = v["n_pos"];
        s.k = v["k"];
        s.d = (int)v["d"];
        s.d_pad = v.count("d_pad") ? (int)v["d_pad"] : (int)b200::round_up(s.d, 64);
        s.sm_count = (int)v["sm_count"];
        s.tc_dtype = (int)v["tc_dtype"];
        s.n_peers = (int)v["n_peers"];
        s.flags = (int32_t)v["flags"];
        s.sparse = v["sparse"] != 0;
        s.rows = v["rows"] != 0;
        s.n_objects = v["n_objects"];
        s.cosine = v["cosine"] != 0;
        const b200::CallPlan p = b200::plan_call(s, b200::read_hooks());
        for (const std::string& h : hooks) unsetenv(h.c_str());
        std::cout << "k_out=" << p.k_out << " path=" << (int)p.path << " mode=" << (int)p.mode << " select=" << (int)p.select << " nw=" << p.nw
                  << " k_cand=" << p.k_cand << " peers=" << p.peers << " T=" << p.geom.T << " cand_stride=" << p.geom.cand_stride
                  << " chunk=" << p.chunk << " n_chunks=" << p.n_chunks << " error=" << p.error << " message=" << p.message
                  << std::endl;
    }
    return 0;
}
