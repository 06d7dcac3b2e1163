// Prints, for tests/test_large_k_select_cpu.py, one line per stdin line:
//  - "key b0 b1 ...": order_key (rectools_b200/csrc/order_key.h) of each fp32 bit pattern (hex in, hex out);
//  - otherwise a call of `name=value` words (CallShape fields and B200_* hooks, the hooks set for that line only):
//    the selection part of its plan (rectools_b200/csrc/plan.h) and the bytes per row of its path-2 / path-3 row chunks.
#include <cstdint>
#include <cstring>
#include <iostream>
#include <map>
#include <sstream>
#include <string>
#include <vector>

#include "../rectools_b200/csrc/order_key.h"
#include "../rectools_b200/csrc/plan.h"

int main() {
    std::string line;
    while (std::getline(std::cin, line)) {
        std::istringstream words(line);
        if (line.rfind("key", 0) == 0) {
            std::string w;
            words >> w;
            for (std::string hex; words >> hex;) {
                const uint32_t bits = (uint32_t)std::stoul(hex, nullptr, 16);
                float s;
                std::memcpy(&s, &bits, sizeof(s));
                std::cout << std::hex << b200::order_key(s) << std::dec << " ";
            }
            std::cout << std::endl;
            continue;
        }
        b200::CallShape s;
        std::map<std::string, long long> v;
        std::vector<std::string> hooks;
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
        s.d_pad = (int)b200::round_up(s.d, 64);
        s.sm_count = (int)v["sm_count"];
        s.tc_dtype = (int)v["tc_dtype"];
        s.flags = (int32_t)v["flags"];
        s.sparse = v["sparse"] != 0;
        const b200::CallPlan p = b200::plan_call(s, b200::read_hooks());
        for (const std::string& h : hooks) unsetenv(h.c_str());
        std::cout << "k_out=" << p.k_out << " path=" << (int)p.path << " mode=" << (int)p.mode << " select=" << (int)p.select
                  << " row_bytes=" << b200::select_row_bytes(s.n_pos, p.k_out, p.select) << " error=" << p.error << std::endl;
    }
    return 0;
}
