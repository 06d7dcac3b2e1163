// Prints the row split of rectools_b200/csrc/group_plan.h for the requests read from stdin, one per line:
//   split n_rows n_members forced   ->  "slice_rows n_slices r0 r1 r0 r1 ..."
//   rebase r0 r1 v0 v1 ... vn       ->  "base w0 w1 ..."  (indptr v cut to rows [r0, r1))
//   hook                            ->  the value of B200_GROUP_SLICE_ROWS as read_group_slice_hook() reads it
// Built and run by tests/test_engine_group_cpu.py.
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "../rectools_b200/csrc/group_plan.h"

int main() {
    std::string line;
    while (std::getline(std::cin, line)) {
        std::istringstream in(line);
        std::string op;
        in >> op;
        if (op == "split") {
            long long n = 0, members = 0, forced = 0;
            in >> n >> members >> forced;
            const int64_t rows = b200::group_slice_rows(n, (int)members, forced);
            const int64_t ns = b200::group_n_slices(n, rows);
            std::cout << rows << " " << ns;
            for (int64_t i = 0; i < ns; ++i) {
                const b200::GroupSlice s = b200::group_slice(n, rows, i);
                std::cout << " " << s.r0 << " " << s.r1;
            }
            std::cout << "\n";
        } else if (op == "rebase") {
            long long r0 = 0, r1 = 0;
            in >> r0 >> r1;
            std::vector<int64_t> v;
            for (long long x; in >> x;) v.push_back(x);
            std::vector<int64_t> out(r1 - r0 + 1);
            const int64_t base = b200::rebase_indptr(v.data(), r0, r1, out.data());
            std::cout << base;
            for (int64_t w : out) std::cout << " " << w;
            std::cout << "\n";
        } else if (op == "hook") {
            std::cout << b200::read_group_slice_hook() << "\n";
        }
    }
    return 0;
}
