// agent_table_harness.cpp — the agent key table of csrc/agr_agents.hpp (the code the engine ships), driven from stdin for
// tests/test_agent_table.py, on the CPU.  One command per line, one answer line each:
//   n <entries>          -> "ok": a new empty table (entries a power of two)
//   i <id> <slot>        -> "<index>": agt_insert of an id the table does not hold
//   d <id>               -> "<index> <count>": agt_delete of the id's entry (count = entries from index on that may have changed)
//   f <id>               -> "<slot>" or "none": agt_find
//   v                    -> "ok <live> <wrapped>" or "bad <reason>": every entry reachable from its home along an unbroken run
//                           of live entries, no id twice; wrapped = 1 when the last and the first entry are both live
// Test infrastructure, no CUDA.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "../agentainer-lab_b200/csrc/agr_agents.hpp"

int main() {
    std::vector<agr_agent_key> t;
    uint32_t mask = 0;
    char line[512];
    while (fgets(line, sizeof line, stdin)) {
        char* tok[4]; int k = 0;
        for (char* p = strtok(line, " \t\n"); p && k < 4; p = strtok(nullptr, " \t\n")) tok[k++] = p;
        if (k == 2 && tok[0][0] == 'n') {
            const uint32_t n = (uint32_t)strtoul(tok[1], nullptr, 0);
            t.assign(n, agr_agent_key{}); mask = n - 1;
            printf("ok\n");
        } else if (k == 3 && tok[0][0] == 'i') {
            agr_agent_key key{};
            agt_pack(tok[1], key.w);
            key.slot = (uint32_t)strtoul(tok[2], nullptr, 0);
            printf("%u\n", agt_insert(t.data(), mask, key));
        } else if (k == 2 && (tok[0][0] == 'd' || tok[0][0] == 'f')) {
            unsigned long long w[4];
            agt_pack(tok[1], w);
            const int64_t i = agt_find(t.data(), mask, w);
            if (tok[0][0] == 'f') { if (i < 0) printf("none\n"); else printf("%u\n", t[i].slot); continue; }
            if (i < 0) { printf("missing\n"); continue; }
            printf("%lld %u\n", (long long)i, agt_delete(t.data(), mask, (uint32_t)i));
        } else if (k == 1 && tok[0][0] == 'v') {
            uint32_t live = 0; const char* bad = nullptr;
            for (uint32_t j = 0; j <= mask && !bad; ++j) {
                if (agt_empty(t[j])) continue;
                ++live;
                for (uint32_t p = agt_home(t[j].w, mask); p != j && !bad; p = (p + 1) & mask)
                    if (agt_empty(t[p])) bad = "hole on a probe path";
                for (uint32_t q = j + 1; q <= mask && !bad; ++q)
                    if (!agt_empty(t[q]) && memcmp(t[q].w, t[j].w, 32) == 0) bad = "id twice";
            }
            if (bad) printf("bad %s\n", bad);
            else printf("ok %u %d\n", live, (!agt_empty(t[mask]) && !agt_empty(t[0])) ? 1 : 0);
        } else {
            fprintf(stderr, "bad command\n");
            return 2;
        }
    }
    return 0;
}
