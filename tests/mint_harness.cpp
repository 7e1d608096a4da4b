// mint_harness.cpp — the engine-minted id functions of csrc/agr_common.h (the code the kernels and the host ship), driven from
// stdin for tests/test_mint_ref.py, on the CPU.  One command per line, one answer line each:
//   m <secret> <shard> <gen> <first row> <n>            -> n lines "<lo> <hi>" (hex): agr_mint_id of rows first .. first + n - 1
//   d <secret> <shard> <gen> <tail> <head> <lo> <hi>    -> "<row>" or "none": agr_unmint_in_window
// Numbers are decimal or 0x-prefixed hex.  Test infrastructure, no CUDA.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../agentainer-lab_b200/csrc/agr_common.h"

static unsigned long long num(const char* s) { return strtoull(s, nullptr, 0); }

int main() {
    char line[512];
    while (fgets(line, sizeof line, stdin)) {
        char* tok[9]; int k = 0;
        for (char* p = strtok(line, " \t\n"); p && k < 9; p = strtok(nullptr, " \t\n")) tok[k++] = p;
        if (k == 6 && tok[0][0] == 'm') {
            const unsigned long long secret = num(tok[1]), first = num(tok[4]), n = num(tok[5]);
            const uint32_t shard = (uint32_t)num(tok[2]), gen = (uint32_t)num(tok[3]);
            for (unsigned long long i = 0; i < n; ++i) {
                unsigned long long lo, hi;
                agr_mint_id(first + i, shard, gen, secret, lo, hi);
                printf("%llx %llx\n", lo, hi);
            }
        } else if (k == 8 && tok[0][0] == 'd') {
            unsigned long long row = 0;
            if (agr_unmint_in_window(num(tok[6]), num(tok[7]), num(tok[1]), (uint32_t)num(tok[2]), (uint32_t)num(tok[3]), num(tok[4]),
                                     num(tok[5]), row))
                printf("%llu\n", row);
            else
                printf("none\n");
        } else {
            fprintf(stderr, "bad command\n");
            return 2;
        }
    }
    return 0;
}
