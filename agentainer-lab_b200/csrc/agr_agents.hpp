// agr_agents.hpp — the agent key table: open addressing with linear probing over agr_agent_key entries (all-zero id words =
// empty), placed by agr_hash_agent of the NUL-padded id.  The engine keeps the table on the host (agr_handle::akeys_host) and
// mirrors it to agr_dev::akeys, where K1 and the service kernel probe it (agr_device.cuh: agent_resolve); tests/agent_table_harness.cpp
// drives the same code on the CPU.  The table has at least twice as many entries as there are agents, so it never fills up.
#pragma once
#include <stdint.h>
#include <string.h>
#include "agr_common.h"

static inline bool agt_empty(const agr_agent_key& e) { return (e.w[0] | e.w[1] | e.w[2] | e.w[3]) == 0ULL; }
static inline uint32_t agt_home(const unsigned long long w[4], uint32_t mask) {
    return (uint32_t)agr_hash_agent(w[0], w[1], w[2], w[3]) & mask;
}
// the id's 32 key bytes: NUL padded, at most 31 characters
static inline void agt_pack(const char* id, unsigned long long w[4]) {
    char buf[32];
    memset(buf, 0, sizeof buf);
    strncpy(buf, id, sizeof buf - 1);
    memcpy(w, buf, 32);
}
// index of the entry that holds id w, or -1
static inline int64_t agt_find(const agr_agent_key* t, uint32_t mask, const unsigned long long w[4]) {
    for (uint32_t i = agt_home(w, mask), k = 0; k <= mask; ++k, i = (i + 1) & mask) {
        if (agt_empty(t[i])) return -1;
        if (memcmp(t[i].w, w, 32) == 0) return i;
    }
    return -1;
}
// puts key (an id the table does not hold) into the first empty entry of its probe path and returns that index
static inline uint32_t agt_insert(agr_agent_key* t, uint32_t mask, const agr_agent_key& key) {
    uint32_t i = agt_home(key.w, mask);
    while (!agt_empty(t[i])) i = (i + 1) & mask;
    t[i] = key;
    return i;
}
// Removes entry idx by backward shift: each later entry of the cluster whose home does not lie cyclically in (hole, its index]
// moves back into the hole, which then continues from where it was.  Every probe path stays unbroken and no tombstone is left,
// so a table under agent churn never fills with dead entries.  Returns how many entries from idx on (cyclically) may have
// changed: all of them lie in idx, idx + 1, ..., idx + count - 1 (mod the table size).
static inline uint32_t agt_delete(agr_agent_key* t, uint32_t mask, uint32_t idx) {
    uint32_t hole = idx, j = idx;
    for (;;) {
        j = (j + 1) & mask;
        if (agt_empty(t[j])) break;
        const uint32_t home = agt_home(t[j].w, mask);
        if (((j - home) & mask) >= ((j - hole) & mask)) { t[hole] = t[j]; hole = j; }
    }
    memset(&t[hole], 0, sizeof t[hole]);
    return ((j - idx) & mask);
}
