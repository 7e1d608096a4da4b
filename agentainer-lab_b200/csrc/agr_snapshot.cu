// agr_snapshot.cu — agr_snapshot and agr_restore: full files (AGRSNAP3), deltas (AGRDELT1), the online cut and the chain.
#include <limits.h>
#include <sys/stat.h>
#include "agr_engine.h"

// ------------------------------------------------------------------------------------------ durability
static int dump_dev(agr_handle* h, FILE* f, void* dsrc, size_t bytes) {
    const size_t chunk = h->bounce_bytes;
    for (size_t o = 0; o < bytes; o += chunk) {
        const size_t m = std::min(chunk, bytes - o);
        CK(cudaMemcpyAsync(h->bounce[0], (const uint8_t*)dsrc + o, m, cudaMemcpyDeviceToHost, h->stream));
        CK(cudaStreamSynchronize(h->stream));
        if (fwrite(h->bounce[0], 1, m, f) != m) return fail(AGR_EINVAL, "snapshot: short write");
    }
    return 0;
}
static int load_dev(agr_handle* h, FILE* f, void* ddst, size_t bytes) {
    const size_t chunk = h->bounce_bytes;
    for (size_t o = 0; o < bytes; o += chunk) {
        const size_t m = std::min(chunk, bytes - o);
        if (fread(h->bounce[0], 1, m, f) != m) return fail(AGR_EINVAL, "restore: short read");
        CK(cudaMemcpyAsync((uint8_t*)ddst + o, h->bounce[0], m, cudaMemcpyHostToDevice, h->stream));
        CK(cudaStreamSynchronize(h->stream));
    }
    return 0;
}
// the physical rows a snapshot holds
static size_t snap_rows(const snap_header& hd) {
    return (hd.flags & AGR_CFG_RING) ? (size_t)std::min<uint64_t>(hd.rows_used, hd.slab_rows) : (size_t)hd.rows_used;
}
// One section of the file: its live device array, its size, and what later calls do to it.  kind SNAP_APPEND: only ever
// appended to inside the window of a snapshot (the slab rows, the record bytes, the response bytes); SNAP_WORDS: per-row words
// rewritten in place; SNAP_LOG: a log, rewritten in place (k_drop_logs) and compacted by agr_reclaim.  The online snapshot
// copies the last two kinds into its shadow at the cut and streams the first from where it lies.
enum { SNAP_APPEND = 0, SNAP_WORDS = 1, SNAP_LOG = 2 };
struct snap_section { void* p; size_t bytes; int kind; };
#define SNAP_NSEC 17
// The sections that follow the header and the agent table, in file order.  Every size comes from the header alone: the one
// description of the layout that agr_snapshot and agr_restore share (tests/test_snapshot_layout_gpu.py reads a file against it).
static void snap_table(agr_handle* h, const snap_header& hd, snap_section out[SNAP_NSEC]) {
    const bool ring = (hd.flags & AGR_CFG_RING) != 0, varlen = (hd.flags & AGR_CFG_VARLEN) != 0;
    const size_t R = snap_rows(hd);
    const snap_section sections[SNAP_NSEC] = {
        {h->d.slab, varlen ? (size_t)(ring ? std::min<uint64_t>(hd.vused, hd.vcap) : hd.vused) : R * AGR_REC, SNAP_APPEND},
        {h->d.state, R * 4, SNAP_WORDS},
        {h->d.route, R * 4, SNAP_WORDS},
        {h->d.aux, R * 4, SNAP_WORDS},
        {h->d.cksum, R * 8, SNAP_WORDS},
        {h->d.voff, varlen ? R * 8 : 0, SNAP_WORDS},
        {h->d.vlen, varlen ? R * 4 : 0, SNAP_WORDS},
        {h->d.completed_log, (size_t)hd.log_len[0] * 4, SNAP_LOG},
        {h->d.failed_log, (size_t)hd.log_len[1] * 4, SNAP_LOG},
        {h->d_resp, (size_t)(ring ? std::min<uint64_t>(hd.resp_used, hd.resp_cap) : hd.resp_used), SNAP_APPEND},
        {h->d_resp_off, R * 8, SNAP_WORDS},
        {h->d_resp_len, R * 4, SNAP_WORDS},
        {h->d_resp_hlen, R * 4, SNAP_WORDS},
        {h->d_err_off, R * 8, SNAP_WORDS},
        {h->d_err_len, R * 4, SNAP_WORDS},
        {h->d.ptime, R * 8, SNAP_WORDS},
        {h->d.mtime, R * 8, SNAP_WORDS},
    };
    for (int k = 0; k < SNAP_NSEC; ++k) out[k] = sections[k];
}
// Hands every section to io (dump_dev, load_dev or the online writer's dump_online) as (device array, bytes).  The source
// table says where each section's bytes are: nullptr = the live arrays; the online writer passes the cut's shadow, which
// holds the sections rewritten in place at h->shadow_off (the append-only ones still come from the live arrays).
static int snap_sections(agr_handle* h, const snap_header& hd, FILE* f, int (*io)(agr_handle*, FILE*, void*, size_t),
                         uint8_t* shadow = nullptr) {
    snap_section sec[SNAP_NSEC];
    snap_table(h, hd, sec);
    for (int k = 0; k < SNAP_NSEC; ++k) TRY(io(h, f, shadow && sec[k].kind != SNAP_APPEND ? shadow + h->shadow_off[k] : sec[k].p, sec[k].bytes));
    return 0;
}

// ---- AGR_CFG_DELTA_SNAPSHOT
// A delta file (AGRDELT1): this header; the parent's absolute path; the agent table, as in a full file; the appended slab rows
// (record bytes with AGR_CFG_VARLEN) [rows_lo, rows_hi), then the appended response bytes [resp_lo, resp_hi), both in physical
// order, in one run or two where the ring wraps; the ascending list of dirty word blocks (u32), then each listed block's slice
// of every SNAP_WORDS section of snap_table, in table order; then per log (completed, failed) the same for its dirty log
// blocks.  Only the last block of a section may be short.  The digests are the compare cut's keyed sums over the word
// sections [0, R) and the log prefixes of the parent's cut and of this one.
#define SNAP_BLOCK_ROWS 256u
#define SNAP_LOG_BLOCK 1024u
struct delta_header {
    char magic[8];                 // "AGRDELT1"
    snap_header cut;               // the state this file brings a restore to
    uint64_t file_bytes;           // a restore refuses a shorter file
    unsigned long long parent_digest[2], digest[2];
    uint32_t block_rows, log_block;
    uint64_t rows_lo, rows_hi, resp_lo, resp_hi;
    uint64_t n_blocks[3];          // listed blocks per table of snap_block_tables
    uint32_t parent_path_len, pad;
};
static_assert(sizeof(delta_header) == 264 && sizeof(snap_header) == 144, "delta_header is a file layout");

// Everything the compare cut, the gather and the scatter use; allocated at agr_create (or by the restore of a delta chain)
static int snap_delta_alloc(agr_handle* h) {
    if (h->d_snap_stage) return 0;
    const size_t nwb = (h->cfg.slab_rows + SNAP_BLOCK_ROWS - 1) / SNAP_BLOCK_ROWS, nlb = (h->d.log_cap + SNAP_LOG_BLOCK - 1) / SNAP_LOG_BLOCK;
    h->snap_bit_off[1] = (nwb + 31) / 32; h->snap_bit_off[2] = h->snap_bit_off[1] + (nlb + 31) / 32;
    h->snap_bit_words = h->snap_bit_off[2] + (nlb + 31) / 32;
    TRY(dev_alloc(h, &h->d_snap_bits, h->snap_bit_words, false));
    TRY(dev_alloc(h, &h->d_snap_digest, (size_t)2, false));
    TRY(host_alloc(h, &h->h_snap_bits, 32 + h->snap_bit_words * 4));
    TRY(dev_alloc(h, &h->d_snap_list, std::max<size_t>(std::max(nwb, nlb), 1), false));
    h->snap_stage_bytes = std::max<size_t>(h->bounce_bytes, (size_t)1 << 20);   // >= one block of every section
    TRY(dev_alloc(h, &h->d_snap_stage, h->snap_stage_bytes, false));
    return 0;
}
static size_t snap_full_bytes(agr_handle* h, const snap_header& hd) {
    snap_section sec[SNAP_NSEC];
    snap_table(h, hd, sec);
    size_t n = sizeof(snap_header) + (size_t)hd.n_agents * (AGR_AGENT_ID_BYTES + 1);
    for (int k = 0; k < SNAP_NSEC; ++k) n += sec[k].bytes;
    return n;
}
// The cut's sections: the SNAP_WORDS ones that hold bytes, then the two logs (whose lengths the kernel reads on the device
// unless lens_from_host).  A word block is 256 rows: 16 * width pieces of 16 B; a log block 1024 entries: 256 pieces.
static void snap_cut_params(agr_handle* h, const snap_header& hd, bool lens_from_host, agr_snap_cmp& c) {
    snap_section sec[SNAP_NSEC];
    snap_table(h, hd, sec);
    const size_t R = snap_rows(hd);
    c = agr_snap_cmp{};
    c.shadow = h->d_shadow; c.bits = h->d_snap_bits; c.digest = h->d_snap_digest; c.key = h->d.id_secret;
    c.lens_from_host = lens_from_host ? 1u : 0u;
    int logs[2], nlog = 0;
    for (int k = 0; k < SNAP_NSEC; ++k) {
        if (sec[k].kind == SNAP_LOG) logs[nlog++] = k;
        if (sec[k].kind != SNAP_WORDS || sec[k].bytes == 0) continue;
        const uint32_t n = c.nrow++;
        c.src[n] = (const uint8_t*)sec[k].p; c.dst_off[n] = h->shadow_off[k]; c.bytes[n] = sec[k].bytes;
        c.pshift[n] = (uint32_t)__builtin_ctzll(16 * (sec[k].bytes / R)); c.bit_off[n] = 0; c.sec_id[n] = (uint32_t)k;
    }
    for (int j = 0; j < 2; ++j) {
        const uint32_t n = c.nrow + j;
        c.src[n] = (const uint8_t*)sec[logs[j]].p; c.dst_off[n] = h->shadow_off[logs[j]]; c.bytes[n] = sec[logs[j]].bytes;
        c.pshift[n] = 8; c.bit_off[n] = (uint32_t)h->snap_bit_off[1 + j]; c.sec_id[n] = (uint32_t)logs[j];
    }
}
// the cut (caller holds HLock): one kernel copies the per-row words of rows [0, R) and the two log prefixes into the shadow;
// with compare, it also marks the blocks that differ from the previous cut and sums the digest of this one
static int snap_cut_locked(agr_handle* h, const snap_header& hd, bool compare) {
    agr_snap_cmp c;
    snap_cut_params(h, hd, false, c);
    if (compare) {
        CK(cudaMemsetAsync(h->d_snap_bits, 0, h->snap_bit_words * 4, h->stream));
        CK(cudaMemsetAsync(h->d_snap_digest, 0, 16, h->stream));
    }
    TRY(op_time_begin(h, 3));
    if (compare) agr_launch_snap_cmp(h->d, c, true, h->sm_count, h->stream);
    else agr_launch_snap_cut(h->d, c, h->sm_count, h->stream);
    CK(cudaGetLastError());
    TRY(op_time_end(h, 3));
    CK(cudaEventRecord(h->snap_ev[0], h->stream));
    return 0;
}
// (restore) the digest of the live arrays as hd describes them.  seed: through the compare cut, which also leaves them in the
// shadow, so that the next snapshot of an AGR_CFG_DELTA_SNAPSHOT engine compares against the restored state
static int snap_digest_locked(agr_handle* h, const snap_header& hd, bool seed, unsigned long long out[2]) {
    agr_snap_cmp c;
    snap_cut_params(h, hd, !seed, c);
    if (seed) CK(cudaMemsetAsync(h->d_snap_bits, 0, h->snap_bit_words * 4, h->stream));
    CK(cudaMemsetAsync(h->d_snap_digest, 0, 16, h->stream));
    agr_launch_snap_cmp(h->d, c, seed, h->sm_count, h->stream);
    CK(cudaGetLastError());
    TRY(d2h_staged(h, out, h->d_snap_digest, 16, h->h_snap_bits));
    return 0;
}
// The block tables of a delta, in file order: [0] the word sections of hd (256 rows per block), [1] and [2] the completed and
// failed logs (1024 entries per block), in the shadow (the writer) or the live arrays (restore).  Table t's bits start at
// snap_bit_off[t].
static void snap_block_tables(agr_handle* h, const snap_header& hd, bool shadow, agr_snap_blocks g[3]) {
    snap_section sec[SNAP_NSEC];
    snap_table(h, hd, sec);
    for (int t = 0; t < 3; ++t) g[t] = agr_snap_blocks{};
    g[0].block_rows = SNAP_BLOCK_ROWS; g[0].rows = snap_rows(hd);
    for (int k = 0, j = 0; k < SNAP_NSEC; ++k) {
        uint8_t* a = shadow ? h->d_shadow + h->shadow_off[k] : (uint8_t*)sec[k].p;
        if (sec[k].kind == SNAP_LOG) {
            agr_snap_blocks& l = g[1 + j];
            l.arr[0] = a; l.nsec = 1; l.width[0] = 4; l.block_rows = SNAP_LOG_BLOCK; l.rows = hd.log_len[j++]; l.rec_bytes = 4ull * SNAP_LOG_BLOCK;
        } else if (sec[k].kind == SNAP_WORDS && sec[k].bytes) {
            agr_snap_blocks& w = g[0];
            w.arr[w.nsec] = a; w.width[w.nsec] = (uint32_t)(sec[k].bytes / w.rows);
            w.rec_bytes += (unsigned long long)w.width[w.nsec] * SNAP_BLOCK_ROWS;
            w.nsec++;
        }
    }
}
// bytes of the slices of n listed blocks (only the table's last block may be short)
static uint64_t snap_blocks_bytes(const agr_snap_blocks& g, const uint32_t* list, size_t n) {
    if (!n) return 0;
    const uint64_t last = list[n - 1], r0 = last * g.block_rows;
    return (n - 1) * g.rec_bytes + std::min<uint64_t>(g.block_rows, g.rows - r0) * (g.rec_bytes / g.block_rows);
}
// The appended pieces of a delta, in file order: the slab rows (record bytes with AGR_CFG_VARLEN) [rows_lo, rows_hi), then the
// response bytes [resp_lo, resp_hi), each in one physical run or two where its ring wraps, as (live device array, bytes)
struct snap_piece { uint8_t* p; uint64_t bytes; };
static int snap_delta_pieces(agr_handle* h, const delta_header& dh, snap_piece out[4]) {
    const snap_header& hd = dh.cut;
    const bool var = (hd.flags & AGR_CFG_VARLEN) != 0, ring = (hd.flags & AGR_CFG_RING) != 0;
    const struct { uint64_t lo, hi, cap; uint8_t* base; uint64_t unit; } spans[2] = {
        {dh.rows_lo, dh.rows_hi, var ? hd.vcap : hd.slab_rows, h->d.slab, var ? 1ull : (uint64_t)AGR_REC}, {dh.resp_lo, dh.resp_hi, hd.resp_cap, h->d_resp, 1}};
    int n = 0;
    for (const auto& s : spans) {
        if (s.hi <= s.lo) continue;
        const uint64_t p = ring ? s.lo % s.cap : s.lo, n0 = ring ? std::min(s.hi - s.lo, s.cap - p) : s.hi - s.lo;
        out[n++] = {s.base + p * s.unit, n0 * s.unit};
        if (s.hi - s.lo > n0) out[n++] = {s.base, (s.hi - s.lo - n0) * s.unit};
    }
    return n;
}
// the absolute name a chain keeps of a file: realpath of its directory, then its name ("" if the directory does not resolve)
static std::string snap_abs_path(const std::string& p) {
    const size_t cut = p.rfind('/');
    const std::string dir = cut == std::string::npos ? "." : (cut == 0 ? "/" : p.substr(0, cut));
    char buf[PATH_MAX];
    if (!realpath(dir.c_str(), buf)) return "";
    std::string out(buf);
    if (out.back() != '/') out += '/';
    return out + (cut == std::string::npos ? p : p.substr(cut + 1));
}

// ---- AGR_CFG_ONLINE_SNAPSHOT
namespace agr_impl __attribute__((visibility("hidden"))) {
// The shadow holds every section rewritten in place at full capacity (slab_rows rows, log_entries entries), each at a 256 B
// boundary behind a 256 B area with the two log lengths the cut read.  Everything is allocated here: nothing is allocated or
// freed while a snapshot runs (cudaFree would wait for the resident service kernel).
int snap_online_create(agr_handle* h) {
    snap_header cap{};
    cap.flags = h->cfg.flags & (AGR_CFG_VARLEN | AGR_CFG_RING);
    cap.rows_used = cap.slab_rows = h->cfg.slab_rows;
    cap.log_len[0] = cap.log_len[1] = h->d.log_cap;
    snap_section sec[SNAP_NSEC];
    snap_table(h, cap, sec);
    size_t at = 256;
    for (int k = 0; k < SNAP_NSEC; ++k) {
        if (sec[k].kind == SNAP_APPEND || sec[k].bytes == 0) continue;
        h->shadow_off[k] = at;
        at += (sec[k].bytes + 255) & ~(size_t)255;
    }
    TRY(dev_alloc(h, &h->d_shadow, at, false));
    h->snap_buf_bytes = h->bounce_bytes;
    for (int b = 0; b < 2; ++b) TRY(host_alloc(h, &h->snap_buf[b], h->snap_buf_bytes));
    for (auto& e : h->snap_ev) CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    // non-blocking: a stream that synchronised with the legacy default stream would also wait behind the resident kernel
    CK(cudaStreamCreateWithFlags(&h->snap_stream, cudaStreamNonBlocking));
    if (h->cfg.flags & AGR_CFG_DELTA_SNAPSHOT) TRY(snap_delta_alloc(h));
    return 0;
}
}  // namespace agr_impl
// the writer stream starts behind the cut; reads what the cut left: the log lengths it read (into hd), and with compare the
// digest and the dirty bits (into h_snap_bits + 16 and + 32)
static int snap_read_cut(agr_handle* h, snap_header& hd, bool compare) {
    if (cudaStreamWaitEvent(h->snap_stream, h->snap_ev[0], 0) != cudaSuccess ||
        cudaMemcpyAsync(h->snap_buf[0], h->d_shadow, 16, cudaMemcpyDeviceToHost, h->snap_stream) != cudaSuccess ||
        (compare && (cudaMemcpyAsync(h->h_snap_bits + 16, h->d_snap_digest, 16, cudaMemcpyDeviceToHost, h->snap_stream) != cudaSuccess ||
                     cudaMemcpyAsync(h->h_snap_bits + 32, h->d_snap_bits, h->snap_bit_words * 4, cudaMemcpyDeviceToHost, h->snap_stream) != cudaSuccess)) ||
        cudaStreamSynchronize(h->snap_stream) != cudaSuccess) return fail(AGR_ECUDA, "snapshot: cut");
    memcpy(hd.log_len, h->snap_buf[0], 16);
    return 0;
}
// writes the chunk waiting in the buffer the next chunk does not use, once its copy has landed
static int snap_drain(agr_handle* h, FILE* f) {
    if (!h->snap_pend) return 0;
    const int b = h->snap_cur ^ 1;
    const size_t m = h->snap_pend;
    h->snap_pend = 0;
    CK(cudaEventSynchronize(h->snap_ev[1 + b]));
    if (fwrite(h->snap_buf[b], 1, m, f) != m) return fail(AGR_EINVAL, "snapshot: short write");
    return 0;
}
// the online writer's io: chunk k's copy on the writer stream overlaps the fwrite of chunk k - 1 (two pinned buffers)
static int dump_online(agr_handle* h, FILE* f, void* dsrc, size_t bytes) {
    for (size_t o = 0; o < bytes;) {
        const size_t m = std::min(h->snap_buf_bytes, bytes - o);
        const int b = h->snap_cur;
        CK(cudaMemcpyAsync(h->snap_buf[b], (const uint8_t*)dsrc + o, m, cudaMemcpyDeviceToHost, h->snap_stream));
        CK(cudaEventRecord(h->snap_ev[1 + b], h->snap_stream));
        TRY(snap_drain(h, f));
        h->snap_cur ^= 1; h->snap_pend = m;
        o += m;
    }
    return 0;
}
static void snap_fill_header(agr_handle* h, snap_header& hd) {
    memcpy(hd.magic, "AGRSNAP3", 8);
    hd.flags = h->cfg.flags & (AGR_CFG_PERSISTENCE | AGR_CFG_MINT_IDS | AGR_CFG_VARLEN | AGR_CFG_RING);
    hd.n_agents = (uint32_t)h->agent_names.size(); hd.shard = h->d.shard_id; hd.gen = h->d.id_gen;
    hd.rows_used = h->rows_used; hd.vused = h->vused; hd.id_secret = h->d.id_secret; hd.scan_lo = h->scan_lo;
    hd.resp_used = h->resp_used; hd.expired_total = h->expired_total; hd.tail = h->tail; hd.released_total = h->released_total; hd.slab_rows = h->cfg.slab_rows; hd.vtail = h->vtail; hd.vcap = h->vcap; hd.resp_tail = h->resp_tail; hd.resp_cap = h->resp_cap;
}
// the agent table as a file holds it: per agent its NUL-padded name (AGR_AGENT_ID_BYTES), then its status byte
static std::vector<char> snap_agents(agr_handle* h) {
    std::vector<char> agents(h->agent_names.size() * (AGR_AGENT_ID_BYTES + 1), 0);
    for (size_t a = 0; a < h->agent_names.size(); ++a) {
        char* e = agents.data() + a * (AGR_AGENT_ID_BYTES + 1);
        strncpy(e, h->agent_names[a].c_str(), AGR_AGENT_ID_BYTES - 1);
        e[AGR_AGENT_ID_BYTES] = (char)h->agent_status[a];
    }
    return agents;
}
// A full file (AGRSNAP3): the header, the agent table, then the sections through io (dump_dev, or dump_online with the cut's
// shadow as in snap_sections) and the drain of the last chunk (nothing is pending after dump_dev)
static int snap_write_full(agr_handle* h, FILE* f, const snap_header& hd, const std::vector<char>& agents,
                           int (*io)(agr_handle*, FILE*, void*, size_t), uint8_t* shadow = nullptr) {
    if (fwrite(&hd, sizeof hd, 1, f) != 1 || fwrite(agents.data(), 1, agents.size(), f) != agents.size())
        return fail(AGR_EINVAL, "snapshot: short write");
    TRY(snap_sections(h, hd, f, io, shadow));
    return snap_drain(h, f);
}
// closes a file a snapshot wrote; a failed close (the last buffered bytes did not reach the file) fails a snapshot that had not
// failed already
static int snap_close(FILE* f, int r) {
    if (fclose(f) != 0 && r == 0) return fail(AGR_EINVAL, "snapshot: close failed");
    return r;
}
// the writer: the list, then the listed blocks of g, packed on the writer stream into the staging buffer (stream order keeps
// a chunk's copies ahead of the next chunk's gather) and streamed through the pinned buffers
static int dump_blocks(agr_handle* h, FILE* f, agr_snap_blocks g, const std::vector<uint32_t>& list) {
    TRY(snap_drain(h, f));
    if (list.empty()) return 0;
    if (fwrite(list.data(), 4, list.size(), f) != list.size()) return fail(AGR_EINVAL, "snapshot: short write");
    CK(cudaMemcpyAsync(h->d_snap_list, list.data(), list.size() * 4, cudaMemcpyHostToDevice, h->snap_stream));
    const size_t per = h->snap_stage_bytes / g.rec_bytes;
    g.stage = h->d_snap_stage;
    for (size_t j = 0; j < list.size(); j += per) {
        const size_t n = std::min(per, list.size() - j);
        g.list = h->d_snap_list + j;
        agr_launch_snap_blocks(g, (uint32_t)n, true, h->snap_stream);
        CK(cudaGetLastError());
        TRY(dump_online(h, f, h->d_snap_stage, snap_blocks_bytes(g, list.data() + j, n)));
    }
    return 0;
}
// AGR_CFG_DELTA_SNAPSHOT: writes a delta on the chain's last file, or a full file when there is no chain, path is one of its
// files, or the deltas would outgrow a full file (hd, the digest and the dirty bits are what the compare cut left)
static int snap_write_chain(agr_handle* h, FILE* f, const char* path, const snap_header& hd, const std::vector<char>& agents, uint64_t bound) {
    unsigned long long digest[2];
    memcpy(digest, h->h_snap_bits + 16, 16);
    const uint32_t* bits = reinterpret_cast<const uint32_t*>(h->h_snap_bits + 32);
    const std::string at = snap_abs_path(path);
    if (at.empty()) return fail(AGR_EINVAL, std::string("snapshot: cannot resolve the directory of ") + path);
    snap_chain& ch = h->chain;
    const size_t full = snap_full_bytes(h, hd);
    bool delta = !ch.paths.empty() && std::find(ch.paths.begin(), ch.paths.end(), at) == ch.paths.end();
    delta_header dh{};
    std::vector<uint32_t> list[3];
    agr_snap_blocks g[3];
    snap_piece pc[4];
    int npc = 0;
    snap_block_tables(h, hd, true, g);
    if (delta) {
        const snap_header& b = ch.base;
        const bool var = (hd.flags & AGR_CFG_VARLEN) != 0;
        memcpy(dh.magic, "AGRDELT1", 8);
        dh.cut = hd;
        memcpy(dh.parent_digest, ch.digest, 16); memcpy(dh.digest, digest, 16);
        dh.block_rows = SNAP_BLOCK_ROWS; dh.log_block = SNAP_LOG_BLOCK;
        // appended since the parent's cut: from the first row (byte) it did not hold yet, clipped to this cut's window
        dh.rows_hi = var ? hd.vused : hd.rows_used;
        dh.rows_lo = std::min(dh.rows_hi, std::max(var ? b.vused : ch.base_bound, var ? hd.vtail : hd.tail));
        dh.resp_hi = hd.resp_used;
        dh.resp_lo = std::min(dh.resp_hi, std::max(b.resp_used, hd.resp_tail));
        dh.parent_path_len = (uint32_t)ch.paths.back().size();
        dh.file_bytes = sizeof dh + dh.parent_path_len + agents.size();
        npc = snap_delta_pieces(h, dh, pc);
        for (int j = 0; j < npc; ++j) dh.file_bytes += pc[j].bytes;
        // dirty blocks, and every block that reaches past what the parent's cut held (the shadow has nothing of it there)
        agr_snap_blocks pg[3];
        snap_block_tables(h, b, true, pg);
        for (int t = 0; t < 3; ++t) {
            const uint32_t* tb = bits + h->snap_bit_off[t];
            const uint64_t first_new = pg[t].rows / pg[t].block_rows;
            for (uint64_t k = 0; k * g[t].block_rows < g[t].rows; ++k)
                if (k >= first_new || ((tb[k >> 5] >> (k & 31)) & 1u)) list[t].push_back((uint32_t)k);
            dh.n_blocks[t] = list[t].size();
            dh.file_bytes += 4 * list[t].size() + snap_blocks_bytes(g[t], list[t].data(), list[t].size());
        }
        delta = ch.delta_bytes + dh.file_bytes <= full;              // else a full file: a restore reads at most ~2 full files
    }
    if (!delta) {
        TRY(snap_write_full(h, f, hd, agents, dump_online, h->d_shadow));
        ch = snap_chain{};
        ch.full_bytes = full;
    } else {
        const std::string& parent = ch.paths.back();
        if (fwrite(&dh, sizeof dh, 1, f) != 1 || fwrite(parent.data(), 1, parent.size(), f) != parent.size() ||
            fwrite(agents.data(), 1, agents.size(), f) != agents.size()) return fail(AGR_EINVAL, "snapshot: short write");
        for (int j = 0; j < npc; ++j) TRY(dump_online(h, f, pc[j].p, pc[j].bytes));
        for (int t = 0; t < 3; ++t) TRY(dump_blocks(h, f, g[t], list[t]));
        TRY(snap_drain(h, f));
        ch.delta_bytes += dh.file_bytes;
    }
    ch.paths.push_back(at);
    ch.base = hd; ch.base_bound = bound;
    memcpy(ch.digest, digest, 16);
    return 0;
}

// The handle is held only while the cut is enqueued; the file is written afterwards while every other call goes on.
static int snapshot_online(agr_handle* h, const char* path) {
    std::lock_guard<std::mutex> one(h->snap_mu);
    CK(cudaSetDevice(h->device));
    FILE* f = fopen(path, "wb");
    if (!f) return fail(AGR_EINVAL, std::string("snapshot: cannot open ") + path);
    const bool chain = (h->cfg.flags & AGR_CFG_DELTA_SNAPSHOT) != 0;
    snap_header hd{};
    std::vector<char> agents;                                  // the agent table as it was at the cut
    uint64_t bound = 0;                                        // rows below were ingested at the cut
    {
        HLock lk(h);
        snap_fill_header(h, hd);
        agents = snap_agents(h);
        bound = ingested_bound(h);
        const int rc = snap_cut_locked(h, hd, chain);
        if (rc < 0) { fclose(f); h->chain = snap_chain{}; return rc; }
        if (is_ring(h)) { h->pinned = true; h->pin_tail = h->tail; h->pin_vtail = h->vtail; h->pin_resp_tail = h->resp_tail; }
    }
    int rc = snap_read_cut(h, hd, chain);
    if (rc == 0) rc = chain ? snap_write_chain(h, f, path, hd, agents, bound) : snap_write_full(h, f, hd, agents, dump_online, h->d_shadow);
    if (cudaStreamSynchronize(h->snap_stream) != cudaSuccess && rc == 0) rc = fail(AGR_ECUDA, "snapshot: writer stream");
    h->snap_pend = 0; h->snap_cur = 0;
    { std::lock_guard<std::mutex> g(h->mu); h->pinned = false; }
    rc = snap_close(f, rc);
    if (rc != 0) h->chain = snap_chain{};                      // a file that failed is no base: the next one is full
    return rc;
}

extern "C" {
int agr_snapshot(agr_handle* h, const char* path) {
    if (!h || !path) return fail(AGR_EINVAL, "NULL argument");
    if (h->cfg.flags & AGR_CFG_ONLINE_SNAPSHOT) return snapshot_online(h, path);
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    CK(cudaStreamSynchronize(h->stream));
    FILE* f = fopen(path, "wb");
    if (!f) return fail(AGR_EINVAL, std::string("snapshot: cannot open ") + path);
    snap_header hd{};
    snap_fill_header(h, hd);
    unsigned long long lens[2] = {0, 0};
    int rc = read_log_lens(h, lens);
    hd.log_len[0] = lens[0]; hd.log_len[1] = lens[1];
    if (rc == 0) rc = snap_write_full(h, f, hd, snap_agents(h), dump_dev);
    return snap_close(f, rc);
}

// ---- restore: a full file, then the deltas of its chain, oldest first
// The agent table of a file: entry a is slot a.  An agent the engine already has (registered before the parent's cut) keeps its
// name and slot, and only its status changes; a new one is registered in table order, so that the slots match.  A delta may name
// another agent than its parent on a slot: the slot was reused between the two cuts (its agent removed before the parent's cut or
// after it, and its rows released), so the old names are forgotten first and the new ones bound to their slots.  The delta was
// written on this parent (restore_locked compares the digests first), so a name that differs can mean nothing else; a name that
// would then stand on two slots is refused.
static int restore_agents_locked(agr_handle* h, FILE* f, uint32_t n) {
    if (n > h->cfg.max_agents) return fail(AGR_ENOSPC, "agent table full");
    std::vector<std::string> names(n);
    std::vector<uint8_t> sts(n);
    for (uint32_t a = 0; a < n; ++a) {
        char name[AGR_AGENT_ID_BYTES];
        if (fread(name, 1, AGR_AGENT_ID_BYTES, f) != AGR_AGENT_ID_BYTES || fread(&sts[a], 1, 1, f) != 1) return fail(AGR_EINVAL, "restore: short read");
        name[AGR_AGENT_ID_BYTES - 1] = 0;
        names[a] = name;
    }
    if (n < h->agent_names.size()) return fail(AGR_EINVAL, "restore: the agent table of a delta does not extend its parent's");
    std::vector<uint32_t> reused;
    for (uint32_t a = 0; a < h->agent_names.size(); ++a)
        if (h->agent_names[a] != names[a]) reused.push_back(a);
    for (uint32_t a : reused) TRY(agent_forget_locked(h, a, true));
    for (uint32_t a : reused) {
        if (h->slot_of.count(names[a])) return fail(AGR_EINVAL, "restore: an agent appears twice in the agent table");
        TRY(agent_bind_locked(h, a, names[a].c_str(), AG_STATUS_REMOVED, true));
    }
    for (uint32_t a = 0; a < n; ++a) {
        const char* name = names[a].c_str();
        const uint8_t st = sts[a];
        const bool removed = (st == AG_STATUS_REMOVED), known = a < h->agent_names.size();
        if (!known || !removed) {
            const int s = set_agent_state_locked(h, name, removed ? (uint8_t)AGR_AGENT_STOPPED : st, true);
            if (s < 0) return s;
            if ((uint32_t)s != a) return fail(AGR_EINVAL, "restore: an agent appears twice in the agent table");
        }
        if (removed) { h->agent_status[a] = AG_STATUS_REMOVED; TRY(push_agent_status(h, a, AG_STATUS_REMOVED)); }
    }
    return 0;
}
// the scatter: n listed blocks of g, read from the file chunk by chunk into the staging buffer and placed into the live arrays
static int load_blocks(agr_handle* h, FILE* f, agr_snap_blocks g, uint64_t n) {
    const uint64_t nb = (g.rows + g.block_rows - 1) / g.block_rows;
    if (n > nb) return fail(AGR_EINVAL, "restore: corrupt delta (more blocks listed than its sections have)");
    std::vector<uint32_t> list(n);
    if (n && fread(list.data(), 4, n, f) != n) return fail(AGR_EINVAL, "restore: short read");
    for (size_t j = 0; j < n; ++j)
        if (list[j] >= nb || (j && list[j] <= list[j - 1])) return fail(AGR_EINVAL, "restore: corrupt delta (block list)");
    if (!n) return 0;
    CK(cudaMemcpyAsync(h->d_snap_list, list.data(), n * 4, cudaMemcpyHostToDevice, h->stream));
    const size_t per = h->snap_stage_bytes / g.rec_bytes;
    g.stage = h->d_snap_stage;
    for (size_t j = 0; j < n; j += per) {
        const size_t m = std::min<size_t>(per, n - j);
        TRY(load_dev(h, f, h->d_snap_stage, snap_blocks_bytes(g, list.data() + j, m)));   // (stream-ordered after the last scatter)
        g.list = h->d_snap_list + j;
        agr_launch_snap_blocks(g, (uint32_t)m, false, h->stream);
        CK(cudaGetLastError());
    }
    CK(cudaStreamSynchronize(h->stream));
    return 0;
}
// applies one delta (f is past its header and parent path) to the live arrays; the header fields are set by the caller
static int restore_delta_locked(agr_handle* h, FILE* f, const delta_header& dh) {
    TRY(restore_agents_locked(h, f, dh.cut.n_agents));
    snap_piece pc[4];
    for (int n = snap_delta_pieces(h, dh, pc), j = 0; j < n; ++j) TRY(load_dev(h, f, pc[j].p, pc[j].bytes));
    agr_snap_blocks g[3];
    snap_block_tables(h, dh.cut, false, g);
    for (int t = 0; t < 3; ++t) TRY(load_blocks(h, f, g[t], dh.n_blocks[t]));
    if ((uint64_t)ftello(f) != dh.file_bytes) return fail(AGR_EINVAL, "restore: corrupt delta (its sections do not add up to its size)");
    return 0;
}
// Follows the parent paths from path back to a full file: files[0] is that file, files[k] (k >= 1) the delta dh[k - 1].
static int restore_chain(const char* path, std::vector<std::string>& files, std::vector<delta_header>& dh) {
    std::string p = path;
    for (;;) {
        const std::string of = files.empty() ? "" : ", the parent of " + files.front();
        if (files.size() > 65536) return fail(AGR_EINVAL, "restore: the chain of parents does not end in a full file");
        FILE* f = fopen(p.c_str(), "rb");
        if (!f) return fail(AGR_EINVAL, "restore: cannot open " + p + of);
        char magic[8] = {0};
        const bool got = fread(magic, 1, 8, f) == 8;
        if (got && memcmp(magic, "AGRSNAP3", 8) == 0) { fclose(f); files.insert(files.begin(), p); return 0; }
        if (!got || memcmp(magic, "AGRDELT1", 8) != 0) { fclose(f); return fail(AGR_EINVAL, files.empty() ? "restore: not a snapshot" : "restore: " + p + of + ", is not a snapshot"); }
        delta_header d{};
        struct stat st{};
        rewind(f);
        const bool ok = fread(&d, sizeof d, 1, f) == 1 && fstat(fileno(f), &st) == 0;
        std::string parent(ok && d.parent_path_len <= PATH_MAX ? d.parent_path_len : 0, '\0');
        const bool named = ok && d.parent_path_len && d.parent_path_len <= PATH_MAX && fread(&parent[0], 1, parent.size(), f) == parent.size();
        fclose(f);
        if (!ok || (uint64_t)st.st_size < d.file_bytes) return fail(AGR_EINVAL, "restore: " + p + of + " is shorter than its header says (truncated)");
        const bool var = (d.cut.flags & AGR_CFG_VARLEN) != 0;
        if (!named || d.block_rows != SNAP_BLOCK_ROWS || d.log_block != SNAP_LOG_BLOCK || d.rows_lo > d.rows_hi ||
            d.rows_hi != (var ? d.cut.vused : d.cut.rows_used) || d.resp_lo > d.resp_hi || d.resp_hi != d.cut.resp_used ||
            d.rows_hi - d.rows_lo > (var ? d.cut.vcap : d.cut.slab_rows) || d.resp_hi - d.resp_lo > d.cut.resp_cap)
            return fail(AGR_EINVAL, "restore: " + p + of + " is not a valid delta");
        files.insert(files.begin(), p);
        dh.insert(dh.begin(), d);
        p = parent;
    }
}
// The state of the whole chain into h: the full file (f, past its header), each delta after a check that the state so far
// is its parent's cut (digest), then the header fields, the log lengths, the dedupe index and the chain an
// AGR_CFG_DELTA_SNAPSHOT engine continues, once.  index = false leaves the dedupe index out (the source engine of a relocation,
// whose rows only move).
static int restore_locked(agr_handle* h, FILE* f, const snap_header& full, const std::vector<std::string>& files, const std::vector<delta_header>& dh,
                          bool index = true) {
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    TRY(restore_agents_locked(h, f, full.n_agents));
    TRY(snap_sections(h, full, f, load_dev));
    const bool chain = (h->cfg.flags & AGR_CFG_DELTA_SNAPSHOT) != 0;
    if (!dh.empty()) TRY(snap_delta_alloc(h));
    const snap_header* at = &full;
    unsigned long long dg[2] = {0, 0};
    for (size_t k = 0; k < dh.size(); ++k) {
        TRY(snap_digest_locked(h, *at, false, dg));
        if (memcmp(dg, dh[k].parent_digest, 16) != 0)
            return fail(AGR_EINVAL, "restore: " + files[k] + " is not the snapshot " + files[k + 1] + " was written on (digest differs): was it replaced?");
        FILE* g = fopen(files[k + 1].c_str(), "rb");
        if (!g) return fail(AGR_EINVAL, "restore: cannot open " + files[k + 1]);
        int rc = fseeko(g, (off_t)(sizeof(delta_header) + dh[k].parent_path_len), SEEK_SET) == 0 ? restore_delta_locked(h, g, dh[k])
                                                                                                : fail(AGR_EINVAL, "restore: short read");
        fclose(g);
        TRY(rc);
        at = &dh[k].cut;
    }
    const snap_header& hd = *at;
    const size_t R = snap_rows(hd);
    h->resp_used = hd.resp_used; h->resp_tail = hd.resp_tail; h->expired_total = hd.expired_total;
    unsigned long long lens[2] = {hd.log_len[0], hd.log_len[1]};
    if (cudaMemcpy(h->d.log_len, lens, sizeof lens, cudaMemcpyHostToDevice) != cudaSuccess) return fail(AGR_ECUDA, "restore: log_len");
    h->rows_used = hd.rows_used; h->vused = hd.vused; h->vtail = hd.vtail; h->scan_lo = hd.scan_lo;
    h->d.shard_id = hd.shard; h->d.id_gen = hd.gen; h->tail = hd.tail; h->released_total = hd.released_total; sync_window(h);
    h->d.idx_base = h->tail;
    h->agent_gen++;                                   // another window: which removed agents' slots it holds is scanned afresh
    TRY(chunk_bounds_unknown(h));
    if (index && !(hd.flags & AGR_CFG_MINT_IDS) && R) {   // hash-id mode: rebuild the dedupe index from the restored rows
        if (is_ring(h)) TRY(ring_reindex_locked(h));     // a ring: the index a release leaves (rows that hold a record)
        else {                                            // append-only: the index never shrinks, so every row K1 stored is in it
            agr_launch_reindex(h->d, (uint32_t)R, h->stream);
            h->k1_launches += 1;
        }
        if (cudaStreamSynchronize(h->stream) != cudaSuccess) return fail(AGR_ECUDA, "restore: reindex");
    }
    if (chain || !dh.empty()) {
        TRY(snap_digest_locked(h, hd, chain, dg));    // an AGR_CFG_DELTA_SNAPSHOT engine: also seeds the shadow
        if (!dh.empty() && memcmp(dg, dh.back().digest, 16) != 0)
            return fail(AGR_EINVAL, "restore: the state after " + files.back() + " differs from the one it was written from (digest)");
    }
    if (chain) {
        snap_chain& ch = h->chain;
        ch = snap_chain{};
        ch.paths = files;
        ch.paths.back() = snap_abs_path(files.back());   // (the parents' paths are absolute already)
        ch.full_bytes = snap_full_bytes(h, full);
        for (const auto& d : dh) ch.delta_bytes += d.file_bytes;
        ch.base = hd; ch.base_bound = hd.rows_used;
        memcpy(ch.digest, dg, 16);
        if (ch.paths.back().empty()) ch = snap_chain{};
    }
    return 0;
}

// ---- restore into other capacities (DESIGN.md section 5)
// Whether the restored state of the last cut s has to move: a ring snapshot into other ring capacities, an append-only
// snapshot into a ring, or either into a ring of the other record form.  Every other restore loads the file in place.
static bool restore_relocates(const agr_handle* h, const snap_header& s) {
    if ((s.flags ^ h->cfg.flags) & AGR_CFG_VARLEN) return true;     // (agr_restore lets the form differ only into a ring)
    if (!(s.flags & AGR_CFG_RING)) return is_ring(h);
    return s.slab_rows != h->cfg.slab_rows || s.resp_cap != h->resp_cap || ((s.flags & AGR_CFG_VARLEN) && s.vcap != h->vcap);
}
static std::string relocation_enomem() {
    return "restore: relocating into other capacities holds the snapshot's engine and the configured one on the device at once, "
           "and both do not fit: " + g_err;
}
// Moves the state of the source engine s (the last cut hd, restored in s's own geometry and record form) into h (a ring): the
// window's rows to row id mod h's slab_rows, the live rows' record and response bytes packed from byte 0, the logs remapped.
// The records take h's form: 512 B rows become compact records, records become 512 B rows (AGR_EINVAL for one longer than
// that).  The header fields other than the byte rings' cursors stay as hd has them.
static int relocate_locked(agr_handle* h, agr_handle* s, const snap_header& hd) {
    HLock lk(h);
    CK(cudaSetDevice(h->device));
    CK(cudaStreamSynchronize(s->stream));
    for (uint32_t a = 0; a < (uint32_t)s->agent_names.size(); ++a) {   // the agent table, slot for slot (as restore_agents_locked)
        const bool removed = s->agent_status[a] == AG_STATUS_REMOVED;
        const int slot = set_agent_state_locked(h, s->agent_names[a].c_str(), removed ? (uint8_t)AGR_AGENT_STOPPED : s->agent_status[a], true);
        if (slot < 0) return slot;
        if ((uint32_t)slot != a) return fail(AGR_EINVAL, "restore: an agent appears twice in the agent table");
        if (removed) { h->agent_status[a] = AG_STATUS_REMOVED; TRY(push_agent_status(h, a, AG_STATUS_REMOVED)); }
    }
    const bool var_s = (hd.flags & AGR_CFG_VARLEN) != 0, var_t = (h->cfg.flags & AGR_CFG_VARLEN) != 0;
    const uint64_t n = hd.rows_used - hd.tail;
    h->rows_used = hd.rows_used; h->tail = hd.tail; h->released_total = hd.released_total; h->scan_lo = hd.scan_lo;
    h->expired_total = hd.expired_total; h->d.shard_id = hd.shard; h->d.id_gen = hd.gen;
    sync_window(h);                                            // h->d now has the target's window and ring geometry
    agr_relayout p{};
    p.s = s->d; p.t = h->d; p.n = n;
    p.sw = agr_relayout_words{s->d_resp_off, s->d_resp_len, s->d_resp_hlen, s->d_err_off, s->d_err_len};
    p.tw = agr_relayout_words{h->d_resp_off, h->d_resp_len, h->d_resp_hlen, h->d_err_off, h->d_err_len};
    {   // scratch of the move: allocated with the source engine, freed with it
        const size_t tiles = std::max<uint32_t>(agr_relayout_tiles(n), 1), rows = std::max<uint64_t>(n, 1);
        const int rc = [&]() {
            TRY(dev_alloc(s, &p.tile_sum, 2 * tiles, false));
            TRY(dev_alloc(s, &p.totals, (size_t)4, false));
            if (var_s || var_t) { TRY(dev_alloc(s, &p.vseg_dst, rows, false)); TRY(dev_alloc(s, &p.vseg_src, rows, false)); TRY(dev_alloc(s, &p.vseg_len, rows, false)); }
            TRY(dev_alloc(s, &p.rseg_dst, 2 * rows, false)); TRY(dev_alloc(s, &p.rseg_src, 2 * rows, false)); TRY(dev_alloc(s, &p.rseg_len, 2 * rows, false));
            return 0;
        }();
        if (rc == AGR_ENOMEM) return fail(rc, relocation_enomem());
        TRY(rc);
    }
    CK(cudaMemsetAsync(p.totals + 2, 0, 8, h->stream));        // k_rl_count's oversized records: none yet, least ~0
    CK(cudaMemsetAsync(p.totals + 3, 0xff, 8, h->stream));
    TRY(op_time_begin(h, 4));
    agr_launch_relayout_count(p, h->stream);
    CK(cudaGetLastError());
    unsigned long long tot[4];
    TRY(d2h_staged(h, tot, p.totals, sizeof tot, h->h_small));
    if (var_s && !var_t && tot[2])
        return fail(AGR_EINVAL, "restore: " + std::to_string(tot[2]) + " live records are longer than the 512 B rows of the fixed "
                                "record form, so they cannot be converted (the first: row " + std::to_string(hd.tail + (tot[3] >> 32)) +
                                    ", " + std::to_string(tot[3] & 0xffffffffull) + " B)");
    if (var_t && tot[0] > h->vcap)
        return fail(AGR_ENOSPC, "restore: the live records take " + std::to_string(tot[0]) + " B, more than vslab_bytes (" +
                                    std::to_string(h->vcap) + " B) by " + std::to_string(tot[0] - h->vcap) + " B");
    if (tot[1] > h->resp_cap)
        return fail(AGR_ENOSPC, "restore: the live response and error bytes take " + std::to_string(tot[1]) + " B, more than resp_bytes (" +
                                    std::to_string(h->resp_cap) + " B) by " + std::to_string(tot[1] - h->resp_cap) + " B");
    agr_launch_relayout_rows(p, h->stream);
    if (var_t) agr_launch_relayout_bytes(s->d.slab, h->d.slab, p.vseg_dst, p.vseg_src, p.vseg_len, n, tot[0], h->stream);
    agr_launch_relayout_bytes(s->d_resp, h->d_resp, p.rseg_dst, p.rseg_src, p.rseg_len, 2 * n, tot[1], h->stream);
    agr_launch_relayout_log(s->d, h->d, s->d.completed_log, h->d.completed_log, hd.log_len[0], h->stream);
    agr_launch_relayout_log(s->d, h->d, s->d.failed_log, h->d.failed_log, hd.log_len[1], h->stream);
    CK(cudaGetLastError());
    TRY(op_time_end(h, 4));
    const unsigned long long lens[2] = {hd.log_len[0], hd.log_len[1]};
    CK(cudaMemcpyAsync(h->d.log_len, lens, sizeof lens, cudaMemcpyHostToDevice, h->stream));
    h->vused = var_t ? tot[0] : 0; h->vtail = 0;
    h->resp_used = tot[1]; h->resp_tail = 0;
    h->d.idx_base = h->tail;
    TRY(chunk_bounds_unknown(h));
    if (!(hd.flags & AGR_CFG_MINT_IDS) && n) TRY(ring_reindex_locked(h));   // hash-id mode: the index a release leaves
    if (cudaStreamSynchronize(h->stream) != cudaSuccess) return fail(AGR_ECUDA, "restore: relocation");
    return 0;
}
// The relocating restore into h: the file (f, past its header) and its deltas go into a source engine of the snapshot's own
// geometry and record form, which is then moved into h and freed.  The source engine is bare: no single-request front end, no snapshot shadows,
// no dedupe index (created in minted-id form, so that it allocates none; nothing of the id mode is in the arrays it holds).
static int restore_relocate(agr_handle* h, FILE* f, const snap_header& full, const std::vector<std::string>& files, const std::vector<delta_header>& dh) {
    const snap_header& last = dh.empty() ? full : dh.back().cut;
    const bool ring = (last.flags & AGR_CFG_RING) != 0;
    const uint64_t window = last.rows_used - last.tail;
    if (window > h->cfg.slab_rows)
        return fail(AGR_ENOSPC, "restore: the live window of the snapshot holds " + std::to_string(window) + " rows, more than slab_rows (" +
                                    std::to_string(h->cfg.slab_rows) + ") by " + std::to_string(window - h->cfg.slab_rows));
    uint64_t logs = 1;
    for (size_t k = 0; k <= dh.size(); ++k) {
        const snap_header& s = k ? dh[k - 1].cut : full;
        if (s.log_len[0] > h->d.log_cap || s.log_len[1] > h->d.log_cap) return fail(AGR_ENOSPC, "restore: snapshot larger than the configured capacities");
        logs = std::max<uint64_t>(logs, std::max(s.log_len[0], s.log_len[1]));
    }
    agr_config sc{};
    sc.flags = AGR_CFG_PERSISTENCE | AGR_CFG_MINT_IDS | (last.flags & (AGR_CFG_VARLEN | AGR_CFG_RING));
    sc.device = h->device; sc.id_secret = last.id_secret; sc.max_agents = h->cfg.max_agents; sc.log_entries = logs;
    sc.max_batch = 1u << 16;                                   // (sizes the staging buffers the load streams through)
    if (ring) { sc.slab_rows = last.slab_rows; sc.vslab_bytes = last.vcap; sc.resp_bytes = last.resp_cap; }
    else {                                                     // append-only: what the file holds (the last cut holds the most)
        sc.slab_rows = std::max<uint64_t>(last.rows_used, 1);
        sc.vslab_bytes = std::max<uint64_t>(last.vused, 16); sc.resp_bytes = std::max<uint64_t>(last.resp_used, 16);
    }
    agr_handle* s = nullptr;
    int rc = agr_create(&sc, &s);
    if (rc == AGR_ENOMEM) return fail(rc, relocation_enomem());
    TRY(rc);
    rc = restore_locked(s, f, full, files, dh, false);
    if (rc == 0) rc = relocate_locked(h, s, last);
    const std::string keep = g_err;
    agr_destroy(s);
    g_err = keep;
    return rc;
}

int agr_restore(const agr_config* cfg, const char* path, agr_handle** out) {
    if (!cfg || !path || !out) return fail(AGR_EINVAL, "NULL argument");
    *out = nullptr;
    std::vector<std::string> files;
    std::vector<delta_header> dh;
    TRY(restore_chain(path, files, dh));
    FILE* f = fopen(files[0].c_str(), "rb");
    if (!f) return fail(AGR_EINVAL, "restore: cannot open " + files[0]);
    snap_header hd{};
    if (fread(&hd, sizeof hd, 1, f) != 1 || memcmp(hd.magic, "AGRSNAP3", 8) != 0) { fclose(f); return fail(AGR_EINVAL, "restore: not a snapshot"); }
    agr_config c = *cfg;
    if (c.flags == 0) c.flags = AGR_CFG_PERSISTENCE;
    const uint32_t mode_bits = AGR_CFG_MINT_IDS | AGR_CFG_VARLEN | AGR_CFG_RING;
    uint32_t form = (hd.flags & AGR_CFG_RING) ? mode_bits : mode_bits & ~AGR_CFG_RING;   // (append-only into a ring relocates)
    if (c.flags & AGR_CFG_RING) form &= ~AGR_CFG_VARLEN;                                  // (into a ring of the other form converts)
    if ((c.flags & form) != (hd.flags & form)) { fclose(f); return fail(AGR_EINVAL, "restore: id mode / record form differ from the snapshot"); }
    if (c.id_secret == 0) c.id_secret = hd.id_secret;
    if (c.id_secret != hd.id_secret) { fclose(f); return fail(AGR_EINVAL, "restore: id_secret differs from the snapshot"); }
    for (size_t k = 0; k < dh.size(); ++k)
        if ((dh[k].cut.flags & mode_bits) != (hd.flags & mode_bits) || dh[k].cut.id_secret != hd.id_secret || dh[k].cut.slab_rows != hd.slab_rows) {
            fclose(f);
            return fail(AGR_EINVAL, "restore: " + files[k + 1] + " and its full file " + files[0] + " come from different engines");
        }
    agr_handle* h = nullptr;
    int rc = agr_create(&c, &h);
    if (rc < 0) { fclose(f); return rc; }
    auto bail = [&](int r) { std::string keep = g_err; fclose(f); agr_destroy(h); g_err = keep; return r; };
    if (restore_relocates(h, dh.empty() ? hd : dh.back().cut)) {
        if ((rc = restore_relocate(h, f, hd, files, dh)) < 0) return bail(rc);
        fclose(f);
        *out = h;
        return 0;
    }
    auto fits = [&](const snap_header& s) -> int {
        const bool snap_ring = (s.flags & AGR_CFG_RING) != 0;
        if (!snap_ring && s.resp_used > h->resp_cap) return fail(AGR_ENOSPC, "restore: stored responses larger than resp_bytes");
        if (snap_ring && s.resp_cap != h->resp_cap) return fail(AGR_EINVAL, "restore: a ring snapshot needs the same resp_bytes");
        if (snap_ring && (s.flags & AGR_CFG_VARLEN) && s.vcap != h->vcap) return fail(AGR_EINVAL, "restore: a ring snapshot needs the same vslab_bytes");
        if (snap_ring && s.slab_rows != h->cfg.slab_rows) return fail(AGR_EINVAL, "restore: a ring snapshot needs the same slab_rows (rows live at logical mod slab_rows)");
        if ((!snap_ring && s.rows_used > h->cfg.slab_rows) || s.log_len[0] > h->d.log_cap || s.log_len[1] > h->d.log_cap || ((s.flags & AGR_CFG_VARLEN) && !snap_ring && s.vused > h->vcap))
            return fail(AGR_ENOSPC, "restore: snapshot larger than the configured capacities");
        return 0;
    };
    if ((rc = fits(hd)) < 0) return bail(rc);
    for (const auto& d : dh) if ((rc = fits(d.cut)) < 0) return bail(rc);
    if ((rc = restore_locked(h, f, hd, files, dh)) < 0) return bail(rc);
    fclose(f);
    *out = h;
    return 0;
}
}  // extern "C"
