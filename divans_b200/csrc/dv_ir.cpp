// dv_ir.cpp -- IR text front-end (SURVEY 8f-3): the reference's textual intermediate representation
// (src/bin/divans.rs:191-483, one command per line, fields separated by single spaces) parsed into the binary
// command-list blob ("DVCL", include/divans_b200.h) that divans_b200_encode_cmds_batch_host consumes.
// Host-side only; the entropy coding of the parsed commands runs on the GPU.
#include <stdint.h>
#include <string.h>

#include <string_view>
#include <vector>

#include "../../include/divans_b200.h"

namespace {

using sv = std::string_view;

struct Cmd { uint32_t type, a, b, c, d; };
struct PredMode {
    uint8_t pred_mode = 0, is_adv = 0, has_speeds = 1;
    uint16_t speed[3][2][2] = {};          // [context-map | stride | combined][low, high][inc, max]
    uint16_t lit_len = 0, dist_len = 0;
    uint8_t lit_map[16384] = {}, dist_map[1024] = {}, mixing[8192] = {};
};

bool number(sv t, long long &v) {
    if (t.empty() || t.size() > 18) return false;
    size_t i = 0; bool neg = false;
    if (t[0] == '-') { neg = true; i = 1; if (t.size() == 1) return false; }
    long long r = 0;
    for (; i < t.size(); i++) { if (t[i] < '0' || t[i] > '9') return false; r = r * 10 + (t[i] - '0'); }
    v = neg ? -r : r;
    return true;
}
int hex(char ch) {
    if (ch >= '0' && ch <= '9') return ch - '0';
    if (ch >= 'a' && ch <= 'f') return ch - 'a' + 10;
    if (ch >= 'A' && ch <= 'F') return ch - 'A' + 10;
    return -1;
}
// str::split(' '): every single space delimits, empty fields are kept
void split(sv line, std::vector<sv> &out) {
    out.clear();
    size_t p = 0;
    for (;;) {
        size_t q = line.find(' ', p);
        if (q == sv::npos) { out.push_back(line.substr(p)); return; }
        out.push_back(line.substr(p, q - p));
        p = q + 1;
    }
}

struct Parser {
    std::vector<Cmd> cmds;
    std::vector<PredMode> pms;
    std::vector<uint8_t> lits;
    int window = 0;

    // numbers following a keyword, up to the first non-number field
    template <typename F> static bool run(const std::vector<sv> &t, size_t from, F &&each) {
        for (size_t j = from; j < t.size(); j++) { long long v; if (!number(t[j], v)) break; if (!each(v)) return false; }
        return true;
    }
    bool prediction(const std::vector<sv> &t) {
        if (t.size() < 2) return false;
        cmds.push_back({7, (uint32_t)pms.size(), 0, 0, 0});
        pms.emplace_back();
        PredMode &pm = pms.back();
        if (t[1] == "lsb6") pm.pred_mode = 0; else if (t[1] == "msb6") pm.pred_mode = 1;
        else if (t[1] == "utf8") pm.pred_mode = 2; else if (t[1] == "sign") pm.pred_mode = 3; else return false;
        static const char *const speed_keys[3][2] = {{"cmspeedinc", "cmspeedmax"}, {"stspeedinc", "stspeedmax"}, {"mxspeedinc", "mxspeedmax"}};
        for (size_t k = 2; k < t.size(); k++) {
            if (t[k] == "lcontextmap") {
                if (!run(t, k + 1, [&](long long v) { if (v < 0 || v > 255) return false; if (pm.lit_len < 16384) pm.lit_map[pm.lit_len++] = (uint8_t)v; return true; })) return false;
            } else if (t[k] == "dcontextmap") {
                if (!run(t, k + 1, [&](long long v) { if (v < 0 || v > 255) return false; if (pm.dist_len < 1024) pm.dist_map[pm.dist_len++] = (uint8_t)v; return true; })) return false;
            } else if (t[k] == "mixingvalues") {
                uint32_t off = 0;
                if (!run(t, k + 1, [&](long long v) { if (off >= 8192 || v < 0 || v > 8) return false; pm.mixing[off++] = (uint8_t)v; return true; })) return false;
            } else {
                for (int w = 0; w < 3; w++) for (int im = 0; im < 2; im++) if (t[k] == speed_keys[w][im]) {
                    for (size_t j = 0; j < 2 && k + 1 + j < t.size(); j++) {
                        long long v; if (!number(t[k + 1 + j], v)) break;
                        if (v < 0 || v > 16384) return false;
                        pm.speed[w][j][im] = (uint16_t)v;
                    }
                }
            }
        }
        return true;
    }
    bool line(sv ln, std::vector<sv> &t) {
        split(ln, t);
        if (t.empty()) return true;
        const sv op = t[0];
        long long v;
        if (op == "window") { if (t.size() > 1 && number(t[1], v)) window = (int)v; return true; }
        if (op == "prediction") return prediction(t);
        if (op == "ctype" || op == "ltype" || op == "dtype") {
            if (t.size() < 2 || !number(t[1], v)) return false;
            Cmd c = {op[0] == 'l' ? 4u : (op[0] == 'c' ? 5u : 6u), (uint32_t)(uint8_t)v, 0, 0, 0};
            if (op[0] == 'l' && t.size() >= 3) { long long sv_; if (!number(t[2], sv_) || sv_ > 8) return false; c.b = (uint32_t)sv_; }
            cmds.push_back(c);
            return true;
        }
        if (op == "copy") {
            long long len, dist;
            if (t.size() < 4 || !number(t[1], len) || t[2] != "from" || !number(t[3], dist)) return false;
            if (len != 0) cmds.push_back({1, (uint32_t)dist, (uint32_t)len, 0, 0});
            return true;
        }
        if (op == "dict") {
            long long flen, wl, wi;
            if (t.size() < 6 || !number(t[1], flen) || t[2] != "word") return false;
            const size_t comma = t[3].find(',');
            if (comma == sv::npos || !number(t[3].substr(0, comma), wl) || !number(t[3].substr(comma + 1), wi)) return false;
            for (size_t k = 5; k < t.size(); k++) if (t[k - 1] == "func") {
                long long tr; if (!number(t[k], tr)) return false;
                cmds.push_back({2, (uint32_t)wi, (uint32_t)(uint8_t)wl, (uint32_t)(uint8_t)tr, (uint32_t)(uint8_t)flen});
                return true;
            }
            return false;
        }
        if (op == "insert" || op == "rndins") {
            long long len;
            if (t.size() < 2 || !number(t[1], len)) return false;
            if (len == 0) return true;
            if (len < 0 || t.size() < 3 || t[2].size() != (size_t)len * 2) return false;
            const size_t off = lits.size();
            lits.resize(off + (size_t)len);
            for (long long k = 0; k < len; k++) {
                const int hi = hex(t[2][2 * k]), lo = hex(t[2][2 * k + 1]);
                if (hi < 0 || lo < 0) return false;
                lits[off + k] = (uint8_t)((hi << 4) | lo);
            }
            cmds.push_back({3, (uint32_t)off, (uint32_t)len, op == "rndins" ? 1u : 0u, 0});
            return true;
        }
        return false;
    }
};

}  // namespace

extern "C" DivansResult divans_b200_ir_to_cmds(const char *ir_text, size_t ir_len, uint8_t *out, size_t out_cap, size_t *blob_len,
                                               int32_t *window_size) {
    if (!ir_text || !blob_len) return DIVANS_FAILURE;
    Parser ps;
    std::vector<sv> toks;
    const sv text(ir_text, ir_len);
    size_t p = 0;
    while (p < text.size()) {
        size_t e = text.find('\n', p);
        if (e == sv::npos) e = text.size();
        sv ln = text.substr(p, e - p);
        if (!ln.empty() && ln.back() == '\r') ln.remove_suffix(1);
        p = e + 1;
        if (ln.empty()) continue;
        if (!ps.line(ln, toks)) return DIVANS_FAILURE;
    }
    constexpr size_t PM_BYTES = 32 + 16384 + 1024 + 8192;
    const size_t need = 32 + ps.cmds.size() * 20 + ps.pms.size() * PM_BYTES + ps.lits.size();
    *blob_len = need;
    if (window_size) *window_size = ps.window;
    if (!out || out_cap < need) return DIVANS_NEEDS_MORE_OUTPUT;
    uint8_t *w = out;
    const uint32_t hdr[8] = {0x4c435644u, 1u, (uint32_t)ps.cmds.size(), (uint32_t)ps.pms.size(), (uint32_t)ps.lits.size(), (uint32_t)ps.window, 0u, 0u};
    memcpy(w, hdr, 32); w += 32;
    if (!ps.cmds.empty()) memcpy(w, ps.cmds.data(), ps.cmds.size() * 20);
    w += ps.cmds.size() * 20;
    for (const PredMode &pm : ps.pms) {
        uint8_t h[32] = {pm.pred_mode, pm.is_adv, pm.has_speeds, 0};
        uint16_t sp[12];
        for (int wch = 0; wch < 3; wch++) for (int k = 0; k < 2; k++) for (int im = 0; im < 2; im++) sp[wch * 4 + k * 2 + im] = pm.speed[wch][k][im];
        memcpy(h + 4, sp, 24);
        memcpy(h + 28, &pm.lit_len, 2); memcpy(h + 30, &pm.dist_len, 2);
        memcpy(w, h, 32); w += 32;
        memcpy(w, pm.lit_map, 16384); w += 16384;
        memcpy(w, pm.dist_map, 1024); w += 1024;
        memcpy(w, pm.mixing, 8192); w += 8192;
    }
    if (!ps.lits.empty()) memcpy(w, ps.lits.data(), ps.lits.size());
    return DIVANS_SUCCESS;
}

// ---------------------------------------------------------------------------------------------------------------
// Command generator for benchmarks and tools (ours, not a reference component): a deterministic hash-chain LZ77 (by default
// greedy with minimum match 4; window 2^window - 16, no dictionary words) that turns raw bytes into a DVCL command list -- one
// PredictionMode command (64-entry identity context map, one mixing value, like raw_to_cmd/mod.rs:116-143), then Literal /
// Copy commands.  SURVEY 8d calls the resulting population "Z": copy-dominated streams like the reference's default
// (brotli-driven) compressor produces.  The command SELECTION of the brotli crate stays out of scope.
// ---------------------------------------------------------------------------------------------------------------
#include <algorithm>
#include <thread>

namespace {
// The parse (include/divans_b200.h, "the LZ77 parse"): best(j) needs every position below j inserted and j not yet, so the
// chain is filled up to j on demand; the (at most three) positions the parse looks at around i are kept in a small cache.
size_t lz77_blob(const uint8_t *in, size_t n, int window, int pred_mode, int mixing_value, const divans_b200_lz77_parse &parse,
                 std::vector<uint8_t> &blob) {
    std::vector<Cmd> cmds;
    cmds.push_back({7, 0, 0, 0, 0});
    const int HB = 15;
    std::vector<int32_t> head((size_t)1 << HB, -1), prev(n + 1, -1);
    const size_t maxdist = ((size_t)1 << window) - 16;
    auto h4 = [&](size_t i) {
        uint32_t v; memcpy(&v, in + i, 4);
        return (v * 2654435761u) >> (32 - HB);
    };
    size_t ins = 0;   // positions below `ins` are in the chain
    auto insert = [&](size_t at) { if (at + 4 <= n) { const uint32_t hh = h4(at); prev[at] = head[hh]; head[hh] = (int32_t)at; } };
    size_t c_pos[4] = {SIZE_MAX, SIZE_MAX, SIZE_MAX, SIZE_MAX}, c_len[4] = {0}, c_dist[4] = {0};
    auto best = [&](size_t i, size_t &best_dist) -> size_t {
        if (c_pos[i & 3] == i) { best_dist = c_dist[i & 3]; return c_len[i & 3]; }
        size_t best_len = 0;
        best_dist = 0;
        if (i + 4 <= n) {
            while (ins < i) insert(ins++);
            int chain = 16;
            for (int32_t c = head[h4(i)]; c >= 0 && chain-- > 0 && i - (size_t)c <= maxdist; c = prev[c]) {
                size_t l = 0, lim = std::min<size_t>(n - i, 65535);
                while (l < lim && in[c + l] == in[i + l]) l++;
                if (l > best_len) { best_len = l; best_dist = i - (size_t)c; }
            }
        }
        c_pos[i & 3] = i; c_len[i & 3] = best_len; c_dist[i & 3] = best_dist;
        return best_len;
    };
    const size_t min_match = (size_t)parse.min_match;
    size_t i = 0, lit_start = 0, d1;
    while (i < n) {
        size_t best_dist;
        const size_t L = best(i, best_dist);
        bool take = L >= min_match;
        if (take && parse.lazy >= 1 && L < 32)
            take = !(best(i + 1, d1) > L || (parse.lazy == 2 && best(i + 2, d1) > L + 1));
        if (take) {
            if (i > lit_start) cmds.push_back({3, (uint32_t)lit_start, (uint32_t)(i - lit_start), 0, 0});
            cmds.push_back({1, (uint32_t)best_dist, (uint32_t)L, 0, 0});
            i += L;
            lit_start = i;
        } else i++;
    }
    if (n > lit_start) cmds.push_back({3, (uint32_t)lit_start, (uint32_t)(n - lit_start), 0, 0});
    constexpr size_t PM_BYTES = 32 + 16384 + 1024 + 8192;
    blob.assign(32 + cmds.size() * 20 + PM_BYTES + n, 0);
    uint8_t *w = blob.data();
    const uint32_t hdr[8] = {0x4c435644u, 1u, (uint32_t)cmds.size(), 1u, (uint32_t)n, (uint32_t)window, 0u, 0u};
    memcpy(w, hdr, 32); w += 32;
    memcpy(w, cmds.data(), cmds.size() * 20); w += cmds.size() * 20;
    w[0] = (uint8_t)pred_mode; w[2] = 1; w[28] = 64; w[30] = 4;
    for (int k = 0; k < 64; k++) w[32 + k] = (uint8_t)k;
    for (int k = 0; k < 4; k++) w[32 + 16384 + k] = (uint8_t)k;
    memset(w + 32 + 16384 + 1024, mixing_value, 8192);
    w += PM_BYTES;
    if (n) memcpy(w, in, n);   // the literal pool is the raw stream itself: a Literal's offset is its position
    return blob.size();
}
}  // namespace

// n raw buffers -> n DVCL blobs written back to back at blob_off[i] (16-byte aligned) of `out`; blob_len[i] receives the sizes.
// With out == NULL or out_cap too small the call returns DIVANS_NEEDS_MORE_OUTPUT and *total receives the size needed.
// `parse` NULL or outside min_match 4..32, lazy 0..2: DIVANS_FAILURE, nothing written.
extern "C" DivansResult divans_b200_lz77_cmds_batch_parse(size_t n, const uint8_t *in, const uint64_t *in_off, const uint64_t *in_len, int32_t window,
                                                          int32_t pred_mode, int32_t mixing_value, uint8_t *out, size_t out_cap, uint64_t *blob_off,
                                                          uint64_t *blob_len, size_t *total, int32_t n_threads, const divans_b200_lz77_parse *parse) {
    if (!in || !in_off || !in_len || !blob_off || !blob_len || !total || window < 10 || window > 24) return DIVANS_FAILURE;
    if (!parse || parse->min_match < 4 || parse->min_match > 32 || parse->lazy < 0 || parse->lazy > 2) return DIVANS_FAILURE;
    const divans_b200_lz77_parse ps = *parse;
    std::vector<std::vector<uint8_t>> blobs(n);
    if (n_threads < 1) n_threads = 1;
    std::vector<std::thread> th;
    for (int t = 0; t < n_threads; t++)
        th.emplace_back([&, t]() { for (size_t i = (size_t)t; i < n; i += (size_t)n_threads) lz77_blob(in + in_off[i], (size_t)in_len[i], window, pred_mode, mixing_value, ps, blobs[i]); });
    for (auto &x : th) x.join();
    size_t pos = 0;
    for (size_t i = 0; i < n; i++) { blob_off[i] = pos; blob_len[i] = blobs[i].size(); pos += (blobs[i].size() + 15) & ~(size_t)15; }
    *total = pos;
    if (!out || out_cap < pos) return DIVANS_NEEDS_MORE_OUTPUT;
    for (size_t i = 0; i < n; i++) memcpy(out + blob_off[i], blobs[i].data(), blobs[i].size());
    return DIVANS_SUCCESS;
}

extern "C" DivansResult divans_b200_lz77_cmds_batch(size_t n, const uint8_t *in, const uint64_t *in_off, const uint64_t *in_len, int32_t window,
                                                    int32_t pred_mode, int32_t mixing_value, uint8_t *out, size_t out_cap, uint64_t *blob_off,
                                                    uint64_t *blob_len, size_t *total, int32_t n_threads) {
    const divans_b200_lz77_parse greedy = DIVANS_B200_LZ77_PARSE_DEFAULT;
    return divans_b200_lz77_cmds_batch_parse(n, in, in_off, in_len, window, pred_mode, mixing_value, out, out_cap, blob_off, blob_len, total,
                                             n_threads, &greedy);
}
