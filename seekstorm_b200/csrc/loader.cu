// loader.cu — parse the reference's on-disk shard files straight into the GPU index (SURVEY.md §8f row 1, §8a rows a3 / a9).
//
//   index.bin  (written by commit.rs:203-467, read back by open_shard index.rs:3253-3516; all integers little endian)
//     [u16 format major][u16 minor]                                           INDEX_HEADER_SIZE = 4   (index.rs:103)
//     per level (= one 64K-doc block of the shard):
//       [u16 longest_field_id]            first level only                                        (index.rs:3326-3345)
//       [indexed fields x 65536 B]        byte4 document-length codes                               (index.rs:3362-3380)
//       [u64 indexed_doc_count][u64 positions_sum_normalized]    cumulative at this level's commit  (index.rs:3418-3426)
//       [segments x (u32 block_length, u32 key_count)]           segments = 1 << segment_number_bits (index.rs:3428-3440)
//       per segment: [key_count x key head][block_length - key_count*key_head_size bytes of key bodies]
//     key head, 20 / 22 / 23 bytes (compress_postinglist.rs:339-409, read at search.rs:2318-2350): u64 key_hash (low 3 bits = n-gram
//       type), u16 posting_count-1, u16 max_docid, u16 max_p_docid, [u8 n-gram df x 0/2/3], u16 pointer_pivot_p_docid,
//       u32 compression_type << 30 | rank_position_pointer_range  (offset inside the segment's body bytes)
//     key body (compress_postinglist.rs:694-977): [position blobs, written backwards] [rank-position pointers: 2 B for postings below
//       the pivot, 3 B from the pivot on] [doc-id container: Array u16 x count | Bitmap 8192 B | RLE u16 runs, (u16 start, u16 len-1) x runs]
//     tf (= positions_count) of posting p (decode_positions_multiterm_singlefield, add_result.rs:2036-2197): top bit of its
//       rank-position pointer clear -> the low bits are the distance back from the pointer array to the posting's blob, which
//       starts with the VINT positions_count (read_singlefield_value, add_result.rs:2584-2606); top bit set -> the positions are
//       embedded in the pointer and the tag bits give the count (2 B: 10 -> 1, 11 -> 2; 3 B: 100 -> 1 ... 111 -> 4).
//   vector.bin (vector.rs:1066-1094): per level [u32 clusters][u32 child_count x clusters][records], record = packed VectorHeader
//       {u16 doc_id, u32 field_id, u32 chunk_id, f32 scale, f32 norm, i16 zero_point, i32 sum_q} (24 B, vector.rs:62-73) + f32[dims].
//
// Supported: one indexed field (the C1-C5 configs), single-term keys (n-gram keys are skipped unless the caller asks for them with
// ssb_load_index_bin_ngrams: their heads carry the components' df bytes at 14..16, their postings are never embedded and their blobs
// start with the component tfs, add_result.rs:2076-2089), Array / Bitmap / RLE containers
// (the writer's Delta container is disabled, compress_postinglist.rs:242), f32 vectors.  Term hashing (hash64 / hash32 = gxhash /
// ahash of the term bytes, index.rs:4165-4225) stays on the host side of the boundary: the file carries the 64-bit keys, queries
// arrive as keys.  No Rust toolchain exists in this environment, so no file written by the reference itself could be tested:
// parity of this loader is pinned only by fixtures manufactured with tests/refwriter.py, a restatement of the reference's writer.
#include <string.h>
#include <algorithm>
#include <functional>
#include <vector>

#include "bm25.h"
#include "common.cuh"

namespace ssb {

namespace {
struct Reader {
    const uint8_t* p; uint64_t n; uint64_t pos = 0; bool ok = true;
    bool need(uint64_t k) { if (pos + k > n || pos + k < pos) { ok = false; return false; } return true; }
    uint16_t u16() { if (!need(2)) return 0; uint16_t v; memcpy(&v, p + pos, 2); pos += 2; return v; }
    uint32_t u32() { if (!need(4)) return 0; uint32_t v; memcpy(&v, p + pos, 4); pos += 4; return v; }
    uint64_t u64() { if (!need(8)) return 0; uint64_t v; memcpy(&v, p + pos, 8); pos += 8; return v; }
};
inline uint16_t rd16(const uint8_t* b) { uint16_t v; memcpy(&v, b, 2); return v; }
inline uint32_t rd32(const uint8_t* b) { uint32_t v; memcpy(&v, b, 4); return v; }
inline uint64_t rd64(const uint8_t* b) { uint64_t v; memcpy(&v, b, 8); return v; }

// read_singlefield_value (add_result.rs:2584-2606): 1-3 byte VINT, 7 bits per byte, most significant group first, STOP_BIT on the last
bool vint(const uint8_t* b, uint64_t len, uint64_t at, uint32_t& out) {
    if (at >= len) return false;
    uint32_t v = b[at];
    if (v & 0x80u) { out = v & 0x7Fu; return true; }
    if (at + 1 >= len) return false;
    v = (v & 0x7Fu) << 7;
    const uint32_t v2 = b[at + 1];
    if (v2 & 0x80u) { out = v | (v2 & 0x7Fu); return true; }
    if (at + 2 >= len) return false;
    out = (v << 7) | ((v2 & 0x7Fu) << 7) | (b[at + 2] & 0x7Fu);
    return true;
}

// a position blob = VINT positions_count, then positions_count VINT deltas (compress_positions, compress_postinglist.rs:946-977)
static bool vint_len(const uint8_t* b, uint64_t len, uint64_t at, uint32_t& out, uint32_t& used) {
    if (!vint(b, len, at, out)) return false;
    used = (b[at] & 0x80u) ? 1u : ((b[at + 1] & 0x80u) ? 2u : 3u);
    return true;
}
static bool push_positions(const uint32_t* deltas, uint32_t n, std::vector<uint16_t>& pos, const char*& why);
static bool blob_positions(const uint8_t* body, uint64_t blen, uint64_t at, uint32_t tf, std::vector<uint16_t>& pos, const char*& why) {
    uint32_t v = 0, used = 0, p = 0;
    if (!vint_len(body, blen, at, v, used)) { why = "position blob out of range"; return false; }
    at += used;
    for (uint32_t i = 0; i < tf; i++) {
        if (!vint_len(body, blen, at, v, used)) { why = "position blob runs past the segment body"; return false; }
        at += used;
        p = i == 0 ? v : p + v + 1u;
        if (p > 65535u) { why = "term position above 65535 (positions are kept as u16)"; return false; }
        pos.push_back((uint16_t)p);
    }
    return true;
}

// one posting list: doc ids + tfs appended to the level's arrays.  body = the segment's body bytes.
// positions of one posting from its delta coding (add_result.rs:38-59 + the phrase matcher's `pos += next + 1`, :3620-3640): the first value is
// the absolute position, every further one the gap minus one
static bool push_positions(const uint32_t* deltas, uint32_t n, std::vector<uint16_t>& pos, const char*& why) {
    uint32_t p = 0;
    for (uint32_t i = 0; i < n; i++) {
        p = i == 0 ? deltas[0] : p + deltas[i] + 1u;
        if (p > 65535u) { why = "term position above 65535 (positions are kept as u16)"; return false; }
        pos.push_back((uint16_t)p);
    }
    return true;
}

// n_comp (n-gram keys: 2 / 3): the blob holds n_comp VINT component tfs ahead of positions_count; they go to ctf_out, 3 per posting
bool decode_key(const uint8_t* body, uint64_t blen, uint32_t count, uint32_t pivot, uint32_t ctp, std::vector<uint16_t>& ids,
                std::vector<uint16_t>& tfs, const char*& why, std::vector<uint16_t>* pos_out = nullptr, uint32_t n_comp = 0,
                std::vector<uint16_t>* ctf_out = nullptr) {
    const uint32_t type = ctp >> 30, range = ctp & 0x3FFFFFFFu;
    // intersection.rs:221-227: pivot*2 + (count - pivot)*3 pointer bytes precede the doc-id container
    const uint64_t psum = (uint64_t)pivot * 2 + (pivot <= count - 1 ? (uint64_t)(count - pivot) * 3 : 0);
    const uint64_t docs = (uint64_t)range + psum;
    if (docs > blen) { why = "rank-position pointers run past the segment body"; return false; }
    const size_t base = ids.size();
    ids.resize(base + count); tfs.resize(base + count);
    if (type == 1) {                                               // Array: sorted u16[count]
        if (docs + (uint64_t)count * 2 > blen) { why = "array container runs past the segment body"; return false; }
        for (uint32_t i = 0; i < count; i++) ids[base + i] = rd16(body + docs + 2 * i);
    } else if (type == 2) {                                        // Bitmap: 8192 B, bit (d & 7) of byte (d >> 3)
        if (docs + 8192 > blen) { why = "bitmap container runs past the segment body"; return false; }
        uint32_t n = 0;
        for (uint32_t w = 0; w < 1024; w++) {
            uint64_t x = rd64(body + docs + 8 * w);
            while (x) { const int b = __builtin_ctzll(x); x &= x - 1; if (n < count) ids[base + n] = (uint16_t)(w * 64 + b); n++; }
        }
        if (n != count) { why = "bitmap population != posting_count"; return false; }
    } else if (type == 3) {                                        // RLE: u16 runs, (u16 start, u16 len-1) x runs
        if (docs + 2 > blen) { why = "rle container runs past the segment body"; return false; }
        const uint32_t runs = rd16(body + docs);
        if (docs + 2 + (uint64_t)runs * 4 > blen) { why = "rle container runs past the segment body"; return false; }
        uint32_t n = 0;
        for (uint32_t r = 0; r < runs; r++) {
            const uint32_t start = rd16(body + docs + 2 + 4 * r), extra = rd16(body + docs + 4 + 4 * r);
            for (uint32_t d = start; d <= start + extra; d++) { if (n < count && d < 65536) ids[base + n] = (uint16_t)d; n++; }
        }
        if (n != count) { why = "rle run lengths != posting_count"; return false; }
    } else { why = "delta container (disabled in the reference writer, compress_postinglist.rs:242) is not supported"; return false; }
    // component tfs of an n-gram posting, read at the start of its blob; `at` moves past them to positions_count
    auto components = [&](uint64_t& at) -> bool {
        if (!n_comp) return true;
        uint16_t c3[3] = {0, 0, 0};
        for (uint32_t c = 0; c < n_comp; c++) {
            uint32_t v = 0, used = 0;
            if (!vint_len(body, blen, at, v, used)) { why = "n-gram component tf out of range"; return false; }
            c3[c] = (uint16_t)(v > 65535u ? 65535u : v); at += used;
        }
        ctf_out->insert(ctf_out->end(), c3, c3 + 3);
        return true;
    };
    // tf from the rank-position pointers
    for (uint32_t p = 0; p < count; p++) {
        uint32_t tf = 0;
        if (p < pivot) {
            const uint64_t at = (uint64_t)range + 2ull * p;
            if (at + 2 > blen) { why = "pointer past the segment body"; return false; }
            const uint32_t rp = rd16(body + at);
            if (rp & 0x8000u) {
                if (n_comp) { why = "embedded n-gram posting (the writer never embeds them, index_posting.rs:445)"; return false; }
                tf = (rp >> 14) == 2u ? 1u : 2u;                                     // embedded: 10 -> 1 position, 11 -> 2
                if (pos_out) {                                                       // 14 payload bits: one 14-bit delta or 7 + 7 (index_posting.rs:590-640)
                    uint32_t dl[2];
                    if (tf == 1) dl[0] = rp & 0x3FFFu; else { dl[0] = (rp >> 7) & 0x7Fu; dl[1] = rp & 0x7Fu; }
                    if (!push_positions(dl, tf, *pos_out, why)) return false;
                }
            } else {
                const uint32_t back = rp & 0x7FFFu;
                uint64_t at = (uint64_t)range - back;
                if (back > range || !components(at) || !vint(body, blen, at, tf)) { if (!*why) why = "position blob out of range"; return false; }
                if (pos_out && !blob_positions(body, blen, at, tf, *pos_out, why)) return false;
            }
        } else {
            const uint64_t at = (uint64_t)range + 3ull * p - pivot;
            if (at + 3 > blen) { why = "pointer past the segment body"; return false; }
            const uint32_t rp = (uint32_t)body[at] | ((uint32_t)body[at + 1] << 8) | ((uint32_t)body[at + 2] << 16);
            if (rp & 0x800000u) {
                if (n_comp) { why = "embedded n-gram posting (the writer never embeds them, index_posting.rs:445)"; return false; }
                tf = ((rp >> 21) & 3u) + 1u;                                         // embedded: 100 -> 1 ... 111 -> 4
                if (pos_out) {                                                       // 21 payload bits: 21 | 10 + 11 | 7 + 7 + 7 | 5 + 5 + 5 + 6
                    uint32_t dl[4];
                    if (tf == 1) dl[0] = rp & 0x1FFFFFu;
                    else if (tf == 2) { dl[0] = (rp >> 11) & 0x3FFu; dl[1] = rp & 0x7FFu; }
                    else if (tf == 3) { dl[0] = (rp >> 14) & 0x7Fu; dl[1] = (rp >> 7) & 0x7Fu; dl[2] = rp & 0x7Fu; }
                    else { dl[0] = (rp >> 16) & 0x1Fu; dl[1] = (rp >> 11) & 0x1Fu; dl[2] = (rp >> 6) & 0x1Fu; dl[3] = rp & 0x3Fu; }
                    if (!push_positions(dl, tf, *pos_out, why)) return false;
                }
            } else {
                const uint32_t back = rp & 0x7FFFFFu;
                uint64_t at = (uint64_t)range - back;
                if (back > range || !components(at) || !vint(body, blen, at, tf)) { if (!*why) why = "position blob out of range"; return false; }
                if (pos_out && !blob_positions(body, blen, at, tf, *pos_out, why)) return false;
            }
        }
        if (tf == 0) { why = "positions_count 0"; return false; }
        if (pos_out && tf > 65535u) { why = "more than 65535 positions in one posting"; return false; }
        tfs[base + p] = (uint16_t)(tf > 65535u ? 65535u : tf);
    }
    return true;
}
}  // namespace

// walk the file; on_level receives every decoded level in the neutral layout (valid during the call only).  ngrams: also decode the n-gram
// keys (key low bits != 0) and hand their component tfs / df bytes over (single-term postings and keys: zeros); otherwise they are
// skipped and the second argument of on_level is null.
static int32_t walk_index_bin(const uint8_t* bytes, uint64_t len, const ssb_index_bin_params* prm,
                              const std::function<int32_t(const ssb_level_desc&, const ssb_level_ngrams*)>& on_level, uint64_t* doc_count_out,
                              uint64_t* pos_sum_out, bool ngrams = false) {
    if (!bytes || !prm) { set_error("load_index_bin: null argument"); return SSB_E_INVALID; }
    if (prm->indexed_field_count != 1) { set_error("load_index_bin: %u indexed fields (only single-field indexes are supported)", prm->indexed_field_count); return SSB_E_UNSUPPORTED; }
    const uint32_t khs = prm->key_head_size;
    if (khs != 20 && khs != 22 && khs != 23) { set_error("load_index_bin: key_head_size must be 20, 22 or 23"); return SSB_E_INVALID; }
    if (prm->segment_number_bits > 16) { set_error("load_index_bin: segment_number_bits > 16"); return SSB_E_INVALID; }
    const uint32_t nseg = 1u << prm->segment_number_bits;
    Reader r{bytes, len};
    const uint16_t major = r.u16(); r.u16();
    if (!r.ok || major != 6) { set_error("load_index_bin: format version %u (this loader reads major version 6, index.rs:105)", (unsigned)major); return SSB_E_UNSUPPORTED; }
    uint64_t doc_count = 0, pos_sum = 0;
    uint32_t level = 0;
    std::vector<uint64_t> keys; std::vector<uint32_t> offs; std::vector<uint16_t> ids, tfs, poss; std::vector<std::pair<uint32_t, uint32_t>> seg;
    std::vector<uint16_t> ctf; std::vector<uint8_t> dfb;                // n-gram mode: [n_postings][3] component tfs, [n_terms][3] df bytes
    if (ngrams && khs == 20) { set_error("load_index_bin_ngrams: key_head_size 20 carries no n-gram df bytes (22 / 23)"); return SSB_E_INVALID; }
    const bool want_pos = prm->decode_positions != 0;   // term positions for phrase queries (off: tf only, as before)
    while (r.pos < len) {
        if (level == 0) r.u16();                                   // longest_field_id
        if (!r.need(65536)) break;
        const uint8_t* doclen = bytes + r.pos; r.pos += 65536;
        doc_count = r.u64(); pos_sum = r.u64();
        seg.clear();
        for (uint32_t s = 0; s < nseg; s++) { const uint32_t bl = r.u32(), kc = r.u32(); seg.emplace_back(bl, kc); }
        if (!r.ok) break;
        if (doc_count <= (uint64_t)level * 65536) { set_error("load_index_bin: level %u: indexed_doc_count %llu", level, (unsigned long long)doc_count); return SSB_E_INVALID; }
        const uint64_t rest = doc_count - (uint64_t)level * 65536;
        const uint32_t n_docs = (uint32_t)(rest < 65536 ? rest : 65536);
        keys.clear(); offs.assign(1, 0); ids.clear(); tfs.clear(); poss.clear(); ctf.clear(); dfb.clear();
        for (uint32_t s = 0; s < nseg; s++) {
            const uint64_t head_bytes = (uint64_t)seg[s].second * khs;
            if (seg[s].first < head_bytes || !r.need(seg[s].first)) { set_error("load_index_bin: level %u segment %u: block_length %u < key heads / past the end", level, s, seg[s].first); return SSB_E_INVALID; }
            const uint8_t* heads = bytes + r.pos;
            const uint8_t* body = heads + head_bytes;
            const uint64_t blen = seg[s].first - head_bytes;
            r.pos += seg[s].first;
            for (uint32_t k = 0; k < seg[s].second; k++) {
                const uint8_t* h = heads + (uint64_t)k * khs;
                const uint64_t key = rd64(h);
                const uint32_t ty = (uint32_t)(key & 7ull);
                if (ty && !ngrams) continue;                       // n-gram posting lists (frequent-term bigrams / trigrams): opt-in
                const uint32_t count = (uint32_t)rd16(h + 8) + 1u;
                const uint32_t pivot = rd16(h + khs - 6), ctp = rd32(h + khs - 4);
                const uint32_t n_comp = ty == 0 ? 0u : (ty <= SSB_NGRAM_RF ? 2u : 3u);
                if (ngrams) {
                    for (uint32_t c = 0; c < 3; c++) dfb.push_back(ty && 14 + c < khs - 6 ? h[14 + c] : (uint8_t)0);
                    if (!ty) ctf.resize(ctf.size() + 3ull * count, 0);
                }
                const char* why = "";
                if (!decode_key(body, blen, count, pivot, ctp, ids, tfs, why, want_pos ? &poss : nullptr, n_comp, &ctf)) {
                    set_error("load_index_bin: level %u segment %u key %016llx: %s", level, s, (unsigned long long)key, why);
                    return SSB_E_INVALID;
                }
                keys.push_back(key); offs.push_back((uint32_t)ids.size());
            }
        }
        ssb_level_desc d{};
        d.level_id = level; d.n_docs = n_docs; d.n_terms = (uint32_t)keys.size();
        d.term_keys = keys.data(); d.posting_offsets = offs.data(); d.doc_ids = ids.data(); d.tfs = tfs.data(); d.doc_len_bytes = doclen;
        if (want_pos) { poss.push_back(0); d.positions = poss.data(); }      // (never null, even for a level without postings)
        ctf.resize(ctf.size() + 3, 0); dfb.resize(dfb.size() + 3, 0);       // (never null either)
        const ssb_level_ngrams ng{ctf.data(), dfb.data()};
        SSB_TRY(on_level(d, ngrams ? &ng : nullptr));
        level++;
    }
    if (!r.ok) { set_error("load_index_bin: truncated file (level %u)", level); return SSB_E_INVALID; }
    if (level == 0) { set_error("load_index_bin: no level in the file"); return SSB_E_INVALID; }
    if (doc_count_out) *doc_count_out = doc_count;
    if (pos_sum_out) *pos_sum_out = pos_sum;
    return SSB_OK;
}

int32_t load_index_bin(LexIndex* lex, const uint8_t* bytes, uint64_t len, const ssb_index_bin_params* prm, uint64_t* n_docs_out, bool ngrams) {
    if (!lex) { set_error("load_index_bin: null argument"); return SSB_E_INVALID; }
    if (lex->n_levels() != 0) { set_error("load_index_bin: the index already holds levels"); return SSB_E_STATE; }
    uint64_t doc_count = 0, pos_sum = 0;
    SSB_TRY(walk_index_bin(bytes, len, prm, [&](const ssb_level_desc& d, const ssb_level_ngrams* ng) { return lex->add_level_ngrams(&d, ng); },
                           &doc_count, &pos_sum, ngrams));
    SSB_TRY(lex->commit(doc_count, pos_sum));     // indexed_doc_count / positions_sum_normalized of the last level = the shard's totals
    if (n_docs_out) *n_docs_out = doc_count;
    return SSB_OK;
}

// host-only walk of the file (no device work): totals + an order-dependent checksum of every (key, doc id, tf) — used by the
// CPU tests of the parser and as a sanity check before a load
int32_t inspect_index_bin(const uint8_t* bytes, uint64_t len, const ssb_index_bin_params* prm, uint64_t out[8]) {
    uint64_t levels = 0, terms = 0, postings = 0, tf_sum = 0, h = 1469598103934665603ull, hp = 1469598103934665603ull;
    auto mix = [&](uint64_t x) { h = (h ^ x) * 1099511628211ull; };
    uint64_t doc_count = 0, pos_sum = 0;
    SSB_TRY(walk_index_bin(bytes, len, prm, [&](const ssb_level_desc& d, const ssb_level_ngrams*) {
        levels++; terms += d.n_terms; postings += d.posting_offsets[d.n_terms];
        for (uint32_t t = 0; t < d.n_terms; t++) {
            mix(d.term_keys[t]);
            for (uint32_t i = d.posting_offsets[t]; i < d.posting_offsets[t + 1]; i++) { mix(((uint64_t)d.level_id << 32) | ((uint64_t)d.doc_ids[i] << 16) | d.tfs[i]); tf_sum += d.tfs[i]; }
        }
        if (d.positions) {     // decode_positions: a second checksum over every position, in posting order
            uint64_t np = 0;
            for (uint32_t i = 0; i < d.posting_offsets[d.n_terms]; i++) np += d.tfs[i];
            for (uint64_t i = 0; i < np; i++) hp = (hp ^ d.positions[i]) * 1099511628211ull;
        }
        return (int32_t)SSB_OK;
    }, &doc_count, &pos_sum));
    out[0] = levels; out[1] = terms; out[2] = postings; out[3] = tf_sum; out[4] = doc_count; out[5] = pos_sum; out[6] = h; out[7] = prm->decode_positions ? hp : 0;
    return SSB_OK;
}

// host-only walk in n-gram mode: out = {levels, n-gram keys, n-gram postings, sum of their tfs, FNV checksum over every n-gram (key, level,
// df bytes) and (doc id, tf, component tfs) in file order, FNV checksum over the n-gram postings' positions (decode_positions) or 0, 0, 0}
int32_t inspect_index_bin_ngrams(const uint8_t* bytes, uint64_t len, const ssb_index_bin_params* prm, uint64_t out[8]) {
    uint64_t levels = 0, terms = 0, postings = 0, tf_sum = 0, h = 1469598103934665603ull, hp = 1469598103934665603ull;
    auto mix = [&](uint64_t x) { h = (h ^ x) * 1099511628211ull; };
    SSB_TRY(walk_index_bin(bytes, len, prm, [&](const ssb_level_desc& d, const ssb_level_ngrams* ng) {
        levels++;
        uint64_t pbase = 0;
        for (uint32_t t = 0; t < d.n_terms; t++) {
            const uint32_t a = d.posting_offsets[t], b = d.posting_offsets[t + 1];
            uint64_t np = 0;
            for (uint32_t i = a; i < b; i++) np += d.tfs[i];
            if (d.term_keys[t] & 7u) {
                terms++; postings += b - a;
                const uint8_t* f = ng->component_df_bytes + 3ull * t;
                mix(d.term_keys[t]); mix(((uint64_t)d.level_id << 32) | ((uint64_t)f[0] << 16) | ((uint64_t)f[1] << 8) | f[2]);
                for (uint32_t i = a; i < b; i++) {
                    const uint16_t* c = ng->component_tfs + 3ull * i;
                    mix(((uint64_t)d.doc_ids[i] << 48) | ((uint64_t)d.tfs[i] << 32) | ((uint64_t)c[0] << 16) | c[1]); mix(c[2]);
                    tf_sum += d.tfs[i];
                }
                if (d.positions) for (uint64_t j = 0; j < np; j++) hp = (hp ^ d.positions[pbase + j]) * 1099511628211ull;
            }
            pbase += np;
        }
        return (int32_t)SSB_OK;
    }, nullptr, nullptr, true));
    out[0] = levels; out[1] = terms; out[2] = postings; out[3] = tf_sum; out[4] = h; out[5] = prm->decode_positions ? hp : 0; out[6] = 0; out[7] = 0;
    return SSB_OK;
}

// vector.bin -> per level (local ids, rows); the caller appends them through the normal add path
int32_t parse_vector_bin(const uint8_t* bytes, uint64_t len, uint32_t dims, std::vector<VectorLevel>& out, bool keep_fields) {
    Reader r{bytes, len};
    const uint64_t rec = 24 + (uint64_t)dims * 4;
    uint32_t level = 0;
    while (r.pos < len) {
        const uint32_t clusters = r.u32();
        if (!r.ok || !r.need((uint64_t)clusters * 4)) { set_error("load_vector_bin: truncated cluster table (level %u)", level); return SSB_E_INVALID; }
        uint64_t n = 0;
        std::vector<uint32_t> counts(clusters);
        for (uint32_t c = 0; c < clusters; c++) { counts[c] = r.u32(); n += counts[c]; }
        if (n > 65536ull * 64) { set_error("load_vector_bin: level %u holds %llu records", level, (unsigned long long)n); return SSB_E_INVALID; }
        if (!r.need(n * rec)) { set_error("load_vector_bin: truncated records (level %u)", level); return SSB_E_INVALID; }
        VectorLevel vl; vl.level_id = level; vl.ids.resize(n); vl.rows.resize(n * dims); vl.cluster_counts = std::move(counts);
        if (keep_fields) { vl.fields.resize(n); vl.chunks.resize(n); }
        for (uint64_t i = 0; i < n; i++) {
            const uint8_t* h = bytes + r.pos + i * rec;
            vl.ids[i] = rd16(h);                                   // VectorHeader.doc_id (vector.rs:65-73); packed: field_id at +2, chunk_id at +6
            if (keep_fields) {
                const uint32_t f = rd32(h + 2);
                if (f >= 32) { set_error("load_vector_bin: field id %u of record %llu (level %u): indexed field ids must be < 32", f, (unsigned long long)i, level); return SSB_E_INVALID; }
                vl.fields[i] = (uint8_t)f; vl.chunks[i] = rd32(h + 6);
            }
            memcpy(vl.rows.data() + i * dims, h + 24, (size_t)dims * 4);
        }
        r.pos += n * rec;
        out.push_back(std::move(vl));
        level++;
    }
    return SSB_OK;
}

}  // namespace ssb
