// Staging: decode the LMDB-format databases (keys per heed_codec/*, values per
// CboRoaringBitmapCodec, crates/milli/src/heed_codec/roaring_bitmap/cbo_roaring_bitmap_codec.rs:15-85)
// into the HBM posting-store layout described in host_index.h.
#include <cmath>
#include "host_index.h"

#include <algorithm>
#include <charconv>
#include <cstdlib>
#include <stdexcept>
#include <set>
#include <thread>

namespace b200 {

namespace {

// Append the docids of one CBO value to `out` (ascending). Returns cardinality.
uint32_t cbo_decode_append(const uint8_t *p, size_t n, std::vector<uint32_t> &out) {
    size_t start = out.size();
    if (n <= 28) {  // raw native-endian u32s (<= THRESHOLD ints)
        for (size_t i = 0; i + 4 <= n; i += 4) {
            uint32_t v;
            memcpy(&v, p + i, 4);
            out.push_back(v);
        }
        return (uint32_t)(out.size() - start);
    }
    uint32_t cookie, nc;
    memcpy(&cookie, p, 4);
    memcpy(&nc, p + 4, 4);
    if (cookie != 12346) throw std::runtime_error("stage: roaring value with run containers / unknown cookie");
    // every length comes from the value itself: check it against the bytes we were given before reading
    if (nc == 0 || nc > 65536 || 8 + 8 * (size_t)nc > n) throw std::runtime_error("stage: malformed roaring value (container count)");
    const uint8_t *desc = p + 8;
    const uint8_t *data = p + 8 + 8 * (size_t)nc;
    const uint8_t *const end = p + n;
    for (uint32_t c = 0; c < nc; c++) {
        uint16_t key, cm1;
        memcpy(&key, desc + 4 * c, 2);
        memcpy(&cm1, desc + 4 * c + 2, 2);
        uint32_t card = (uint32_t)cm1 + 1, hi = (uint32_t)key << 16;
        if ((size_t)(end - data) < (card <= 4096 ? 2 * (size_t)card : (size_t)8192)) throw std::runtime_error("stage: malformed roaring value (truncated container)");
        if (card <= 4096) {
            for (uint32_t i = 0; i < card; i++) {
                uint16_t lo;
                memcpy(&lo, data + 2 * i, 2);
                out.push_back(hi | lo);
            }
            data += 2 * (size_t)card;
        } else {
            for (uint32_t w = 0; w < 1024; w++) {
                uint64_t bits;
                memcpy(&bits, data + 8 * w, 8);
                while (bits) {
                    out.push_back(hi | (w * 64 + (uint32_t)__builtin_ctzll(bits)));
                    bits &= bits - 1;
                }
            }
            data += 8192;
        }
    }
    return (uint32_t)(out.size() - start);
}

// Append one posting list (ascending docids) to the pool.  A list is stored as a dense bitmap over the docid space when card >
// n_docs / 128 (B200_DENSE_DIV): a bitmap costs n_docs / 8 bytes, i.e. at most 4x the sorted-docid form at that density, and turns
// the scatter of the list into a coalesced gather by universe row instead of one random row lookup per docid (DESIGN.md §2).
uint32_t dense_min_card(const HostIndex &ix) {
    uint32_t dense_div = 128;
    if (const char *env = getenv("B200_DENSE_DIV")) dense_div = (uint32_t)std::max(8, atoi(env));
    return ix.n_docs / dense_div;
}
void append_list(HostIndex &ix, const uint32_t *src, uint32_t c, uint32_t dense_min) {
    if (ix.pool.size() & 1) ix.pool.push_back(0);  // keep every list 8-byte aligned
    ListRef r{ix.pool.size(), c, 0};
    if (c > dense_min && c > 64) {
        r.dense = 1;
        size_t base = ix.pool.size();
        ix.pool.resize(base + 2 * (size_t)ix.n_words64, 0);
        uint64_t *words = reinterpret_cast<uint64_t *>(ix.pool.data() + base);
        for (uint32_t k = 0; k < c; k++) {
            uint32_t d = src[k];
            if (d < ix.n_docs) words[d >> 6] |= 1ull << (d & 63);
        }
    } else {
        ix.pool.insert(ix.pool.end(), src, src + c);
    }
    ix.lists.push_back(r);
}

struct Builder {
    HostIndex &ix;
    const RawDb *dbs_base = nullptr;
    explicit Builder(HostIndex &i) : ix(i) {}
    // decode values [k0,k1) of a db in parallel, then append to the pool in key order; returns first list id
    uint32_t add_lists(const RawDb &db, const std::vector<uint8_t> &keep /* per key: 1 = stage */) {
        uint64_t n = db.n;
        if (dbs_base && &db >= dbs_base && &db < dbs_base + 10) {
            ix.db_first[&db - dbs_base] = (uint32_t)ix.lists.size();
            ix.db_keys[&db - dbs_base] = (uint32_t)n;
        }
        unsigned nt = std::max(1u, std::min(16u, std::thread::hardware_concurrency()));
        std::vector<std::vector<uint32_t>> parts(nt);
        std::vector<std::vector<uint32_t>> cards(nt);
        std::vector<std::thread> th;
        std::vector<std::string> errs(nt);
        for (unsigned t = 0; t < nt; t++) {
            th.emplace_back([&, t]() {
                uint64_t a = n * t / nt, b = n * (t + 1) / nt;
                try {
                    for (uint64_t i = a; i < b; i++) {
                        if (!keep.empty() && !keep[i]) {
                            cards[t].push_back(0xffffffffu);
                            continue;
                        }
                        uint32_t c = cbo_decode_append(db.vals.data() + db.voff[i], db.voff[i + 1] - db.voff[i], parts[t]);
                        cards[t].push_back(c);
                    }
                } catch (const std::exception &e) {
                    errs[t] = e.what();
                }
            });
        }
        for (auto &x : th) x.join();
        for (auto &e : errs)
            if (!e.empty()) throw std::runtime_error(e);
        uint32_t first = (uint32_t)ix.lists.size();
        const uint32_t dense_min = dense_min_card(ix);
        for (unsigned t = 0; t < nt; t++) {
            size_t at = 0;
            for (uint32_t c : cards[t]) {
                if (c == 0xffffffffu) {
                    ix.lists.push_back(ListRef{0, 0, 0});
                    continue;
                }
                append_list(ix, parts[t].data() + at, c, dense_min);
                at += c;
            }
            std::vector<uint32_t>().swap(parts[t]);
        }
        return first;
    }
};

}  // namespace

void build_host_index(const std::vector<uint8_t> &dict_bytes, const std::vector<uint64_t> &dict_off, const RawDb *dbs,
                      const std::vector<uint8_t> &docids_cbo, HostIndex &ix) {
    ix.dict_bytes = dict_bytes;
    ix.dict_off = dict_off;
    ix.n_words = dict_off.empty() ? 0 : dict_off.size() - 1;
    if (ix.n_words >= (1u << 21)) throw std::runtime_error("stage: dictionary larger than 2^21 words (packed pair keys)");
    // universe
    std::vector<uint32_t> docs;
    cbo_decode_append(docids_cbo.data(), docids_cbo.size(), docs);
    ix.n_documents = docs.size();
    ix.n_docs = docs.empty() ? 0 : docs.back() + 1;
    for (auto d : docs) ix.n_docs = std::max(ix.n_docs, d + 1);
    ix.n_words64 = (ix.n_docs + 63) / 64;
    ix.base_ub.assign(ix.n_words64, 0);
    for (auto d : docs) ix.base_ub[d >> 6] |= 1ull << (d & 63);
    ix.lists.clear();
    ix.pool.clear();
    Builder b(ix);
    b.dbs_base = dbs;
    std::vector<uint8_t> all;

    auto word_of_key = [&](const RawDb &db, uint64_t i, size_t trim) -> int64_t {
        size_t kn = db.koff[i + 1] - db.koff[i];
        if (kn < trim) return -1;
        return ix.find_word(db.keys.data() + db.koff[i], kn - trim);
    };
    // word_docids / exact_word_docids
    for (int which = 0; which < 2; which++) {
        const RawDb &db = dbs[which];
        std::vector<uint32_t> &dir = which == 0 ? ix.wd_list : ix.ewd_list;
        dir.assign(ix.n_words, NO_LIST);
        uint32_t first = b.add_lists(db, all);
        for (uint64_t i = 0; i < db.n; i++) {
            int64_t w = word_of_key(db, i, 0);
            if (w >= 0) dir[w] = first + (uint32_t)i;
        }
    }
    // word_fid / word_position: key = word \0 u16be
    auto csr_u16 = [&](const RawDb &db, std::vector<uint32_t> &off, std::vector<uint16_t> &val, std::vector<uint32_t> &lst) {
        uint32_t first = b.add_lists(db, all);
        off.assign(ix.n_words + 1, 0);
        std::vector<int64_t> wk(db.n);
        for (uint64_t i = 0; i < db.n; i++) {
            wk[i] = word_of_key(db, i, 3);
            if (wk[i] >= 0) off[wk[i] + 1]++;
        }
        for (uint64_t w = 0; w < ix.n_words; w++) off[w + 1] += off[w];
        val.assign(off[ix.n_words], 0);
        lst.assign(off[ix.n_words], NO_LIST);
        std::vector<uint32_t> cur(off.begin(), off.end() - 1);
        for (uint64_t i = 0; i < db.n; i++) {
            if (wk[i] < 0) continue;
            const uint8_t *k = db.keys.data() + db.koff[i + 1] - 2;
            uint32_t at = cur[wk[i]]++;
            val[at] = (uint16_t)((k[0] << 8) | k[1]);
            lst[at] = first + (uint32_t)i;
        }
    };
    csr_u16(dbs[6], ix.wf_off, ix.wf_fid, ix.wf_list);
    csr_u16(dbs[5], ix.wp_off, ix.wp_pos, ix.wp_list);
    // prefixes: union of the keys of the two prefix docids dbs
    {
        std::vector<std::string> ps;
        for (int which : {2, 3})
            for (uint64_t i = 0; i < dbs[which].n; i++)
                ps.emplace_back((const char *)dbs[which].keys.data() + dbs[which].koff[i], dbs[which].koff[i + 1] - dbs[which].koff[i]);
        std::sort(ps.begin(), ps.end());
        ps.erase(std::unique(ps.begin(), ps.end()), ps.end());
        ix.prefixes = ps;
        size_t np = ps.size();
        ix.pd_list.assign(np, NO_LIST);
        ix.epd_list.assign(np, NO_LIST);
        for (int which : {2, 3}) {
            const RawDb &db = dbs[which];
            uint32_t first = b.add_lists(db, all);
            for (uint64_t i = 0; i < db.n; i++) {
                std::string k((const char *)db.keys.data() + db.koff[i], db.koff[i + 1] - db.koff[i]);
                int32_t p = ix.find_prefix(k);
                if (p >= 0) (which == 2 ? ix.pd_list : ix.epd_list)[p] = first + (uint32_t)i;
            }
        }
        auto csr_p = [&](const RawDb &db, std::vector<uint32_t> &off, std::vector<uint16_t> &val, std::vector<uint32_t> &lst) {
            uint32_t first = b.add_lists(db, all);
            off.assign(np + 1, 0);
            std::vector<int32_t> pk(db.n);
            for (uint64_t i = 0; i < db.n; i++) {
                size_t kn = db.koff[i + 1] - db.koff[i];
                pk[i] = kn >= 3 ? ix.find_prefix(std::string((const char *)db.keys.data() + db.koff[i], kn - 3)) : -1;
                if (pk[i] >= 0) off[pk[i] + 1]++;
            }
            for (size_t p = 0; p < np; p++) off[p + 1] += off[p];
            val.assign(off[np], 0);
            lst.assign(off[np], NO_LIST);
            std::vector<uint32_t> cur(off.begin(), off.end() - 1);
            for (uint64_t i = 0; i < db.n; i++) {
                if (pk[i] < 0) continue;
                const uint8_t *k = db.keys.data() + db.koff[i + 1] - 2;
                uint32_t at = cur[pk[i]]++;
                val[at] = (uint16_t)((k[0] << 8) | k[1]);
                lst[at] = first + (uint32_t)i;
            }
        };
        csr_p(dbs[8], ix.pf_off, ix.pf_fid, ix.pf_list);
        csr_p(dbs[7], ix.pp_off, ix.pp_pos, ix.pp_list);
    }
    // field_id_word_count: key = u16be fid | u8 count
    {
        const RawDb &db = dbs[9];
        uint32_t first = b.add_lists(db, all);
        for (uint64_t i = 0; i < db.n; i++) {
            const uint8_t *k = db.keys.data() + db.koff[i];
            if (db.koff[i + 1] - db.koff[i] != 3) continue;
            uint32_t fid = (k[0] << 8) | k[1];
            ix.fwc_list[(fid << 8) | k[2]] = first + (uint32_t)i;
        }
    }
    // word pair proximity: key = prox | w1 | 0 | w2, already sorted by (prox, w1, w2) == packed key order
    {
        const RawDb &db = dbs[4];
        std::vector<uint64_t> keys(db.n, ~0ull);
        std::vector<uint8_t> keep(db.n, 0);
        unsigned nt = std::max(1u, std::min(16u, std::thread::hardware_concurrency()));
        std::vector<std::thread> th;
        for (unsigned t = 0; t < nt; t++)
            th.emplace_back([&, t]() {
                uint64_t a = db.n * t / nt, e = db.n * (t + 1) / nt;
                std::string last_w1;
                int64_t last_r1 = -1;
                for (uint64_t i = a; i < e; i++) {
                    const uint8_t *k = db.keys.data() + db.koff[i];
                    size_t kn = db.koff[i + 1] - db.koff[i];
                    if (kn < 3) continue;
                    const uint8_t *z = (const uint8_t *)memchr(k + 1, 0, kn - 1);
                    if (!z) continue;
                    size_t l1 = z - (k + 1);
                    int64_t r1;
                    if (last_r1 >= 0 && last_w1.size() == l1 && memcmp(last_w1.data(), k + 1, l1) == 0)
                        r1 = last_r1;
                    else {
                        r1 = ix.find_word(k + 1, l1);
                        last_w1.assign((const char *)k + 1, l1);
                        last_r1 = r1;
                    }
                    int64_t r2 = ix.find_word(z + 1, kn - 2 - l1);
                    if (r1 < 0 || r2 < 0) continue;
                    keys[i] = HostIndex::pair_key(k[0], (uint32_t)r1, (uint32_t)r2);
                    keep[i] = 1;
                }
            });
        for (auto &x : th) x.join();
        // keys whose words are unknown are dropped; the rest must be strictly ascending
        bool all_kept = true;
        for (auto kflag : keep) all_kept = all_kept && kflag;
        uint32_t first = b.add_lists(db, keep);
        ix.pair_list_base = first;
        if (all_kept) {
            ix.pair_keys = std::move(keys);
        } else {
            // compact: list ids must stay contiguous with the keys, so rebuild the list table slice
            std::vector<ListRef> kept;
            for (uint64_t i = 0; i < db.n; i++)
                if (keep[i]) {
                    ix.pair_keys.push_back(keys[i]);
                    kept.push_back(ix.lists[first + i]);
                }
            ix.lists.resize(first);
            ix.lists.insert(ix.lists.end(), kept.begin(), kept.end());
        }
        for (size_t i = 1; i < ix.pair_keys.size(); i++)
            if (ix.pair_keys[i - 1] >= ix.pair_keys[i]) throw std::runtime_error("stage: word_pair_proximity_docids keys not in LMDB order");
    }
}

void build_presence(const RawDb &db, int which, HostIndex &ix) {
    std::vector<uint32_t> docs;
    for (uint64_t i = 0; i < db.n; i++) {
        const uint8_t *k = db.keys.data() + db.koff[i];
        if (db.koff[i + 1] - db.koff[i] != 2) throw std::runtime_error("stage: facet presence key is not a u16 BE field id");
        std::vector<uint64_t> &bm = ix.presence[which][(uint16_t)(k[0] << 8 | k[1])];
        bm.assign(ix.n_words64, 0);
        docs.clear();
        cbo_decode_append(db.vals.data() + db.voff[i], db.voff[i + 1] - db.voff[i], docs);
        for (uint32_t d : docs)
            if (d < ix.n_docs) bm[d >> 6] |= 1ull << (d & 63);
    }
}

void build_sort_fields(const RawDb &f64_db, const RawDb &string_db, HostIndex &ix) {
    ix.sort_fields.clear();
    struct Val {
        uint16_t fid;
        uint32_t key_index;  // among the level-0 keys of its database
        std::vector<uint32_t> docs;
        std::string bound;  // strings: the normalised key
    };
    // level-0 entries in LMDB order (u16 BE fid | u8 level | bound): per field, numbers and strings each come in ascending order
    auto level0 = [&](const RawDb &db, bool numbers) {
        std::vector<Val> out;
        uint32_t l0 = 0;
        for (uint64_t i = 0; i < db.n; i++) {
            const uint8_t *k = db.keys.data() + db.koff[i];
            size_t kn = db.koff[i + 1] - db.koff[i];
            if (kn < 3) throw std::runtime_error("stage: facet key shorter than fid + level");
            if (k[2] != 0) continue;  // group levels: only level 0 is read
            if (numbers && kn != 3 + 16) throw std::runtime_error("stage: facet_id_f64_docids key without a 16-byte OrderedF64 bound");
            const uint8_t *v = db.vals.data() + db.voff[i];
            size_t vn = db.voff[i + 1] - db.voff[i];
            if (vn < 1) throw std::runtime_error("stage: facet value without its group size byte");
            Val x;
            x.fid = (uint16_t)(k[0] << 8 | k[1]);
            x.key_index = l0++;
            if (!numbers) x.bound.assign((const char *)k + 3, kn - 3);
            cbo_decode_append(v + 1, vn - 1, x.docs);
            out.push_back(std::move(x));
        }
        return out;
    };
    std::vector<Val> nums = level0(f64_db, true), strs = level0(string_db, false);
    for (auto &x : nums) {
        SortField &f = ix.sort_fields[x.fid];
        f.num_key.push_back(x.key_index);
        f.n_num++;
    }
    for (auto &x : strs) {
        SortField &f = ix.sort_fields[x.fid];
        f.str_key.push_back(x.key_index);
        f.str_val.push_back(x.bound);
        f.n_str++;
    }
    for (auto &kv : ix.sort_fields) {
        SortField &f = kv.second;
        f.key[0].assign(ix.n_docs, f.n_values());
        f.key[1].assign(ix.n_docs, f.n_values());
    }
    // ordinal of the i-th number / j-th string of a field in each direction; a document keeps the smallest (its first bucket)
    std::map<uint16_t, uint32_t> seen;
    auto fold = [&](std::vector<Val> &vals, bool numbers) {
        seen.clear();
        for (auto &x : vals) {
            SortField &f = ix.sort_fields[x.fid];
            uint32_t i = seen[x.fid]++;
            uint32_t oa = numbers ? i : f.n_num + i;
            uint32_t od = numbers ? f.n_num - 1 - i : f.n_num + (f.n_str - 1 - i);
            for (uint32_t d : x.docs) {
                if (d >= ix.n_docs) continue;  // not in documents_ids
                f.key[0][d] = std::min(f.key[0][d], oa);
                f.key[1][d] = std::min(f.key[1][d], od);
            }
        }
    };
    fold(nums, true);
    fold(strs, false);
    // facet distribution: each number's f64 (the bound's last 8 bytes, big-endian), the number ordinals in Display-string order, and
    // the document-major ordinals.  Filling the table value by value in ascending ordinal order leaves each document's run sorted.
    for (uint64_t i = 0, l0 = 0; i < f64_db.n; i++) {
        const uint8_t *k = f64_db.keys.data() + f64_db.koff[i];
        if (k[2] != 0) continue;
        uint64_t bits = 0;
        for (int b = 0; b < 8; b++) bits = bits << 8 | k[11 + b];
        double v;
        memcpy(&v, &bits, 8);
        ix.sort_fields[nums[l0++].fid].num_val.push_back(v);
    }
    for (auto &kv : ix.sort_fields) {
        SortField &f = kv.second;
        std::vector<std::string> shown(f.n_num);
        for (uint32_t o = 0; o < f.n_num; o++) shown[o] = rust_f64_display(f.num_val[o]);
        f.disp.resize(f.n_num);
        for (uint32_t o = 0; o < f.n_num; o++) f.disp[o] = o;
        std::sort(f.disp.begin(), f.disp.end(), [&](uint32_t a, uint32_t b) { return shown[a] < shown[b]; });
        f.doc_off.assign(ix.n_docs + 1, 0);
    }
    auto each_value = [&](auto fn) {
        seen.clear();
        for (auto &x : nums) fn(ix.sort_fields[x.fid], seen[x.fid]++, x);
        seen.clear();
        for (auto &x : strs) {
            SortField &f = ix.sort_fields[x.fid];
            fn(f, f.n_num + seen[x.fid]++, x);
        }
    };
    each_value([&](SortField &f, uint32_t, const Val &x) {
        for (uint32_t d : x.docs)
            if (d < ix.n_docs) f.doc_off[d + 1]++;
    });
    for (auto &kv : ix.sort_fields) {
        SortField &f = kv.second;
        for (uint32_t d = 0; d < ix.n_docs; d++) f.doc_off[d + 1] += f.doc_off[d];
        f.doc_ord.resize(f.doc_off[ix.n_docs]);
    }
    std::map<uint16_t, std::vector<uint32_t>> fill;
    each_value([&](SortField &f, uint32_t o, const Val &x) {
        std::vector<uint32_t> &at = fill[x.fid];
        if (at.empty()) at.assign(f.doc_off.begin(), f.doc_off.end() - 1);
        for (uint32_t d : x.docs)
            if (d < ix.n_docs) f.doc_ord[at[d]++] = o;
    });
}

std::string rust_f64_display(double v) {
    if (std::isnan(v)) return "NaN";
    if (std::isinf(v)) return v > 0 ? "inf" : "-inf";
    // to_chars in scientific notation gives the shortest round-trip digits d[.ddd]e±x; fixed notation would print the exact binary
    // expansion of a large value ("99999999999999991611392" for 1e23) where Rust pads the shortest digits with zeros
    char buf[64];
    const auto res = std::to_chars(buf, buf + sizeof buf, v, std::chars_format::scientific);
    std::string s(buf, res.ptr), sign;
    if (s[0] == '-') {
        sign = "-";
        s.erase(0, 1);
    }
    const size_t e = s.find('e');
    const int point = 1 + atoi(s.c_str() + e + 1);  // decimal point position after the first digit, shifted by the exponent
    std::string digits = s.substr(0, e);
    if (digits.size() > 1) digits.erase(1, 1);  // the '.'
    if (point <= 0) return sign + "0." + std::string((size_t)-point, '0') + digits;
    if ((size_t)point >= digits.size()) return sign + digits + std::string((size_t)point - digits.size(), '0');
    return sign + digits.substr(0, (size_t)point) + "." + digits.substr((size_t)point);
}

void build_geo_field(const RawDb &f64_db, const RawDb &string_db, HostIndex &ix) {
    GeoField &g = ix.geo;
    g.lat.assign(ix.n_docs, 0.0);
    g.lng.assign(ix.n_docs, 0.0);
    g.ub.assign(ix.n_words64, 0);
    g.n_geo = 0;
    if (g.lat_fid == 0xFFFF || g.lng_fid == 0xFFFF) return;
    // per coordinate: 0 none, 1 from a number, 2 from a string
    std::vector<uint8_t> have[2] = {std::vector<uint8_t>(ix.n_docs, 0), std::vector<uint8_t>(ix.n_docs, 0)};
    std::vector<double> *dst[2] = {&g.lat, &g.lng};
    const uint16_t fids[2] = {g.lat_fid, g.lng_fid};
    std::vector<uint32_t> docs;
    // level-0 entries come in ascending value order per field, so the first value a document meets is its smallest (geo_value
    // takes the first entry of field_id_docid_facet_{f64s,strings} for (fid, docid), ordered the same way)
    auto scan = [&](const RawDb &db, bool numbers) {
        for (uint64_t i = 0; i < db.n; i++) {
            const uint8_t *k = db.keys.data() + db.koff[i];
            const size_t kn = db.koff[i + 1] - db.koff[i];
            if (kn < 3 || k[2] != 0) continue;
            const uint16_t fid = (uint16_t)(k[0] << 8 | k[1]);
            for (int c = 0; c < 2; c++) {
                if (fid != fids[c]) continue;
                double v = 0;
                if (numbers) {
                    if (kn != 3 + 16) throw std::runtime_error("stage: facet_id_f64_docids key without a 16-byte OrderedF64 bound");
                    uint64_t bits = 0;
                    for (int b = 0; b < 8; b++) bits = bits << 8 | k[11 + b];
                    memcpy(&v, &bits, 8);
                } else {
                    // str::parse::<f64>: the whole string, no surrounding blanks
                    std::string str((const char *)k + 3, kn - 3);
                    char *end = nullptr;
                    v = str.empty() || isspace((unsigned char)str[0]) || str.find('x') != std::string::npos ? 0.0 : strtod(str.c_str(), &end);
                    if (!end || *end) v = std::nan("");
                }
                docs.clear();
                cbo_decode_append(db.vals.data() + db.voff[i] + 1, db.voff[i + 1] - db.voff[i] - 1, docs);
                for (uint32_t d : docs) {
                    if (d >= ix.n_docs || have[c][d]) continue;
                    if (!numbers && std::isnan(v))
                        throw std::runtime_error("stage: a geo coordinate stored as a string does not parse as f64 (docid " + std::to_string(d) + ")");
                    have[c][d] = numbers ? 1 : 2;
                    (*dst[c])[d] = v;
                }
            }
        }
    };
    scan(f64_db, true);
    scan(string_db, false);
    for (uint32_t d = 0; d < ix.n_docs; d++) {
        if (!have[0][d] && !have[1][d]) continue;
        if (!have[0][d] || !have[1][d])
            throw std::runtime_error("stage: document " + std::to_string(d) + " has one geo coordinate without the other");
        if (!(ix.base_ub[d >> 6] >> (d & 63) & 1)) continue;  // not in documents_ids
        g.ub[d >> 6] |= 1ull << (d & 63);
        g.n_geo++;
    }
}

bool parse_json_string_array(const uint8_t *s, size_t n, std::vector<std::string> &out) {
    out.clear();
    size_t i = 0;
    auto ws = [&]() {
        while (i < n && (s[i] == ' ' || s[i] == '\t' || s[i] == '\n' || s[i] == '\r')) i++;
    };
    auto hex4 = [&](uint32_t &v) {
        if (i + 4 > n) return false;
        v = 0;
        for (int k = 0; k < 4; k++) {
            const uint8_t c = s[i++];
            const int d = c >= '0' && c <= '9' ? c - '0' : c >= 'a' && c <= 'f' ? c - 'a' + 10 : c >= 'A' && c <= 'F' ? c - 'A' + 10 : -1;
            if (d < 0) return false;
            v = v << 4 | (uint32_t)d;
        }
        return true;
    };
    auto put_utf8 = [](std::string &o, uint32_t c) {
        if (c < 0x80) {
            o += (char)c;
        } else if (c < 0x800) {
            o += (char)(0xC0 | c >> 6);
            o += (char)(0x80 | (c & 63));
        } else if (c < 0x10000) {
            o += (char)(0xE0 | c >> 12);
            o += (char)(0x80 | (c >> 6 & 63));
            o += (char)(0x80 | (c & 63));
        } else {
            o += (char)(0xF0 | c >> 18);
            o += (char)(0x80 | (c >> 12 & 63));
            o += (char)(0x80 | (c >> 6 & 63));
            o += (char)(0x80 | (c & 63));
        }
    };
    ws();
    if (i >= n || s[i++] != '[') return false;
    ws();
    if (i < n && s[i] == ']') {
        i++;
        ws();
        return i == n;
    }
    for (;;) {
        ws();
        if (i >= n || s[i++] != '"') return false;
        std::string v;
        for (;;) {
            if (i >= n) return false;
            const uint8_t c = s[i++];
            if (c == '"') break;
            if (c < 0x20) return false;
            if (c != '\\') {
                v += (char)c;
                continue;
            }
            if (i >= n) return false;
            const uint8_t e = s[i++];
            uint32_t cp = 0;
            switch (e) {
                case '"': v += '"'; break;
                case '\\': v += '\\'; break;
                case '/': v += '/'; break;
                case 'b': v += '\b'; break;
                case 'f': v += '\f'; break;
                case 'n': v += '\n'; break;
                case 'r': v += '\r'; break;
                case 't': v += '\t'; break;
                case 'u':
                    if (!hex4(cp)) return false;
                    if (cp >= 0xD800 && cp < 0xDC00) {  // a surrogate pair
                        uint32_t lo = 0;
                        if (i + 2 > n || s[i] != '\\' || s[i + 1] != 'u') return false;
                        i += 2;
                        if (!hex4(lo) || lo < 0xDC00 || lo >= 0xE000) return false;
                        cp = 0x10000 + ((cp - 0xD800) << 10) + (lo - 0xDC00);
                    } else if (cp >= 0xDC00 && cp < 0xE000) {
                        return false;
                    }
                    put_utf8(v, cp);
                    break;
                default: return false;
            }
        }
        out.push_back(std::move(v));
        ws();
        if (i >= n) return false;
        if (s[i] == ',') {
            i++;
            continue;
        }
        if (s[i++] != ']') return false;
        ws();
        return i == n;
    }
}

bool utf8_decode(const uint8_t *s, size_t n, std::vector<uint32_t> &out) {
    out.clear();
    for (size_t i = 0; i < n;) {
        const uint8_t c = s[i];
        const int len = c < 0x80 ? 1 : (c >> 5) == 6 ? 2 : (c >> 4) == 14 ? 3 : (c >> 3) == 30 ? 4 : 0;
        if (!len || i + len > n) return false;
        uint32_t cp = len == 1 ? c : (c & (0x7F >> len));
        for (int k = 1; k < len; k++) {
            if ((s[i + k] & 0xC0) != 0x80) return false;
            cp = cp << 6 | (s[i + k] & 63);
        }
        static const uint32_t least[5] = {0, 0, 0x80, 0x800, 0x10000};  // overlong forms are not UTF-8
        if (cp < least[len] || cp > 0x10FFFF || (cp >= 0xD800 && cp < 0xE000)) return false;
        out.push_back(cp);
        i += len;
    }
    return true;
}

void build_facet_search(const RawDb &string_db, const RawDb &norm_db, const RawDb &orig_db, HostIndex &ix) {
    FacetSearchIndex &fs = ix.fsearch;
    fs = FacetSearchIndex();
    // the level-0 string keys, their posting lists (appended to the pool in key order) and smallest docids
    std::map<std::pair<uint16_t, std::string>, uint32_t> key_of;
    std::map<uint16_t, std::pair<uint32_t, uint32_t>> range;  // fid -> (first key, number of keys)
    std::map<uint16_t, uint32_t> list0;  // fid -> the list id of its first level-0 string key
    const uint32_t dense_min = dense_min_card(ix);
    std::vector<uint32_t> docs, kept, chars;
    // the fields facet search can reach: those with normalised strings (a field without them has no FST)
    std::set<uint16_t> searchable;
    for (uint64_t i = 0; i < norm_db.n; i++)
        if (norm_db.koff[i + 1] - norm_db.koff[i] >= 2) {
            const uint8_t *k = norm_db.keys.data() + norm_db.koff[i];
            searchable.insert((uint16_t)(k[0] << 8 | k[1]));
        }
    for (uint64_t i = 0; i < string_db.n; i++) {
        const uint8_t *k = string_db.keys.data() + string_db.koff[i];
        const size_t kn = string_db.koff[i + 1] - string_db.koff[i];
        if (kn < 3 || k[2] != 0) continue;
        const uint16_t fid = (uint16_t)(k[0] << 8 | k[1]);
        const uint32_t at = (uint32_t)fs.key.size();
        auto r = range.emplace(fid, std::make_pair(at, 0u)).first;
        r->second.second++;
        if (!searchable.count(fid)) {  // no list, key or original for it: a placeholder keeps the key positions
            fs.key.emplace_back();
            fs.min_doc.push_back(0);
            continue;
        }
        if (r->second.second == 1) list0[fid] = (uint32_t)ix.lists.size();
        docs.clear();
        cbo_decode_append(string_db.vals.data() + string_db.voff[i] + 1, string_db.voff[i + 1] - string_db.voff[i] - 1, docs);
        kept.clear();
        for (uint32_t d : docs)
            if (d < ix.n_docs) kept.push_back(d);
        append_list(ix, kept.data(), (uint32_t)kept.size(), dense_min);
        fs.key.emplace_back((const char *)k + 3, kn - 3);
        fs.min_doc.push_back(docs.empty() ? 0 : docs[0]);
        key_of.emplace(std::make_pair(fid, fs.key.back()), at);
    }
    // the original naming each key: field_id_docid_facet_strings at (fid, smallest docid, key)
    fs.has_orig.assign(fs.key.size(), 0);
    fs.orig.assign(fs.key.size(), std::string());
    for (auto &kv : key_of) {
        std::string probe(6, '\0');
        const uint32_t d = fs.min_doc[kv.second];
        probe[0] = (char)(kv.first.first >> 8);
        probe[1] = (char)(kv.first.first & 255);
        for (int b = 0; b < 4; b++) probe[2 + b] = (char)(d >> (24 - 8 * b) & 255);
        probe += kv.first.second;
        uint64_t lo = 0, hi = orig_db.n;
        while (lo < hi) {
            const uint64_t mid = (lo + hi) / 2;
            const size_t mn = orig_db.koff[mid + 1] - orig_db.koff[mid];
            const int c = memcmp(orig_db.keys.data() + orig_db.koff[mid], probe.data(), std::min(mn, probe.size()));
            if (c < 0 || (c == 0 && mn < probe.size()))
                lo = mid + 1;
            else
                hi = mid;
        }
        if (lo < orig_db.n && orig_db.koff[lo + 1] - orig_db.koff[lo] == probe.size() &&
            memcmp(orig_db.keys.data() + orig_db.koff[lo], probe.data(), probe.size()) == 0) {
            fs.has_orig[kv.second] = 1;
            fs.orig[kv.second].assign((const char *)orig_db.vals.data() + orig_db.voff[lo], orig_db.voff[lo + 1] - orig_db.voff[lo]);
        }
    }
    // the hyper-normalised strings, field by field in key order, and the keys each one walks
    std::vector<std::string> set;
    for (uint64_t i = 0; i < norm_db.n; i++) {
        const uint8_t *k = norm_db.keys.data() + norm_db.koff[i];
        const size_t kn = norm_db.koff[i + 1] - norm_db.koff[i];
        if (kn < 2) throw std::runtime_error("stage: facet_id_normalized_string_strings key shorter than its field id");
        const uint16_t fid = (uint16_t)(k[0] << 8 | k[1]);
        if (!parse_json_string_array(norm_db.vals.data() + norm_db.voff[i], norm_db.voff[i + 1] - norm_db.voff[i], set))
            throw std::runtime_error("stage: a facet_id_normalized_string_strings value is not a JSON array of strings");
        std::sort(set.begin(), set.end());  // a BTreeSet<String>: byte order, no duplicates, whatever order the bytes list them in
        set.erase(std::unique(set.begin(), set.end()), set.end());
        const uint32_t h = (uint32_t)fs.char_off.size() - 1;
        auto ins = fs.fields.emplace(fid, FacetSearchField());
        FacetSearchField &f = ins.first->second;
        if (ins.second) {
            f.h0 = h;
            auto r = range.find(fid);
            if (r != range.end()) {
                f.k0 = r->second.first;
                f.n_str = r->second.second;
                f.list0 = list0[fid];
            }
        } else if (f.h1 != h) {
            throw std::runtime_error("stage: facet_id_normalized_string_strings keys not in LMDB order");
        }
        f.h1 = h + 1;
        if (!utf8_decode(k + 2, kn - 2, chars)) throw std::runtime_error("stage: a facet_id_normalized_string_strings key is not valid UTF-8");
        fs.chars.insert(fs.chars.end(), chars.begin(), chars.end());
        fs.char_off.push_back((uint32_t)fs.chars.size());
        for (const std::string &s : set) {
            auto it = key_of.find(std::make_pair(fid, s));
            if (it == key_of.end()) break;  // the reference logs the missing key and skips the rest of this entry
            fs.csr_key.push_back(it->second);
        }
        fs.csr_off.push_back((uint32_t)fs.csr_key.size());
        f.n_entries += fs.csr_off[h + 1] - fs.csr_off[h];
    }
}

}  // namespace b200
