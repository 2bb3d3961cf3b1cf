/* indexgen — test/bench infrastructure, NOT product and NOT oracle.
 *
 * Replaces milli's (out-of-scope) indexer for this project: it tokenises documents,
 * and writes the posting databases the query-time path reads, in the reference's own
 * on-disk formats (SURVEY.md §A.7, §B.1, §B.2):
 *   keys   : LMDB byte keys  (word | word\0u16be | u8 prox,w1,\0,w2 | u16be fid,u8 count)
 *   values : CboRoaringBitmapCodec bytes (<=7 ints raw native-endian u32, else portable roaring)
 * What the indexer writes follows
 *   crates/milli/src/update/new/extract/searchable/extract_word_docids.rs:67-190
 *   crates/milli/src/update/new/extract/searchable/extract_word_pair_proximity_docids.rs:470-560
 *   crates/milli/src/update/new/extract/searchable/tokenize_document.rs:13-14,128-150
 *   crates/milli/src/update/new/word_fst_builder.rs:71-131 (prefix dbs)
 * Both the CPU oracle and the CUDA library are fed from these byte images, exactly as a
 * deployment would feed them from the LMDB environment.
 */
#ifndef B200_INDEXGEN_H
#define B200_INDEXGEN_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

enum ig_db_id {
    IG_DB_WORD_DOCIDS = 0,
    IG_DB_EXACT_WORD_DOCIDS = 1,
    IG_DB_WORD_PREFIX_DOCIDS = 2,
    IG_DB_EXACT_WORD_PREFIX_DOCIDS = 3,
    IG_DB_WORD_PAIR_PROXIMITY_DOCIDS = 4,
    IG_DB_WORD_POSITION_DOCIDS = 5,
    IG_DB_WORD_FID_DOCIDS = 6,
    IG_DB_WORD_PREFIX_POSITION_DOCIDS = 7,
    IG_DB_WORD_PREFIX_FID_DOCIDS = 8,
    IG_DB_FIELD_ID_WORD_COUNT_DOCIDS = 9,
    IG_DB_COUNT = 10
};

/* One LMDB-like database: n sorted byte keys and their values. */
typedef struct {
    uint64_t n_keys;
    const uint8_t *key_bytes;
    const uint64_t *key_offsets; /* n_keys+1 */
    const uint8_t *val_bytes;
    const uint64_t *val_offsets; /* n_keys+1 */
} ig_db_view;

typedef struct ig_builder ig_builder;

/* n_fields searchable fields, fid = 0..n_fields-1, weight(fid) = fid.
 * exact_mask bit f set => field f is an "exact attribute". */
ig_builder *ig_new(uint32_t n_fields, uint32_t exact_mask);
void ig_free(ig_builder *);
/* stop words: space separated, lowercase */
void ig_set_stop_words(ig_builder *, const char *words);
/* add one field value of one document (docids must be < 2^32; call per field in fid order) */
void ig_add_text(ig_builder *, uint32_t docid, uint32_t fid, const char *text);
/* Synthetic corpus (SURVEY §8(d) cfg 1-3): n_docs docs, field 0 gets len_lo..len_hi Zipf(s) words
 * over a vocab of `vocab` words (base-26 strings len 3-12, 30% are one-edit mutations of earlier
 * words so typo neighbourhoods are non-trivial); if n_fields>1, field 1 gets 20-80 words. */
void ig_add_synthetic(ig_builder *, uint32_t n_docs, uint32_t vocab, double zipf_s, uint32_t len_lo,
                      uint32_t len_hi, uint64_t seed);
/* Draw `n` query strings from the synthetic corpus per SURVEY §8(d) cfg 2:
 * 2-4 consecutive words of a random doc, 40% clean / 40% one edit / 20% two edits,
 * last word truncated to a prefix with p=0.3. Returns a malloc'ed '\n'-joined buffer. */
char *ig_synthetic_queries(ig_builder *, uint32_t n, uint64_t seed, int with_typos);
void ig_free_str(char *);
/* Same query stream as ig_synthetic_queries, from the arrays of ig_query_source (so that a corpus cached on disk can still
 * produce queries): words by intern id (bytes + n_words+1 offsets), field-0 word ids of every document (n_docs+1 offsets). */
char *ig_queries_from_arrays(const uint8_t *word_bytes, const uint64_t *word_off, const uint32_t *doc_off, uint32_t n_docs,
                             const uint32_t *doc_words, uint32_t n, uint64_t seed, int with_typos);
void ig_query_source(const ig_builder *, uint8_t **word_bytes, uint64_t **word_off, uint64_t *n_words, const uint32_t **doc_off,
                     uint64_t *n_docs, const uint32_t **doc_words, uint64_t *n_doc_words);
/* SURVEY §8(d) cfg 4 embeddings: rows [first_row, first_row + n) of an i.i.d. N(0,1), L2-normalised matrix as IEEE binary16;
 * deterministic in (seed, row), multi-threaded. */
void ig_fill_embeddings_f16(uint16_t *out, uint64_t first_row, uint64_t n, uint32_t d, uint64_t seed);
/* sort + build every database */
void ig_build(ig_builder *);
uint32_t ig_n_docs(const ig_builder *);        /* max docid + 1 */
uint64_t ig_n_words(const ig_builder *);       /* dictionary size (words fst) */
/* sorted dictionary = union of word_docids and exact_word_docids keys */
void ig_dictionary(const ig_builder *, const uint8_t **bytes, const uint64_t **offsets);
void ig_db(const ig_builder *, int db_id, ig_db_view *out);
/* all document ids, CBO encoded (main["documents-ids"]) */
void ig_documents_ids(const ig_builder *, const uint8_t **bytes, uint64_t *len);

#ifdef __cplusplus
}
#endif
#endif
