// ingest_dev.cuh -- PAF text -> sorted hit array, entirely on the GPU (SURVEY.md 8f.1; reference: paf.c:34-67
// paf_parse/paf_read, hit.c:70-107 ma_hit_read, sdict.c:27-45 sd_put).
#pragma once
#include "mab_common.cuh"
#include "hit_dev.cuh"

// name table of the reads, in id order (id = rank of first appearance among filter-passing lines,
// query before target: hit.c:87-90 + sdict.c:27-45)
struct DNames {
	uint32_t n_seq = 0;
	uint64_t *off = nullptr;     // byte offset of the name in the PAF text (first occurrence)
	uint32_t *nlen = nullptr;    // name length in bytes
	uint32_t *slen = nullptr;    // sequence length recorded at first appearance
};

// name_regrow: how often the ingest built its read-name table again.  Not only dictionary overflows: it counts the resident parse
// regrown after a probe run hit its limit; every rerun of windowed pass 1, whether the dictionary or only the name store was full;
// every streamed parse given up for the resident one, whether for a full dictionary, more lines than estimated or a line cut at a
// chunk; and every re-seed of the sharded global table (hash_retries of them)
struct IngestStats { uint64_t n_lines, n_parsed, n_hits, n_seq, tot_len, n_dropped; int hash_retries; uint32_t name_regrow; };
struct NoContParams { int max_hang; float int_frac; }; // -R (ma_hit_no_cont, hit.c:38-68)

// d_text: the PAF bytes in device memory.  On return `h` holds the sorted hits (ma_hit_sort order, stable) and
// `names` the dictionary.  Exits loudly on malformed sizes (> 2^31 hits per GPU).
// nocont != nullptr: the reference's -R, i.e. reads clearly contained in a much longer read are dropped together with every
// line that names them before ids are assigned (st.n_dropped = their number).
void ingest_paf(MabDev &d, const char *d_text, size_t len, int min_span, int min_match, int bi_dir,
                DHits &h, DNames &names, IngestStats &st, const NoContParams *nocont = nullptr);
// load + ingest overlapped: host_text -> d_text in chunks on MabDev::copy_stream while arrived chunks are scanned and parsed
void ingest_paf_stream(MabDev &d, char *d_text, const char *host_text, size_t len, int min_span, int min_match, int bi_dir,
                       DHits &h, DNames &names, IngestStats &st);
// Windowed ingest: the text is delivered in order by `src` (read: the next bytes, 0 at the end; rewind: back to byte 0, nonzero
// if impossible) and read twice, window_bytes (>= 64 KB, grown to the longest line) at a time; the device holds two windows, the
// dictionary, a packed name store and the hits, never the text.  Same hits, names (names.off indexes *name_text_out, which the
// caller frees) and counters as ingest_paf.  size_hint: bytes of the text when known (sizes the dictionary), else 0.
// false: the source could not be rewound and nothing was ingested.  A source whose second delivery differs exits with code 78.
// A device source (read == nullptr, fill set) writes the text straight into the device windows on the ingest's stream: fill returns
// the bytes written (0 at the end), TS_FULL when its next piece is longer than cap (the window is cut at its last line, or grows),
// or TS_FAIL; a TS_FAIL in pass 1 gives false with nothing ingested, in pass 2 exit 78.
enum { TS_FULL = -3, TS_FAIL = -2 };
struct TextSource {
	size_t (*read)(void *ud, char *dst, size_t cap); int (*rewind)(void *ud); void *ud;
	int64_t (*fill)(void *ud, char *d_dst, size_t cap);
};
bool ingest_paf_windowed(MabDev &d, const TextSource &src, size_t window_bytes, size_t size_hint, int min_span, int min_match, int bi_dir,
                         DHits &h, DNames &names, char **name_text_out, IngestStats &st);
void names_free(MabDev &d, DNames &n);
// byte offsets of the line starts of a text in device memory (len > 0); free with d.free.  start[n_lines] is not set.
uint64_t *dev_line_starts(MabDev &d, const char *d_text, size_t len, uint64_t *n_lines_out);
// FNV-1a + finaliser over the bytes [s, t) of p, never 0: the read-name hash of the dictionaries
__host__ __device__ __forceinline__ uint64_t fmix64(uint64_t k)
{
	k ^= k >> 33; k *= 0xff51afd7ed558ccdULL; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ULL; k ^= k >> 33;
	return k;
}

__host__ __device__ __forceinline__ uint64_t name_hash(const char *p, uint32_t s, uint32_t t, uint64_t seed)
{
	uint64_t h = 1469598103934665603ULL ^ seed;
	for (uint32_t i = s; i < t; ++i) h = (h ^ (uint8_t)p[i]) * 1099511628211ULL;
	h = fmix64(h);
	return h ? h : 1;
}



struct ShardComm;
// Sharded variant: this rank's byte range of the PAF in, the hits of the reads this rank owns out (SURVEY.md 8e).
// *name_text_out receives a device buffer with all read names packed (names.off indexes it); the caller frees it.
// host_text != nullptr: the bytes are still on the host and cross PCIe in chunks while the arrived chunks are parsed.
void ingest_paf_sharded(MabDev &d, ShardComm &sc, char *d_text, size_t len, int min_span, int min_match, int bi_dir,
                        DHits &h, DNames &names, char **name_text_out, IngestStats &st, const char *host_text = nullptr);
