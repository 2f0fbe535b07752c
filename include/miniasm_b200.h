/* miniasm_b200.h -- C ABI of libminiasm_b200.so (plain pointers and sizes; no torch, no C++ types).
 *
 * Two levels (SURVEY.md section 8b):
 *
 *  1. DROP-IN level.  The reference (lh3/miniasm @ v0.3-r179) has no plugin layer; its seam is the C API
 *     its own driver main.c:108-199 calls.  Every entry point below has the same name, argument meaning,
 *     ownership rules and stderr/exit behaviour as the reference function it replaces, so the reference's
 *     main.o links against this library unchanged (INTEGRATION.md, "link seam").  Arrays are host memory
 *     (malloc/calloc/realloc family); each call moves its operands to the GPU, runs the CUDA path and
 *     moves the result back.  The struct layouts are ABI: main.c and the writers read fields directly.
 *
 *  2. FUSED level (mab_*).  One opaque device-resident context keeps hits, arcs and the graph in HBM
 *     across stages; only counts and the final unitig graph cross PCIe.  The CLI and bench.py use this.
 *
 * There is no CPU fallback: without a usable CUDA device every entry point prints "[E::miniasm_b200]"
 * and exits non-zero.
 */
#ifndef MINIASM_B200_H
#define MINIASM_B200_H

#include <stdio.h>
#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------ ABI structs ------------------- */

/* replaces sd_seq_t / sdict_t, sdict.h:6-15 */
typedef struct { char *name; uint32_t len, aux:31, del:1; } sd_seq_t;
typedef struct { uint32_t n_seq, m_seq; sd_seq_t *seq; void *h; } sdict_t;

/* replaces asg_arc_t / asg_seq_t / asg_t, asg.h:7-23 */
typedef struct { uint64_t ul; uint32_t v; uint32_t ol:31, del:1; } asg_arc_t;
typedef struct { uint32_t len:31, del:1; } asg_seq_t;
typedef struct {
	uint32_t m_arc, n_arc:31, is_srt:1;
	asg_arc_t *arc;
	uint32_t m_seq, n_seq:31, is_symm:1;
	asg_seq_t *seq;
	uint64_t *idx;
} asg_t;

/* replaces ma_opt_t / ma_hit_t / ma_sub_t / ma_utg_t / ma_ug_t, miniasm.h:12-55 */
typedef struct {
	int min_span, min_match, min_dp;
	float min_iden;
	int max_hang, min_ovlp;
	float int_frac;
	int gap_fuzz, n_rounds, bub_dist, max_ext;
	float min_ovlp_drop_ratio, max_ovlp_drop_ratio, final_ovlp_drop_ratio;
} ma_opt_t;

typedef struct {
	uint64_t qns;
	uint32_t qe, tn, ts, te;
	uint32_t ml:31, rev:1;
	uint32_t bl:31, del:1;
} ma_hit_t;

typedef struct { uint32_t s:31, del:1, e; } ma_sub_t;

typedef struct {
	uint32_t len:31, circ:1;
	uint32_t start, end;
	uint32_t m, n;
	uint64_t *a;
	char *s;
} ma_utg_t;

typedef struct { size_t n, m; ma_utg_t *a; } ma_utg_v;
typedef struct { ma_utg_v u; asg_t *g; } ma_ug_t;

/* replaces paf_file_t / paf_rec_t, paf.h:9-24 */
#ifndef KSTRING_T
#define KSTRING_T kstring_t
typedef struct __kstring_t { size_t l, m; char *s; } kstring_t;
#endif
typedef struct { void *fp; kstring_t buf; } paf_file_t;
typedef struct {
	const char *qn, *tn;
	uint32_t ql, qs, qe, tl, ts, te;
	uint32_t ml:31, rev:1, bl;
} paf_rec_t;

extern int ma_verbose;                                   /* common.c:3 */

/* ------------------------------------------------------------------ drop-in level ------------------ */
/* host utilities (host C in the reference too): sys.c:7-46, sdict.c:8-86, paf.c:9-67, common.c:5-23 */
double sys_cputime(void);
double sys_realtime(void);
void sys_init(void);
const char *sys_timestamp(void);
sdict_t *sd_init(void);
void sd_destroy(sdict_t *d);
int32_t sd_put(sdict_t *d, const char *name, uint32_t len);
int32_t sd_get(const sdict_t *d, const char *name);
int32_t *sd_squeeze(sdict_t *d);
paf_file_t *paf_open(const char *fn);
int paf_close(paf_file_t *pf);
int paf_read(paf_file_t *pf, paf_rec_t *r);
void ma_opt_init(ma_opt_t *opt);

/* stage (i): hit.c:38-256 (miniasm.h:61-68) */
sdict_t *ma_hit_no_cont(const char *fn, int min_span, int min_match, int max_hang, float int_frac);
ma_hit_t *ma_hit_read(const char *fn, int min_span, int min_match, sdict_t *d, size_t *n, int bi_dir, const sdict_t *excl);
ma_sub_t *ma_hit_sub(int min_dp, float min_iden, int end_clip, size_t n, const ma_hit_t *a, size_t n_sub);
size_t ma_hit_cut(const ma_sub_t *reg, int min_span, size_t n, ma_hit_t *a);
size_t ma_hit_flt(const ma_sub_t *sub, int max_hang, int min_ovlp, size_t n, ma_hit_t *a, float *cov);
void ma_sub_merge(size_t n_sub, ma_sub_t *a, const ma_sub_t *b);
size_t ma_hit_contained(const ma_opt_t *opt, sdict_t *d, ma_sub_t *sub, size_t n, ma_hit_t *a);

/* stage (ii): asm.c:9-39, asg.c:11-193 (miniasm.h:70, asg.h:31-38) */
asg_t *ma_sg_gen(const ma_opt_t *opt, const sdict_t *d, const ma_sub_t *sub, size_t n_hits, const ma_hit_t *hit);
asg_t *asg_init(void);
void asg_destroy(asg_t *g);
void asg_seq_set(asg_t *g, int sid, int len, int del);
void asg_arc_sort(asg_t *g);
void asg_arc_index(asg_t *g);
void asg_arc_rm(asg_t *g);
void asg_cleanup(asg_t *g);
void asg_symm(asg_t *g);
int asg_arc_del_multi(asg_t *g);
int asg_arc_del_asymm(asg_t *g);
int asg_arc_del_trans(asg_t *g, int fuzz);

/* stage (iii): asg.c:83-101,199-433, asm.c:41-290 (asg.h:36-42, miniasm.h:71-75) */
int asg_arc_del_short(asg_t *g, float drop_ratio);
int asg_cut_tip(asg_t *g, int max_ext);
int asg_cut_internal(asg_t *g, int max_ext);
int asg_cut_biloop(asg_t *g, int max_ext);
int asg_pop_bubble(asg_t *g, int max_dist);
ma_ug_t *ma_ug_gen(asg_t *g);
int ma_ug_seq(ma_ug_t *g, const sdict_t *d, const ma_sub_t *sub, const char *fn);
void ma_ug_print(const ma_ug_t *ug, const sdict_t *d, const ma_sub_t *sub, FILE *fp);
void ma_sg_print(const asg_t *g, const sdict_t *d, const ma_sub_t *sub, FILE *fp);
void ma_ug_destroy(ma_ug_t *ug);

/* ------------------------------------------------------------------ fused level -------------------- */
typedef struct mab_ctx mab_ctx_t;

/* counters a run exposes (reference prints the same numbers in its [M::...] stderr lines) */
typedef struct {
	uint64_t n_lines, n_hits_stored, n_seq_in;          /* ma_hit_read */
	uint64_t n_hits_final, n_seq_final;                 /* after ma_hit_contained */
	uint64_t n_arc_sg;                                  /* ma_sg_gen */
	uint64_t n_arc_trans_in, n_reduced, trans_inner;    /* asg_arc_del_trans: arcs in, reduced, inner-loop iterations */
	uint64_t n_arc_final, n_utg;
	double   ms_del_trans_kernel;                       /* CUDA-event time of the transitive-reduction kernel */
	uint64_t n_kernel_launches, n_lib_calls;
	double   ms_ingest, ms_select, ms_layout, ms_unitigs; /* CUDA-event time of the last call of each step */
	uint64_t n_name_regrow;                             /* last ingest: read-name tables built again, not only for a full
	                                                       dictionary: resident parse regrown (probe limit), windowed pass 1 rerun
	                                                       (dictionary or name store full), streamed parse redone resident (full
	                                                       dictionary, more lines than estimated, line cut at a chunk), sharded
	                                                       global table re-seeded */
} mab_stats_t;

mab_ctx_t *mab_create(int device);                      /* exits if the device cannot be initialised */
void mab_destroy(mab_ctx_t *ctx);
void mab_set_verbose(int level);                        /* 0 silences the [M::...] lines of both levels */
const mab_stats_t *mab_stats(const mab_ctx_t *ctx);

/* Step 1, main.c:117-118 / hit.c:70-107.  The PAF bytes go to HBM once (from a host buffer, or from a plain/gzip
 * file through pinned staging buffers); parsing, the name dictionary, mirrored hits and ma_hit_sort run there.
 * mab_load_paf_file: a regular file that starts with the gzip magic crosses PCIe compressed and is inflated on the GPU
 * (single or concatenated members, CRC-32 and ISIZE checked); a stream the GPU decoder rejects (damaged, trailing bytes, ...)
 * and stdin ("-") go through zlib's gzread on the host, so the loaded bytes are the same either way. */
int mab_load_paf_text(mab_ctx_t *ctx, const char *text, size_t len);
int mab_load_paf_file(mab_ctx_t *ctx, const char *fn);  /* -1 if the file cannot be opened */
/* gzip-compressed PAF held in host memory, inflated on the GPU.  Returns 0, or -2 when the GPU decoder rejects the stream:
 * then nothing is loaded (the text is empty) and the caller inflates on the host and uses mab_load_paf_text. */
int mab_load_paf_gz(mab_ctx_t *ctx, const void *gz, size_t len);
/* Copies min(cap, length) bytes of the resident PAF text to dst; returns its length. */
size_t mab_paf_text(const mab_ctx_t *ctx, char *dst, size_t cap);
int mab_ingest(mab_ctx_t *ctx, int min_span, int min_match, int bi_dir);
/* load + ingest overlapped: chunks of the host text are parsed while the next ones cross PCIe (same result as the two calls) */
int mab_load_ingest_text(mab_ctx_t *ctx, const char *text, size_t len, int min_span, int min_match, int bi_dir);
/* Step 1 without the text in HBM: the PAF is taken from a source in windows of window_bytes (0 = 256 MB; at least 64 KB; a
 * longer line grows the windows) and read twice -- names, ids and hit counts first, then the hits straight into their sorted
 * place -- so the device holds two windows, the read names and the hits, whatever the size of the text.  Leaves the state
 * mab_ingest leaves (a text loaded before is dropped).  The source must deliver the same bytes after rewind: a difference
 * ends the process with exit code 78.  Returns 0; mab_ingest_windowed -1 when rewind fails (nothing ingested, the context stays
 * usable); mab_ingest_file_windowed -1 when the file cannot be opened and -2 when it cannot be rewound ("-" on a pipe).  A
 * gzip file is inflated by zlib on the host here, twice. */
typedef struct {
	size_t (*read)(void *ud, char *dst, size_t cap);  /* next bytes in order, 0 at the end */
	int    (*rewind)(void *ud);                       /* back to byte 0; -1 if impossible */
	void   *ud;
} mab_text_source_t;
int mab_ingest_windowed(mab_ctx_t *ctx, const mab_text_source_t *src, size_t window_bytes, int min_span, int min_match, int bi_dir);
int mab_ingest_file_windowed(mab_ctx_t *ctx, const char *fn, size_t window_bytes, int min_span, int min_match, int bi_dir);
/* high-water mark, in bytes, of the device memory the context's allocator handed out; reset != 0 restarts it at the current use */
size_t mab_mem_peak(mab_ctx_t *ctx, int reset);
/* device memory, in bytes, the context could still take: what the driver reports free plus what its allocator holds unused */
size_t mab_mem_free(mab_ctx_t *ctx);
/* -R: ma_hit_no_cont (hit.c:38-68) + ma_hit_read with its exclusion list (hit.c:86) as one pass over the resident text */
int mab_ingest_nocont(mab_ctx_t *ctx, int min_span, int min_match, int bi_dir, int max_hang, float int_frac);
/* alternative to load+ingest: hits and dictionary produced by the drop-in ma_hit_read (host arrays) */
int mab_load_hits(mab_ctx_t *ctx, const ma_hit_t *a, size_t n, const sdict_t *dict);

/* Steps 2-3, main.c:119-142 (ma_hit_sub/cut/flt/sub_merge/contained).  stage = the reference's -S. */
int mab_select(mab_ctx_t *ctx, const ma_opt_t *opt, int no_first, int no_second, int stage);
/* Step 4, main.c:155-188 (ma_sg_gen, asg_arc_del_trans, tip/bubble/short/internal/biloop passes) */
int mab_layout(mab_ctx_t *ctx, const ma_opt_t *opt, int stage);
/* Step 5, main.c:190-192 (ma_ug_gen) */
int mab_unitigs(mab_ctx_t *ctx);

/* Host copies in the reference's own structures (caller owns them: sd_destroy / free / asg_destroy / ma_ug_destroy) */
sdict_t *mab_export_dict(mab_ctx_t *ctx);               /* names and lengths of the current reads, ids = graph ids */
ma_sub_t *mab_export_sub(mab_ctx_t *ctx);               /* NULL when no read selection ran */
ma_hit_t *mab_export_hits(mab_ctx_t *ctx, size_t *n);
asg_t *mab_export_sg(mab_ctx_t *ctx);
ma_ug_t *mab_export_ug(mab_ctx_t *ctx);
float mab_coverage(const mab_ctx_t *ctx);
/* The bytes of ma_ug_print(mab_export_ug(), mab_export_dict(), mab_export_sub(), fp) (asm.c:77-116) for a layout without
 * unitig sequences, formatted on the GPU and written with one fwrite: no host copies of the tables.  Returns the number
 * of bytes written, -1 before mab_unitigs.  (The CLI's default writer; MAB_GPU_GFA=0 selects the host route.) */
long mab_write_gfa(mab_ctx_t *ctx, FILE *fp);
/* The other outputs of the reference's -p, formatted on the GPU and written in chunks of bounded size (device scratch and pinned
 * memory do not grow with the output).  Each returns the number of bytes written and exits with code 74 on a short write.
 * They work on a single-GPU context and on rank 0's context after mab_layout_sharded. */
long mab_write_paf(mab_ctx_t *ctx, FILE *fp); /* print_hits of main.c:21-30; -1 (nothing written) when no read selection ran */
long mab_write_bed(mab_ctx_t *ctx, FILE *fp); /* print_subs of main.c:13-19; -1 when no read selection ran */
long mab_write_sg(mab_ctx_t *ctx, FILE *fp);  /* ma_sg_print(mab_export_sg, mab_export_dict, mab_export_sub); -1 before mab_layout */
/* -f reads: ma_ug_seq (asm.c:236-290) + ma_ug_print on the GPU.  mab_reads_prefetch starts streaming the FASTA/FASTQ file (plain
 * or gzip, "-" = stdin) into HBM on a thread and stream of its own -- call it before mab_ingest and the copy hides behind the
 * graph stages; a regular gzip file crosses PCIe compressed and is inflated on the GPU, with zlib's gzread as the fallback for
 * a stream the GPU decoder rejects, as in mab_load_paf_file.  mab_write_gfa_reads indexes the records in HBM (line starts, headers, a name table of the layout's reads),
 * gathers / reverse-complements the bases straight into the S lines of the GFA text and writes it.  Returns the bytes written;
 * -1 before mab_unitigs; -2 (nothing written) when the file is neither FASTA-like nor 4-line FASTQ -- multi-line FASTQ cannot be
 * cut into records in parallel -- in which case the caller uses mab_export_* + ma_ug_seq + ma_ug_print. */
int mab_reads_prefetch(mab_ctx_t *ctx, const char *fn);
long mab_write_gfa_reads(mab_ctx_t *ctx, FILE *fp, const char *fn_reads);

/* Hash-sharded multi-GPU run (one process per GPU, read r owned by rank r mod world, NCCL on the context's stream).
 * rank 0: mab_nccl_unique_id -> launcher broadcasts the bytes -> every rank: mab_shard_init.  Each rank loads ITS byte
 * range of the PAF (ranges in rank order, cut at line ends), then ingest/select/layout_sharded; afterwards every rank
 * holds the reduced graph of the whole PAF and mab_unitigs / mab_export_* work as in a single-GPU run. */
int mab_nccl_unique_id(void *out128);
int mab_shard_init(mab_ctx_t *ctx, int rank, int world, const void *id128);
int mab_ingest_sharded(mab_ctx_t *ctx, int min_span, int min_match, int bi_dir);
int mab_load_ingest_text_sharded(mab_ctx_t *ctx, const char *text, size_t len, int min_span, int min_match, int bi_dir); /* load (this rank's byte range) + ingest, overlapped */
int mab_select_sharded(mab_ctx_t *ctx, const ma_opt_t *opt);
int mab_layout_sharded(mab_ctx_t *ctx, const ma_opt_t *opt);

/* timing helpers for bench.py: CUDA events on the context's stream */
void *mab_event_create(void);
void mab_event_record(mab_ctx_t *ctx, void *ev);
float mab_event_elapsed_ms(void *ev_begin, void *ev_end);
void mab_event_destroy(void *ev);
void mab_sync(mab_ctx_t *ctx);
void mab_last_del_trans(uint64_t *n_arc_in, uint64_t *inner, uint64_t *n_reduced, uint64_t *n_big, double *kernel_ms);
void mab_last_clean(uint32_t *rounds, uint32_t *committed);
void mab_clean_totals(uint32_t *passes, uint32_t *max_sweeps, uint32_t *sweeps, uint32_t *actions); /* tip/bubble/internal/bi-loop passes of the last mab_layout */
void mab_count_del_trans_inner(int on);                /* 1: asg_arc_del_trans also counts inner-loop iterations (mab_stats_t::trans_inner); costs time */

#ifdef __cplusplus
}
#endif

#endif
