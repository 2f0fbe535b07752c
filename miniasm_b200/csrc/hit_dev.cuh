// hit_dev.cuh -- stage (i): per-read coverage trimming and containment filtering of PAF hits on the GPU.
// Counterpart of hit.c:109-256 and the shared classifier ma_hit2arc (miniasm.h:86-104).
#pragma once
#include "mab_common.cuh"
#include "asg_dev.cuh"
#include <functional>

// sharded runs: sums the per-rank counters of a log line over all ranks (installed by mab_select_sharded; null = single GPU)
typedef void (*MabCountHook)(void *ctx, unsigned long long *v, int n);
extern thread_local MabCountHook mab_count_hook;
extern thread_local void *mab_count_hook_ctx;

struct DHits {
	DHit *a = nullptr, *a2 = nullptr;   // hit array + ping-pong buffer for compaction
	size_t n = 0, m = 0;
	uint32_t n_seq = 0;
	// per-read bounds of the sorted hits, first << 32 | end (0 = the read heads no hits), n_seq entries; left by the sort and by
	// dh_select for the renumbered reads, dropped by every other pass that moves, drops or renumbers hits (null = unknown:
	// ma_hit_sub and ma_sg_gen derive them from the hits)
	uint64_t *grp = nullptr;
	// Selected, not compacted (left by dh_select; null = the hits are dense): the n kept hits still lie in their read's buckets
	// of a, under the old read ids, and grp[new id] holds those bucket bounds, which also cover the read's hits to dropped
	// targets.  map[old id] = new id or -1; off[new id] = where the read's kept hits start in the dense order (n_seq + 1 entries).
	// ma_sg_gen reads the buckets through map; every other reader calls dh_hits_dense first.
	int32_t *map = nullptr;
	uint32_t *off = nullptr;
};

struct HitArcParams { int max_hang; float int_frac; int min_ovlp; };

void dh_reserve(MabDev &d, DHits &h, size_t m);
void dh_free(MabDev &d, DHits &h);

// ma_hit_sort (hit.c:19-22): sort by the 64-bit qns (query id, then query start); stable.  A per-read bucket sort: counts per
// query read, every record scattered into its read's bucket in h.a2 with its input position i in the query-id half of qns
// (requires n < 2^32), then each bucket sorted by qs << 32 | i into h.a.  Sets h.grp.
void dh_sort(MabDev &d, DHits &h);
// The same for a caller that built the buckets itself: first = exclusive scan of the per-read counts (n_seq + 1 entries, from
// dh_bucket_first); h.a2[first[q] ..< first[q + 1]] = read q's records in any order, each with an ordinal in the query-id half of
// qns that is distinct within the bucket and increases with the hit's input order.  Sorts every bucket by qs << 32 | ordinal into
// the same positions of h.a, with q written back into the query-id half; h.a2 is left as scratch.
void dh_bucket_first(MabDev &d, const uint32_t *cnt, uint32_t n_seq, uint32_t *first);
void dh_sort_buckets(MabDev &d, DHits &h, const uint32_t *first);

// ma_hit_sub (hit.c:109-160).  sub_out: n_seq entries, fully written (zeros for reads heading no group).
// Returns the number of reads that keep an interval ("query sequences remain after sub").
uint64_t dh_sub(MabDev &d, const DHits &h, int min_dp, float min_iden, int end_clip, DSub *sub_out);

// ma_hit_cut (hit.c:162-193): clip hits to the kept intervals, drop short ones; returns the new count.
size_t dh_cut(MabDev &d, DHits &h, const DSub *reg, int min_span);

// ma_hit_flt (hit.c:195-216): drop internal / short hits; cov as the reference computes it (logged only).
size_t dh_flt(MabDev &d, DHits &h, const DSub *sub, int max_hang, int min_ovlp, float *cov);

// ma_sub_merge (hit.c:218-223)
void dh_sub_merge(MabDev &d, uint32_t n_sub, DSub *a, const DSub *b);

// ma_hit_contained (hit.c:225-256) + ma_hit_mark_unused (hit.c:24-36) + the id part of sd_squeeze
// (sdict.c:69-86).  seq_del: per-read deletion flags of the dictionary on entry (may be null = none).
// On return sub is compacted in place, hits renumbered/compacted, map_out[old] = new id or -1, and
// h.n_seq is the surviving read count.  Returns the new hit count.
size_t dh_contained(MabDev &d, DHits &h, DSub *sub, const uint8_t *seq_del, const HitArcParams &p, int32_t *map_out);
// The default read selection (main.c:119-142, -S 5 and up): ma_hit_sub, ma_hit_cut, ma_hit_flt, ma_hit_sub with end clipping,
// ma_sub_merge, ma_hit_cut and ma_hit_contained, with the same results and [M::...] lines as calling the steps above in turn.
// Runs as per-read passes over the hits' per-read buckets (h.grp; derived from the hits when null).  sub: n_seq entries, the
// merged table compacted like dh_contained's.  Returns the new hit count; h.n_seq is the surviving read count and
// map_out[old] = new id or -1.  The hits are left selected, not compacted (see DHits::map).
struct SelectParams { int min_dp; float min_iden; int min_span; int flt_max_hang, flt_min_ovlp; HitArcParams cont; };
// Callbacks of dh_select; an empty member is skipped.  step3: where the second round begins (after the ma_hit_flt line).
// sub_done(table): after each ma_hit_sub, with the n_seq rows it wrote.  flags_done(sub, used, n_seq): after the containment
// flags and "used" marks are raised, before the renumbering reads them.  A sharded run completes its per-rank rows there.
struct SelectHooks {
	std::function<void()> step3;
	std::function<void(DSub*)> sub_done;
	std::function<void(DSub*, uint8_t*, uint32_t)> flags_done;
};
size_t dh_select(MabDev &d, DHits &h, DSub *sub, const SelectParams &o, int32_t *map_out, float *cov, const SelectHooks &hk);
// The hits as the dense, qid-ordered array the step functions leave: copies the kept hits of a selection out of their buckets
// and renumbers them (nothing to do when they are dense already).
void dh_hits_dense(MabDev &d, DHits &h);
// ma_sg_gen without the final asg_cleanup: seq table + sorted local arcs (sharded runs clean up after exchanging seq flags).
// Returns the number of deleted reads when the emit counted them, else -1.  Selected hits stay in their buckets unless the
// column sort has to take them.
int64_t dh_sg_emit(MabDev &d, DHits &h, const uint32_t *len, const uint8_t *del, const HitArcParams &p, DGraph &g);

// ma_sg_gen (asm.c:9-39): lens/del per read -> graph with arcs emitted in hit order, then asg_cleanup.
void dh_sg_gen(MabDev &d, DHits &h, const uint32_t *len, const uint8_t *del, const HitArcParams &p, DGraph &g);
