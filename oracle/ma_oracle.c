/* ma_oracle.c -- ORACLE / TEST INFRASTRUCTURE.  NOT part of the product: nothing under miniasm_b200/ links,
 * loads or calls this file; only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may.
 *
 * A sequential CPU restatement, in plain C, of the PAF -> string graph -> unitig path of lh3/miniasm
 * v0.3-r179, written from the behaviour of the reference (citations are file:line into the reference's sources).
 * It exports the reference's own C API names, so the same ctypes driver (miniasm_b200/pipeline.py) can run
 * the reference, this port and the CUDA product side by side.
 *
 * PARITY PIN: the reference ships no tests or golden vectors (SURVEY.md section 4).  This port is pinned by
 * (a) tests/test_oracle_cpu.py, which runs it step by step against the unmodified reference compiled into
 * oracle/_ref/libminiasm_ref.so, and (b) the committed fixtures under tests/golden/ that were produced by
 * the reference binary (tests/golden/make_golden.py).
 *
 * Known, documented difference: both sorts here are STABLE merge sorts; the reference uses an in-place
 * unstable radix sort (ksort.h:134-183), so records with equal keys may come out in another order.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <stdint.h>
#include <assert.h>
#include "ma_oracle.h"

int ma_verbose = 0;

/* ------------------------------------------------------------------ options: common.c:5-23 */
void ma_opt_init(ma_opt_t *o)
{
	o->min_span = 2000; o->min_match = 100; o->min_dp = 3; o->min_iden = .05f;
	o->max_hang = 1000; o->min_ovlp = o->min_span; o->int_frac = .8f;
	o->gap_fuzz = 1000; o->n_rounds = 2; o->bub_dist = 50000; o->max_ext = 4;
	o->min_ovlp_drop_ratio = .5f; o->max_ovlp_drop_ratio = .7f; o->final_ovlp_drop_ratio = .8f;
}

/* ------------------------------------------------------------------ dictionary: sdict.c:8-86 (linear-probing table) */
typedef struct { uint32_t cap, used; int32_t *slot; } oidx_t;

static uint32_t ohash(const char *s) { uint32_t h = 2166136261u; for (; *s; ++s) h = (h ^ (uint8_t)*s) * 16777619u; return h; }

static void oidx_put(oidx_t *x, const sdict_t *d, int32_t id)
{
	uint32_t k = ohash(d->seq[id].name) & (x->cap - 1);
	while (x->slot[k] >= 0) k = (k + 1) & (x->cap - 1);
	x->slot[k] = id; ++x->used;
}

static void oidx_build(sdict_t *d, uint32_t min_cap)
{
	oidx_t *x = (oidx_t*)calloc(1, sizeof(oidx_t));
	uint32_t i;
	x->cap = 64;
	while (x->cap < min_cap || x->cap < 2 * d->n_seq + 2) x->cap <<= 1;
	x->slot = (int32_t*)malloc(4 * (size_t)x->cap);
	memset(x->slot, 0xff, 4 * (size_t)x->cap);
	for (i = 0; i < d->n_seq; ++i) oidx_put(x, d, (int32_t)i);
	if (d->h) { free(((oidx_t*)d->h)->slot); free(d->h); }
	d->h = x;
}

sdict_t *sd_init(void) { sdict_t *d = (sdict_t*)calloc(1, sizeof(sdict_t)); oidx_build(d, 64); return d; }

void sd_destroy(sdict_t *d)
{
	uint32_t i;
	if (!d) return;
	for (i = 0; i < d->n_seq; ++i) free(d->seq[i].name);
	if (d->h) { free(((oidx_t*)d->h)->slot); free(d->h); }
	free(d->seq); free(d);
}

int32_t sd_get(const sdict_t *d, const char *name)
{
	const oidx_t *x = (const oidx_t*)d->h;
	uint32_t k;
	for (k = ohash(name) & (x->cap - 1); x->slot[k] >= 0; k = (k + 1) & (x->cap - 1))
		if (strcmp(d->seq[x->slot[k]].name, name) == 0) return x->slot[k];
	return -1;
}

int32_t sd_put(sdict_t *d, const char *name, uint32_t len)
{
	int32_t id = sd_get(d, name);
	if (id >= 0) return id;
	if (d->n_seq == d->m_seq) { d->m_seq = d->m_seq ? d->m_seq * 2 : 16; d->seq = (sd_seq_t*)realloc(d->seq, d->m_seq * sizeof(sd_seq_t)); }
	d->seq[d->n_seq].name = strdup(name); d->seq[d->n_seq].len = len; d->seq[d->n_seq].aux = 0; d->seq[d->n_seq].del = 0;
	++d->n_seq;
	if (2 * d->n_seq + 2 > ((oidx_t*)d->h)->cap) oidx_build(d, 0);
	else oidx_put((oidx_t*)d->h, d, (int32_t)d->n_seq - 1);
	return (int32_t)d->n_seq - 1;
}

int32_t *sd_squeeze(sdict_t *d)
{
	int32_t *map = (int32_t*)calloc(d->n_seq ? d->n_seq : 1, 4);
	uint32_t i, j;
	for (i = j = 0; i < d->n_seq; ++i)
		if (d->seq[i].del) { free(d->seq[i].name); map[i] = -1; }
		else { d->seq[j] = d->seq[i]; map[i] = (int32_t)j++; }
	d->n_seq = j;
	oidx_build(d, 0);
	return map;
}

/* ------------------------------------------------------------------ stable sorts by a 64-bit key */
static void msort64(size_t n, void *base, size_t width, size_t key_off)
{ /* bottom-up merge sort of records whose uint64 key sits at key_off */
	char *a = (char*)base, *b = (char*)malloc(n * width + 1), *src = a, *dst = b, *t;
	size_t w, i;
	for (w = 1; w < n; w <<= 1) {
		for (i = 0; i < n; i += 2 * w) {
			size_t l = i, m = i + w < n ? i + w : n, r = i + 2 * w < n ? i + 2 * w : n, p = l, q = m, k = l;
			while (p < m && q < r) {
				uint64_t kp, kq;
				memcpy(&kp, src + p * width + key_off, 8); memcpy(&kq, src + q * width + key_off, 8);
				if (kq < kp) memcpy(dst + k++ * width, src + q++ * width, width);
				else memcpy(dst + k++ * width, src + p++ * width, width);
			}
			if (p < m) memcpy(dst + k * width, src + p * width, (m - p) * width), k += m - p;
			if (q < r) memcpy(dst + k * width, src + q * width, (r - q) * width);
		}
		t = src; src = dst; dst = t;
	}
	if (src != a) memcpy(a, src, n * width);
	free(b);
}

static int cmp_u32(const void *x, const void *y) { uint32_t a = *(const uint32_t*)x, b = *(const uint32_t*)y; return a < b ? -1 : a > b; }

/* ------------------------------------------------------------------ PAF reading + hit loading: paf.c:34-67, hit.c:70-107 */
typedef struct { char *qn, *tn; uint32_t ql, qs, qe, tl, ts, te, ml, bl, rev; } oline_t;

/* one PAF line (terminated in place) -> fields; 0 if it has fewer than 10 columns (paf.c:34-56).  *stale_bl carries the 11th
 * column of the last line that had one: a 10-column line keeps it */
static int paf_fields(char *line, ssize_t len, oline_t *r, uint32_t *stale_bl)
{
	char *f[12], *p = line;
	int nf = 0;
	if (len && line[len - 1] == '\n') line[--len] = 0;
	if (len > 1 && line[len - 1] == '\r') line[--len] = 0;       /* kseq.h:143 */
	for (f[nf++] = p; *p && nf < 12; ++p) if (*p == '\t') { *p = 0; f[nf++] = p + 1; }
	if (nf < 10) return 0;                                       /* paf.c:54 */
	r->qn = f[0], r->tn = f[5];
	r->ql = (uint32_t)strtol(f[1], 0, 10); r->qs = (uint32_t)strtol(f[2], 0, 10); r->qe = (uint32_t)strtol(f[3], 0, 10);
	r->rev = f[4][0] == '-';
	r->tl = (uint32_t)strtol(f[6], 0, 10); r->ts = (uint32_t)strtol(f[7], 0, 10); r->te = (uint32_t)strtol(f[8], 0, 10);
	r->ml = (uint32_t)strtol(f[9], 0, 10) & 0x7fffffffu;
	if (nf >= 11) { char *e = strchr(f[10], '\t'); if (e) *e = 0; *stale_bl = (uint32_t)strtol(f[10], 0, 10); }
	r->bl = *stale_bl;
	return 1;
}

/* the filter both passes over the PAF apply before anything else (hit.c:57 and hit.c:85): unsigned spans, signed match count */
static int too_small(const oline_t *r, int min_span, int min_match)
{
	return r->qe - r->qs < (uint32_t)min_span || r->te - r->ts < (uint32_t)min_span || (int)r->ml < min_match;
}

ma_hit_t *ma_hit_read(const char *fn, int min_span, int min_match, sdict_t *d, size_t *n, int bi_dir, const sdict_t *excl)
{
	FILE *fp = fopen(fn, "rb");
	char *line = 0;
	size_t cap = 0, n_a = 0, m_a = 0;
	ssize_t len;
	ma_hit_t *a = 0;
	uint32_t stale_bl = 0;
	if (!fp) { fprintf(stderr, "[E::%s] could not open PAF file %s\n", __func__, fn); exit(1); }
	while ((len = getline(&line, &cap, fp)) >= 0) {
		oline_t r;
		if (!paf_fields(line, len, &r, &stale_bl)) continue;
		if (too_small(&r, min_span, min_match)) continue;        /* hit.c:85 */
		if (excl && (sd_get(excl, r.qn) >= 0 || sd_get(excl, r.tn) >= 0)) continue;
		if (n_a + 2 > m_a) { m_a = m_a ? m_a * 2 : 256; a = (ma_hit_t*)realloc(a, m_a * sizeof(ma_hit_t)); }
		{
			uint32_t qid = (uint32_t)sd_put(d, r.qn, r.ql), tid = (uint32_t)sd_put(d, r.tn, r.tl);
			ma_hit_t *h = &a[n_a++];
			memset(h, 0, sizeof(*h));
			h->qns = (uint64_t)qid << 32 | r.qs; h->qe = r.qe; h->tn = tid; h->ts = r.ts; h->te = r.te; h->rev = r.rev; h->ml = r.ml; h->bl = r.bl;
			if (bi_dir && qid != tid) {                          /* mirrored hit, hit.c:92-98 */
				h = &a[n_a++];
				memset(h, 0, sizeof(*h));
				h->qns = (uint64_t)tid << 32 | r.ts; h->qe = r.te; h->tn = qid; h->ts = r.qs; h->te = r.qe; h->rev = r.rev; h->ml = r.ml; h->bl = r.bl;
			}
		}
	}
	free(line); fclose(fp);
	msort64(n_a, a, sizeof(ma_hit_t), 0);                        /* ma_hit_sort, hit.c:19-22 */
	*n = n_a;
	return a;
}

/* ------------------------------------------------------------------ -R prefilter: hit.c:38-68
 * A first pass over the PAF that names the reads to leave out: a read lying, with short overhangs, well inside a read more
 * than twice its length.  The result is the `excl` dictionary of ma_hit_read. */
sdict_t *ma_hit_no_cont(const char *fn, int min_span, int min_match, int max_hang, float int_frac)
{
	FILE *fp = fopen(fn, "rb");
	char *line = 0;
	size_t cap = 0;
	ssize_t len;
	uint32_t stale_bl = 0;
	sdict_t *d;
	const int near = max_hang >> 2, far = max_hang << 1;
	if (!fp) { fprintf(stderr, "[E::%s] could not open PAF file %s\n", __func__, fn); exit(1); }
	d = sd_init();
	while ((len = getline(&line, &cap, fp)) >= 0) {
		oline_t r;
		int t5, t3;                                              /* target bases beyond the match, at the query's 5' / 3' side */
		if (!paf_fields(line, len, &r, &stale_bl) || too_small(&r, min_span, min_match)) continue;
		t5 = (int)(r.rev ? r.tl - r.te : r.ts), t3 = (int)(r.rev ? r.ts : r.tl - r.te);
		if (r.ql >> 1 > r.tl) {                                  /* long query, short target: hit.c:60-63 */
			if (t5 > near || t3 > near || (float)(r.te - r.ts) < (float)r.tl * int_frac) continue;
			if ((int)r.qs - t5 > far && (int)(r.ql - r.qe) - t3 > far) sd_put(d, r.tn, r.tl);
		} else if (r.ql < r.tl >> 1) {                           /* the mirror case: hit.c:64-67 (unsigned compares on the query side) */
			if (r.qs > (uint32_t)near || r.ql - r.qe > (uint32_t)near || (float)(r.qe - r.qs) < (float)r.ql * int_frac) continue;
			if (t5 - (int)r.qs > far && t3 - (int)(r.ql - r.qe) > far) sd_put(d, r.qn, r.ql);
		}
	}
	free(line); fclose(fp);
	if (ma_verbose >= 3) fprintf(stderr, "[M::%s] dropped %d contained reads\n", __func__, d->n_seq);
	return d;
}

/* ------------------------------------------------------------------ the classifier: miniasm.h:86-104 */
enum { O_INT = -1, O_QCONT = -2, O_TCONT = -3, O_SHORT = -4 };

static int hit2arc(const ma_hit_t *h, int ql, int tl, int max_hang, float int_frac, int min_ovlp, asg_arc_t *p)
{
	int32_t qs = (int32_t)(uint32_t)h->qns, tl5, tl3, ext5, ext3;
	uint32_t q3 = (uint32_t)ql - h->qe, span = h->qe - (uint32_t)qs, full, u, v, l;
	if (h->rev) tl5 = (int32_t)((uint32_t)tl - h->te), tl3 = (int32_t)h->ts;
	else tl5 = (int32_t)h->ts, tl3 = (int32_t)((uint32_t)tl - h->te);
	ext5 = qs < tl5 ? qs : tl5;
	ext3 = (int32_t)(q3 < (uint32_t)tl3 ? q3 : (uint32_t)tl3);
	full = span + (uint32_t)ext5 + (uint32_t)ext3;
	if (ext5 > max_hang || ext3 > max_hang || (float)span < (float)full * int_frac) return O_INT;
	if (qs <= tl5 && q3 <= (uint32_t)tl3) return O_QCONT;
	if (qs >= tl5 && q3 >= (uint32_t)tl3) return O_TCONT;
	if (qs > tl5) u = 0, v = !!h->rev, l = (uint32_t)qs - (uint32_t)tl5;
	else u = 1, v = !h->rev, l = q3 - (uint32_t)tl3;
	if (full < (uint32_t)min_ovlp || h->te - h->ts + (uint32_t)ext5 + (uint32_t)ext3 < (uint32_t)min_ovlp) return O_SHORT;
	u |= (uint32_t)(h->qns >> 32) << 1; v |= h->tn << 1;
	p->ul = (uint64_t)u << 32 | l; p->v = v; p->ol = (uint32_t)ql - l; p->del = 0;
	return (int)l;
}

/* ------------------------------------------------------------------ stage (i): hit.c:109-256 */
ma_sub_t *ma_hit_sub(int min_dp, float min_iden, int end_clip, size_t n, const ma_hit_t *a, size_t n_sub)
{
	ma_sub_t *sub = (ma_sub_t*)calloc(n_sub ? n_sub : 1, sizeof(ma_sub_t));
	uint32_t *ev = 0;
	size_t i, j, first, m_ev = 0;
	for (first = 0, i = 1; i <= n; ++i) {
		uint32_t qid, n_ev = 0, start = 0, best_s = 0, best_e = 0;
		int depth = 0;
		if (i < n && a[i].qns >> 32 == a[i - 1].qns >> 32) continue;
		qid = (uint32_t)(a[i - 1].qns >> 32);
		if (2 * (i - first) > m_ev) { m_ev = 2 * (i - first); ev = (uint32_t*)realloc(ev, 4 * m_ev); }
		for (j = first; j < i; ++j) {            /* interval ends of the usable hits of this read */
			uint32_t s, e;
			if (a[j].tn == qid || (float)(int)a[j].ml < (float)(int)a[j].bl * min_iden) continue;
			s = (uint32_t)a[j].qns + (uint32_t)end_clip; e = a[j].qe - (uint32_t)end_clip;
			if (e > s) { ev[n_ev++] = s << 1; ev[n_ev++] = e << 1 | 1; }
		}
		qsort(ev, n_ev, 4, cmp_u32);
		for (j = 0; j < n_ev; ++j) {             /* depth sweep; the first longest stretch with depth >= min_dp wins */
			int before = depth;
			depth += ev[j] & 1 ? -1 : 1;
			if (before < min_dp && depth >= min_dp) start = ev[j] >> 1;
			else if (before >= min_dp && depth < min_dp && (ev[j] >> 1) - start > best_e - best_s) best_s = start, best_e = ev[j] >> 1;
		}
		if (best_e - best_s > 0) { sub[qid].s = best_s - (uint32_t)end_clip; sub[qid].e = best_e + (uint32_t)end_clip; sub[qid].del = 0; }
		else sub[qid].del = 1;
		first = i;
	}
	free(ev);
	return sub;
}

size_t ma_hit_cut(const ma_sub_t *reg, int min_span, size_t n, ma_hit_t *a)
{
	size_t i, m = 0;
	for (i = 0; i < n; ++i) {
		ma_hit_t h = a[i];
		const ma_sub_t *rq = &reg[h.qns >> 32], *rt = &reg[h.tn];
		uint32_t pqs = (uint32_t)h.qns, rqs = rq->s, rts = rt->s, uqs, uqe, uts, ute;
		int qs, qe, ts, te;
		if (rq->del || rt->del) continue;
		if (h.rev) {   /* clip of the target maps to the opposite end of the query (hit.c:169-174) */
			uqs = h.te < rt->e ? pqs : pqs + (h.te - rt->e);
			uqe = h.ts > rts ? h.qe : h.qe - (rts - h.ts);
			uts = h.qe < rq->e ? h.ts : h.ts + (h.qe - rq->e);
			ute = pqs > rqs ? h.te : h.te - (rqs - pqs);
		} else {
			uqs = h.ts > rts ? pqs : pqs + (rts - h.ts);
			uqe = h.te < rt->e ? h.qe : h.qe - (h.te - rt->e);
			uts = pqs > rqs ? h.ts : h.ts + (rqs - pqs);
			ute = h.qe < rq->e ? h.te : h.te - (h.qe - rq->e);
		}
		qs = (int)uqs; qe = (int)uqe; ts = (int)uts; te = (int)ute;
		qs = (qs > (int)rqs ? qs : (int)rqs) - (int)rqs;
		qe = (int)(((uint32_t)qe < rq->e ? (uint32_t)qe : rq->e) - rqs);
		ts = (ts > (int)rts ? ts : (int)rts) - (int)rts;
		te = (int)(((uint32_t)te < rt->e ? (uint32_t)te : rt->e) - rts);
		if (qe - qs >= min_span && te - ts >= min_span) {
			h.qns = (h.qns >> 32 << 32) | (uint64_t)(int64_t)qs; h.qe = (uint32_t)qe; h.ts = (uint32_t)ts; h.te = (uint32_t)te;
			a[m++] = h;
		}
	}
	return m;
}

size_t ma_hit_flt(const ma_sub_t *sub, int max_hang, int min_ovlp, size_t n, ma_hit_t *a, float *cov)
{
	size_t i, m = 0;
	uint64_t tot_dp = 0, tot_len = 0;
	asg_arc_t t;
	for (i = 0; i < n; ++i) {
		const ma_sub_t *sq = &sub[a[i].qns >> 32], *st = &sub[a[i].tn];
		int r;
		if (sq->del || st->del) continue;
		r = hit2arc(&a[i], (int)(sq->e - sq->s), (int)(st->e - st->s), max_hang, .5f, min_ovlp, &t);
		if (r >= 0 || r == O_QCONT || r == O_TCONT) {
			tot_dp += r >= 0 ? (uint32_t)r : r == O_QCONT ? sq->e - sq->s : st->e - st->s;
			a[m++] = a[i];
		}
	}
	for (i = 1; i <= m; ++i)
		if (i == m || a[i].qns >> 32 != a[i - 1].qns >> 32) tot_len += sub[a[i - 1].qns >> 32].e - sub[a[i - 1].qns >> 32].s;
	*cov = (float)((double)tot_dp / tot_len);
	return m;
}

void ma_sub_merge(size_t n_sub, ma_sub_t *a, const ma_sub_t *b)
{
	size_t i;
	for (i = 0; i < n_sub; ++i) { a[i].e = a[i].s + b[i].e; a[i].s += b[i].s; }
}

size_t ma_hit_contained(const ma_opt_t *opt, sdict_t *d, ma_sub_t *sub, size_t n, ma_hit_t *a)
{
	size_t i, m = 0, n_old = d->n_seq;
	int32_t *map;
	asg_arc_t t;
	for (i = 0; i < d->n_seq; ++i) d->seq[i].aux = 0;
	for (i = 0; i < n; ++i) {
		ma_sub_t *sq = &sub[a[i].qns >> 32], *st = &sub[a[i].tn];
		int r = hit2arc(&a[i], (int)(sq->e - sq->s), (int)(st->e - st->s), opt->max_hang, opt->int_frac, opt->min_ovlp, &t);
		if (r == O_QCONT) sq->del = 1; else if (r == O_TCONT) st->del = 1;
		d->seq[a[i].qns >> 32].aux = d->seq[a[i].tn].aux = 1;   /* ma_hit_mark_unused, hit.c:24-36 */
	}
	for (i = 0; i < d->n_seq; ++i) { if (sub[i].del || !d->seq[i].aux) d->seq[i].del = 1; d->seq[i].aux = 0; }
	map = sd_squeeze(d);
	for (i = 0; i < n_old; ++i) if (map[i] >= 0) sub[map[i]] = sub[i];
	for (i = 0; i < n; ++i) {
		int32_t q = map[a[i].qns >> 32], t2 = map[a[i].tn];
		if (q < 0 || t2 < 0) continue;
		a[i].qns = (uint64_t)(uint32_t)q << 32 | (uint32_t)a[i].qns; a[i].tn = (uint32_t)t2;
		a[m++] = a[i];
	}
	free(map);
	return m;
}

/* ------------------------------------------------------------------ graph container: asg.c:11-145 */
#define A_N(g, v) ((uint32_t)(g)->idx[(v)])
#define A_A(g, v) (&(g)->arc[(g)->idx[(v)] >> 32])

asg_t *asg_init(void) { return (asg_t*)calloc(1, sizeof(asg_t)); }
void asg_destroy(asg_t *g) { if (g) { free(g->seq); free(g->idx); free(g->arc); free(g); } }

void asg_seq_set(asg_t *g, int sid, int len, int del)
{
	if ((uint32_t)sid >= g->m_seq) { uint32_t m = 16; while (m <= (uint32_t)sid) m <<= 1; g->m_seq = m; g->seq = (asg_seq_t*)realloc(g->seq, 4 * (size_t)m); }
	if ((uint32_t)sid >= g->n_seq) g->n_seq = sid + 1;
	g->seq[sid].len = len; g->seq[sid].del = !!del;
}

static asg_arc_t *arc_push(asg_t *g)
{
	if (g->n_arc == g->m_arc) { g->m_arc = g->m_arc ? g->m_arc * 2 : 16; g->arc = (asg_arc_t*)realloc(g->arc, 16 * (size_t)g->m_arc); }
	return &g->arc[g->n_arc++];
}

void asg_arc_rm(asg_t *g)
{
	uint32_t i, n = 0;
	for (i = 0; i < g->n_arc; ++i) {
		const asg_arc_t *a = &g->arc[i];
		if (!a->del && !g->seq[a->ul >> 33].del && !g->seq[a->v >> 1].del) g->arc[n++] = *a;
	}
	if (n < g->n_arc) { free(g->idx); g->idx = 0; }
	g->n_arc = n;
}

void asg_arc_sort(asg_t *g) { msort64(g->n_arc, g->arc, sizeof(asg_arc_t), 0); }

void asg_arc_index(asg_t *g)
{
	uint32_t i, first = 0;
	free(g->idx);
	g->idx = (uint64_t*)calloc((size_t)g->n_seq * 2 + 1, 8);
	for (i = 1; i <= g->n_arc; ++i)
		if (i == g->n_arc || g->arc[i].ul >> 32 != g->arc[i - 1].ul >> 32) { g->idx[g->arc[i - 1].ul >> 32] = (uint64_t)first << 32 | (i - first); first = i; }
}

void asg_cleanup(asg_t *g)
{
	asg_arc_rm(g);
	if (!g->is_srt) { asg_arc_sort(g); g->is_srt = 1; }
	if (!g->idx) asg_arc_index(g);
}

int asg_arc_del_multi(asg_t *g)
{
	uint32_t v, n_vtx = g->n_seq * 2, n = 0;
	for (v = 0; v < n_vtx; ++v) {
		asg_arc_t *av = A_A(g, v);
		uint32_t i, j, nv = A_N(g, v);
		for (i = 1; i < nv; ++i)                    /* an arc with an earlier arc to the same target goes */
			for (j = 0; j < i; ++j) if (av[j].v == av[i].v) { av[i].del = 1; ++n; break; }
	}
	if (n) asg_cleanup(g);
	return (int)n;
}

int asg_arc_del_asymm(asg_t *g)
{
	uint32_t e, n = 0;
	for (e = 0; e < g->n_arc; ++e) {
		uint32_t v = g->arc[e].v ^ 1, u = (uint32_t)(g->arc[e].ul >> 32) ^ 1, i, nv = A_N(g, v);
		const asg_arc_t *av = A_A(g, v);
		for (i = 0; i < nv && av[i].v != u; ++i);
		if (i == nv) { g->arc[e].del = 1; ++n; }
	}
	if (n) asg_cleanup(g);
	return (int)n;
}

void asg_symm(asg_t *g) { asg_arc_del_multi(g); asg_arc_del_asymm(g); g->is_symm = 1; }

/* ------------------------------------------------------------------ ma_sg_gen: asm.c:9-39 */
asg_t *ma_sg_gen(const ma_opt_t *opt, const sdict_t *d, const ma_sub_t *sub, size_t n_hits, const ma_hit_t *hit)
{
	asg_t *g = asg_init();
	size_t i;
	for (i = 0; i < d->n_seq; ++i)
		asg_seq_set(g, (int)i, sub ? (int)(sub[i].e - sub[i].s) : (int)d->seq[i].len, sub ? (sub[i].del || d->seq[i].del) : d->seq[i].del);
	for (i = 0; i < n_hits; ++i) {
		const ma_hit_t *h = &hit[i];
		uint32_t q = (uint32_t)(h->qns >> 32);
		asg_arc_t t;
		/* the 32-bit lengths (asm.c:23-24): asg_seq_t::len keeps only 31 bits of them */
		int ql = sub ? (int)(sub[q].e - sub[q].s) : (int)d->seq[q].len, tl = sub ? (int)(sub[h->tn].e - sub[h->tn].s) : (int)d->seq[h->tn].len;
		int r = hit2arc(h, ql, tl, opt->max_hang, opt->int_frac, opt->min_ovlp, &t);
		if (r >= 0) {
			if (q == h->tn) { if ((uint32_t)h->qns == h->ts && h->qe == h->te && h->rev) g->seq[q].del = 1; }
			else *arc_push(g) = t;
		} else if (r == O_QCONT) g->seq[q].del = 1;
	}
	asg_cleanup(g);
	return g;
}

/* ------------------------------------------------------------------ transitive reduction, short overlaps: asg.c:83-101,148-193 */
int asg_arc_del_trans(asg_t *g, int fuzz)
{
	uint32_t v, n_vtx = g->n_seq * 2, n = 0;
	uint8_t *mark = (uint8_t*)calloc(n_vtx ? n_vtx : 1, 1);
	for (v = 0; v < n_vtx; ++v) {
		uint32_t i, j, nv = A_N(g, v), L;
		asg_arc_t *av = A_A(g, v);
		if (nv == 0) continue;
		if (g->seq[v >> 1].del) { for (i = 0; i < nv; ++i) av[i].del = 1; n += nv; continue; }
		for (i = 0; i < nv; ++i) mark[av[i].v] = 1;
		L = (uint32_t)av[nv - 1].ul + (uint32_t)fuzz;
		for (i = 0; i < nv; ++i) {
			uint32_t w = av[i].v, nw = A_N(g, w);
			const asg_arc_t *aw = A_A(g, w);
			if (mark[w] != 1) continue;
			for (j = 0; j < nw && (uint32_t)aw[j].ul + (uint32_t)av[i].ul <= L; ++j) if (mark[aw[j].v]) mark[aw[j].v] = 2;
		}
		for (i = 0; i < nv; ++i) { if (mark[av[i].v] == 2) av[i].del = 1, ++n; mark[av[i].v] = 0; }
	}
	free(mark);
	if (n) { asg_cleanup(g); asg_symm(g); }
	return (int)n;
}

int asg_arc_del_short(asg_t *g, float ratio)
{
	uint32_t v, n_vtx = g->n_seq * 2, n = 0;
	for (v = 0; v < n_vtx; ++v) {
		asg_arc_t *av = A_A(g, v);
		uint32_t i, nv = A_N(g, v), thres;
		if (nv < 2) continue;
		thres = (uint32_t)((int)av[0].ol * ratio + .499);
		for (i = nv - 1; i >= 1 && av[i].ol < thres; --i);
		for (++i; i < nv; ++i) av[i].del = 1, ++n;
	}
	if (n) { asg_cleanup(g); asg_symm(g); }
	return (int)n;
}

/* ------------------------------------------------------------------ short unitig cutters: asg.c:199-306 */
enum { E_MERGE = 0, E_TIP = 1, E_MOUT = 2, E_MNEI = 3 };

static int utg_end(const asg_t *g, uint32_t v, uint64_t *lw)
{
	const asg_arc_t *av = A_A(g, v ^ 1), *aw;
	uint32_t i, n = 0, last = 0, nv = A_N(g, v ^ 1), w, nw;
	for (i = 0; i < nv; ++i) if (!av[i].del) last = i, ++n;
	if (n == 0) return E_TIP;
	if (n > 1) return E_MOUT;
	if (lw) *lw = av[last].ul << 32 | av[last].v;
	w = av[last].v ^ 1; aw = A_A(g, w); nw = A_N(g, w);
	for (i = n = 0; i < nw; ++i) if (!aw[i].del) ++n;
	return n == 1 ? E_MERGE : E_MNEI;
}

static int walk(const asg_t *g, uint32_t v, int max_ext, uint32_t *path, uint32_t *n_path)
{
	int r;
	uint64_t lw = 0;
	*n_path = 0; path[(*n_path)++] = v;
	do {
		r = utg_end(g, v ^ 1, &lw);
		if (r != E_MERGE) break;
		v = (uint32_t)lw; path[(*n_path)++] = v;
	} while (--max_ext > 0);
	return r;
}

static void arc_set_del(asg_t *g, uint32_t v, uint32_t w, int del)
{
	asg_arc_t *av = A_A(g, v);
	uint32_t i, nv = A_N(g, v);
	for (i = 0; i < nv; ++i) if (av[i].v == w) av[i].del = !!del;
}

static void read_del(asg_t *g, uint32_t s)
{
	uint32_t k, i;
	g->seq[s].del = 1;
	for (k = 0; k < 2; ++k) {
		uint32_t v = s << 1 | k, nv = A_N(g, v);
		asg_arc_t *av = A_A(g, v);
		for (i = 0; i < nv; ++i) { av[i].del = 1; arc_set_del(g, av[i].v ^ 1, v ^ 1, 1); }
	}
}

static int cut_generic(asg_t *g, int max_ext, int first_type, int want_end, int negate)
{ /* tips: first TIP, end != MERGE;  internal: first MNEI, end == MNEI */
	uint32_t v, n_vtx = g->n_seq * 2, cnt = 0, np, i, *path = (uint32_t*)malloc(4 * ((size_t)(max_ext > 0 ? max_ext : 1) + 2));
	for (v = 0; v < n_vtx; ++v) {
		int r;
		if (g->seq[v >> 1].del || utg_end(g, v, 0) != first_type) continue;
		r = walk(g, v, max_ext, path, &np);
		if (negate ? r == want_end : r != want_end) continue;
		for (i = 0; i < np; ++i) read_del(g, path[i] >> 1);
		++cnt;
	}
	free(path);
	if (cnt) asg_cleanup(g);
	return (int)cnt;
}

int asg_cut_tip(asg_t *g, int max_ext) { return cut_generic(g, max_ext, E_TIP, E_MERGE, 1); }
int asg_cut_internal(asg_t *g, int max_ext) { return cut_generic(g, max_ext, E_MNEI, E_MNEI, 0); }

int asg_cut_biloop(asg_t *g, int max_ext)
{
	uint32_t v, n_vtx = g->n_seq * 2, cnt = 0, np, i, *path = (uint32_t*)malloc(4 * ((size_t)(max_ext > 0 ? max_ext : 1) + 2));
	for (v = 0; v < n_vtx; ++v) {
		uint32_t w = UINT32_MAX, x, ov = 0, ox = 0, nv, nw;
		const asg_arc_t *av, *aw;
		if (g->seq[v >> 1].del || utg_end(g, v, 0) != E_MNEI) continue;
		if (walk(g, v, max_ext, path, &np) != E_MOUT) continue;
		x = path[np - 1] ^ 1;
		av = A_A(g, v ^ 1); nv = A_N(g, v ^ 1);
		for (i = 0; i < nv; ++i) if (!av[i].del) w = av[i].v ^ 1;
		aw = A_A(g, w); nw = A_N(g, w);
		for (i = 0; i < nw; ++i) { if (aw[i].del) continue; if (aw[i].v == x) ox = aw[i].ol; if (aw[i].v == v) ov = aw[i].ol; }
		if ((ov == 0 && ox == 0) || ov <= ox) continue;
		arc_set_del(g, w, x, 1); arc_set_del(g, x ^ 1, w ^ 1, 1);
		++cnt;
	}
	free(path);
	if (cnt) asg_cleanup(g);
	return (int)cnt;
}

/* ------------------------------------------------------------------ bubble popping: asg.c:312-433 */
typedef struct { uint32_t p, d, c, r, s; } binfo_t;
typedef struct { uint32_t n, m, *a; } u32v;
static void vpush(u32v *v, uint32_t x) { if (v->n == v->m) { v->m = v->m ? v->m * 2 : 16; v->a = (uint32_t*)realloc(v->a, 4 * (size_t)v->m); } v->a[v->n++] = x; }

static uint64_t pop_one(asg_t *g, uint32_t v0, int max_dist, binfo_t *a, u32v *S, u32v *T, u32v *b, u32v *e)
{
	uint32_t i, pending = 0;
	uint64_t ret = 0;
	if (g->seq[v0 >> 1].del || A_N(g, v0) < 2) return 0;
	S->n = T->n = b->n = e->n = 0;
	a[v0].c = a[v0].d = 0;
	vpush(S, v0);
	do {
		uint32_t v = S->a[--S->n], d = a[v].d, c = a[v].c, nv = A_N(g, v);
		const asg_arc_t *av = A_A(g, v);
		for (i = 0; i < nv; ++i) {
			uint32_t w = av[i].v, l = (uint32_t)av[i].ul;
			binfo_t *t = &a[w];
			if (w == v0) goto reset;
			if (av[i].del) continue;
			vpush(e, (uint32_t)(g->idx[v] >> 32) + i);
			if (d + l > (uint32_t)max_dist) break;
			if (!t->s) {
				uint32_t k, nx = A_N(g, w ^ 1);
				const asg_arc_t *ax = A_A(g, w ^ 1);
				vpush(b, w);
				t->p = v; t->s = 1; t->d = d + l; t->r = 0;
				for (k = 0; k < nx; ++k) t->r += !ax[k].del;
				++pending;
			} else {
				if (c + 1 > t->c || (c + 1 == t->c && d + l > t->d)) t->p = v;
				if (c + 1 > t->c) t->c = c + 1;
				if (d + l < t->d) t->d = d + l;
			}
			t->r = (t->r - 1) & 0x7fffffffu;
			if (t->r == 0) { if (A_N(g, w)) vpush(S, w); else vpush(T, w); --pending; }
		}
		if (i < nv || S->n == 0) goto reset;
	} while (S->n > 1 || pending);
	for (i = 0; i < b->n; ++i) g->seq[b->a[i] >> 1].del = 1;       /* backtrack, asg.c:338-357 */
	for (i = 0; i < e->n; ++i) { asg_arc_t *x = &g->arc[e->a[i]]; x->del = 1; arc_set_del(g, x->v ^ 1, (uint32_t)(x->ul >> 32) ^ 1, 1); }
	{
		uint32_t v = S->a[0];
		do { uint32_t u = a[v].p; g->seq[v >> 1].del = 0; arc_set_del(g, u, v, 0); arc_set_del(g, v ^ 1, u ^ 1, 0); v = u; } while (v != v0);
	}
	ret = 1 | (uint64_t)T->n << 32;
reset:
	for (i = 0; i < b->n; ++i) { binfo_t *t = &a[b->a[i]]; t->s = t->c = t->d = 0; }
	return ret;
}

int asg_pop_bubble(asg_t *g, int max_dist)
{
	uint32_t v, n_vtx = g->n_seq * 2;
	uint64_t n_pop = 0;
	binfo_t *a;
	u32v S = {0,0,0}, T = {0,0,0}, b = {0,0,0}, e = {0,0,0};
	if (!g->is_symm) asg_symm(g);
	a = (binfo_t*)calloc(n_vtx ? n_vtx : 1, sizeof(binfo_t));
	for (v = 0; v < n_vtx; ++v) {
		uint32_t i, live = 0, nv = A_N(g, v);
		const asg_arc_t *av = A_A(g, v);
		if (nv < 2 || g->seq[v >> 1].del) continue;
		for (i = 0; i < nv; ++i) live += !av[i].del;
		if (live > 1) n_pop += pop_one(g, v, max_dist, a, &S, &T, &b, &e);
	}
	free(a); free(S.a); free(T.a); free(b.a); free(e.a);
	if (n_pop) asg_cleanup(g);
	return (int)n_pop;
}

/* ------------------------------------------------------------------ unitigs: asm.c:121-210 */
ma_ug_t *ma_ug_gen(asg_t *g)
{
	uint32_t v, n_vtx = g->n_seq * 2, i;
	int32_t *mark = (int32_t*)calloc(n_vtx ? n_vtx : 1, 4);
	uint64_t *fw = (uint64_t*)malloc(8 * ((size_t)n_vtx + 2)), *bw = (uint64_t*)malloc(8 * ((size_t)n_vtx + 2));
	ma_ug_t *ug = (ma_ug_t*)calloc(1, sizeof(ma_ug_t));
	ug->g = asg_init();
	for (v = 0; v < n_vtx; ++v) {
		uint32_t w, x, l, start = v, end = v ^ 1, len = 0, nf = 0, nb = 0;
		ma_utg_t *p;
		if (g->seq[v >> 1].del || A_N(g, v) == 0 || mark[v]) continue;
		mark[v] = 1;
		for (w = v; A_N(g, w) == 1; ) {                 /* forward while out(w) == 1 and in(x) == 1 */
			x = A_A(g, w)->v;
			if (A_N(g, x ^ 1) != 1) break;
			mark[x] = mark[w ^ 1] = 1;
			l = (uint32_t)A_A(g, w)->ul;
			fw[nf++] = (uint64_t)w << 32 | l;
			end = x ^ 1; len += l; w = x;
			if (x == v) break;
		}
		if (start != (end ^ 1) || nf == 0) {            /* linear: close with the last read, then grow backwards */
			l = g->seq[end >> 1].len;
			fw[nf++] = (uint64_t)(end ^ 1) << 32 | l; len += l;
			for (x = v; A_N(g, x ^ 1) == 1; x = w) {
				w = A_A(g, x ^ 1)->v ^ 1;
				if (A_N(g, w) != 1) break;
				mark[x] = mark[w ^ 1] = 1;
				l = (uint32_t)A_A(g, w)->ul;
				bw[nb++] = (uint64_t)w << 32 | l;
				start = w; len += l;
			}
		} else start = end = UINT32_MAX;                /* circular */
		if (start != UINT32_MAX) mark[start] = mark[end] = 1;
		if (ug->u.n == ug->u.m) { ug->u.m = ug->u.m ? ug->u.m * 2 : 16; ug->u.a = (ma_utg_t*)realloc(ug->u.a, ug->u.m * sizeof(ma_utg_t)); }
		p = &ug->u.a[ug->u.n++];
		p->s = 0; p->start = start; p->end = end; p->len = len; p->circ = start == UINT32_MAX; p->n = p->m = nf + nb;
		p->a = (uint64_t*)malloc(8 * (size_t)(p->n ? p->n : 1));
		for (i = 0; i < nb; ++i) p->a[i] = bw[nb - 1 - i];
		for (i = 0; i < nf; ++i) p->a[nb + i] = fw[i];
	}
	free(fw); free(bw);
	for (v = 0; v < n_vtx; ++v) mark[v] = -1;           /* unitig ends -> oriented unitig ids */
	for (i = 0; i < ug->u.n; ++i) if (!ug->u.a[i].circ) { mark[ug->u.a[i].start] = (int32_t)(i << 1); mark[ug->u.a[i].end] = (int32_t)(i << 1 | 1); }
	for (i = 0; i < g->n_arc; ++i) {
		const asg_arc_t *p = &g->arc[i];
		int32_t mu, mv;
		if (p->del) continue;
		mu = mark[(uint32_t)(p->ul >> 32) ^ 1]; mv = mark[p->v];
		if (mu >= 0 && mv >= 0) {
			uint32_t u = (uint32_t)mu ^ 1;
			int l = (int)(ug->u.a[u >> 1].len - p->ol);
			asg_arc_t *q = arc_push(ug->g);
			if (l < 0) l = 1;
			q->ol = p->ol; q->del = 0; q->ul = (uint64_t)u << 32 | (uint32_t)l; q->v = (uint32_t)mv;
		}
	}
	for (i = 0; i < ug->u.n; ++i) asg_seq_set(ug->g, (int)i, (int)ug->u.a[i].len, 0);
	asg_cleanup(ug->g);
	free(mark);
	return ug;
}

void ma_ug_destroy(ma_ug_t *ug)
{
	size_t i;
	if (!ug) return;
	for (i = 0; i < ug->u.n; ++i) { free(ug->u.a[i].a); free(ug->u.a[i].s); }
	free(ug->u.a); asg_destroy(ug->g); free(ug);
}

/* ------------------------------------------------------------------ unitig sequences: asm.c:212-290, kseq.h:163-211
 * The reads file (FASTA or FASTQ, plain or gzip, "-" = stdin) is walked record by record the way kseq_read does:
 *   header   : '>' or '@', name = bytes up to the first white space, rest of the line ignored;
 *   sequence : following lines joined, until a line STARTS with '>', '@' or '+'; empty lines skipped; after every line one
 *              trailing CR is dropped from what has been collected so far (if more than one byte has);
 *   '+'      : rest of that line skipped, then quality lines (same CR rule) until they are at least as long as the
 *              sequence; a different length ends the whole scan (kseq_read returns -2, asm.c:261 stops);
 *   after a FASTQ record the next header is hunted for byte by byte (any '>' or '@'), after a FASTA record it is the
 *   byte that ended the sequence. */
#include <zlib.h>
#include <ctype.h>

typedef struct { gzFile f; unsigned char buf[1 << 16]; int n, at; } rd_t;
typedef struct { size_t l, m; char *s; } ostr_t;

static int rd_byte(rd_t *r)
{
	if (r->at >= r->n) {
		r->n = gzread(r->f, r->buf, sizeof(r->buf)), r->at = 0;
		if (r->n <= 0) { r->n = 0; return -1; }
	}
	return r->buf[r->at++];
}
static int rd_more(rd_t *r) { int c = rd_byte(r); if (c >= 0) --r->at; return c >= 0; }
static void ostr_push(ostr_t *s, int c) { if (s->l + 2 > s->m) { s->m = s->m ? s->m * 2 : 256; s->s = (char*)realloc(s->s, s->m); } s->s[s->l++] = (char)c; s->s[s->l] = 0; }
/* rest of the current line appended to s, CR rule applied; -1 if the input was already exhausted */
static int rd_rest_of_line(rd_t *r, ostr_t *s)
{
	int c;
	if (!rd_more(r)) return -1;
	while ((c = rd_byte(r)) >= 0 && c != '\n') ostr_push(s, c);
	if (s->l > 1 && s->s[s->l - 1] == '\r') s->s[--s->l] = 0;
	return 0;
}

/* next record: >= 0 length of the sequence, -1 end of input, -2 broken quality.  *head = the header byte already consumed (0: hunt) */
static int next_record(rd_t *r, int *head, ostr_t *name, ostr_t *seq, ostr_t *qual)
{
	int c;
	if (*head == 0) {
		while ((c = rd_byte(r)) >= 0 && c != '>' && c != '@');
		if (c < 0) return -1;
		*head = c;
	}
	name->l = seq->l = qual->l = 0;
	if (!rd_more(r)) return -1;
	while ((c = rd_byte(r)) >= 0 && !isspace(c)) ostr_push(name, c);
	if (name->l == 0) ostr_push(name, 0), name->l = 0;           /* keep name->s a valid empty string */
	if (c >= 0 && c != '\n') while ((c = rd_byte(r)) >= 0 && c != '\n');
	while ((c = rd_byte(r)) >= 0 && c != '>' && c != '+' && c != '@') {
		if (c == '\n') continue;
		ostr_push(seq, c);
		rd_rest_of_line(r, seq);                                 /* (at the end of the input nothing is appended and no CR is dropped) */
	}
	if (c == '>' || c == '@') *head = c;
	if (c != '+') return (int)seq->l;
	while ((c = rd_byte(r)) >= 0 && c != '\n');
	if (c < 0) return -2;
	while (rd_rest_of_line(r, qual) >= 0 && qual->l < seq->l);
	*head = 0;
	return seq->l == qual->l ? (int)seq->l : -2;
}

static unsigned char comp_of[128];
static void comp_init(void)                                     /* asm.c:224-233 as a rule: IUPAC pairs swap, U -> A, the rest stays */
{
	static const char pair[] = "ATCGMKRYVBHD";
	int i;
	for (i = 0; i < 128; ++i) comp_of[i] = (unsigned char)i;
	for (i = 0; pair[i]; i += 2) {
		comp_of[(int)pair[i]] = pair[i + 1], comp_of[(int)pair[i + 1]] = pair[i];
		comp_of[pair[i] | 32] = pair[i + 1] | 32, comp_of[pair[i + 1] | 32] = pair[i] | 32;
	}
	comp_of['U'] = 'A', comp_of['u'] = 'a';
	comp_of[96] = 64;                                            /* the table's row of lower-case letters starts with '@' (asm.c:231) */
}

int ma_ug_seq(ma_ug_t *ug, const sdict_t *d, const ma_sub_t *sub, const char *fn)
{
	typedef struct { uint32_t utg:31, rev:1, at, len; } place_t;  /* where a read goes: asm.c:246-257 */
	rd_t *r;
	place_t *pl;
	ostr_t name = {0,0,0}, seq = {0,0,0}, qual = {0,0,0};
	int head = 0, l;
	size_t i, j;
	gzFile f = fn && strcmp(fn, "-") ? gzopen(fn, "r") : gzdopen(fileno(stdin), "r");
	if (f == 0) return -1;
	comp_init();
	r = (rd_t*)calloc(1, sizeof(rd_t));
	r->f = f;
	pl = (place_t*)calloc(d->n_seq ? d->n_seq : 1, sizeof(place_t));
	for (i = 0; i < ug->u.n; ++i) {
		ma_utg_t *u = &ug->u.a[i];
		uint32_t at = 0;
		u->s = (char*)calloc(1, (size_t)u->len + 1);
		memset(u->s, 'N', u->len);                               /* reads missing from the file stay N (asm.c:249) */
		for (j = 0; j < u->n; ++j) {
			place_t *p = &pl[u->a[j] >> 33];
			assert(p->len == 0);                                 /* a read sits in one place only (asm.c:252) */
			p->utg = (uint32_t)i, p->rev = u->a[j] >> 32 & 1, p->at = at, p->len = (uint32_t)u->a[j];
			at += p->len;
		}
	}
	while ((l = next_record(r, &head, &name, &seq, &qual)) >= 0) {
		int32_t id = sd_get(d, name.s);
		const place_t *p;
		const char *b = seq.s;
		size_t bl = seq.l;
		char *dst;
		uint32_t k;
		if (id < 0 || pl[id].len == 0) continue;
		p = &pl[id];
		if (sub) {                                               /* only the kept interval of the read counts (asm.c:262-266) */
			assert(sub[id].e - sub[id].s <= bl);
			b += sub[id].s, bl = sub[id].e - sub[id].s;
		}
		dst = ug->u.a[p->utg].s + p->at;
		if (!p->rev) memcpy(dst, b, p->len);
		else for (k = 0; k < p->len; ++k) { unsigned char c = (unsigned char)b[bl - 1 - k]; dst[k] = c >= 128 ? 'N' : (char)comp_of[c]; }
	}
	free(name.s); free(seq.s); free(qual.s); free(pl);
	gzclose(f); free(r);
	return 0;
}

/* ------------------------------------------------------------------ writers: asm.c:41-55,77-116 */
void ma_sg_print(const asg_t *g, const sdict_t *d, const ma_sub_t *sub, FILE *fp)
{
	uint32_t i;
	for (i = 0; i < g->n_arc; ++i) {
		const asg_arc_t *a = &g->arc[i];
		uint32_t u = (uint32_t)(a->ul >> 32), v = a->v;
		if (sub) fprintf(fp, "L\t%s:%d-%d\t%c\t%s:%d-%d\t%c\t%d:\tL1:i:%d\n", d->seq[u >> 1].name, sub[u >> 1].s + 1, sub[u >> 1].e, "+-"[u & 1],
						 d->seq[v >> 1].name, sub[v >> 1].s + 1, sub[v >> 1].e, "+-"[v & 1], a->ol, (uint32_t)a->ul);
		else fprintf(fp, "L\t%s\t%c\t%s\t%c\t%d:\tL1:i:%d\n", d->seq[u >> 1].name, "+-"[u & 1], d->seq[v >> 1].name, "+-"[v & 1], a->ol, (uint32_t)a->ul);
	}
}

void ma_ug_print(const ma_ug_t *ug, const sdict_t *d, const ma_sub_t *sub, FILE *fp)
{
	uint32_t i, j;
	for (i = 0; i < ug->u.n; ++i) {
		const ma_utg_t *p = &ug->u.a[i];
		uint32_t off = 0;
		char nm[32];
		sprintf(nm, "utg%.6d%c", i + 1, "lc"[p->circ]);
		fprintf(fp, "S\t%s\t%s\tLN:i:%d\n", nm, p->s ? p->s : "*", p->len);
		if (p->circ) fprintf(fp, "L\t%s\t+\t%s\t+\t0M\nL\t%s\t-\t%s\t-\t0M\n", nm, nm, nm, nm);
		for (j = 0; j < p->n; off += (uint32_t)p->a[j++]) {
			uint32_t r = (uint32_t)(p->a[j] >> 33);
			if (sub) fprintf(fp, "a\t%s\t%d\t%s:%d-%d\t%c\t%d\n", nm, off, d->seq[r].name, sub[r].s + 1, sub[r].e, "+-"[p->a[j] >> 32 & 1], (uint32_t)p->a[j]);
			else fprintf(fp, "a\t%s\t%d\t%s\t%c\t%d\n", nm, off, d->seq[r].name, "+-"[p->a[j] >> 32 & 1], (uint32_t)p->a[j]);
		}
	}
	for (i = 0; i < ug->g->n_arc; ++i) {
		uint32_t u = (uint32_t)(ug->g->arc[i].ul >> 32), v = ug->g->arc[i].v;
		fprintf(fp, "L\tutg%.6d%c\t%c\tutg%.6d%c\t%c\t%dM\tSD:i:%d\n", (u >> 1) + 1, "lc"[ug->u.a[u >> 1].circ], "+-"[u & 1],
				(v >> 1) + 1, "lc"[ug->u.a[v >> 1].circ], "+-"[v & 1], ug->g->arc[i].ol, (uint32_t)ug->g->arc[i].ul);
	}
	for (i = 0; i < ug->u.n; ++i) {
		const ma_utg_t *p = &ug->u.a[i];
		if (p->start == UINT32_MAX) { fprintf(fp, "x\tutg%.6dc\t%d\t%d\n", i + 1, p->len, p->n); continue; }
		if (sub) fprintf(fp, "x\tutg%.6dl\t%d\t%d\t%d\t%d\t%s:%d-%d\t%c\t%s:%d-%d\t%c\n", i + 1, p->len, p->n, A_N(ug->g, i << 1 | 1), A_N(ug->g, i << 1),
						 d->seq[p->start >> 1].name, sub[p->start >> 1].s + 1, sub[p->start >> 1].e, "+-"[p->start & 1],
						 d->seq[p->end >> 1].name, sub[p->end >> 1].s + 1, sub[p->end >> 1].e, "+-"[p->end & 1]);
		else fprintf(fp, "x\tutg%.6dl\t%d\t%d\t%d\t%d\t%s\t%c\t%s\t%c\n", i + 1, p->len, p->n, A_N(ug->g, i << 1 | 1), A_N(ug->g, i << 1),
					 d->seq[p->start >> 1].name, "+-"[p->start & 1], d->seq[p->end >> 1].name, "+-"[p->end & 1]);
	}
}
