// capi_hit.cu -- drop-in level C ABI for stage (i) and graph construction (miniasm.h:61-70 of the reference).
// Host arrays in, CUDA passes (hit_dev.cu), host arrays out; same ownership rules as the reference.
#include "../../include/miniasm_b200.h"
#include "capi_util.cuh"
#include "hit_dev.cuh"

static_assert(sizeof(ma_hit_t) == sizeof(DHit), "hit ABI");
static_assert(sizeof(ma_sub_t) == sizeof(DSub), "sub ABI");

static void hits_upload(MabDev &d, const ma_hit_t *a, size_t n, uint32_t n_seq, DHits &h)
{
	dh_reserve(d, h, n ? n : 1);
	h.n = n, h.n_seq = n_seq;
	if (n) MAB_CUDA(cudaMemcpyAsync(h.a, a, n * sizeof(DHit), cudaMemcpyHostToDevice, d.stream));
}

static void hits_download(MabDev &d, const DHits &h, ma_hit_t *a)
{
	if (h.n) MAB_CUDA(cudaMemcpyAsync(a, h.a, h.n * sizeof(DHit), cudaMemcpyDeviceToHost, d.stream));
	d.sync();
}

// the reference passes interval tables without a length: size them by the largest read id the hits name
static uint32_t max_id_plus1(size_t n, const ma_hit_t *a)
{
	uint32_t m = 0;
	for (size_t i = 0; i < n; ++i) {
		uint32_t q = (uint32_t)(a[i].qns >> 32), t = a[i].tn;
		if (q >= m) m = q + 1;
		if (t >= m) m = t + 1;
	}
	return m;
}

template <typename T> static T *to_dev(MabDev &d, const T *host, size_t n)
{
	T *p = mab_alloc<T>(d, n);
	if (n) MAB_CUDA(cudaMemcpyAsync(p, host, n * sizeof(T), cudaMemcpyHostToDevice, d.stream));
	return p;
}

extern "C" {

/* hit.c:70-107.  Parsing and the name dictionary stay on the host at this level (the fused level parses on
 * the GPU); the mirrored hits are sorted on the device. */
ma_hit_t *ma_hit_read(const char *fn, int min_span, int min_match, sdict_t *d, size_t *n, int bi_dir, const sdict_t *excl)
{
	paf_file_t *fp = paf_open(fn);
	paf_rec_t r;
	ma_hit_t *a = 0;
	size_t n_a = 0, m_a = 0, tot = 0, tot_len = 0;
	if (fp == 0) {
		fprintf(stderr, "[E::%s] could not open PAF file %s\n", __func__, fn);
		exit(1);
	}
	memset(&r, 0, sizeof(r));
	while (paf_read(fp, &r) >= 0) {
		++tot;
		if (r.qe - r.qs < (uint32_t)min_span || r.te - r.ts < (uint32_t)min_span || (int)r.ml < min_match) continue;
		if (excl && (sd_get(excl, r.qn) >= 0 || sd_get(excl, r.tn) >= 0)) continue;
		if (n_a + 2 > m_a) { m_a = m_a ? m_a << 1 : 1024; a = (ma_hit_t*)realloc(a, m_a * sizeof(ma_hit_t)); }
		ma_hit_t *p = &a[n_a++];
		uint32_t qid = (uint32_t)sd_put(d, r.qn, r.ql), tid = (uint32_t)sd_put(d, r.tn, r.tl);
		p->qns = (uint64_t)qid << 32 | r.qs, p->qe = r.qe, p->tn = tid;
		p->ts = r.ts, p->te = r.te, p->rev = r.rev, p->ml = r.ml, p->bl = r.bl, p->del = 0;
		if (bi_dir && qid != tid) { // the same overlap seen from the target (hit.c:92-98)
			ma_hit_t *m = &a[n_a++];
			m->qns = (uint64_t)tid << 32 | r.ts, m->qe = r.te, m->tn = qid;
			m->ts = r.qs, m->te = r.qe, m->rev = r.rev, m->ml = r.ml, m->bl = r.bl, m->del = 0;
		}
	}
	paf_close(fp);
	for (uint32_t i = 0; i < d->n_seq; ++i) tot_len += d->seq[i].len;
	if (ma_verbose >= 3)
		fprintf(stderr, "[M::%s::%s] read %ld hits; stored %ld hits and %d sequences (%ld bp)\n", __func__, sys_timestamp(),
				(long)tot, (long)n_a, d->n_seq, (long)tot_len);
	if (n_a > 1) {
		MabDev &dev = mab_default_dev();
		DHits h;
		hits_upload(dev, a, n_a, d->n_seq, h);
		dh_sort(dev, h);
		hits_download(dev, h, a);
		dh_free(dev, h);
		dev.sync();
	}
	*n = n_a;
	return a;
}

/* hit.c:109-160 */
ma_sub_t *ma_hit_sub(int min_dp, float min_iden, int end_clip, size_t n, const ma_hit_t *a, size_t n_sub)
{
	ma_sub_t *sub = (ma_sub_t*)calloc(n_sub ? n_sub : 1, sizeof(ma_sub_t));
	MabDev &dev = mab_default_dev();
	DHits h;
	hits_upload(dev, a, n, (uint32_t)n_sub, h);
	DSub *dsub = mab_alloc<DSub>(dev, n_sub);
	dh_sub(dev, h, min_dp, min_iden, end_clip, dsub);
	if (n_sub) MAB_CUDA(cudaMemcpyAsync(sub, dsub, n_sub * sizeof(DSub), cudaMemcpyDeviceToHost, dev.stream));
	dev.sync();
	dev.free(dsub);
	dh_free(dev, h);
	dev.sync();
	return sub;
}

/* hit.c:162-193 */
size_t ma_hit_cut(const ma_sub_t *reg, int min_span, size_t n, ma_hit_t *a)
{
	MabDev &dev = mab_default_dev();
	DHits h;
	uint32_t n_sub = max_id_plus1(n, a);
	hits_upload(dev, a, n, n_sub, h);
	DSub *dreg = to_dev(dev, (const DSub*)reg, n_sub);
	size_t m = dh_cut(dev, h, dreg, min_span);
	hits_download(dev, h, a);
	dev.free(dreg);
	dh_free(dev, h);
	dev.sync();
	return m;
}

/* hit.c:195-216 */
size_t ma_hit_flt(const ma_sub_t *sub, int max_hang, int min_ovlp, size_t n, ma_hit_t *a, float *cov)
{
	MabDev &dev = mab_default_dev();
	DHits h;
	uint32_t n_sub = max_id_plus1(n, a);
	hits_upload(dev, a, n, n_sub, h);
	DSub *dsub = to_dev(dev, (const DSub*)sub, n_sub);
	size_t m = dh_flt(dev, h, dsub, max_hang, min_ovlp, cov);
	hits_download(dev, h, a);
	dev.free(dsub);
	dh_free(dev, h);
	dev.sync();
	return m;
}

/* hit.c:218-223 */
void ma_sub_merge(size_t n_sub, ma_sub_t *a, const ma_sub_t *b)
{
	MabDev &dev = mab_default_dev();
	DSub *da = to_dev(dev, (const DSub*)a, n_sub), *db = to_dev(dev, (const DSub*)b, n_sub);
	dh_sub_merge(dev, (uint32_t)n_sub, da, db);
	if (n_sub) MAB_CUDA(cudaMemcpyAsync(a, da, n_sub * sizeof(DSub), cudaMemcpyDeviceToHost, dev.stream));
	dev.sync();
	dev.free(da); dev.free(db);
	dev.sync();
}

/* hit.c:225-256: containment flags on the device, the name side of sd_squeeze on the host */
size_t ma_hit_contained(const ma_opt_t *opt, sdict_t *d, ma_sub_t *sub, size_t n, ma_hit_t *a)
{
	MabDev &dev = mab_default_dev();
	DHits h;
	const uint32_t old_n_seq = d->n_seq;
	hits_upload(dev, a, n, old_n_seq, h);
	DSub *dsub = to_dev(dev, (const DSub*)sub, old_n_seq);
	uint8_t *h_del = (uint8_t*)malloc(old_n_seq ? old_n_seq : 1);
	for (uint32_t i = 0; i < old_n_seq; ++i) h_del[i] = d->seq[i].del;
	uint8_t *d_del = to_dev(dev, h_del, old_n_seq);
	int32_t *d_map = mab_alloc<int32_t>(dev, old_n_seq);
	HitArcParams p = { opt->max_hang, opt->int_frac, opt->min_ovlp };
	int vsave = ma_verbose;
	ma_verbose = 0; // the summary line is printed below, once the dictionary is squeezed
	size_t m = dh_contained(dev, h, dsub, d_del, p, d_map);
	ma_verbose = vsave;
	int32_t *map = (int32_t*)malloc((old_n_seq ? old_n_seq : 1) * 4);
	if (old_n_seq) {
		MAB_CUDA(cudaMemcpyAsync(map, d_map, (size_t)old_n_seq * 4, cudaMemcpyDeviceToHost, dev.stream));
		MAB_CUDA(cudaMemcpyAsync(sub, dsub, (size_t)old_n_seq * sizeof(DSub), cudaMemcpyDeviceToHost, dev.stream));
	}
	hits_download(dev, h, a);
	for (uint32_t i = 0; i < old_n_seq; ++i)
		if (map[i] < 0) d->seq[i].del = 1;
	int32_t *map2 = sd_squeeze(d);
	for (uint32_t i = 0; i < old_n_seq; ++i)
		if (map[i] != map2[i]) { fprintf(stderr, "[E::%s] device/host id map mismatch at read %u\n", __func__, i); exit(74); }
	free(map2); free(map); free(h_del);
	dev.free(dsub); dev.free(d_del); dev.free(d_map);
	dh_free(dev, h);
	dev.sync();
	if (ma_verbose >= 3)
		fprintf(stderr, "[M::%s::%s] %d sequences and %ld hits remain after containment removal\n", __func__, sys_timestamp(), d->n_seq, (long)m);
	return m;
}

/* asm.c:9-39 */
asg_t *ma_sg_gen(const ma_opt_t *opt, const sdict_t *d, const ma_sub_t *sub, size_t n_hits, const ma_hit_t *hit)
{
	MabDev &dev = mab_default_dev();
	const uint32_t n_seq = d->n_seq;
	uint32_t *len = (uint32_t*)malloc((n_seq ? n_seq : 1) * 4);
	uint8_t *del = (uint8_t*)malloc(n_seq ? n_seq : 1);
	for (uint32_t i = 0; i < n_seq; ++i) {
		if (sub) len[i] = sub[i].e - sub[i].s, del[i] = sub[i].del || d->seq[i].del;
		else len[i] = d->seq[i].len, del[i] = d->seq[i].del;
	}
	DHits h;
	DGraph dg;
	hits_upload(dev, hit, n_hits, n_seq, h);
	uint32_t *d_len = to_dev(dev, len, n_seq);
	uint8_t *d_del = to_dev(dev, del, n_seq);
	HitArcParams p = { opt->max_hang, opt->int_frac, opt->min_ovlp };
	dh_sg_gen(dev, h, d_len, d_del, p, dg);
	asg_t *g = asg_init();
	g->n_seq = n_seq, g->m_seq = n_seq ? n_seq : 1;
	g->seq = (asg_seq_t*)malloc((size_t)g->m_seq * sizeof(asg_seq_t));
	g->m_arc = dg.n_arc ? dg.n_arc : 1;
	g->arc = (asg_arc_t*)malloc((size_t)g->m_arc * sizeof(asg_arc_t));
	mab_graph_download(dev, dg, g);
	dev.free(d_len); dev.free(d_del);
	dh_free(dev, h);
	dg_free(dev, dg);
	dev.sync();
	free(len); free(del);
	return g;
}

}
