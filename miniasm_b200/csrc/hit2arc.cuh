// hit2arc.cuh -- the hit classifier shared by ma_hit_flt, ma_hit_contained and ma_sg_gen.
//
// Restates ma_hit2arc (miniasm.h:86-104) with the C integer-conversion rules of the original written out:
// the reference mixes int32, uint32 and 31-bit fields, so which comparisons are signed and which are
// unsigned is part of the behaviour (SURVEY.md section 7, hard part 2).  One float32 product decides the
// "internal match" test; it is computed with an explicit round-to-nearest multiply (no FMA contraction).
#pragma once
#include "mab_common.cuh"

#define MAB_HT_INT        (-1)
#define MAB_HT_QCONT      (-2)
#define MAB_HT_TCONT      (-3)
#define MAB_HT_SHORT_OVLP (-4)

// ql, tl: lengths of the (trimmed) query / target reads.  On a non-negative return *arc holds the arc.
__host__ __device__ __forceinline__ int mab_hit2arc(const DHit &h, int ql, int tl, int max_hang, float int_frac, int min_ovlp, DArc *arc)
{
	const int32_t qs = (int32_t)(uint32_t)h.qns;
	const uint32_t qe = h.qe, rev = h.ml_rev >> 31;
	int32_t tl5, tl3; // target overhang beyond the query's 5' / 3' end, on the query strand
	if (rev) tl5 = (int32_t)((uint32_t)tl - h.te), tl3 = (int32_t)h.ts;
	else tl5 = (int32_t)h.ts, tl3 = (int32_t)((uint32_t)tl - h.te);
	const uint32_t q3 = (uint32_t)ql - qe;                       // query bases right of the hit (unsigned in the reference)
	const int32_t ext5 = qs < tl5 ? qs : tl5;                    // signed compare
	const int32_t ext3 = (int32_t)(q3 < (uint32_t)tl3 ? q3 : (uint32_t)tl3); // unsigned compare
	const uint32_t span = qe - (uint32_t)qs;
	const uint32_t full = span + (uint32_t)ext5 + (uint32_t)ext3;
#ifdef __CUDA_ARCH__
	const float bound = __fmul_rn((float)full, int_frac);
#else
	const float bound = (float)full * int_frac;
#endif
	if (ext5 > max_hang || ext3 > max_hang || (float)span < bound) return MAB_HT_INT;
	if (qs <= tl5 && q3 <= (uint32_t)tl3) return MAB_HT_QCONT;    // query contained (tested first: ties delete both reads)
	if (qs >= tl5 && q3 >= (uint32_t)tl3) return MAB_HT_TCONT;    // target contained
	uint32_t u, v, l;
	if (qs > tl5) u = 0, v = rev, l = (uint32_t)qs - (uint32_t)tl5;
	else u = 1, v = !rev, l = q3 - (uint32_t)tl3;
	if (full < (uint32_t)min_ovlp || h.te - h.ts + (uint32_t)ext5 + (uint32_t)ext3 < (uint32_t)min_ovlp) return MAB_HT_SHORT_OVLP;
	u |= (uint32_t)(h.qns >> 32) << 1, v |= h.tn << 1;
	arc->ul = (uint64_t)u << 32 | l;
	arc->v = v;
	arc->ol_del = ((uint32_t)ql - l) & 0x7fffffffu;
	return (int)l;
}

// ---------------------------------------------------------------------------------------------
// ma_hit_cut (hit.c:162-193).  The reference computes in `int` locals from uint32 operands and compares
// against a 31-bit field (signed after promotion) or a uint32 field (unsigned); restated with explicit types.
// ---------------------------------------------------------------------------------------------
// clips hit p to the kept intervals rq (query read) / rt (target read); true if both spans stay >= min_span
__host__ __device__ __forceinline__ bool mab_cut_hit(DHit &p, const DSub rq, const DSub rt, int min_span)
{
	{
		if ((rq.s_del | rt.s_del) & MAB_DEL_BIT) return false;
		const uint32_t rqs = rq.s_del, rts = rt.s_del, rqe = rq.e, rte = rt.e; // del bits are clear here
		const uint32_t pqs = (uint32_t)p.qns;
		uint32_t uqs, uqe, uts, ute;
		if (p.ml_rev >> 31) {
			uqs = p.te < rte ? pqs : pqs + (p.te - rte);
			uqe = p.ts > rts ? p.qe : p.qe - (rts - p.ts);
			uts = p.qe < rqe ? p.ts : p.ts + (p.qe - rqe);
			ute = pqs > rqs ? p.te : p.te - (rqs - pqs);
		} else {
			uqs = p.ts > rts ? pqs : pqs + (rts - p.ts);
			uqe = p.te < rte ? p.qe : p.qe - (p.te - rte);
			uts = pqs > rqs ? p.ts : p.ts + (rqs - pqs);
			ute = p.qe < rqe ? p.te : p.te - (p.qe - rqe);
		}
		int qs = (int)uqs, qe = (int)uqe, ts = (int)uts, te = (int)ute;
		qs = (qs > (int)rqs ? qs : (int)rqs) - (int)rqs;                      // signed compare (31-bit field promotes to int)
		qe = (int)(((uint32_t)qe < rqe ? (uint32_t)qe : rqe) - rqs);          // unsigned compare (uint32 field)
		ts = (ts > (int)rts ? ts : (int)rts) - (int)rts;
		te = (int)(((uint32_t)te < rte ? (uint32_t)te : rte) - rts);
		bool keep = qe - qs >= min_span && te - ts >= min_span;
		if (keep) {
			p.qns = (p.qns >> 32 << 32) | (uint64_t)(int64_t)qs;
			p.qe = (uint32_t)qe, p.ts = (uint32_t)ts, p.te = (uint32_t)te;
		}
		return keep;
	}
}

// ma_hit_flt (hit.c:195-216): true if hit h of query interval sq / target interval st classifies as an arc or a containment under
// the (already relaxed) thresholds; *dp is then what it adds to the numerator of the coverage estimate the reference logs
__host__ __device__ __forceinline__ bool mab_flt_hit(const DHit &h, const DSub sq, const DSub st, int max_hang, int min_ovlp, uint32_t *dp)
{
	if ((sq.s_del | st.s_del) & MAB_DEL_BIT) return false;
	const uint32_t ql = sq.e - sq.s_del, tl = st.e - st.s_del;
	DArc t;
	const int r = mab_hit2arc(h, (int)ql, (int)tl, max_hang, .5f, min_ovlp, &t);
	*dp = r >= 0 ? (uint32_t)r : r == MAB_HT_QCONT ? ql : tl;
	return r >= 0 || r == MAB_HT_QCONT || r == MAB_HT_TCONT;
}
