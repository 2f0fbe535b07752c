// hit_host.cpp -- TEST INFRASTRUCTURE (never linked into the product): the functions that carry the reference's integer
// conversion rules -- mab_cut_hit (ma_hit_cut's clipping, hit.c:162-193), mab_flt_hit (ma_hit_flt's keep rule, hit.c:195-216)
// and mab_hit2arc (miniasm.h:86-104), all in miniasm_b200/csrc/hit2arc.cuh, the very header the CUDA kernels are built from --
// compiled for the host and put behind the loops of ma_hit_cut / ma_hit_flt / ma_sg_gen, so that the CPU tier can fuzz them
// against the unmodified reference with inputs no synthetic PAF produces (hits reaching outside the kept intervals, wrapped spans,
// empty intervals, self hits):
// tests/test_hitrules_cpu.py.  Also here: mab_comp_of (basecomp.cuh), the reverse-strand complement of `-f reads`, all 256 byte values.
#include "../../miniasm_b200/csrc/hit2arc.cuh"
#include "../../miniasm_b200/csrc/basecomp.cuh"

extern "C" {

// ma_hit_cut (hit.c:162-193): clip every hit to the kept intervals of both reads, stable in-place compaction
size_t hs_hit_cut(const DSub *reg, int min_span, size_t n, DHit *a)
{
	size_t m = 0;
	for (size_t i = 0; i < n; ++i) {
		DHit p = a[i];
		if (mab_cut_hit(p, reg[p.qns >> 32], reg[p.tn], min_span)) a[m++] = p;
	}
	return m;
}

// ma_hit_flt (hit.c:195-216): stable in-place compaction by mab_flt_hit; *tot_dp is the numerator of the coverage estimate
size_t hs_hit_flt(const DSub *sub, int max_hang, int min_ovlp, size_t n, DHit *a, unsigned long long *tot_dp)
{
	size_t m = 0;
	unsigned long long dp = 0;
	for (size_t i = 0; i < n; ++i) {
		const DHit h = a[i];
		uint32_t l;
		if (mab_flt_hit(h, sub[h.qns >> 32], sub[h.tn], max_hang, min_ovlp, &l)) a[m++] = h, dp += l;
	}
	*tot_dp = dp;
	return m;
}

// the arc-emission loop of ma_sg_gen (asm.c:14-36) before asg_cleanup: arcs in hit order, seq[i] = len | del<<31.
// `seq` comes in holding the lengths and deletion flags of asm.c:14-17; len32 the 32-bit lengths the classifier takes (asm.c:23-24).
size_t hs_sg_arcs(int max_hang, float int_frac, int min_ovlp, size_t n, const DHit *a, const uint32_t *len32, uint32_t *seq, DArc *out)
{
	size_t m = 0;
	for (size_t i = 0; i < n; ++i) {
		const DHit h = a[i];
		const uint32_t qn = (uint32_t)(h.qns >> 32);
		DArc t;
		const int r = mab_hit2arc(h, (int)len32[qn], (int)len32[h.tn], max_hang, int_frac, min_ovlp, &t);
		if (r >= 0) {
			if (qn == h.tn) {
				if ((uint32_t)h.qns == h.ts && h.qe == h.te && (h.ml_rev >> 31)) seq[qn] |= MAB_DEL_BIT;
				continue;
			}
			out[m++] = t;
		} else if (r == MAB_HT_QCONT) seq[qn] |= MAB_DEL_BIT;
	}
	return m;
}

// the complement of a sequence byte as the gather kernel of `-f reads` applies it (asm.c:224-233,281)
unsigned char hs_comp(unsigned char c) { return mab_comp_of(c); }

// the classification alone, for a histogram of what the fuzz reached
int hs_hit2arc(const DHit *h, int ql, int tl, int max_hang, float int_frac, int min_ovlp, DArc *t) { return mab_hit2arc(*h, ql, tl, max_hang, int_frac, min_ovlp, t); }

}
