// gfa_dev.cu -- the GFA text of ma_ug_print (asm.c:77-116) produced on the GPU from the device-resident layout.
//
// Why: after mab_unitigs everything the writer needs is in HBM (unitig layout, unitig graph, read names, kept
// intervals).  The host writer first has to copy those tables down and rebuild host structs (one malloc per unitig,
// a name index per read) before it formats ~1 line per read; on 1 M reads that tail is ~20 ms of a 120 ms
// end-to-end step.  Here every output line ("record") is formatted by one thread straight into one text buffer, which
// then crosses PCIe once (~45 MB) and goes to the FILE with a single fwrite.
//
// Two passes over the same emitter (so the lengths cannot disagree with the bytes): pass 0 counts the bytes of each
// record, an exclusive scan places them, pass 1 writes.  Record order = the reference's line order:
//   for each unitig i: S line (+ the two circularising L lines), then its `a` lines   -> records [0, n_utg + n_items)
//   L lines of the unitig graph                                                        -> next n_arc records
//   x lines                                                                            -> last n_utg records
// Integer formats are the reference's: "%d" of the 32-bit value, "utg%.6d" zero-padded.  Without unitig sequences the S line
// carries "*"; with them (-f reads) it reserves `len` bytes, pre-filled with 'N', that ugseq_dev.cu fills in place.
// This is the default writer of the CLI and of bench.py (MAB_GPU_GFA=0 / --host-gfa: host structs + ma_ug_print).
#include "gfa_dev.cuh"
#include "fmt_sink.cuh"
#include <cub/cub.cuh>

struct GfaView {
	const DUtgMeta *meta; const uint64_t *items; const uint32_t *ioff; // ioff: exclusive (mod 2^32) sum of item lengths
	uint32_t n_utg; uint64_t n_items;
	const DArc *uarc; uint32_t n_uarc; const uint64_t *uidx;
	ReadNames nm;
	uint64_t *seq_pos;             // non-null: S lines reserve `len` bytes for the unitig sequence; seq_pos[i] = where (filled by the write pass)
	const char *out_base;
};

template <class Sink> __host__ __device__ __forceinline__ void put_utg(Sink &s, uint32_t i, bool circ) // "utg%.6d%c" of i + 1
{
	s.c('u'); s.c('t'); s.c('g');
	put_dec(s, i + 1, 6);
	s.c(circ ? 'c' : 'l');
}
template <class Sink> __host__ __device__ void emit_record(const GfaView &v, uint64_t rec, Sink &s)
{
	const uint64_t n_block = (uint64_t)v.n_utg + v.n_items;
	if (rec < n_block) {
		// unitig i = the last one whose block starts at or before rec; block start of unitig i = i + meta[i].first
		uint32_t lo = 0, hi = v.n_utg;
		while (hi - lo > 1) {
			const uint32_t mid = lo + (hi - lo) / 2;
			if ((uint64_t)mid + v.meta[mid].first <= rec) lo = mid; else hi = mid;
		}
		const uint32_t i = lo;
		const DUtgMeta m = v.meta[i];
		const uint64_t j = rec - ((uint64_t)i + m.first);
		if (j == 0) {
			s.c('S'); s.c('\t'); put_utg(s, i, m.circ != 0); s.c('\t');
			if (v.seq_pos) s.hole(m.len, v.seq_pos + i, v.out_base); else s.c('*');       // asm.c:83: u->s or "*"
			put_lit(s, "\tLN:i:", 6); put_int(s, (int32_t)m.len); s.c('\n');
			if (m.circ)
				for (int k = 0; k < 2; ++k) {
					s.c('L'); s.c('\t'); put_utg(s, i, true); s.c('\t'); s.c(k ? '-' : '+'); s.c('\t');
					put_utg(s, i, true); s.c('\t'); s.c(k ? '-' : '+'); s.c('\t'); s.c('0'); s.c('M'); s.c('\n');
				}
		} else {
			const uint64_t k = (uint64_t)m.first + (j - 1);
			const uint64_t it = v.items[k];
			const uint32_t off = v.ioff[k] - v.ioff[m.first];
			s.c('a'); s.c('\t'); put_utg(s, i, m.circ != 0); s.c('\t'); put_int(s, (int32_t)off); s.c('\t');
			put_read(s, v.nm, (uint32_t)(it >> 33));
			s.c('\t'); s.c((it >> 32 & 1) ? '-' : '+'); s.c('\t'); put_int(s, (int32_t)(uint32_t)it); s.c('\n');
		}
	} else if (rec < n_block + v.n_uarc) {
		const DArc a = v.uarc[rec - n_block];
		const uint32_t u = (uint32_t)(a.ul >> 32), w = a.v;
		s.c('L'); s.c('\t'); put_utg(s, u >> 1, v.meta[u >> 1].circ != 0); s.c('\t'); s.c((u & 1) ? '-' : '+'); s.c('\t');
		put_utg(s, w >> 1, v.meta[w >> 1].circ != 0); s.c('\t'); s.c((w & 1) ? '-' : '+'); s.c('\t');
		put_int(s, (int32_t)(a.ol_del & 0x7fffffffu)); s.c('M'); put_lit(s, "\tSD:i:", 6); put_int(s, (int32_t)(uint32_t)a.ul); s.c('\n');
	} else {
		const uint32_t i = (uint32_t)(rec - n_block - v.n_uarc);
		const DUtgMeta m = v.meta[i];
		s.c('x'); s.c('\t');
		if (m.start == 0xffffffffu) {
			put_utg(s, i, true); s.c('\t'); put_int(s, (int32_t)m.len); s.c('\t'); put_int(s, (int32_t)m.n); s.c('\n');
		} else {
			put_utg(s, i, false); s.c('\t'); put_int(s, (int32_t)m.len); s.c('\t'); put_int(s, (int32_t)m.n); s.c('\t');
			put_int(s, (int32_t)(uint32_t)v.uidx[(size_t)i << 1 | 1]); s.c('\t'); put_int(s, (int32_t)(uint32_t)v.uidx[(size_t)i << 1 | 0]); s.c('\t');
			put_read(s, v.nm, m.start >> 1); s.c('\t'); s.c((m.start & 1) ? '-' : '+'); s.c('\t');
			put_read(s, v.nm, m.end >> 1); s.c('\t'); s.c((m.end & 1) ? '-' : '+'); s.c('\n');
		}
	}
}

__global__ void k_gfa_count(GfaView v, uint64_t n_rec, uint32_t *len)
{
	for (uint64_t r = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; r < n_rec; r += (uint64_t)gridDim.x * blockDim.x) {
		CountSink s{0};
		emit_record(v, r, s);
		len[r] = s.n;
	}
}

__global__ void k_gfa_write(GfaView v, uint64_t n_rec, const uint64_t *pos, char *out)
{
	v.out_base = out;
	for (uint64_t r = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; r < n_rec; r += (uint64_t)gridDim.x * blockDim.x) {
		WriteSink s{out + pos[r]};
		emit_record(v, r, s);
	}
}

struct ItemLen { __host__ __device__ __forceinline__ uint32_t operator()(uint64_t x) const { return (uint32_t)x; } };
struct U32ToU64 { __host__ __device__ __forceinline__ uint64_t operator()(uint32_t x) const { return x; } };

// Formats the GFA into a fresh device buffer (*d_text_out, caller frees through d.free); returns its size in bytes.
size_t dg_gfa_text(MabDev &d, const DUnitigs &ug, const uint32_t *orig, const uint64_t *noff, const uint32_t *nlen, const char *name_text,
                   const DSub *sub, char **d_text_out, uint64_t *seq_pos, uint32_t **ioff_out)
{
	*d_text_out = nullptr;
	if (ioff_out) *ioff_out = nullptr;
	const uint64_t n_rec = (uint64_t)ug.n_utg * 2 + ug.n_items + ug.g.n_arc;
	if (n_rec == 0) return 0;
	if (ug.n_items >= (1ull << 32)) { fprintf(stderr, "[E::miniasm_b200] more than 2^32 layout entries\n"); exit(73); }
	uint32_t *ioff = mab_alloc<uint32_t>(d, ug.n_items ? ug.n_items : 1);
	size_t tb = 0;
	void *tmp;
	if (ug.n_items) {
		cub::TransformInputIterator<uint32_t, ItemLen, const uint64_t*> in(ug.items, ItemLen());
		cub::DeviceScan::ExclusiveSum(nullptr, tb, in, ioff, (int64_t)ug.n_items, d.stream);
		tmp = d.tmp(tb);
		cub::DeviceScan::ExclusiveSum(tmp, tb, in, ioff, (int64_t)ug.n_items, d.stream);
		++d.n_lib;
	}
	GfaView v{ug.meta, ug.items, ioff, ug.n_utg, ug.n_items, ug.g.arc, ug.g.n_arc, ug.g.idx, {orig, noff, nlen, name_text, sub}, seq_pos, nullptr};
	uint32_t *len = mab_alloc<uint32_t>(d, n_rec);
	uint64_t *pos = mab_alloc<uint64_t>(d, n_rec + 1);
	MAB_LAUNCH(d, k_gfa_count, mab_grid(n_rec, 256), 256, 0, v, n_rec, len);
	cub::TransformInputIterator<uint64_t, U32ToU64, const uint32_t*> lin(len, U32ToU64());
	cub::DeviceScan::ExclusiveSum(nullptr, tb, lin, pos, (int64_t)n_rec, d.stream);
	tmp = d.tmp(tb);
	cub::DeviceScan::ExclusiveSum(tmp, tb, lin, pos, (int64_t)n_rec, d.stream);
	++d.n_lib;
	uint64_t last_pos = 0;
	uint32_t last_len = 0;
	MAB_CUDA(cudaMemcpyAsync(&last_pos, pos + n_rec - 1, 8, cudaMemcpyDeviceToHost, d.stream));
	MAB_CUDA(cudaMemcpyAsync(&last_len, len + n_rec - 1, 4, cudaMemcpyDeviceToHost, d.stream));
	d.sync();
	const size_t bytes = (size_t)(last_pos + last_len);
	char *out = (char*)d.alloc(bytes ? bytes : 1);
	if (seq_pos && bytes) MAB_CUDA(cudaMemsetAsync(out, 'N', bytes, d.stream)); // asm.c:249: a unitig starts as N's; the gather overwrites what the reads file holds
	MAB_LAUNCH(d, k_gfa_write, mab_grid(n_rec, 256), 256, 0, v, n_rec, pos, out);
	if (ioff_out) *ioff_out = ioff; else d.free(ioff);
	d.free(len); d.free(pos);
	*d_text_out = out;
	return bytes;
}

// ---- host probe (tests only): the same emitter compiled for the CPU, fed from the reference's host structs ------------
// Lets the CPU test tier compare the formatter with ma_ug_print byte for byte without a GPU (tests/test_host_cpu.py).
#include "../../include/miniasm_b200.h"
#include <vector>
#include <string>

extern "C" size_t mab_test_gfa_host(const ma_ug_t *ug, const sdict_t *d, const ma_sub_t *sub, char *out, size_t cap)
{
	std::vector<DUtgMeta> meta(ug->u.n ? ug->u.n : 1);
	std::vector<uint64_t> items;
	for (size_t i = 0; i < ug->u.n; ++i) {
		const ma_utg_t *p = &ug->u.a[i];
		meta[i].len = p->len, meta[i].circ = p->circ, meta[i].start = p->start, meta[i].end = p->end, meta[i].n = p->n, meta[i].first = (uint32_t)items.size();
		items.insert(items.end(), p->a, p->a + p->n);
	}
	std::vector<uint32_t> ioff(items.size() + 1, 0);
	for (size_t k = 0; k < items.size(); ++k) ioff[k + 1] = ioff[k] + (uint32_t)items[k];
	std::string text;
	std::vector<uint64_t> noff(d->n_seq ? d->n_seq : 1);
	std::vector<uint32_t> nlen(d->n_seq ? d->n_seq : 1);
	for (uint32_t r = 0; r < d->n_seq; ++r) noff[r] = text.size(), nlen[r] = (uint32_t)strlen(d->seq[r].name), text += d->seq[r].name;
	GfaView v{meta.data(), items.data(), ioff.data(), (uint32_t)ug->u.n, (uint64_t)items.size(),
	          (const DArc*)ug->g->arc, ug->g->n_arc, ug->g->idx, {nullptr, noff.data(), nlen.data(), text.data(), (const DSub*)sub}, nullptr, nullptr};
	const uint64_t n_rec = (uint64_t)v.n_utg * 2 + v.n_items + v.n_uarc;
	size_t tot = 0;
	for (uint64_t r = 0; r < n_rec; ++r) { CountSink s{0}; emit_record(v, r, s); tot += s.n; }
	if (out && tot <= cap) {
		char *p = out;
		for (uint64_t r = 0; r < n_rec; ++r) { WriteSink s{p}; emit_record(v, r, s); p = s.p; }
	}
	return tot;
}
