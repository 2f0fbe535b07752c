// ugseq_dev.cu -- ma_ug_seq (asm.c:236-290) on the GPU: the reads file (FASTA/FASTQ, as kseq.h:163-211 reads it) is indexed in
// HBM, every record is matched to a read of the layout through a name table, and the bases of the layout's pieces are
// gathered (forward, or reverse-complemented through asm.c:224-233's table) straight into the sequence fields of the GFA
// text that gfa_dev.cu formats -- the unitig sequences never exist as separate strings.
//
// What the reference does per record: kseq_read -> name = header up to the first white space; sequence = the following
// lines joined (one trailing '\r' per line dropped) until a line starts with '>', '@' or '+'; after a '+' line, quality
// lines until they are as long as the sequence.  A record whose name is a read of the layout overwrites that read's piece
// of its unitig (a later record with the same name wins).
//
// A general multi-line FASTQ cannot be cut into records without walking it (a quality line may start with '@'); the two
// layouts every tool writes can, and a parallel check PROVES the layout before it is trusted:
//   FASTA-like : no line starts with '+'; then every line starting with '>' or '@' is a header and everything else is
//                sequence (exactly kseq's loop); any line width, CRLF, empty lines;
//   FASTQ-4    : 4 lines per record: '@' header, one sequence line, '+' line, one quality line of the same length.
// Anything else (multi-line FASTQ, junk before the first header, a line that is a lone '\r') returns UGSEQ_UNSUPPORTED and
// the caller falls back to the host reader (host/gfa.c ma_ug_seq), which walks the file like kseq does.
#include "ugseq_dev.cuh"
#include "ingest_dev.cuh"
#include "basecomp.cuh"
#include <cub/cub.cuh>

enum { LT_EMPTY = 0, LT_HEADER = 1, LT_PLUS = 2, LT_SEQ = 3 };

// per line: type by first byte, sequence bytes it contributes (length without the '\n' and without one trailing '\r')
__global__ void k_fx_lines(const char *__restrict__ text, size_t len, const uint64_t *__restrict__ start, uint64_t n_lines,
                           uint8_t *type, uint32_t *slen, unsigned long long *counts)
{	// counts: [0] headers, [1] '+' lines, [2] lone-'\r' lines, [3] lines longer than 2^31
	unsigned nh = 0, np = 0, ncr = 0, nbig = 0;
	for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n_lines; i += (uint64_t)gridDim.x * blockDim.x) {
		const uint64_t s = start[i];
		uint64_t e = i + 1 < n_lines ? start[i + 1] - 1 : (text[len - 1] == '\n' ? len - 1 : len);
		uint64_t l = e - s;
		uint8_t t = LT_EMPTY;
		if (l) {
			const char c = text[s];
			if (text[e - 1] == '\r') { if (l == 1) ++ncr; --l; }
			t = c == '>' || c == '@' ? LT_HEADER : (c == '+' ? LT_PLUS : LT_SEQ);
			if (l == 0) t = LT_EMPTY;
		}
		if (l >> 31) ++nbig, l = 0;
		type[i] = t, slen[i] = (uint32_t)l;
		nh += t == LT_HEADER, np += t == LT_PLUS;
	}
	nh = __reduce_add_sync(0xffffffffu, nh), np = __reduce_add_sync(0xffffffffu, np);
	ncr = __reduce_add_sync(0xffffffffu, ncr), nbig = __reduce_add_sync(0xffffffffu, nbig);
	if ((threadIdx.x & 31) == 0) {
		if (nh) atomicAdd(counts + 0, (unsigned long long)nh);
		if (np) atomicAdd(counts + 1, (unsigned long long)np);
		if (ncr) atomicAdd(counts + 2, (unsigned long long)ncr);
		if (nbig) atomicAdd(counts + 3, (unsigned long long)nbig);
	}
}

// FASTQ-4 hypothesis, one thread per record
__global__ void k_fq4_check(const uint8_t *type, const uint32_t *slen, const char *text, const uint64_t *start, uint64_t n_rec, unsigned long long *n_bad)
{
	unsigned bad = 0;
	for (uint64_t r = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; r < n_rec; r += (uint64_t)gridDim.x * blockDim.x) {
		const uint64_t l = 4 * r;
		const bool ok = type[l] == LT_HEADER && text[start[l]] == '@' && type[l + 1] == LT_SEQ && type[l + 2] == LT_PLUS && slen[l + 3] == slen[l + 1];
		bad += !ok;
	}
	bad = __reduce_add_sync(0xffffffffu, bad);
	if ((threadIdx.x & 31) == 0 && bad) atomicAdd(n_bad, (unsigned long long)bad);
}

__global__ void k_times4(uint64_t *a, uint64_t n) { for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) a[i] = 4 * i; }

struct IsHeader { const uint8_t *type; __device__ __forceinline__ bool operator()(uint64_t i) const { return type[i] == LT_HEADER; } };
struct SeqBytes { const uint8_t *type; const uint32_t *slen; __device__ __forceinline__ uint64_t operator()(uint64_t i) const { return type[i] == LT_SEQ ? slen[i] : 0; } };

// ---- name table of the layout's reads ---------------------------------------------------------------------------------
struct RTab { unsigned long long *key; uint32_t *id; uint64_t mask; };

__global__ void k_rtab_insert(uint32_t n, const uint32_t *orig, const uint64_t *noff, const uint32_t *nlen, const char *ntext, RTab t, unsigned long long *overflow)
{
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const uint32_t o = orig ? orig[i] : i;
		const unsigned long long h = name_hash(ntext + noff[o], 0, nlen[o], 0);
		uint64_t s = h & t.mask;
		int probe = 0;
		for (; probe < 1 << 16; ++probe, s = (s + 1) & t.mask)
			if (atomicCAS(&t.key[s], 0ull, h) == 0ull) { t.id[s] = i; break; } // names are distinct: equal hashes simply take separate slots
		if (probe == 1 << 16) atomicAdd(overflow, 1ull);
	}
}

// record r: name = header line after its first byte up to the first white-space byte (isspace: ' ', \t \n \v \f \r)
__global__ void k_rec_lookup(uint64_t n_rec, const uint64_t *hdr_line, const char *text, size_t len, const uint64_t *start, uint64_t n_lines,
                             RTab t, const uint32_t *orig, const uint64_t *noff, const uint32_t *nlen, const char *ntext, unsigned long long *rec_of_read)
{
	for (uint64_t r = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; r < n_rec; r += (uint64_t)gridDim.x * blockDim.x) {
		const uint64_t l = hdr_line[r];
		const uint64_t s = start[l] + 1, e = l + 1 < n_lines ? start[l + 1] - 1 : (text[len - 1] == '\n' ? len - 1 : len);
		uint64_t q = s;
		while (q < e) { const char c = text[q]; if (c == ' ' || (c >= '\t' && c <= '\r')) break; ++q; }
		const uint32_t nl = (uint32_t)(q - s);
		const unsigned long long h = name_hash(text + s, 0, nl, 0);
		for (uint64_t p = h & t.mask;; p = (p + 1) & t.mask) {
			const unsigned long long k = t.key[p];
			if (k == 0) break;                                     // not a read of the layout
			if (k != h) continue;
			const uint32_t id = t.id[p], o = orig ? orig[id] : id;
			if (nlen[o] != nl) continue;
			const char *a = ntext + noff[o], *b = text + s;
			bool same = true;
			for (uint32_t x = 0; same && x < nl; ++x) same = a[x] == b[x];
			if (same) { atomicMax(&rec_of_read[id], (unsigned long long)(r + 1)); break; } // the last record of a name wins (0 = none)
		}
	}
}

// ---- gather -----------------------------------------------------------------------------------------------------------
struct SeqSrc { // where the bases of a record are
	const char *text; const uint64_t *start; const uint8_t *type; const uint32_t *slen; const uint64_t *cum; // cum: sequence bytes before line i, over the whole file
	const uint64_t *hdr_line; uint64_t n_rec, n_lines; int fq4;
};

// text position of base p of the record whose sequence lines are [l0, l1) (FASTA-like: binary search on cum; FASTQ-4: one line)
__device__ __forceinline__ char seq_base(const SeqSrc &f, uint64_t l0, uint64_t l1, uint64_t p)
{
	if (f.fq4) return f.text[f.start[l0] + p];
	const uint64_t want = f.cum[l0] + p;
	uint64_t a = l0, b = l1;              // last line with cum[line] <= want
	while (b - a > 1) { const uint64_t m = a + (b - a) / 2; if (f.cum[m] <= want) a = m; else b = m; }
	return f.text[f.start[a] + (want - f.cum[a])];
}

// one warp per layout item k = (read, strand, length); its bytes go to out + seq_pos[unitig] + offset of the item in the unitig
__global__ void k_ugseq_gather(SeqSrc f, const DUtgMeta *meta, uint32_t n_utg, const uint64_t *items, const uint32_t *ioff, uint64_t n_items,
                               const unsigned long long *rec_of_read, const DSub *sub, const uint64_t *seq_pos, char *out, unsigned long long *n_short)
{
	const uint64_t warp = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5, n_warp = ((uint64_t)gridDim.x * blockDim.x) >> 5;
	const uint32_t lane = threadIdx.x & 31;
	for (uint64_t k = warp; k < n_items; k += n_warp) {
		const uint64_t it = items[k];
		const uint32_t id = (uint32_t)(it >> 33), rev = (uint32_t)(it >> 32) & 1, ln = (uint32_t)it;
		const unsigned long long rr = rec_of_read[id];
		if (rr == 0 || ln == 0) continue;                          // the read is not in the file: its piece stays 'N'
		const uint64_t r = rr - 1;
		uint32_t lo = 0, hi = n_utg;                               // unitig of item k: last one with first <= k
		while (hi - lo > 1) { const uint32_t m = lo + (hi - lo) / 2; if (meta[m].first <= k) lo = m; else hi = m; }
		const uint32_t off = ioff[k] - ioff[meta[lo].first];
		char *dst = out + seq_pos[lo] + off;
		const uint64_t l0 = f.hdr_line[r] + 1, l1 = f.fq4 ? l0 + 1 : (r + 1 < f.n_rec ? f.hdr_line[r + 1] : f.n_lines);
		const uint64_t sl = f.fq4 ? f.slen[l0] : (l1 < f.n_lines ? f.cum[l1] : f.cum[f.n_lines]) - f.cum[l0]; // bases in the record
		const uint64_t s0 = sub ? (sub[id].s_del & 0x7fffffffu) : 0, e0 = sub ? sub[id].e : sl;
		if (sub ? e0 > sl : ln > sl) { if (lane == 0) atomicAdd(n_short, 1ull); continue; } // asm.c:263 asserts it
		for (uint32_t i = lane; i < ln; i += 32)
			dst[i] = rev ? (char)mab_comp_of((unsigned char)seq_base(f, l0, l1, e0 - 1 - i)) : seq_base(f, l0, l1, s0 + i);
	}
}

void dg_reads_free(MabDev &d, DReadsIndex &ix)
{
	d.free(ix.start); d.free(ix.type); d.free(ix.slen); d.free(ix.cum); d.free(ix.hdr_line);
	ix = DReadsIndex();
}

int dg_reads_index(MabDev &d, const char *text, size_t len, DReadsIndex &ix)
{
	ix = DReadsIndex();
	if (len == 0) return 0;
	char first;
	MAB_CUDA(cudaMemcpyAsync(&first, text, 1, cudaMemcpyDeviceToHost, d.stream));
	ix.start = dev_line_starts(d, text, len, &ix.n_lines);         // (synchronises)
	if (first != '>' && first != '@') return UGSEQ_UNSUPPORTED;    // kseq would hunt for the first '>' or '@' byte anywhere
	const uint64_t n = ix.n_lines;
	ix.type = mab_alloc<uint8_t>(d, n); ix.slen = mab_alloc<uint32_t>(d, n);
	d.zero_scal(SC_TMP0, 4);
	MAB_LAUNCH(d, k_fx_lines, mab_grid(n, 256), 256, 0, text, len, ix.start, n, ix.type, ix.slen, d.d_scal + SC_TMP0);
	const uint64_t n_hdr = d.get_scal(SC_TMP0), n_plus = d.h_scal[SC_TMP0 + 1];
	if (d.h_scal[SC_TMP0 + 2] || d.h_scal[SC_TMP0 + 3]) return UGSEQ_UNSUPPORTED;
	if (n_plus == 0) ix.fq4 = 0;
	else {
		if (n % 4) return UGSEQ_UNSUPPORTED;
		d.zero_scal(SC_TMP0, 1);
		MAB_LAUNCH(d, k_fq4_check, mab_grid(n / 4, 256), 256, 0, ix.type, ix.slen, text, ix.start, n / 4, d.d_scal + SC_TMP0);
		if (d.get_scal(SC_TMP0)) return UGSEQ_UNSUPPORTED;
		ix.fq4 = 1;
	}
	cub::CountingInputIterator<uint64_t> pos(0);
	size_t tb = 0;
	void *tmp;
	if (ix.fq4) {
		ix.n_rec = n / 4;
		ix.hdr_line = mab_alloc<uint64_t>(d, ix.n_rec);
		MAB_LAUNCH(d, k_times4, mab_grid(ix.n_rec, 256), 256, 0, ix.hdr_line, ix.n_rec);
	} else {
		ix.n_rec = n_hdr;
		ix.hdr_line = mab_alloc<uint64_t>(d, n_hdr);
		unsigned long long *d_n = d.d_scal + SC_NSEL;
		IsHeader ish{ix.type};
		cub::DeviceSelect::If(nullptr, tb, pos, ix.hdr_line, d_n, (int64_t)n, ish, d.stream);
		tmp = d.tmp(tb);
		cub::DeviceSelect::If(tmp, tb, pos, ix.hdr_line, d_n, (int64_t)n, ish, d.stream);
		++d.n_lib;
		ix.cum = mab_alloc<uint64_t>(d, n + 1);
		SeqBytes sb{ix.type, ix.slen};
		cub::TransformInputIterator<uint64_t, SeqBytes, cub::CountingInputIterator<uint64_t>> in(pos, sb);
		cub::DeviceScan::ExclusiveSum(nullptr, tb, in, ix.cum, (int64_t)n, d.stream);
		tmp = d.tmp(tb);
		cub::DeviceScan::ExclusiveSum(tmp, tb, in, ix.cum, (int64_t)n, d.stream); // n items; the total is appended below
		++d.n_lib;
		uint64_t last_cum;
		uint32_t last_len; uint8_t last_type;
		MAB_CUDA(cudaMemcpyAsync(&last_cum, ix.cum + n - 1, 8, cudaMemcpyDeviceToHost, d.stream));
		MAB_CUDA(cudaMemcpyAsync(&last_len, ix.slen + n - 1, 4, cudaMemcpyDeviceToHost, d.stream));
		MAB_CUDA(cudaMemcpyAsync(&last_type, ix.type + n - 1, 1, cudaMemcpyDeviceToHost, d.stream));
		d.sync();
		const uint64_t total = last_cum + (last_type == LT_SEQ ? last_len : 0);
		MAB_CUDA(cudaMemcpyAsync(ix.cum + n, &total, 8, cudaMemcpyHostToDevice, d.stream));
		d.sync();
	}
	return 0;
}

int dg_ugseq_fill(MabDev &d, const char *text, size_t len, const DReadsIndex &ix, const DUnitigs &ug, const uint32_t *ioff,
                  uint32_t n_seq, const uint32_t *orig, const uint64_t *noff, const uint32_t *nlen, const char *ntext, const DSub *sub,
                  const uint64_t *seq_pos, char *out)
{
	if (ix.n_rec == 0 || ug.n_items == 0 || n_seq == 0) return 0;
	RTab t;
	uint64_t cap = 1024; while (cap < 2ull * n_seq) cap <<= 1;
	t.key = (unsigned long long*)mab_alloc<uint64_t>(d, cap); t.id = mab_alloc<uint32_t>(d, cap); t.mask = cap - 1;
	MAB_CUDA(cudaMemsetAsync(t.key, 0, cap * 8, d.stream));
	unsigned long long *rec_of_read = (unsigned long long*)mab_alloc<uint64_t>(d, n_seq);
	MAB_CUDA(cudaMemsetAsync(rec_of_read, 0, (size_t)n_seq * 8, d.stream));
	d.zero_scal(SC_TMP0, 2);
	MAB_LAUNCH(d, k_rtab_insert, mab_grid(n_seq, 256), 256, 0, n_seq, orig, noff, nlen, ntext, t, d.d_scal + SC_TMP0);
	MAB_LAUNCH(d, k_rec_lookup, mab_grid(ix.n_rec, 256), 256, 0, ix.n_rec, ix.hdr_line, text, len, ix.start, ix.n_lines, t, orig, noff, nlen, ntext, rec_of_read);
	SeqSrc f{text, ix.start, ix.type, ix.slen, ix.cum, ix.hdr_line, ix.n_rec, ix.n_lines, ix.fq4};
	const uint64_t n_warp = ug.n_items < (uint64_t)MAB_SMS * 64 ? ug.n_items : (uint64_t)MAB_SMS * 64;
	MAB_LAUNCH(d, k_ugseq_gather, (unsigned)((n_warp * 32 + 255) / 256), 256, 0, f, ug.meta, ug.n_utg, ug.items, ioff, ug.n_items, rec_of_read, sub, seq_pos, out, d.d_scal + SC_TMP0 + 1);
	const uint64_t overflow = d.get_scal(SC_TMP0), n_short = d.h_scal[SC_TMP0 + 1];
	d.free(t.key); d.free(t.id); d.free(rec_of_read);
	if (overflow) { fprintf(stderr, "[E::miniasm_b200] read-name table overflow\n"); exit(77); }
	return n_short ? UGSEQ_SHORT_RECORD : 0;
}
