// dump_dev.cu -- the stage dumps of the command line formatted on the GPU:
//   -p paf  print_hits  (main.c:21-30): one record per hit, in array order
//   -p bed  print_subs  (main.c:13-19): one record per current read; empty when the kept interval is empty (s == e)
//   -p sg   ma_sg_print (asm.c:41-55):  one record per arc of the string graph, in array order
// Each record is formatted by one thread with the sinks of fmt_sink.cuh (count pass, scan, write pass).
//
// Why chunked: a -S 2 -p paf dump of 100 M hits is ~9 GB of text, which must not need a device buffer and a pinned buffer of
// its own size.  The driver counts a window of records, scans the lengths into 64-bit positions, cuts the window into chunks
// of at most CHUNK bytes (a record longer than that is a chunk of its own), and writes the chunks one by one.  The pinned
// landing buffers are double-buffered: the fwrite of chunk k runs on the host while chunk k+1 is formatted and copied down.
#include "dump_dev.cuh"
#include <cub/cub.cuh>
#include <algorithm>

// "name:s+1-e\t" followed by e - s: the interval fields of print_hits, with e - s computed unsigned and printed as "%d"
template <class Sink> __host__ __device__ __forceinline__ void put_hit_read(Sink &s, const ReadNames &v, uint32_t r)
{
	put_read(s, v, r);
	const DSub b = v.sub[r];
	s.c('\t'); put_int(s, (int32_t)(b.e - (b.s_del & 0x7fffffffu)));
}

template <int K, class Sink> __host__ __device__ void emit_dump(const DumpView &v, uint64_t rec, Sink &s)
{
	if (K == DUMP_PAF) {
		const DHit h = v.hit[rec];
		put_hit_read(s, v.nm, (uint32_t)(h.qns >> 32)); s.c('\t');
		put_int(s, (int32_t)(uint32_t)h.qns); s.c('\t'); put_int(s, (int32_t)h.qe); s.c('\t'); s.c((h.ml_rev >> 31) ? '-' : '+'); s.c('\t');
		put_hit_read(s, v.nm, h.tn); s.c('\t');
		put_int(s, (int32_t)h.ts); s.c('\t'); put_int(s, (int32_t)h.te); s.c('\t');
		put_int(s, (int32_t)(h.ml_rev & 0x7fffffffu)); s.c('\t'); put_int(s, (int32_t)(h.bl_del & 0x7fffffffu));
		put_lit(s, "\t255\n", 5);
	} else if (K == DUMP_BED) {
		const DSub b = v.nm.sub[rec];
		const uint32_t s0 = b.s_del & 0x7fffffffu;
		if (s0 != b.e) {
			put_name(s, v.nm, (uint32_t)rec); s.c('\t'); put_int(s, (int32_t)s0); s.c('\t'); put_int(s, (int32_t)b.e); s.c('\n');
		}
	} else {
		const DArc a = v.arc[rec];
		const uint32_t u = (uint32_t)(a.ul >> 32), w = a.v;
		s.c('L'); s.c('\t'); put_read(s, v.nm, u >> 1); s.c('\t'); s.c((u & 1) ? '-' : '+'); s.c('\t');
		put_read(s, v.nm, w >> 1); s.c('\t'); s.c((w & 1) ? '-' : '+'); s.c('\t');
		put_int(s, (int32_t)(a.ol_del & 0x7fffffffu)); put_lit(s, ":\tL1:i:", 7); put_int(s, (int32_t)(uint32_t)a.ul); s.c('\n');
	}
}

template <int K> __global__ void k_dump_count(DumpView v, uint64_t r0, uint32_t n, uint64_t *len)
{
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		CountSink s{0};
		emit_dump<K>(v, r0 + i, s);
		len[i] = s.n;
	}
}

template <int K> __global__ void k_dump_write(DumpView v, uint64_t r0, uint32_t k0, uint32_t k1, const uint64_t *pos, char *out)
{
	const uint64_t base = pos[k0];
	for (uint32_t i = k0 + blockIdx.x * blockDim.x + threadIdx.x; i < k1; i += gridDim.x * blockDim.x) {
		WriteSink s{out + (pos[i] - base)};
		emit_dump<K>(v, r0 + i, s);
	}
}

// Greedy cut of a window into chunks: chunk j ends at record cut[2j] (exclusive) and text position cut[2j+1], the longest run of
// records from the previous end whose text fits `cap` bytes, or the single next record when it alone is longer.  pos[i] is the
// text position of record i, pos[n] the window's size.  One thread: a window has a handful of chunks.
__global__ void k_dump_cuts(const uint64_t *pos, uint32_t n, uint64_t cap, uint64_t *cut, unsigned long long *n_cut)
{
	uint32_t k = 0, j = 0;
	while (k < n) {
		const uint64_t base = pos[k];
		uint32_t lo = k + 1, hi = n;
		while (lo < hi) {
			const uint32_t mid = lo + (hi - lo + 1) / 2;
			if (pos[mid] - base <= cap) lo = mid; else hi = mid - 1;
		}
		cut[2 * j] = lo, cut[2 * j + 1] = pos[lo];
		++j, k = lo;
	}
	*n_cut = j;
}

template <int K> static size_t dump_write(MabDev &d, const DumpView &v, uint64_t n_rec, FILE *fp, char **pin, size_t &pin_cap)
{
	static const char *what[] = { "PAF", "BED", "string graph" };
	const uint32_t WIN = 1u << 20;         // records per window: 8 + 8 + 16 bytes of scratch each
	const uint64_t CHUNK = 64ull << 20;    // text per chunk
	if (n_rec == 0) return 0;
	const uint32_t nw_max = (uint32_t)std::min<uint64_t>(n_rec, WIN);
	uint64_t *len = mab_alloc<uint64_t>(d, nw_max);
	uint64_t *pos = mab_alloc<uint64_t>(d, (size_t)nw_max + 1);
	uint64_t *cut = mab_alloc<uint64_t>(d, 2 * (size_t)nw_max);
	MAB_CUDA(cudaMemsetAsync(pos, 0, 8, d.stream));
	size_t tb = 0;
	cub::DeviceScan::InclusiveSum(nullptr, tb, len, pos + 1, (int)nw_max, d.stream);
	char *dbuf = nullptr;
	size_t dcap = 0, total = 0, pend_bytes = 0;
	int b = 0, pend = -1;
	cudaEvent_t ev[2];
	for (int i = 0; i < 2; ++i) MAB_CUDA(cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming));
	auto flush = [&] {
		if (pend < 0) return;
		MAB_CUDA(cudaEventSynchronize(ev[pend]));
		if (fwrite(pin[pend], 1, pend_bytes, fp) != pend_bytes) { fprintf(stderr, "[E::miniasm_b200] short write of the %s text\n", what[K]); exit(74); }
		total += pend_bytes, pend = -1;
	};
	std::vector<uint64_t> hcut;
	for (uint64_t r0 = 0; r0 < n_rec; r0 += WIN) {
		const uint32_t nw = (uint32_t)std::min<uint64_t>(n_rec - r0, WIN);
		MAB_LAUNCH(d, k_dump_count<K>, mab_grid(nw, 256), 256, 0, v, r0, nw, len);
		void *tmp = d.tmp(tb);
		cub::DeviceScan::InclusiveSum(tmp, tb, len, pos + 1, (int)nw, d.stream);
		++d.n_lib;
		MAB_LAUNCH(d, k_dump_cuts, 1, 1, 0, pos, nw, CHUNK, cut, d.d_scal + SC_COUNT);
		flush();                                                     // the previous window's last chunk, while this one is counted
		const uint32_t n_cut = (uint32_t)d.get_scal(SC_COUNT);
		hcut.resize(2 * (size_t)n_cut);
		MAB_CUDA(cudaMemcpyAsync(hcut.data(), cut, hcut.size() * 8, cudaMemcpyDeviceToHost, d.stream));
		d.sync();
		uint32_t k0 = 0;
		uint64_t p0 = 0;
		for (uint32_t j = 0; j < n_cut; ++j) {
			const uint32_t k1 = (uint32_t)hcut[2 * j];
			const uint64_t p1 = hcut[2 * j + 1];
			const size_t bytes = (size_t)(p1 - p0);
			if (bytes) {
				const size_t want = std::max<size_t>(bytes, std::min<size_t>(CHUNK, 2 * bytes)); // grow-only, to a full chunk when chunks are large
				if (bytes > dcap) { d.free(dbuf); dbuf = (char*)d.alloc(want); dcap = want; }
				if (bytes > pin_cap) {
					flush();
					for (int i = 0; i < 2; ++i) { if (pin[i]) MAB_CUDA(cudaFreeHost(pin[i])); MAB_CUDA(cudaMallocHost(&pin[i], want)); }
					pin_cap = want;
				}
				MAB_LAUNCH(d, k_dump_write<K>, mab_grid(k1 - k0, 256), 256, 0, v, r0, k0, k1, pos, dbuf);
				MAB_CUDA(cudaMemcpyAsync(pin[b], dbuf, bytes, cudaMemcpyDeviceToHost, d.stream));
				MAB_CUDA(cudaEventRecord(ev[b], d.stream));
				flush();                                             // chunk k goes to the FILE while chunk k+1 is formatted
				pend = b, pend_bytes = bytes, b ^= 1;
			}
			k0 = k1, p0 = p1;
		}
	}
	flush();
	if (getenv("MAB_TRACE"))
		fprintf(stderr, "[T::dg_dump_write] %s: %llu records, %zu bytes; device scratch %zu bytes, pinned %zu bytes\n", what[K],
		        (unsigned long long)n_rec, total, (size_t)nw_max * 8 + ((size_t)nw_max + 1) * 8 + (size_t)nw_max * 16 + tb + dcap, 2 * pin_cap);
	for (int i = 0; i < 2; ++i) MAB_CUDA(cudaEventDestroy(ev[i]));
	d.free(dbuf); d.free(len); d.free(pos); d.free(cut);
	d.sync();
	return total;
}

size_t dg_dump_write(MabDev &d, DumpKind kind, const DumpView &v, uint64_t n_rec, FILE *fp, char **pin, size_t &pin_cap)
{
	if (kind == DUMP_PAF) return dump_write<DUMP_PAF>(d, v, n_rec, fp, pin, pin_cap);
	if (kind == DUMP_BED) return dump_write<DUMP_BED>(d, v, n_rec, fp, pin, pin_cap);
	return dump_write<DUMP_SG>(d, v, n_rec, fp, pin, pin_cap);
}

// ---- host probe (tests only): the same emitters compiled for the CPU, fed from the reference's host structs ------------------
// kind DUMP_PAF: recs = ma_hit_t[n]; DUMP_BED: n = d->n_seq, recs unused; DUMP_SG: recs = asg_arc_t[n].  Returns the size of the
// text; writes it to out when it fits cap.  Lets the CPU test tier compare the emitters with print_hits / print_subs /
// ma_sg_print byte for byte without a GPU (tests/test_dump_writers_cpu.py).
#include "../../include/miniasm_b200.h"
#include <string>

template <int K> static size_t dump_host(const DumpView &v, size_t n, char *out, size_t cap)
{
	size_t tot = 0;
	for (size_t r = 0; r < n; ++r) { CountSink s{0}; emit_dump<K>(v, r, s); tot += s.n; }
	if (out && tot <= cap)
		for (size_t r = 0; r < n; ++r) { WriteSink s{out}; emit_dump<K>(v, r, s); out = s.p; }
	return tot;
}

extern "C" size_t mab_test_dump_host(int kind, const void *recs, size_t n, const sdict_t *d, const ma_sub_t *sub, char *out, size_t cap)
{
	std::string text;
	std::vector<uint64_t> noff(d->n_seq ? d->n_seq : 1);
	std::vector<uint32_t> nlen(d->n_seq ? d->n_seq : 1);
	for (uint32_t r = 0; r < d->n_seq; ++r) noff[r] = text.size(), nlen[r] = (uint32_t)strlen(d->seq[r].name), text += d->seq[r].name;
	const DumpView v{{nullptr, noff.data(), nlen.data(), text.data(), (const DSub*)sub}, (const DHit*)recs, (const DArc*)recs};
	if (kind == DUMP_PAF) return dump_host<DUMP_PAF>(v, n, out, cap);
	if (kind == DUMP_BED) return dump_host<DUMP_BED>(v, n, out, cap);
	return dump_host<DUMP_SG>(v, n, out, cap);
}
