// fmt_sink.cuh -- the text formatting shared by the GPU writers (gfa_dev.cu: -p ug, dump_dev.cu: -p paf|bed|sg).
//
// One thread formats one output record into a Sink.  A count pass runs the emitter with CountSink, a scan places the records,
// and a write pass runs the same emitter with WriteSink, so the lengths cannot disagree with the bytes.  Integer formats are the
// reference's: "%d" of the 32-bit value.
#pragma once
#include "mab_common.cuh"

struct CountSink {
	uint32_t n;
	__host__ __device__ __forceinline__ void c(char) { ++n; }
	__host__ __device__ __forceinline__ void bytes(const char *, uint32_t l) { n += l; }
	__host__ __device__ __forceinline__ void hole(uint32_t l, uint64_t *, const char *) { n += l; }
};
struct WriteSink {
	char *p;
	__host__ __device__ __forceinline__ void c(char ch) { *p++ = ch; }
	__host__ __device__ __forceinline__ void bytes(const char *s, uint32_t l) { for (uint32_t k = 0; k < l; ++k) p[k] = s[k]; p += l; }
	__host__ __device__ __forceinline__ void hole(uint32_t l, uint64_t *where, const char *base) { *where = (uint64_t)(p - base); p += l; } // left as the buffer was pre-filled
};

template <class Sink> __host__ __device__ __forceinline__ void put_dec(Sink &s, uint32_t x, int min_digits)
{
	char t[10];
	int n = 0;
	do t[n++] = (char)('0' + x % 10), x /= 10; while (x);
	for (int k = n; k < min_digits; ++k) s.c('0');
	while (n) s.c(t[--n]);
}
template <class Sink> __host__ __device__ __forceinline__ void put_int(Sink &s, int32_t v) // "%d"
{
	uint32_t x = (uint32_t)v;
	if (v < 0) s.c('-'), x = 0u - x;
	put_dec(s, x, 1);
}
template <class Sink> __host__ __device__ __forceinline__ void put_lit(Sink &s, const char *lit, uint32_t l) { for (uint32_t k = 0; k < l; ++k) s.c(lit[k]); }

// Read names by current id: orig maps a current id to the original one (null = identity), noff/nlen locate the name in text;
// sub holds the kept interval of each current read (null = no read selection ran: names print without the :s+1-e suffix).
struct ReadNames {
	const uint32_t *orig; const uint64_t *noff; const uint32_t *nlen; const char *text; const DSub *sub;
};

template <class Sink> __host__ __device__ __forceinline__ void put_name(Sink &s, const ReadNames &v, uint32_t r)
{
	const uint32_t o = v.orig ? v.orig[r] : r;
	s.bytes(v.text + v.noff[o], v.nlen[o]);
}
template <class Sink> __host__ __device__ __forceinline__ void put_read(Sink &s, const ReadNames &v, uint32_t r) // name or name:s+1-e
{
	put_name(s, v, r);
	if (v.sub) {
		const DSub b = v.sub[r];
		s.c(':'); put_int(s, (int32_t)((b.s_del & 0x7fffffffu) + 1)); s.c('-'); put_int(s, (int32_t)b.e);
	}
}
