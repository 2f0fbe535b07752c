// gzstream.cuh -- the stepping decisions of the streaming gzip decoder (GzStream in gunzip_dev.cu, DESIGN.md section 3c):
// which units of a compressed segment chain, where the next segment starts, what history is handed on and how a member's
// CRC-32 is carried across segments.  __host__ __device__, so that tests/hostsim/gzstream_host.cpp runs exactly these steps.
//
// A segment is the compressed bytes from the carried position (an absolute bit: unit 0) up to a length or the end of the file.
// Its units are decoded by inf_run over the segment alone, so a unit that reaches the segment's last byte reports INF_SHORT
// (or, when a trailer ends exactly there, INF_END): in a segment that is not the file's end neither means the stream ends.
#pragma once
#include "inflate.cuh"

// what the chain does with a unit: take it and go on to its landing, take it as the stream's last, stop before it (the next
// segment starts at it), or reject the stream
enum { GZS_TAKE = 0, GZS_LAST = 1, GZS_STOP = 2, GZS_BAD = 3 };
// a chain that took no unit: unit 0 needs a longer segment, or its output alone is longer than the output room
enum { GZS_GROW = 4, GZS_SMALL = 5 };

// unit of status st and output length olen, after `total` bytes of output of this segment's chain, with room for cap in all
INF_HD int gzs_unit(int st, bool final, uint64_t total, uint64_t olen, uint64_t cap)
{
	if (st == INF_ERR) return GZS_BAD;                       // a fault inside the bytes present: damage
	if (st == INF_SHORT) return final ? GZS_BAD : GZS_STOP;  // ran past the segment: truncation only at the file's end
	if (st == INF_END && !final) return GZS_STOP;            // a trailer at the segment's end, not the file's
	if (olen > cap - total) return GZS_STOP;
	return st == INF_END ? GZS_LAST : GZS_TAKE;
}

struct GzsChain {
	uint32_t nc;       // units taken
	uint32_t stop;     // GZS_STOP: the unit the next segment starts at
	int kind;          // GZS_LAST, GZS_STOP (nc > 0), GZS_BAD, GZS_GROW or GZS_SMALL (nc == 0)
	uint64_t total, members;
};

// walk the units from unit 0 along their landings; chain[c] / off[c] / mbase[c] as k_gz_chain writes them
INF_HD void gzs_chain(const int *st, const uint32_t *land, const uint64_t *olen, const uint32_t *nmem, bool final, uint64_t cap,
                      uint32_t *chain, uint64_t *off, uint32_t *mbase, GzsChain &r)
{
	uint64_t total = 0, members = 0;
	uint32_t c = 0, u = 0;
	int k;
	for (;;) {
		k = gzs_unit(st[u], final, total, olen[u], cap);
		if (k == GZS_BAD || k == GZS_STOP) break;
		chain[c] = u, off[c] = total, mbase[c] = (uint32_t)members;
		total += olen[u], members += nmem[u], ++c;
		if (k == GZS_LAST) break;
		u = land[u]; // > u: the chain always moves on
	}
	if (k == GZS_STOP && c == 0) k = st[0] == INF_LAND || olen[0] > cap ? GZS_SMALL : GZS_GROW; // (a landing unit 0 stops only for room)
	r.nc = c, r.stop = u, r.kind = k, r.total = total, r.members = members;
}

// The CRC carry.  The segment's output [0, total) holds the tail of the member open at its start (raw CRC register carry_raw
// over its carry_len earlier bytes), then whole members, then the head of the member left open.  Piece m of the output is
// [m ? m_end[m-1] : 0, m < members ? m_end[m] : total) with raw CRC raw and length len; the first piece continues the carry.
INF_HD void gzs_piece(const uint32_t *x2k, uint32_t carry_raw, uint64_t carry_len, uint32_t m, uint32_t &raw, uint64_t &len)
{
	if (m == 0) raw = inf_crc_join(x2k, carry_raw, raw, len), len += carry_len;
}

// a member's trailer against its joined raw CRC and length
INF_HD bool gzs_member_ok(const uint32_t *x2k, uint32_t raw, uint64_t len, uint32_t crc, uint32_t isize)
{
	return inf_crc_final(x2k, raw, len) == crc && (uint32_t)len == isize;
}

// history and `valid` handed on: the window after the last unit taken (win[nc], valid[nc] of the window step seeded with the
// carried ones); the next segment starts at bit seg_bit + starts[stop], never at a member header
INF_HD uint64_t gzs_next_bit(uint64_t seg_bit, const uint64_t *starts, uint32_t stop) { return seg_bit + starts[stop]; }

// Segment lengths.  A fill takes about cap bytes of output; its segment is chosen when the segment before it is chained (from that
// fill's cap and the compressed / inflated ratio so far, 0.35 before 1 MB has come out), so that the next segment's pass 1 can
// start while the current one is still being resolved.  The first segment of a pass uses the fill's own cap.
INF_HD uint64_t gzs_seg_len(uint64_t cap, uint64_t in_used, uint64_t out_made)
{
	const double ratio = out_made > (1u << 20) ? (double)in_used / (double)out_made : 0.35;
	const uint64_t seg = (uint64_t)((double)cap * ratio * 1.1) + (16u << 10);
	return seg > cap + (16u << 10) ? cap + (16u << 10) : seg;
}

// The room memo: a fill that stopped before a landing unit of need_next bytes for want of room (the chain took total of cap)
// remembers that length; a later fill with less room than that returns at once, asking for more (a segment that starts there
// might cut the unit shorter, so this only leaves a window a little less full).
INF_HD uint64_t gzs_need_after(uint64_t need_next, uint64_t cap, uint64_t total) { return need_next > cap - total ? need_next : 0; }
INF_HD bool gzs_room_short(uint64_t need, uint64_t cap) { return need > cap; }

// units of a segment: the chunk size that gives about 16 K units, between 4 KiB and 64 KiB
INF_HD uint64_t gzs_chunk_for(uint64_t seg)
{
	uint64_t c = 4096;
	while (c < 65536 && c * 16384 < seg) c <<= 1;
	return c;
}
