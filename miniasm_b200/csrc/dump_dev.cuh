// dump_dev.cuh -- the -p paf | bed | sg texts (main.c:13-30 print_subs / print_hits, asm.c:41-55 ma_sg_print) formatted on the
// GPU and written in chunks of bounded size; see dump_dev.cu.
#pragma once
#include "fmt_sink.cuh"

enum DumpKind { DUMP_PAF = 0, DUMP_BED = 1, DUMP_SG = 2 };

// What the emitters read.  nm: names and kept intervals by current read id (nm.sub is required for paf and bed);
// hit: the hits (paf); arc: the string graph's arcs (sg).
struct DumpView {
	ReadNames nm;
	const DHit *hit;
	const DArc *arc;
};

// Formats records [0, n_rec) of `kind` and writes them to fp in record order.  Device scratch and pinned memory are bounded
// by a fixed window of records and a fixed chunk of text, except that a single record longer than the chunk gets a buffer
// of its own size.  pin[2] / pin_cap: the caller's pair of pinned landing buffers and their size (grown here when a chunk needs
// more; chunk k+1 lands in one while chunk k is written to the FILE from the other).  Returns the number of bytes written;
// exits with code 74 on a short write.
size_t dg_dump_write(MabDev &d, DumpKind kind, const DumpView &v, uint64_t n_rec, FILE *fp, char **pin, size_t &pin_cap);
