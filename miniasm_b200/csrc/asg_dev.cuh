// asg_dev.cuh -- device-resident string graph (stage ii + the arc-level parts of stage iii).
// Counterpart of the reference's asg_t container and passes (asg.h:13-42, asg.c:22-193).
#pragma once
#include "mab_common.cuh"

struct DGraph {
	uint32_t n_seq = 0;       // reads; vertices = 2*n_seq
	uint32_t n_arc = 0;
	size_t   m_arc = 0;       // capacity of arc / arc2 (elements)
	bool is_srt = false, is_symm = false, has_idx = false;
	uint32_t len_bits = 32;   // every arc length < 2^len_bits (lets the radix sort skip dead key bits)
	DArc *arc = nullptr;      // canonical AoS arc array
	DArc *arc2 = nullptr;     // ping-pong buffer for compaction / sort output
	uint32_t *seq = nullptr;  // len:31 | del<<31 per read
	uint64_t *idx = nullptr;  // first<<32 | count per vertex
};

void dg_reserve(MabDev &d, DGraph &g, size_t m_arc);
void dg_set_nseq(MabDev &d, DGraph &g, uint32_t n_seq);
void dg_free(MabDev &d, DGraph &g);

// asg.c:57-70 (+ optional external deletion flags produced by dg_del_trans)
void dg_arc_rm(MabDev &d, DGraph &g, const uint8_t *flag);
uint32_t dg_n_del_seq(MabDev &d, const DGraph &g); // reads with the del bit set
void dg_arc_sort(MabDev &d, DGraph &g);          // asg.c:22-25
void dg_build_sorted(MabDev &d, DGraph &g, uint64_t *key, uint64_t *val, uint64_t *key2, uint64_t *val2, uint32_t n_in, uint32_t n_real, uint32_t lb, bool has_sentinel);
void dg_arc_index(MabDev &d, DGraph &g);         // asg.c:27-42
void dg_cleanup(MabDev &d, DGraph &g, const uint8_t *flag = nullptr); // asg.c:72-80
uint32_t dg_del_multi(MabDev &d, DGraph &g);     // asg.c:104-121
uint32_t dg_del_asymm(MabDev &d, DGraph &g);     // asg.c:124-138
void dg_symm(MabDev &d, DGraph &g);              // asg.c:140-145
uint32_t dg_del_trans(MabDev &d, DGraph &g, uint32_t fuzz);  // asg.c:148-193
// peer != null: neighbour slabs are read from peer[owner] + (nidx[w] >> 32) (sharded run with CUDA IPC peer access)
uint32_t dg_del_trans_flags(MabDev &d, DGraph &g, uint32_t fuzz, uint32_t own_lo, uint32_t own_hi, uint8_t **flag_out,
                            const DArc *const *peer = nullptr, const uint64_t *nidx = nullptr, const uint32_t *orig = nullptr, uint32_t world = 1);
uint32_t dg_del_short(MabDev &d, DGraph &g, float ratio);    // asg.c:83-101

// statistics of the last dg_del_trans call (for the roofline arithmetic in bench.py)
struct DelTransStats { uint64_t n_arc_in, n_vtx, inner_iters, n_reduced, n_big; float kernel_ms; };
extern thread_local DelTransStats g_del_trans_stats; // of the calling thread's last call (one thread drives one GPU)

extern int mab_del_trans_count_inner; // 1: asg_arc_del_trans also counts its inner-loop iterations (slower kernel variant)
extern thread_local int mab_mute; // 1: this thread is a non-zero rank of a multi-GPU run and prints no [M::...] lines
#define MAB_V(level) (!mab_mute && mab_verbose >= (level))
extern int mab_verbose;   // mirrors ma_verbose (common.c:3): >=3 prints the reference's [M::...] lines
