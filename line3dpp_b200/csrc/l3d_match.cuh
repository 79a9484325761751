// l3d_match.cuh — launch geometry + kernel declarations shared by l3d_match.cu and l3d_capi.cu
#pragma once
#include "l3d_device.cuh"
#include "../../include/l3d_capi.h"

/* geometry of k_match_topk (one CTA per SM); every knob can be overridden with -D for the sweep (tools/sweep_tiles.py) */
#ifndef MK_WARPS
#define MK_WARPS 32
#endif
#define MK_THREADS (32 * MK_WARPS)
#ifndef MK_SLOTS
#define MK_SLOTS 8                      /* row slots per warp: key list, threshold, count and constants of a row in flight */
#endif
#define MK_NSLOT (MK_WARPS * MK_SLOTS)  /* row slots per CTA; also the most rows of a unit whose target view takes several passes */
static_assert(MK_NSLOT <= 256, "a queue entry is (slot << 24) | ring position: 8 bits of slot");
#ifndef MK_UNIT_ROWS
#define MK_UNIT_ROWS 1024               /* most source rows per work unit (one CTA) of a pair whose target view is resident */
#endif
#ifndef MK_TT
#define MK_TT 512                       /* level-1 entries (target segments) per TMA stage (16 B arc + 16 B segment each: 16 KB) */
#endif
#ifndef MK_STAGES
#define MK_STAGES 6                     /* TMA ring depth: 3072 target segments resident; larger target views take several passes */
#endif
#ifndef MK_CAP
#define MK_CAP 32                       /* survivor keys kept per row before pruning to k (<= 32: one key per lane) */
#endif
#ifndef MK_SCAN_ORDER
#define MK_SCAN_ORDER 1                 /* order of a row's window pieces: 1 = arc class nearest the row's own span first, 0 = class
                                           order 0 .. NCLS - 1 (A/B builds only; the matches are the same either way) */
#endif

#define DK_THREADS 256
#ifndef DK_MINB
#define DK_MINB 4                       /* resident CTAs per SM of the dense kernel (register budget 64) */
#endif
#define DK_WARPS 8
#define DK_ROWS 32                      /* MAXIMUM source rows per CTA of the dense kernel; the launch picks 8..32 so that the tile
                                           count fills whole waves of 4 CTAs per SM (l3d_dense_rows_per_cta) */
#define DK_T 4                          /* target columns per lane: a CTA covers DK_ROWS x (8*4*32 = 1024) cells */
#define DKN_ROWS 32                     /* rows per CTA of the unfiltered test kernel */

struct L3DMat3 { float m[9]; };

size_t l3d_match_smem_bytes(int sem);        // dynamic shared memory of k_match_topk<sem, *>
size_t l3d_dense_smem_bytes();

__global__ void k_prep_segments(const float4* __restrict__ segs, const L3DViewDev* __restrict__ views, int num_views,
                                long long total, float4* __restrict__ cache);
// parameters of k_match_topk, passed by value
struct MatchArgs {
    const float4* segs; const float4* cache; const double* cache_d;       // segments, their float / double ray caches (cache_d: REF_CPU)
    const L3DViewDev* views; const L3DPairDev* pairs; const int4* units;  // units: (pair, first source row, rows, 0) of every CTA
    const uint4* arcs; const float4* arc_segs;                            // level-1 table (k_arcs_gather): packed arcs and their target segments,
    const L3DPairBasis* basis;                                            // both in window order; the pencil bases (k_pair_arcs)
    const uint4* wins; long long win_row0;                                // row windows (k_row_windows) of the rows from win_row0 on
    int* counts; l3d_match_rec* recs;                                     // per-row match count and records
    int knn;                                                              // TopK: k; Store: row stride; Count: unused
    float epi;
};
// what k_match_topk keeps of the matches of a row: the kNN best, only their number, or all of them
enum class Keep { TopK, Count, Store };
template <int SEM, Keep KEEP> __global__ void k_match_topk(MatchArgs A);    // SEM: L3D_SEM_REF_GPU / L3D_SEM_REF_CPU
#ifdef L3D_MATCH_PROBE
/* probe build only (tools/probe_match_phases.py): clock64 spans (a row's set-up: its constants, its window positions, the concatenation
   of its window pieces) of every warp by phase, counters (exact evaluations, those that pass the overlap test (REF_GPU), then the depth test, keys
   pushed into row lists, prune_row calls), and per CTA the longest, shortest and
   summed warp busy time, all summed over the CTAs of the launches since the last reset; read with l3d_match_probe (extern "C") */
enum { MP_SETUP, MP_WINDOW, MP_PIECES, MP_SCAN, MP_EXACT, MP_FINAL, MP_WAIT, MP_TAIL, MP_ROWS, MP_ENTRIES, MP_SURVIVORS, MP_EVALS, MP_DRAINS,
       MP_OVERLAP_PASS, MP_DEPTH_PASS, MP_PUSHED, MP_PRUNES, MP_CTAS, MP_BUSY_MAX, MP_BUSY_MIN, MP_BUSY_SUM, MP_N };
#endif
extern void (*const l3d_match_kernels[2][3])(MatchArgs);                   // every instantiation of k_match_topk: [SEM][KEEP]
// Caller-given candidates (l3d_match_pairs_cand): a candidate is the key (global row << 24) | target segment, global row = the pair's
// row_off + source segment.  k_cand_keys turns the caller's (pair, src_seg, tgt_seg) triples into keys (L3D_CAND_NONE for a triple of a
// pair that is not restricted or not evaluated by the call); a radix sort and a unique pass leave them sorted and distinct.
#define L3D_CAND_NONE 0xFFFFFFFFFFFFFFFFull
__global__ void k_cand_keys(long long n, const int32_t* __restrict__ trip, const L3DPairDev* __restrict__ pairs, const int* __restrict__ restricted,
                            int first_pair, int last_pair, unsigned long long* __restrict__ keys);
// parameters of k_match_cand, passed by value
struct CandArgs {
    const float4* segs; const float4* cache; const double* cache_d;       // as MatchArgs
    const L3DViewDev* views; const L3DPairDev* pairs;
    const longlong2* rpairs; int nrp; long long nrows;                    // (pair, its first row among the restricted rows) of every restricted
                                                                          // pair of the call, nrp of them; nrows restricted rows in all
    const unsigned long long* keys; const int* nkeys;                     // sorted distinct candidate keys, their number (device)
    int* counts; l3d_match_rec* recs;                                     // as MatchArgs
    int knn;                                                              // TopK: k; Store: row stride; Count: unused
    float epi;
};
// one warp per restricted row, CAND_WARPS warps per CTA: the row's candidates only, with k_match_topk's exact arithmetic and keep policy
#define CAND_WARPS 8
template <int SEM, Keep KEEP> __global__ void k_match_cand(CandArgs A);
extern void (*const l3d_cand_kernels[2][3])(CandArgs);                     // every instantiation of k_match_cand: [SEM][KEEP]
// level-1 pre-filter tables: one CTA per view pair of [first_pair, first_pair + gridDim.x): raw arcs + sort keys; after the sort
// k_arcs_gather writes the packed arcs and, in a parallel array, their target segments, in window order
__global__ void k_pair_arcs(const float4* __restrict__ segs, const L3DViewDev* __restrict__ views, const L3DPairDev* __restrict__ pairs,
                            int first_pair, int enabled, double ext, const int* __restrict__ restricted, uint4* __restrict__ raw,
                            unsigned long long* __restrict__ keys, unsigned int* __restrict__ vals, L3DPairBasis* __restrict__ basis);
__global__ void k_arcs_gather(long long n, const unsigned long long* __restrict__ keys, const unsigned int* __restrict__ vals,
                              const uint4* __restrict__ raw, const float4* __restrict__ segs, const L3DViewDev* __restrict__ views,
                              const L3DPairDev* __restrict__ pairs, int first_pair, uint4* __restrict__ out, float4* __restrict__ out_segs);
// row windows of the work units of one call (k_match_topk reads them): L3D_RW_WORDS words per row, 16-byte aligned, row r of the
// call (counted from win_row0) at wins + r * (L3D_RW_WORDS / 4):
//   word 0, 1: the pencil parameters k1, k2 of the row's two epipolar lines (line_kappa); word 2: 1 if the row skips level 1; word 3: 0;
//   word 4 + 2c, 5 + 2c (arc class c < L3D_ARC_NCLS): the first entry of the pair's sorted table inside class c whose arc start is not
//   below ka - 2^(L3D_ARC_CLS0 + c), resp. above kb (the class end when kb = 2^32 - 1); pair-relative, over the whole class
#define L3D_RW_WORDS 20
#define L3D_RW_STAGE 12000      /* most arc starts of a pair k_row_windows stages in shared memory: 47 KB, plus its static shared memory within
                                   the 48 KB a launch gets without opting in; larger tables are searched in place */
__global__ void k_row_windows(const float4* __restrict__ segs, const L3DViewDev* __restrict__ views, const L3DPairDev* __restrict__ pairs,
                              const int4* __restrict__ units, const L3DPairBasis* __restrict__ basis, const uint4* __restrict__ arcs,
                              long long win_row0, uint4* __restrict__ wins);
__global__ void k_sort_rows(int* __restrict__ counts, l3d_match_rec* __restrict__ recs, int stride, long long rows, int topk);
__global__ void k_prep_segments_f64(const float4* __restrict__ segs, const L3DViewDev* __restrict__ views, int num_views,
                                    long long total, double* __restrict__ cache);
int l3d_dense_rows_per_cta(int Ns, int Nt, int num_sms);
struct L3DDenseJob {            // one view pair of the dense contract; colb / tile0: its tiles in a batched launch
    const float4* ssegs; const float4* tsegs; const float4* scache; const float4* tcache; float4* depths; float* overlaps;
    L3DMat3 F; float3 Cs, Ct; int Ns, Nt, rows_per_cta, colb; long long tile0;
};
__global__ void k_match_dense(L3DDenseJob J, float epi);
__global__ void k_match_dense_batch(const L3DDenseJob* __restrict__ jobs, int njobs, float epi);
__global__ void k_match_dense_nofilter(L3DDenseJob J, float epi);
__global__ void k_compact_matches(const int* __restrict__ counts, const long long* __restrict__ row_ptr,
                                  const l3d_match_rec* __restrict__ recs, int knn, long long rows,
                                  l3d_match_rec* __restrict__ out);
__global__ void k_fp32_peak(float* __restrict__ out, int iters, float a, float b);
