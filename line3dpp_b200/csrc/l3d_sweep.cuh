// l3d_sweep.cuh — layout of the scoring sweep's match store (l3d_pipeline.cu), shared with the affinity stage.
//
// Every view owns a REGION of entries: all matches its segments can ever have in matches_[view] (line3D.h:387) - the direct
// records of the pairs it is the source of and the records of the pairs it is the target of (storeInverseMatches,
// line3D.cc:1672-1699) - already filtered by orientation (checkMatchOrientation, 811-858) and already in the reference's list
// order.  A region is a sequence of CHUNKS: (segment, neighbouring view) -> the entries of that segment with that view.
// Persistent state per entry: 9 bytes
//      e_val   u32   index g of the match record (l3d_match_rec, row-major fixed slots) | bit 31: the entry is the INVERSE view of it
//      e_score f32   score3D
//      e_flag  u8    bit 0 active (a direct match, or an inverse match whose source scored it > 0), bit 1 kept by filterMatches
// everything else (segment, target view/segment, depths, overlap) is re-read from the record.
#pragma once
#include "l3d_device.cuh"
#include "../../include/l3d_capi.h"

#define SW_ACTIVE 1u
#define SW_KEPT 2u
#define SW_INV 0x80000000u

struct SwView {               // per view (by view index)
    long long chunk_base;     // first chunk of the view: chunk(seg, c) = chunk_base + seg * np + c
    long long region_off;     // first entry of the view's region
    int ci_off, np;           // the view's chunk descriptors: cinfo[ci_off .. ci_off + np)
};

struct SwEntry { int seg, tgt_view, tgt_seg; float4 dep; float overlap; };

// pair of a record row: last p with row_off[p] <= row
__device__ __forceinline__ int sw_pair_of_row(const long long* __restrict__ row_off, int num_pairs, long long row)
{
    return last_le(num_pairs, row, [&](int i) { return __ldg(row_off + i); });
}

// what matches_[view][seg] holds for this entry: Match{src = (view, seg), tgt = (tgt_view, tgt_seg), depths from the entry's side}
__device__ __forceinline__ SwEntry sw_decode(unsigned int val, const L3DPairDev* __restrict__ pairs, const long long* __restrict__ row_off,
                                             int num_pairs, int knn, const l3d_match_rec* __restrict__ recs)
{
    const unsigned int g = val & ~SW_INV;
    const l3d_match_rec rec = recs[g];
    const long long row = (long long)(g / (unsigned int)knn);
    const int p = sw_pair_of_row(row_off, num_pairs, row);
    const int r = (int)(row - __ldg(row_off + p));
    SwEntry e;
    e.overlap = rec.overlap;
    if (val & SW_INV) { e.seg = (int)rec.tgt_seg; e.tgt_view = pairs[p].src; e.tgt_seg = r; e.dep = make_float4(rec.d_q1, rec.d_q2, rec.d_p1, rec.d_p2); }
    else { e.seg = r; e.tgt_view = pairs[p].tgt; e.tgt_seg = (int)rec.tgt_seg; e.dep = make_float4(rec.d_p1, rec.d_p2, rec.d_q1, rec.d_q2); }
    return e;
}
// depths only (p-side first), no pair lookup
__device__ __forceinline__ float4 sw_depths(unsigned int val, const l3d_match_rec* __restrict__ recs)
{
    const l3d_match_rec rec = recs[val & ~SW_INV];
    return (val & SW_INV) ? make_float4(rec.d_q1, rec.d_q2, rec.d_p1, rec.d_p2) : make_float4(rec.d_p1, rec.d_p2, rec.d_q1, rec.d_q2);
}

struct SwScoreArgs;
extern void (*const l3d_sw_score_kernels[2][2])(SwScoreArgs);     // every instantiation of the chain kernel k_sw_score: [REF_CPU][tables in shared memory]
size_t l3d_sw_score_smem_bytes(bool cpu_sem);                     // the most dynamic shared memory a k_sw_score launch uses
