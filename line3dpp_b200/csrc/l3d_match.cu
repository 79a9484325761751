// l3d_match.cu — matching kernels for sm_90a (compiled with -fmad=false, see l3d_device.cuh).
//
//   k_prep_segments : per-segment pre-pass; caches viewing rays and the interpretation-plane normal of every 2D
//                     segment (the reference recomputes 4 mat-vecs + 5 normalisations per surviving PAIR,
//                     cudawrapper.cu:148-154).
//   k_pair_arcs,    : level-1 tables of the view pairs of one call (l3d_device.cuh "pencil parameter"): every target segment as an arc of
//   k_arcs_gather     the epipolar pencil, grouped by arc length and sorted by arc start (one radix sort in between, l3d_capi.cu); the
//                     table carries each arc's target segment in a parallel array (32 B per pair and target).
//   k_row_windows   : per source row of every work unit, before k_match_topk: the pencil parameters of its epipolar lines (FP64) and
//                     the two ends of its window in every arc class (binary searches of the sorted table), 80 B per row, so that
//                     k_match_topk's row set-up is one load instead of a dependent FP64 chain and 16 searches on 16 of 32 lanes.
//   k_match_topk    : production kernel.  One CTA per SM (32 warps) = one work unit: a view pair and up to 1024 of its source rows.
//                     The pair's table (arcs + segments) is staged in shared memory by 1-D TMA (cp.async.bulk + mbarrier, 6 stages x
//                     512 entries x 32 B in flight from the first instruction): a target view of up to 3072 segments is resident in one
//                     pass, and a warp takes the unit's rows one at a time from a shared counter into one of its 8 row slots (constants,
//                     key list, score-to-beat), with no CTA barrier; larger target views take several passes over units of at most 256
//                     rows, each slot bound to one row.  Per row the warp clips the window of every arc class (k_row_windows) to the
//                     resident entries and scans only those entries, all windows as one concatenation (full warps), the
//                     class nearest the row's own span first so that its score-to-beat rises early: each
//                     lane runs the arc test (13 integer instructions) and the conservative float filter (27 flop + 2 rcp on the
//                     staged target segment) on its entry, branch-free, the survivors of both are ballot-compacted into a per-warp
//                     queue of ring positions (emptied before every refill) and evaluated 32 at a time on the staged segment with the
//                     exact, reference-order arithmetic; per-row survivor keys live in shared
//                     memory and the k best are selected and written once.  Replaces K_match_lines + the dense D2H + host
//                     priority-queue pass (cudawrapper.cu:186-253, 570-650).  Instruction-issue / latency bound; compulsory HBM
//                     traffic ~0.1 B/pair-eval.  One instantiation per semantics (REF_GPU / REF_CPU exact arithmetic) and keep
//                     policy (top-k, or the count and store passes of "keep all matches").
//   k_match_dense   : the reference's device contract (float4 depths + float overlap for EVERY cell,
//                     cudawrapper.cu:186-253), same filter + exact path, coalesced 20 B/cell writes: HBM-write bound.
#include "l3d_match.cuh"
#include "l3d_device_f64.cuh"

// ------------------------------------------------------------------------------------------------ pre-pass
__global__ void __launch_bounds__(256) k_prep_segments(const float4* __restrict__ segs, const L3DViewDev* __restrict__ views,
                                                       int num_views, long long total, float4* __restrict__ cache)
{
    long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const L3DViewDev* v = views + last_le(num_views, idx, [&](int i) { return views[i].seg_off; });
    float4 s = segs[idx];
    float3 r1 = normalize3(mulmat_h(v->RtKinv, s.x, s.y));
    float3 r2 = normalize3(mulmat_h(v->RtKinv, s.z, s.w));
    float3 n = normalize3(cross3(r1, r2));
    cache[3 * idx] = make_float4(r1.x, r1.y, r1.z, r2.x);
    cache[3 * idx + 1] = make_float4(r2.y, r2.z, n.x, n.y);
    cache[3 * idx + 2] = make_float4(n.z, 0.f, 0.f, 0.f);
}

// same for the double path (REF_CPU semantics): rays and plane normal exactly as triangulationDepths forms them
__global__ void __launch_bounds__(256) k_prep_segments_f64(const float4* __restrict__ segs, const L3DViewDev* __restrict__ views,
                                                           int num_views, long long total, double* __restrict__ cache)
{
    long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const L3DViewDev* v = views + last_le(num_views, idx, [&](int i) { return views[i].seg_off; });
    float4 s = segs[idx];
    D3 r1 = dray(v->RtKinv_d, (double)s.x, (double)s.y), r2 = dray(v->RtKinv_d, (double)s.z, (double)s.w);
    D3 n = dnormalized(dcross(r1, r2));
    double* o = cache + 9 * idx;
    o[0] = r1.x; o[1] = r1.y; o[2] = r1.z; o[3] = r2.x; o[4] = r2.y; o[5] = r2.z; o[6] = n.x; o[7] = n.y; o[8] = n.z;
}

// ------------------------------------------------------------------------------------------------ fused match + top-k
#ifdef L3D_MATCH_PROBE
__device__ unsigned long long g_match_probe[MP_N];
#define MPROBE(...) __VA_ARGS__
#else
#define MPROBE(...)
#endif

// A slot is the state of one source row in flight: key list, score-to-beat, count and the row's filter constants.  Every slot array
// is indexed by CTA slot (warp * MK_SLOTS + i); slot_row names the unit's row the slot holds.
struct MatchSmem {
    uint4 stage[MK_STAGES][MK_TT];                   // TMA-staged target arcs in window order (arc_may_match, l3d_device.cuh)
    float4 stage_seg[MK_STAGES][MK_TT];              // their target segments, same order (two arrays: both 16-byte loads of a warp are conflict-free)
    unsigned long long lists[MK_NSLOT][MK_CAP + 1];  // per-slot survivor keys (+1: slots start on different banks, lanes that push keys of different rows do not collide)
    float4 rowA[MK_NSLOT];                           // (e1.x, e1.y, e1.z, e2.x)
    float4 rowB[MK_NSLOT];                           // (e2.y, e2.z, g, 0.95 * score-to-beat)
    uint2 rowK[MK_NSLOT];                            // pencil parameters of the row's two epipolar lines (l3d_device.cuh, k_row_windows)
    float row_thr[MK_NSLOT];                         // overlap of the current k-th best survivor (0 until k are known)
    int list_cnt[MK_NSLOT];
    int slot_row[MK_NSLOT];                          // row of the unit (0 .. rows - 1) the slot holds; -1: never used
    unsigned char rowall[MK_NSLOT];                  // 1: an epipolar line of this row is not a pencil member to within the margins (source point at the epipole): no level 1
    unsigned int queue[MK_WARPS][96];                // survivors of both filters per warp: (slot << 24) | position in the ring, evaluated
                                                     // exactly 32 at a time (up to 64 pushed per scan step onto at most 31 waiting)
    L3DPairBasis B;                                  // the pair's pencil basis and the first sorted entry of every arc class, and the end (k_pair_arcs)
    float F[9];                                      // the pair's float fundamental matrix (row constants)
    int next_row;                                    // single-pass units: the next row a warp takes
    int nrows, nt, npass, pass;                      // rows of the unit, target segments, passes over the target view and the current pass
                                                     // (read here, not held in registers across the exact path)
    unsigned long long bars[MK_STAGES];
    // per-CTA constants of the (rarely executed, deliberately out-of-line) exact path
    const float4* cache; const float4* ssegs;        // float ray cache; the unit's first source segment
    const uint4* tarcs; const float4* tasegs;        // the pair's level-1 table (TMA sources of the refills)
    const unsigned int* wins;                        // row windows of the unit's rows (k_row_windows), L3D_RW_WORDS words per row
    long long src_base, toff;
    float3 Cs, Ct;
    float epi; int knn;
    int cap;                                         // keys a row list collects before it is cut to its k best (and the score-to-beat rises); a list holds at most cap keys, so the kNN <= 32 this kernel serves need 32 (smaller caps: sweep builds for kNN 10 only, DESIGN.md section 8)
    // REF_CPU semantics only: the exact path is matchingCPU's double arithmetic; the float filter stays the same
    const double* cache_d;
    double Fd[9]; D3 Csd, Ctd;
    // output: row base of the unit, per-row counts and records (row stride knn; keep-all modes: knn holds the stride found by Count)
    long long R0; int* counts_out; l3d_match_rec* recs_out;
#ifdef L3D_MATCH_PROBE
    unsigned long long probe[MK_WARPS][MP_N];
#endif
    // REF_GPU only, last: REF_CPU launches without them (l3d_match_smem_bytes), which leaves it 32 KB more L1 (DESIGN.md section 8)
    float4 srays[MK_NSLOT][3];                       // the row's cached rays and plane normal (k_prep_segments), for its depths
    float snum[MK_NSLOT];                            // the row's depth numerator depth_num(n, Cs, Ct) (depths_in_front)
};
size_t l3d_match_smem_bytes(int sem) { return sem == L3D_SEM_REF_GPU ? sizeof(MatchSmem) : offsetof(MatchSmem, srays); }

#ifdef L3D_MATCH_PROBE
__device__ __forceinline__ void probe_add(MatchSmem& S, int warp, int lane, int k, unsigned long long v) { if (lane == 0) S.probe[warp][k] += v; }
extern "C" int l3d_match_probe(unsigned long long* out, int reset)
{
    if (cudaMemcpyFromSymbol(out, g_match_probe, sizeof(unsigned long long) * MP_N) != cudaSuccess) return -1;
    if (reset) {
        static const unsigned long long zero[MP_N] = {};
        if (cudaMemcpyToSymbol(g_match_probe, zero, sizeof(zero)) != cudaSuccess) return -1;
    }
    return MP_N;
}
#endif

// rank of lane's key among the n <= 32 keys of a row list (number of larger keys; keys are unique)
__device__ __forceinline__ int rank_in_row(const unsigned long long* list, int n, unsigned long long k)
{
    int r = 0;
    for (int j = 0; j < n; ++j) r += list[j] > k;
    return r;
}

// the same rank when lane's key is one of the `rounds` best keys of the active lanes, 64 otherwise: `rounds` rounds of warp maximum
// (keys are unique and > 0) instead of ranking all keys against each other.  rounds is warp-uniform.
__device__ __forceinline__ int top_rank(unsigned long long k, bool active, int rounds)
{
    const unsigned int hi = (unsigned int)(k >> 32), lo = (unsigned int)k;
    int r = 64;
    for (int i = 0; i < rounds; ++i) {
        const unsigned int m = __reduce_max_sync(0xffffffffu, active ? hi : 0u);
        bool c = active && hi == m;
        unsigned int bm = __ballot_sync(0xffffffffu, c);
        if (__popc(bm) > 1) { const unsigned int l = __reduce_max_sync(0xffffffffu, c ? lo : 0u); c = c && lo == l; }
        if (c) { r = i; active = false; }
    }
    return r;
}

// keep the k best keys of a full row list (sorted, best first) and raise the row's score-to-beat
__device__ __noinline__ void prune_row(MatchSmem& S, int slot, int lane)
{
    const int knn = S.knn; const float epi = S.epi;
    MPROBE(probe_add(S, threadIdx.x >> 5, lane, MP_PRUNES, 1);)
    __syncwarp();
    const int n = min(S.list_cnt[slot], S.cap);
    const unsigned long long k = lane < n ? S.lists[slot][lane] : 0ull;
    const int r = knn <= 16 ? top_rank(k, lane < n, min(knn, n)) : rank_in_row(S.lists[slot], n, k);
    __syncwarp();
    if (lane < n && r < knn) S.lists[slot][r] = k;
    __syncwarp();
    if (lane == 0) {
        S.list_cnt[slot] = min(n, knn);
        if (n >= knn) {
            const float kth = key_overlap(S.lists[slot][knn - 1]);
            S.row_thr[slot] = kth;
            S.rowB[slot].w = 0.95f * fmaxf(kth, epi);
        }
    }
    __syncwarp();
}

// depths (d_p1, d_p2, d_q1, d_q2) of target j for the unit's row rl in slot sl, stored as Match stores them (floats, commons.h:186-203);
// true when all four are in front of the cameras: > 0 in float (REF_GPU, cudawrapper.cu:186-253; the row's rays from its slot) or
// > 1e-12 in double (REF_CPU, line3D.cc:925-1003)
template <int SEM>
__device__ __forceinline__ bool target_depths(const MatchSmem& S, int sl, int rl, unsigned int j, float* d)
{
    if (SEM == L3D_SEM_REF_CPU) {
        const SegRaysD s = load_rays_d(S.cache_d, S.src_base + rl), t = load_rays_d(S.cache_d, S.toff + j);
        double dd[4];
        exact_depths_f64(s, t, S.Csd, S.Ctd, dd);
        d[0] = (float)dd[0]; d[1] = (float)dd[1]; d[2] = (float)dd[2]; d[3] = (float)dd[3];
        return dd[0] > L3D_EPS_D && dd[1] > L3D_EPS_D && dd[2] > L3D_EPS_D && dd[3] > L3D_EPS_D;
    }
    const SegRays s = rays_from_smem(S.srays[sl]), t = load_rays(S.cache, S.toff + j);
    exact_depths(s, t, S.Cs, S.Ct, d);
    return d[0] > 0.0f && d[1] > 0.0f && d[2] > 0.0f && d[3] > 0.0f;
}

// REF_GPU: the overlap test of a candidate (target segment q) for the row held by slot sl (has == false: padding lane, never a match),
// K_match_lines' float overlap with the row's cached epipolar lines: it must exceed epi and reach the row's current k-th best (below it
// the candidate can never be selected).  Inline: the lanes stay converged through it.
__device__ __forceinline__ bool overlap_pass(const MatchSmem& S, int sl, float4 q, bool has, float* ov)
{
    const float4 rA = S.rowA[sl], rB = S.rowB[sl];
    bool inv;
    *ov = exact_overlap(q, make_float3(rA.x, rA.y, rA.z), make_float3(rA.w, rB.x, rB.y), &inv);
    return has && *ov > S.epi && *ov >= S.row_thr[sl];
}
// REF_CPU: the same test with matchingCPU's double overlap (line3D.cc:925-1003) and epipolar lines from the double F, then the depth
// test; out of line, so that its double values are not live in exact_batch
__device__ __noinline__ bool eval_candidate_f64(const MatchSmem& S, int sl, int rl, unsigned int j, float4 q, bool has, float* ov, float* d)
{
    if (!has) return false;
    const float4 sp = __ldg(S.ssegs + rl);
    const D3 e1 = dmulmat(S.Fd, d3((double)sp.x, (double)sp.y, 1.0)), e2 = dmulmat(S.Fd, d3((double)sp.z, (double)sp.w, 1.0));
    bool valid;
    *ov = exact_overlap_f64(q, e1, e2, &valid);
    return valid && *ov > S.epi && *ov >= S.row_thr[sl] && target_depths<L3D_SEM_REF_CPU>(S, sl, rl, j, d);
}

// exact evaluation of up to 32 queued candidates (one per lane): REF_GPU the overlap test (overlap_pass), then the depth test on the
// lanes that passed it; REF_CPU both in eval_candidate_f64.  Out of line on purpose: the hot filter loop must
// stay inside the instruction cache (the first version inlined this 5x -> 64 KB of SASS, 55 % "no instruction" stalls).
// A match is kept per KEEP: TopK pushes its key into the slot's list (cut to the kNN best when full), Count only counts it,
// Store writes its record (row stride S.knn, slot = arrival order; k_sort_rows puts the rows into the reference's
// ascending-target order afterwards).
template <int SEM, Keep KEEP>
__device__ __noinline__ void exact_batch(MatchSmem& S, unsigned int entry, bool has, int lane)
{
    const int knn = S.knn;
    MPROBE(const int warp = threadIdx.x >> 5;)
    const int sl = has ? (int)(entry >> 24) : 0;
    const int rl = S.slot_row[sl];
    const unsigned int pos = entry & 0xFFFFFFu;                      // position in the resident ring: target index and segment are staged
    const unsigned int j = (&S.stage[0][0])[pos].w;
    float ov = 0.0f, d[4];
    const float4 q = (&S.stage_seg[0][0])[pos];
    bool pending;
    if (SEM == L3D_SEM_REF_CPU) pending = eval_candidate_f64(S, sl, rl, j, q, has, &ov, d);
    else {
        // TopK and Count only need the depth test's outcome: a sign test without the divisions (depths_in_front), on the target's rays
        // loaded before the overlap arithmetic, which hides their L2 latency (Store holds the depths too and would spill with them)
        const SegRays t = KEEP != Keep::Store ? load_rays(S.cache, S.toff + j) : SegRays{};
        pending = overlap_pass(S, sl, q, has, &ov);
        MPROBE(probe_add(S, warp, lane, MP_OVERLAP_PASS, __popc(__ballot_sync(0xffffffffu, pending)));)
        if (pending)
            pending = KEEP == Keep::Store ? target_depths<SEM>(S, sl, rl, j, d) : depths_in_front(rays_from_smem(S.srays[sl]), t, S.Cs, S.Ct, S.snum[sl]);
    }
    MPROBE(probe_add(S, warp, lane, MP_DEPTH_PASS, __popc(__ballot_sync(0xffffffffu, pending)));)
    if (KEEP != Keep::TopK) {
        if (pending) {
            const int slot = atomicAdd(&S.list_cnt[sl], 1);             // a row belongs to one warp: no cross-warp contention
            if (KEEP == Keep::Store && slot < knn) {
                l3d_match_rec rec;
                rec.tgt_seg = j; rec.overlap = ov; rec.d_p1 = d[0]; rec.d_p2 = d[1]; rec.d_q1 = d[2]; rec.d_q2 = d[3];
                S.recs_out[(S.R0 + rl) * knn + slot] = rec;
            }
        }
        __syncwarp();
        return;
    }
    const unsigned long long key = make_key(ov, j);
    while (true) {
        MPROBE(bool pushed = false;)
        if (pending) {
            int slot = atomicAdd(&S.list_cnt[sl], 1);
            if (slot < S.cap) { S.lists[sl][slot] = key; pending = false; MPROBE(pushed = true;) }
        }
        MPROBE(probe_add(S, warp, lane, MP_PUSHED, __popc(__ballot_sync(0xffffffffu, pushed)));)
        unsigned int pm = __ballot_sync(0xffffffffu, pending);
        if (!pm) break;
        unsigned int todo = pm;                       // a row list is full: keep its k best and retry
        while (todo) {
            int leader = __ffs(todo) - 1;
            int row = __shfl_sync(0xffffffffu, sl, leader);
            prune_row(S, row, lane);
            unsigned int mine = __ballot_sync(0xffffffffu, pending && sl == row);
            todo &= ~mine;
            if (knn >= S.cap) {                       // list stays full (k == capacity): fold the pending keys in one by one
                while (mine) {
                    int l = __ffs(mine) - 1;
                    mine &= mine - 1;
                    unsigned long long k = __shfl_sync(0xffffffffu, key, l);
                    if (lane == 0 && k > S.lists[row][S.cap - 1]) S.lists[row][S.cap - 1] = k;
                    if (lane == l) pending = false;
                    prune_row(S, row, lane);   // re-sort; also refreshes the score-to-beat
                }
            }
        }
    }
    __syncwarp();
}

// write the match count of the row held by slot sl; TopK also selects its k best survivors and writes their records.  Runs once per
// row, when the slot is about to be reused or at the end of the unit: out of line.
template <int SEM, Keep KEEP>
__device__ __noinline__ void finalize_row(MatchSmem& S, int sl, int lane)
{
    const int knn = S.knn, rl = S.slot_row[sl];
    const long long R = S.R0 + rl;
    if (KEEP != Keep::TopK) { if (lane == 0) S.counts_out[R] = S.list_cnt[sl]; return; }
    const int n = min(S.list_cnt[sl], S.cap);
    if (lane == 0) S.counts_out[R] = min(n, knn);
    if (n == 0) return;
    const unsigned long long key = lane < n ? S.lists[sl][lane] : 0ull;
    const unsigned int j = key_tgt(key);
    // REF_GPU: the target's rays loaded before the ranking, which hides their latency
    const SegRays t = SEM == L3D_SEM_REF_GPU ? load_rays(S.cache, S.toff + (lane < n ? j : 0u)) : SegRays{};
    // REF_GPU kNN <= 16: prune_row's selection; REF_CPU ranks by counting (the selection makes its finalize_row spill, 18 % slower on
    // the benchmark's first 500 view pairs, H100 80GB HBM3, 700 W)
    const int rank = SEM == L3D_SEM_REF_GPU && knn <= 16 ? top_rank(key, lane < n, min(knn, n)) : rank_in_row(S.lists[sl], n, key);
    if (lane < n && rank < knn) {
        float d[4];
        if (SEM == L3D_SEM_REF_GPU) exact_depths(rays_from_smem(S.srays[sl]), t, S.Cs, S.Ct, d);
        else target_depths<SEM>(S, sl, rl, j, d);
        l3d_match_rec rec;
        rec.tgt_seg = j; rec.overlap = key_overlap(key);
        rec.d_p1 = d[0]; rec.d_p2 = d[1]; rec.d_q1 = d[2]; rec.d_q2 = d[3];
        S.recs_out[R * knn + rank] = rec;
    }
}

// ---- level-1 tables ------------------------------------------------------------------------------------------------
// orthonormal basis (u, v) of the pencil's subspace in scaled coordinates; NaN when F has no usable null vector
__device__ void pair_basis(const float* F, L3DPairBasis* B)
{
    double c[3][3];
    for (int k = 0; k < 3; ++k) {                         // columns of F: the epipolar lines of (1,0,0), (0,1,0), (0,0,1)
        const double x = F[k], y = F[3 + k], z = F[6 + k], n = sqrt(x * x + y * y + z * z);
        c[k][0] = n > 0.0 ? x / n : 0.0; c[k][1] = n > 0.0 ? y / n : 0.0; c[k][2] = n > 0.0 ? z / n : 0.0;
    }
    double E[3] = {0.0, 0.0, 0.0}, best = 0.0;
    for (int a = 0; a < 3; ++a)
        for (int b = a + 1; b < 3; ++b) {                 // E is orthogonal to every column: the best-conditioned cross product
            const double x = c[a][1] * c[b][2] - c[a][2] * c[b][1], y = c[a][2] * c[b][0] - c[a][0] * c[b][2], z = c[a][0] * c[b][1] - c[a][1] * c[b][0];
            const double n = x * x + y * y + z * z;
            if (n > best) { best = n; E[0] = x; E[1] = y; E[2] = z; }
        }
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    double n[3] = {E[0] / L3D_ARC_SCALE, E[1] / L3D_ARC_SCALE, E[2]};       // the epipole in scaled coordinates
    const double len = sqrt(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
    if (!(best > 1e-20) || !(len > 0.0) || !isfinite(len)) { for (int i = 0; i < 3; ++i) B->u[i] = B->v[i] = nan; return; }
    for (int i = 0; i < 3; ++i) n[i] /= len;
    int ax = 0;
    if (fabs(n[1]) < fabs(n[ax])) ax = 1;
    if (fabs(n[2]) < fabs(n[ax])) ax = 2;
    double a[3] = {0.0, 0.0, 0.0}; a[ax] = 1.0;
    double u[3] = {n[1] * a[2] - n[2] * a[1], n[2] * a[0] - n[0] * a[2], n[0] * a[1] - n[1] * a[0]};
    const double ul = sqrt(u[0] * u[0] + u[1] * u[1] + u[2] * u[2]);
    for (int i = 0; i < 3; ++i) u[i] /= ul;
    const double v[3] = {n[1] * u[2] - n[2] * u[1], n[2] * u[0] - n[0] * u[2], n[0] * u[1] - n[1] * u[0]};     // u x v = n
    for (int i = 0; i < 3; ++i) { B->u[i] = u[i]; B->v[i] = v[i]; }
}

// raw arc of one target segment: x = start A of T (absolute units), y = length of T, z / w = length of T_ext below / above T; y ==
// 0xFFFFFFFF: no usable arc.  Margins: a displacement of delta = 0.05 px + 0.4 % of the segment length of the pencil line at the point
// in question (200 x the rounding error of the reference's float intersection, 2.4e-4 px / sin(phi), and above the float filter's own
// margins), plus 4e-6 rad for the rounding of the angles themselves.  Everything uncertain (epipole within the margin of the extended
// segment or of its line, degenerate segment, non-monotone or non-finite values, T_ext longer than pi/2) has no arc.
__device__ uint4 target_arc(const L3DPairBasis& B, float4 q, double ext, bool enabled)
{
    const uint4 none = make_uint4(0u, 0xFFFFFFFFu, 0u, 0u);
    if (!enabled) return none;
    const double x1 = (double)q.x / L3D_ARC_SCALE, y1 = (double)q.y / L3D_ARC_SCALE, x2 = (double)q.z / L3D_ARC_SCALE, y2 = (double)q.w / L3D_ARC_SCALE;
    const double a1 = x1 * B.u[0] + y1 * B.u[1] + B.u[2], b1 = x1 * B.v[0] + y1 * B.v[1] + B.v[2];
    const double dx = x2 - x1, dy = y2 - y1, ac = dx * B.u[0] + dy * B.u[1], bc = dx * B.v[0] + dy * B.v[1];
    const double len = sqrt(dx * dx + dy * dy), rhoc = sqrt(ac * ac + bc * bc);
    const double delta = (0.05 + 4e-3 * len * L3D_ARC_SCALE) / L3D_ARC_SCALE;
    if (!(len > 1e-9) || !isfinite(rhoc) || !(rhoc > 1e-3 * len) || !(ext >= 0.0)) return none;
    {   // the target line through the epipole: (x1 x x2) . n ~ 0, n = u x v
        const double lx = y1 - y2, ly = x2 - x1, lz = x1 * y2 - y1 * x2;
        const double nx = B.u[1] * B.v[2] - B.u[2] * B.v[1], ny = B.u[2] * B.v[0] - B.u[0] * B.v[2], nz = B.u[0] * B.v[1] - B.u[1] * B.v[0];
        if (!(fabs(lx * nx + ly * ny + lz * nz) > 1e-4 * sqrt(lx * lx + ly * ly + lz * lz))) return none;
    }
    const double to_units = 4294967296.0 / 3.14159265358979323846;
    const unsigned int kc = arc_units(atan2(ac, -bc));
    const double ts[4] = {-ext, 0.0, 1.0, 1.0 + ext};
    double al[4], mg[4];
    for (int i = 0; i < 4; ++i) {          // (x.u, x.v) is linear along the line
        const double a = a1 + ts[i] * ac, b = b1 + ts[i] * bc, rho = sqrt(a * a + b * b);
        if (!isfinite(rho) || !(delta < 0.25 * rho)) return none;
        al[i] = (double)(unsigned int)(arc_units(atan2(a, -b)) - kc);
        mg[i] = (1.2 * delta / rho + 4e-6) * to_units;
    }
    const bool up = al[0] <= al[1] && al[1] <= al[2] && al[2] <= al[3], down = al[0] >= al[1] && al[1] >= al[2] && al[2] >= al[3];
    if (!up && !down) return none;
    const int i0 = up ? 0 : 3, i1 = up ? 1 : 2, i2 = up ? 2 : 1, i3 = up ? 3 : 0;      // ascending in cut coordinates
    const double top = 4294967295.0;
    double lo = fmax(al[i1] - mg[i1], 0.0), hi = fmin(al[i2] + mg[i2], top);
    double lox = fmin(fmax(al[i0] - mg[i0], 0.0), lo), hix = fmax(fmin(al[i3] + mg[i3], top), hi);
    lo = floor(lo); lox = floor(lox); hi = ceil(hi); hix = ceil(hix);
    if (!(hix - lox < 2147483648.0 - 524288.0)) return none;
    return make_uint4(kc + (unsigned int)lo, (unsigned int)(hi - lo), (unsigned int)(lo - lox), (unsigned int)(hix - hi));
}

// one CTA per view pair: basis, raw arcs, class sizes and the sort keys (pair, class, start of T).  A pair restricted to caller-given
// candidates (restricted non-null and set for it: l3d_match_pairs_cand) has an empty table.
__global__ void __launch_bounds__(256)
k_pair_arcs(const float4* __restrict__ segs, const L3DViewDev* __restrict__ views, const L3DPairDev* __restrict__ pairs, int first_pair,
            int enabled, double ext, const int* __restrict__ restricted, uint4* __restrict__ raw, unsigned long long* __restrict__ keys,
            unsigned int* __restrict__ vals, L3DPairBasis* __restrict__ basis)
{
    __shared__ L3DPairBasis B;
    __shared__ int cnt[L3D_ARC_NCLS + 1];
    const L3DPairDev* P = pairs + first_pair + blockIdx.x;
    if (threadIdx.x == 0) pair_basis(P->F, &B);
    if (threadIdx.x <= L3D_ARC_NCLS) cnt[threadIdx.x] = 0;
    __syncthreads();
    const L3DViewDev* vt = views + P->tgt;
    const float4* t = segs + vt->seg_off;
    const int Nt = restricted && restricted[first_pair + blockIdx.x] ? 0 : vt->nseg;
    for (int j = threadIdx.x; j < Nt; j += 256) {
        const uint4 r = target_arc(B, t[j], ext, enabled != 0);
        const int c = arc_class(r.y);
        raw[P->arc_off + j] = r;
        keys[P->arc_off + j] = ((unsigned long long)blockIdx.x << 36) | ((unsigned long long)c << 32) | (c == L3D_ARC_NCLS ? (unsigned long long)j : (unsigned long long)r.x);
        vals[P->arc_off + j] = (unsigned int)(P->arc_off + j);
        atomicAdd(&cnt[c], 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int off = 0;
        for (int c = 0; c <= L3D_ARC_NCLS; ++c) { B.cls_off[c] = off; off += cnt[c]; }
        B.cls_off[L3D_ARC_NCLS + 1] = off;
        basis[first_pair + blockIdx.x] = B;
    }
}

// packed entries in sorted order (arc_may_match, l3d_device.cuh) and, in a parallel array, their target segments
__global__ void __launch_bounds__(256)
k_arcs_gather(long long n, const unsigned long long* __restrict__ keys, const unsigned int* __restrict__ vals, const uint4* __restrict__ raw,
              const float4* __restrict__ segs, const L3DViewDev* __restrict__ views, const L3DPairDev* __restrict__ pairs, int first_pair,
              uint4* __restrict__ out, float4* __restrict__ out_segs)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned long long k = keys[i];
    const unsigned int src = vals[i];
    const uint4 r = raw[src];
    const bool wide = ((k >> 32) & 0xFull) == (unsigned long long)L3D_ARC_NCLS;
    const L3DPairDev* P = pairs + first_pair + (int)(k >> 36);
    const unsigned int j = src - (unsigned int)P->arc_off;
    const unsigned int w16 = (r.y + 65535u) >> 16, e1 = (r.z + 65535u) >> 16, eh = (r.w + 65535u) >> 16;
    out[i] = wide ? make_uint4(0u, 0u, L3D_ARC_WIDE, j) : make_uint4(r.x, e1 | (w16 << 16), eh, j);
    out_segs[i] = segs[views[P->tgt].seg_off + j];
}

// One CTA per work unit of k_match_topk: the row windows of its rows (l3d_match.cuh), one row per thread.  This is the arithmetic
// k_match_topk's row set-up needs before a row's scan, the same operations on the same values: the float epipolar lines F*p
// (mulmat_h), their pencil parameters (line_kappa, double) and per arc class the lower bounds of the two window keys in the sorted
// table (a row outside the pencil model, rall, needs none: the class start).  The arc starts of classes 0 .. NCLS - 1 are staged in
// shared memory when there are at most L3D_RW_STAGE of them (the launch sizes the dynamic shared memory), searched in the table otherwise.
__global__ void __launch_bounds__(256)
k_row_windows(const float4* __restrict__ segs, const L3DViewDev* __restrict__ views, const L3DPairDev* __restrict__ pairs,
              const int4* __restrict__ units, const L3DPairBasis* __restrict__ basis, const uint4* __restrict__ arcs, long long win_row0,
              uint4* __restrict__ wins)
{
    extern __shared__ unsigned int rw_starts[];
    __shared__ L3DPairBasis B;
    __shared__ float F[9];
    const int4 unit = units[blockIdx.x];
    const L3DPairDev* P = pairs + unit.x;
    constexpr int NB = (int)(sizeof(L3DPairBasis) / sizeof(int));
    static_assert(L3D_RW_WORDS == 4 + 2 * L3D_ARC_NCLS && NB + 9 <= 256, "row window layout; one word of the pair per thread");
    if (threadIdx.x < NB) reinterpret_cast<int*>(&B)[threadIdx.x] = reinterpret_cast<const int*>(basis + unit.x)[threadIdx.x];
    else if (threadIdx.x < NB + 9) F[threadIdx.x - NB] = P->F[threadIdx.x - NB];
    __syncthreads();
    const uint4* tab = arcs + P->arc_off;
    const bool staged = B.cls_off[L3D_ARC_NCLS] <= L3D_RW_STAGE;
    if (staged)
        for (int i = threadIdx.x; i < B.cls_off[L3D_ARC_NCLS]; i += blockDim.x) rw_starts[i] = tab[i].x;
    __syncthreads();
    const float4* ssegs = segs + views[P->src].seg_off + unit.y;
    uint4* out = wins + (P->row_off + unit.y - win_row0) * (L3D_RW_WORDS / 4);
    for (int r = threadIdx.x; r < unit.z; r += blockDim.x) {
        const float4 s = ssegs[r];
        const float3 e1 = mulmat_h(F, s.x, s.y), e2 = mulmat_h(F, s.z, s.w);
        bool off1, off2;
        const unsigned int k1 = line_kappa(B, e1, &off1), k2 = line_kappa(B, e2, &off2);
        const bool rall = off1 || off2;
        const bool fwd = (k2 - k1) < 0x80000000u;
        const unsigned int ka = fwd ? k1 : k2, kb = fwd ? k2 : k1;
        unsigned int pos[2 * L3D_ARC_NCLS];
#pragma unroll
        for (int i = 0; i < 2 * L3D_ARC_NCLS; ++i) {
            const int c = i >> 1;
            const bool upper = i & 1;
            int lo = B.cls_off[c], hi = B.cls_off[c + 1];
            const unsigned int key = upper ? kb + 1u : ka - (1u << (L3D_ARC_CLS0 + c));
            if (rall) hi = lo;
            else if (upper && kb == 0xFFFFFFFFu) lo = hi;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if ((staged ? rw_starts[mid] : __ldg(&tab[mid].x)) < key) lo = mid + 1; else hi = mid;
            }
            pos[i] = (unsigned int)lo;
        }
        uint4* o = out + (size_t)r * (L3D_RW_WORDS / 4);
        o[0] = make_uint4(k1, k2, rall ? 1u : 0u, 0u);
#pragma unroll
        for (int i = 0; i < L3D_ARC_NCLS / 2; ++i) o[1 + i] = make_uint4(pos[4 * i], pos[4 * i + 1], pos[4 * i + 2], pos[4 * i + 3]);
    }
}

// thread 0: start the TMA copies of the level-1 entries of pass `pass` of a pair into the ring; the arcs and the segments of a stage
// complete on the stage's barrier together
__device__ __forceinline__ void stage_entries(MatchSmem& S, int pass)
{
    const uint4* arcs = S.tarcs; const float4* asegs = S.tasegs;
    for (int i = 0; i < MK_STAGES; ++i) {
        const int o = (pass * MK_STAGES + i) * MK_TT, n = min(MK_TT, S.nt - o);
        if (n <= 0) break;
        const unsigned int bytes = (unsigned int)n * 16u;
        mbar_expect_tx(&S.bars[i], 2u * bytes);
        tma_load_1d(S.stage[i], arcs + o, bytes, &S.bars[i]);
        tma_load_1d(S.stage_seg[i], asegs + o, bytes, &S.bars[i]);
    }
}

// Does staged entry i pass both filters for a row (kappas k1, k2; rall: the row skips level 1; rA / rB: its float filter constants)?
// Level 1 (arc_may_match) and level 2 (filter_may_survive on the staged target segment) are both evaluated and ANDed without a branch:
// the arc test rejects only about a quarter of a window's entries.
__device__ __forceinline__ bool entry_may_match(const MatchSmem& S, int i, unsigned int k1, unsigned int k2, bool rall, float4 rA, float4 rB)
{
    const uint4 arc = (&S.stage[0][0])[i];
    return (arc_may_match(arc, k1, k2) | rall) & filter_may_survive((&S.stage_seg[0][0])[i], rA, rB);
}

// Entry index of position G + lane (clamped to the last position, tot - 1) of a row's concatenated window pieces (np pieces, lane q < np:
// position pE and shift pshift of piece q, positions strictly increasing).  Warp-uniform G; piece of G by one ballot, the pieces that
// start inside [G, G + 32) as bits of one reduction.
__device__ __forceinline__ int flat_entry(int G, int lane, int np, int pE, int pshift, int tot)
{
    const bool mine = lane < np;
    const int r0 = __popc(__ballot_sync(0xffffffffu, mine && pE <= G)) - 1;
    const unsigned int starts = __reduce_or_sync(0xffffffffu, mine && pE > G && pE < G + 32 ? 1u << (pE - G) : 0u);
    const int r = r0 + __popc(starts & ((2u << lane) - 1u));
    return min(G + lane, tot - 1) + __shfl_sync(0xffffffffu, pshift, r);
}

// the row windows of the unit's row rl (k_row_windows), one word per lane: the pencil parameters, the level-1 flag and the window
// positions of every arc class
__device__ __forceinline__ unsigned int row_window(const MatchSmem& S, int rl, int lane)
{ return lane < L3D_RW_WORDS ? __ldg(S.wins + (size_t)rl * L3D_RW_WORDS + lane) : 0u; }

// the constants of the unit's row rl into slot sl, and an empty key list: the epipolar lines F*p (cudawrapper.cu:216-217) and the float
// filter's scale; REF_GPU also its cached rays (lanes 0 .. 2, one float4 each) and their depth numerator, which every depth test of
// the row uses.  Returns the row's windows (row_window), loaded together with its segment and rays so that the loads overlap.
template <int SEM>
__device__ __forceinline__ unsigned int setup_row(MatchSmem& S, int sl, int rl, int lane)
{
    const unsigned int rw = row_window(S, rl, lane);
    const float4 s = __ldg(S.ssegs + rl);
    if (SEM == L3D_SEM_REF_GPU) {
        const float4 ray = lane < 3 ? __ldg(S.cache + 3 * (S.src_base + rl) + lane) : make_float4(0.f, 0.f, 0.f, 0.f);
        const float nz = __shfl_sync(0xffffffffu, ray.x, 2);                 // n = (c1.z, c1.w, c2.x), rays_from_smem
        if (lane < 3) S.srays[sl][lane] = ray;
        if (lane == 1) S.snum[sl] = depth_num(make_float3(ray.z, ray.w, nz), S.Cs, S.Ct);
    }
    const float3 e1 = mulmat_h(S.F, s.x, s.y), e2 = mulmat_h(S.F, s.z, s.w);
    if (lane == 0) {
        const float g = L3D_FILTER_C1 * fmaxf(sqrtf(e1.x * e1.x + e1.y * e1.y), sqrtf(e2.x * e2.x + e2.y * e2.y));
        S.rowA[sl] = make_float4(e1.x, e1.y, e1.z, e2.x);
        S.rowB[sl] = make_float4(e2.y, e2.z, g, 0.95f * S.epi);
        S.list_cnt[sl] = 0;
        S.row_thr[sl] = 0.0f;
        S.slot_row[sl] = rl;
    }
    __syncwarp();
    return rw;
}

// evaluate every pending candidate of the warp's queue (qn < 32 of them)
template <int SEM, Keep KEEP>
__device__ __forceinline__ void drain_queue(MatchSmem& S, int warp, int lane, int& qn)
{
    __syncwarp();
    if (qn > 0) {
        MPROBE(const long long t0 = clock64();)
        const bool has = lane < qn;
        exact_batch<SEM, KEEP>(S, has ? S.queue[warp][lane] : 0u, has, lane);
        MPROBE(probe_add(S, warp, lane, MP_EXACT, clock64() - t0); probe_add(S, warp, lane, MP_EVALS, qn);)
        qn = 0;
    }
}

// Scan the window entries of the row in slot sl (its row windows rw, row_window) that lie in the ring entries [base, base + cnt) of the
// pair's level-1 table resident in the current pass, and queue the survivors of both filters; the queue is evaluated 32 at a time.
template <int SEM, Keep KEEP>
__device__ __forceinline__ void scan_row(MatchSmem& S, int sl, unsigned int rw, int warp, int lane, int& qn)
{
    const int base = S.pass * (MK_STAGES * MK_TT), cnt = min(MK_STAGES * MK_TT, S.nt - base);
    MPROBE(const long long t_row = clock64(); long long t_exact = 0;)
    const unsigned int lt_mask = (1u << lane) - 1u;
    const int* cls_off = S.B.cls_off;
    // the row's constants, re-read from shared memory after exact batches instead of held across them (register budget of 32 warps);
    // rB.w: the score-to-beat, which the batches may raise (a stale value only rejects less)
    uint2 kr = make_uint2(__shfl_sync(0xffffffffu, rw, 0), __shfl_sync(0xffffffffu, rw, 1));
    bool rall = __shfl_sync(0xffffffffu, rw, 2) != 0u;
    if (lane == 0) { S.rowK[sl] = kr; S.rowall[sl] = rall ? 1 : 0; }
    float4 rA = S.rowA[sl];
    float4 rB = S.rowB[sl];
    // short arc [ka, kb] between the two kappa values: a target of class c can only match if its arc starts in [ka - 2^(CLS0 + c), kb]
    const bool fwd = (kr.y - kr.x) < 0x80000000u;
    const unsigned int ka = fwd ? kr.x : kr.y, kb = fwd ? kr.y : kr.x;
    // Lanes 2i and 2i + 1 (i < NCLS) work on class c, the i-th class of the row's scan order.  The best overlaps come from targets
    // whose arc is about as long as the row's own span kb - ka, so the class of that span goes first, then the classes on either
    // side of it by distance (the smaller class first on a tie): the row's score-to-beat rises after fewer exact evaluations.  The
    // order only changes when candidates arrive, not which of them are kept.
    int c = min(lane >> 1, L3D_ARC_NCLS - 1);
#if MK_SCAN_ORDER
    {
        const int rc = min(arc_class(kb - ka), L3D_ARC_NCLS - 1), m = min(rc, L3D_ARC_NCLS - 1 - rc);   // m classes on both sides
        const int d = c <= 2 * m ? (c + 1) >> 1 : c - m;
        const bool below = c <= 2 * m ? (c & 1) != 0 : 2 * rc > L3D_ARC_NCLS - 1;
        c = below ? rc - d : rc + d;
    }
#endif
    // lanes 0 .. 2 * NCLS - 1: lower / upper end of the window of class c inside the resident part of that class.  The row's window
    // position over the whole class, clipped to the resident entries [base, base + cnt): a class is sorted, so that is the first resident
    // entry of the class at or after the key, as a search of the resident part would find it.
    const int res = min(max((int)__shfl_sync(0xffffffffu, rw, 4 + 2 * c + (lane & 1)) - base, 0), cnt);
    MPROBE(const long long t_win = clock64(); probe_add(S, warp, lane, MP_WINDOW, t_win - t_row);)
    // lane p < 2 * NCLS: piece p & 1 of the window of class c (two pieces when the window wraps around 2^32); lane 2 * NCLS: the
    // targets every row looks at, last.  A row outside the pencil model (rall) takes everything as one piece.
    int plo = 0, phi = 0;
    {
        const int i0 = __shfl_sync(0xffffffffu, res, lane & ~1), i1 = __shfl_sync(0xffffffffu, res, lane | 1);
        const int s_c = min(max(cls_off[c] - base, 0), cnt), e_c = min(max(cls_off[c + 1] - base, 0), cnt);
        const bool wrap = ka - (1u << (L3D_ARC_CLS0 + c)) > kb;
        if (lane < 2 * L3D_ARC_NCLS) {
            if (!(lane & 1)) { plo = wrap ? s_c : i0; phi = i1; }
            else if (wrap) { plo = i0; phi = e_c; }
        } else if (lane == 2 * L3D_ARC_NCLS) { plo = min(max(cls_off[L3D_ARC_NCLS] - base, 0), cnt); phi = cnt; }
        if (rall) { plo = 0; phi = lane == 0 ? cnt : 0; }
    }
    // The pieces are scanned as one concatenation, so that every step but the row's last fills all 64 lanes: a window piece
    // averages a few dozen entries.  Lane q < np holds the q-th non-empty piece: its position E in the concatenation and the
    // shift (first entry - E) that turns a position of that piece into an entry index.
    const int len = phi - plo;
    const unsigned int ne = __ballot_sync(0xffffffffu, len > 0);
    int ex = len;
    for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, ex, o); if (lane >= o) ex += v; }
    const int tot = __shfl_sync(0xffffffffu, ex, 31), np = __popc(ne);
    ex -= len;
    const int src = lane < np ? (int)__fns(ne, 0u, lane + 1) : 0;
    const int pE = __shfl_sync(0xffffffffu, ex, src), pshift = __shfl_sync(0xffffffffu, plo - ex, src);
    MPROBE(probe_add(S, warp, lane, MP_PIECES, clock64() - t_win); const long long t_scan = clock64(); probe_add(S, warp, lane, MP_ENTRIES, tot);)
    for (int G = 0; G < tot; G += 64) {                 // two entries per lane: half the loop / vote / push overhead per entry
        const int ia = flat_entry(G, lane, np, pE, pshift, tot), ib = flat_entry(G + 32, lane, np, pE, pshift, tot);
        const bool pa = entry_may_match(S, ia, kr.x, kr.y, rall, rA, rB) & (G + lane < tot);
        const bool pb = entry_may_match(S, ib, kr.x, kr.y, rall, rA, rB) & (G + 32 + lane < tot);
        const unsigned int ba = __ballot_sync(0xffffffffu, pa), bb = __ballot_sync(0xffffffffu, pb);
        if (ba | bb) {
            MPROBE(probe_add(S, warp, lane, MP_SURVIVORS, __popc(ba) + __popc(bb));)
            if (pa) S.queue[warp][qn + __popc(ba & lt_mask)] = ((unsigned int)sl << 24) | (unsigned int)ia;
            qn += __popc(ba);
            if (pb) S.queue[warp][qn + __popc(bb & lt_mask)] = ((unsigned int)sl << 24) | (unsigned int)ib;
            qn += __popc(bb);
            __syncwarp();
            if (qn >= 32) {
                MPROBE(const long long t0 = clock64();)
                do { qn -= 32; exact_batch<SEM, KEEP>(S, S.queue[warp][qn + lane], true, lane); MPROBE(probe_add(S, warp, lane, MP_EVALS, 32);) } while (qn >= 32);
                MPROBE(t_exact += clock64() - t0;)
                kr = S.rowK[sl]; rall = S.rowall[sl] != 0; rA = S.rowA[sl]; rB = S.rowB[sl];
            }
        }
    }
    MPROBE(probe_add(S, warp, lane, MP_SCAN, clock64() - t_scan - t_exact); probe_add(S, warp, lane, MP_EXACT, t_exact);)
}

// One instantiation per semantics (L3D_SEM_*: the exact path's arithmetic; the staging, scan and float filter are the same) and
// keep policy.  TopK is the production kernel.  kNN <= 0 ("keep all matches", cudawrapper.cu:628-636 / line3D.cc:988-996) runs
// Count (A.knn unused), then Store with the row stride found by Count in A.knn.
// One CTA per SM and per work unit (a pair and a range of its source rows, stage_pairs in l3d_capi.cu).  A target view of up to
// MK_STAGES * MK_TT segments is resident in one pass: a warp takes the unit's rows one at a time from a shared counter as soon as it
// has a slot, so no warp waits for another until the unit ends.  Larger target views take several passes with a CTA barrier each; their
// units have at most MK_NSLOT rows, every warp's slots hold fixed rows and keep their lists across the passes.
// The pair, view and basis records are read with explicit __ldg: pointers taken from a parameter block carry no __restrict__.
template <int SEM, Keep KEEP>
__global__ void __launch_bounds__(MK_THREADS, 1) k_match_topk(const MatchArgs A)
{
    MPROBE(const long long t_start = clock64();)
    extern __shared__ __align__(128) unsigned char smem_raw[];
    MatchSmem& S = *reinterpret_cast<MatchSmem*>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int4 unit = __ldg(A.units + blockIdx.x);
    const L3DPairDev* P = A.pairs + unit.x;
    const int row0 = unit.y, nrows = unit.z;
    const L3DViewDev* vs = A.views + __ldg(&P->src);
    const L3DViewDev* vt = A.views + __ldg(&P->tgt);
    const int Nt = __ldg(&vt->nseg);
    const int RES = MK_STAGES * MK_TT;                     // entries resident at a time; larger target views take several passes
    const int npass = (Nt + RES - 1) / RES;
    if (tid == 0) {
        const long long soff = __ldg(&vs->seg_off);
        S.cache = A.cache; S.ssegs = A.segs + soff + row0; S.src_base = soff + row0; S.toff = __ldg(&vt->seg_off);
        S.epi = A.epi; S.knn = A.knn; S.cap = MK_CAP; S.next_row = 0; S.nrows = nrows; S.nt = Nt; S.npass = npass; S.pass = 0;
        S.tarcs = A.arcs + __ldg(&P->arc_off); S.tasegs = A.arc_segs + __ldg(&P->arc_off);
        S.Cs = make_float3(__ldg(&vs->C[0]), __ldg(&vs->C[1]), __ldg(&vs->C[2])); S.Ct = make_float3(__ldg(&vt->C[0]), __ldg(&vt->C[1]), __ldg(&vt->C[2]));
        S.R0 = __ldg(&P->row_off) + row0; S.counts_out = A.counts; S.recs_out = A.recs;
        S.wins = reinterpret_cast<const unsigned int*>(A.wins + (S.R0 - A.win_row0) * (L3D_RW_WORDS / 4));
        if (SEM == L3D_SEM_REF_CPU) {
            S.cache_d = A.cache_d;
            for (int i = 0; i < 9; ++i) S.Fd[i] = __ldg(&P->Fd[i]);
            S.Csd = d3(__ldg(&vs->C_d[0]), __ldg(&vs->C_d[1]), __ldg(&vs->C_d[2])); S.Ctd = d3(__ldg(&vt->C_d[0]), __ldg(&vt->C_d[1]), __ldg(&vt->C_d[2]));
        }
        for (int i = 0; i < MK_STAGES; ++i) mbar_init(&S.bars[i], 1);
        mbar_fence_init();
        stage_entries(S, 0);                            // the first pass is in flight while the rows are set up
    }
    constexpr int NB = (int)(sizeof(L3DPairBasis) / sizeof(int));
    static_assert(sizeof(L3DPairBasis) % sizeof(int) == 0 && NB + 9 + 1 <= MK_THREADS, "one word per thread");
    if (tid < NB) reinterpret_cast<int*>(&S.B)[tid] = __ldg(reinterpret_cast<const int*>(A.basis + unit.x) + tid);
    else if (tid < NB + 9) S.F[tid - NB] = __ldg(&P->F[tid - NB]);
    for (int i = tid; i < MK_NSLOT; i += MK_THREADS) S.slot_row[i] = -1;
    MPROBE(if (tid < MP_N * MK_WARPS) (&S.probe[0][0])[tid] = 0ull; long long t_wait = clock64();)
    __syncthreads();
    MPROBE(probe_add(S, warp, lane, MP_WAIT, clock64() - t_wait);)

    int qn = 0;    // warp-uniform fill of the candidate queue
    MPROBE(t_wait = clock64();)
    while (S.pass < S.npass) {                         // passes over the target view
        for (int i = 0; i < MK_STAGES && (S.pass * MK_STAGES + i) * MK_TT < S.nt; ++i) mbar_wait(&S.bars[i], (unsigned int)(S.pass & 1));
        MPROBE(probe_add(S, warp, lane, MP_WAIT, clock64() - t_wait);)
        for (int sl = warp * MK_SLOTS;;) {
            // next row: single pass, the next untaken row of the unit; several passes, the warp's fixed rows (slot sl holds row sl)
            int rl = sl;
            if (S.npass == 1) {
                if (lane == 0) rl = atomicAdd(&S.next_row, 1);
                rl = __shfl_sync(0xffffffffu, rl, 0);
            }
            if (rl >= S.nrows) break;
            unsigned int rw;
            if (S.pass == 0) {
                if (S.slot_row[sl] >= 0) {             // the slot's previous row: its queued candidates first (rarely any), then its result
                    if (__any_sync(0xffffffffu, lane < qn && (S.queue[warp][lane] >> 24) == (unsigned int)sl)) {
                        MPROBE(probe_add(S, warp, lane, MP_DRAINS, 1);)
                        drain_queue<SEM, KEEP>(S, warp, lane, qn);
                    }
                    MPROBE(const long long t0 = clock64();)
                    finalize_row<SEM, KEEP>(S, sl, lane);
                    MPROBE(probe_add(S, warp, lane, MP_FINAL, clock64() - t0);)
                }
                MPROBE(const long long t0 = clock64();)
                rw = setup_row<SEM>(S, sl, rl, lane);
                MPROBE(probe_add(S, warp, lane, MP_SETUP, clock64() - t0); probe_add(S, warp, lane, MP_ROWS, 1);)
            } else rw = row_window(S, rl, lane);
            scan_row<SEM, KEEP>(S, sl, rw, warp, lane, qn);
            if (++sl == (warp + 1) * MK_SLOTS) {       // the warp's slots hold its rows in turn; several passes: one row per slot
                if (S.npass > 1) break;
                sl = warp * MK_SLOTS;
            }
        }
        drain_queue<SEM, KEEP>(S, warp, lane, qn);     // the queue holds ring positions: empty it before the ring is refilled
        MPROBE(t_wait = clock64();)
        if (S.pass + 1 == S.npass) break;
        __syncthreads();                               // everybody is done with the resident entries: refill
        if (tid == 0) { ++S.pass; stage_entries(S, S.pass); }
        __syncthreads();                               // the new pass index is visible to every warp
    }
    MPROBE(const long long t_fin = clock64();)
    for (int i = 0; i < MK_SLOTS; ++i) {
        const int sl = warp * MK_SLOTS + i;
        if (S.slot_row[sl] >= 0) finalize_row<SEM, KEEP>(S, sl, lane);
    }
#ifdef L3D_MATCH_PROBE
    const long long t_done = clock64();
    probe_add(S, warp, lane, MP_FINAL, t_done - t_fin);
    __shared__ unsigned long long busy[MK_WARPS];
    if (lane == 0) busy[warp] = (unsigned long long)(t_done - t_start);
    __syncthreads();
    probe_add(S, warp, lane, MP_TAIL, clock64() - t_done);
    __syncthreads();
    if (tid == 0) {
        unsigned long long mx = 0ull, mn = ~0ull, sum = 0ull;
        for (int w = 0; w < MK_WARPS; ++w) { mx = max(mx, busy[w]); mn = min(mn, busy[w]); sum += busy[w]; }
        S.probe[0][MP_CTAS] += 1; S.probe[0][MP_BUSY_MAX] += mx; S.probe[0][MP_BUSY_MIN] += mn; S.probe[0][MP_BUSY_SUM] += sum;
    }
    __syncthreads();
    if (tid < MP_N) {
        unsigned long long v = 0ull;
        for (int w = 0; w < MK_WARPS; ++w) v += S.probe[w][tid];
        atomicAdd(&g_match_probe[tid], v);
    }
#endif
}

static_assert(L3D_SEM_REF_GPU == 0 && L3D_SEM_REF_CPU == 1 && (int)Keep::TopK == 0 && (int)Keep::Count == 1 && (int)Keep::Store == 2,
              "l3d_match_kernels is indexed [L3D_SEM_*][Keep]");
void (*const l3d_match_kernels[2][3])(MatchArgs) = {
    {k_match_topk<L3D_SEM_REF_GPU, Keep::TopK>, k_match_topk<L3D_SEM_REF_GPU, Keep::Count>, k_match_topk<L3D_SEM_REF_GPU, Keep::Store>},
    {k_match_topk<L3D_SEM_REF_CPU, Keep::TopK>, k_match_topk<L3D_SEM_REF_CPU, Keep::Count>, k_match_topk<L3D_SEM_REF_CPU, Keep::Store>},
};

// ------------------------------------------------------------------------------------------------ caller-given candidates
__global__ void __launch_bounds__(256) k_cand_keys(long long n, const int32_t* __restrict__ trip, const L3DPairDev* __restrict__ pairs,
                                                   const int* __restrict__ restricted, int first_pair, int last_pair,
                                                   unsigned long long* __restrict__ keys)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int p = trip[3 * i];
    const bool use = p >= first_pair && p < last_pair && restricted[p];
    keys[i] = use ? ((unsigned long long)(pairs[p].row_off + trip[3 * i + 1]) << 24) | (unsigned long long)trip[3 * i + 2] : L3D_CAND_NONE;
}

// first index in the sorted keys [0, n) whose key is not below k
__device__ __forceinline__ int cand_lower_bound(const unsigned long long* __restrict__ keys, int n, unsigned long long k)
{
    int lo = 0, hi = n;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (__ldg(keys + mid) < k) lo = mid + 1; else hi = mid; }
    return lo;
}

// One warp per source row of a restricted pair; lane i takes the row's candidates i, i + 32, ...  The decisions are k_match_topk's on
// the same values: the row's epipolar lines F*p from the float F (REF_GPU) or the double F (REF_CPU), exact_overlap / exact_overlap_f64
// on the target segment, the overlap above epi, then the depth test (depths_in_front where only the outcome is needed, the depths
// themselves where they are stored), keys make_key.  k_match_topk's pre-filters are conservative, so with every target as a candidate
// the matches are its own.  TopK keeps the row's k best keys in shared memory, sorted best first: every batch of 32 is ranked against
// them and the list by counting.  Count / Store keep every match; the candidates arrive in ascending target order, so Store writes
// the row in the order k_sort_rows leaves it.
template <int SEM, Keep KEEP>
__global__ void __launch_bounds__(32 * CAND_WARPS) k_match_cand(const CandArgs A)
{
    __shared__ unsigned long long best[CAND_WARPS][32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long g = (long long)blockIdx.x * CAND_WARPS + warp;
    if (g >= A.nrows) return;
    const int ip = last_le(A.nrp, g, [&](int i) { return A.rpairs[i].y; });
    const L3DPairDev* P = A.pairs + A.rpairs[ip].x;
    const int r = (int)(g - A.rpairs[ip].y);
    const L3DViewDev* vs = A.views + __ldg(&P->src);
    const L3DViewDev* vt = A.views + __ldg(&P->tgt);
    const long long R = __ldg(&P->row_off) + r, sidx = __ldg(&vs->seg_off) + r, toff = __ldg(&vt->seg_off);
    const int nk = *A.nkeys;
    const int b = cand_lower_bound(A.keys, nk, (unsigned long long)R << 24), e = cand_lower_bound(A.keys, nk, (unsigned long long)(R + 1) << 24);
    const float4 s = __ldg(A.segs + sidx);
    const float3 Cs = make_float3(vs->C[0], vs->C[1], vs->C[2]), Ct = make_float3(vt->C[0], vt->C[1], vt->C[2]);
    float3 e1, e2;
    SegRays sr;
    float snum = 0.0f;
    D3 e1d, e2d, Csd, Ctd;
    if (SEM == L3D_SEM_REF_CPU) {
        e1d = dmulmat(P->Fd, d3((double)s.x, (double)s.y, 1.0)); e2d = dmulmat(P->Fd, d3((double)s.z, (double)s.w, 1.0));
        Csd = d3(vs->C_d[0], vs->C_d[1], vs->C_d[2]); Ctd = d3(vt->C_d[0], vt->C_d[1], vt->C_d[2]);
    } else {
        e1 = mulmat_h(P->F, s.x, s.y); e2 = mulmat_h(P->F, s.z, s.w);
        sr = load_rays(A.cache, sidx);
        snum = depth_num(sr.n, Cs, Ct);
    }
    const int K = min(A.knn, 32);
    unsigned long long mine = 0ull;     // TopK: the lane-th best key so far (0: none)
    int cnt = 0;                        // TopK: keys in the list; Count / Store: matches so far
    for (int i0 = b; i0 < e; i0 += 32) {
        const int i = i0 + lane;
        const bool has = i < e;
        const unsigned int j = has ? (unsigned int)(__ldg(A.keys + i) & 0xFFFFFFull) : 0u;
        const float4 q = __ldg(A.segs + toff + j);
        float ov = 0.0f, d[4];
        bool pass;
        if (SEM == L3D_SEM_REF_CPU) {
            bool valid;
            ov = exact_overlap_f64(q, e1d, e2d, &valid);
            pass = has && valid && ov > A.epi;
            if (pass) {
                double dd[4];
                exact_depths_f64(load_rays_d(A.cache_d, sidx), load_rays_d(A.cache_d, toff + j), Csd, Ctd, dd);
                d[0] = (float)dd[0]; d[1] = (float)dd[1]; d[2] = (float)dd[2]; d[3] = (float)dd[3];
                pass = dd[0] > L3D_EPS_D && dd[1] > L3D_EPS_D && dd[2] > L3D_EPS_D && dd[3] > L3D_EPS_D;
            }
        } else {
            bool inv;
            ov = exact_overlap(q, e1, e2, &inv);
            pass = has && ov > A.epi;
            if (pass) {
                const SegRays t = load_rays(A.cache, toff + j);
                if (KEEP == Keep::Store) { exact_depths(sr, t, Cs, Ct, d); pass = d[0] > 0.0f && d[1] > 0.0f && d[2] > 0.0f && d[3] > 0.0f; }
                else pass = depths_in_front(sr, t, Cs, Ct, snum);
            }
        }
        const unsigned int bal = __ballot_sync(0xffffffffu, pass);
        if (KEEP != Keep::TopK) {
            if (KEEP == Keep::Store && pass) {
                const int slot = cnt + __popc(bal & ((1u << lane) - 1u));
                if (slot < A.knn) {
                    l3d_match_rec rec;
                    rec.tgt_seg = j; rec.overlap = ov; rec.d_p1 = d[0]; rec.d_p2 = d[1]; rec.d_q1 = d[2]; rec.d_q2 = d[3];
                    A.recs[R * A.knn + slot] = rec;
                }
            }
            cnt += __popc(bal);
            continue;
        }
        if (!bal) continue;
        // rank of every new key and of every listed key among both (keys are distinct and > 0; 0 marks no key)
        const unsigned long long key = pass ? make_key(ov, j) : 0ull;
        int rk = 0, rm = lane;
        for (int l = 0; l < 32; ++l) {
            const unsigned long long ok = __shfl_sync(0xffffffffu, mine, l), nk2 = __shfl_sync(0xffffffffu, key, l);
            rk += (ok > key) + (nk2 > key);
            rm += nk2 > mine;
        }
        __syncwarp();
        if (mine && rm < K) best[warp][rm] = mine;
        if (key && rk < K) best[warp][rk] = key;
        cnt = min(cnt + __popc(bal), K);
        __syncwarp();
        mine = lane < cnt ? best[warp][lane] : 0ull;
    }
    if (lane == 0) A.counts[R] = cnt;
    if (KEEP != Keep::TopK || lane >= cnt) return;
    const unsigned int j = key_tgt(mine);
    float d[4];
    if (SEM == L3D_SEM_REF_CPU) {
        double dd[4];
        exact_depths_f64(load_rays_d(A.cache_d, sidx), load_rays_d(A.cache_d, toff + j), Csd, Ctd, dd);
        d[0] = (float)dd[0]; d[1] = (float)dd[1]; d[2] = (float)dd[2]; d[3] = (float)dd[3];
    } else exact_depths(sr, load_rays(A.cache, toff + j), Cs, Ct, d);
    l3d_match_rec rec;
    rec.tgt_seg = j; rec.overlap = key_overlap(mine); rec.d_p1 = d[0]; rec.d_p2 = d[1]; rec.d_q1 = d[2]; rec.d_q2 = d[3];
    A.recs[R * A.knn + lane] = rec;
}

void (*const l3d_cand_kernels[2][3])(CandArgs) = {
    {k_match_cand<L3D_SEM_REF_GPU, Keep::TopK>, k_match_cand<L3D_SEM_REF_GPU, Keep::Count>, k_match_cand<L3D_SEM_REF_GPU, Keep::Store>},
    {k_match_cand<L3D_SEM_REF_CPU, Keep::TopK>, k_match_cand<L3D_SEM_REF_CPU, Keep::Count>, k_match_cand<L3D_SEM_REF_CPU, Keep::Store>},
};

// keep-all rows arrive in queue order; the reference appends them in ascending target order.  One warp per row, the row
// staged in shared memory (stride * 24 B per warp), rank = number of smaller target indices (unique per row).
// topk > 0 (kNN beyond the fused kernel's 32 keys per row): the rows keep their `topk` best matches instead, in the order the
// reference pops its priority queue (descending overlap, cudawrapper.cu:637-645; equal overlaps by target index), counts clipped.
__global__ void __launch_bounds__(128) k_sort_rows(int* __restrict__ counts, l3d_match_rec* __restrict__ recs, int stride, long long rows, int topk)
{
    extern __shared__ __align__(16) unsigned char sort_smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
    l3d_match_rec* buf = reinterpret_cast<l3d_match_rec*>(sort_smem) + (size_t)warp * stride;
    for (long long row = (long long)blockIdx.x * wpb + warp; row < rows; row += (long long)gridDim.x * wpb) {
        const int n = min(counts[row], stride);
        if (n > 1) {
            l3d_match_rec* g = recs + row * stride;
            for (int i = lane; i < n; i += 32) buf[i] = g[i];
            __syncwarp();
            for (int i = lane; i < n; i += 32) {
                const unsigned int t = buf[i].tgt_seg;
                const float ov = buf[i].overlap;
                int r = 0;
                if (topk > 0) { for (int j = 0; j < n; ++j) r += (buf[j].overlap > ov || (buf[j].overlap == ov && buf[j].tgt_seg < t)) ? 1 : 0; if (r < topk) g[r] = buf[i]; }
                else { for (int j = 0; j < n; ++j) r += buf[j].tgt_seg < t; g[r] = buf[i]; }
            }
        }
        if (topk > 0 && lane == 0 && n > topk) counts[row] = topk;
        __syncwarp();
    }
}

// ------------------------------------------------------------------------------------------------ dense contract
// K_match_lines' device contract: depths[Ns][Nt] (float4) + overlaps[Ns][Nt] (float) for EVERY cell, 20 B written per
// pair evaluation -> HBM-write bound.  A warp owns DK_T*32 consecutive target columns and walks DK_ROWS source rows:
// cells the filter proves empty are stored at once, coalesced ((-1,-1,-1,-1), 0); the others are ballot-compacted into
// a per-warp queue and evaluated 32 at a time by the exact path, which stores its 20 bytes itself.
struct DenseSmem {
    float4 rowA[DK_ROWS], rowB[DK_ROWS];
    float4 sray[DK_ROWS][3];                       // cached rays / plane normal of the CTA's source rows
    float4 tq[DK_WARPS][32 * DK_T];                // target segments of each warp's columns
    unsigned int queue[DK_WARPS][64];
    float4* depths; float* overlaps;
    const float4* tcache;                          // cached rays / plane normals of the target view: only the ~1 % of cells whose
                                                   // overlap exceeds the threshold read them (L2), not worth 48 KB of shared memory
    float3 Cs, Ct;
    float epi; int Nt, row0;
};
size_t l3d_dense_smem_bytes() { return sizeof(DenseSmem); }
// Rows per CTA (8..DK_ROWS) such that the tile count fills whole waves of the 4 resident CTAs per SM: a 3000 x 3000 pair
// with a fixed 16 rows gives 564 CTAs = 1.07 waves on 132 SMs, i.e. a second wave that is 93 % idle.
int l3d_dense_rows_per_cta(int Ns, int Nt, int num_sms)
{
    const long long slots = (long long)DK_MINB * (num_sms > 0 ? num_sms : 132);
    const long long colb = (Nt + DK_WARPS * DK_T * 32 - 1) / (DK_WARPS * DK_T * 32);
    int best = 16; double best_eff = -1.0;
    for (int R = 8; R <= DK_ROWS; ++R) {
        const long long tiles = colb * ((Ns + R - 1) / R);
        const long long waves = (tiles + slots - 1) / slots;
        const double eff = (double)tiles / (double)(waves * slots);
        if (eff > best_eff + 1e-9 || (eff > best_eff - 1e-9 && R > best)) { best_eff = eff; best = R; }
    }
    return best;
}

__device__ __noinline__ void dense_exact_batch(DenseSmem& S, unsigned int entry, bool has, int warp, int x0)
{
    if (!has) return;
    const int r = (int)(entry >> 24), x = (int)(entry & 0xFFFFFFu), col = x - x0;
    const float4 q = S.tq[warp][col];
    const float4 rA = S.rowA[r], rB = S.rowB[r];
    float4 res = make_float4(-1.f, -1.f, -1.f, -1.f);
    bool inv;
    const float ov = exact_overlap(q, make_float3(rA.x, rA.y, rA.z), make_float3(rA.w, rB.x, rB.y), &inv);
    if (ov > S.epi) {
        const SegRays s = rays_from_smem(S.sray[r]), t = load_rays(S.tcache, x);
        float d[4];
        exact_depths(s, t, S.Cs, S.Ct, d);
        res = make_float4(d[0], d[1], d[2], d[3]);
    }
    const size_t o = (size_t)(S.row0 + r) * S.Nt + x;
    __stcs(S.depths + o, res);
    __stcs(S.overlaps + o, ov);
}

// one tile (rows_per_cta source rows x DK_WARPS * DK_T * 32 target columns) of one view pair; (bx, by) = the tile's column / row block
__device__ __forceinline__ void dense_tile(const float4* __restrict__ ssegs, int Ns, const float4* __restrict__ tsegs, int Nt,
                                           const float4* __restrict__ scache, const float4* __restrict__ tcache, const L3DMat3& F, float3 Cs, float3 Ct,
                                           float epi, float4* __restrict__ depths, float* __restrict__ overlaps, int rows_per_cta, int bx, int by)
{
    extern __shared__ __align__(128) unsigned char dense_smem_raw[];
    DenseSmem& S = *reinterpret_cast<DenseSmem*>(dense_smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int row0 = by * rows_per_cta;
    const int nrows = min(rows_per_cta, Ns - row0);
    if (tid == 0) { S.depths = depths; S.overlaps = overlaps; S.tcache = tcache; S.Cs = Cs; S.Ct = Ct; S.epi = epi; S.Nt = Nt; S.row0 = row0; }
    if (tid < nrows) {
        float4 s = __ldg(ssegs + row0 + tid);
        float3 e1 = mulmat_h(F.m, s.x, s.y), e2 = mulmat_h(F.m, s.z, s.w);
        float g = L3D_FILTER_C1 * fmaxf(sqrtf(e1.x * e1.x + e1.y * e1.y), sqrtf(e2.x * e2.x + e2.y * e2.y));
        S.rowA[tid] = make_float4(e1.x, e1.y, e1.z, e2.x);
        S.rowB[tid] = make_float4(e2.y, e2.z, g, 0.f);      // threshold 0: reject only provably empty cells
    }
    if (tid < 3 * nrows) S.sray[tid / 3][tid % 3] = __ldg(scache + 3 * (size_t)row0 + tid);
    const int x0 = (bx * DK_WARPS + warp) * (32 * DK_T);
    float4 q[DK_T];
    bool ok[DK_T];
#pragma unroll
    for (int t = 0; t < DK_T; ++t) {
        const int x = x0 + t * 32 + lane;
        ok[t] = x < Nt;
        q[t] = __ldg(tsegs + (ok[t] ? x : 0));
        S.tq[warp][t * 32 + lane] = q[t];
    }
    __syncthreads();
    if (x0 >= Nt) return;
    const unsigned int lt_mask = (1u << lane) - 1u;
    const float4 none = make_float4(-1.f, -1.f, -1.f, -1.f);
    int qn = 0;
    for (int r = 0; r < nrows; ++r) {
        const float4 rA = S.rowA[r], rB = S.rowB[r];
        const size_t orow = (size_t)(row0 + r) * Nt;
        bool pass[DK_T];
#pragma unroll
        for (int t = 0; t < DK_T; ++t) pass[t] = ok[t] && filter_may_survive(q[t], rA, rB);
#pragma unroll
        for (int t = 0; t < DK_T; ++t) {
            const int x = x0 + t * 32 + lane;
            if (ok[t] && !pass[t]) { __stcs(depths + orow + x, none); __stcs(overlaps + orow + x, 0.0f); }
            const unsigned int b = __ballot_sync(0xffffffffu, pass[t]);
            if (b) {
                if (pass[t]) S.queue[warp][qn + __popc(b & lt_mask)] = ((unsigned int)r << 24) | (unsigned int)x;
                qn += __popc(b);
                __syncwarp();
                if (qn >= 32) { qn -= 32; dense_exact_batch(S, S.queue[warp][qn + lane], true, warp, x0); }
            }
        }
    }
    if (qn > 0) dense_exact_batch(S, lane < qn ? S.queue[warp][lane] : 0u, lane < qn, warp, x0);
}

// one view pair: a 2-D grid of (column block, row block) tiles
__global__ void __launch_bounds__(DK_THREADS, DK_MINB) k_match_dense(const L3DDenseJob J, float epi)
{ dense_tile(J.ssegs, J.Ns, J.tsegs, J.Nt, J.scache, J.tcache, J.F, J.Cs, J.Ct, epi, J.depths, J.overlaps, J.rows_per_cta, blockIdx.x, blockIdx.y); }

// The same contract for MANY view pairs in one launch (l3d_match_dense_pairs): a 1-D grid over the tiles of all jobs, so the tail of
// one pair's tiles overlaps the head of the next pair's instead of leaving SMs idle at the end of every 88 us launch.
__global__ void __launch_bounds__(DK_THREADS, DK_MINB)
k_match_dense_batch(const L3DDenseJob* __restrict__ jobs, int njobs, float epi)
{
    __shared__ int job_s;
    if (threadIdx.x == 0) job_s = last_le(njobs, (long long)blockIdx.x, [&](int i) { return jobs[i].tile0; });
    __syncthreads();
    const L3DDenseJob& J = jobs[job_s];
    const int t = (int)((long long)blockIdx.x - J.tile0);
    dense_tile(J.ssegs, J.Ns, J.tsegs, J.Nt, J.scache, J.tcache, J.F, J.Cs, J.Ct, epi, J.depths, J.overlaps, J.rows_per_cta, t % J.colb, t / J.colb);
}

// same contract, NO pre-filter: every cell goes through the exact path.  Test-only cross-check of the filter.
__global__ void __launch_bounds__(DK_THREADS) k_match_dense_nofilter(const L3DDenseJob J, float epi)
{
    const float4 *ssegs = J.ssegs, *tsegs = J.tsegs, *scache = J.scache, *tcache = J.tcache;
    const int Ns = J.Ns, Nt = J.Nt; const L3DMat3& F = J.F; const float3 Cs = J.Cs, Ct = J.Ct;
    const int x = blockIdx.x * DK_THREADS + threadIdx.x;
    const int row0 = blockIdx.y * DKN_ROWS;
    const int nrows = min(DKN_ROWS, Ns - row0);
    if (x >= Nt) return;
    const float4 q = __ldg(tsegs + x);
    for (int r = 0; r < nrows; ++r) {
        float4 s4 = __ldg(ssegs + row0 + r);
        float3 e1 = mulmat_h(F.m, s4.x, s4.y), e2 = mulmat_h(F.m, s4.z, s4.w);
        float4 res = make_float4(-1.f, -1.f, -1.f, -1.f);
        bool inv;
        float ov = exact_overlap(q, e1, e2, &inv);
        if (ov > epi) {
            SegRays s = load_rays(scache, row0 + r), t = load_rays(tcache, x);
            float d[4];
            exact_depths(s, t, Cs, Ct, d);
            res = make_float4(d[0], d[1], d[2], d[3]);
        }
        const size_t o = (size_t)(row0 + r) * Nt + x;
        J.depths[o] = res;
        J.overlaps[o] = ov;
    }
}

// ------------------------------------------------------------------------------------------------ CSR compaction
__global__ void __launch_bounds__(256) k_compact_matches(const int* __restrict__ counts, const long long* __restrict__ row_ptr,
                                                         const l3d_match_rec* __restrict__ recs, int knn, long long rows,
                                                         l3d_match_rec* __restrict__ out)
{
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // one thread per (row, slot)
    long long row = i / knn;
    int slot = (int)(i - row * knn);
    if (row >= rows) return;
    if (slot < counts[row]) out[row_ptr[row] + slot] = recs[row * knn + slot];
}

// ------------------------------------------------------------------------------------------------ FP32 peak probe
// 16 independent FFMA chains per thread, no memory traffic: the non-tensor FP32 roofline denominator, measured in the
// same process and clocks as the bench (MEASURED_PEAKS.json only carries HBM and bf16-tensor peaks).
__global__ void __launch_bounds__(256) k_fp32_peak(float* __restrict__ out, int iters, float a, float b)
{
    float x[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) x[i] = (float)(threadIdx.x + i);
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < 16; ++i) x[i] = __fmaf_rn(x[i], a, b);
    }
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i) s += x[i];
    if (s == 123.456f) out[0] = s;   // never true; keeps the chains alive
}
