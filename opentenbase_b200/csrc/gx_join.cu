// gx_join.cu — K2 open-addressing hash build and K3 probe (materialising).
//
// Table: power-of-two array of 16-byte slots {int64 key, uint64 payload},
// linear probing, load factor in (0.33, 0.67].  Empty = key INT64_MIN; rows
// whose key IS INT64_MIN live in a small side list.  The payload holds up to
// eight bytes of carried build-side columns (or the build row number), so a
// probe hit costs one 32-byte sector and no second gather.
//
// Replaces MultiExecPrivateHash / ExecHashTableInsert (nodeHash.c:157,1828:
// chained buckets of MinimalTuple copies in 32 KB chunks) and
// ExecScanHashBucket / ExecHashJoinImpl (nodeHash.c:2174, nodeHashjoin.c:186).
#include "gx_internal.cuh"
#include <type_traits>

int gx_fill_dpreds(gx_ctx *ctx, const gx_table *t, int n_preds, const gx_pred *preds, gx_dpred *out);

struct gx_build_args {
    gx_dcol key;
    int npreds, n_payload;
    gx_dpred preds[GX_MAX_PREDS];
    gx_dcol payload[GX_MAX_PAYLOAD];
    long long nrows;
    gx_slot *slots; unsigned long long mask;
    unsigned long long *special; int special_cap;
    gx_slotfn sf;                 // gx_slot_index
    long long *counters;          // ctx->d_scratch: the SW_* words
    // direct build only: rows claimed per sub-table, how many one sub-table may hold, and the largest
    // claim count seen past that limit (0 = none)
    unsigned int *sub_claims; unsigned int sub_limit; unsigned int *sub_over;
};
// Words of ctx->d_scratch / h_scratch the build uses (word 2 is gx_hash_probe_ex's output cursor).  The sample's key range
// shares word 5 with the chain steps, which are counted only after it is read.  OVF_*: bits of the key-ordered fill's
// overflow word; OVF_FULL also flags the bucketing's overflow.
enum {
    SW_INSERTED = 0, SW_SPECIAL = 1,    // entries the direct build inserted; side-list rows
    SW_PLACED = 3, SW_STEPS = 5,        // entries the fills placed; their chain steps
    SW_KRANGE = 4, SW_PRANGE = 16,      // the sample's key, payload min and max
    SW_UNSORTED = 6, SW_OVERFLOW = 7,   // key-ordered build: rows out of key order; OVF_* bits (both int)
    SW_ENDS = 20,                       // the key column's first and last key
    SW_ORDER = 18,                      // the sample's order bits (gx_k_key_range, int)
    OVF_FULL = 1, OVF_STUCK = 2, OVF_PAYLOAD = 4   // a sub-table is full; a staged wait gave up; a payload outside the narrow window
};

__device__ __forceinline__ unsigned long long pack_payload(const gx_build_args &a, long long r)
{
    if (a.n_payload == 0) return (unsigned long long) r;
    unsigned long long p = 0; int shift = 0;
#pragma unroll
    for (int i = 0; i < GX_MAX_PAYLOAD; i++) {
        if (i >= a.n_payload) break;
        int t = a.payload[i].type;
        unsigned long long v = (unsigned long long) gx_load_int(a.payload[i], r);
        int bytes = (t == GX_INT8 || t == GX_FLOAT8) ? 8 : (t == GX_CHAR ? 1 : 4);
        if (bytes < 8) v &= (1ULL << (8 * bytes)) - 1;
        p |= v << shift;
        shift += 8 * bytes;
    }
    return p;
}

__global__ void __launch_bounds__(256) gx_k_hash_build(gx_build_args a)
{
    long long stride = (long long) gridDim.x * blockDim.x;
    long long inserted = 0;
    for (long long r = (long long) blockIdx.x * blockDim.x + threadIdx.x; r < a.nrows; r += stride) {
        bool ok = !gx_is_null(a.key, r);               // hashStrict: NULL keys never match
#pragma unroll
        for (int p = 0; p < GX_MAX_PREDS; p++) if (p < a.npreds) ok = ok && gx_eval_pred(a.preds[p], r);
        if (!ok) continue;
        long long key = gx_load_int(a.key, r);
        unsigned long long payload = pack_payload(a, r);
        if (key == GX_EMPTY_KEY) {
            int idx = (int) atomicAdd((unsigned long long *) &a.counters[SW_SPECIAL], 1ULL);
            if (idx < a.special_cap) a.special[idx] = payload;
            continue;
        }
        unsigned long long s = gx_slot_index(key, a.sf);
        // a sub-table must keep a free slot, or probe walks that miss in it never end: rows past the limit
        // are not inserted and fail the build.  So the CAS walk below always meets an empty slot.
        const unsigned int claim = atomicAdd(&a.sub_claims[s >> GX_SUB_LOG2], 1u);
        if (claim >= a.sub_limit) { atomicMax(a.sub_over, claim + 1); continue; }
        bool placed = false;
        for (int step = 0; step < GX_SUB; step++) {
            long long old = (long long) atomicCAS((unsigned long long *) &a.slots[s].key,
                                                  (unsigned long long) GX_EMPTY_KEY, (unsigned long long) key);
            if (old == GX_EMPTY_KEY) { a.slots[s].payload = payload; placed = true; break; }
            s = gx_next_slot(s, a.mask);
        }
        if (!placed) { atomicMax(a.sub_over, claim + 1); continue; }
        inserted++;
    }
    // one atomic per warp
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) inserted += __shfl_down_sync(0xffffffffu, inserted, o);
    if ((threadIdx.x & 31) == 0 && inserted) atomicAdd((unsigned long long *) &a.counters[SW_INSERTED], (unsigned long long) inserted);
}

__global__ void gx_k_fill_slots(gx_slot *slots, long long n)
{
    long long stride = (long long) gridDim.x * blockDim.x;
    // 16-byte stores
    for (long long i = (long long) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        longlong2 v; v.x = GX_EMPTY_KEY; v.y = 0;
        ((longlong2 *) slots)[i] = v;
    }
}


// ---------------------------------------------------------------------------
// Bucketed build.  Random CAS into a table much larger than L2 is bound by
// DRAM latency: every
// insert is a DRAM read-modify-write of a sector that was just cleared.  So the
// table is cut into sub-tables of GX_SUB slots (32 KB); linear probing wraps
// INSIDE a sub-table (all probe kernels use gx_next_slot()).  Build rows are
// bucketed by sub-table (sequential read, 16-byte scattered stores that
// write-combine in L2), then one CTA builds one sub-table entirely in shared
// memory and streams it out with coalesced 16-byte stores: the table is written
// exactly once, never read, never cleared, and sees no global atomics.
struct gx_bbuild_args {
    gx_build_args b;
    long long nsub;
    unsigned int *cursor;       // [nsub] rows scattered to each sub-table so far
    gx_slot *pairs;             // nsub fixed-capacity buckets of GX_SUB pairs (a fuller bucket cannot be built anyway)
    int *overflow;
    long long *start; int *unsorted;   // key-ordered build: first row of every sub-table
    gx_cslot *cslots;                  // compact output (gx_k_sorted_fill<GX_SLOTS_COMPACT, ..>)
    unsigned int *narrow;              // narrow output (gx_k_sorted_fill<GX_SLOTS_NARROW, ..>)
};

__device__ __forceinline__ bool build_row_ok(const gx_build_args &a, long long r)
{
    bool ok = !gx_is_null(a.key, r);
#pragma unroll
    for (int p = 0; p < GX_MAX_PREDS; p++) if (p < a.npreds) ok = ok && gx_eval_pred(a.preds[p], r);
    return ok;
}

// Scatter (key, payload) pairs into their sub-table's bucket.  The position
// comes from one L2 atomic; the chain load -> atomic -> store is latency bound,
// so every thread keeps BSCAT rows in flight.
#define BSCAT 4
__global__ void __launch_bounds__(256) gx_k_bbuild_scatter(gx_bbuild_args a)
{
    const long long tile = (long long) blockDim.x * BSCAT;
    const long long ntiles = (a.b.nrows + tile - 1) / tile;
    for (long long t = blockIdx.x; t < ntiles; t += gridDim.x) {
        long long key[BSCAT]; unsigned long long payload[BSCAT], sub[BSCAT]; unsigned int pos[BSCAT]; bool ok[BSCAT];
#pragma unroll
        for (int u = 0; u < BSCAT; u++) {
            long long r = t * tile + (long long) u * blockDim.x + threadIdx.x;     // coalesced per u
            ok[u] = r < a.b.nrows && build_row_ok(a.b, r);
            key[u] = ok[u] ? gx_load_int(a.b.key, r) : 0;
            payload[u] = ok[u] ? pack_payload(a.b, r) : 0;
        }
#pragma unroll
        for (int u = 0; u < BSCAT; u++) {
            if (ok[u] && key[u] == GX_EMPTY_KEY) {
                int idx = (int) atomicAdd((unsigned long long *) &a.b.counters[SW_SPECIAL], 1ULL);
                if (idx < a.b.special_cap) a.b.special[idx] = payload[u];
                ok[u] = false;
            }
            sub[u] = gx_slot_index(key[u], a.b.sf) >> GX_SUB_LOG2;
            if (ok[u]) pos[u] = atomicAdd(&a.cursor[sub[u]], 1u);
        }
#pragma unroll
        for (int u = 0; u < BSCAT; u++) {
            if (!ok[u]) continue;
            if (pos[u] >= GX_SUB - 1) { *a.overflow = OVF_FULL; continue; }      // a sub-table keeps one slot free
            longlong2 v; v.x = key[u]; v.y = (long long) payload[u];
            ((longlong2 *) a.pairs)[sub[u] * GX_SUB + pos[u]] = v;
        }
    }
}
// ---------------------------------------------------------------------------
// Two-level write-combined bucketing (replaces the one-pass scatter above for
// big tables), which spends its time in per-row L2 atomics and 16-byte
// scattered stores.  Here a CTA takes a
// tile of 4096 rows, ranks them by bucket digit in shared memory (native 32-bit
// shared atomics), stages them bucket by bucket and copies each bucket's run out
// as one contiguous piece: one global atomic per (tile, bucket) instead of one
// per row, and 256-byte runs instead of 16-byte stores.  Level 1 splits on the
// high bits of the sub-table number, level 2 on the low bits.
#define BP_TILE 4096
#define BP_THREADS 512
#define BP_PER (BP_TILE / BP_THREADS)
struct gx_bpart_args {
    gx_build_args b;
    int bits_hi, bits_lo;
    long long nsub;
    gx_slot *l1; long long cap1; unsigned int *cur1;      // level-1 regions
    gx_slot *pairs; unsigned int *cursor; int *overflow;  // final buckets
    long long tiles_per_l1;
};

struct bp_smem {
    longlong2 *stage; unsigned short *bid; unsigned int *hist, *base, *gbase;
};
__device__ __forceinline__ bp_smem bp_carve(unsigned char *raw, int nb)
{
    bp_smem m;
    m.stage = (longlong2 *) raw;
    m.hist = (unsigned int *) (raw + (size_t) BP_TILE * 16);
    m.base = m.hist + nb; m.gbase = m.base + nb;
    m.bid = (unsigned short *) (m.gbase + nb);
    return m;
}
static size_t bp_smem_bytes(int nb) { return (size_t) BP_TILE * 16 + (size_t) nb * 12 + (size_t) BP_TILE * 2 + 64; }

// rank + stage one tile; returns after the staging buffer is complete
__device__ __forceinline__ void bp_stage_tile(const bp_smem &m, int nb, const long long *key, const unsigned long long *payload,
                                              const bool *ok, const unsigned int *digit, long long *scan_smem)
{
    unsigned int rank[BP_PER];
    for (int i = threadIdx.x; i < nb; i += blockDim.x) m.hist[i] = 0;
    __syncthreads();
    // Sorted build input (serial keys + order-preserving slots) sends a whole warp to the same
    // bucket: aggregate per warp first so the shared atomic is issued once per distinct bucket.
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int u = 0; u < BP_PER; u++) {
        unsigned int am = __ballot_sync(0xffffffffu, ok[u]);
        if (!ok[u]) continue;
        unsigned int peers = __match_any_sync(am, digit[u]);
        int leader = __ffs(peers) - 1;
        unsigned int base = 0;
        if (lane == leader) base = atomicAdd(&m.hist[digit[u]], (unsigned int) __popc(peers));
        rank[u] = __shfl_sync(peers, base, leader) + __popc(peers & ((1u << lane) - 1));
    }
    __syncthreads();
    {   // exclusive scan of the histogram (nb <= blockDim.x)
        long long tot;
        long long h = (int) threadIdx.x < nb ? (long long) m.hist[threadIdx.x] : 0;
        long long ex = gx_block_exscan(h, &tot, scan_smem);
        if ((int) threadIdx.x < nb) m.base[threadIdx.x] = (unsigned int) ex;
    }
    __syncthreads();
#pragma unroll
    for (int u = 0; u < BP_PER; u++) {
        if (!ok[u]) continue;
        unsigned int p = m.base[digit[u]] + rank[u];
        longlong2 v; v.x = key[u]; v.y = (long long) payload[u];
        m.stage[p] = v; m.bid[p] = (unsigned short) digit[u];
    }
}

__global__ void __launch_bounds__(BP_THREADS, 2) gx_k_bpart1(gx_bpart_args a)
{
    extern __shared__ unsigned char bp_raw[];
    __shared__ long long scan_smem[33];
    const int nb = 1 << a.bits_hi;
    bp_smem m = bp_carve(bp_raw, nb);
    const long long ntiles = (a.b.nrows + BP_TILE - 1) / BP_TILE;
    for (long long t = blockIdx.x; t < ntiles; t += gridDim.x) {
        long long key[BP_PER]; unsigned long long payload[BP_PER]; bool ok[BP_PER]; unsigned int digit[BP_PER];
#pragma unroll
        for (int u = 0; u < BP_PER; u++) {
            long long r = t * BP_TILE + (long long) u * BP_THREADS + threadIdx.x;
            ok[u] = r < a.b.nrows && build_row_ok(a.b, r);
            key[u] = ok[u] ? gx_load_int(a.b.key, r) : 0;
            payload[u] = ok[u] ? pack_payload(a.b, r) : 0;
            if (ok[u] && key[u] == GX_EMPTY_KEY) {
                int idx = (int) atomicAdd((unsigned long long *) &a.b.counters[SW_SPECIAL], 1ULL);
                if (idx < a.b.special_cap) a.b.special[idx] = payload[u];
                ok[u] = false;
            }
            digit[u] = (unsigned int) ((gx_slot_index(key[u], a.b.sf) >> GX_SUB_LOG2) >> a.bits_lo);
        }
        bp_stage_tile(m, nb, key, payload, ok, digit, scan_smem);
        if ((int) threadIdx.x < nb) m.gbase[threadIdx.x] = m.hist[threadIdx.x] ? atomicAdd(&a.cur1[threadIdx.x], m.hist[threadIdx.x]) : 0;
        __syncthreads();
        const unsigned int total = m.base[nb - 1] + m.hist[nb - 1];
        for (unsigned int j = threadIdx.x; j < total; j += blockDim.x) {
            unsigned int d = m.bid[j];
            long long pos = (long long) m.gbase[d] + (j - m.base[d]);
            if (pos >= a.cap1) { *a.overflow = OVF_FULL; continue; }
            ((longlong2 *) a.l1)[(long long) d * a.cap1 + pos] = m.stage[j];
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(BP_THREADS, 2) gx_k_bpart2(gx_bpart_args a)
{
    extern __shared__ unsigned char bp_raw[];
    __shared__ long long scan_smem[33];
    const int nb = 1 << a.bits_lo;
    bp_smem m = bp_carve(bp_raw, nb);
    const long long nwork = ((long long) 1 << a.bits_hi) * a.tiles_per_l1;
    for (long long w = blockIdx.x; w < nwork; w += gridDim.x) {
        const long long b1 = w / a.tiles_per_l1, t = w % a.tiles_per_l1;
        long long n1 = a.cur1[b1]; if (n1 > a.cap1) n1 = a.cap1;
        if (t * BP_TILE >= n1) continue;                       // uniform per CTA
        const longlong2 *src = (const longlong2 *) a.l1 + b1 * a.cap1;
        long long key[BP_PER]; unsigned long long payload[BP_PER]; bool ok[BP_PER]; unsigned int digit[BP_PER];
#pragma unroll
        for (int u = 0; u < BP_PER; u++) {
            long long i = t * BP_TILE + (long long) u * BP_THREADS + threadIdx.x;
            ok[u] = i < n1;
            longlong2 v; v.x = 0; v.y = 0;
            if (ok[u]) v = src[i];
            key[u] = v.x; payload[u] = (unsigned long long) v.y;
            digit[u] = (unsigned int) ((gx_slot_index(key[u], a.b.sf) >> GX_SUB_LOG2) & (unsigned long long) (nb - 1));
        }
        bp_stage_tile(m, nb, key, payload, ok, digit, scan_smem);
        if ((int) threadIdx.x < nb)
            m.gbase[threadIdx.x] = m.hist[threadIdx.x] ? atomicAdd(&a.cursor[(b1 << a.bits_lo) | threadIdx.x], m.hist[threadIdx.x]) : 0;
        __syncthreads();
        const unsigned int total = m.base[nb - 1] + m.hist[nb - 1];
        for (unsigned int j = threadIdx.x; j < total; j += blockDim.x) {
            unsigned int d = m.bid[j];
            unsigned int pos = m.gbase[d] + (j - m.base[d]);
            if (pos >= GX_SUB - 1) { *a.overflow = OVF_FULL; continue; }       // a sub-table keeps one slot free
            ((longlong2 *) a.pairs)[(((long long) b1 << a.bits_lo) | d) * GX_SUB + pos] = m.stage[j];
        }
        __syncthreads();
    }
}

// ---------------------------------------------------------------------------
// Building one sub-table (GX_SUB slots) in shared memory WITHOUT a compare-and-swap loop.
// A linear-probing table filled in slot order has a closed form: with c[s] rows hashing to
// slot s, the first of them lands at s + e[s], where e[s] = max(0, e[s-1] + c[s-1] - 1) is
// the overflow carried in from the left.  With P[s] = sum_{t<s} (c[t] - 1) this is
// e[s] = P[s] - min_{j<=s} P[j]: one histogram (native 32-bit shared atomics, which also
// hand every row its rank among the rows of its slot), one block-wide scan of the pair
// (sum, prefix-minimum), one conflict-free placement pass.  Rows pushed past the end of
// the sub-table wrap to its start; they are rare and go through a CAS loop afterwards.
// Any prober that walks from slot(key) to the right (gx_next_slot) finds every key before
// it meets an empty slot, exactly as with CAS insertion.
// The caller's LOAD hands over row i: from the bucket pairs (gx_k_bbuild_fill), straight from the
// columns (gx_k_sorted_fill), or from the shared-memory stage the copy engine filled while the
// previous sub-table was built (gx_k_sorted_fill_staged, which puts its two stages behind this struct).
// The finished sub-table leaves with plain 16-byte stores; the trailing barrier frees the table, the
// histogram and the caller's rows for the next sub-table.
#define FILL_THREADS 256
#define FILL_ROWS (GX_SUB / FILL_THREADS)          // rows (and slots) per thread
template <int F> struct gx_slot_of { typedef gx_slot type; };
template <> struct gx_slot_of<GX_SLOTS_COMPACT> { typedef gx_cslot type; };
template <> struct gx_slot_of<GX_SLOTS_NARROW> { typedef unsigned int type; };
template <int F> struct gx_fill_smem_t {
    typename gx_slot_of<F>::type tab[GX_SUB];
    unsigned int cnt[GX_SUB];                      // histogram, then e[s]
    int wsum[FILL_THREADS / 32], wmin[FILL_THREADS / 32];
};
typedef gx_fill_smem_t<GX_SLOTS_WIDE> gx_fill_smem;
#define FILL_SMEM_BYTES ((int) sizeof(gx_fill_smem))
#define FILL_INF (1 << 29)

// F = the slot format GX_SLOTS_*; dst points at that slot type.  A narrow row whose payload does not fit the slot's
// payload bits raises pay_miss (and is placed with a truncated payload: the host rebuilds in the 8-byte form).
template <int F, class LOAD>
__device__ __forceinline__ void gx_subtable_build(gx_fill_smem_t<F> &sm, unsigned int n, const gx_slotfn &sf, LOAD load, void *dst,
                                                  unsigned int &steps, unsigned int &placed, int &pay_miss,
                                                  long long want_sub = -1, int *misplaced = nullptr)
{
    constexpr bool C = F != GX_SLOTS_WIDE;                     // 32-bit key words (compact and narrow)
    constexpr int SB = (int) sizeof(typename gx_slot_of<F>::type);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // ---- clear: histogram and table
    {
        uint4 z = make_uint4(0, 0, 0, 0);
        uint4 *c4 = (uint4 *) sm.cnt;
        for (int i = tid; i < GX_SUB / 4; i += FILL_THREADS) c4[i] = z;
        if (C) {
            uint4 *t4 = (uint4 *) sm.tab;
#pragma unroll
            for (int u = 0; u < FILL_ROWS * SB / 16; u++) t4[tid + u * FILL_THREADS] = z;
        } else {
            longlong2 e; e.x = GX_EMPTY_KEY; e.y = 0;
            longlong2 *t2 = (longlong2 *) sm.tab;
#pragma unroll
            for (int u = 0; u < FILL_ROWS; u++) t2[tid + u * FILL_THREADS] = e;
        }
    }
    __syncthreads();
    // ---- histogram + rank
    // what is kept per row until placement: the slot's two words (compact: two 32-bit values)
    typename std::conditional<C, unsigned int, long long>::type key[FILL_ROWS];
    typename std::conditional<C, unsigned int, unsigned long long>::type pay[FILL_ROWS];
    unsigned int sr[FILL_ROWS];
#pragma unroll
    for (int u = 0; u < FILL_ROWS; u++) {
        unsigned int i = tid + u * FILL_THREADS;
        sr[u] = 0xffffffffu;
        long long k64; unsigned long long p64;
        if (i < n && load(i, k64, p64)) {
            const unsigned long long fs = gx_slot_index(k64, sf);
            if (want_sub >= 0 && (long long) (fs >> GX_SUB_LOG2) != want_sub) *misplaced = 1;   // caller's row range was wrong
            unsigned int sl = (unsigned int) (fs & (GX_SUB - 1));
            sr[u] = sl | (atomicAdd(&sm.cnt[sl], 1u) << GX_SUB_LOG2);
            if (F == GX_SLOTS_NARROW) {
                const long long pv = (long long) (int) (unsigned int) p64;       // the 4-byte payload column is signed
                if (!gx_nslot_fits(pv, sf)) pay_miss = 1;
                key[u] = gx_nslot_make(k64, pv, sf); pay[u] = 0;
            } else if (C) { key[u] = GX_CSLOT_D(k64, sf.kmin); pay[u] = (unsigned int) p64; }
            else { key[u] = k64; pay[u] = p64; }
        }
    }
    __syncthreads();
    // ---- e[s] for the FILL_ROWS slots this thread owns
    {
        int c[FILL_ROWS];
        const uint4 *c4 = (const uint4 *) (sm.cnt + tid * FILL_ROWS);
#pragma unroll
        for (int q = 0; q < FILL_ROWS / 4; q++) { uint4 v = c4[q]; c[4 * q] = (int) v.x; c[4 * q + 1] = (int) v.y; c[4 * q + 2] = (int) v.z; c[4 * q + 3] = (int) v.w; }
        int p[FILL_ROWS], run = 0, lmin = 0;
#pragma unroll
        for (int j = 0; j < FILL_ROWS; j++) { p[j] = run; lmin = min(lmin, run); run += c[j] - 1; }
        // inclusive warp scan of (sum, prefix-min) with combine(a, b) = (a.s + b.s, min(a.m, a.s + b.m))
        int S = run, M = lmin;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            int ps = __shfl_up_sync(0xffffffffu, S, o), pm = __shfl_up_sync(0xffffffffu, M, o);
            if (lane >= o) { M = min(pm, ps + M); S = ps + S; }
        }
        if (lane == 31) { sm.wsum[warp] = S; sm.wmin[warp] = M; }
        int xs = __shfl_up_sync(0xffffffffu, S, 1), xm = __shfl_up_sync(0xffffffffu, M, 1);
        if (lane == 0) { xs = 0; xm = FILL_INF; }
        __syncthreads();
        int bs = 0, bm = FILL_INF;                    // everything in the warps before this one
        for (int w = 0; w < warp; w++) { bm = min(bm, bs + sm.wmin[w]); bs += sm.wsum[w]; }
        const int base = bs + xs, mprev = min(bm, bs + xm);   // P at this thread's first slot; min of P over all earlier slots
        int rmin = mprev;
        uint4 o4[FILL_ROWS / 4];
        unsigned int *o = (unsigned int *) o4;
#pragma unroll
        for (int j = 0; j < FILL_ROWS; j++) { int P = base + p[j]; rmin = min(rmin, P); o[j] = (unsigned int) (P - rmin); }
        uint4 *d4 = (uint4 *) (sm.cnt + tid * FILL_ROWS);
#pragma unroll
        for (int q = 0; q < FILL_ROWS / 4; q++) d4[q] = o4[q];
    }
    __syncthreads();
    // ---- placement
    int wrapped = 0;
#pragma unroll
    for (int u = 0; u < FILL_ROWS; u++) {
        if (sr[u] == 0xffffffffu) continue;
        unsigned int sl = sr[u] & (GX_SUB - 1), pos = sl + sm.cnt[sl] + (sr[u] >> GX_SUB_LOG2);
        steps += pos - sl; placed++;
        if (pos < GX_SUB) {
            if (F == GX_SLOTS_NARROW) ((unsigned int *) sm.tab)[pos] = (unsigned int) key[u];
            else if (C) { uint2 v; v.x = (unsigned int) key[u]; v.y = (unsigned int) pay[u]; ((uint2 *) sm.tab)[pos] = v; }
            else { longlong2 v; v.x = key[u]; v.y = (long long) pay[u]; ((longlong2 *) sm.tab)[pos] = v; }
            sr[u] = 0xffffffffu;
        } else wrapped = 1;
    }
    if (__syncthreads_or(wrapped)) {
#pragma unroll
        for (int u = 0; u < FILL_ROWS; u++) {
            if (sr[u] == 0xffffffffu) continue;
            unsigned int sl = 0;                      // everything from its slot to the end is full: continue from the start
            for (;;) {
                bool won;
                if (F == GX_SLOTS_NARROW) won = atomicCAS((unsigned int *) sm.tab + sl, 0u, (unsigned int) key[u]) == 0u;
                else if (C) {
                    gx_cslot *t = (gx_cslot *) sm.tab;
                    won = atomicCAS(&t[sl].d, 0u, (unsigned int) key[u]) == 0u;
                    if (won) t[sl].payload = (unsigned int) pay[u];
                } else {
                    gx_slot *t = (gx_slot *) sm.tab;
                    won = (long long) atomicCAS((unsigned long long *) &t[sl].key, (unsigned long long) GX_EMPTY_KEY, (unsigned long long) key[u]) == GX_EMPTY_KEY;
                    if (won) t[sl].payload = pay[u];
                }
                if (won) break;
                sl = (sl + 1) & (GX_SUB - 1); steps++;
            }
        }
        __syncthreads();
    }
    // ---- stream the finished sub-table out
    if (C) {
        const uint4 *t4 = (const uint4 *) sm.tab;
        uint4 *d4 = (uint4 *) dst;
#pragma unroll
        for (int u = 0; u < FILL_ROWS * SB / 16; u++) d4[tid + u * FILL_THREADS] = t4[tid + u * FILL_THREADS];
    } else {
        const longlong2 *t2 = (const longlong2 *) sm.tab;
        longlong2 *d2 = (longlong2 *) dst;
#pragma unroll
        for (int u = 0; u < FILL_ROWS; u++) d2[tid + u * FILL_THREADS] = t2[tid + u * FILL_THREADS];
    }
    __syncthreads();
}

__device__ __forceinline__ void fill_report(const gx_build_args &b, unsigned int steps, unsigned int placed)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { steps += __shfl_down_sync(0xffffffffu, steps, o); placed += __shfl_down_sync(0xffffffffu, placed, o); }
    if ((threadIdx.x & 31) == 0) {
        if (steps) atomicAdd((unsigned long long *) &b.counters[SW_STEPS], (unsigned long long) steps);      // chain statistics decide whether
        if (placed) atomicAdd((unsigned long long *) &b.counters[SW_PLACED], (unsigned long long) placed);    // the slot function is kept
    }
}

// one CTA per sub-table (grid-strided) over the buckets the scatter passes produced
__global__ void __launch_bounds__(FILL_THREADS, 4) gx_k_bbuild_fill(gx_bbuild_args a)
{
    extern __shared__ __align__(16) unsigned char fill_smem_raw[];
    gx_fill_smem &sm = *(gx_fill_smem *) fill_smem_raw;
    unsigned int steps = 0, placed = 0;
    int pay_miss = 0;                                  // narrow form only
    for (long long sub = blockIdx.x; sub < a.nsub; sub += gridDim.x) {
        unsigned int n = a.cursor[sub];
        if (n >= GX_SUB) n = 0;                        // overflowed: the host rebuilds directly
        const longlong2 *src = (const longlong2 *) a.pairs + sub * GX_SUB;
        gx_subtable_build<GX_SLOTS_WIDE>(sm, n, a.b.sf,
                          [&](unsigned int i, long long &k, unsigned long long &p) { longlong2 v = src[i]; k = v.x; p = (unsigned long long) v.y; return true; },
                          a.b.slots + sub * GX_SUB, steps, placed, pay_miss);
    }
    fill_report(a.b, steps, 0);                        // entries are counted from the cursors (gx_k_bbuild_total)
}

// ---------------------------------------------------------------------------
// Partition-free build for a build side that is stored in key order (a table kept in
// primary-key order, e.g. TPC-H orders) when the order-preserving slot function is in
// use: the rows of one sub-table are then one CONTIGUOUS row range, found by binary
// search, so no bucketing pass is needed at all — each CTA reads its rows straight from
// the columns (coalesced), builds the sub-table in shared memory and streams it out.
// one coalesced pass over the key column: verifies ascending order and records, for every
// sub-table, the first row that maps to it (start[nsub] = nrows)
__global__ void gx_k_sorted_bounds(gx_build_args a, long long nsub, long long *start, int *unsorted)
{
    long long stride = (long long) gridDim.x * blockDim.x;
    for (long long i = (long long) blockIdx.x * blockDim.x + threadIdx.x; i < a.nrows; i += stride) {
        if (gx_is_null(a.key, i)) { *unsorted = 1; return; }
        long long k = gx_load_int(a.key, i);
        long long sb = (k == GX_EMPTY_KEY) ? -1 : (long long) (gx_slot_index(k, a.sf) >> GX_SUB_LOG2);
        long long sp = -1;
        if (i > 0) {
            long long kp = gx_load_int(a.key, i - 1);
            if (kp > k) { *unsorted = 1; return; }
            sp = (kp == GX_EMPTY_KEY) ? -1 : (long long) (gx_slot_index(kp, a.sf) >> GX_SUB_LOG2);
        }
        for (long long s2 = sp + 1; s2 <= sb; s2++) start[s2] = i;
        if (i == a.nrows - 1) for (long long s2 = sb + 1; s2 <= nsub; s2++) start[s2] = a.nrows;
    }
}

// the same for an int8 key column without NULLs: 4 consecutive keys per lane (two 16-byte
// loads), the predecessor of a lane's first key comes from the lane below by shuffle
__global__ void __launch_bounds__(256) gx_k_sorted_bounds_i8(const long long *__restrict__ keys, long long nrows, gx_slotfn sf,
                                                             long long nsub, long long *start, int *unsorted)
{
    const int lane = threadIdx.x & 31;
    const long long nwarp = ((long long) gridDim.x * blockDim.x) >> 5, wid = ((long long) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long ngroups = (nrows + 127) >> 7;
    bool bad = false;
    for (long long gq = wid; gq < ngroups; gq += nwarp) {
        const long long r0 = (gq << 7) + lane * 4;
        long long k[4];
        if (r0 + 3 < nrows) {
            longlong2 a = __ldg((const longlong2 *) (keys + r0)), b = __ldg((const longlong2 *) (keys + r0 + 2));
            k[0] = a.x; k[1] = a.y; k[2] = b.x; k[3] = b.y;
        } else {
#pragma unroll
            for (int j = 0; j < 4; j++) k[j] = r0 + j < nrows ? __ldg(keys + r0 + j) : 0x7fffffffffffffffLL;
        }
        long long sb[4];
#pragma unroll
        for (int j = 0; j < 4; j++) sb[j] = (k[j] == GX_EMPTY_KEY) ? -1 : (long long) (gx_slot_index(k[j], sf) >> GX_SUB_LOG2);
        long long kp = __shfl_up_sync(0xffffffffu, k[3], 1), sp = __shfl_up_sync(0xffffffffu, sb[3], 1);
        if (lane == 0) {
            if (r0 == 0) { kp = k[0]; sp = -1; }
            else { kp = __ldg(keys + r0 - 1); sp = (kp == GX_EMPTY_KEY) ? -1 : (long long) (gx_slot_index(kp, sf) >> GX_SUB_LOG2); }
        }
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const long long r = r0 + j;
            if (r < nrows) {
                if (kp > k[j]) bad = true;
                if (sb[j] != sp) for (long long s2 = sp + 1; s2 <= sb[j]; s2++) start[s2] = r;
                if (r == nrows - 1) for (long long s2 = sb[j] + 1; s2 <= nsub; s2++) start[s2] = nrows;
                kp = k[j]; sp = sb[j];
            }
        }
    }
    if (__any_sync(0xffffffffu, bad) && lane == 0) *unsorted = 1;
}

// The generic row loader (any key type, NULLs, build-side quals, packed payload); in the VERIFY form an int8 key
// without NULLs.  The shapes of a plain key + one 4-byte column (or none) go to gx_k_sorted_fill_staged below.
// Output of the key-ordered fills in slot format F
template <int F> __device__ __forceinline__ char *fill_out(const gx_bbuild_args &a)
{
    return F == GX_SLOTS_NARROW ? (char *) a.narrow : F == GX_SLOTS_COMPACT ? (char *) a.cslots : (char *) a.b.slots;
}
template <int F, bool VERIFY>
__global__ void __launch_bounds__(FILL_THREADS, F != GX_SLOTS_WIDE ? 5 : 4) gx_k_sorted_fill(gx_bbuild_args a)      // 5 CTAs/SM
{
    extern __shared__ __align__(16) unsigned char fill_smem_raw[];
    gx_fill_smem_t<F> &sm = *(gx_fill_smem_t<F> *) fill_smem_raw;
    char *const out = fill_out<F>(a);
    const size_t slot_bytes = sizeof(typename gx_slot_of<F>::type);
    if (!VERIFY && *a.unsorted) return;
    unsigned int steps = 0, placed = 0;
    int bad = 0, pay_miss = 0;
    const long long *keys = (const long long *) a.b.key.data;
    long long lo = 0, hi = 0;
    if (blockIdx.x < a.nsub) { lo = a.start[blockIdx.x]; hi = a.start[blockIdx.x + 1]; }
    for (long long sub = blockIdx.x; sub < a.nsub; sub += gridDim.x) {
        long long nlo = 0, nhi = 0;
        const long long nsubn = sub + gridDim.x;
        if (nsubn < a.nsub) { nlo = a.start[nsubn]; nhi = a.start[nsubn + 1]; }
        unsigned int n = (unsigned int) (hi - lo);
        if (hi - lo >= GX_SUB) { n = 0; if (threadIdx.x == 0) atomicOr(a.overflow, OVF_FULL); }     // a sub-table keeps one slot free
        if (VERIFY && hi < lo) { n = 0; bad = 1; }
        if (!VERIFY)
            gx_subtable_build<F>(sm, n, a.b.sf,
                              [&](unsigned int i, long long &k, unsigned long long &p) {
                                  long long r = lo + i;
                                  if (!build_row_ok(a.b, r)) return false;
                                  k = gx_load_int(a.b.key, r); p = pack_payload(a.b, r); return true; },
                              out + (size_t) sub * GX_SUB * slot_bytes, steps, placed, pay_miss);
        else                                                   // int8 key without NULLs; quals and any payload
            gx_subtable_build<F>(sm, n, a.b.sf,
                              [&](unsigned int i, long long &k, unsigned long long &p) {
                                  const long long r = lo + i;
                                  k = __ldg(keys + r);
                                  const long long kp = r > 0 ? __ldg(keys + r - 1) : k;
                                  if (kp > k || k == GX_EMPTY_KEY) bad = 1;          // order is checked on every row, kept or not
                                  if (!build_row_ok(a.b, r)) return false;
                                  p = pack_payload(a.b, r); return true; },
                              out + (size_t) sub * GX_SUB * slot_bytes, steps, placed, pay_miss, sub, &bad);
        lo = nlo; hi = nhi;
    }
    if (VERIFY && bad) *a.unsorted = 1;
    if (pay_miss) atomicOr(a.overflow, OVF_PAYLOAD);
    fill_report(a.b, steps, placed);
}

// ---------------------------------------------------------------------------
// The key-ordered fill for the loader shapes of a table kept in primary-key order (TPC-H orders):
// PK 1 = an int8 key without NULLs or quals + one 4-byte payload column, PK 2 = the same key, payload = row number.
// Persistent: CTA b owns the contiguous block of sub-tables [nsub b / grid, nsub (b + 1) / grid), so its input is one
// contiguous row range and its output one contiguous piece of the table.  The rows of a sub-table never pass through
// a global load in the row loop: thread 0 copies them into a two-deep stage ring with cp.async.bulk (completion counted
// on the stage's mbarrier) two sub-tables ahead, so the copy of sub-table s + 1 travels while s is histogrammed,
// scanned and placed.  A stage holds a 16-byte aligned superset of the key range including the row before it (the
// order check's predecessor) and of the payload range; the rounding reads at most 15 bytes past a column's last row,
// inside the last row's 16-byte block.  The finished sub-table leaves with plain 16-byte stores, which the CTA does
// not wait for.  Checks, flags and chain counters are those of gx_k_sorted_fill; a wait that gives up raises bit 2 of
// *overflow and the host rebuilds with gx_k_sorted_fill.  Both raise bit 4 for a payload outside the narrow form's window.
#define FSTAGE_KEYS (GX_SUB + 4)                   // rows [lo - 1, hi) rounded out to even rows: at most 2047 + 3
#define FSTAGE_PAYS (GX_SUB + 8)                   // rows [lo, hi) rounded out to multiples of 4: at most 2047 + 6
template <int PK> struct __align__(16) gx_fill_stage {
    long long key[FSTAGE_KEYS];
    unsigned int pay[PK == 1 ? FSTAGE_PAYS : 4];
    unsigned long long bar;
    long long lo, hi;                              // the staged sub-table's row range, written by thread 0 before its arrive
};
template <int PK, int F> constexpr int staged_smem_bytes() { return (int) (sizeof(gx_fill_smem_t<F>) + 2 * sizeof(gx_fill_stage<PK>)); }

template <int PK, int F, bool VERIFY>
__global__ void __launch_bounds__(FILL_THREADS, F != GX_SLOTS_WIDE ? 3 : 2) gx_k_sorted_fill_staged(gx_bbuild_args a)      // what shared memory allows
{
    extern __shared__ __align__(16) unsigned char fill_smem_raw[];
    gx_fill_smem_t<F> &sm = *(gx_fill_smem_t<F> *) fill_smem_raw;
    gx_fill_stage<PK> *const stage = (gx_fill_stage<PK> *) (fill_smem_raw + sizeof(gx_fill_smem_t<F>));
    char *const out = fill_out<F>(a);
    const size_t slot_bytes = sizeof(typename gx_slot_of<F>::type);
    if (!VERIFY && *a.unsorted) return;
    const long long s0 = a.nsub * blockIdx.x / gridDim.x, s1 = a.nsub * (blockIdx.x + 1) / gridDim.x;
    const long long *keys = (const long long *) a.b.key.data;
    const unsigned int *pay4 = (const unsigned int *) a.b.payload[0].data;
    // thread 0: stage the rows of sub-table s.  An empty or overflowing range stages nothing and completes the phase at once.
    auto issue = [&](long long s, gx_fill_stage<PK> &st) {
        const long long lo = a.start[s], hi = a.start[s + 1];
        st.lo = lo; st.hi = hi;
        if (hi <= lo || hi - lo >= GX_SUB) { gx_mbar_arrive(&st.bar); return; }
        const long long k0 = (lo > 0 ? lo - 1 : 0) & ~1LL, k1 = (hi + 1) & ~1LL;
        const long long p0 = lo & ~3LL, p1 = (hi + 3) & ~3LL;
        const unsigned int kb = (unsigned int) (k1 - k0) * 8u, pb = PK == 1 ? (unsigned int) (p1 - p0) * 4u : 0u;
        // the CTA's generic-proxy reads of the stage's previous rows are ordered before the copy engine's writes
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        gx_mbar_arrive_expect_tx(&st.bar, kb + pb);
        gx_bulk_g2s(st.key, keys + k0, kb, &st.bar);
        if (PK == 1) gx_bulk_g2s(st.pay, pay4 + p0, pb, &st.bar);
    };
    if (threadIdx.x == 0) {
        gx_mbar_init(&stage[0].bar, 1); gx_mbar_init(&stage[1].bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        if (s0 < s1) issue(s0, stage[0]);
        if (s0 + 1 < s1) issue(s0 + 1, stage[1]);
    }
    __syncthreads();
    unsigned int steps = 0, placed = 0;
    int bad = 0, pay_miss = 0;
    bool stuck = false;
    for (long long s = s0; s < s1; s++) {
        gx_fill_stage<PK> &st = stage[(s - s0) & 1];
        if (__syncthreads_or(!gx_mbar_wait(&st.bar, (unsigned int) ((s - s0) >> 1) & 1u))) { stuck = true; break; }
        const long long lo = st.lo, hi = st.hi;
        unsigned int n = (unsigned int) (hi - lo);
        if (hi - lo >= GX_SUB) { n = 0; if (threadIdx.x == 0) atomicOr(a.overflow, OVF_FULL); }       // a sub-table keeps one slot free
        if (hi < lo) { n = 0; bad = 1; }
        const long long *sk = st.key + (lo - ((lo > 0 ? lo - 1 : 0) & ~1LL));                 // row lo; sk[-1] is row lo - 1
        const unsigned int *sp = st.pay + (lo & 3);
        gx_subtable_build<F>(sm, n, a.b.sf,
                          [&](unsigned int i, long long &k, unsigned long long &p) {
                              k = sk[i];
                              if (VERIFY) {
                                  const long long kp = lo + i > 0 ? sk[(int) i - 1] : k;
                                  if (kp > k || k == GX_EMPTY_KEY) bad = 1;
                              }
                              p = PK == 1 ? (unsigned long long) sp[i] : (unsigned long long) (lo + i);
                              return true; },
                          out + (size_t) s * GX_SUB * slot_bytes, steps, placed, pay_miss, VERIFY ? s : -1, &bad);
        // gx_subtable_build ends with a barrier: nobody reads this stage any more
        if (threadIdx.x == 0 && s + 2 < s1) issue(s + 2, st);
    }
    if (stuck && threadIdx.x == 0) atomicOr(a.overflow, OVF_STUCK);
    if (VERIFY && bad) *a.unsorted = 1;
    if (pay_miss) atomicOr(a.overflow, OVF_PAYLOAD);
    fill_report(a.b, steps, placed);
}
// ---------------------------------------------------------------------------
// Bounds by SEARCH instead of by a pass over the key column (int8 key without NULLs).
//  * lower_bound(s) = first row whose key maps to sub-table >= s.  One warp: the 32 rows around
//    the interpolated position s * rows-per-sub-table decide it in one round when the keys are
//    as uniform as the slot function assumes; otherwise a bracket is grown (x16 per round) and
//    narrowed 32-ary.  All nsub + 1 bounds cost microseconds (gx_k_sorted_bounds_search).
//  * what the pass over the column used to establish is then VERIFIED by the fill itself
//    (gx_k_sorted_fill<.., VERIFY>): every CTA checks that its rows map to its sub-table and
//    ascend (each row against its predecessor, including the one before its range).
//    start[0] = 0 and start[nsub] = nrows are fixed and the ranges [start[s], start[s+1]) tile
//    [0, nrows), so if no CTA raises the flag every adjacent pair of rows has been compared and
//    every row sits in the right sub-table — whatever the search returned.  A raised flag sends
//    the host down the bucketing path.  The search itself: sorted_lower_bound (gx_internal.cuh).

// start[s] for every sub-table by search: one warp per bound, ~one 256-byte read each
__global__ void __launch_bounds__(256) gx_k_sorted_bounds_search(const long long *__restrict__ keys, long long nrows, gx_slotfn sf,
                                                                 long long nsub, long long nslots, long long *start)
{
    const int lane = threadIdx.x & 31;
    const long long nwarp = ((long long) gridDim.x * blockDim.x) >> 5, wid = ((long long) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const double rows_per_sub = (double) nrows * (double) GX_SUB / (double) (nslots - GX_SUB);
    // a warp takes a CONTIGUOUS block of bounds and seeds each search with the previous result
    const long long per = (nsub + 1 + nwarp - 1) / nwarp, s0 = wid * per;
    long long prev = -1;
    for (long long s = s0; s < s0 + per && s <= nsub; s++) {
        const long long v = sorted_lower_bound(keys, nrows, sf, s, nsub, rows_per_sub, lane, prev);
        if (lane == 0) start[s] = v;
        prev = (s > 0 && s < nsub) ? v : -1;
    }
}

// rows with the reserved key INT64_MIN sort first: move them to the side list
__global__ void gx_k_sorted_special(gx_build_args a, const long long *start, const int *unsorted)
{
    if (*unsorted) return;
    const long long n = start[0];
    for (long long r = threadIdx.x; r < n; r += blockDim.x) {
        if (gx_is_null(a.key, r) || gx_load_int(a.key, r) != GX_EMPTY_KEY) continue;
        if (!build_row_ok(a, r)) continue;
        int idx = (int) atomicAdd((unsigned long long *) &a.counters[SW_SPECIAL], 1ULL);
        if (idx < a.special_cap) a.special[idx] = pack_payload(a, r);
    }
}

// entries actually placed = sum of the cursors
__global__ void gx_k_bbuild_total(const unsigned int *cursor, long long n, long long *total)
{
    long long sum = 0;
    for (long long i = (long long) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long) gridDim.x * blockDim.x) sum += cursor[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_down_sync(0xffffffffu, sum, o);
    if ((threadIdx.x & 31) == 0 && sum) atomicAdd((unsigned long long *) total, (unsigned long long) sum);
}
__global__ void gx_k_scan_i64(long long *v, long long n, long long *total);   // gx_agg.cu

// key-density estimate for the slot function: min / max over a strided sample; the same for the payload column
// (pay.data non-null: the narrow slot form's payload window) of the sampled rows with a key.  *order (when not null): bit 0
// = a sampled key is below the one a stride before it, bit 1 = equal to it (a NULL counts as neither)
__global__ void gx_k_key_range(gx_dcol key, gx_dcol pay, long long nrows, long long stride, long long *minmax, long long *pminmax, int *order)
{
    long long i = ((long long) blockIdx.x * blockDim.x + threadIdx.x) * stride;
    long long lo = 0x7fffffffffffffffLL, hi = -0x7fffffffffffffffLL - 1, plo = lo, phi = hi;
    if (i < nrows && !gx_is_null(key, i)) {
        lo = hi = gx_load_int(key, i);
        if (pay.data) plo = phi = gx_load_int(pay, i);
        if (order && i + stride < nrows && !gx_is_null(key, i + stride)) {
            const long long next = gx_load_int(key, i + stride);
            if (next <= lo) atomicOr(order, next < lo ? 1 : 2);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        long long a = __shfl_down_sync(0xffffffffu, lo, o), b = __shfl_down_sync(0xffffffffu, hi, o);
        lo = a < lo ? a : lo; hi = b > hi ? b : hi;
        a = __shfl_down_sync(0xffffffffu, plo, o); b = __shfl_down_sync(0xffffffffu, phi, o);
        plo = a < plo ? a : plo; phi = b > phi ? b : phi;
    }
    if ((threadIdx.x & 31) == 0 && minmax) {
        atomicMin(&minmax[0], lo); atomicMax(&minmax[1], hi);
        if (pay.data) { atomicMin(&pminmax[0], plo); atomicMax(&pminmax[1], phi); }
    }
}

// Interpolation is tried when the key span is at most this many times the row count: TPC-H order
// keys use 8 of every 32 values (spread 4), and each of N datanodes holds a pseudo-random 1/N of
// them (spread 4 N).  Uniformity itself is not sampled: a build whose sub-tables overflow or whose
// average chain exceeds 4 is redone with the mixing hash.
#define GX_INTERP_MAX_SPREAD 256.0

// the build's environment switches (README), read once per build
struct build_switches {
    unsigned int win;                 // GX_SLOT_WIN (31)
    int slot_mode;                    // GX_SLOT_MODE: 0 mixing hash without a sample, 1 interpolation at any key spread (-1)
    bool wide, direct, nosorted, onepass, nosearch, nocompact;   // GX_SLOT_WIDE, GX_BUILD_{DIRECT,NOSORTED,ONEPASS},
};                                                               // GX_NO_BOUNDS_SEARCH, GX_NO_COMPACT = 1
static bool switch_on(const char *name) { const char *e = getenv(name); return e && e[0] == '1'; }
static build_switches read_build_switches()
{
    const char *win = getenv("GX_SLOT_WIN"), *mode = getenv("GX_SLOT_MODE");
    return { win ? (unsigned int) atoi(win) : 31u, mode ? atoi(mode) : -1, switch_on("GX_SLOT_WIDE"), switch_on("GX_BUILD_DIRECT"),
             switch_on("GX_BUILD_NOSORTED"), switch_on("GX_BUILD_ONEPASS"), switch_on("GX_NO_BOUNDS_SEARCH"), switch_on("GX_NO_COMPACT") };
}

// interpolation slot function over [kmin, kmin + range): slots [0, nslots - GX_SUB), monotone in the key.
// Narrow ranges (< 2^32, the usual case: at most 16 keys of range per row) use 32-bit arithmetic unless `wide`.
static void gx_set_interpolation(gx_hash *h, long long kmin, double range_d, bool wide)
{
    const long double ratio = (long double) (h->nslots - GX_SUB) / (long double) range_d;
    h->kmin = kmin;
    if (range_d < 4294967295.0 && !wide) {
        int sh = 0;
        while (sh < 62 && ratio * (long double) (1ULL << (sh + 1)) < 4294967295.0L) sh++;
        h->mode = 2; h->shift = (unsigned int) sh;
        h->scale = (unsigned long long) (ratio * (long double) (1ULL << sh));
        return;
    }
    h->mode = 1; h->shift = 0;
    const long double sc = (long double) 18446744073709551616.0L * ratio;
    h->scale = sc >= 18446744073709551615.0L ? ~0ULL : (unsigned long long) sc;
}

// The fill of the key-ordered build.  pk 1 / 2: gx_k_sorted_fill_staged, one resident grid; pk 0 (and the rebuild after
// a staged wait gave up): gx_k_sorted_fill.  The second profile name tells which one ran.
template <int PK, int F, bool VERIFY> static void sorted_fill_staged(gx_ctx *ctx, const gx_bbuild_args &ba)
{
    static int per_sm = 0;
    if (!per_sm) {
        cudaFuncSetAttribute(gx_k_sorted_fill_staged<PK, F, VERIFY>, cudaFuncAttributeMaxDynamicSharedMemorySize, staged_smem_bytes<PK, F>());
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gx_k_sorted_fill_staged<PK, F, VERIFY>, FILL_THREADS,
                                                          staged_smem_bytes<PK, F>()) != cudaSuccess || per_sm < 1) per_sm = 1;
    }
    gx_launch_scope which(ctx, "build_fill_staged", 0);
    gx_k_sorted_fill_staged<PK, F, VERIFY><<<per_sm * ctx->sm_count, FILL_THREADS, staged_smem_bytes<PK, F>(), ctx->stream>>>(ba);
}
// F: slot format; the narrow form only serves pk 1 (and pk 0, the generic loader)
template <int F, bool VERIFY> static void sorted_fill(gx_ctx *ctx, const gx_bbuild_args &ba, int pk)
{
    if (pk == 1) { sorted_fill_staged<1, F, VERIFY>(ctx, ba); return; }
    if constexpr (F != GX_SLOTS_NARROW) { if (pk == 2) { sorted_fill_staged<2, F, VERIFY>(ctx, ba); return; } }
    const int bytes = (int) sizeof(gx_fill_smem_t<F>);
    static bool attr = false;
    if (!attr) { cudaFuncSetAttribute(gx_k_sorted_fill<F, VERIFY>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes); attr = true; }
    gx_launch_scope which(ctx, "build_fill_rows", 0);
    gx_k_sorted_fill<F, VERIFY><<<ctx->sm_count * (F != GX_SLOTS_WIDE ? 10 : 8), FILL_THREADS, bytes, ctx->stream>>>(ba);
}

// gx_hash_slotfn's inverse (the mask follows nslots)
static void set_slotfn(gx_hash *h, const gx_slotfn &f)
{ h->mode = f.mode; h->win = f.win; h->kmin = f.kmin; h->scale = f.scale; h->shift = f.shift; h->amask = f.amask; h->tbits = f.tbits; h->pbase = f.pbase; }
template <class T> struct tmp_buf {                 // a temporary device buffer, freed at scope exit
    gx_ctx *ctx; T *p = nullptr;
    explicit tmp_buf(gx_ctx *c) : ctx(c) {}
    ~tmp_buf() { gx_tmp_free(ctx, p); }
    cudaError_t alloc(size_t n) { cudaError_t e = gx_tmp_alloc(ctx, (void **) &p, n * sizeof(T)); if (e != cudaSuccess) p = nullptr; return e; }
};
static cudaError_t clear_scratch(gx_ctx *ctx, int w0, int w1) { return cudaMemsetAsync(ctx->d_scratch + w0, 0, (w1 - w0 + 1) * sizeof(long long), ctx->stream); }
static double fill_avg_chain(const long long *w) { return w[SW_PLACED] > 0 ? (double) w[SW_STEPS] / (double) w[SW_PLACED] : 0.0; }
// One join-table build.  h owns the slot function: a.sf = gx_hash_slotfn(h) before every launch.
struct build_job {
    gx_ctx *ctx; const gx_table *inner; int key_col; build_switches sw;
    gx_build_args a; int payload_bytes;
    gx_hash *h;                       // freed unless handed out
    build_job(gx_ctx *c, const gx_table *t, int k) : ctx(c), inner(t), key_col(k), sw(read_build_switches()), payload_bytes(0), h(nullptr) { memset(&a, 0, sizeof(a)); }
    ~build_job() { if (h) gx_hash_free(h); }
};

// argument checks, build arguments, and the table's slots and side list
static int build_setup(build_job &j, int n_preds, const gx_pred *preds, int n_payload, const int32_t *payload_cols, int unique)
{
    gx_ctx *ctx = j.ctx; const gx_table *inner = j.inner; const int key_col = j.key_col; gx_build_args &a = j.a;
    GX_CHECK_ARG(ctx, key_col >= 0 && key_col < inner->ncols, "hash_build: key column %d out of range", key_col);
    int kt = inner->types[key_col];
    GX_CHECK_ARG(ctx, kt == GX_INT4 || kt == GX_INT8 || kt == GX_DATE, "hash_build: key type %d not hashable here (int4/int8/date only)", kt);
    GX_CHECK_ARG(ctx, n_payload >= 0 && n_payload <= GX_MAX_PAYLOAD, "hash_build: n_payload %d", n_payload);
    a.key.data = inner->cols[key_col]; a.key.nulls = inner->nulls[key_col]; a.key.type = kt;
    a.npreds = n_preds; a.n_payload = n_payload; a.nrows = inner->nrows;
    int rc = gx_fill_dpreds(ctx, inner, n_preds, preds, a.preds); if (rc) return rc;
    gx_hash *h = j.h = (gx_hash *) calloc(1, sizeof(gx_hash));
    h->ctx = ctx; h->key_type = kt; h->n_payload = n_payload; h->unique = unique; h->src = inner; h->src_version = inner->version; h->n_preds = n_preds;
    if (n_preds > 0) memcpy(h->preds, preds, (size_t) n_preds * sizeof(gx_pred));      // n_preds checked by gx_fill_dpreds
    for (int i = 0; i < n_payload; i++) {
        int c = payload_cols[i];
        if (c < 0 || c >= inner->ncols) { GX_SET_ERR(ctx, "hash_build: payload column %d out of range", c); return GX_ERR_ARG; }
        if (inner->nulls[c]) { GX_SET_ERR(ctx, "hash_build: nullable payload column %d not supported in-slot", c); return GX_ERR_ARG; }
        a.payload[i].data = inner->cols[c]; a.payload[i].nulls = nullptr; a.payload[i].type = inner->types[c];
        h->payload_types[i] = inner->types[c];
        j.payload_bytes += gx_type_size(inner->types[c]);
    }
    if (j.payload_bytes > 8) { GX_SET_ERR(ctx, "hash_build: payload columns total %d bytes > 8", j.payload_bytes); return GX_ERR_ARG; }
    h->nslots = gx_pow2_ceil(inner->nrows + inner->nrows / 2 + 16); h->special_cap = 1 << 16;      // load factor <= 0.67
    h->win = j.sw.win; h->amask = 1u;                           // the mixing hash until the sample says otherwise
    a.mask = (unsigned long long) h->nslots - 1; a.special_cap = h->special_cap; a.counters = ctx->d_scratch;
    return GX_OK;
}
// the table's slots and side list
static int alloc_table(build_job &j)
{
    gx_ctx *ctx = j.ctx; gx_hash *h = j.h;
    cudaError_t e = gx_tmp_alloc(ctx, (void **) &h->slots, (size_t) h->nslots * sizeof(gx_slot));
    if (e == cudaSuccess) e = gx_tmp_alloc(ctx, (void **) &h->special_payload, (size_t) h->special_cap * sizeof(unsigned long long));
    if (e != cudaSuccess) { GX_SET_ERR(ctx, "hash_build: cudaMalloc of %lld slots failed: %s", (long long) h->nslots, cudaGetErrorString(e)); return GX_ERR_NOMEM; }
    j.a.slots = h->slots; j.a.special = h->special_payload;
    return GX_OK;
}
// the sample's key and payload ranges, the key column's first and last key, and the slot function chosen
struct key_sample { long long lo, hi, pmin, pmax, first, last; bool have_prange, have_ends, sampled; int order; gx_slotfn sf; };
// the key column's first and last key (this synchronises the stream)
static int fetch_key_ends(const build_job &j, key_sample &s)
{
    gx_ctx *ctx = j.ctx; const int ksz = gx_type_size(j.a.key.type); const char *col = (const char *) j.a.key.data;
    long long *w = ctx->h_scratch + SW_ENDS; w[0] = w[1] = 0;
    GX_CUDA(ctx, cudaMemcpyAsync(w, col, ksz, cudaMemcpyDeviceToHost, ctx->stream));
    GX_CUDA(ctx, cudaMemcpyAsync(w + 1, col + (size_t) (j.inner->nrows - 1) * ksz, ksz, cudaMemcpyDeviceToHost, ctx->stream));
    GX_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    s.first = ksz == 4 ? (long long) (int) w[0] : w[0]; s.last = ksz == 4 ? (long long) (int) w[1] : w[1]; s.have_ends = true;
    return GX_OK;
}
// choose the slot function from a strided key sample (64 K keys): interpolation when the
// keys span at most GX_INTERP_MAX_SPREAD x their count
static int sample_keys(build_job &j, key_sample &s)
{
    gx_ctx *ctx = j.ctx; const long long nrows = j.inner->nrows; s = key_sample();
    if (nrows >= 4096 && j.h->nslots >= 64 * GX_SUB && j.sw.slot_mode != 0) {
        long long stride = nrows / 65536; if (stride < 1) stride = 1;
        const long long nthreads = (nrows + stride - 1) / stride, init[2] = { 0x7fffffffffffffffLL, -0x7fffffffffffffffLL - 1 };
        long long *krange = ctx->d_scratch + SW_KRANGE, *prange = ctx->d_scratch + SW_PRANGE;
        GX_CUDA(ctx, cudaMemcpyAsync(krange, init, sizeof(init), cudaMemcpyHostToDevice, ctx->stream));
        GX_CUDA(ctx, cudaMemcpyAsync(prange, init, sizeof(init), cudaMemcpyHostToDevice, ctx->stream));
        int *order = (int *) (ctx->d_scratch + SW_ORDER);
        GX_CUDA(ctx, cudaMemsetAsync(order, 0, sizeof(long long), ctx->stream));
        // one int4/date payload column: its sampled range decides whether the narrow slot form can hold it
        const bool pay4 = j.a.n_payload == 1 && (j.a.payload[0].type == GX_INT4 || j.a.payload[0].type == GX_DATE);
        gx_dcol pay; memset(&pay, 0, sizeof(pay)); if (pay4) pay = j.a.payload[0];
        { gx_launch_scope ls(ctx, "build_sample"); gx_k_key_range<<<(unsigned) ((nthreads + 255) / 256), 256, 0, ctx->stream>>>(j.a.key, pay, nrows, stride, krange, prange, order); }
        GX_CUDA(ctx, cudaMemcpyAsync(ctx->h_scratch + SW_KRANGE, krange, 2 * sizeof(long long), cudaMemcpyDeviceToHost, ctx->stream));
        GX_CUDA(ctx, cudaMemcpyAsync(ctx->h_scratch + SW_PRANGE, prange, 2 * sizeof(long long), cudaMemcpyDeviceToHost, ctx->stream));
        GX_CUDA(ctx, cudaMemcpyAsync(ctx->h_scratch + SW_ORDER, order, sizeof(long long), cudaMemcpyDeviceToHost, ctx->stream));
        int rc = fetch_key_ends(j, s); if (rc) return rc;          // the sample's one synchronise
        const long long *w = ctx->h_scratch;
        s.lo = w[SW_KRANGE]; s.hi = w[SW_KRANGE + 1]; s.pmin = w[SW_PRANGE]; s.pmax = w[SW_PRANGE + 1]; s.have_prange = pay4 && s.pmin <= s.pmax;
        s.sampled = true; s.order = *(const int *) (w + SW_ORDER);
        // widen the sampled range a little: keys outside it still map (they just wrap)
        const double range = (double) s.hi - (double) s.lo + 1.0, pad = range / 1024.0 + 64.0, lo_d = (double) s.lo - pad, range_d = range + 2 * pad;
        if (s.hi > s.lo && (range <= GX_INTERP_MAX_SPREAD * (double) nrows || j.sw.slot_mode == 1) && lo_d > -9.0e18 && lo_d + range_d < 9.0e18)
            gx_set_interpolation(j.h, (long long) lo_d, range_d, j.sw.wide);
    }
    s.sf = gx_hash_slotfn(j.h);
    return GX_OK;
}
// the key-ordered build's form: pk, the staged fill's loader (1: one 4-byte payload column, 2: row number, 0: generic);
// searched: bounds by search; compact: 8-byte slots; narrow: 4-byte slots instead of compact ones
struct sorted_form { int pk; bool searched, compact, narrow; };
// One key-ordered fill (the bounds pass's first with gx_k_sorted_special), then the scratch words read back.
// The second profile names tell the path, the form and `why`: the narrow form, or the refill that replaced it.
static int sorted_fill_pass(build_job &j, const gx_bbuild_args &ba, const sorted_form &f, int pk, const char *why, bool refill)
{
    gx_ctx *ctx = j.ctx; const bool special = !refill && !f.searched;
    if (refill) GX_CUDA(ctx, clear_scratch(ctx, SW_PLACED, SW_OVERFLOW));
    {
        gx_launch_scope ls(ctx, "build", special ? 2 : 1);
        gx_launch_scope path(ctx, f.searched ? "build_sorted_search" : "build_sorted_pass", 0);
        gx_launch_scope form(ctx, f.compact ? "build_compact" : nullptr, 0);
        gx_launch_scope nform(ctx, why, 0);
        if (special) gx_k_sorted_special<<<1, 256, 0, ctx->stream>>>(ba.b, ba.start, ba.unsorted);
        if (f.narrow) { if (f.searched) sorted_fill<GX_SLOTS_NARROW, true>(ctx, ba, pk); else sorted_fill<GX_SLOTS_NARROW, false>(ctx, ba, pk); }
        else if (f.compact) { if (f.searched) sorted_fill<GX_SLOTS_COMPACT, true>(ctx, ba, pk); else sorted_fill<GX_SLOTS_COMPACT, false>(ctx, ba, pk); }
        else if (f.searched) sorted_fill<GX_SLOTS_WIDE, true>(ctx, ba, pk);
        else sorted_fill<GX_SLOTS_WIDE, false>(ctx, ba, pk);
    }
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(ctx->h_scratch, ctx->d_scratch, (SW_OVERFLOW + 1) * sizeof(long long), cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) { GX_SET_ERR(ctx, "hash_build: %s", cudaGetErrorString(e)); return GX_ERR_CUDA; }
    return GX_OK;
}
// a bounded wait of the staged fill gave up: the same build with the generic row loader
static int staged_fallback(build_job &j, const gx_bbuild_args &ba, const sorted_form &f, const char *why)
{
    if (f.pk == 0 || !((int) j.ctx->h_scratch[SW_OVERFLOW] & OVF_STUCK)) return GX_OK;
    fprintf(stderr, "gpuexec: a bounded mbarrier wait of gx_k_sorted_fill_staged gave up; rebuilding with gx_k_sorted_fill\n");
    return sorted_fill_pass(j, ba, f, 0, why, true);
}
// a payload outside the narrow window (a value the sample missed): the same build in the 8-byte form
static int narrow_refill(build_job &j, gx_bbuild_args &ba, sorted_form &f)
{
    gx_hash *h = j.h; gx_tmp_free(j.ctx, h->narrow); h->narrow = nullptr; f.narrow = false; h->tbits = 0; h->pbase = 0;
    if (gx_tmp_alloc(j.ctx, (void **) &h->cslots, (size_t) h->nslots * sizeof(gx_cslot)) != cudaSuccess)
        { h->cslots = nullptr; GX_SET_ERR(j.ctx, "hash_build: cudaMalloc of %lld compact slots failed", (long long) h->nslots); return GX_ERR_NOMEM; }
    j.a.sf = gx_hash_slotfn(h); ba.b = j.a; ba.cslots = h->cslots; ba.narrow = nullptr;
    int rc = sorted_fill_pass(j, ba, f, f.pk, "build_narrow_refill", true);
    return rc ? rc : staged_fallback(j, ba, f, "build_narrow_refill");
}
// Key-ordered build side: no bucketing, a sub-table's rows are one row range.  Not tried (UNORDERED, h unchanged) when the
// key span is too wide; unless BUILT, h is left in 16-byte slots.
enum sorted_outcome { SORTED_BUILT, SORTED_CLUSTERED, SORTED_UNORDERED };
static int sorted_build(build_job &j, key_sample &ks, sorted_outcome &out, long long &nplaced)
{
    gx_ctx *ctx = j.ctx; gx_hash *h = j.h; const gx_build_args &a = j.a; const long long *w = ctx->h_scratch; out = SORTED_UNORDERED;
    GX_CUDA(ctx, clear_scratch(ctx, SW_UNSORTED, SW_OVERFLOW));
    if (!ks.have_ends) { int rc = fetch_key_ends(j, ks); if (rc) return rc; }
    const long long kmin = ks.first == GX_EMPTY_KEY ? ks.first + 1 : ks.first, kmax = ks.last;      // the reserved key lives in the side list
    const double range_d = (double) kmax - (double) kmin + 1.0;
    const long long nsub = h->nslots / GX_SUB;
    tmp_buf<long long> start(ctx);
    if (!(range_d >= 1.0 && range_d < 9.0e18 && range_d <= GX_INTERP_MAX_SPREAD * (double) a.nrows && start.alloc(nsub + 1) == cudaSuccess)) return GX_OK;
    // exact bounds (if the column really is ordered): every key maps below nslots - GX_SUB, monotonically
    gx_set_interpolation(h, kmin, range_d, j.sw.wide);
    GX_CUDA(ctx, clear_scratch(ctx, SW_INSERTED, SW_SPECIAL));
    GX_CUDA(ctx, clear_scratch(ctx, SW_PLACED, SW_STEPS));
    const bool i8 = a.key.type == GX_INT8 && a.key.nulls == nullptr, pay4 = a.n_payload == 1 && (a.payload[0].type == GX_INT4 || a.payload[0].type == GX_DATE);
    sorted_form f = { i8 && a.npreds == 0 ? (a.n_payload == 0 ? 2 : pay4 ? 1 : 0) : 0, false, false, false };
    // int8 key without NULLs whose first key is an ordinary key: bounds by search, order and
    // placement verified by the fill (see sorted_lower_bound)
    f.searched = i8 && ks.first != GX_EMPTY_KEY && ((uintptr_t) a.key.data & 15) == 0 && !j.sw.nosearch;
    // compact 8-byte slots when the exact key span and the payload fit 32 bits each (a sub-table's keys must be told
    // apart by 31 bits: its key span is range / #sub-tables)
    const bool small_payload = a.n_payload == 0 ? a.nrows < 0xffffffffLL : j.payload_bytes <= 4;
    const double keys_per_slot = range_d / (double) (h->nslots - GX_SUB);
    f.compact = (f.pk != 0 || f.searched) && small_payload && h->mode != 0 && keys_per_slot * GX_SUB < 268435456.0 && !j.sw.nocompact;
    // narrow 4-byte slots (pk 1) when the tag the key span needs leaves room for the sampled payload range, which
    // is centred in the window; a payload the sample missed is caught by the fill (OVF_PAYLOAD)
    if (f.compact && f.pk == 1 && ks.have_prange) {
        const unsigned int tbits = gx_nslot_tbits(keys_per_slot);
        const long long pwin = tbits < 32 ? 1LL << (32 - tbits) : 0;         // payload values a slot holds
        if (ks.pmax - ks.pmin < pwin) {
            long long pb = ks.pmin - (pwin - 1 - (ks.pmax - ks.pmin)) / 2;
            if (pb < (long long) INT32_MIN) pb = INT32_MIN;                     // the window stays inside int4
            if (pb > (long long) INT32_MAX - (pwin - 1)) pb = (long long) INT32_MAX - (pwin - 1);
            f.narrow = true; h->tbits = tbits; h->pbase = (int) pb;
        }
    }
    h->keys_per_slot = keys_per_slot;
    if (f.narrow && gx_tmp_alloc(ctx, (void **) &h->narrow, (size_t) h->nslots * sizeof(unsigned int)) != cudaSuccess) { h->narrow = nullptr; f.narrow = false; }
    if (!f.narrow) { h->tbits = 0; h->pbase = 0; }
    if (f.compact && !f.narrow && gx_tmp_alloc(ctx, (void **) &h->cslots, (size_t) h->nslots * sizeof(gx_cslot)) != cudaSuccess) { h->cslots = nullptr; f.compact = false; }
    h->amask = f.compact ? 3u : 1u; h->cspan = f.compact ? (unsigned long long) (kmax - kmin) + 1ULL : 0ULL;
    // the staged fill copies 16-byte aligned blocks of the key and payload columns
    if (f.pk != 0 && (((uintptr_t) a.key.data & 15) != 0 || (f.pk == 1 && ((uintptr_t) a.payload[0].data & 15) != 0))) f.pk = 0;
    j.a.sf = gx_hash_slotfn(h);
    gx_bbuild_args ba; memset(&ba, 0, sizeof(ba));
    ba.b = a; ba.nsub = nsub; ba.start = start.p; ba.cslots = h->cslots; ba.narrow = h->narrow;
    ba.unsorted = (int *) (ctx->d_scratch + SW_UNSORTED); ba.overflow = (int *) (ctx->d_scratch + SW_OVERFLOW);
    {
        gx_launch_scope ls(ctx, "build_bounds");
        const long long *keys = (const long long *) a.key.data;
        if (f.searched) gx_k_sorted_bounds_search<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(keys, a.nrows, a.sf, nsub, h->nslots, ba.start);
        else if (a.key.type == GX_INT8 && a.key.nulls == nullptr && ((uintptr_t) keys & 15) == 0) gx_k_sorted_bounds_i8<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(keys, a.nrows, a.sf, nsub, ba.start, ba.unsorted);
        else gx_k_sorted_bounds<<<ctx->sm_count * 16, 256, 0, ctx->stream>>>(a, nsub, ba.start, ba.unsorted);
    }
    const char *why = f.narrow ? "build_narrow" : nullptr;
    int rc = sorted_fill_pass(j, ba, f, f.pk, why, false);
    if (!rc) rc = staged_fallback(j, ba, f, why);
    if (!rc && f.narrow && ((int) w[SW_OVERFLOW] & OVF_PAYLOAD) && (int) w[SW_UNSORTED] == 0) rc = narrow_refill(j, ba, f);
    if (rc) return rc;
    if ((int) w[SW_UNSORTED] == 0) {
        h->avg_chain = fill_avg_chain(w);
        if (((int) w[SW_OVERFLOW] & ~OVF_PAYLOAD) == 0 && h->avg_chain <= 4.0) {     // OVF_PAYLOAD was answered by narrow_refill
            nplaced = w[SW_PLACED]; h->sorted_build = 1; out = SORTED_BUILT;
            if (f.compact) { gx_tmp_free(ctx, h->slots); h->slots = nullptr; }      // the 16-byte form is made on demand (gx_hash_wide)
            return GX_OK;
        }
        out = SORTED_CLUSTERED;
    }
    gx_tmp_free(ctx, h->cslots); gx_tmp_free(ctx, h->narrow); h->cslots = nullptr; h->narrow = nullptr; h->amask = 1u; h->cspan = 0; h->tbits = 0; h->pbase = 0;
    return GX_OK;
}

// Bucketed build (two-level scatter for 2^12 .. 2^18 sub-tables).  REHASH: interpolation overflowed a sub-table or made long
// chains (keys less uniform than sampled); OVERFLOW: the mixing hash did.
enum bucket_outcome { BUCKET_BUILT, BUCKET_REHASH, BUCKET_OVERFLOW };
static int bucketed_build(build_job &j, bucket_outcome &out, long long &nplaced)
{
    gx_ctx *ctx = j.ctx; gx_hash *h = j.h; const long long nrows = j.inner->nrows;
    GX_CUDA(ctx, clear_scratch(ctx, SW_INSERTED, SW_SPECIAL));
    j.a.sf = gx_hash_slotfn(h);
    gx_bbuild_args ba; memset(&ba, 0, sizeof(ba)); ba.b = j.a; ba.nsub = h->nslots / GX_SUB;
    tmp_buf<unsigned int> cursor(ctx); tmp_buf<gx_slot> pairs(ctx);
    cudaError_t e = cursor.alloc(ba.nsub + 1);                      // the last word is the overflow flag
    if (e == cudaSuccess) e = pairs.alloc(h->nslots);
    if (e != cudaSuccess) { GX_SET_ERR(ctx, "hash_build: cudaMalloc of the bucketing buffers failed: %s", cudaGetErrorString(e)); return GX_ERR_NOMEM; }
    ba.cursor = cursor.p; ba.pairs = pairs.p; ba.overflow = (int *) (ba.cursor + ba.nsub);
    GX_CUDA(ctx, cudaMemsetAsync(ba.cursor, 0, (size_t) ba.nsub * sizeof(unsigned int) + sizeof(int), ctx->stream));
    GX_CUDA(ctx, clear_scratch(ctx, SW_PLACED, SW_STEPS));
    long long ntiles = (nrows + 256 * BSCAT - 1) / (256 * BSCAT), maxb = (long long) ctx->sm_count * 8;
    unsigned grid = (unsigned) (ntiles < maxb ? ntiles : maxb);
    int log2nsub = 0; while (((long long) 1 << log2nsub) < ba.nsub) log2nsub++;
    bool two_level = log2nsub >= 12 && log2nsub <= 18 && !j.sw.onepass;
    if (two_level) {
        gx_bpart_args pa; memset(&pa, 0, sizeof(pa));
        pa.b = ba.b; pa.nsub = ba.nsub; pa.bits_hi = (log2nsub + 1) / 2; pa.bits_lo = log2nsub - pa.bits_hi;
        pa.pairs = ba.pairs; pa.cursor = ba.cursor; pa.overflow = ba.overflow;
        const long long B1 = (long long) 1 << pa.bits_hi;
        pa.cap1 = (nrows / B1) + (nrows / B1) / 4 + 2 * BP_TILE; pa.tiles_per_l1 = (pa.cap1 + BP_TILE - 1) / BP_TILE;
        tmp_buf<gx_slot> l1(ctx); tmp_buf<unsigned int> cur1(ctx);
        e = l1.alloc((size_t) B1 * pa.cap1); if (e == cudaSuccess) e = cur1.alloc((size_t) B1);
        if (e == cudaSuccess) {
            pa.l1 = l1.p; pa.cur1 = cur1.p;
            GX_CUDA(ctx, cudaMemsetAsync(pa.cur1, 0, (size_t) B1 * sizeof(unsigned int), ctx->stream));
            static bool attr = false;
            if (!attr) { cudaFuncSetAttribute(gx_k_bpart1, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) bp_smem_bytes(512));
                         cudaFuncSetAttribute(gx_k_bpart2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) bp_smem_bytes(512)); attr = true; }
            gx_launch_scope ls(ctx, "build_scatter", 2);
            gx_launch_scope which(ctx, "build_bucket2", 0);
            gx_k_bpart1<<<ctx->sm_count * 2, BP_THREADS, bp_smem_bytes(1 << pa.bits_hi), ctx->stream>>>(pa);
            gx_k_bpart2<<<ctx->sm_count * 2, BP_THREADS, bp_smem_bytes(1 << pa.bits_lo), ctx->stream>>>(pa);
        } else two_level = false;                                   // no room for the level-1 buffer: one-pass scatter
    }
    if (!two_level) {
        gx_launch_scope ls(ctx, "build_scatter");
        gx_launch_scope which(ctx, "build_bucket1", 0);
        gx_k_bbuild_scatter<<<grid, 256, 0, ctx->stream>>>(ba);
    }
    {
        static bool attr = false;
        if (!attr) { cudaFuncSetAttribute(gx_k_bbuild_fill, cudaFuncAttributeMaxDynamicSharedMemorySize, FILL_SMEM_BYTES); attr = true; }
        gx_launch_scope ls(ctx, "build", 2);
        gx_k_bbuild_fill<<<ctx->sm_count * 8, FILL_THREADS, FILL_SMEM_BYTES, ctx->stream>>>(ba);
        gx_k_bbuild_total<<<ctx->sm_count, 256, 0, ctx->stream>>>(ba.cursor, ba.nsub, ctx->d_scratch + SW_PLACED);
    }
    int h_over = 0; e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(ctx->h_scratch + SW_PLACED, ctx->d_scratch + SW_PLACED, (SW_STEPS - SW_PLACED + 1) * sizeof(long long), cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(&h_over, ba.overflow, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) { GX_SET_ERR(ctx, "hash_build: %s", cudaGetErrorString(e)); return GX_ERR_CUDA; }
    h->avg_chain = fill_avg_chain(ctx->h_scratch);
    if (h->mode != 0 && (h_over || h->avg_chain > 4.0)) out = BUCKET_REHASH;
    else if (h_over) out = BUCKET_OVERFLOW;
    else { out = BUCKET_BUILT; nplaced = ctx->h_scratch[SW_PLACED]; }
    return GX_OK;
}

// Direct build: CAS insertion into the cleared table
static int direct_build(build_job &j)
{
    gx_ctx *ctx = j.ctx; gx_hash *h = j.h; gx_build_args &a = j.a;
    GX_CUDA(ctx, clear_scratch(ctx, SW_INSERTED, SW_SPECIAL));
    { gx_launch_scope ls(ctx, "build_clear"); gx_k_fill_slots<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(h->slots, h->nslots); }
    // probe walks wrap inside a sub-table (or the whole table when it is smaller): each keeps a free slot
    const long long wrap = h->nslots < GX_SUB ? h->nslots : GX_SUB, nsub = h->nslots / wrap;
    tmp_buf<unsigned int> claims(ctx); GX_CUDA(ctx, claims.alloc(nsub + 1));
    GX_CUDA(ctx, cudaMemsetAsync(claims.p, 0, (size_t) (nsub + 1) * sizeof(unsigned int), ctx->stream));
    a.sf = gx_hash_slotfn(h); a.sub_claims = claims.p; a.sub_limit = (unsigned int) (wrap - 1); a.sub_over = claims.p + nsub;
    unsigned int h_sub_over = 0; cudaError_t e;
    {
        gx_launch_scope ls(ctx, "build");
        gx_launch_scope which(ctx, "build_direct", 0);
        const long long nb = (a.nrows + 255) / 256, maxb = (long long) ctx->sm_count * 8;
        gx_k_hash_build<<<(unsigned) (nb < maxb ? nb : maxb), 256, 0, ctx->stream>>>(a);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(&h_sub_over, a.sub_over, sizeof(unsigned int), cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) { GX_SET_ERR(ctx, "hash_build: %s", cudaGetErrorString(e)); return GX_ERR_CUDA; }
    if (h_sub_over) {
        GX_SET_ERR(ctx, "hash_build: %u build rows hash into one %lld-slot sub-table of the join table, which holds at most %lld "
                   "(a build key repeated that often, or keys that collide under the table's hash)", h_sub_over, wrap, wrap - 1);
        return GX_ERR_ARG;
    }
    return GX_OK;
}

// The table from the sample on: slots, fill, entry count and side list
static int build_fill(build_job &j, key_sample &ks)
{
    gx_ctx *ctx = j.ctx; const gx_table *inner = j.inner; gx_hash *h = j.h; long long *w = ctx->h_scratch;
    int rc = alloc_table(j); if (rc) return rc;
    GX_CUDA(ctx, clear_scratch(ctx, SW_INSERTED, SW_SPECIAL));
    long long nplaced = -1;                                         // entries a fill placed (key-ordered or bucketed build)
    if (inner->nrows == 0) { gx_launch_scope ls(ctx, "build_clear"); gx_k_fill_slots<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(h->slots, h->nslots); }
    else {
        bool direct = h->nslots < 64 * GX_SUB || j.sw.direct;      // big tables: bucket by sub-table, build each in shared memory
        sorted_outcome so = SORTED_UNORDERED;
        if (!direct && h->mode != 0 && !j.sw.nosorted) {
            rc = sorted_build(j, ks, so, nplaced); if (rc) return rc;
            if (so == SORTED_CLUSTERED) h->mode = 0;               // clustered keys: the mixing hash
            else if (so == SORTED_UNORDERED) set_slotfn(h, ks.sf);  // not in key order: back to the sampled slot function
        }
        if (!direct && so != SORTED_BUILT) {
            bucket_outcome bo; rc = bucketed_build(j, bo, nplaced); if (rc) return rc;
            if (bo == BUCKET_REHASH) { h->mode = 0; rc = bucketed_build(j, bo, nplaced); if (rc) return rc; }
            direct = bo == BUCKET_OVERFLOW;
        }
        if (direct) { rc = direct_build(j); if (rc) return rc; }
    }
    // the entry count and the side list (the key-ordered build read them with its fill's counters)
    GX_CUDA(ctx, cudaGetLastError());
    if (!h->sorted_build) {
        GX_CUDA(ctx, cudaMemcpyAsync(w, ctx->d_scratch, 2 * sizeof(long long), cudaMemcpyDeviceToHost, ctx->stream));
        GX_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    if (nplaced >= 0) w[SW_INSERTED] = nplaced;
    h->nentries = w[SW_INSERTED] + w[SW_SPECIAL];
    h->special_count = (int) w[SW_SPECIAL];
    GX_CHECK_ARG(ctx, h->special_count <= h->special_cap, "hash_build: %d rows carry key INT64_MIN (side list holds %d)", h->special_count, h->special_cap);
    return GX_OK;
}

// What a deferred build keeps for its fill: the build as gx_hash_build set it up and sampled it
struct gx_deferred { gx_build_args a; int payload_bytes; build_switches sw; key_sample ks; };

// Defer the fill?  A key-ordered merge (gx_agg.cu, gx_k_mergejoin) can then read the build rows themselves instead of a table
// written once and read once.  Only the staged narrow build's shape (unique int8 key without NULLs, one int4/date payload, no
// quals, 16-byte aligned columns) over strictly ascending sampled keys, and only when even its narrowest table (4-byte
// slots) is larger than L2: a smaller table stays in L2 between the fill and the probe, and every other reader fills it
// anyway.
static bool defer_fill(const build_job &j, const key_sample &ks)
{
    const gx_build_args &a = j.a; const gx_hash *h = j.h;
    return ks.sampled && ks.order == 0 && h->unique && a.key.type == GX_INT8 && a.key.nulls == nullptr && a.npreds == 0 &&
           a.n_payload == 1 && (a.payload[0].type == GX_INT4 || a.payload[0].type == GX_DATE) &&
           ((uintptr_t) a.key.data & 15) == 0 && ((uintptr_t) a.payload[0].data & 15) == 0 &&
           (size_t) h->nslots * sizeof(unsigned int) > j.ctx->l2_bytes && !j.sw.direct && !j.sw.nosorted;
}

extern "C" int gx_hash_build(gx_ctx *ctx, const gx_table *inner, int key_col, int n_preds, const gx_pred *preds,
                             int n_payload, const int32_t *payload_cols, int unique, gx_hash **out)
{
    if (!ctx || !inner || !out) return GX_ERR_ARG;
    build_job j(ctx, inner, key_col);
    int rc = build_setup(j, n_preds, preds, n_payload, payload_cols, unique); if (rc) return rc;
    key_sample ks; rc = sample_keys(j, ks); if (rc) return rc;
    gx_hash *h = j.h;
    if (defer_fill(j, ks)) {
        h->deferred = new gx_deferred{ j.a, j.payload_bytes, j.sw, ks };
        h->bkey = (const long long *) j.a.key.data; h->bpay = (const int *) j.a.payload[0].data; h->nbuild = inner->nrows;
        gx_table *src = const_cast<gx_table *>(inner);
        h->next_deferred = src->deferred; src->deferred = h;
    } else {
        rc = build_fill(j, ks); if (rc) return rc;
    }
    *out = h; j.h = nullptr;
    return GX_OK;
}

static void unlink_deferred(gx_hash *h)
{
    gx_table *src = const_cast<gx_table *>(h->src);
    if (!src) return;                               // its table is gone (gx_table_settle): nothing links to it
    for (gx_hash **p = &src->deferred; *p; p = &(*p)->next_deferred)
        if (*p == h) { *p = h->next_deferred; break; }
    h->next_deferred = nullptr;
}
// the buffers and statistics of a fill, back to what the sample left
static void drop_fill(gx_hash *h)
{
    gx_tmp_free(h->ctx, h->slots); gx_tmp_free(h->ctx, h->cslots); gx_tmp_free(h->ctx, h->narrow); gx_tmp_free(h->ctx, h->special_payload);
    h->slots = nullptr; h->cslots = nullptr; h->narrow = nullptr; h->special_payload = nullptr;
    h->nentries = 0; h->special_count = 0; h->avg_chain = 0.0; h->sorted_build = 0; h->cspan = 0; h->keys_per_slot = 0.0;
}
int hash_materialize(gx_hash *h)
{
    if (!h->deferred) return GX_OK;
    if (h->nbuild < 0) { GX_SET_ERR(h->ctx, "join table: its build table was freed before the deferred fill could run"); return GX_ERR_STATE; }
    gx_deferred *d = h->deferred;
    build_job j(h->ctx, h->src, 0);
    j.a = d->a; j.payload_bytes = d->payload_bytes; j.sw = d->sw; j.h = h;
    set_slotfn(h, d->ks.sf);
    key_sample ks = d->ks;
    const int rc = build_fill(j, ks);
    j.h = nullptr;                                  // the caller's handle: never freed here
    if (rc) { drop_fill(h); set_slotfn(h, d->ks.sf); return rc; }     // still deferred: a later call tries again
    unlink_deferred(h);
    delete d; h->deferred = nullptr;
    return GX_OK;
}
int gx_table_settle(gx_table *t, bool freeing)
{
    while (t->deferred) {
        gx_hash *h = t->deferred;
        const int rc = hash_materialize(h);
        if (rc && !freeing) return rc;
        if (rc) { unlink_deferred(h); h->nbuild = -1; h->src = nullptr; }      // its rows are gone: every later use reports the failure
    }
    return GX_OK;
}
// a strided sample of 64 K keys, as the build's
int gx_sample_order(gx_ctx *ctx, const long long *keys, long long nrows, int *order)
{
    long long stride = nrows / 65536; if (stride < 1) stride = 1;
    const long long nthreads = (nrows + stride - 1) / stride;
    int *d_order = (int *) (ctx->d_scratch + SW_ORDER);
    gx_dcol key; memset(&key, 0, sizeof(key)); key.data = keys; key.type = GX_INT8;
    gx_dcol pay; memset(&pay, 0, sizeof(pay));
    GX_CUDA(ctx, cudaMemsetAsync(d_order, 0, sizeof(long long), ctx->stream));
    { gx_launch_scope ls(ctx, "agg_sample"); gx_k_key_range<<<(unsigned) ((nthreads + 255) / 256), 256, 0, ctx->stream>>>(key, pay, nrows, stride, nullptr, nullptr, d_order); }
    GX_CUDA(ctx, cudaGetLastError());
    GX_CUDA(ctx, cudaMemcpyAsync(ctx->h_scratch + SW_ORDER, d_order, sizeof(long long), cudaMemcpyDeviceToHost, ctx->stream));
    GX_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    *order = *(const int *) (ctx->h_scratch + SW_ORDER);
    return GX_OK;
}

// compact or narrow table -> 16-byte slots, for the consumers that only read that form.  The full key is rebuilt from
// its stored tag bits and the slot's position (gx_tag_key): the interpolation maps slot i back to key offset
// ~ i * keys_per_slot, and the entry's home lies in the same sub-table.
template <int F>
__global__ void gx_k_expand_slots(const void *c, gx_slot *w, long long nslots, gx_slotfn f, double keys_per_slot)
{
    long long stride = (long long) gridDim.x * blockDim.x;
    for (long long i = (long long) blockIdx.x * blockDim.x + threadIdx.x; i < nslots; i += stride) {
        longlong2 o;
        o.x = GX_EMPTY_KEY; o.y = 0;
        if (F == GX_SLOTS_NARROW) {
            const unsigned int v = ((const unsigned int *) c)[i];
            if (v) {
                o.x = gx_tag_key(i, (v & ((1u << f.tbits) - 1u)) >> 1, (int) f.tbits - 1, f.kmin, keys_per_slot);
                o.y = (long long) (unsigned long long) (unsigned int) gx_nslot_payload(v, f);
            }
        } else {
            const gx_cslot v = ((const gx_cslot *) c)[i];
            if (v.d) { o.x = gx_tag_key(i, v.d >> 1, 31, f.kmin, keys_per_slot); o.y = (long long) (unsigned long long) v.payload; }
        }
        ((longlong2 *) w)[i] = o;
    }
}
int gx_hash_wide(gx_ctx *ctx, gx_hash *h)
{
    int rc = hash_materialize(h); if (rc) return rc;
    if (h->slots || (!h->cslots && !h->narrow)) return GX_OK;
    cudaError_t e = gx_tmp_alloc(ctx, (void **) &h->slots, (size_t) h->nslots * sizeof(gx_slot));
    if (e != cudaSuccess) { h->slots = nullptr; GX_SET_ERR(ctx, "hash table: cudaMalloc of %lld slots failed: %s", (long long) h->nslots, cudaGetErrorString(e)); return GX_ERR_NOMEM; }
    gx_launch_scope ls(ctx, "build_expand");
    if (h->narrow) gx_k_expand_slots<GX_SLOTS_NARROW><<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(h->narrow, h->slots, h->nslots, gx_hash_slotfn(h), h->keys_per_slot);
    else gx_k_expand_slots<GX_SLOTS_COMPACT><<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(h->cslots, h->slots, h->nslots, gx_hash_slotfn(h), h->keys_per_slot);
    GX_CUDA(ctx, cudaGetLastError());
    return GX_OK;
}

// the statistics describe the filled table: a deferred one is filled first (a failure: -1 / the error, gx_last_error says why)
extern "C" int64_t gx_hash_nentries(const gx_hash *h) { return h && hash_materialize(const_cast<gx_hash *>(h)) == GX_OK ? h->nentries : -1; }
extern "C" int64_t gx_hash_nslots(const gx_hash *h) { return h && hash_materialize(const_cast<gx_hash *>(h)) == GX_OK ? h->nslots : -1; }
extern "C" int gx_hash_info(const gx_hash *h, int *slot_mode, double *avg_chain)
{
    if (!h) return GX_ERR_ARG;
    int rc = hash_materialize(const_cast<gx_hash *>(h)); if (rc) return rc;
    if (slot_mode) *slot_mode = h->sorted_build ? 2 : (h->mode != 0 ? 1 : 0);
    if (avg_chain) *avg_chain = h->avg_chain;
    return GX_OK;
}
extern "C" void gx_hash_free(gx_hash *h)
{
    if (!h) return;
    if (h->deferred) { unlink_deferred(h); delete h->deferred; }
    gx_tmp_free(h->ctx, h->slots);
    gx_tmp_free(h->ctx, h->cslots);
    gx_tmp_free(h->ctx, h->narrow);
    gx_tmp_free(h->ctx, h->special_payload);
    free(h);
}

// ------------------------------------------------------------ K3 probe
struct gx_probe_args {
    gx_dcol key;
    int npreds, n_out_outer, n_payload, unique;
    gx_dpred preds[GX_MAX_PREDS];
    long long nrows;
    const gx_slot *slots; unsigned long long mask;
    const gx_cslot *cslots; unsigned long long cspan;       // compact 8-byte form (half the bytes: an L2-resident table more often)
    const unsigned int *narrow;                            // narrow 4-byte form (gx_nslot_*), same cspan
    const unsigned long long *special; int special_count; int _pad2; gx_slotfn sf;
    gx_dcol out_src[GX_MAX_COLS];
    void *out[GX_MAX_COLS];
    uint8_t *out_nulls[GX_MAX_COLS];
    int payload_types[GX_MAX_PAYLOAD];
    long long *cursor;             // global output cursor
    long long out_cap;
    int count_only; int join_type;  // GX_JOIN_*
};

__device__ __forceinline__ void emit_payload(const gx_probe_args &a, long long dst, unsigned long long payload, bool matched);
__device__ __forceinline__ void emit_row(const gx_probe_args &a, long long dst, long long r, unsigned long long payload, bool matched = true)
{
    for (int c = 0; c < a.n_out_outer; c++) {
        switch (a.out_src[c].type) {
            case GX_INT4: case GX_DATE: ((int *) a.out[c])[dst] = ((const int *) a.out_src[c].data)[r]; break;
            case GX_CHAR: ((signed char *) a.out[c])[dst] = ((const signed char *) a.out_src[c].data)[r]; break;
            default: ((long long *) a.out[c])[dst] = ((const long long *) a.out_src[c].data)[r]; break;
        }
        if (a.out_nulls[c]) a.out_nulls[c][dst] = a.out_src[c].nulls ? a.out_src[c].nulls[r] : 0;
    }
    emit_payload(a, dst, payload, matched);
}
__device__ __forceinline__ void emit_payload(const gx_probe_args &a, long long dst, unsigned long long payload, bool matched)
{
    if (a.join_type == GX_JOIN_SEMI || a.join_type == GX_JOIN_ANTI) return;      // the inner side is not part of the target list
    const int npo = a.n_payload ? a.n_payload : 1;
    if (a.join_type == GX_JOIN_LEFT)                                               // hj_NullInnerTupleSlot for an unmatched outer row
        for (int i = 0; i < npo; i++) if (a.out_nulls[a.n_out_outer + i]) a.out_nulls[a.n_out_outer + i][dst] = matched ? 0 : 1;
    if (!matched) payload = 0;
    if (a.n_payload == 0) { ((long long *) a.out[a.n_out_outer])[dst] = (long long) payload; return; }
    int shift = 0;
    for (int i = 0; i < a.n_payload; i++) {
        int t = a.payload_types[i]; void *o = a.out[a.n_out_outer + i];
        switch (t) {
            case GX_INT4: case GX_DATE: ((int *) o)[dst] = (int) (payload >> shift); shift += 32; break;
            case GX_CHAR: ((signed char *) o)[dst] = (signed char) (payload >> shift); shift += 8; break;
            default: ((long long *) o)[dst] = (long long) payload; shift += 64; break;
        }
    }
}

// One pass.  Each thread walks its row's probe sequence; matches are appended
// through a warp-aggregated cursor (join output order is unspecified in the
// reference as well).  count_only sizes the output for non-unique builds.
__global__ void __launch_bounds__(256) gx_k_hash_probe(gx_probe_args a)
{
    long long stride = (long long) gridDim.x * blockDim.x;
    long long nloop = (a.nrows + stride - 1) / stride;
    long long r = (long long) blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    for (long long it = 0; it < nloop; it++, r += stride) {
        bool ok = r < a.nrows && !gx_is_null(a.key, r);
        if (ok) {
#pragma unroll
            for (int p = 0; p < GX_MAX_PREDS; p++) if (p < a.npreds) ok = ok && gx_eval_pred(a.preds[p], r);
        }
        long long key = ok ? gx_load_int(a.key, r) : 0;
        // walk: the warp iterates until every lane has exhausted its chain
        unsigned long long s = gx_slot_index(key, a.sf);
        bool special = ok && key == GX_EMPTY_KEY;
        int sp_i = 0;
        bool active = ok;
        while (__any_sync(0xffffffffu, active)) {
            bool hit = false; unsigned long long payload = 0;
            if (active) {
                if (special) {
                    if (sp_i < a.special_count) { hit = true; payload = a.special[sp_i++]; if (a.unique) active = false; }
                    else active = false;
                } else {
                    gx_slot sl = a.slots[s];
                    if (sl.key == GX_EMPTY_KEY) active = false;
                    else {
                        if (sl.key == key) { hit = true; payload = sl.payload; if (a.unique) active = false; }
                        s = gx_next_slot(s, a.mask);
                    }
                }
            }
            unsigned int m = __ballot_sync(0xffffffffu, hit);
            if (m) {
                long long base = 0;
                if (lane == 0) base = (long long) atomicAdd((unsigned long long *) a.cursor, (unsigned long long) __popc(m));
                base = __shfl_sync(0xffffffffu, base, 0);
                if (hit && !a.count_only) {
                    long long dst = base + __popc(m & ((1u << lane) - 1));
                    if (dst < a.out_cap) emit_row(a, dst, r, payload);
                }
            }
        }
    }
}

// Unique build side (inner_unique, nodeHashjoin.c:859-861): at most one match per outer row.  A warp takes
// tiles of 4 x 32 rows: the four key loads and then the four home-pair loads (one 32-byte sector each) are in
// flight together, matches are numbered with ballots and the warp claims its output range with ONE atomic per
// tile; the surviving rows are copied column by column.
template <int F> __global__ void gx_k_hash_probe_unique(gx_probe_args a);
template <int F>
// no min-blocks on purpose: any value (even 1 or 4, which leave the occupancy as it is) changes ptxas' schedule
// of the independent loads this kernel keeps in flight
__global__ void __launch_bounds__(256) gx_k_hash_probe_unique(gx_probe_args a)
{
    const int lane = threadIdx.x & 31;
    const unsigned int lt = (1u << lane) - 1;
    const long long nwarp = ((long long) gridDim.x * blockDim.x) >> 5, wid = ((long long) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long tile = 32LL * PT_K;
    for (long long base = wid * tile; base < a.nrows; base += nwarp * tile) {
        long long r[PT_K], key[PT_K]; bool ok[PT_K], hit[PT_K], quals_ok[PT_K]; unsigned long long pay[PT_K];
#pragma unroll
        for (int j = 0; j < PT_K; j++) { r[j] = base + j * 32 + lane; quals_ok[j] = r[j] < a.nrows; }
        for (int p = 0; p < a.npreds; p++) {
#pragma unroll
            for (int j = 0; j < PT_K; j++) if (quals_ok[j]) quals_ok[j] = gx_eval_pred(a.preds[p], r[j]);
        }
#pragma unroll
        for (int j = 0; j < PT_K; j++) ok[j] = quals_ok[j] && !gx_is_null(a.key, r[j]);      // a NULL key never matches (hashStrict)
#pragma unroll
        for (int j = 0; j < PT_K; j++) key[j] = ok[j] ? gx_load_int(a.key, r[j]) : 0;
        gx_probe_first<F, PT_K>(a, ok, key, hit, pay);
        __syncwarp();
        // which rows produce output (nodeHashjoin.c:569-668): INNER/SEMI the matched ones, ANTI the unmatched ones
        // (HJ_FILL_OUTER_TUPLE without a match), LEFT all of them (unmatched with a NULL inner side)
        bool matched[PT_K];
#pragma unroll
        for (int j = 0; j < PT_K; j++) {
            matched[j] = hit[j];
            const bool scanned = quals_ok[j];                   // passed the scan quals (a NULL key included: it just never matches)
            if (a.join_type == GX_JOIN_ANTI) hit[j] = scanned && !matched[j];
            else if (a.join_type == GX_JOIN_LEFT) hit[j] = scanned;
        }
        unsigned int m[PT_K]; int total = 0;
#pragma unroll
        for (int j = 0; j < PT_K; j++) { m[j] = __ballot_sync(0xffffffffu, hit[j]); total += __popc(m[j]); }
        if (total == 0) continue;
        long long dst0 = 0;
        if (lane == 0) dst0 = (long long) atomicAdd((unsigned long long *) a.cursor, (unsigned long long) total);
        dst0 = __shfl_sync(0xffffffffu, dst0, 0);
        if (a.count_only) continue;
        // outer columns: column by column, the tile's loads in flight together; then the inner side
        long long dd[PT_K];
#pragma unroll
        for (int j = 0; j < PT_K; j++) { dd[j] = dst0 + __popc(m[j] & lt); hit[j] = hit[j] && dd[j] < a.out_cap; dst0 += __popc(m[j]); }
        for (int c = 0; c < a.n_out_outer; c++) gx_copy_rows<PT_K>(a.out_src[c], a.out[c], a.out_nulls[c], r, dd, hit);
        if (a.join_type != GX_JOIN_SEMI && a.join_type != GX_JOIN_ANTI) {
#pragma unroll
            for (int j = 0; j < PT_K; j++) if (hit[j]) emit_payload(a, dd[j], pay[j], matched[j]);
        }
    }
}

extern "C" int gx_hash_probe_ex(gx_ctx *ctx, const gx_table *outer, int key_col, int n_preds, const gx_pred *preds,
                                const gx_hash *h, int join_type, int n_out_outer, const int32_t *out_outer_cols, gx_table **out);
extern "C" int gx_hash_probe(gx_ctx *ctx, const gx_table *outer, int key_col, int n_preds, const gx_pred *preds,
                             const gx_hash *h, int n_out_outer, const int32_t *out_outer_cols, gx_table **out)
{
    return gx_hash_probe_ex(ctx, outer, key_col, n_preds, preds, h, GX_JOIN_INNER, n_out_outer, out_outer_cols, out);
}
extern "C" int gx_hash_probe_ex(gx_ctx *ctx, const gx_table *outer, int key_col, int n_preds, const gx_pred *preds,
                                const gx_hash *h, int join_type, int n_out_outer, const int32_t *out_outer_cols, gx_table **out)
{
    if (!ctx || !outer || !h || !out) return GX_ERR_ARG;
    int rc = hash_materialize(const_cast<gx_hash *>(h)); if (rc) return rc;
    GX_CHECK_ARG(ctx, key_col >= 0 && key_col < outer->ncols, "hash_probe: key column %d out of range", key_col);
    int kt = outer->types[key_col];
    GX_CHECK_ARG(ctx, kt == GX_INT4 || kt == GX_INT8 || kt == GX_DATE, "hash_probe: key type %d not supported", kt);
    GX_CHECK_ARG(ctx, join_type == GX_JOIN_INNER || join_type == GX_JOIN_LEFT || join_type == GX_JOIN_SEMI || join_type == GX_JOIN_ANTI,
                 "hash_probe: join type %d not supported (inner, left, semi, anti)", join_type);
    GX_CHECK_ARG(ctx, join_type != GX_JOIN_LEFT || h->unique, "hash_probe: LEFT JOIN needs a unique build side (inner_unique)");
    const bool no_inner_cols = join_type == GX_JOIN_SEMI || join_type == GX_JOIN_ANTI;
    int n_pay_out = no_inner_cols ? 0 : (h->n_payload ? h->n_payload : 1);
    GX_CHECK_ARG(ctx, n_out_outer >= 0 && n_out_outer + n_pay_out <= GX_MAX_COLS && n_out_outer + n_pay_out > 0, "hash_probe: bad output column count");
    gx_probe_args a; memset(&a, 0, sizeof(a));
    a.key.data = outer->cols[key_col]; a.key.nulls = outer->nulls[key_col]; a.key.type = kt;
    a.npreds = n_preds; a.n_out_outer = n_out_outer; a.n_payload = h->n_payload; a.unique = h->unique; a.join_type = join_type;
    const bool first_match_only_c = h->unique || join_type != GX_JOIN_INNER;
    const bool use_compact = (h->cslots != nullptr || h->narrow != nullptr) && first_match_only_c;   // 8- and 4-byte slots are probed as they are
    if (!use_compact) { int wrc = gx_hash_wide(ctx, const_cast<gx_hash *>(h)); if (wrc) return wrc; }
    a.nrows = outer->nrows; a.slots = h->slots; a.mask = (unsigned long long) h->nslots - 1;
    a.cslots = h->cslots; a.narrow = h->narrow; a.cspan = h->cspan;
    a.special = h->special_payload; a.special_count = h->special_count;
    a.sf = gx_hash_slotfn(h);
    rc = gx_fill_dpreds(ctx, outer, n_preds, preds, a.preds); if (rc) return rc;
    int32_t types[GX_MAX_COLS]; bool hn[GX_MAX_COLS];
    for (int c = 0; c < n_out_outer; c++) {
        int oc = out_outer_cols[c];
        GX_CHECK_ARG(ctx, oc >= 0 && oc < outer->ncols, "hash_probe: output column %d out of range", oc);
        a.out_src[c].data = outer->cols[oc]; a.out_src[c].nulls = outer->nulls[oc]; a.out_src[c].type = outer->types[oc];
        types[c] = outer->types[oc]; hn[c] = outer->nulls[oc] != nullptr;
    }
    const bool left = join_type == GX_JOIN_LEFT;
    if (!no_inner_cols && h->n_payload == 0) { types[n_out_outer] = GX_INT8; hn[n_out_outer] = left; }
    for (int i = 0; i < h->n_payload; i++) { if (!no_inner_cols) { types[n_out_outer + i] = h->payload_types[i]; hn[n_out_outer + i] = left; } a.payload_types[i] = h->payload_types[i]; }
    a.cursor = ctx->d_scratch + 2;
    long long nb = (outer->nrows + 255) / 256, maxb = (long long) ctx->sm_count * 8;
    unsigned grid = (unsigned) (nb < maxb ? (nb > 0 ? nb : 1) : maxb);
    long long out_cap = outer->nrows;
    const bool first_match_only = h->unique || join_type != GX_JOIN_INNER;      // semi/anti stop at the first match
    if (!first_match_only) {
        // size the output first
        a.count_only = 1; a.out_cap = 0;
        GX_CUDA(ctx, cudaMemsetAsync(a.cursor, 0, sizeof(long long), ctx->stream));
        { gx_launch_scope ls(ctx, "probe_count"); gx_k_hash_probe<<<grid, 256, 0, ctx->stream>>>(a); }
        GX_CUDA(ctx, cudaMemcpyAsync(ctx->h_scratch, a.cursor, sizeof(long long), cudaMemcpyDeviceToHost, ctx->stream));
        GX_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        out_cap = ctx->h_scratch[0];
    }
    gx_table *t;
    rc = gx_table_alloc_like(ctx, n_out_outer + n_pay_out, types, hn, out_cap, &t); if (rc) return rc;
    for (int c = 0; c < t->ncols; c++) { a.out[c] = t->cols[c]; a.out_nulls[c] = t->nulls[c]; }
    a.count_only = 0; a.out_cap = out_cap;
    GX_CUDA(ctx, cudaMemsetAsync(a.cursor, 0, sizeof(long long), ctx->stream));
    {
        gx_launch_scope ls(ctx, "probe");
        if (first_match_only) {
            long long nt = (outer->nrows + 32 * PT_K * 8 - 1) / (32 * PT_K * 8);
            const unsigned pgrid = (unsigned) (nt < maxb ? (nt > 0 ? nt : 1) : maxb);
            if (use_compact && h->narrow) gx_k_hash_probe_unique<GX_SLOTS_NARROW><<<pgrid, 256, 0, ctx->stream>>>(a);
            else if (use_compact) gx_k_hash_probe_unique<GX_SLOTS_COMPACT><<<pgrid, 256, 0, ctx->stream>>>(a);
            else gx_k_hash_probe_unique<GX_SLOTS_WIDE><<<pgrid, 256, 0, ctx->stream>>>(a);
        } else gx_k_hash_probe<<<grid, 256, 0, ctx->stream>>>(a);
    }
    cudaError_t e = cudaMemcpyAsync(ctx->h_scratch, a.cursor, sizeof(long long), cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) { gx_table_free(t); GX_SET_ERR(ctx, "hash_probe: %s", cudaGetErrorString(e)); return GX_ERR_CUDA; }
    t->nrows = ctx->h_scratch[0] < out_cap ? ctx->h_scratch[0] : out_cap;
    *out = t;
    return GX_OK;
}

// ------------------------------------------------- right semi / anti join under an aggregate
// JOIN_SEMI_RIGHT / JOIN_ANTI_RIGHT (nodes.h:897-900): the preserved relation is the build side, and the probe side only
// decides which build rows survive (the bucket-delete arms of nodeHashjoin.c:580-607, HJ_FILL_INNER for ANTI_RIGHT).
// Three steps: a marking probe sets one bit per build row that has a partner, the build rows are compacted by their bit
// (gx_k_filter_onepass, build row order kept), and the aggregate runs over the compacted rows without a join.
struct gx_mark_args {
    gx_dcol key;
    int npreds, _pad;
    gx_dpred preds[GX_MAX_PREDS];
    long long nrows;
    const gx_slot *slots; unsigned long long mask;
    const gx_cslot *cslots; unsigned long long cspan;
    const unsigned int *narrow;
    const unsigned long long *special; int special_count; int _pad2; gx_slotfn sf;
    unsigned int *bits;                 // one bit per build row (the build stored the row number as payload)
};

// set a build row's bit; a bit already set costs a load instead of an atomic
__device__ __forceinline__ void gx_mark_row(unsigned int *bits, unsigned long long row)
{
    unsigned int *w = bits + (row >> 5);
    const unsigned int b = 1u << (row & 31);
    if (!(__ldcg(w) & b)) atomicOr(w, b);
}

// A warp takes tiles of PT_K x 32 probe rows, as gx_k_hash_probe_unique does: quals tile-wise, NULL keys skipped.  A lane
// whose key equals the key of the lane below it marks nothing (the lane below marks the same rows), which keeps the
// atomics down on a probe side clustered on the key (lineitem: ~4 rows per order).  WALK = false: a unique build, read in
// the format the build wrote through gx_probe_first; WALK = true: every partner, walked in the 16-byte form.  Rows with
// key INT64_MIN mark the side list.
template <int F, bool WALK>
__global__ void __launch_bounds__(256) gx_k_probe_mark(gx_mark_args a)
{
    const int lane = threadIdx.x & 31;
    const long long nwarp = ((long long) gridDim.x * blockDim.x) >> 5, wid = ((long long) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long tile = 32LL * PT_K;
    for (long long base = wid * tile; base < a.nrows; base += nwarp * tile) {
        long long r[PT_K], key[PT_K]; bool ok[PT_K];
#pragma unroll
        for (int j = 0; j < PT_K; j++) { r[j] = base + j * 32 + lane; ok[j] = r[j] < a.nrows; }
        for (int p = 0; p < a.npreds; p++) pred_tile<PT_K>(a.preds[p], r, ok);
#pragma unroll
        for (int j = 0; j < PT_K; j++) {
            ok[j] = ok[j] && !gx_is_null(a.key, r[j]);                     // a NULL key never matches (hashStrict)
            key[j] = ok[j] ? gx_load_int(a.key, r[j]) : 0;
            const long long kd = __shfl_up_sync(0xffffffffu, key[j], 1);
            const bool od = __shfl_up_sync(0xffffffffu, ok[j], 1);
            if (lane > 0 && od && kd == key[j]) ok[j] = false;
            if (ok[j] && key[j] == GX_EMPTY_KEY) {
                for (int i = 0; i < a.special_count; i++) gx_mark_row(a.bits, a.special[i]);
                ok[j] = false;
            }
        }
        if (!WALK) {
            bool hit[PT_K]; unsigned long long pay[PT_K];
            gx_probe_first<F, PT_K>(a, ok, key, hit, pay);
#pragma unroll
            for (int j = 0; j < PT_K; j++) if (hit[j]) gx_mark_row(a.bits, pay[j]);
        } else {
            unsigned long long s[PT_K]; long long k0[PT_K], k1[PT_K]; unsigned long long p0[PT_K], p1[PT_K];
#pragma unroll
            for (int j = 0; j < PT_K; j++) {                                // the home pairs' loads in flight together
                s[j] = gx_slot_index(key[j], a.sf); k0[j] = k1[j] = GX_EMPTY_KEY; p0[j] = p1[j] = 0;
                if (ok[j]) gx_ld_pair(a.slots + s[j], k0[j], p0[j], k1[j], p1[j]);
            }
#pragma unroll
            for (int j = 0; j < PT_K; j++) {
                if (!ok[j]) continue;
                for (;;) {                                                  // linear probing: the run ends at an empty slot
                    if (k0[j] == GX_EMPTY_KEY) break;
                    if (k0[j] == key[j]) gx_mark_row(a.bits, p0[j]);
                    if (k1[j] == GX_EMPTY_KEY) break;
                    if (k1[j] == key[j]) gx_mark_row(a.bits, p1[j]);
                    s[j] = gx_next_pair(s[j], a.mask);
                    gx_ld_pair(a.slots + s[j], k0[j], p0[j], k1[j], p1[j]);
                }
            }
        }
    }
}

// the plan's build columns -> compacted table columns; GX_ERR_ARG for a column the build table does not have
static int right_columns(gx_ctx *ctx, const gx_table *build, const gx_agg_plan *plan, bool plan_keeps_preds, int *map, int32_t *out_cols, int *n_out)
{
    for (int c = 0; c < GX_MAX_COLS; c++) map[c] = -1;
    *n_out = 0;
    auto use = [&](int col, const char *what, int i) -> int {
        GX_CHECK_ARG(ctx, col >= 0 && col < build->ncols, "hash_agg_right: %s %d reads column %d of a %d-column build table", what, i, col, build->ncols);
        if (map[col] < 0) { map[col] = *n_out; out_cols[(*n_out)++] = col; }
        return GX_OK;
    };
    int rc;
    GX_CHECK_ARG(ctx, plan->n_group_cols >= 0 && plan->n_group_cols <= GX_MAX_GROUP_COLS, "agg plan: n_group_cols %d", plan->n_group_cols);
    GX_CHECK_ARG(ctx, plan->n_aggs >= 0 && plan->n_aggs <= GX_MAX_AGGS, "agg plan: n_aggs %d", plan->n_aggs);
    GX_CHECK_ARG(ctx, plan->n_preds >= 0 && plan->n_preds <= GX_MAX_PREDS, "too many predicates (%d)", plan->n_preds);
    for (int c = 0; c < plan->n_group_cols; c++) {
        GX_CHECK_ARG(ctx, plan->group_cols[c].side == 0, "hash_agg_right: group column %d is on side %d (the build table is side 0)", c, plan->group_cols[c].side);
        if ((rc = use(plan->group_cols[c].col, "group column", c))) return rc;
    }
    for (int a = 0; a < plan->n_aggs; a++) {
        if (plan->aggs[a].fn == GX_AGG_COUNT_STAR) continue;              // takes no argument: its program is not read
        const gx_expr &e = plan->aggs[a].arg;
        GX_CHECK_ARG(ctx, e.nops >= 0 && e.nops <= GX_MAX_EXPR_OPS, "agg %d: %d ops", a, e.nops);
        for (int k = 0; k < e.nops; k++) if (e.ops[k].op == GX_OP_COL && (rc = use(e.ops[k].col, "aggregate", a))) return rc;
    }
    if (plan_keeps_preds)
        for (int p = 0; p < plan->n_preds; p++) if ((rc = use(plan->preds[p].col, "predicate", p))) return rc;
    return GX_OK;
}

extern "C" int gx_hash_agg_right(gx_ctx *ctx, const gx_table *probe, int probe_key_col, int n_probe_preds, const gx_pred *probe_preds,
                                 const gx_table *build, const gx_hash *h, int join_type, const gx_agg_plan *plan, gx_result **out)
{
    if (!ctx || !probe || !build || !plan || !out) return GX_ERR_ARG;
    GX_CHECK_ARG(ctx, join_type == GX_JOIN_SEMI_RIGHT || join_type == GX_JOIN_ANTI_RIGHT,
                 "hash_agg_right: join type %d (right semi %d, right anti %d)", join_type, GX_JOIN_SEMI_RIGHT, GX_JOIN_ANTI_RIGHT);
    GX_CHECK_ARG(ctx, h != nullptr, "hash_agg_right: no join table");
    int rc = hash_materialize(const_cast<gx_hash *>(h)); if (rc) return rc;
    GX_CHECK_ARG(ctx, h->n_payload == 0, "hash_agg_right: the join table carries %d payload columns (it must carry the build row number)", h->n_payload);
    GX_CHECK_ARG(ctx, h->src == build && h->src_version == build->version,
                 "hash_agg_right: the join table was not built from this build table as it is now");
    GX_CHECK_ARG(ctx, probe_key_col >= 0 && probe_key_col < probe->ncols, "hash_agg_right: probe key column %d out of range", probe_key_col);
    const int kt = probe->types[probe_key_col];
    GX_CHECK_ARG(ctx, kt == GX_INT4 || kt == GX_INT8 || kt == GX_DATE, "hash_agg_right: probe key type %d (int4, int8 or date)", kt);
    GX_CHECK_ARG(ctx, plan->outer_key_col < 0, "hash_agg_right: the plan's outer_key_col must be -1 (the probe key is an argument)");
    GX_CHECK_ARG(ctx, plan->join_type == GX_JOIN_INNER, "hash_agg_right: the plan's join type must be inner (%d given)", plan->join_type);
    gx_mark_args a; memset(&a, 0, sizeof(a));
    rc = gx_fill_dpreds(ctx, probe, n_probe_preds, probe_preds, a.preds); if (rc) return rc;
    // the plan's quals join the build quals in the compaction when they fit one qual list, else the aggregate applies them
    const bool plan_keeps_preds = h->n_preds + plan->n_preds > GX_MAX_PREDS;
    int map[GX_MAX_COLS]; int32_t out_cols[GX_MAX_COLS]; int n_out = 0;
    rc = right_columns(ctx, build, plan, plan_keeps_preds, map, out_cols, &n_out); if (rc) return rc;
    if (n_out == 0) out_cols[n_out++] = 0;                                  // count(*) alone: the table needs a column
    gx_pred cpreds[GX_MAX_PREDS]; int ncp = h->n_preds;                 // at most GX_MAX_PREDS: see plan_keeps_preds
    memcpy(cpreds, h->preds, sizeof(h->preds));
    if (!plan_keeps_preds) for (int p = 0; p < plan->n_preds; p++) cpreds[ncp++] = plan->preds[p];
    gx_agg_plan p = *plan;                                                  // the plan over the compacted columns
    for (int c = 0; c < p.n_group_cols; c++) p.group_cols[c].col = map[p.group_cols[c].col];
    for (int i = 0; i < p.n_aggs; i++) {
        if (p.aggs[i].fn == GX_AGG_COUNT_STAR) continue;
        for (int k = 0; k < p.aggs[i].arg.nops; k++) if (p.aggs[i].arg.ops[k].op == GX_OP_COL) p.aggs[i].arg.ops[k].col = map[p.aggs[i].arg.ops[k].col];
    }
    if (plan_keeps_preds) for (int i = 0; i < p.n_preds; i++) p.preds[i].col = map[p.preds[i].col];
    else p.n_preds = 0;
    p.outer_key_col = -1; p.join_type = GX_JOIN_INNER;
    {
        // what the aggregate would reject is rejected before any device work: the compacted table's shape is known
        gx_table shape; memset(&shape, 0, sizeof(shape));
        shape.ctx = ctx; shape.ncols = n_out; shape.nrows = build->nrows; shape.capacity = build->nrows;
        for (int c = 0; c < n_out; c++) {
            shape.types[c] = build->types[out_cols[c]]; shape.cols[c] = build->cols[out_cols[c]]; shape.nulls[c] = build->nulls[out_cols[c]];
        }
        rc = gx_check_agg_plan(ctx, &shape, &p); if (rc) return rc;
        gx_dpred dp[GX_MAX_PREDS];                                          // the compaction's quals: columns and operators
        rc = gx_fill_dpreds(ctx, build, ncp, cpreds, dp); if (rc) return rc;
    }

    // 1. marking probe
    // a row-number payload is never narrow (the narrow form carries one 4-byte payload column): wide or compact
    const bool walk = !h->unique;
    if (walk && probe->nrows > 0) { rc = gx_hash_wide(ctx, const_cast<gx_hash *>(h)); if (rc) return rc; }
    const size_t nwords = (size_t) ((build->nrows + 31) / 32);
    unsigned int *bits = nullptr;
    cudaError_t e = gx_tmp_alloc(ctx, (void **) &bits, (nwords ? nwords : 1) * sizeof(unsigned int));
    if (e == cudaSuccess) e = cudaMemsetAsync(bits, 0, (nwords ? nwords : 1) * sizeof(unsigned int), ctx->stream);
    if (e == cudaSuccess && probe->nrows > 0) {
        a.key.data = probe->cols[probe_key_col]; a.key.nulls = probe->nulls[probe_key_col]; a.key.type = kt;
        a.npreds = n_probe_preds; a.nrows = probe->nrows;
        a.slots = h->slots; a.mask = (unsigned long long) h->nslots - 1;
        a.cslots = h->cslots; a.cspan = h->cspan;
        a.special = h->special_payload; a.special_count = h->special_count;
        a.sf = gx_hash_slotfn(h); a.bits = bits;
        const long long nt = (probe->nrows + 32 * PT_K * 8 - 1) / (32 * PT_K * 8), maxb = (long long) ctx->sm_count * 8;
        const unsigned grid = (unsigned) (nt < maxb ? nt : maxb);
        gx_launch_scope ls(ctx, "probe_mark");
        gx_launch_scope which(ctx, walk ? "probe_mark_walk" : h->cslots ? "probe_mark_compact" : "probe_mark_wide", 0);
        if (walk) gx_k_probe_mark<GX_SLOTS_WIDE, true><<<grid, 256, 0, ctx->stream>>>(a);
        else if (h->cslots) gx_k_probe_mark<GX_SLOTS_COMPACT, false><<<grid, 256, 0, ctx->stream>>>(a);
        else gx_k_probe_mark<GX_SLOTS_WIDE, false><<<grid, 256, 0, ctx->stream>>>(a);
        e = cudaGetLastError();
    }
    if (e != cudaSuccess) {
        gx_tmp_free(ctx, bits);
        GX_SET_ERR(ctx, "hash_agg_right: %s", cudaGetErrorString(e));
        return e == cudaErrorMemoryAllocation ? GX_ERR_NOMEM : GX_ERR_CUDA;
    }
    // 2. the build rows the join consumes, in build row order
    gx_table *kept = nullptr;
    rc = gx_filter_marked(ctx, build, ncp, cpreds, n_out, out_cols, bits, join_type == GX_JOIN_SEMI_RIGHT, &kept);
    gx_tmp_free(ctx, bits);
    if (rc) return rc;
    // 3. the aggregate, without a join
    rc = gx_hash_agg(ctx, kept, nullptr, &p, out);
    gx_table_free(kept);
    return rc;
}
