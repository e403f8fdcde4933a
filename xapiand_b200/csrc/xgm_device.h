/* xgm_device.h — kernel parameter block and launcher prototypes (host <-> kernels, internal). */
#ifndef XGM_DEVICE_H
#define XGM_DEVICE_H
#include <cuda_runtime.h>
#include <stdint.h>

#include "xgm_format.h"

#define XGM_MAX_SLOTS 8

struct XgmDevSlot {
    const uint32_t* voff; /* [lastdocid+2] CSR offsets, NULL = slot absent */
    const uint64_t* vals; /* order-preserving numeric keys, ascending per doc */
};

struct XgmDevResult {
    uint32_t n;      /* entries written to out_* (<= topk) */
    uint32_t exact;  /* documents matching the boolean structure */
    uint32_t known;  /* ProtoMSet::known_matching_docs */
    uint32_t flags;  /* XGM_RES_* */
    double max_w;    /* dense kernel: best weight seen */
    uint32_t max_subqs;
    uint32_t pad;
};
#define XGM_RES_LOST 1u        /* candidates were lost: the overflow pool could not take the second pass */
#define XGM_RES_APPROX 2u      /* the match-count bounds are approximate (pruned run) */
#define XGM_RES_PENDING 4u     /* the first pass overflowed: a second pass is pending */
#define XGM_RES_SKIPPED 8u     /* whole work items were skipped by MaxScore: the match count is a lower bound */
#define XGM_RES_SECOND_PASS 16u /* produced by the second pass */

/* Slots of XgmKernelParams::work_counter, zeroed before every batch.  A counter of per-pass work has one slot per
 * pass, slot + pass. */
#define XGM_WC_AND 0        /* [0],[1]   items of xgm_and_kernel taken */
#define XGM_WC_OR 2         /* [2],[3]   items of xgm_or_kernel taken */
#define XGM_WC_RERUN 4      /* [4]       queries the second pass re-runs */
#define XGM_WC_AND_BM 6     /* [6],[7]   items of xgm_and_bm3_kernel taken */
#define XGM_WC_POOL 8       /* [8..9]    64-bit overflow-pool reservation, in entries */
#define XGM_WC_OR3 10       /* [10],[11] items of xgm_or3_kernel<0> taken */
#define XGM_WC_TILE 12      /* [12],[13] tiles of xgm_or_tile_kernel taken */
#define XGM_WC_OR3_SINGLE 14 /* [14],[15] items of xgm_or3_kernel<1> taken */
#define XGM_WC_TOPK_FRONT 16 /* [16]      topk_list entries written from the front */
#define XGM_WC_TOPK 17      /* [17],[18] entries handed to the CTAs of xgm_topk_kernel */
#define XGM_WC_TOPK_BACK 19 /* [19]      topk_list entries written from the back */

struct XgmKernelParams {
    /* index */
    const XgmBlockHdr* hdr;
    const uint4* docs;
    const uint4* tfs;
    const uint32_t* doclen;
    const uint32_t* bitmaps;
    const uint32_t* coarse;       /* a bit per 8 docids of bitmaps[]: word bm_off / 8 + (d >> 8), bit (d >> 3) & 31 */
    const uint32_t* ranks;
    uint32_t lastdocid;
    uint32_t doclen_lb;           /* Database::get_doclength_lower_bound: block-level weight bounds */
    XgmDevSlot slots[XGM_MAX_SLOTS];
    /* batch */
    const XgmDevQuery* queries;
    const XgmWorkItem* items;     /* AND kernel work list */
    const XgmWorkItem* items_or;  /* OR kernel work list */
    const XgmWorkItem* items_bm;  /* bitmap AND kernel work list */
    uint32_t nitems, nitems_or, nitems_bm;
    const uint32_t* nitems_bm_dev; /* non-null: item count of the bitmap AND list lives on the device (range-major expansion) */
    /* range-major bitmap AND list: its segments, sorted by driver list.  An item serves the run of queries
     * bm_segs[query .. query + pad).query, which share the driver.  Null (level order): the item's query field is
     * its one query. */
    const XgmWorkItem* bm_segs;
    uint32_t nq;
    uint32_t* work_counter;       /* batch counters, slots XGM_WC_* */
    uint32_t pass;                /* 0 = first pass, 1 = re-run of overflowed queries with their exact b* */
    XgmQState* qstate;            /* [nq] */
    uint32_t* hist;               /* [nq][XGM_NBINS] */
    /* per-query match buffers */
    uint32_t match_cap;
    uint32_t keep_cap;            /* survivors the top-k kernel can rank in shared memory */
    double* match_w;
    uint32_t* match_d;
    uint64_t* match_k;
    /* overflow pool: second-pass candidates of queries whose first-pass buffer overflowed */
    uint32_t pool_total;
    double* pool_w;
    uint32_t* pool_d;
    uint64_t* pool_k;
    /* results */
    uint32_t out_stride;
    double* out_w;
    uint32_t* out_d;
    uint64_t* out_k;
    XgmDevResult* out_info;
    XgmRaise* raise_log;          /* [nq][XGM_RAISE_LOG] */
    /* xgm_or_tile_kernel's work list: the queries with or_fast == XGM_OR_FAST_TILE (xgm_or3_kernel<1> finds their
     * items in items_or) */
    const uint32_t* tileq;
    uint32_t ntileq;
    /* top-k: queries xgm_topk_small_kernel left to xgm_topk_kernel (XGM_WC_TOPK_FRONT counts the expensive ones from
     * the front of the list, XGM_WC_TOPK_BACK the others from its back); null = every query of the batch.
     * XGM_WC_TOPK + pass hands the entries out. */
    uint32_t* topk_list;
};
#define XGM_CTRL_HDR 128 /* bytes of work counters in front of the per-query state */
static_assert(4 * (XGM_WC_TOPK_BACK + 1) <= XGM_CTRL_HDR, "the work counters fit their header");

/* Largest keep_cap of a searcher: the top-k kernel holds XGM_KEEP_PER_THREAD survivors per thread in registers. */
#define XGM_KEEP_CAP_MAX 8192u

/* Resident-CTA grids of the persistent kernels for one searcher. */
struct XgmGrids {
    int and_, and_bm, or_, or3, or_tile, topk;
};
/* The grids on the current device at sm_count SMs, the top-k kernel's at keep_cap.  Also opts the kernels with large
 * dynamic shared memory in on the current device, each at a constant size: the bitmap AND and or3 kernels at their
 * fixed scratch, the top-k kernel at XGM_KEEP_CAP_MAX.  Searchers of any keep_cap, created on any thread, write the
 * same values. */
cudaError_t xgm_kernel_grids(int sm_count, uint32_t keep_cap, XgmGrids& g);

cudaError_t xgm_launch_and(const XgmKernelParams& p, int grid, cudaStream_t s);
cudaError_t xgm_launch_and_bm(const XgmKernelParams& p, int grid, cudaStream_t s);
cudaError_t xgm_launch_expand(const XgmWorkItem* seg, uint32_t total, const uint32_t* level_start, uint32_t nlevels,
                              uint32_t bpi, XgmWorkItem* out, cudaStream_t s);
cudaError_t xgm_launch_expand_ranges(const XgmWorkItem* runs, uint32_t nruns, const XgmBlockHdr* hdr, uint32_t nranges,
                                     uint32_t range_bits, uint32_t bpi, uint32_t* lo, uint32_t* cnt, uint32_t* off,
                                     uint32_t* total, XgmWorkItem* out, cudaStream_t s);
cudaError_t xgm_launch_or(const XgmKernelParams& p, int grid, cudaStream_t s);
cudaError_t xgm_launch_or3(const XgmKernelParams& p, int grid, int phase, cudaStream_t s);
cudaError_t xgm_launch_or_tile(const XgmKernelParams& p, int grid, cudaStream_t s);
/* Ranks the batch's nq queries on at most `grid` CTAs; adds the kernels it enqueued (one or two) to `launches`. */
cudaError_t xgm_launch_topk(const XgmKernelParams& p, uint32_t nq, int grid, uint32_t& launches, cudaStream_t s);
cudaError_t xgm_launch_coarse(const uint32_t* bitmaps, size_t ncoarse, uint32_t* coarse, cudaStream_t s);
cudaError_t xgm_launch_decode(const XgmKernelParams& p, uint32_t blk_begin, uint32_t nblocks, int sm_count,
                              uint32_t* out_d, uint32_t* out_w, cudaStream_t s);
size_t xgm_topk_smem_bytes(uint32_t keep_cap);
/* xgm_merge_kernel's inputs: nparts gathered parts, part p of each array at base + p * part_* bytes, [query][rank]
 * records of `stride` per query; outputs [nq][maxitems] records and [nq] counts. */
struct XgmMergeArgs {
    const double* gw;
    const uint32_t* gd;
    const uint64_t* gk;          /* sort keys; null: no order reads them (then out_k is not written) */
    const XgmDevResult* ginfo;
    size_t part_w, part_d, part_k, part_info;
    const uint8_t* orders;       /* [nq]: bits 0-1 XGM_SORT_*, bit 2 reverse; null: relevance for every query */
    uint32_t nparts, nq, stride, first, maxitems;
    double* out_w;
    uint32_t* out_d;
    uint64_t* out_k;
    uint32_t* out_n;
};
#define XGM_MERGE_MAX_PARTS 64
#define XGM_MERGE_MAX_SMEM (200 * 1024) /* bytes of dynamic shared memory a merge may take */
/* xgm_merge_kernel's dynamic shared memory: weight, docid and, when keys are read, key of m records per part */
static inline uint64_t xgm_merge_smem_bytes(uint32_t nparts, uint64_t m, bool keys) {
    return nparts * m * (keys ? 20 : 12);
}
/* The caller checks nparts and xgm_merge_smem_bytes against the limits above. */
cudaError_t xgm_launch_merge(const XgmMergeArgs& a, cudaStream_t s);

#endif
