/* gsb_internal.h — interfaces between the translation units of libgpushare_b200.so (not installed). */
#ifndef GSB_INTERNAL_H_
#define GSB_INTERNAL_H_

#include <cuda_runtime_api.h>
#include <stdint.h>

#include "../../include/gpushare_b200.h"

/* What one CTA leaves behind; the last CTA to finish folds all slots into gsb_kernel_out. */
struct gsb_partial {
  unsigned long long mismatch_words;
  unsigned long long mismatch_bits;
  unsigned long long first_bad_word; /* absolute 16 B-word index, ~0ull if none */
  unsigned long long words;          /* words this CTA processed */
  uint32_t checksum_xor;
  uint32_t checksum_sum;
};

/* Written by the kernel into pinned, device-mapped host memory (one per device). */
struct gsb_kernel_out {
  unsigned long long mismatch_words;
  unsigned long long mismatch_bits;
  unsigned long long first_bad_word;
  uint32_t checksum_xor;
  uint32_t checksum_sum;
  unsigned long long words_done; /* Σ words every CTA processed — must equal n_words */
  uint32_t done_flag;            /* launch sequence number echoed by the finishing CTA */
  uint32_t pad;
};

/* One mismatching word as the kernel saw it. */
struct gsb_fault_word {
  unsigned long long word; /* absolute 16 B-word index */
  uint32_t observed[4];
  uint32_t expected[4];
};

/* Fault log of one device. The device copy is filled by the mismatch branch of every comparing kernel and emptied by
 * the last CTA of a faulted launch, which first copies it into the pinned, device-mapped host copy (launch_seq tells
 * the host which launch that copy belongs to). A clean launch touches neither. */
struct gsb_fault_log {
  unsigned long long flips[2][128]; /* [0]: expected 0 observed 1, [1]: expected 1 observed 0; bit 32 * lane + bit */
  unsigned int count;               /* device: slots claimed (may pass GSB_FAULT_RECORDS); host: records filled */
  uint32_t launch_seq;              /* host copy only */
  gsb_fault_word rec[GSB_FAULT_RECORDS];
};

/* The link ops (gsb_link_probe) use neither the window's first word, the generation table's arena size nor March C-'s
 * backgrounds, so their four fields share storage with those in anonymous unions of the same types: no field moves,
 * the struct keeps its size and no pointer gains an alias. That keeps every other kernel's code as it was (ptxas
 * schedules them differently once the parameter block grows). A link launch: CTAs [0, link_down_ctas) read the host
 * buffer at `base` (n_words words, compared with seed_expect's pattern; word offsets from the buffer's start) and the
 * others write seed_write's pattern into the host buffer at device address link_up (link_up_words words), both
 * link_passes times over. The copy verify ops (gsb_copy_probe) use none of those three either: copy_begin and copy_end
 * are the destination byte range [begin, end) the copy wrote and copy_delta = src_offset - dst_offset mod 2^32 (the
 * copy geometry of gsb_pattern.h); `base` is the destination, n_words its words, seed_expect its background and
 * seed_write the source's seed. */
struct gsb_kernel_args {
  uint4 *base;                 /* arena base (device VA of absolute word 0) */
  union {
    unsigned long long first_word; /* absolute index of the window's first 16 B word */
    unsigned long long link_up_words;
    unsigned long long copy_begin;
  };
  unsigned long long n_words;    /* words in the window */
  uint32_t seed_expect;        /* raw seed (the kernel mixes it) */
  uint32_t seed_write;
  const uint32_t *seed_table;  /* optional: raw expected seed per granule, indexed (w >> granule_shift) */
  uint32_t *table_update;      /* optional: last CTA stores seed_write for every granule the window covers */
  union {
    unsigned long long arena_words; /* words in the whole arena (tail-granule rule of table_update) */
    unsigned long long link_up;
    unsigned long long copy_end;
  };
  uint32_t granule_shift;      /* log2(words per granule) */
  uint32_t launch_seq;
  uint32_t opaque_zero;        /* always 0; only the compiler does not know (DIRECT refill: a real load->store dependency) */
  gsb_partial *partials;       /* [grid] device memory */
  unsigned int *ticket;        /* device memory, self-resetting */
  /* device memory, self-resetting, two counters of BULKD: [0] the dynamic tile scheduler's claims, [1] the verify
   * tiles a refill has consumed */
  unsigned long long *tile_counter;
  gsb_kernel_out *out;         /* device pointer of the mapped host struct */
  gsb_fault_log *fault;        /* device memory, self-resetting (zero between faulted launches) */
  gsb_fault_log *fault_out;    /* device pointer of the mapped host copy */
  /* March C- ops only: the background each lane of a word is compared with, and the one stored (0 or 0xFFFFFFFF);
   * last, so that no field above moves */
  union {
    uint32_t solid_expect;
    uint32_t link_down_ctas;
    uint32_t copy_delta;
  };
  union {
    uint32_t solid_write;
    uint32_t link_passes;
  };
};

struct gsb_launch_geom {
  uint32_t variant; /* resolved GSB_VARIANT_* */
  uint32_t grid;
  uint32_t block;
  uint32_t smem_bytes;
};

/* Resolve variant/grid for the CURRENT device (occupancy query); grid_request == 0 => auto. */
int gsb_kernel_geometry(uint32_t op, uint32_t variant, uint32_t grid_request, int sm_count,
                        gsb_launch_geom *geom);
/* Enqueue one probe launch on `stream` of the current context. Returns cudaError_t as int. */
int gsb_kernel_launch(uint32_t op, const gsb_launch_geom *geom, const gsb_kernel_args *args,
                      cudaStream_t stream);
/* Test hook: one thread spinning on %globaltimer for `ns` nanoseconds on `stream`. Returns cudaError_t as int. */
int gsb_kernel_stall(unsigned long long ns, cudaStream_t stream);
/* Test hook of gsb_copy_probe: XOR xr into the 16-byte word at p (device memory) on `stream`. Returns cudaError_t. */
int gsb_kernel_xor_word(uint4 *p, uint4 xr, cudaStream_t stream);
/* CTAs of one side (down or up) of a PCIe link launch on a device with `sm_count` SMs. */
uint32_t gsb_kernel_link_ctas(int sm_count);
/* Load every kernel this library can launch into the CURRENT context. Returns cudaError_t as int. */
int gsb_kernel_preload(void);
/* Upper bound of CTAs any geometry will use on a device with `sm_count` SMs (sizes `partials`). */
uint32_t gsb_kernel_max_grid(int sm_count);

/* What one SM-check launch (sm_check_sm90a.cu) leaves in device memory; the host zeroes it before every launch. */
struct gsb_sm_log {
  unsigned int covered[GSB_SM_MAX / 32]; /* bit %smid: a CTA of the launch ran there */
  unsigned int faulty[GSB_SM_MAX / 32];  /* bit %smid: a wrong word there */
  unsigned long long words;              /* result words compared */
  unsigned long long mismatch_words;
  unsigned long long mismatch_bits;
  unsigned int count;                    /* records claimed (may pass GSB_SM_RECORDS) */
  unsigned int pad;
  gsb_sm_record rec[GSB_SM_RECORDS];
};

struct gsb_sm_args {
  gsb_sm_log *log;
  const void *expected;         /* the unit's answers (gsb_sm_expected): uint64 per chain thread, uint32 per D word */
  unsigned long long hook_xr;   /* test hook: XORed into word hook_index of the CTA on SM hook_smid */
  uint32_t seed;                /* operands' seed */
  uint32_t hook_smid;           /* GSB_SM_MAX: no hook */
  uint32_t hook_index;
  uint32_t smem_bytes;          /* dynamic shared memory of every CTA */
};

/* Enqueue one SM-check launch of `unit` with `grid` CTAs on `stream`. Returns cudaError_t as int. */
int gsb_sm_kernel_launch(uint32_t unit, uint32_t grid, const gsb_sm_args *a, cudaStream_t stream);
/* The same for a tensor unit's test-only twin (mma_operands_sm90a.cu, gsb_test_sm_operands): its operands are the table
 * after the 8192 expected words at a->expected (gsb_sm_table_* in gsb_sm_kat.h). */
int gsb_sm_operands_launch(uint32_t unit, uint32_t grid, const gsb_sm_args *a, cudaStream_t stream);
/* Load the SM-check kernels into the CURRENT context and let each take `smem_bytes` of dynamic shared memory. */
int gsb_sm_kernel_preload(int smem_bytes);
/* The same for the four test-only twins. */
int gsb_sm_operands_preload(int smem_bytes);

/* Enqueue one tensor-core format check launch (tensor_check_sm90a.cu) of GSB_TENSOR_UNIT_* `unit` with `grid` CTAs on
 * `stream`. Its log and arguments are the SM check's: gsb_sm_log, and gsb_sm_args whose `expected` holds the 8192 D
 * words (gsb_tensor_word_bytes each). Returns cudaError_t as int. */
int gsb_tensor_kernel_launch(uint32_t unit, uint32_t grid, const gsb_sm_args *a, cudaStream_t stream);
/* The same for a unit's test-only twin (tensor_operands_sm90a.cu, gsb_test_tensor_operands): its operands are the
 * table after the 8192 expected words (gsb_sm_table_* in gsb_sm_kat.h). */
int gsb_tensor_operands_launch(uint32_t unit, uint32_t grid, const gsb_sm_args *a, cudaStream_t stream);
/* Load the tensor-core format check's kernels (and, for the second, their twins) into the CURRENT context and let each
 * take `smem_bytes` of dynamic shared memory. */
int gsb_tensor_kernel_preload(int smem_bytes);
int gsb_tensor_operands_preload(int smem_bytes);

/* Enqueue one sparse tensor-core check launch (sparse_check_sm90a.cu, libgpushare_b200_sparse.so) of
 * GSB_SPARSE_UNIT_* `unit` with `grid` CTAs on `stream`. Its log and arguments are the SM check's: gsb_sm_log, and
 * gsb_sm_args whose `expected` holds the 8192 D words (uint32 each). Returns cudaError_t as int. */
int gsb_sparse_kernel_launch(uint32_t unit, uint32_t grid, const gsb_sm_args *a, cudaStream_t stream);
/* The same for a unit's test-only twin (sparse_operands_sm90a.cu, gsb_test_sparse_operands): its operands and patterns
 * are the table after the 8192 expected words (gsb_sparse_table_* in gsb_sparse_kat.h). */
int gsb_sparse_operands_launch(uint32_t unit, uint32_t grid, const gsb_sm_args *a, cudaStream_t stream);
/* Load the sparse check's kernels (and, for the second, their twins) into the CURRENT context and let each take
 * `smem_bytes` of dynamic shared memory. */
int gsb_sparse_kernel_preload(int smem_bytes);
int gsb_sparse_operands_preload(int smem_bytes);

/* Arguments of one SM special-function check launch (sfu_check_sm90a.cu): the SM check's, whose `expected` holds an
 * exact unit's folds (uint64, index op * 256 + thread), and for MUFU where each CTA writes its folds, raw results and
 * %smid (indexed by blockIdx; layout as gsb_sfu_vote reads them). */
struct gsb_sfu_args {
  gsb_sm_args sm;
  unsigned long long *folds;
  uint32_t *raw;
  uint32_t *smid;
};

/* Enqueue one SM special-function check launch of GSB_SFU_UNIT_* `unit` with `grid` CTAs on `stream`. Returns
 * cudaError_t as int. */
int gsb_sfu_kernel_launch(uint32_t unit, uint32_t grid, const gsb_sfu_args *a, cudaStream_t stream);
/* Load its kernels into the CURRENT context and let each take `smem_bytes` of dynamic shared memory. */
int gsb_sfu_kernel_preload(int smem_bytes);

/* Arguments of one chosen-input launch of an SFU value unit's test-only twin (sfu_operands_sm90a.cu,
 * gsb_test_sfu_inputs): every CTA runs instruction `op` of the unit on the n operand pairs (a[i], b[i]) as the shipped
 * kernel's instruction takes them, writes result i to out[blockIdx * n + i] and its %smid to smid[blockIdx], and sets
 * its coverage bit in log. */
struct gsb_sfu_table_args {
  gsb_sm_log *log;
  const unsigned long long *a;
  const unsigned long long *b;
  unsigned long long *out;
  uint32_t *smid;
  uint32_t n;
  uint32_t op;
  uint32_t smem_bytes;
};

/* Enqueue one such launch of GSB_SFU_UNIT_* `unit` (not WARP) with `grid` CTAs on `stream`. Returns cudaError_t as
 * int. */
int gsb_sfu_operands_launch(uint32_t unit, uint32_t grid, const gsb_sfu_table_args *a, cudaStream_t stream);
/* The same preload for the twins. */
int gsb_sfu_operands_preload(int smem_bytes);

/* What one L1 check launch (l1_check_sm90a.cu) leaves in device memory; the host zeroes it before every launch. Its
 * leading fields are the SM check's, so fold_log serves it; the host classifies the records afterwards. */
struct gsb_l1_log {
  unsigned int covered[GSB_SM_MAX / 32]; /* bit %smid: a CTA of the launch ran there */
  unsigned int faulty[GSB_SM_MAX / 32];  /* bit %smid: a wrong word there */
  unsigned long long words;              /* 16-byte words compared */
  unsigned long long mismatch_words;
  unsigned long long mismatch_bits;
  unsigned int count;                    /* records claimed (may pass GSB_L1_RECORDS) */
  unsigned int pad;
  gsb_l1_record rec[GSB_L1_RECORDS];
};

struct gsb_l1_args {
  gsb_l1_log *log;
  uint4 *buf;                      /* sm_count regions of GSB_L1_REGION_WORDS words, filled with seed's pattern */
  unsigned long long *spans;       /* [blockIdx][GSB_L1_FORMS][2]: clock64 span of the cold pass, of the warm passes */
  unsigned long long tex_linear;   /* TEX: cudaTextureObject_t of buf as one linear uint4 resource */
  unsigned long long tex_clamp;    /* TEX: buf as a pitch-2D array of GSB_L1_TEX_WIDTH x rows uint4, clamp addressing */
  unsigned long long tex_border;   /* the same with border addressing */
  unsigned long long hook_xr;      /* test hook: XORed into lanes 0-1 of observed word hook_index on SM hook_smid */
  uint32_t seed;                   /* the pattern the buffer, bank and parameters hold; L1_STORE stores generation 2 */
  uint32_t seed_expect;            /* the pattern the kernels compare against */
  uint32_t passes;                 /* L1_LOAD and NC */
  uint32_t rows;                   /* TEX: rows of the 2-D array (GSB_L1_TEX_ROWS per CTA) */
  uint32_t hook_smid;              /* GSB_SM_MAX: no corrupt hook */
  uint32_t hook_index;
  uint32_t skip_smid;              /* L1_STORE: the CTA on this SM stores nothing; GSB_SM_MAX: none */
  uint32_t reserved0;
};

/* Enqueue one L1 check launch of GSB_L1_UNIT_* `unit` with `grid` CTAs on `stream`. PARAM launches with `param`
 * (GSB_L1_PARAM_WORDS words) as its parameter. Returns cudaError_t as int. */
int gsb_l1_kernel_launch(uint32_t unit, uint32_t grid, const gsb_l1_args *a, const uint4 *param, cudaStream_t stream);
/* What a test-only twin l1_from_table<UNIT> reads besides gsb_l1_args (gsb_test_l1_table, include/gpushare_b200.h). */
struct gsb_l1_table_args {
  const uint32_t *table;     /* n entries */
  const uint32_t *expected;  /* L1_STORE: [cta][region word][4]; TEX: [cta][read][2]; else unused */
  uint32_t n;
  uint32_t region_words;     /* words of each CTA's region (TEX, CONST, PARAM: the fixed size) */
};

/* Enqueue one launch of `unit`'s twin (l1_table_sm90a.cu) with `grid` CTAs on `stream`, as gsb_l1_kernel_launch; CONST
 * first enqueues the copy of GSB_L1_CONST_WORDS words at `bank` into the twin's own bank (`bank` must stay valid until
 * it has run). Returns cudaError_t as int. */
int gsb_l1_table_launch(uint32_t unit, uint32_t grid, const gsb_l1_args *a, const gsb_l1_table_args *t,
                        const uint4 *bank, const uint4 *param, cudaStream_t stream);
/* Enqueue the copy of GSB_L1_CONST_WORDS words at `host` into the CONST unit's bank on `stream`; `host` must stay
 * valid until the copy has run. Returns cudaError_t as int. */
int gsb_l1_const_upload(const uint4 *host, cudaStream_t stream);
/* cudaOccupancyMaxActiveBlocksPerMultiprocessor of `unit`'s kernel. Returns cudaError_t as int. */
int gsb_l1_occupancy(uint32_t unit, int *ctas);
/* Load the L1 check's kernels into the CURRENT context and ask for the largest L1 (carveout 0) for its buffer units. */
int gsb_l1_kernel_preload(void);

/* What one memory-ordering check launch (order_check_sm90a.cu) leaves in device memory; the host zeroes it before every
 * launch. Its leading fields are the SM check's, so fold_log serves it. */
struct gsb_order_log {
  unsigned int covered[GSB_SM_MAX / 32]; /* bit %smid: a CTA of the launch ran there */
  unsigned int faulty[GSB_SM_MAX / 32];  /* bit %smid: a consumer there recorded a bad outcome */
  unsigned long long words;              /* u64 words read and checked */
  unsigned long long mismatch_words;     /* observations and final reads classed CORRUPT, FORBIDDEN or LOST */
  unsigned long long mismatch_bits;
  unsigned int count;                    /* records claimed (may pass GSB_ORDER_RECORDS) */
  unsigned int barrier;                  /* the grid barriers' arrival counter */
  unsigned long long corrupt, forbidden, lost, timeout, overlap, weak;
  gsb_order_record rec[GSB_ORDER_RECORDS];
};

struct gsb_order_args {
  gsb_order_log *log;
  unsigned long long *locs;  /* sm_count blocks of GSB_ORDER_LOC_WORDS u64 */
  uint4 *scratch;            /* sm_count stress regions of GSB_ORDER_SCRATCH_WORDS */
  unsigned long long *obs;   /* [rank][observation][GSB_ORDER_OBS_WORDS]: SB and IRIW reads, classified after the barrier */
  uint32_t *smids;           /* [rank]: %smid, published before the first barrier */
  uint32_t seed;             /* the seed the words are stored under */
  uint32_t seed_expect;      /* the seed the kernel checks hashes against */
  uint32_t unit;             /* GSB_ORDER_UNIT_* */
  uint32_t distance;         /* d */
  uint32_t dist_index;       /* 0..GSB_ORDER_DISTANCES-1, for the records */
  uint32_t observations;     /* iterations per CTA */
  uint32_t inject_smid;      /* test hook: the consumer on this SM forges observation inject_index; GSB_SM_MAX: none */
  uint32_t inject_index;
  uint32_t skip_smid;        /* test hook: the CTA on this SM stores nothing; GSB_SM_MAX: none */
  uint32_t smem_bytes;       /* dynamic shared memory of every CTA */
};

/* Enqueue one cooperative memory-ordering launch of `grid` CTAs on `stream`. Returns cudaError_t as int
 * (cudaErrorCooperativeLaunchTooLarge: the CTAs could not all be co-resident). */
int gsb_order_kernel_launch(uint32_t grid, const gsb_order_args *a, cudaStream_t stream);
/* Load its kernel into the CURRENT context and let it take `smem_bytes` of dynamic shared memory. */
int gsb_order_kernel_preload(int smem_bytes);

/* What one SM-stress slice (sm_stress_sm90a.cu) leaves in device memory; the host zeroes it before every slice. */
struct gsb_stress_log {
  unsigned int covered[GSB_SM_MAX / 32];
  unsigned int faulty[GSB_SM_MAX / 32];
  unsigned long long words;                             /* D words checked */
  unsigned long long mismatch_words;
  unsigned long long mismatch_bits;
  unsigned int count;                                   /* records claimed (may pass GSB_SM_RECORDS) */
  unsigned int pad;
  unsigned long long set_iterations[GSB_STRESS_SETS_MAX];
  unsigned long long sm_iterations[GSB_SM_MAX];         /* by %smid */
  gsb_stress_record rec[GSB_SM_RECORDS];
};

struct gsb_stress_args {
  gsb_stress_log *log;
  const uint32_t *expected;     /* sets x 8192 D words, row-major: gsb_sm_expected(unit, seed_expect + s) */
  const uint32_t *folds;        /* sets x GSB_STRESS_FOLD_THREADS: gsb_stress_fold of the same */
  unsigned long long slice_ns;  /* each CTA stops iterating this long after it started */
  unsigned long long max_iters; /* and after this many iterations of a warpgroup, whatever %globaltimer says */
  uint32_t seed;                /* set s uses the SM probe's operands at seed + s */
  uint32_t slice;               /* the run's slice (for the records) */
  uint32_t smem_bytes;
  uint32_t hook_smid;           /* GSB_SM_MAX: no hook */
  uint32_t hook_index;
  uint32_t hook_xr;
};

/* Enqueue one SM-stress slice of tensor unit `unit` with `grid` CTAs on `stream`. Returns cudaError_t as int. */
int gsb_stress_kernel_launch(uint32_t unit, uint32_t grid, const gsb_stress_args *a, cudaStream_t stream);
/* Let the SM-stress kernels take `smem_bytes` of dynamic shared memory. Returns cudaError_t as int. */
int gsb_stress_kernel_preload(int smem_bytes);
/* Iterations one warpgroup of `unit` cannot exceed per microsecond (twice the SM's dense tensor peak at 2 GHz). */
uint32_t gsb_stress_iters_per_us(uint32_t unit);

/* What one SM-to-SM launch (cluster_check_sm90a.cu) leaves in device memory; the host zeroes it before every launch. */
struct gsb_cluster_log {
  unsigned int covered[GSB_CLUSTER_SM_MAX / 32]; /* bit %smid: a CTA of the launch ran there */
  unsigned int faulty[GSB_CLUSTER_SM_MAX / 32];  /* bit %smid: one end of a wrong word */
  unsigned long long words;                      /* 16-byte words compared */
  unsigned long long mismatch_words;
  unsigned long long mismatch_bits;
  unsigned int timeouts;                         /* mbarrier waits that ran out */
  unsigned int count;                            /* records claimed (may pass GSB_CLUSTER_RECORDS) */
  gsb_cluster_record rec[GSB_CLUSTER_RECORDS];
};

struct gsb_cluster_args {
  gsb_cluster_log *log;
  const void *mc_src;           /* MULTICAST: n segments of region_words words, segment s what rank s multicasts */
  unsigned long long hook_xr;   /* test hook: XORed into lanes 0-1 of checked word hook_index of the CTA on hook_smid */
  uint32_t seed;                /* the words sent and the background */
  uint32_t seed_expect;         /* the words checked against */
  uint32_t hook_smid;           /* GSB_CLUSTER_SM_MAX: no corrupt hook */
  uint32_t hook_index;
  uint32_t skip_smid;           /* test hook: the CTA on this SM sends nothing; GSB_CLUSTER_SM_MAX: none */
  uint32_t smem_bytes;          /* dynamic shared memory of every CTA */
};

/* Enqueue one SM-to-SM launch of `path`: `clusters` clusters of n CTAs on `stream`. Returns cudaError_t as int. */
int gsb_cluster_kernel_launch(uint32_t path, uint32_t n, uint32_t clusters, const gsb_cluster_args *a,
                              cudaStream_t stream);
/* cudaOccupancyMaxActiveClusters of clusters of n CTAs with `smem_bytes` each (0 when none fits). */
int gsb_cluster_max_active(uint32_t n, int smem_bytes, int *clusters);
/* Load the SM-to-SM kernels into the CURRENT context, let each take `smem_bytes` of dynamic shared memory and allow
 * clusters of 16. */
int gsb_cluster_kernel_preload(int smem_bytes);
/* gsb_test_cluster_script: enqueue the test-only twin of `path`'s launch (cluster_script_sm90a.cu, in
 * libgpushare_b200_cluster_script.so), its region size and
 * routes read from `s` in device memory. Returns cudaError_t as int. */
int gsb_cluster_script_launch(uint32_t path, uint32_t n, uint32_t clusters, const gsb_cluster_args *a,
                              const struct gsb_cluster_script *s, cudaStream_t stream);
int gsb_cluster_script_preload(int smem_bytes);

/* What one L2 atomic launch (atomic_check_sm90a.cu) leaves in device memory; the host zeroes it before every launch.
 * A run launch fills the first part, a check launch the counts and records. */
struct gsb_atomic_log {
  unsigned int covered[GSB_ATOMIC_SM_MAX / 32];  /* bit %smid: a CTA of the run launch ran there */
  unsigned int cta_smid[GSB_ATOMIC_SM_MAX];      /* %smid of each run CTA, by blockIdx */
  unsigned long long issued;                     /* atomics the run launch issued (CAS: successful swaps) */
  unsigned long long words;                      /* words the check launch compared */
  unsigned long long mismatch_words;
  unsigned long long mismatch_bits;
  unsigned int timeouts;                         /* CAS loops that ran out */
  unsigned int out_of_range;                     /* tickets returned at or past the word's contributor count */
  unsigned int cas_max_ns;                       /* the longest CAS loop */
  unsigned int skipped_cta;                      /* blockIdx + 1 of the CTA that applied the skip hook; 0: none */
  unsigned int count;                            /* records claimed (may pass GSB_ATOMIC_RECORDS) */
  unsigned int reserved0;
  gsb_atomic_record rec[GSB_ATOMIC_RECORDS];
};

struct gsb_atomic_args {
  gsb_atomic_log *log;
  void *buf;                  /* GSB_ATOMIC_BYTES: the words the atomics land on */
  const void *expected;       /* GSB_ATOMIC_BYTES: what the check launch compares them with */
  uint32_t *slots;            /* TICKET, CAS: GSB_ATOMIC_HOT_WORDS x gsb_atomic_hot_count ticket slots */
  unsigned long long hook_xr; /* test hook: XORed into observed word hook_word by the check launch */
  uint32_t op;
  uint32_t seed;              /* the starting words and the contributions */
  uint32_t ctas;              /* CTAs of the run launch: the contributor count derives from it */
  uint32_t hook_word;         /* 0xFFFFFFFF: no corrupt hook */
  uint32_t skip_smid;         /* test hook: the run CTA on this SM issues nothing; GSB_ATOMIC_SM_MAX: none */
  uint32_t smem_bytes;        /* dynamic shared memory of every run CTA */
};

enum { GSB_ATOMIC_STAGE_INIT = 0, GSB_ATOMIC_STAGE_RUN = 1, GSB_ATOMIC_STAGE_CHECK = 2 };
/* Enqueue one L2 atomic launch of `stage` for a->op on `stream` (a->ctas CTAs). Returns cudaError_t as int. */
int gsb_atomic_kernel_launch(uint32_t stage, const gsb_atomic_args *a, cudaStream_t stream);
/* Load the L2 atomic kernels into the CURRENT context and let each run kernel take `smem_bytes` of shared memory. */
int gsb_atomic_kernel_preload(int smem_bytes);
/* gsb_test_atomic_values: enqueue the test-only twin of a->op's run launch (atomic_values_sm90a.cu), each operand read
 * from `values` (gsb_atomic_value_count(a->ctas) words, gsb_atomic_value_index). Not for TICKET or CAS. */
int gsb_atomic_values_launch(const gsb_atomic_args *a, const uint64_t *values, cudaStream_t stream);
int gsb_atomic_values_preload(int smem_bytes);

/* What one shared-memory atomic launch (shared_atomic_check_sm90a.cu, libgpushare_b200_shared_atomic.so) leaves in
 * device memory; the host zeroes it before every launch. Its leading fields are the SM check's, so fold_log serves it. */
struct gsb_shared_atomic_log {
  unsigned int covered[GSB_SM_MAX / 32]; /* bit %smid: a CTA of the launch ran there */
  unsigned int faulty[GSB_SM_MAX / 32];  /* bit %smid: a wrong word or an out-of-range ticket there */
  unsigned long long words;              /* area words compared */
  unsigned long long mismatch_words;
  unsigned long long mismatch_bits;
  unsigned int count;                    /* records claimed (may pass GSB_SHARED_ATOMIC_RECORDS) */
  unsigned int skipped_cta;              /* blockIdx + 1 of the CTA that applied the skip hook; 0: none */
  unsigned long long issued;             /* atomics issued (CAS: successful swaps) */
  unsigned int timeouts;                 /* CAS loops and REDAS waits that ran out */
  unsigned int faults;                   /* tickets returned at or past the count, torn b128 pairs */
  unsigned int cas_max_ns;               /* the longest CAS loop */
  unsigned int reserved0;
  unsigned int cta_smid[GSB_SM_MAX];     /* %smid of each CTA, by blockIdx */
  gsb_shared_atomic_record rec[GSB_SHARED_ATOMIC_RECORDS];
};

struct gsb_shared_atomic_args {
  gsb_shared_atomic_log *log;
  const uint32_t *expected;   /* GSB_SHARED_ATOMIC_AREA_WORDS: every CTA's area after a clean run (DSMEM, REDAS: one
                                 area per cluster rank) */
  uint32_t *slots;            /* TICKET, CAS: grid x GSB_SHARED_ATOMIC_SLOT_WORDS (gsb_shared_atomic_slot) */
  unsigned long long hook_xr; /* test hook: XORed into observed word hook_index by the CTA on hook_smid */
  uint32_t seed;              /* the starting words and the contributions */
  uint32_t hook_smid;         /* GSB_SM_MAX: no corrupt hook */
  uint32_t hook_index;
  uint32_t skip_smid;         /* test hook: the CTA on this SM issues no atomic; GSB_SM_MAX: none */
  uint32_t smem_bytes;        /* dynamic shared memory of every CTA */
  uint32_t reserved0;
};

/* Enqueue one shared-memory atomic launch of GSB_SHARED_ATOMIC_UNIT_* `unit` with `grid` CTAs on `stream`. Returns
 * cudaError_t as int. */
int gsb_shared_atomic_kernel_launch(uint32_t unit, uint32_t grid, const gsb_shared_atomic_args *a, cudaStream_t stream);
/* Enqueue one DSMEM or REDAS launch: `clusters` clusters of n CTAs on `stream`; a->expected holds the n ranks' areas.
 * Returns cudaError_t as int. */
int gsb_shared_atomic_cluster_launch(uint32_t unit, uint32_t n, uint32_t clusters, const gsb_shared_atomic_args *a,
                                     cudaStream_t stream);
/* cudaOccupancyMaxActiveClusters of `unit`'s clusters of n CTAs with `smem_bytes` each (0 when none fits). */
int gsb_shared_atomic_max_clusters(uint32_t unit, uint32_t n, int smem_bytes, int *clusters);
/* Load its kernels into the CURRENT context, let each take `smem_bytes` of dynamic shared memory and allow clusters of
 * 16. */
int gsb_shared_atomic_kernel_preload(int smem_bytes);

#endif /* GSB_INTERNAL_H_ */
