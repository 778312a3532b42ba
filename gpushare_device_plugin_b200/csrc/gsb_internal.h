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

struct gsb_kernel_args {
  uint4 *base;                 /* arena base (device VA of absolute word 0) */
  unsigned long long first_word; /* absolute index of the window's first 16 B word */
  unsigned long long n_words;    /* words in the window */
  uint32_t seed_expect;        /* raw seed (the kernel mixes it) */
  uint32_t seed_write;
  const uint32_t *seed_table;  /* optional: raw expected seed per granule, indexed (w >> granule_shift) */
  uint32_t *table_update;      /* optional: last CTA stores seed_write for every granule the window covers */
  unsigned long long arena_words; /* words in the whole arena (tail-granule rule of table_update) */
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
/* Load every kernel this library can launch into the CURRENT context. Returns cudaError_t as int. */
int gsb_kernel_preload(void);
/* Upper bound of CTAs any geometry will use on a device with `sm_count` SMs (sizes `partials`). */
uint32_t gsb_kernel_max_grid(int sm_count);

#endif /* GSB_INTERNAL_H_ */
