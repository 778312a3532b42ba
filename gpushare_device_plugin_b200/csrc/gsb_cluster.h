/*
 * gsb_cluster.h — the SM-to-SM check's geometry and words, shared by its sm_90a kernels (cluster_check_sm90a.cu), the
 * host half of the probe (gsb_device.cu, gsb_cluster.cc) and, compiled as C, the tests' host build.
 *
 * A CTA's dynamic shared memory of smem_bytes is a GSB_CLUSTER_HEADER_BYTES header and then its area of
 * area_words = (smem_bytes - header) / 16 words of 16 bytes. The area holds `slots` regions of region_words words each:
 * one per peer (n - 1 slots), or one per rank for MULTICAST (n slots). BULK_S2S only gives half the area to its regions:
 * its send tiles, one per peer, lie right after them. region_words is a multiple of 8 words (128 bytes).
 *
 * In the area of owner o, the region of peer q is slot (q - o - 1) mod n, and slot j belongs to peer (o + 1 + j) mod n
 * (MULTICAST: slot j is rank j's). The owner is the receiver on every path but DSMEM_LD, where each CTA fills its own
 * area for its peers to read.
 *
 * Word i of what rank s sends rank d on path p is gsb_pattern_word(word_addr(p, n, s, d, i), gsb_seed_key(seed)), and
 * word j of owner o's background is gsb_pattern_word(bg_addr(p, n, o, j), bg_key(seed)): both addresses are unique in
 * a launch, so a word that landed in the wrong CTA or region, or never landed, is wrong and says where it came from.
 */
#ifndef GSB_CLUSTER_H_
#define GSB_CLUSTER_H_

#include <stdint.h>

#include "../../include/gpushare_b200.h"
#include "gsb_pattern.h"

#define GSB_CLUSTER_BG_SALT 0x4247424Bu  /* "BGBK": the background's seed differs from the data's */
#define GSB_CLUSTER_REGION_ALIGN 8u      /* words */

GSB_HD uint32_t gsb_cluster_area_words(uint32_t smem_bytes) {
  return smem_bytes > GSB_CLUSTER_HEADER_BYTES ? (smem_bytes - GSB_CLUSTER_HEADER_BYTES) / 16u : 0u;
}

GSB_HD uint32_t gsb_cluster_slots(uint32_t p, uint32_t n) { return p == GSB_CLUSTER_PATH_MULTICAST ? n : n - 1u; }

GSB_HD uint32_t gsb_cluster_region_words(uint32_t p, uint32_t n, uint32_t smem_bytes) {
  uint32_t aw = gsb_cluster_area_words(smem_bytes);
  if (p == GSB_CLUSTER_PATH_BULK_S2S) aw /= 2u;
  return aw / gsb_cluster_slots(p, n) / GSB_CLUSTER_REGION_ALIGN * GSB_CLUSTER_REGION_ALIGN;
}

/* the slot of peer q's region in owner o's area */
GSB_HD uint32_t gsb_cluster_slot(uint32_t p, uint32_t n, uint32_t o, uint32_t q) {
  return p == GSB_CLUSTER_PATH_MULTICAST ? q : (q + n - o - 1u) % n;
}

/* the peer whose region is slot j of owner o's area */
GSB_HD uint32_t gsb_cluster_peer(uint32_t p, uint32_t n, uint32_t o, uint32_t j) {
  return p == GSB_CLUSTER_PATH_MULTICAST ? j : (o + 1u + j) % n;
}

GSB_HD uint64_t gsb_cluster_word_addr(uint32_t p, uint32_t n, uint32_t s, uint32_t d, uint32_t i) {
  return (uint64_t)p << 56 | (uint64_t)(n - 1u) << 48 | (uint64_t)s << 40 | (uint64_t)(d & 0xFFu) << 32 | i;
}

GSB_HD uint64_t gsb_cluster_bg_addr(uint32_t p, uint32_t n, uint32_t o, uint32_t j) {
  return 1ull << 63 | (uint64_t)p << 56 | (uint64_t)(n - 1u) << 48 | (uint64_t)o << 40 | 0xFEull << 32 | j;
}

GSB_HD uint32_t gsb_cluster_bg_key(uint32_t seed) { return gsb_seed_key(seed ^ GSB_CLUSTER_BG_SALT); }

/* the dynamic shared memory the hook's region sizes are bounded at: the H100's 227 KiB opt-in maximum */
#define GSB_CLUSTER_SCRIPT_SMEM (GSB_CLUSTER_HEADER_BYTES + 16u * GSB_CLUSTER_HOOK_INDEX_MAX)

/* gsb_test_cluster_script's script, as the twin kernels (cluster_script_sm90a.cu) read it from device memory: route is
 * indexed s * n + d with the launch's n */
typedef struct gsb_cluster_script {
  uint32_t region_words;
  uint8_t route[GSB_CLUSTER_MAX_N * GSB_CLUSTER_MAX_N];
} gsb_cluster_script;

#ifdef __cplusplus
/* gsb_test_cluster_script's refusals (gsb_cluster.cc); route NULL checks the path and n only */
bool gsb_cluster_script_valid(uint32_t p, uint32_t n, uint32_t region_words, const uint8_t *route);
#endif

#endif /* GSB_CLUSTER_H_ */
