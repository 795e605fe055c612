/* wide_oracle.c -- the sequential oracle (oracle/grove_oracle_seq.c, unchanged) compiled a second time for wide submissions:
 * clique records with 16-bit MinReplicas / replicas and GROVE_MAX_WIDE_GANG_PODS pods per gang.  The loops, the ordering and
 * the arithmetic are the oracle's own; only the clique record type, the per-gang pod limit (which also sizes the entry stack of
 * one evaluation: a fixed 2048 entries, 16 KB in the one evaluation record a cycle allocates) and the exported names differ.
 * TEST INFRASTRUCTURE ONLY (tests/wide_oracle.py).
 *
 * This holds as long as grove_oracle_seq.c (a) names the clique record only as grove_clique_t and reads its counts through it,
 * never holding a MinReplicas / replicas value in an 8-bit variable, and (b) bounds a gang's pods only by GROVE_MAX_GANG_PODS.
 * An edit there that breaks either makes this build diverge from the pass it restates; test_oracle_wide.py's hand cases
 * (600-pod PodGroups) and its equality with the ordinary oracle within the old limits are there to catch that. */
#include "../include/grove_place.h"

typedef struct wide_clique {
  uint32_t req_cpu_milli;
  uint32_t req_mem_mib;
  uint16_t req_gpu;
  uint16_t min_replicas;
  uint16_t replicas;
  uint16_t class_mask;
  uint8_t level;
  uint8_t scope;
} wide_clique_t;

#define grove_clique_t wide_clique_t
#undef GROVE_MAX_GANG_PODS
#define GROVE_MAX_GANG_PODS GROVE_MAX_WIDE_GANG_PODS
#define oracle_validate oracle_validate_wide
#define oracle_run_cycle oracle_run_cycle_wide
#define oracle_topology oracle_topology_wide
#define oracle_abi_version oracle_abi_version_wide

#include "../oracle/grove_oracle_seq.c"
