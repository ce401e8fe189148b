/* Synthetic Filecoin tipset builder — C ABI (test / bench infrastructure).
 *
 * Produces, deterministically from (seed, params), the IPLD block set a Lotus node
 * would serve for one parent/child tipset pair, in the flat form the engine ingests:
 *   cids[n][38] | offsets[n] | lengths[n] | blob        (blocks 16-byte aligned)
 * plus the "what came over RPC" descriptor (reference src/client/types.rs:13-58:
 * ApiTipset.cids / blocks[].messages / parent_message_receipts / parent_state_root,
 * and the ChainGetParentReceipts events roots used at events/generator.rs:199-211).
 *
 * Shapes follow SURVEY.md §8(d) / Appendix A. CPU only; never linked into the
 * product library.
 */
#ifndef IPCFP_SYNTH_H
#define IPCFP_SYNTH_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct synth_params {
    uint64_t seed;
    uint64_t n_receipts;        /* N messages / receipts in the parent tipset              */
    uint32_t events_per_receipt;/* E                                                        */
    uint32_t match_ppm;         /* receipts carrying exactly one forced matching event      */
    uint32_t has_actor_filter;  /* spec carries actor_id_filter = Some(target_actor)        */
    uint64_t target_actor;      /* emitter of forced events when has_actor_filter           */
    uint32_t bw3_permille;      /* events AMTs with bit_width 3 (else 5)                    */
    uint32_t case_a_permille;   /* events encoded as `topics`/`data` (evm.rs:20-30)         */
    uint32_t malformed_permille;/* Case-B events whose t2 is 31 bytes (evm.rs:45-47)        */
    uint32_t null_root_permille;/* receipts with events_root = null (generator.rs:210)      */
    uint32_t n_parents;         /* parent blocks (each has a BLS and a SECP message AMT)    */
    uint32_t dup_msgs;          /* messages repeated in a later block's BLS AMT             */
    uint32_t with_state_tree;   /* build StateRoot + actors HAMT + EVM actors               */
    uint32_t n_actors;          /* actors in the state tree (IDs 1000..)                    */
    uint64_t hamt_entries;      /* entries in the target actor's storage HAMT               */
    uint64_t shard_lo, shard_hi;/* materialise events blocks only for receipts in [lo,hi);
                                   0,0 = everything                                          */
    uint32_t threads;           /* 0 = hardware_concurrency                                 */
    uint32_t same_topic1;       /* config 1: every event shares the target topic1           */
    uint32_t event_shapes;      /* 0: the fixed shapes above; 1: varied events (emitter heads, topic
                                   counts, data sizes, codecs, flags, duplicate / unknown keys,
                                   near misses) and 0..events_per_receipt events per receipt  */
} synth_params;

typedef struct synth_tipset synth_tipset;

void synth_default_params(synth_params* p);
synth_tipset* synth_build(const synth_params* p);
void synth_free(synth_tipset* t);

/* flat block set */
uint64_t synth_n_blocks(const synth_tipset*);
const uint8_t* synth_cids(const synth_tipset*);      /* n × 38 */
const uint64_t* synth_offsets(const synth_tipset*);  /* n      */
const uint32_t* synth_lengths(const synth_tipset*);  /* n      */
const uint8_t* synth_blob(const synth_tipset*);
uint64_t synth_blob_size(const synth_tipset*);

/* tipset descriptor */
int64_t synth_parent_epoch(const synth_tipset*);
int64_t synth_child_epoch(const synth_tipset*);
uint32_t synth_n_parents(const synth_tipset*);
const uint8_t* synth_parent_cids(const synth_tipset*);        /* n_parents × 38 */
const uint8_t* synth_parent_txmeta_cids(const synth_tipset*); /* n_parents × 38 */
const uint8_t* synth_child_cid(const synth_tipset*);          /* 38 */
const uint8_t* synth_receipts_root(const synth_tipset*);      /* 38 */
const uint8_t* synth_parent_state_root(const synth_tipset*);  /* 38 (child.blocks[0].parent_state_root) */
uint64_t synth_n_receipts(const synth_tipset*);
const uint8_t* synth_events_roots(const synth_tipset*);       /* n_receipts × 38 (zeros when absent) */
const uint8_t* synth_has_events_root(const synth_tipset*);    /* n_receipts */

/* what the spec should be */
const char* synth_event_signature(const synth_tipset*);
const char* synth_topic1(const synth_tipset*);
uint64_t synth_target_actor(const synth_tipset*);
/* ground truth by construction: receipts that carry a forced matching event */
uint64_t synth_n_selected(const synth_tipset*);
const uint64_t* synth_selected(const synth_tipset*);

/* storage side */
const uint8_t* synth_storage_root(const synth_tipset*);  /* contract_state CID of target actor, 38 */
/* key32 / value of storage entry k (k < hamt_entries; k == hamt_entries → the
 * calculate_storage_slot("calib-subnet-1", 0) entry). Returns value length. */
uint32_t synth_storage_entry(const synth_tipset*, uint64_t k, uint8_t key32[32], uint8_t value[32]);
/* an absent key */
void synth_storage_absent_key(const synth_tipset*, uint64_t k, uint8_t key32[32]);

/* CPU hash helpers exported for test vectors */
void synth_blake2b256(const uint8_t* in, uint64_t len, uint8_t out[32]);
void synth_keccak256(const uint8_t* in, uint64_t len, uint8_t out[32]);
void synth_sha256(const uint8_t* in, uint64_t len, uint8_t out[32]);

#ifdef __cplusplus
}
#endif
#endif
