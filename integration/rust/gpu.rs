//! `src/proofs/gpu.rs` — drop-in GPU path for consensus-shipyard/ipc-filecoin-proofs over `libipcfp.so`.
//!
//! What a maintainer adds to the reference crate (with `ipcfp-sys = { path = "…/integration/rust/ipcfp-sys" }` in Cargo.toml and
//! `pub mod gpu;` in `src/proofs/mod.rs`). It keeps the reference's own types and signatures:
//!
//! * `GpuBlockstore` implements `fvm_ipld_blockstore::Blockstore` (the trait the generators are generic over —
//!   `src/proofs/events/generator.rs:60`, `src/proofs/storage/generator.rs:29`, `src/proofs/storage/decode.rs:36`);
//! * `generate_event_proof_gpu` replaces the body of `generate_event_proof` (`src/proofs/events/generator.rs:60-107`);
//! * `generate_storage_proof_gpu` replaces `generate_storage_proof` (`src/proofs/storage/generator.rs:29-67`), batched;
//! * `generate_proof_bundle_gpu` replaces the two loops of `generate_proof_bundle` (`src/proofs/generator.rs:25-95`);
//!   `generate_proof_bundle_logs_gpu` is the same bundle with eth_getLogs-style log filters in place of event specs;
//! * `verify_event_proof_gpu` / `verify_storage_proof_gpu` replace `verify_event_proof` / `verify_storage_proof`
//!   (`src/proofs/events/verifier.rs:51-74`, `src/proofs/storage/verifier.rs:24-63`) with every witness block CID-checked.
//!
//! NOT COMPILED IN THE ENGINE'S REPO (its build image has no Rust toolchain and the reference's crates are not vendored there);
//! the same C-ABI calls, in the same order, are exercised through Python `ctypes` by the engine's tests and bench.
use std::ffi::CString;
use std::os::raw::c_void;

use anyhow::{anyhow, bail, Result};
use cid::Cid;
use ethereum_types::H256;
use fvm_ipld_blockstore::Blockstore;
use ipcfp_sys as sys;

use crate::client::types::{ApiReceipt, ApiTipset};
use crate::proofs::common::bundle::{ProofBlock, UnifiedProofBundle, UnifiedVerificationResult};
use crate::proofs::events::bundle::{EventData, EventProof, EventProofBundle};
use crate::proofs::generator::{EventProofSpec, StorageProofSpec};
use crate::proofs::storage::bundle::StorageProof;

const CID_LEN: usize = sys::IPCFP_CID_LEN;

fn check(st: sys::ipcfp_status) -> Result<()> {
    if st == sys::IPCFP_OK {
        return Ok(());
    }
    let msg = unsafe { std::ffi::CStr::from_ptr(sys::ipcfp_last_error()) }.to_string_lossy().into_owned();
    let idx = unsafe { sys::ipcfp_last_error_index() };
    Err(anyhow!("ipcfp status {} at index {}: {}", st, idx as i64, msg))
}

/// 38 raw bytes of a Filecoin chain CID (v1, 32-byte digest) — the form the C ABI carries.
fn cid38(c: &Cid) -> Result<[u8; CID_LEN]> {
    let b = c.to_bytes();
    if b.len() != CID_LEN {
        bail!("CID {} is not a 38-byte CIDv1 with a 32-byte digest", c);
    }
    let mut out = [0u8; CID_LEN];
    out.copy_from_slice(&b);
    Ok(out)
}
fn cid_of_str(s: &str) -> Result<[u8; CID_LEN]> {
    cid38(&Cid::try_from(s)?)
}
fn cid_from38(b: &[u8]) -> Result<Cid> {
    Ok(Cid::try_from(b)?)
}
fn hex0x(b: &[u8]) -> String {
    format!("0x{}", hex::encode(b))
}

/// Device-resident block store: the `Blockstore` the generators read from, instead of `RpcBlockstore` / `CachedBlockstore`
/// (`src/client/blockstore.rs:20-37`, `src/client/cached_blockstore.rs:53-85`).
pub struct GpuBlockstore {
    h: *mut sys::ipcfp_store,
    /// the packed block bytes as handed to `ipcfp_store_create`, kept when the caller asked for it (`ingest_keeping_blocks`): the
    /// array a by-reference witness (`IPCFP_WITNESS_BY_REFERENCE`) points into
    kept_blob: Option<Vec<u8>>,
}
unsafe impl Send for GpuBlockstore {}

impl GpuBlockstore {
    /// `blocks`: what the RPC layer fetched (`ChainReadObj` results, or a `CachedBlockstore`'s shared cache), in any order.
    /// `verify`: Blake2b-256 every block against its CID on the GPU (the check the reference never makes — SURVEY F6).
    pub fn ingest<'a, I>(blocks: I, device: i32, verify: bool) -> Result<Self>
    where
        I: IntoIterator<Item = (&'a Cid, &'a [u8])>,
    {
        Self::ingest_impl(blocks, device, verify, false)
    }
    /// As `ingest`, and the store keeps its host copy of the packed blocks: witnesses can then come back by reference
    /// (`generate_event_proof_gpu_by_reference`) — what a `CachedBlockstore` that outlives the proof holds anyway.
    pub fn ingest_keeping_blocks<'a, I>(blocks: I, device: i32, verify: bool) -> Result<Self>
    where
        I: IntoIterator<Item = (&'a Cid, &'a [u8])>,
    {
        Self::ingest_impl(blocks, device, verify, true)
    }
    fn ingest_impl<'a, I>(blocks: I, device: i32, verify: bool, keep: bool) -> Result<Self>
    where
        I: IntoIterator<Item = (&'a Cid, &'a [u8])>,
    {
        let mut cids: Vec<u8> = Vec::new();
        let mut offsets: Vec<u64> = Vec::new();
        let mut lengths: Vec<u32> = Vec::new();
        let mut blob: Vec<u8> = Vec::new();
        for (c, data) in blocks {
            cids.extend_from_slice(&cid38(c)?);
            while blob.len() % 16 != 0 {
                blob.push(0);
            }
            offsets.push(blob.len() as u64);
            lengths.push(u32::try_from(data.len())?);
            blob.extend_from_slice(data);
        }
        let mut h = std::ptr::null_mut();
        let st = unsafe {
            sys::ipcfp_store_create(
                cids.as_ptr(),
                offsets.as_ptr(),
                lengths.as_ptr(),
                blob.as_ptr(),
                blob.len() as u64,
                lengths.len() as u64,
                device,
                if verify { sys::IPCFP_STORE_VERIFY_CIDS } else { 0 },
                &mut h,
            )
        };
        if st != sys::IPCFP_OK {
            if !h.is_null() {
                unsafe { sys::ipcfp_store_destroy(h) };
            }
            check(st)?;
        }
        Ok(Self { h, kept_blob: if keep { Some(blob) } else { None } })
    }
    /// A CARv1 archive (`lotus chain export`, `Filecoin.ChainExport`, a decompressed snapshot) as the store, its sections found on the
    /// GPU (`ipcfp_store_create_car`): block k is section k, and the store keeps `car`, which by-reference witnesses index.
    pub fn from_car(car: Vec<u8>, device: i32, verify: bool) -> Result<Self> {
        let mut h = std::ptr::null_mut();
        let st = unsafe {
            sys::ipcfp_store_create_car(
                car.as_ptr(),
                car.len() as u64,
                device,
                if verify { sys::IPCFP_STORE_VERIFY_CIDS } else { 0 },
                &mut h,
                std::ptr::null_mut(),
            )
        };
        if st != sys::IPCFP_OK {
            if !h.is_null() {
                unsafe { sys::ipcfp_store_destroy(h) };
            }
            check(st)?;
        }
        Ok(Self { h, kept_blob: Some(car) })
    }
    /// The witness of a bundle as a store of its own (every block CID-checked): what the verifiers replay against.
    pub fn from_witness(blocks: &[ProofBlock], device: i32) -> Result<Self> {
        Self::ingest(blocks.iter().map(|b| (&b.cid, b.data.as_slice())), device, true)
    }
    pub fn raw(&self) -> *mut sys::ipcfp_store {
        self.h
    }
}
impl Drop for GpuBlockstore {
    fn drop(&mut self) {
        unsafe { sys::ipcfp_store_destroy(self.h) }
    }
}
impl Blockstore for GpuBlockstore {
    fn get(&self, k: &Cid) -> Result<Option<Vec<u8>>> {
        let c = cid38(k)?;
        let (mut len, mut found) = (0u32, 0i32);
        check(unsafe { sys::ipcfp_store_get(self.h, c.as_ptr(), std::ptr::null_mut(), 0, &mut len, &mut found) })?;
        if found == 0 {
            return Ok(None);
        }
        let mut buf = vec![0u8; len as usize];
        check(unsafe { sys::ipcfp_store_get(self.h, c.as_ptr(), buf.as_mut_ptr(), len, &mut len, &mut found) })?;
        Ok(Some(buf))
    }
    fn has(&self, k: &Cid) -> Result<bool> {
        let c = cid38(k)?;
        let mut found = 0i32;
        check(unsafe { sys::ipcfp_store_has(self.h, c.as_ptr(), &mut found) })?;
        Ok(found != 0)
    }
    fn put_keyed(&self, _k: &Cid, _block: &[u8]) -> Result<()> {
        unreachable!("read-only store, like RpcBlockstore (src/client/blockstore.rs:31)")
    }
}

/// Owned backing arrays of an `ipcfp_tipset_desc` (the inputs that came over RPC: `ApiTipset`, `Vec<ApiReceipt>`).
pub struct TipsetDesc {
    parent_cids: Vec<u8>,
    txmeta_cids: Vec<u8>,
    child_cid: [u8; CID_LEN],
    receipts_root: [u8; CID_LEN],
    state_root: [u8; CID_LEN],
    events_roots: Vec<u8>,
    has_root: Vec<u8>,
    parent_epoch: i64,
    child_epoch: i64,
}
impl TipsetDesc {
    /// `receipts`: `ChainGetParentReceipts(child.cids[0])` (events/generator.rs:199-204); may be empty for storage-only bundles.
    pub fn new(parent: &ApiTipset, child: &ApiTipset, receipts: &[ApiReceipt]) -> Result<Self> {
        if child.cids.is_empty() || child.blocks.is_empty() {
            bail!("child tipset has no blocks"); // extract_child_info, events/generator.rs:112-119
        }
        let mut parent_cids = Vec::with_capacity(parent.cids.len() * CID_LEN);
        for c in &parent.cids {
            parent_cids.extend_from_slice(&cid_of_str(&c.cid)?);
        }
        let mut txmeta_cids = Vec::with_capacity(parent.blocks.len() * CID_LEN);
        for b in &parent.blocks {
            txmeta_cids.extend_from_slice(&cid_of_str(&b.messages.cid)?);
        }
        if parent.cids.len() != parent.blocks.len() {
            bail!("parent tipset: {} cids but {} blocks", parent.cids.len(), parent.blocks.len());
        }
        let mut events_roots = vec![0u8; receipts.len() * CID_LEN];
        let mut has_root = vec![0u8; receipts.len()];
        for (i, r) in receipts.iter().enumerate() {
            if let Some(m) = &r.events_root {
                events_roots[i * CID_LEN..(i + 1) * CID_LEN].copy_from_slice(&cid_of_str(&m.cid)?);
                has_root[i] = 1;
            }
        }
        Ok(Self {
            parent_cids,
            txmeta_cids,
            child_cid: cid_of_str(&child.cids[0].cid)?,
            receipts_root: cid_of_str(&child.blocks[0].parent_message_receipts.cid)?,
            state_root: cid_of_str(&child.blocks[0].parent_state_root.cid)?,
            events_roots,
            has_root,
            parent_epoch: parent.height,
            child_epoch: child.height,
        })
    }
    fn raw(&self) -> sys::ipcfp_tipset_desc {
        sys::ipcfp_tipset_desc {
            parent_epoch: self.parent_epoch,
            child_epoch: self.child_epoch,
            n_parents: (self.parent_cids.len() / CID_LEN) as u32,
            parent_cids: self.parent_cids.as_ptr(),
            parent_txmeta_cids: self.txmeta_cids.as_ptr(),
            child_cid: self.child_cid.as_ptr(),
            receipts_root: self.receipts_root.as_ptr(),
            child_parent_state_root: self.state_root.as_ptr(),
            n_receipts: self.has_root.len() as u64,
            events_roots: self.events_roots.as_ptr(),
            has_events_root: self.has_root.as_ptr(),
        }
    }
}

struct SpecC {
    sig: CString,
    topic: CString,
    raw: sys::ipcfp_event_spec,
}
fn spec_c(event_signature: &str, topic_1: &str, actor_id_filter: Option<u64>) -> Result<SpecC> {
    let sig = CString::new(event_signature)?;
    let topic = CString::new(topic_1)?;
    let raw = sys::ipcfp_event_spec {
        event_signature: sig.as_ptr(),
        topic_1: topic.as_ptr(),
        has_actor_id_filter: actor_id_filter.is_some() as u8,
        actor_id_filter: actor_id_filter.unwrap_or(0),
    };
    Ok(SpecC { sig, topic, raw })
}

fn witness_blocks(w: &sys::ipcfp_witness) -> Result<Vec<ProofBlock>> {
    let n = w.n_blocks as usize;
    let mut out = Vec::with_capacity(n);
    for i in 0..n {
        let cid = cid_from38(unsafe { std::slice::from_raw_parts(w.cids.add(i * CID_LEN), CID_LEN) })?;
        let off = unsafe { *w.offsets.add(i) } as usize;
        let len = unsafe { *w.lengths.add(i) } as usize;
        let data = unsafe { std::slice::from_raw_parts(w.blob.add(off), len) }.to_vec();
        out.push(ProofBlock { cid, data });
    }
    Ok(out) // already in `Cid` Ord order, like WitnessCollector::materialize (common/witness.rs:43-56)
}

fn event_proofs_of(r: &sys::ipcfp_event_result, parent: &ApiTipset, child: &ApiTipset) -> Result<Vec<EventProof>> {
    let parent_tipset_cids: Vec<String> = parent.cids.iter().map(|m| m.cid.clone()).collect();
    let child_block_cid = child.cids[0].cid.clone();
    let mut proofs = Vec::with_capacity(r.n_proofs as usize);
    for k in 0..r.n_proofs as usize {
        let p = unsafe { &*r.proofs.add(k) };
        let topics = (0..p.n_topics as usize)
            .map(|t| hex0x(unsafe { std::slice::from_raw_parts(r.data_blob.add(p.topics_off as usize + 32 * t), 32) }))
            .collect();
        let data = hex0x(unsafe { std::slice::from_raw_parts(r.data_blob.add(p.data_off as usize), p.data_len as usize) });
        proofs.push(EventProof {
            parent_epoch: parent.height,
            child_epoch: child.height,
            parent_tipset_cids: parent_tipset_cids.clone(),
            child_block_cid: child_block_cid.clone(),
            message_cid: cid_from38(&p.message_cid)?.to_string(),
            exec_index: p.exec_index,
            event_index: p.event_index,
            event_data: EventData { emitter: p.emitter, topics, data }, // events/generator.rs:274-293
        });
    }
    Ok(proofs)
}

/// `generate_event_proof` (`src/proofs/events/generator.rs:60-107`) on the GPU: base witness, message-AMT recording, execution
/// order, two-pass scan, materialise — one C-ABI call.
pub fn generate_event_proof_gpu(
    store: &GpuBlockstore,
    parent: &ApiTipset,
    child: &ApiTipset,
    receipts: &[ApiReceipt],
    event_signature: &str,
    topic_1: &str,
    actor_id_filter: Option<u64>,
) -> Result<EventProofBundle> {
    let desc = TipsetDesc::new(parent, child, receipts)?;
    let spec = spec_c(event_signature, topic_1, actor_id_filter)?;
    let mut out = std::ptr::null_mut();
    check(unsafe { sys::ipcfp_generate_event_proof(store.h, &desc.raw(), &spec.raw, 0, &mut out) })?;
    let r = unsafe { &*out };
    let res = (|| -> Result<EventProofBundle> {
        Ok(EventProofBundle { proofs: event_proofs_of(r, parent, child)?, blocks: witness_blocks(&r.witness)? })
    })();
    unsafe { sys::ipcfp_event_result_free(out) };
    let _keep = (&spec.sig, &spec.topic);
    res
}

/// One rank's handle on the library's cross-shard protocol (`ipcfp_comm_init`, DESIGN.md §6): two NCCL communicators and the
/// exchange streams of this process's GPU. Rank 0 makes the id with [`ShardedComm::unique_id`] and hands the 128 bytes to the other
/// ranks by any means the host already has (the reference's own RPC, MPI, a file).
pub struct ShardedComm {
    h: *mut sys::ipcfp_comm,
    world: u32,
    rank: u32,
}
unsafe impl Send for ShardedComm {}

impl ShardedComm {
    pub fn unique_id() -> Result<[u8; sys::IPCFP_COMM_ID_BYTES]> {
        let mut id = [0u8; sys::IPCFP_COMM_ID_BYTES];
        check(unsafe { sys::ipcfp_comm_unique_id(id.as_mut_ptr()) })?;
        Ok(id)
    }
    pub fn new(id: &[u8; sys::IPCFP_COMM_ID_BYTES], world: u32, rank: u32, device: i32) -> Result<Self> {
        let mut h = std::ptr::null_mut();
        check(unsafe { sys::ipcfp_comm_init(id.as_ptr(), world, rank, device, &mut h) })?;
        Ok(Self { h, world, rank })
    }
}
impl Drop for ShardedComm {
    fn drop(&mut self) {
        unsafe { sys::ipcfp_comm_destroy(self.h) }
    }
}

/// What one rank holds after a sharded call: its own proofs and witness blocks, and its part of the merged witness CID set.
pub struct ShardedEventProof {
    /// proofs of the receipts this rank owns (`message_cid` and `exec_index` final: the execution order was resolved across shards)
    pub proofs: Vec<EventProof>,
    /// this shard's witness blocks in `Cid` order
    pub blocks: Vec<ProofBlock>,
    /// entries `[union_first, union_first + union_part.len())` of the `BTreeSet<Cid>` union over ALL shards (`common/witness.rs:24-40`);
    /// the parts of ranks 0..world, concatenated, are the whole sorted set of `union_total` CIDs
    pub union_part: Vec<Cid>,
    pub union_first: u64,
    pub union_total: u64,
    pub total_matching: u64,
    pub total_proofs: u64,
}

/// `generate_event_proof` (`src/proofs/events/generator.rs:60-107`) for ONE tipset split over `comm.world` GPUs by receipt index:
/// rank r scans receipts `bounds[r]..bounds[r+1]` out of a store that holds the blocks that range needs. Every rank must make the
/// call; they succeed or fail together, naming the error the single-store call on the whole tipset would have named.
pub fn generate_event_proof_sharded_gpu(
    comm: &ShardedComm,
    store: &GpuBlockstore,
    parent: &ApiTipset,
    child: &ApiTipset,
    receipts: &[ApiReceipt],
    bounds: &[u64],
    event_signature: &str,
    topic_1: &str,
    actor_id_filter: Option<u64>,
) -> Result<ShardedEventProof> {
    if bounds.len() != comm.world as usize + 1 {
        return Err(anyhow!("bounds must hold world + 1 receipt indices"));
    }
    let desc = TipsetDesc::new(parent, child, receipts)?;
    let spec = spec_c(event_signature, topic_1, actor_id_filter)?;
    let mut tip = std::ptr::null_mut();
    check(unsafe { sys::ipcfp_tipset_upload(store.h, &desc.raw(), &mut tip) })?;
    let mut out = std::ptr::null_mut();
    let st = unsafe {
        sys::ipcfp_generate_event_proof_sharded(comm.h, store.h, tip, &spec.raw, bounds.as_ptr(), sys::IPCFP_SHARDED_UNION_TO_HOST, &mut out)
    };
    unsafe { sys::ipcfp_tipset_free(tip) };
    check(st)?;
    let r = unsafe { &*out };
    let res = (|| -> Result<ShardedEventProof> {
        let part = unsafe { std::slice::from_raw_parts(r.union_cids, r.n_union_part as usize * CID_LEN) };
        let mut union_part = Vec::with_capacity(r.n_union_part as usize);
        for c in part.chunks_exact(CID_LEN) {
            union_part.push(Cid::try_from(c)?);
        }
        Ok(ShardedEventProof {
            proofs: event_proofs_of(r, parent, child)?,
            blocks: witness_blocks(&r.witness)?,
            union_part,
            union_first: r.union_part_first,
            union_total: r.n_union_cids,
            total_matching: r.total_matching,
            total_proofs: r.total_proofs,
        })
    })();
    unsafe { sys::ipcfp_event_result_free(out) };
    let _keep = (&spec.sig, &spec.topic, comm.rank);
    res
}

/// `generate_event_proof_gpu` with the witness BY REFERENCE (`IPCFP_WITNESS_BY_REFERENCE`): the GPU returns CIDs / offsets / lengths
/// only and `ProofBlock.data` is sliced out of the store's own host copy of the blocks — 50 bytes per witness block cross PCIe instead
/// of the block bytes. The store must have been built with `ingest_keeping_blocks`.
pub fn generate_event_proof_gpu_by_reference(
    store: &GpuBlockstore,
    parent: &ApiTipset,
    child: &ApiTipset,
    receipts: &[ApiReceipt],
    event_signature: &str,
    topic_1: &str,
    actor_id_filter: Option<u64>,
) -> Result<EventProofBundle> {
    let blob = store.kept_blob.as_ref().ok_or_else(|| anyhow!("store was not built with ingest_keeping_blocks"))?;
    let desc = TipsetDesc::new(parent, child, receipts)?;
    let spec = spec_c(event_signature, topic_1, actor_id_filter)?;
    let mut out = std::ptr::null_mut();
    check(unsafe { sys::ipcfp_generate_event_proof(store.h, &desc.raw(), &spec.raw, sys::IPCFP_WITNESS_BY_REFERENCE, &mut out) })?;
    let r = unsafe { &*out };
    let res = (|| -> Result<EventProofBundle> {
        let w = &r.witness;
        let mut blocks = Vec::with_capacity(w.n_blocks as usize);
        for i in 0..w.n_blocks as usize {
            let cid = cid_from38(unsafe { std::slice::from_raw_parts(w.cids.add(i * CID_LEN), CID_LEN) })?;
            let off = unsafe { *w.offsets.add(i) } as usize; // into the blob this store was created from
            let len = unsafe { *w.lengths.add(i) } as usize;
            let data = blob.get(off..off + len).ok_or_else(|| anyhow!("witness block {} outside the kept blob", i))?.to_vec();
            blocks.push(ProofBlock { cid, data });
        }
        Ok(EventProofBundle { proofs: event_proofs_of(r, parent, child)?, blocks })
    })();
    unsafe { sys::ipcfp_event_result_free(out) };
    let _keep = (&spec.sig, &spec.topic);
    res
}

fn storage_proof_of(p: &sys::ipcfp_storage_proof, child: &ApiTipset, desc: &TipsetDesc) -> Result<StorageProof> {
    Ok(StorageProof {
        child_epoch: child.height,
        child_block_cid: child.cids[0].cid.clone(),
        parent_state_root: cid_from38(&desc.state_root)?.to_string(),
        actor_id: p.actor_id,
        actor_state_cid: cid_from38(&p.actor_state_cid)?.to_string(),
        storage_root: cid_from38(&p.storage_root)?.to_string(),
        slot: hex0x(&p.slot),
        value: hex0x(&p.value), // create_proof_claim, storage/generator.rs:158-178
    })
}

/// `generate_storage_proof` (`src/proofs/storage/generator.rs:29-67`), batched over specs: → per spec `(StorageProof, Vec<ProofBlock>)`.
pub fn generate_storage_proof_gpu(
    store: &GpuBlockstore,
    parent: &ApiTipset,
    child: &ApiTipset,
    specs: &[StorageProofSpec],
) -> Result<Vec<(StorageProof, Vec<ProofBlock>)>> {
    let desc = TipsetDesc::new(parent, child, &[])?;
    let cs: Vec<sys::ipcfp_storage_spec> = specs.iter().map(|s| sys::ipcfp_storage_spec { actor_id: s.actor_id, slot: s.slot.0 }).collect();
    let mut out = std::ptr::null_mut();
    check(unsafe { sys::ipcfp_generate_storage_proofs(store.h, &desc.raw(), cs.as_ptr(), cs.len() as u64, &mut out) })?;
    let r = unsafe { &*out };
    let res = (|| -> Result<Vec<(StorageProof, Vec<ProofBlock>)>> {
        let all = witness_blocks(&r.witness)?;
        let mut v = Vec::with_capacity(cs.len());
        for i in 0..r.n_proofs as usize {
            let p = unsafe { &*r.proofs.add(i) };
            let (a, b) = unsafe { (*r.spec_witness_offsets.add(i) as usize, *r.spec_witness_offsets.add(i + 1) as usize) };
            let blocks = (a..b).map(|k| all[unsafe { *r.spec_witness_index.add(k) } as usize].clone()).collect();
            v.push((storage_proof_of(p, child, &desc)?, blocks));
        }
        Ok(v)
    })();
    unsafe { sys::ipcfp_storage_result_free(out) };
    res
}

/// One Solidity value by its storage path (`ipcfp.h`, "Storage paths"): the caller's `ipcfp_storage_path` (steps and keys borrowed for
/// the call) → its status, its value (the words, or the decoded bytes) and the proofs of its expanded specs with their blocks, as
/// `generate_storage_proof_gpu` returns them.
pub struct StoragePathValue {
    pub status: u32,
    pub value: Vec<u8>,
    pub proofs: Vec<(StorageProof, Vec<ProofBlock>)>,
}
pub fn generate_storage_path_proofs_gpu(
    store: &GpuBlockstore,
    parent: &ApiTipset,
    child: &ApiTipset,
    paths: &[sys::ipcfp_storage_path],
) -> Result<Vec<StoragePathValue>> {
    let desc = TipsetDesc::new(parent, child, &[])?;
    let mut tip = std::ptr::null_mut();
    check(unsafe { sys::ipcfp_tipset_upload(store.h, &desc.raw(), &mut tip) })?;
    let mut out = std::ptr::null_mut();
    let st = unsafe { sys::ipcfp_generate_storage_path_proofs_resident(store.h, tip, paths.as_ptr(), paths.len() as u64, 0, &mut out) };
    unsafe { sys::ipcfp_tipset_free(tip) };
    check(st)?;
    let r = unsafe { &*out };
    let res = (|| -> Result<Vec<StoragePathValue>> {
        let s = unsafe { &*r.storage };
        let all = witness_blocks(&s.witness)?;
        let mut v = Vec::with_capacity(paths.len());
        for i in 0..r.n_paths as usize {
            let pv = unsafe { &*r.paths.add(i) };
            let value = unsafe { std::slice::from_raw_parts(r.value_blob.add(pv.value_off as usize), pv.value_len as usize) }.to_vec();
            let mut proofs = Vec::with_capacity(pv.n_specs as usize);
            for k in pv.first_spec as usize..(pv.first_spec + pv.n_specs) as usize {
                let p = unsafe { &*s.proofs.add(k) };
                let (a, b) = unsafe { (*s.spec_witness_offsets.add(k) as usize, *s.spec_witness_offsets.add(k + 1) as usize) };
                let blocks = (a..b).map(|j| all[unsafe { *s.spec_witness_index.add(j) } as usize].clone()).collect();
                proofs.push((storage_proof_of(p, child, &desc)?, blocks));
            }
            v.push(StoragePathValue { status: pv.status, value, proofs });
        }
        Ok(v)
    })();
    unsafe { sys::ipcfp_path_result_free(out) };
    res
}

/// `resolve_eth_address_to_actor_id` (`src/proofs/common/address.rs:8-62`) from the state tree at `state_root` (the child header's
/// ParentStateRoot) instead of `Filecoin.EthAddressToFilecoinAddress` + `Filecoin.StateLookupID`: the same validation and messages,
/// then the Init actor's address map walked on the GPU.
pub fn resolve_eth_address_to_actor_id_gpu(store: &GpuBlockstore, state_root: &Cid, eth_addr: &str) -> Result<u64> {
    let eth_addr = eth_addr.trim_start_matches("0x");
    let bytes = hex::decode(eth_addr).map_err(|e| anyhow!("Invalid hex in Ethereum address: {}", e))?;
    if bytes.len() != 20 {
        return Err(anyhow!("Invalid Ethereum address length: expected 20 bytes, got {}", bytes.len()));
    }
    let mut addr = sys::ipcfp_address { len: 0, bytes: [0u8; sys::IPCFP_ADDRESS_MAX] };
    check(unsafe { sys::ipcfp_address_from_eth(bytes.as_ptr(), &mut addr) })?;
    let root = cid38(state_root)?;
    let mut out = std::ptr::null_mut();
    check(unsafe { sys::ipcfp_resolve_addresses(store.h, root.as_ptr(), &addr, 1, &mut out) })?;
    let (st, id) = unsafe { (*(*out).status, *(*out).actor_ids) };
    unsafe { sys::ipcfp_resolve_result_free(out) };
    if st != sys::IPCFP_OK {
        bail!("Failed to lookup ID address: ipcfp status {}", st);
    }
    Ok(id)
}

/// An actor proof: the C record (actor_id, sequence, balance, code, head, delegated address, the EVM fields, `status`) with the bytecode
/// when asked for, and the blocks that prove it.
pub struct ActorProofGpu {
    pub proof: sys::ipcfp_actor_proof,
    pub bytecode: Vec<u8>,
    pub blocks: Vec<ProofBlock>,
}

/// `ipcfp_generate_actor_proofs`: what the state tree under `child`'s ParentStateRoot holds for each address (`Address::to_bytes()`),
/// or a proven absence. `evm_code_cids`: the EVM actor code CIDs of the network's manifests; `with_code`: the bytecode joins the proof.
pub fn generate_actor_proofs_gpu(
    store: &GpuBlockstore,
    child: &Cid,
    parent_state_root: &Cid,
    addresses: &[Vec<u8>],
    evm_code_cids: &[Cid],
    with_code: bool,
) -> Result<Vec<ActorProofGpu>> {
    let mut addrs = Vec::with_capacity(addresses.len());
    for a in addresses {
        if a.is_empty() || a.len() > sys::IPCFP_ADDRESS_MAX {
            bail!("address of {} bytes", a.len());
        }
        let mut c = sys::ipcfp_address { len: a.len() as u8, bytes: [0u8; sys::IPCFP_ADDRESS_MAX] };
        c.bytes[..a.len()].copy_from_slice(a);
        addrs.push(c);
    }
    let mut evm = Vec::with_capacity(CID_LEN * evm_code_cids.len());
    for c in evm_code_cids {
        evm.extend_from_slice(&cid38(c)?);
    }
    let (child_b, root_b, receipts) = (cid38(child)?, cid38(parent_state_root)?, [0u8; CID_LEN]);
    let mut d: sys::ipcfp_tipset_desc = unsafe { std::mem::zeroed() };
    d.child_cid = child_b.as_ptr();
    d.child_parent_state_root = root_b.as_ptr();
    d.receipts_root = receipts.as_ptr();   // not read by actor proofs
    let flags = if with_code { sys::IPCFP_ACTOR_WITH_CODE } else { 0 };
    let mut out = std::ptr::null_mut();
    check(unsafe {
        sys::ipcfp_generate_actor_proofs(store.h, &d, addrs.as_ptr(), addrs.len() as u64, evm.as_ptr(), evm_code_cids.len() as u64, flags, &mut out)
    })?;
    let r = unsafe { &*out };
    let result = (|| {
        let all = witness_blocks(&r.witness)?;
        let mut proofs = Vec::with_capacity(r.n_proofs as usize);
        for i in 0..r.n_proofs as usize {
            let p = unsafe { *r.proofs.add(i) };
            let bytecode = if p.code_len > 0 {
                unsafe { std::slice::from_raw_parts(r.code_blob.add(p.code_off as usize), p.code_len as usize) }.to_vec()
            } else {
                Vec::new()
            };
            let (lo, hi) = unsafe { (*r.proof_witness_offsets.add(i), *r.proof_witness_offsets.add(i + 1)) };
            let blocks = (lo..hi)
                .map(|k| {
                    let b = &all[unsafe { *r.proof_witness_index.add(k as usize) } as usize];
                    ProofBlock { cid: b.cid, data: b.data.clone() }
                })
                .collect();
            proofs.push(ActorProofGpu { proof: p, bytecode, blocks });
        }
        Ok(proofs)
    })();
    unsafe { sys::ipcfp_actor_result_free(out) };
    result
}

/// `generate_proof_bundle` (`src/proofs/generator.rs:25-95`): ONE store built from everything the RPC layer fetched for this tipset
/// pair, storage specs first, then event specs, then the `BTreeSet<(Cid, Vec<u8>)>` union of the witnesses.
pub fn generate_proof_bundle_gpu(
    store: &GpuBlockstore,
    parent: &ApiTipset,
    child: &ApiTipset,
    receipts: &[ApiReceipt],
    storage_specs: Vec<StorageProofSpec>,
    event_specs: Vec<EventProofSpec>,
) -> Result<UnifiedProofBundle> {
    let desc = TipsetDesc::new(parent, child, receipts)?;
    let ss: Vec<sys::ipcfp_storage_spec> = storage_specs.iter().map(|s| sys::ipcfp_storage_spec { actor_id: s.actor_id, slot: s.slot.0 }).collect();
    let es: Vec<SpecC> = event_specs
        .iter()
        .map(|s| spec_c(&s.event_signature, &s.topic_1, s.actor_id_filter))
        .collect::<Result<_>>()?;
    let es_raw: Vec<sys::ipcfp_event_spec> = es
        .iter()
        .map(|s| sys::ipcfp_event_spec {
            event_signature: s.sig.as_ptr(),
            topic_1: s.topic.as_ptr(),
            has_actor_id_filter: s.raw.has_actor_id_filter,
            actor_id_filter: s.raw.actor_id_filter,
        })
        .collect();
    let mut out = std::ptr::null_mut();
    check(unsafe {
        sys::ipcfp_generate_proof_bundle(store.h, &desc.raw(), ss.as_ptr(), ss.len() as u64, es_raw.as_ptr(), es_raw.len() as u64, &mut out)
    })?;
    unified_bundle_of(out, parent, child, &desc)
}

/// An eth_getLogs-style log filter (`ipcfp_log_filter`): `emitters` empty for any emitter, else actor IDs; `topics[k]` `None` for any
/// value at position k, else the 32-byte values topic k may take. A log needs at least `topics.len()` topics. The spec
/// `{sig, t1, actor}` is `LogFilter { emitters: actor.into_iter().collect(), topics: vec![Some(vec![keccak(sig)]), Some(vec![ascii_to_bytes32(t1)])] }`.
pub struct LogFilter {
    pub emitters: Vec<u64>,
    pub topics: Vec<Option<Vec<[u8; 32]>>>,
}

fn log_filter_c(f: &LogFilter) -> Result<sys::ipcfp_log_filter> {
    if f.topics.len() > 4 {
        bail!("a log filter has at most 4 topic positions");
    }
    let mut c = sys::ipcfp_log_filter {
        n_emitters: f.emitters.len() as u64,
        emitters: f.emitters.as_ptr(),
        n_positions: f.topics.len() as u32,
        _pad: 0,
        n_values: [0; 4],
        values: [std::ptr::null(); 4],
    };
    for (k, t) in f.topics.iter().enumerate() {
        if let Some(v) = t {
            c.n_values[k] = v.len() as u64;
            c.values[k] = v.as_ptr() as *const u8;
        }
    }
    Ok(c)
}

/// `generate_proof_bundle` with log filters in place of event specs (`ipcfp_generate_log_bundle`): the storage specs, then one
/// EventProofBundle per filter in order, then the union of the witnesses. A bundle of the filters the specs stand for is the spec
/// bundle, byte for byte.
pub fn generate_proof_bundle_logs_gpu(
    store: &GpuBlockstore,
    parent: &ApiTipset,
    child: &ApiTipset,
    receipts: &[ApiReceipt],
    storage_specs: Vec<StorageProofSpec>,
    log_filters: &[LogFilter],
) -> Result<UnifiedProofBundle> {
    let desc = TipsetDesc::new(parent, child, receipts)?;
    let ss: Vec<sys::ipcfp_storage_spec> = storage_specs.iter().map(|s| sys::ipcfp_storage_spec { actor_id: s.actor_id, slot: s.slot.0 }).collect();
    let fs: Vec<sys::ipcfp_log_filter> = log_filters.iter().map(log_filter_c).collect::<Result<_>>()?;
    let mut out = std::ptr::null_mut();
    check(unsafe {
        sys::ipcfp_generate_log_bundle(store.h, &desc.raw(), ss.as_ptr(), ss.len() as u64, fs.as_ptr(), fs.len() as u64, 0, &mut out)
    })?;
    unified_bundle_of(out, parent, child, &desc)
}

/// The logs of given messages with their proofs (`ipcfp_generate_message_log_proof`): the EventProofBundle of `log_filter` (`None`:
/// every log) restricted to the receipts of `message_cids`, and every message's position in the execution order (`None`: the tipset
/// did not execute it). Only the selected receipts' events AMTs are read.
pub fn generate_message_log_proof_gpu(
    store: &GpuBlockstore,
    parent: &ApiTipset,
    child: &ApiTipset,
    receipts: &[ApiReceipt],
    message_cids: &[Cid],
    log_filter: Option<&LogFilter>,
) -> Result<(EventProofBundle, Vec<Option<u64>>)> {
    let desc = TipsetDesc::new(parent, child, receipts)?;
    let mut cids = Vec::with_capacity(message_cids.len() * CID_LEN);
    for c in message_cids {
        cids.extend_from_slice(&cid38(c)?);
    }
    let f = log_filter.map(log_filter_c).transpose()?;
    let fp = f.as_ref().map_or(std::ptr::null(), |f| f as *const sys::ipcfp_log_filter);
    let mut idx = vec![0u64; message_cids.len()];
    let mut out = std::ptr::null_mut();
    check(unsafe {
        sys::ipcfp_generate_message_log_proof(store.h, &desc.raw(), cids.as_ptr(), message_cids.len() as u64, fp, 0, idx.as_mut_ptr(), &mut out)
    })?;
    let r = unsafe { &*out };
    let res = (|| -> Result<EventProofBundle> {
        Ok(EventProofBundle { proofs: event_proofs_of(r, parent, child)?, blocks: witness_blocks(&r.witness)? })
    })();
    unsafe { sys::ipcfp_event_result_free(out) };
    Ok((res?, idx.into_iter().map(|i| if i == u64::MAX { None } else { Some(i) }).collect()))
}

/// A message proof: the C record (`status`, `exec_index`, `exit_code`, `gas_used`, `events_root`, and with the body the message's
/// fields) with its return data and params. The witness is one union for all proofs.
pub struct MessageProofGpu {
    pub proof: sys::ipcfp_message_proof,
    pub return_data: Vec<u8>,
    pub params: Vec<u8>,
}

/// `ipcfp_generate_message_proofs`: whether each message (`message_cids`, as the parent blocks' message AMTs hold them) executed in the
/// tipset pair and how it ended, from the receipts AMT under the child header; `with_body`: the message block joins the witness and its
/// fields the proof. → (one proof per message in request order, the witness union in `Cid` order)
pub fn generate_message_proofs_gpu(
    store: &GpuBlockstore,
    parent: &ApiTipset,
    child: &ApiTipset,
    receipts: &[ApiReceipt],
    message_cids: &[Cid],
    with_body: bool,
) -> Result<(Vec<MessageProofGpu>, Vec<ProofBlock>)> {
    let desc = TipsetDesc::new(parent, child, receipts)?;
    let mut cids = Vec::with_capacity(message_cids.len() * CID_LEN);
    for c in message_cids {
        cids.extend_from_slice(&cid38(c)?);
    }
    let flags = if with_body { sys::IPCFP_MESSAGE_WITH_BODY } else { 0 };
    let mut out = std::ptr::null_mut();
    check(unsafe { sys::ipcfp_generate_message_proofs(store.h, &desc.raw(), cids.as_ptr(), message_cids.len() as u64, flags, &mut out) })?;
    let r = unsafe { &*out };
    let result = (|| {
        let bytes = |off: u64, len: u64| {
            if len == 0 { Vec::new() } else { unsafe { std::slice::from_raw_parts(r.data_blob.add(off as usize), len as usize) }.to_vec() }
        };
        let mut proofs = Vec::with_capacity(r.n_proofs as usize);
        for i in 0..r.n_proofs as usize {
            let p = unsafe { *r.proofs.add(i) };
            proofs.push(MessageProofGpu { proof: p, return_data: bytes(p.return_off, p.return_len), params: bytes(p.params_off, p.params_len) });
        }
        Ok((proofs, witness_blocks(&r.witness)?))
    })();
    unsafe { sys::ipcfp_message_result_free(out) };
    result
}

/// The UnifiedProofBundle of an `ipcfp_bundle`, which it frees.
fn unified_bundle_of(out: *mut sys::ipcfp_bundle, parent: &ApiTipset, child: &ApiTipset, desc: &TipsetDesc) -> Result<UnifiedProofBundle> {
    let b = unsafe { &*out };
    let res = (|| -> Result<UnifiedProofBundle> {
        let mut storage_proofs = Vec::new();
        if !b.storage.is_null() {
            let s = unsafe { &*b.storage };
            for i in 0..s.n_proofs as usize {
                storage_proofs.push(storage_proof_of(unsafe { &*s.proofs.add(i) }, child, desc)?);
            }
        }
        let mut event_proofs = Vec::new();
        for k in 0..b.n_event_results as usize {
            event_proofs.extend(event_proofs_of(unsafe { &**b.events.add(k) }, parent, child)?);
        }
        Ok(UnifiedProofBundle { storage_proofs, event_proofs, blocks: witness_blocks(&b.witness)? })
    })();
    unsafe { sys::ipcfp_bundle_free(out) };
    res
}

fn unhex32(s: &str) -> Result<[u8; 32]> {
    let mut b = [0u8; 32];
    hex::decode_to_slice(s.trim_start_matches("0x"), &mut b)?;
    Ok(b)
}

/// `verify_event_proof` (`src/proofs/events/verifier.rs:51-74`) on the GPU. The trust closures stay on the host (they are policy,
/// `:124-144`); `check_event` becomes an optional spec the event must match. Every witness block is hashed against its CID.
pub fn verify_event_proof_gpu(
    bundle: &EventProofBundle,
    is_trusted_parent_ts: &dyn Fn(i64, &[Cid]) -> bool,
    is_trusted_child_header: &dyn Fn(i64, &Cid) -> bool,
    check_event: Option<&EventProofSpec>,
    device: i32,
) -> Result<Vec<bool>> {
    if bundle.proofs.is_empty() {
        return Ok(vec![]);
    }
    let store = GpuBlockstore::from_witness(&bundle.blocks, device)?;
    let filter = match check_event {
        Some(s) => Some(spec_c(&s.event_signature, &s.topic_1, s.actor_id_filter)?),
        None => None,
    };
    let mut results = vec![false; bundle.proofs.len()];
    // proofs of one bundle share the tipset pair; group them by it so that each group is ONE batched call
    let mut groups: std::collections::BTreeMap<(i64, i64, Vec<String>, String), Vec<usize>> = Default::default();
    for (i, p) in bundle.proofs.iter().enumerate() {
        groups.entry((p.parent_epoch, p.child_epoch, p.parent_tipset_cids.clone(), p.child_block_cid.clone())).or_default().push(i);
    }
    for ((parent_epoch, child_epoch, parents, child), idxs) in groups {
        let parent_cids: Vec<Cid> = parents.iter().map(|s| Cid::try_from(s.as_str())).collect::<std::result::Result<_, _>>()?;
        let child_cid = Cid::try_from(child.as_str())?;
        if !is_trusted_parent_ts(parent_epoch, &parent_cids) || !is_trusted_child_header(child_epoch, &child_cid) {
            continue; // verify_trust_anchors → Ok(false)
        }
        let mut pc = Vec::with_capacity(parent_cids.len() * CID_LEN);
        for c in &parent_cids {
            pc.extend_from_slice(&cid38(c)?);
        }
        let cc = cid38(&child_cid)?;
        let desc = sys::ipcfp_tipset_desc {
            parent_epoch,
            child_epoch,
            n_parents: parent_cids.len() as u32,
            parent_cids: pc.as_ptr(),
            parent_txmeta_cids: std::ptr::null(),
            child_cid: cc.as_ptr(),
            receipts_root: std::ptr::null(),
            child_parent_state_root: std::ptr::null(),
            n_receipts: 0,
            events_roots: std::ptr::null(),
            has_events_root: std::ptr::null(),
        };
        let mut blob: Vec<u8> = Vec::new();
        let mut raw: Vec<sys::ipcfp_event_proof> = Vec::with_capacity(idxs.len());
        for &i in &idxs {
            let p = &bundle.proofs[i];
            let topics_off = blob.len() as u64;
            for t in &p.event_data.topics {
                blob.extend_from_slice(&unhex32(t)?);
            }
            let data_off = blob.len() as u64;
            let data = hex::decode(p.event_data.data.trim_start_matches("0x"))?;
            blob.extend_from_slice(&data);
            raw.push(sys::ipcfp_event_proof {
                exec_index: p.exec_index,
                event_index: p.event_index,
                emitter: p.event_data.emitter,
                n_topics: p.event_data.topics.len() as u32,
                data_len: data.len() as u32,
                data_off,
                topics_off,
                message_cid: cid_of_str(&p.message_cid)?,
                _pad: [0; 2],
            });
        }
        let mut res = vec![0u8; raw.len()];
        check(unsafe {
            sys::ipcfp_verify_event_proofs(
                store.h,
                &desc,
                raw.as_ptr(),
                raw.len() as u64,
                blob.as_ptr(),
                blob.len() as u64,
                filter.as_ref().map_or(std::ptr::null(), |f| &f.raw as *const _),
                res.as_mut_ptr(),
            )
        })?;
        for (k, &i) in idxs.iter().enumerate() {
            results[i] = res[k] != 0;
        }
    }
    Ok(results)
}

/// `verify_storage_proof` (`src/proofs/storage/verifier.rs:24-63`) for all storage proofs of a bundle at once.
pub fn verify_storage_proof_gpu(
    proofs: &[StorageProof],
    blocks: &[ProofBlock],
    is_trusted_child_header: &dyn Fn(i64, &Cid) -> bool,
    device: i32,
) -> Result<Vec<bool>> {
    if proofs.is_empty() {
        return Ok(vec![]);
    }
    let store = GpuBlockstore::from_witness(blocks, device)?;
    let mut results = vec![false; proofs.len()];
    let mut groups: std::collections::BTreeMap<(i64, String, String), Vec<usize>> = Default::default();
    for (i, p) in proofs.iter().enumerate() {
        groups.entry((p.child_epoch, p.child_block_cid.clone(), p.parent_state_root.clone())).or_default().push(i);
    }
    for ((child_epoch, child, psr), idxs) in groups {
        let child_cid = Cid::try_from(child.as_str())?;
        if !is_trusted_child_header(child_epoch, &child_cid) {
            continue; // verify_trust_anchor → Ok(false)
        }
        let cc = cid38(&child_cid)?;
        let sr = cid_of_str(&psr)?;
        let desc = sys::ipcfp_tipset_desc {
            parent_epoch: 0,
            child_epoch,
            n_parents: 0,
            parent_cids: std::ptr::null(),
            parent_txmeta_cids: std::ptr::null(),
            child_cid: cc.as_ptr(),
            receipts_root: std::ptr::null(),
            child_parent_state_root: sr.as_ptr(),
            n_receipts: 0,
            events_roots: std::ptr::null(),
            has_events_root: std::ptr::null(),
        };
        let mut raw = Vec::with_capacity(idxs.len());
        for &i in &idxs {
            let p = &proofs[i];
            raw.push(sys::ipcfp_storage_proof {
                actor_id: p.actor_id,
                actor_state_cid: cid_of_str(&p.actor_state_cid)?,
                storage_root: cid_of_str(&p.storage_root)?,
                slot: unhex32(&p.slot)?,
                value: unhex32(&p.value)?,
                found: 0,
                _pad: [0; 3],
                raw_len: 0,
            });
        }
        let mut res = vec![0u8; raw.len()];
        check(unsafe { sys::ipcfp_verify_storage_proofs(store.h, &desc, raw.as_ptr(), raw.len() as u64, res.as_mut_ptr()) })?;
        for (k, &i) in idxs.iter().enumerate() {
            results[i] = res[k] != 0;
        }
    }
    Ok(results)
}

struct TrustCtx<'a> {
    parent: &'a dyn Fn(i64, &[Cid]) -> bool,
    child: &'a dyn Fn(i64, &Cid) -> bool,
}
unsafe extern "C" fn trust_parent_tramp(ctx: *mut c_void, epoch: i64, cids: *const u8, n: u32) -> std::os::raw::c_int {
    let t = &*(ctx as *const TrustCtx);
    let raw = if n == 0 { &[][..] } else { std::slice::from_raw_parts(cids, n as usize * CID_LEN) };
    let parsed: std::result::Result<Vec<Cid>, _> = raw.chunks(CID_LEN).map(Cid::try_from).collect();
    parsed.map_or(0, |v| (t.parent)(epoch, &v) as std::os::raw::c_int)
}
unsafe extern "C" fn trust_child_tramp(ctx: *mut c_void, epoch: i64, cid: *const u8) -> std::os::raw::c_int {
    let t = &*(ctx as *const TrustCtx);
    Cid::try_from(std::slice::from_raw_parts(cid, CID_LEN)).map_or(0, |c| (t.child)(epoch, &c) as std::os::raw::c_int)
}

/// `verify_proof_bundle` (`src/proofs/verifier.rs:12-60`) straight from the bundle's JSON text (EventProofBundle or UnifiedProofBundle):
/// the parse, the witness store and both verifiers run on the GPU; text not in serde_json's canonical form is read by the host parser
/// with the same results. The trust closures are called at most once each, on this thread.
pub fn verify_proof_bundle_json(
    text: &str,
    is_trusted_parent_ts: &dyn Fn(i64, &[Cid]) -> bool,
    is_trusted_child_header: &dyn Fn(i64, &Cid) -> bool,
    check_event: Option<&EventProofSpec>,
    device: i32,
) -> Result<UnifiedVerificationResult> {
    let filter = match check_event {
        Some(s) => Some(spec_c(&s.event_signature, &s.topic_1, s.actor_id_filter)?),
        None => None,
    };
    let ctx = TrustCtx { parent: is_trusted_parent_ts, child: is_trusted_child_header };
    let mut out = std::ptr::null_mut();
    check(unsafe {
        sys::ipcfp_verify_bundle_json(
            text.as_ptr() as *const std::os::raw::c_char,
            text.len() as u64,
            device,
            Some(trust_parent_tramp),
            Some(trust_child_tramp),
            &ctx as *const TrustCtx as *mut c_void,
            filter.as_ref().map_or(std::ptr::null(), |f| &f.raw as *const _),
            &mut out,
        )
    })?;
    let v = unsafe { &*out };
    let bools = |p: *const u8, n: u64| if n == 0 { vec![] } else { unsafe { std::slice::from_raw_parts(p, n as usize) }.iter().map(|&x| x != 0).collect() };
    let res = UnifiedVerificationResult {
        storage_results: bools(v.storage_results, v.n_storage_proofs),
        event_results: bools(v.event_results, v.n_event_proofs),
    };
    unsafe { sys::ipcfp_bundle_verdict_free(out) };
    Ok(res)
}

/// `calculate_storage_slot` / `compute_mapping_slot` (`src/proofs/storage/utils.rs:5-19`) on the GPU, batched.
pub fn compute_mapping_slots_gpu(keys: &[[u8; 32]], slot_indices: &[u64], device: i32) -> Result<Vec<H256>> {
    if keys.len() != slot_indices.len() {
        bail!("keys / slot indices length mismatch");
    }
    let flat: Vec<u8> = keys.iter().flat_map(|k| k.iter().copied()).collect();
    let mut out = vec![0u8; 32 * keys.len()];
    check(unsafe { sys::ipcfp_compute_mapping_slots(flat.as_ptr(), slot_indices.as_ptr(), keys.len() as u64, device, out.as_mut_ptr()) })?;
    Ok(out.chunks(32).map(H256::from_slice).collect())
}

#[allow(dead_code)]
fn _assert_ffi_types(_: *mut c_void) {}
