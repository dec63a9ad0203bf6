"""Document-sharded /retrieve across the GPUs of one box: one process per GPU
(`torch.distributed`, NCCL over NVLink), each rank holding rows
[rank*N/G, (rank+1)*N/G) of the dense matrix and the postings restricted to them
(SURVEY.md section 8e; the reference itself is single-process, manifests.go:81).

Per batch:  local dense top-P + local BM25 top-P (CUDA, per rank)
            -> ONE all-gather of the two key lists (B * 2P * 8 bytes per rank)
            -> merge G*P -> P per list, global BM25 ranks, fuse, top-k (CUDA, every rank).
BM25 statistics (N, avgdl, df[V]) are made global once at commit by an all-reduce, so the
scores do not depend on the sharding.

The stage kernels are reached through the `stages` object so that the distributed plumbing
(row partition, stats all-reduce, gather layout, ordinal bases) can be exercised on CPU
with gloo by the tests; the product always uses `NativeStages` (libkaito_rag, no fallback).
"""
from __future__ import annotations

import os

import numpy as np
import torch
import torch.distributed as dist


def shard_range(n_total: int, world_size: int, rank: int) -> tuple[int, int]:
    """Contiguous row range of `rank`: [lo, hi). Remainder rows go to the first ranks."""
    base, rem = divmod(n_total, world_size)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


class NativeStages:
    """CUDA stages of one shard (kaito_b200._native.Index on this rank's GPU)."""

    def __init__(self, ctx, index):
        self.ctx, self.index = ctx, index
        self.device = torch.device("cuda", ctx.device_id)

    def stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    # ---- mutations (the multi-GPU service: kaito_b200/sharded_engine.py)
    def add(self, node_ids, vecs, term_offsets=None, term_ids=None, term_tf=None, doc_len=None):
        self.index.add(node_ids, vecs, term_offsets, term_ids, term_tf, doc_len)

    def remove(self, node_ids) -> int:
        return self.index.remove(node_ids)

    def set_ordinal_map(self, base: int, stride: int):
        self.index.set_ordinal_map(base, stride)

    def n_rows(self) -> int:
        return int(self.index.stats().n_rows)

    def dim_padded(self) -> int:
        return int(self.index.stats().dim_padded)

    def persist(self, path: str):
        self.index.persist(path)

    def drop(self):
        if getattr(self, "_p2p", None) is not None:
            self._p2p.destroy()
            self._p2p = None
        self.index.drop()

    def commit_local(self, vocab):
        return self.index.commit_local(vocab)

    # redeal: compaction of the round-robin shards together (ShardedRetriever.compact)
    def alive_bitmap(self) -> np.ndarray:
        return self.index.alive_bitmap()

    def redeal_begin(self, alive_all: np.ndarray, window_rows: int):
        return self.index.redeal_begin(alive_all, window_rows)

    def redeal_prepare(self, recv_entries: np.ndarray):
        self.index.redeal_prepare(recv_entries)

    def redeal_pack(self, window: int, rows: torch.Tensor, entries: torch.Tensor):
        self.index.dev_redeal_pack(window, rows.data_ptr(), entries.data_ptr(), self.stream())

    def redeal_unpack(self, window: int, rows: torch.Tensor, entries: torch.Tensor):
        self.index.dev_redeal_unpack(window, rows.data_ptr(), entries.data_ptr(), self.stream())

    def redeal_finish(self) -> int:
        return self.index.redeal_finish(self.stream())

    def redeal_abort(self):
        self.index.redeal_abort()

    def commit_global(self, vocab, df, n_docs, total_len, ordinal_base):
        self.index.commit_global(vocab, df, n_docs, total_len, ordinal_base)

    def dense_candidates(self, q: torch.Tensor, P: int, out: torch.Tensor):
        self.index.dev_dense_candidates(q.shape[0], q.data_ptr(), P, out.data_ptr(), self.stream())

    def bm25_candidates(self, terms: torch.Tensor, toff: torch.Tensor, batch: int, P: int, out: torch.Tensor, toff_host=None):
        self.index.dev_bm25_candidates(batch, terms.data_ptr(), toff.data_ptr(), P, out.data_ptr(), self.stream(), toff_host)

    def merge(self, gathered: torch.Tensor, n_lists: int, batch: int, P: int, out: torch.Tensor):
        self.ctx.dev_merge(n_lists, batch, P, gathered.data_ptr(), out.data_ptr(), self.stream())

    # peer-memory exchange (our kernels over NVLink instead of NCCL all-gather + merge); ShardedRetriever sets it up
    P2P_MAX_BATCH, P2P_MAX_P = 1024, 256      # mailbox slot = 2 lists x 1024 x 256 keys (4 MiB per rank and parity)

    def p2p_setup(self, rank: int, world: int, group):
        from . import _native
        p = _native.P2PExchange(self.ctx, rank, world, self.P2P_MAX_BATCH, self.P2P_MAX_P)
        handles = [None] * world
        dist.all_gather_object(handles, p.handle.tobytes(), group=group)
        p.connect(np.frombuffer(b"".join(handles), np.uint8).copy())   # the caller's all-reduce is the barrier
        self._p2p = p

    def p2p_fits(self, nl: int, B: int, P: int) -> bool:
        return nl * B * P <= 2 * self.P2P_MAX_BATCH * self.P2P_MAX_P and P <= 1024

    def exchange_merge(self, local: torch.Tensor, merged: torch.Tensor):
        nl, B, P = local.shape
        self._p2p.exchange_merge(nl, B, P, local.data_ptr(), merged.data_ptr(), self.stream())

    def fuse(self, batch, P, k, dense_keys, bm25_keys, vw, tw, mode, out, allow=None):
        self.ctx.dev_fuse(batch, P, k, dense_keys.data_ptr(), None if bm25_keys is None else bm25_keys.data_ptr(), vw, tw,
                          mode, None if allow is None else allow.data_ptr(), out["final"].data_ptr(), out["dense"].data_ptr(), out["sparse"].data_ptr(),
                          out["rank"].data_ptr(), out["ordinal"].data_ptr(), out["count"].data_ptr(), self.stream())


class ShardedRetriever:
    """HybridRetriever._aretrieve (hybrid_retriever.py:205-237) over document shards."""

    def __init__(self, stages, device: torch.device, dim_padded: int, group=None):
        self.stages, self.device, self.dpad, self.group = stages, device, dim_padded, group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.hybrid = False
        self._buf = {}
        self.last_lists = None
        self._p2p_state = None

    # ------------------------------------------------------------------ index time
    def commit(self, vocab: int, n_local_rows: int, ordinal_base: int | None = None):
        """Global BM25 statistics: one all-reduce (df[V] + 2 scalars) and an all-gather of shard
        sizes for the ordinal bases (contiguous shards); `ordinal_base` overrides the base for shards that carry
        their own ordinal map (round-robin shards of the service: base = rank, stride = world)."""
        df, n_live, total_len = self.stages.commit_local(vocab)
        stats = torch.tensor([n_live, total_len], dtype=torch.int64, device=self.device)
        df_t = torch.from_numpy(df.astype(np.int64)).to(self.device)
        sizes = torch.zeros(self.world, dtype=torch.int64, device=self.device)
        sizes[self.rank] = n_local_rows
        if self.world > 1:
            dist.all_reduce(stats, group=self.group)
            dist.all_reduce(df_t, group=self.group)
            dist.all_reduce(sizes, group=self.group)
        n_docs, total = int(stats[0].item()), int(stats[1].item())
        base = int(sizes[: self.rank].sum().item()) if ordinal_base is None else int(ordinal_base)
        self.stages.commit_global(vocab, df_t.cpu().numpy().astype(np.uint32), n_docs, total, base)
        self.hybrid = True
        return n_docs, total, base

    # ------------------------------------------------------------------ compaction
    COMPACT_WINDOW_ROWS = 1 << 15     # new ordinals per window: at 768 dims about 150 MB of send staging per rank at most
    REDEAL_ENTRY_BYTES = 8

    def compact(self, vocab: int, window_rows: int | None = None) -> tuple[int, int]:
        """Remove the dead rows of round-robin shards (base = rank, stride = world) together, every rank in lock step: the live
        rows are renumbered in their old order and re-dealt across the shards as a fresh service would have dealt them
        (kaito_rag.h, krag_redeal_begin), then committed again.  The index must be unchanged since its last commit.
        Returns (rows reclaimed over all shards, this shard's rows afterwards).  A refusal or an allocation failure on any
        rank leaves every shard unchanged; a failure once rows have moved leaves the index unusable (drop it)."""
        st, dev, G = self.stages, self.device, self.world
        window_rows = window_rows or self.COMPACT_WINDOW_ROWS
        n_rows = st.n_rows()
        bm = st.alive_bitmap()
        meta = torch.zeros((G, 2), dtype=torch.int64, device=dev)
        meta[self.rank, 0], meta[self.rank, 1] = len(bm), n_rows
        if G > 1:
            dist.all_reduce(meta, group=self.group)
        words, n_total = int(meta[:, 0].max().item()), int(meta[:, 1].sum().item())
        loc = torch.zeros(max(words, 1), dtype=torch.int32, device=dev)
        if len(bm):
            loc[: len(bm)] = torch.from_numpy(bm.view(np.int32)).to(dev)
        gathered = torch.empty(G * loc.numel(), dtype=torch.int32, device=dev)
        if G > 1:
            dist.all_gather_into_tensor(gathered, loc, group=self.group)
        else:
            gathered.copy_(loc)
        alive_all = np.ascontiguousarray(gathered.cpu().numpy().view(np.uint32).reshape(G, -1)[:, :words])

        plan, err = None, None
        try:
            plan = st.redeal_begin(alive_all, window_rows)
        except Exception as e:
            err = e
        row_bytes = plan[2] if plan is not None else 0
        flag = self._sum(torch.tensor([0 if err is None else 1, row_bytes], dtype=torch.int64, device=dev))
        if flag[0] or flag[1] != G * row_bytes:
            if plan is not None:
                st.redeal_abort()
            raise err or RuntimeError("compaction refused on another rank (or the shards disagree on the row layout); "
                                      "every shard is unchanged")
        n_windows, n_live, row_bytes, send_rows, send_ents, recv_rows = plan
        if n_live == n_total:              # nothing dead: every rank sees the same bitmaps
            st.redeal_abort()
            return 0, n_rows

        recv_ents = np.zeros((n_windows, G), np.int64)
        if n_windows > 0:                  # recv_ents[k][t] = what shard t sends this shard in window k
            se = torch.from_numpy(send_ents).to(dev)
            g = torch.empty((G * n_windows, G), dtype=torch.int64, device=dev)
            if G > 1:
                dist.all_gather_into_tensor(g, se, group=self.group)
            else:
                g.copy_(se)
            recv_ents = np.ascontiguousarray(g.view(G, n_windows, G)[:, :, self.rank].T.cpu().numpy())
        err, bufs = None, None
        try:
            st.redeal_prepare(recv_ents)
            peak = lambda tab, per: max(1, int(tab.sum(axis=1).max(initial=0)) * per)
            bufs = [torch.empty(peak(send_rows, row_bytes), dtype=torch.uint8, device=dev),
                    torch.empty(peak(recv_rows, row_bytes), dtype=torch.uint8, device=dev),
                    torch.empty(peak(send_ents, self.REDEAL_ENTRY_BYTES), dtype=torch.uint8, device=dev),
                    torch.empty(peak(recv_ents, self.REDEAL_ENTRY_BYTES), dtype=torch.uint8, device=dev)]
        except Exception as e:
            err = e
        if self._sum(torch.tensor([0 if err is None else 1], dtype=torch.int64, device=dev))[0]:
            st.redeal_abort()
            raise err or RuntimeError("compaction failed on another rank before any row moved; every shard is unchanged")
        s_rows, r_rows, s_ents, r_ents = bufs
        try:
            for k in range(n_windows):
                st.redeal_pack(k, s_rows, s_ents)
                self._all_to_all(r_rows, s_rows, recv_rows[k] * row_bytes, send_rows[k] * row_bytes)
                self._all_to_all(r_ents, s_ents, recv_ents[k] * self.REDEAL_ENTRY_BYTES, send_ents[k] * self.REDEAL_ENTRY_BYTES)
                st.redeal_unpack(k, r_rows, r_ents)
            n_new = st.redeal_finish()
        except Exception:
            try:
                st.redeal_abort()        # rows were in flight: the shard is now unusable (drop it)
            except Exception:
                pass
            raise
        del bufs, s_rows, r_rows, s_ents, r_ents
        self.commit(vocab, n_new, ordinal_base=self.rank)
        return n_total - n_live, n_new

    def _sum(self, t: torch.Tensor) -> list[int]:
        if self.world > 1:
            dist.all_reduce(t, group=self.group)
        return [int(v) for v in t.cpu().tolist()]

    def _all_to_all(self, out: torch.Tensor, inp: torch.Tensor, out_splits, in_splits):
        o, i = int(np.sum(out_splits)), int(np.sum(in_splits))
        if self.world == 1:
            out[:o].copy_(inp[:i])
            return
        dist.all_to_all_single(out[:o], inp[:i], output_split_sizes=[int(x) for x in out_splits],
                               input_split_sizes=[int(x) for x in in_splits], group=self.group)

    # ------------------------------------------------------------------ query time
    def _use_p2p(self, nl: int, B: int, P: int) -> bool:
        """Peer-memory exchange when the stages provide it (NativeStages on a multi-GPU box); KRAG_P2P=0 keeps NCCL.
        Every rank takes the same decision: it depends only on (stages type, env, shapes) and setup is collective."""
        if self._p2p_state is None:
            ok = hasattr(self.stages, "p2p_setup") and self.device.type == "cuda" and os.environ.get("KRAG_P2P", "1") != "0"
            if ok:
                err = None
                try:
                    self.stages.p2p_setup(self.rank, self.world, self.group)
                except Exception as e:  # no peer access on this box: keep the NCCL path, loudly
                    err = e
                flag = torch.tensor([0 if err is None else 1], dtype=torch.int32, device=self.device)
                dist.all_reduce(flag, group=self.group)
                if int(flag.item()):
                    print(f"[kaito_b200] rank {self.rank}: peer-memory exchange unavailable ({err}); using NCCL all-gather", flush=True)
                    ok = False
            self._p2p_state = ok
        return self._p2p_state and self.stages.p2p_fits(nl, B, P)

    @staticmethod
    def _numel(shape) -> int:
        n = 1
        for s in shape:
            n *= int(s)
        return n

    def _storage(self, key, numel, dtype, **kw):
        """flat buffer of at least `numel` elements, grown in powers of two: the service's batches differ in size from call to
        call, and re-allocating (above all re-PINNING host memory: cudaHostAlloc synchronises the device and costs
        milliseconds) on every new shape was most of a sharded /retrieve batch"""
        t = self._buf.get(key)
        if t is None or t.dtype != dtype or t.numel() < numel:
            cap = 1024
            while cap < numel:
                cap <<= 1
            t = torch.empty((cap,), dtype=dtype, **kw)
            self._buf[key] = t
        return t

    def _tensor(self, name, shape, dtype):
        n = self._numel(shape)
        return self._storage(("dev", name), n, dtype, device=self.device)[:n].view(shape)

    def retrieve_dev(self, q: torch.Tensor, terms: torch.Tensor | None, toff: torch.Tensor | None, k: int,
                     cand_mult: float = 3.0, vector_weight: float = 0.7, text_weight: float = 0.3, mode: int = 0,
                     toff_host: np.ndarray | None = None, allow: torch.Tensor | None = None):
        """Inputs already on this rank's device (q: [B, dim_padded] fp32 zero padded).
        Returns a dict of device tensors [B, k] (+ count [B])."""
        B = q.shape[0]
        P = int(k * max(1.0, cand_mult))
        hybrid = self.hybrid and terms is not None
        nl = 2 if hybrid else 1
        local = self._tensor("local", (nl, B, P), torch.int64)
        self.stages.dense_candidates(q, P, local[0])
        if hybrid:
            self.stages.bm25_candidates(terms, toff, B, P, local[1], toff_host)
        if self.world > 1 and self._use_p2p(nl, B, P):
            merged = self._tensor("merged", (nl, B, P), torch.int64)
            self.stages.exchange_merge(local, merged)          # P2P stores + flag-waiting merge (our kernels over NVLink)
        elif self.world > 1:
            flat = self._tensor("gathered", (self.world * nl, B, P), torch.int64)
            dist.all_gather_into_tensor(flat, local, group=self.group)   # concatenation along dim 0
            gathered = flat.view(self.world, nl, B, P)
            merged = self._tensor("merged", (nl, B, P), torch.int64)
            # [G, nl, B, P] -> per list a [G, B, P] view (list stride = nl*B*P is handled by a copy-free slice
            # only when nl == 1; otherwise gather the two lists into contiguous blocks)
            if nl == 1:
                self.stages.merge(gathered, self.world, B, P, merged[0])
            else:
                per_list = gathered.transpose(0, 1).contiguous()  # [nl, G, B, P]
                self.stages.merge(per_list[0], self.world, B, P, merged[0])
                self.stages.merge(per_list[1], self.world, B, P, merged[1])
        else:
            merged = local
        self.last_lists = merged      # [nl, B, P] u64 keys: the global candidate lists of this call (dense, then BM25)
        out = {
            "final": self._tensor("final", (B, k), torch.float64), "dense": self._tensor("dense", (B, k), torch.float32),
            "sparse": self._tensor("sparse", (B, k), torch.float32), "rank": self._tensor("rank", (B, k), torch.int32),
            "ordinal": self._tensor("ordinal", (B, k), torch.int64), "count": self._tensor("count", (B,), torch.int32),
        }
        if allow is not None:       # keyword-side metadata post-filter (hybrid_retriever.py:227-235): bitmap over GLOBAL ordinals
            self.stages.fuse(B, P, k, merged[0], merged[1] if hybrid else None, vector_weight, text_weight, mode, out, allow=allow)
        else:
            self.stages.fuse(B, P, k, merged[0], merged[1] if hybrid else None, vector_weight, text_weight, mode, out)
        return out

    def embed_into(self, embedder, flat_tok: np.ndarray, tok_off: np.ndarray, q: torch.Tensor):
        """Query embeddings (K5) into q [B, dim_padded] on every rank.  The embedder weights are replicated; the
        QUERIES are split across the ranks (each embeds B/G of them) and the rows are all-gathered, so the
        embedding stage scales with the number of GPUs like the corpus scan does."""
        B = len(tok_off) - 1
        if self.dpad != embedder.hidden:
            q.zero_()                            # padding columns of the row layout must be zero
        if self.world == 1 or B % self.world:
            embedder.embed_dev(flat_tok, tok_off, q.data_ptr(), self.dpad, self.stages.stream())
            return
        per = B // self.world
        lo = self.rank * per
        f = np.ascontiguousarray(flat_tok[tok_off[lo]:tok_off[lo + per]])
        o = np.ascontiguousarray(tok_off[lo:lo + per + 1] - tok_off[lo])
        loc = self._tensor("q_local", (per, self.dpad), torch.float32)
        if self.dpad != embedder.hidden:
            loc.zero_()
        embedder.embed_dev(f, o, loc.data_ptr(), self.dpad, self.stages.stream())
        dist.all_gather_into_tensor(q, loc, group=self.group)

    def retrieve(self, q_host: np.ndarray | None, q_terms_list, k: int, embedder=None, tokens=None, allow_bitmap: np.ndarray | None = None, **kw):
        """End to end with HOST buffers: pinned H2D of the queries, the pipeline, D2H of the result.
        With `embedder` (kaito_b200._native.Embedder) and `tokens` = (flat int32 token ids, int32 offsets [B+1])
        the query vectors are produced on the GPU by the BERT forward (K5) instead of being uploaded."""
        if embedder is not None:
            flat_tok, tok_off = tokens
            B = len(tok_off) - 1
            q = self._tensor("q", (B, self.dpad), torch.float32)
            self.embed_into(embedder, flat_tok, tok_off, q)
        else:
            B, d = q_host.shape
            pin_q = self._pinned("pin_q", (B, self.dpad), torch.float32)
            pin_q.zero_()
            pin_q[:, :d] = torch.from_numpy(q_host)
            q = self._tensor("q", (B, self.dpad), torch.float32)
            q.copy_(pin_q, non_blocking=True)
        terms = toff = None
        if q_terms_list is not None:
            offs = np.zeros(B + 1, np.int32)
            for i, t in enumerate(q_terms_list):
                offs[i + 1] = offs[i] + len(t)
            flat = np.concatenate([np.asarray(t, np.uint32) for t in q_terms_list]) if offs[-1] else np.zeros(1, np.uint32)
            pin_t = self._pinned("pin_t", (max(len(flat), 1),), torch.int32)
            pin_t[: len(flat)] = torch.from_numpy(flat.view(np.int32))
            pin_o = self._pinned("pin_o", (B + 1,), torch.int32)
            pin_o.copy_(torch.from_numpy(offs))
            terms = self._tensor("terms", (max(len(flat), 1),), torch.int32)
            toff = self._tensor("toff", (B + 1,), torch.int32)
            terms.copy_(pin_t, non_blocking=True)
            toff.copy_(pin_o, non_blocking=True)
        allow = None
        if allow_bitmap is not None:
            ab = np.ascontiguousarray(allow_bitmap, np.uint32)
            pin_a = self._pinned("pin_allow", (max(len(ab), 1),), torch.int32)
            pin_a[: len(ab)] = torch.from_numpy(ab.view(np.int32))
            allow = self._tensor("allow", (max(len(ab), 1),), torch.int32)
            allow.copy_(pin_a, non_blocking=True)
        out = self.retrieve_dev(q, terms, toff, k, toff_host=offs if q_terms_list is not None else None, allow=allow, **kw)
        host = {name: self._pinned("pin_out_" + name, tuple(t.shape), t.dtype) for name, t in out.items()}
        for name, t in out.items():
            host[name].copy_(t, non_blocking=True)
        if self.device.type == "cuda":
            torch.cuda.current_stream(self.device).synchronize()
        return {name: t.numpy().copy() for name, t in host.items()}

    def _pinned(self, name, shape, dtype):
        n = self._numel(shape)
        return self._storage(("pin", name), n, dtype, pin_memory=(self.device.type == "cuda"))[:n].view(shape)

    @staticmethod
    def io_bytes(B: int, dim: int, n_terms: int, k: int) -> tuple[int, int]:
        """(host->device, device->host) bytes per retrieve() call."""
        return B * dim * 4 + n_terms * 4 + (B + 1) * 4, B * k * (8 + 4 + 4 + 4 + 8) + B * 4
