"""Job plugins: thin subclasses of the reference's own training jobs whose `_process_subbatch` calls the FUSED
entry points of libb200kge (score + loss in one launch sequence, scores never reach HBM).

Selected through the reference's job factory (kge/job/train.py:127-137: `init_from(config.get("<type>.class_name"),
config.modules(), ...)`), i.e. in a LibKGE config:

    modules: [kge.job, kge.model, kge.model.embedder, kge_b200.plugin]
    model: b200_complex
    1vsAll.class_name: B200TrainingJob1vsAll
    KvsAll.class_name: B200TrainingJobKvsAll
    negative_sampling.class_name: B200TrainingJobNegativeSampling

Everything else of the job (data loading, collate, sub-batching, trace entries, penalties, optimizer, hooks,
checkpoints) is the reference's code, unchanged.  Whenever a fused form is not available for the configured
combination (a non-b200 model, a loss outside the fused set, ...) the method falls through to the reference
implementation, which then still reaches the kernels through `model.score_*`.  Embedding dropout in training takes the
dropout entry points in the 1vsAll and KvsAll jobs (masks drawn on the device, keyed per sub-batch).  The
negative-sampling job with dropout keeps the reference step unless `user.b200_ns_dropout: true` opts into the dropout
kernels: the option chooses which random stream supplies the masks (the library's Philox key instead of torch's
generator), as `user.b200_device_sampling` does for the negatives.

LibKGE's `reciprocal_relations_model` over a b200 base model takes the base model's fused and dropout forms too: the
1vsAll reciprocal step, KvsAll's _po query type as the sp_ query (o, p + R), and the negative-sampling S slot as
O-slot triples (o, p + R, s).  The P slot, `s_o` and negative-sampling dropout keep the reference's step.

Evaluation: `entity_ranking.class_name: B200EntityRankingJob` selects the entity-ranking job below (eval.py:36-48); the
training jobs' validation (`valid.every`) is created by the same factory and picks it up too.
"""
from __future__ import annotations

import math
import sys
import time

import torch

from kge.job.eval_entity_ranking import EntityRankingJob
from kge.job.train_1vsAll import TrainingJob1vsAll
from kge.job.train_KvsAll import TrainingJobKvsAll
from kge.job.train import TrainingJob
from kge.job.train_negative_sampling import TrainingJobNegativeSampling
from kge.job import Job
from kge.model.reciprocal_relations_model import ReciprocalRelationsModel
from kge.util.loss import (BCEWithLogitsKgeLoss, KLDivWithSoftmaxKgeLoss, MarginRankingKgeLoss, SEKgeLoss,
                           SoftMarginKgeLoss)
from kge.util.sampler import KgeSampler

from .. import engine
from ..optim import install_native_step

S, P, O = 0, 1, 2
SLOT_STR = ["s", "p", "o"]


def _fused_loss_kind(loss):
    """("bce"|"kl", offset) if the job's KgeLoss has a fused form, else None (loss.py:139-213)."""
    if type(loss) is BCEWithLogitsKgeLoss and loss._bce_type is None:
        return "bce", float(loss._offset)
    if type(loss) is KLDivWithSoftmaxKgeLoss:
        return "kl", 0.0
    return None


def _ns_loss_kind(loss):
    """(name, arg, temperature) of the job's KgeLoss if the negative-sampling kernels cover it, else None: every loss
    KgeLoss.create builds for a negative-sampling job (loss.py:30-90; "ce" is not one of its names)."""
    t = type(loss)
    if t is BCEWithLogitsKgeLoss:
        name = {None: "bce", "mean": "bce_mean", "self_adversarial": "bce_self_adversarial"}.get(loss._bce_type)
        if name is None:
            return None
        return name, float(loss._offset), float(getattr(loss, "_temperature", 1.0))
    if t is KLDivWithSoftmaxKgeLoss:
        return "kl", 0.0, 1.0
    if t is MarginRankingKgeLoss and loss._loss.reduction == "sum":
        return "margin_ranking", float(loss._loss.margin), 1.0
    if t is SoftMarginKgeLoss and loss._loss.reduction == "sum":
        return "soft_margin", 0.0, 1.0
    if t is SEKgeLoss and loss._loss.reduction == "sum":
        return "se", 0.0, 1.0
    return None


def _fused_model(model):
    """The b200 model if its fused entry points can read the tables in place, else None."""
    if getattr(model, "_b200_name", None) is None or not hasattr(model, "b200_fusable"):
        return None
    return model if model.b200_fusable() else None


def _dropout_model(model):
    """(b200 model, (p_ent, p_rel)) if embedding dropout is active and the dropout entry points can serve the model's
    tables, else (None, None)."""
    if getattr(model, "_b200_name", None) is None or not hasattr(model, "b200_dropout_rates"):
        return None, None
    rates = model.b200_dropout_rates()
    return (model, rates) if rates is not None else (None, None)


def _reciprocal_base(model):
    """(base model, R) for a LibKGE ReciprocalRelationsModel whose base model is a b200 model, else (None, None).  Its
    score_po is the base model's sp_ query (o, p + R) against the same table (reciprocal_relations_model.py:85-92), so
    the fused and dropout forms of the base model serve both directions; R = dataset.num_relations()."""
    if type(model) is not ReciprocalRelationsModel:
        return None, None
    base = getattr(model, "_base_model", None)
    if getattr(base, "_b200_name", None) is None or not hasattr(base, "b200_fusable"):
        return None, None
    return base, int(model.dataset.num_relations())


def dropout_call(epoch, batch_index, ordinal):
    """The `call` word of a sub-batch's dropout key: a pure function of (epoch, batch index, sub-batch ordinal within
    the batch), so a resumed run draws the same masks."""
    return ((int(epoch) << 40) | (int(batch_index) << 16) | int(ordinal)) & (2 ** 64 - 1)


class _DropoutKeys:
    """One engine.DropoutKey per sub-batch: seed = torch.initial_seed() (as the device sampler), call from
    (epoch, batch index, sub-batch ordinal), row_base = the sub-batch's first row in the batch."""

    def _b200_dropout_key(self, rates, batch_index, subbatch_slice):
        pos = (self.epoch, batch_index)
        ordinal = self._b200_drop_ordinal + 1 if getattr(self, "_b200_drop_pos", None) == pos else 0
        self._b200_drop_pos, self._b200_drop_ordinal = pos, ordinal
        return engine.DropoutKey(rates[0], rates[1], torch.initial_seed(), dropout_call(self.epoch, batch_index, ordinal),
                                 subbatch_slice.start or 0)


def _user_option(config, key, default=None):
    try:
        return config.get("user." + key)
    except KeyError:
        return default


class _NativeOptimizer:
    """`user.b200_native_optimizer: true`: the training job's optimizer (Adagrad or SparseAdam) steps on the library's
    kernels (kge_b200.optim).  Only `step` of the instance is replaced; its state and state_dict() stay torch's, so
    checkpoints resume with the option on or off.  A configuration the native step cannot serve raises when the job
    is created."""

    def _b200_native_optimizer(self):
        if self.is_forward_only or not _user_option(self.config, "b200_native_optimizer", False):
            return
        try:
            install_native_step(self.optimizer)
        except NotImplementedError as e:
            raise NotImplementedError(f"user.b200_native_optimizer: {e}") from None


class _BatchSplit:
    """Replicas + batch split over the processes of a torch.distributed group (SURVEY 8e, "small tables": every GPU
    holds the whole tables, scores its share of the batch's rows against them, and the dense table gradients are
    all-reduced before the optimizer step; no collective on the forward data path).

    Enabled by `user.b200_batch_split: true` when a process group with more than one rank is initialised (one process
    per GPU, `job.device: cuda:<LOCAL_RANK>`, one output folder per rank, the same random seed on every rank so that
    all ranks draw the same batches).  Rank r takes rows [r*B/W, (r+1)*B/W) of every batch; the per-row losses are
    divided by the size of the WHOLE batch (as for sub-batches, train_1vsAll.py:65), so the all-reduced gradients and
    avg_loss are those of the single-process job.  Penalties and the optimizer step run identically on every rank
    (kge/job/train.py:411-470), which keeps the replicas in step without a broadcast."""

    def _b200_ranks(self):
        r = getattr(self, "_b200_rank_world", None)
        if r is None:
            r = (0, 1)
            if _user_option(self.config, "b200_batch_split", False):
                import torch.distributed as dist

                if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
                    r = (dist.get_rank(), dist.get_world_size())
            self._b200_rank_world = r
        return r

    def _b200_my_rows(self, subbatch_slice, batch_size):
        """This rank's part of a sub-batch slice, or None if it has none."""
        rank, world = self._b200_ranks()
        if world == 1:
            return subbatch_slice
        lo, hi = rank * batch_size // world, (rank + 1) * batch_size // world
        start = max(subbatch_slice.start or 0, lo)
        stop = min(batch_size if subbatch_slice.stop is None else subbatch_slice.stop, hi)
        return slice(start, stop) if stop > start else None

    def _process_batch(self, batch_index, batch):
        result = super()._process_batch(batch_index, batch)
        rank, world = self._b200_ranks()
        if world == 1:
            return result
        import torch.distributed as dist

        if not self.is_forward_only:
            for p in self.model.parameters():
                if not p.requires_grad:
                    continue
                if p.grad is None:                      # a rank without rows (batch smaller than the group)
                    p.grad = torch.zeros_like(p)
                if p.grad.is_sparse:
                    raise NotImplementedError("user.b200_batch_split all-reduces dense gradients (sparse: False)")
                dist.all_reduce(p.grad)
        total = torch.tensor([result.avg_loss], dtype=torch.float64, device=self.device)
        dist.all_reduce(total)
        result.avg_loss = float(total.item())
        return result


class B200TrainingJob1vsAll(_DropoutKeys, _NativeOptimizer, _BatchSplit, TrainingJob1vsAll):
    """`TrainingJob1vsAll` (train_1vsAll.py:10-82) with the sub-batch step as ONE fused call:
    (loss(score_sp, o) + loss(score_po, s)) / batch_size, both directions stacked into one problem."""

    def __init__(self, config, dataset, parent_job=None, model=None, forward_only=False):
        super().__init__(config, dataset, parent_job, model=model, forward_only=forward_only)
        self._b200_native_optimizer()
        if self.__class__ == B200TrainingJob1vsAll:
            for f in Job.job_created_hooks:
                f(self)

    def _process_subbatch(self, batch_index, batch, subbatch_slice, result):
        subbatch_slice = self._b200_my_rows(subbatch_slice, result.size)
        if subbatch_slice is None:
            return
        base, recip = _reciprocal_base(self.model)
        target = self.model if base is None else base
        model, kind = _fused_model(target), _fused_loss_kind(self.loss)
        rates = None
        if model is None:
            model, rates = _dropout_model(target)
            if model is not None and not self.is_forward_only and not model.b200_1vsall_native_backward_ok():
                model = None
        elif recip is not None and not self.is_forward_only and not model.b200_1vsall_native_backward_ok():
            model = None                # the reciprocal step has no recompute backward
        if model is None or kind is None:
            return super()._process_subbatch(batch_index, batch, subbatch_slice, result)
        batch_size = result.size
        drop = None if rates is None else self._b200_dropout_key(rates, batch_index, subbatch_slice)

        host = batch["triples"][subbatch_slice]
        if (drop is None and recip is None and self.is_forward_only and not host.is_cuda and host.dtype == torch.int64
                and host.is_contiguous() and len(host) > 0):
            # forward only: batch copy, kernels and the scalar read-back in ONE library call (no torch ops in between)
            result.forward_time -= time.time()
            value = model.loss_1vsall_host(host, kind[0], kind[1])
            if len(host) != batch_size:
                value *= len(host) / batch_size
            result.avg_loss += value
            result.forward_time += time.time()
            return

        result.prepare_time -= time.time()
        triples = host.to(self.device, non_blocking=True)
        result.prepare_time += time.time()

        result.forward_time -= time.time()
        # sum over both directions and all rows of the sub-batch, divided by the sub-batch size by the kernel's
        # finaliser; the reference divides by the size of the whole batch (train_1vsAll.py:65,76)
        kw = {} if drop is None else {"dropout": drop}
        if recip is not None:
            kw["reciprocal"] = recip
        loss_value = model.loss_1vsall(triples, kind[0], kind[1], need_grad=not self.is_forward_only, **kw)
        if len(triples) != batch_size:
            loss_value = loss_value * (len(triples) / batch_size)
        result.avg_loss += loss_value.item()
        result.forward_time += time.time()

        result.backward_time -= time.time()
        if not self.is_forward_only:
            loss_value.backward()
        result.backward_time += time.time()


class B200TrainingJobKvsAll(_DropoutKeys, _NativeOptimizer, _BatchSplit, TrainingJobKvsAll):
    """`TrainingJobKvsAll` (train_KvsAll.py:205-294): per query type one fused score+loss call that consumes the
    batch's label coordinates as CSR (no dense [n, E] label matrix: job/util.py:32-60 + `.to_dense()`,
    train_KvsAll.py:242-266 are not executed).  The s_o query type (relation prediction) is served for the dot family
    (model.b200_kvsall_so_ok) against the relation table; otherwise a job with s_o keeps the reference step."""

    def __init__(self, config, dataset, parent_job=None, model=None, forward_only=False):
        super().__init__(config, dataset, parent_job, model=model, forward_only=forward_only)
        self._b200_native_optimizer()
        if self.__class__ == B200TrainingJobKvsAll:
            for f in Job.job_created_hooks:
                f(self)

    def _process_subbatch(self, batch_index, batch, subbatch_slice, result):
        subbatch_slice = self._b200_my_rows(subbatch_slice, result.size)
        if subbatch_slice is None:
            return
        base, recip = _reciprocal_base(self.model)
        target = self.model if base is None else base
        model, kind = _fused_model(target), _fused_loss_kind(self.loss)
        rates = None
        if model is None:
            model, rates = _dropout_model(target)
        # s_o: the dot family's relation-candidate kernels; a reciprocal-relations model has no score_so
        # (reciprocal_relations_model.py), so its reference step raises before anything is computed
        so_ok = "s_o" not in self.query_types or (recip is None and model is not None and model.b200_kvsall_so_ok())
        if (model is None or kind is None or not so_ok or not model.b200_csr_labels_ok(self.label_smoothing)
                or (not self.is_forward_only and not model.b200_kvsall_native_backward_ok(rates is not None))):
            return super()._process_subbatch(batch_index, batch, subbatch_slice, result)
        batch_size = result.size
        # one key per sub-batch: the sp_, _po and s_o query types draw disjoint mask streams under it
        kw = {} if rates is None else {"dropout": self._b200_dropout_key(rates, batch_index, subbatch_slice)}

        result.prepare_time -= time.time()
        queries = batch["queries"][subbatch_slice].to(self.device)
        qt = batch["query_type_indexes"][subbatch_slice].to(self.device)
        coords = batch["label_coords"]                       # [nnz, 2] int, rows ascending (collate order)
        start, stop = subbatch_slice.start or 0, subbatch_slice.stop
        rows = coords[:, 0].long()
        if start != 0 or stop < batch_size:
            keep = (rows >= start) & (rows < stop)
            rows, cols = rows[keep] - start, coords[keep, 1].long()
        else:
            cols = coords[:, 1].long()
        n_sub = len(queries)
        result.prepare_time += time.time()

        for query_type_index, query_type in enumerate(self.query_types):
            result.prepare_time -= time.time()
            examples = (qt == query_type_index).nonzero(as_tuple=False).view(-1)
            if len(examples) == 0:
                result.prepare_time += time.time()
                continue
            # CSR of the selected rows: counts per selected row, columns in row order
            sel = torch.zeros(n_sub, dtype=torch.bool, device=self.device)
            sel[examples] = True
            keep = sel[rows]
            counts = torch.bincount(rows[keep], minlength=n_sub)[examples]
            offsets = torch.zeros(len(examples) + 1, dtype=torch.int64, device=self.device)
            torch.cumsum(counts, 0, out=offsets[1:])
            ccols = cols[keep]
            result.prepare_time += time.time()

            result.forward_time -= time.time()
            # sp_ queries are (s, p) pairs, _po queries are (p, o) pairs, s_o queries (s, o) pairs (indexing.py:197-235)
            qkw, smoothing = kw, self.label_smoothing
            if query_type == "s_o":
                # relation targets are never smoothed (train_KvsAll.py:263)
                combine, ent_idx, rel_idx, smoothing = "s_o", queries[examples, 0], queries[examples, 1], 0.0
            elif query_type == "sp_":
                combine, ent_idx, rel_idx = "sp_", queries[examples, 0], queries[examples, 1]
            elif recip is not None:
                # reciprocal relations: the sp_ query (o, p + R), masks on the _po streams
                combine, ent_idx, rel_idx = "sp_", queries[examples, 1], queries[examples, 0] + recip
                if rates is not None:
                    qkw = dict(kw, dropout_streams="_po")
            else:
                combine, ent_idx, rel_idx = "_po", queries[examples, 1], queries[examples, 0]
            if self.is_forward_only:
                loss_value = model.loss_kvsall(combine, ent_idx, rel_idx, offsets, ccols, kind[0], kind[1],
                                               smoothing, **qkw) / batch_size
            else:
                loss_value = model.loss_kvsall_train(combine, ent_idx, rel_idx, offsets, ccols, kind[0], kind[1],
                                                     smoothing, batch_size, **qkw)
            result.avg_loss += loss_value.item()
            result.forward_time += time.time()
            result.backward_time -= time.time()
            if not self.is_forward_only:
                loss_value.backward()
            result.backward_time += time.time()


class B200FrequencySampler(KgeSampler):
    """`negative_sampling.sampling_type: frequency` on the device route of B200TrainingJobNegativeSampling: the options
    and filtering indexes of KgeSampler.__init__, plus the weights KgeFrequencySampler.__init__ defines
    (sampler.py:762-780), kept as `counts[slot]` = bincount(train[:, slot]) and `smoothing` (w = counts + smoothing).
    KgeFrequencySampler itself cannot be built on current torch (torch._multinomial_alias_setup is gone); the job draws
    on the device (engine.sample_frequency and sample_frequency_filtered), so the host `_sample` refuses."""

    def __init__(self, config, configuration_key, dataset):
        super().__init__(config, configuration_key, dataset)
        self.smoothing = float(self.get_option("frequency.smoothing"))
        train = dataset.split(config.get("train.split"))
        self.counts = []
        for slot in (S, P, O):
            vocab = int(self.vocabulary_size[slot])
            c = torch.bincount(train[:, slot].long(), minlength=vocab)
            if c.numel() != vocab:
                raise ValueError(f"{config.get('train.split')} holds {SLOT_STR[slot]} ids outside [0, {vocab})")
            self.counts.append(c)

    def _sample(self, positive_triples, slot, num_samples):
        raise NotImplementedError("frequency negative sampling is drawn on the device only: use "
                                  "B200TrainingJobNegativeSampling with user.b200_device_sampling: true")


class B200TrainingJobNegativeSampling(_DropoutKeys, _NativeOptimizer, _BatchSplit, TrainingJobNegativeSampling):
    """`TrainingJobNegativeSampling` (train_negative_sampling.py:103-164): per slot ONE kernel gathers the sampled
    rows and scores them, with the positive triple in column 0 — neither `[n*K, D]` gathers (`triple`
    implementation, sampler.py:294-305) nor scoring against all unique targets (`batch`, :306-339).

    With `user.b200_device_sampling: true` (LibKGE's free-form `user.*` option space) and a uniform, not shared
    sampler the negatives are also DRAWN on the device (Philox, keyed by the torch seed, counter = batch / slot): the
    DataLoader workers only slice the triples, and no [n, K] id tensors travel host -> device
    (KgeUniformSampler._sample, sampler.py:588-596, is a CPU torch.randint).  `negative_sampling.filtering.<slot>` is
    served there too: the sampling kernel replaces positives of the filtering split with uniform non-positives
    (engine.sample_uniform_filtered), from an index uploaded once when the job is created.

    `negative_sampling.sampling_type: frequency` (not shared) is served on this route only: the job builds
    B200FrequencySampler instead of the reference's KgeFrequencySampler, uploads one weight table per sampled slot and
    draws with engine.sample_frequency, or engine.sample_frequency_filtered for a filtered slot.

    With `user.b200_ns_p_slot: true` a sampled P slot (relation negatives) trains natively too, through
    model.loss_negatives_p (b200kge_ns_p_backward), when the model passes b200_ns_p_slot_ok(); without the option a P slot
    sends the whole sub-batch to the reference step, as before.

    With `user.b200_ns_shared: true` and the reference's uniform sampler with `shared: True` (naive or default, with
    or without replacement), the S and O slots train through model.loss_negatives_shared (b200kge_ns_shared_score /
    _backward) when the model passes b200_ns_shared_ok(): each row's pair is scored against the U' shared rows once, and
    the backward sums the block's gradient per shared id.  The host sampler, and so every draw, is the reference's.
    A sampled P slot, embedding dropout and frequency sampling keep the route they take without the option."""

    def __init__(self, config, dataset, parent_job=None, model=None, forward_only=False):
        want = bool(_user_option(config, "b200_device_sampling", False))
        if (want and config.get("negative_sampling.sampling_type") == "frequency"
                and not config.get("negative_sampling.shared")):
            # TrainingJobNegativeSampling.__init__ (train_negative_sampling.py:16-27) with the plugin's sampler in place
            # of KgeSampler.create, which would build KgeFrequencySampler
            TrainingJob.__init__(self, config, dataset, parent_job, model=model, forward_only=forward_only)
            self._sampler = B200FrequencySampler(config, "negative_sampling", dataset)
            self.type_str = "negative_sampling"
        else:
            super().__init__(config, dataset, parent_job, model=model, forward_only=forward_only)
        sm = self._sampler
        frequency = isinstance(sm, B200FrequencySampler)
        self._device_sampling = bool(
            want and (frequency or type(sm).__name__ == "KgeUniformSampler") and not sm.shared)
        self._frequency = self._b200_frequency_tables() if frequency else {}
        self._filter_index = self._b200_filter_indexes() if self._device_sampling else {}
        self._sample_calls = 0
        self._b200_native_optimizer()
        if self.__class__ == B200TrainingJobNegativeSampling:
            for f in Job.job_created_hooks:
                f(self)

    def _get_collate_fun(self):
        if not self._device_sampling:
            return super()._get_collate_fun()

        def collate(batch):          # the triples only: negatives are drawn on the device
            return {"triples": self.dataset.split(self.train_split)[batch, :].long(), "negative_samples": []}
        return collate

    def _b200_filter_indexes(self):
        """{slot: engine.FilterIndex} for every sampled slot with `negative_sampling.filtering.<slot>`: the positives of
        the sampler's filtering split (the index the sampler created, sampler.py:44-48), uploaded once.  A key whose
        positives cover the vocabulary is refused here: the reference's redraw loop would never end on it."""
        sm = self._sampler
        filtered = [slot for slot in (S, P, O) if sm.filter_positives[slot] and sm.num_samples[slot] > 0]
        if self._frequency and filtered and sm.filter_implementation == "fast":
            # what KgeSampler._filter_and_resample_fast raises for every sampler but the uniform one (sampler.py:197-210)
            raise NotImplementedError("Use filtering.implementation=standard for this sampler.")
        out = {}
        for slot in filtered:
            name = f"{sm.filtering_split}_{['po', 'so', 'sp'][slot]}_to_{SLOT_STR[slot]}"
            vocab = int(sm.vocabulary_size[slot])
            index = engine.FilterIndex(self.dataset.index(name), vocab, self.device)
            if index.max_count >= vocab:
                raise NotImplementedError(
                    f"negative_sampling.filtering.{SLOT_STR[slot]}: a key of {name} has all {vocab} ids as positives, "
                    "so no negative exists for it")
            table = self._frequency.get(slot)
            if table is not None and table.attach(index).full_keys:
                raise NotImplementedError(
                    f"negative_sampling.filtering.{SLOT_STR[slot]}: the positives of key {index.first_full_key} of "
                    f"{name} carry all the frequency weight (smoothing {table.smoothing}), so no negative exists for it")
            out[slot] = index
        return out

    def _b200_frequency_tables(self):
        """{slot: engine.FrequencyTable} for every sampled slot: the sampler's counts and smoothing, uploaded once."""
        sm = self._sampler
        return {slot: engine.FrequencyTable(sm.counts[slot], sm.smoothing, self.device)
                for slot in (S, P, O) if sm.num_samples[slot] > 0}

    def _device_negatives(self, n, slot, batch_index, triples):
        sm = self._sampler
        # one independent stream per (epoch, batch, slot); the key follows torch.manual_seed
        offset = ((self.epoch * (1 << 24) + batch_index) << 2) | slot
        self._sample_calls += 1
        K, vocab = int(sm.num_samples[slot]), int(sm.vocabulary_size[slot])
        index, table = self._filter_index.get(slot), self._frequency.get(slot)
        if table is not None:
            if index is None:
                return engine.sample_frequency(n, K, table, torch.initial_seed(), offset)
            return engine.sample_frequency_filtered(n, K, table, torch.initial_seed(), offset, triples, slot, index)
        if index is None:
            return engine.sample_uniform(n, K, vocab, torch.initial_seed(), offset, self.device)
        # the dataset's own triples: with reciprocal relations the S slot is filtered on (p, o), as the reference's
        # sampler sees them; the (o, p + R, s') rewrite happens only when scoring
        return engine.sample_uniform_filtered(n, K, vocab, torch.initial_seed(), offset, triples, slot, index)

    def _b200_ns_dropout_route(self, kind, slots):
        """(b200 model, (p_ent, p_rel)) if `user.b200_ns_dropout` is on, embedding dropout is active and the dropout
        kernels serve the configuration, else (None, None).  With device sampling an unserved configuration raises
        (the reference step cannot consume device-drawn negatives)."""
        model, rates = _dropout_model(self.model)
        if model is None or not _user_option(self.config, "b200_ns_dropout", False):
            return None, None
        reason = None
        if kind is None:
            reason = f"the loss {type(self.loss).__name__} has no negative-sampling kernel"
        elif any(sl == P for sl in slots):
            reason = "the P slot is not served"
        elif not all(model.b200_ns_dropout_ok(sl) for sl in slots):
            reason = f"model {model._b200_name} with l_norm {model._b200_args()[0]} and this embedding width is not served"
        if reason is None:
            return model, rates
        if self._device_sampling:
            raise NotImplementedError(f"user.b200_ns_dropout with user.b200_device_sampling: {reason}")
        return None, None

    def _process_subbatch(self, batch_index, batch, subbatch_slice, result):
        subbatch_slice = self._b200_my_rows(subbatch_slice, result.size)
        if subbatch_slice is None:
            return
        kind = _ns_loss_kind(self.loss)
        slots = [sl for sl in (S, P, O) if self._sampler.num_samples[sl] > 0]
        base, recip = _reciprocal_base(self.model)
        if base is None:
            model = _fused_model(self.model)
        else:
            # reciprocal relations: the S slot scores (o, p + R, s') through the O-slot kernels
            # (reciprocal_relations_model.py:74-78); the P slot falls through (the reference raises there), and so
            # does embedding dropout (the NS dropout kernels do not serve the wrapper)
            model = _fused_model(base) if P not in slots else None
            if model is None and self._device_sampling:
                why = ("the P slot is not served" if P in slots else
                       "embedding dropout is not served" if base.b200_dropout_rates() is not None else
                       "the base model's tables cannot be read in place")
                raise NotImplementedError(f"user.b200_device_sampling with reciprocal_relations_model: {why}")
        # user.b200_ns_p_slot: the P slot trains through b200kge_ns_p_backward where the model serves it
        p_native = (model is not None and P in slots and _user_option(self.config, "b200_ns_p_slot", False)
                    and model.b200_ns_p_slot_ok())
        trainable = (model is not None and kind is not None
                     and all((p_native if sl == P else model.b200_ns_native_backward_ok(O if recip is not None else sl))
                             for sl in slots))
        drop = None
        if model is None and base is None:
            model, rates = self._b200_ns_dropout_route(kind, slots)
            if model is not None:
                # one key per sub-batch; the S and O slots draw disjoint mask streams under it
                drop = self._b200_dropout_key(rates, batch_index, subbatch_slice)
                trainable = True
        # "all" draws the masks of "batch" (embed_all() gives the same distribution); `auto` is resolved by _prepare
        impl = "triple" if getattr(self, "_implementation", "batch") == "triple" else "batch"
        dkw = {} if drop is None else {"dropout": drop, "implementation": impl}
        # user.b200_ns_shared: the S / O slots of a shared uniform sample train through b200kge_ns_shared_*
        shared = (model is not None and drop is None and P not in slots and trainable and not self.is_forward_only
                  and self._sampler.shared and type(self._sampler).__name__ == "KgeUniformSampler"
                  and _user_option(self.config, "b200_ns_shared", False) and model.b200_ns_shared_ok())
        if model is not None and any(model.b200_sparse_grads()):
            # the row set of a sparse gradient: `all` scores against embed_all(), so every entity row is in it
            dkw["implementation"] = getattr(self, "_implementation", "batch")
        if model is None or (not self.is_forward_only and not trainable):
            if self._device_sampling:
                raise NotImplementedError("user.b200_device_sampling needs a b200_* model whose slots the fused "
                                          "gradient kernel covers (S / O slots; the P slot with user.b200_ns_p_slot)")
            return super()._process_subbatch(batch_index, batch, subbatch_slice, result)
        batch_size = result.size
        result.prepare_time -= time.time()
        triples = batch["triples"]
        if self._filter_index:
            # one device copy of the batch's triples serves the filtered sampling of every slot and the scoring
            if "b200_triples" not in batch:
                batch["b200_triples"] = triples.to(self.device)
            triples = batch["b200_triples"]
        triples = triples[subbatch_slice]
        negs = batch["negative_samples"]
        subbatch_size = len(triples)
        labels = batch["labels"]
        result.prepare_time += time.time()

        for slot in [S, P, O]:
            num_samples = self._sampler.num_samples[slot]
            if num_samples <= 0:
                continue
            result.prepare_time -= time.time()
            if self._device_sampling:
                if negs == [] or len(negs) < 3:
                    negs = batch["negative_samples"] = [None, None, None]
                if negs[slot] is None:          # drawn once per batch and slot, sliced per sub-batch
                    negs[slot] = self._device_negatives(batch_size, slot, batch_index, batch.get("b200_triples"))
                negatives = negs[slot][subbatch_slice]
            elif shared:
                negatives = None
            else:
                # the whole batch's samples, sliced: NaiveSharedNegativeSample.samples takes no slice (sampler.py:414)
                negatives = negs[slot].samples()
                if subbatch_size != batch_size:
                    negatives = negatives[subbatch_slice]
            tri, kslot = triples, slot
            if recip is not None and slot == S:
                tri, kslot = torch.stack((triples[:, 2], triples[:, 1] + recip, triples[:, 0]), dim=1), O
            result.prepare_time += time.time()

            result.forward_time -= time.time()
            if not self.is_forward_only:
                # training: forward + the fused NS gradient kernel behind one autograd node
                if shared:
                    sm = negs[slot]
                    drop_index = getattr(sm, "_drop_index", None)        # DefaultSharedNegativeSample only
                    if drop_index is not None:
                        drop_index = drop_index.to(self.device)[subbatch_slice]
                    loss_value = model.loss_negatives_shared(
                        tri, kslot, sm._unique_samples.to(self.device), sm._repeat_indexes.to(self.device),
                        drop_index, num_samples, kind[1], batch_size, kind[0], kind[2],
                        getattr(self, "_implementation", "batch"))
                elif slot == P:
                    loss_value = model.loss_negatives_p(tri, negatives.to(self.device), kind[1], batch_size, kind[0],
                                                        kind[2], getattr(self, "_implementation", "batch"))
                else:
                    loss_value = model.loss_negatives(tri, negatives.to(self.device), kslot, kind[1], batch_size,
                                                      kind[0], kind[2], **dkw)
                result.avg_loss += loss_value.item()
                result.forward_time += time.time()
                result.backward_time -= time.time()
                loss_value.backward()
                result.backward_time += time.time()
                continue
            scores = model.score_negatives(tri, negatives.to(self.device), kslot, **dkw)  # [n, 1+K], positive first
            if kind is not None and kind[0] == "bce":
                # labels are 1 in column 0 and 0 elsewhere (train_negative_sampling.py:128-137): index labels
                lab = torch.zeros(subbatch_size, dtype=torch.int64, device=self.device)
                loss_value = model.loss_dense(scores, lab, "bce", kind[1]) / batch_size
            elif kind is not None:
                # the row-loss kernel, positive in column 0 (train_negative_sampling.py:126-156)
                loss_value = model.loss_negatives_forward(scores, kind[0], kind[1], kind[2]) / batch_size
            else:
                if labels[slot] is None or labels[slot].shape != (subbatch_size, 1 + num_samples):
                    labels[slot] = torch.zeros((subbatch_size, 1 + num_samples), device=self.device)
                    labels[slot][:, 0] = 1
                loss_value = self.loss(scores, labels[slot], num_negatives=num_samples) / batch_size
            result.avg_loss += loss_value.item()
            result.forward_time += time.time()


# ------------------------------------------------------------------------------------------------------------------
# Entity-ranking evaluation

#: precision modes b200kge_rank_sp_po_eval serves (the in-kernel split modes keep the reference's _evaluate)
_EVAL_PRECISIONS = ("auto", "fp32", "f16x3")


def _row_keys(offsets, cols, row0, E):
    """row * E + col for every entry of a CSR (rows numbered from row0)."""
    n = offsets.numel() - 1
    rows = torch.repeat_interleave(torch.arange(row0, row0 + n), offsets[1:] - offsets[:-1])
    return rows * E + cols


def eval_filter_csr(batch, E, sp_index, po_index, exclude=None):
    """(offsets [2n+1], cols, keys) over the stacked rows of an evaluation batch [n, 3]: row i lists the known objects of
    (s_i, p_i, ?), row n+i the known subjects of (?, p_i, o_i), as entity ids, sorted and unique per row — the
    coordinates get_sp_po_coords_from_spo_batch (kge/job/util.py:6-29) yields, with the _po block moved from columns
    [E, 2E) to rows [n, 2n).  keys = row * E + col (sorted); entries whose key is in `exclude` (sorted) are dropped."""
    n = batch.shape[0]
    o_sp, c_sp = sp_index.get_all_csr(batch[:, [S, P]])
    o_po, c_po = po_index.get_all_csr(batch[:, [P, O]])
    keys = torch.unique(torch.cat((_row_keys(o_sp, c_sp, 0, E), _row_keys(o_po, c_po, n, E))))
    if exclude is not None and exclude.numel() and keys.numel():
        keys = keys[~torch.isin(keys, exclude)]
    offsets = torch.zeros(2 * n + 1, dtype=torch.int64)
    torch.cumsum(torch.bincount(keys // E, minlength=2 * n), 0, out=offsets[1:])
    return offsets, keys % E, keys


class B200EntityRankingJob(EntityRankingJob):
    """`EntityRankingJob` (eval_entity_ranking.py:12-487) whose batch is ranked by ONE library call
    (b200kge_rank_sp_po_eval) against the whole entity table: the raw, filtered and filtered-with-test counts come from a
    single scoring pass, with the filters as CSR built on the host by the DataLoader workers (kge_b200.indexing).  No
    [n, 2E] score, label or coordinate tensor exists.  The counts are additive over the table and nothing of size [n, E]
    is allocated, so `entity_ranking.chunk_size` is not needed and not read.

    The true scores are taken as the reference takes them (score_sp / score_po on the unique targets, :192-203) and the
    reference's tie-handling consistency check (:240-274) compares them with the scores the kernel computed at the true
    answers.  Final ranks, histograms (every `metrics_per.*` hook), metrics, hooks and trace entries are the reference
    job's own (`_get_ranks`, `hist_hooks`, `_compute_metrics`).

    The fused route needs a b200 model whose tables can be read in place (or a ReciprocalRelationsModel over one) and
    a precision the library's ranking entry serves; everything else, collate included, is the reference's."""

    def __init__(self, config, dataset, parent_job, model):
        super().__init__(config, dataset, parent_job, model)
        self._b200_route = None
        if self.__class__ == B200EntityRankingJob:
            for f in Job.job_created_hooks:
                f(self)

    def _b200_select_route(self):
        """(b200 model, R or None) when the fused route serves this job's model, else None."""
        base, recip = _reciprocal_base(self.model)
        target = self.model if base is None else base
        if getattr(target, "_b200_name", None) is None or not hasattr(target, "b200_fusable"):
            return None
        was = target.training
        try:
            target.train(False)             # evaluation runs in eval mode: embedding dropout is inactive there
            ok = target.b200_fusable()
        finally:
            target.train(was)
        if not ok or target._b200_args()[1] not in _EVAL_PRECISIONS:
            return None
        return target, recip

    def _prepare(self):
        super()._prepare()
        self._b200_route = self._b200_select_route()
        if self._b200_route is None:
            return
        from ..indexing import index_KvsAll

        # the reference appended the evaluation split to filter_splits (:27-29)
        known = torch.cat([self.dataset.split(sp) for sp in self.filter_splits])
        self._b200_index = (index_KvsAll(known, "sp"), index_KvsAll(known, "po"))
        self._b200_test_index = None
        if "test" not in self.filter_splits and self.filter_with_test:
            test = self.dataset.split("test")
            self._b200_test_index = (index_KvsAll(test, "sp"), index_KvsAll(test, "po"))

    def _collate(self, batch):
        if self._b200_route is None:
            return super()._collate(batch)
        batch = torch.cat(batch).reshape((-1, 3))
        E = self.dataset.num_entities()
        tri = batch.long()
        f_off, f_col, f_keys = eval_filter_csr(tri, E, *self._b200_index)
        test = ()
        if self._b200_test_index is not None:
            t_off, t_col, _ = eval_filter_csr(tri, E, *self._b200_test_index, exclude=f_keys)
            test = (t_off, t_col)
        own = torch.cat((tri[:, O], tri[:, S]))
        return batch, (f_off, f_col), test, own

    def _b200_tie_check(self, own_score, true2n):
        """The reference's check that the ranking pass scored the true answers as score_sp / score_po did (:240-274):
        on failure log the mean and max difference, then raise or (tie_handling.warn_only) print and go on."""
        if torch.allclose(own_score, true2n, rtol=self.tie_rtol, atol=self.tie_atol):
            return
        diff = torch.abs(own_score - true2n)
        self.config.log(f"Tie-handling: mean difference between scores was: {diff.mean()}.")
        self.config.log(f"Tie-handling: max difference between scores was: {diff.max()}.")
        msg = ("Error in tie-handling: the ranking pass and score_sp / score_po scored a true answer differently beyond "
               "entity_ranking.tie_handling.rtol / atol. Verify the model's scoring implementations or consider "
               "increasing the tie-handling tolerances.")
        if self.config.get("entity_ranking.tie_handling.warn_only"):
            print(msg, file=sys.stderr)
        else:
            raise ValueError(msg)

    def _b200_true_scores(self, s, p, o):
        """[2n]: o's score of each sp_ row, then s's score of each _po row, from the model's score_sp / score_po on the
        unique targets (:192-203)."""
        uo, io = torch.unique(o, return_inverse=True)
        o_true = torch.gather(self.model.score_sp(s, p, uo), 1, io.view(-1, 1)).view(-1)
        us, is_ = torch.unique(s, return_inverse=True)
        s_true = torch.gather(self.model.score_po(p, o, us), 1, is_.view(-1, 1)).view(-1)
        return torch.cat((o_true, s_true))

    @torch.no_grad()
    def _evaluate(self):
        if self._b200_route is None:
            return super()._evaluate()
        model, recip = self._b200_route
        with_test = "test" not in self.filter_splits and self.filter_with_test
        suffixes = ["", "_filtered"] + (["_filtered_with_test"] if with_test else [])
        hists = [dict() for _ in suffixes]
        nb = len(self.loader)
        common = dict(type="entity_ranking", split=self.eval_split, filter_splits=self.filter_splits)
        self.current_trace["epoch"] = dict(common, scope="epoch", epoch=self.epoch, batches=nb,
                                           size=len(self.triples))
        for f in self.pre_epoch_hooks:
            f(self)

        metrics = {}
        epoch_time = -time.time()
        for batch_number, (batch, filt, test, own) in enumerate(self.loader):
            self.current_trace["batch"] = dict(common, scope="batch", epoch=self.epoch, batch=batch_number,
                                               size=len(batch), batches=nb)
            for f in self.pre_batch_hooks:
                f(self)

            batch = batch.to(self.device)
            s, p, o = batch[:, 0], batch[:, 1], batch[:, 2]
            n = len(batch)
            filt = tuple(t.to(self.device, non_blocking=True) for t in filt)
            test = tuple(t.to(self.device, non_blocking=True) for t in test) if with_test else None
            own = own.to(self.device, non_blocking=True)
            true2n = self._b200_true_scores(s, p, o)
            rank, ties, own_score = model.rank_eval(s, p, o, true2n, filt, test, self.tie_rtol, self.tie_atol,
                                                    reciprocal=recip, own_col=own)
            self._b200_tie_check(own_score, true2n)

            # per ranking: (s ranks, o ranks); stacked rows 0..n-1 rank the objects, n..2n-1 the subjects
            ranks = []
            for k in range(len(suffixes)):
                r = self._get_ranks(rank[k], ties[k])
                ranks.append((r[n:], r[:n]))
            batch_hists = [dict() for _ in suffixes]
            for f in self.hist_hooks:
                for k in (0, 1):
                    f(batch_hists[k], s, p, o, ranks[k][0], ranks[k][1], job=self)
            if with_test:
                for f in self.hist_hooks:
                    f(batch_hists[2], s, p, o, ranks[2][0], ranks[2][1], job=self)

            if self.trace_examples:
                self._b200_trace_examples(s, p, o, ranks, with_test, nb)

            metrics = {}
            for k, suffix in enumerate(suffixes):
                metrics.update(self._compute_metrics(batch_hists[k]["all"], suffix=suffix))
            self.current_trace["batch"].update(metrics)
            for f in self.post_batch_hooks:
                f(self)
            if self.trace_batch:
                self.trace(**self.current_trace["batch"])
            self.current_trace["batch"] = None
            self._b200_print_progress(batch_number, nb, metrics)

            for k in range(len(suffixes)):
                for key, h in batch_hists[k].items():
                    hists[k][key] = hists[k][key] + h if key in hists[k] else h

        self.config.print("\033[2K\r", end="", flush=True)
        for key in hists[0]:
            name = "_" + key if key != "all" else ""
            for k, suffix in enumerate(suffixes):
                metrics.update(self._compute_metrics(hists[k][key], suffix=suffix + name))
        epoch_time += time.time()
        self.current_trace["epoch"].update(dict(epoch_time=epoch_time, event="eval_completed", **metrics))

    def _b200_trace_examples(self, s, p, o, ranks, with_test, nb):
        """One `example_rank` entry per task and triple, as the reference writes them (:364-403)."""
        entry = dict(type="entity_ranking", scope="example", split=self.eval_split, filter_splits=self.filter_splits,
                     size=len(s), batches=nb, epoch=self.epoch)
        for i in range(len(s)):
            entry["batch"] = i
            entry["s"], entry["p"], entry["o"] = s[i].item(), p[i].item(), o[i].item()
            for task, side in (("sp", 1), ("po", 0)):
                if with_test:
                    entry["rank_filtered_with_test"] = ranks[2][side][i].item() + 1
                self.trace(event="example_rank", task=task, rank=ranks[0][side][i].item() + 1,
                           rank_filtered=ranks[1][side][i].item() + 1, **entry)

    def _b200_print_progress(self, batch_number, nb, metrics):
        """The reference's console progress line (:429-453)."""
        k = self.hits_at_k_s[-1]
        width = 1 + int(math.ceil(math.log10(nb)))
        self.config.print(
            f"\r{self.config.log_prefix}  batch:{batch_number: {width}d}/{nb - 1}, "
            f"mrr (filt.): {metrics['mean_reciprocal_rank']:4.3f} ({metrics['mean_reciprocal_rank_filtered']:4.3f}), "
            f"hits@1: {metrics['hits_at_1']:4.3f} ({metrics['hits_at_1_filtered']:4.3f}), "
            f"hits@{k}: {metrics[f'hits_at_{k}']:4.3f} ({metrics[f'hits_at_{k}_filtered']:4.3f})\033[K",
            end="", flush=True)
