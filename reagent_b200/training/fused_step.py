"""Whole-update CUDA graphs: replay sample -> TD step -> weight gradients -> Adam + Polyak.

`FusedDqnStep` is the public fast path for the reference workflow "rb.sample_transition_batch
-> trainer_preprocessor -> Lightning optimizer loop" (reagent/gym/datasets/
replay_buffer_dataset.py:122-133 + reagent/training/reagent_lightning_module.py:108-133):
per update the host only draws the random numbers (Python's `random` stream for the
prioritized buffer, torch.randint for the uniform one -- bit-exact index parity with the
reference), writes them to pinned memory and replays one captured graph that does the
host->device copy, the kernels and the device->host copy of the loss.

`prefetch=True` pipelines the sampler one update ahead, the way the reference's DataLoader
over ReplayBufferDataset prefetches batches: the graph of update k trains on the batch drawn
during update k-1 while the replay-sample kernel for update k+1 runs on a second stream (it
does not depend on the parameters).  The host's random stream is consumed in the same order;
the only observable difference is that a transition added between two `step()` calls can be
sampled one update later.

`FusedDqnStep` drives DQNTrainer, QRDQNTrainer and C51Trainer on sample_discrete_dqn_batch and
ParametricDQNTrainer on sample_parametric_dqn_batch (one-hot actions as features, the identity
tiling of the possible actions); the latter without `per` and on one GPU.  DiscreteCRRTrainer runs
on sample_discrete_dqn_batch under the same two limits; its exploration noise is drawn with
torch.randn inside the graph, and a step returns its q1 loss.

`FusedPolicyStep` is the device-resident online step for SACTrainer and TD3Trainer (continuous
actions), with the same staging, draw, status words, optional prioritized replay and data
parallel (`shard` + `process_group`).
"""
from typing import Optional

import numpy as np
import torch

from ..replay_memory.device_replay import DeviceReplay, PrioritizedUpdate, PriorityShard
from ..replay_memory.prioritized_replay_buffer import PrioritizedReplayBuffer
from .c51_trainer import C51Trainer
from .discrete_crr_trainer import DiscreteCRRTrainer
from .dqn_trainer import DQNTrainer
from .parametric_dqn_trainer import ParametricDQNTrainer
from .qrdqn_trainer import QRDQNTrainer
from .sac_trainer import SACTrainer
from .td3_trainer import TD3Trainer

# Prioritized replay: each trainer's priority source, keyed on the exact type (a subclass could
# change what its per-row workspace values mean) -- the DeviceReplay write-back and a function of
# (trainer, workspace) giving its inputs after the update.  DQN: the TD error; QR-DQN: the row's
# loss over its N^2 quantile pairs; C51: its cross entropy; SAC / TD3: the larger critic TD error.
_PRIORITY_SOURCES = {
    DQNTrainer: (DeviceReplay.write_back_priorities, lambda t, ws: (ws["td_target"], ws["q_sel"])),
    QRDQNTrainer: (DeviceReplay.write_back_row_priorities,
                   lambda t, ws: (ws["loss_partials"], float(t.num_atoms) * float(t.num_atoms))),
    C51Trainer: (DeviceReplay.write_back_row_priorities, lambda t, ws: (ws["loss_partials"], 1.0)),
    SACTrainer: (DeviceReplay.write_back_row_priorities, lambda t, ws: (ws["td_error"], 1.0)),
    TD3Trainer: (DeviceReplay.write_back_row_priorities, lambda t, ws: (ws["td_error"], 1.0)),
}


def _priority_shard(batch_size, shard, process_group) -> PriorityShard:
    """The PriorityShard of a prioritized step's `shard = (rank, world)` on `process_group`;
    world > 1 needs the group, and the group must have `world` ranks with this one `rank`."""
    from .data_parallel import shard_rows

    rank, world = (0, 1) if shard is None else (int(shard[0]), int(shard[1]))
    if process_group is None:
        if world > 1:
            raise ValueError("per with shard needs process_group: every rank's priorities are "
                             "gathered over it")
    else:
        import torch.distributed as dist

        if world != dist.get_world_size(process_group) or rank != dist.get_rank(process_group):
            raise ValueError(f"per with shard={tuple(shard) if shard else None} needs the "
                             f"process group's (rank, world), "
                             f"({dist.get_rank(process_group)}, "
                             f"{dist.get_world_size(process_group)})")
    row0, _ = shard_rows(batch_size, rank, world)
    return PriorityShard(row0, batch_size, process_group)


def _query_keyword(rb) -> str:
    """sample_discrete_dqn_batch's keyword for the device random numbers of `rb`'s draw."""
    return "query_dev" if isinstance(rb, PrioritizedReplayBuffer) else "ranks_dev"


class FusedDqnStep:
    _per_trainers = (DQNTrainer, QRDQNTrainer, C51Trainer)  # exact types `per` covers
    _index_buffers = 2  # of a device draw: the prefetch path alternates two
    _beta_net = "q_network"  # the network whose Adam step count anneals per's beta

    def __init__(self, trainer, replay_buffer, batch_size: int, process_group=None,
                 slots: int = 2, prefetch: bool = False, shard=None, rng: str = "host",
                 online: bool = False, per: Optional[PrioritizedUpdate] = None):
        """`shard = (rank, world)`: data-parallel strong scaling (SURVEY.md 8e).  `batch_size`
        is the GLOBAL minibatch; the replay buffer is replicated and every rank consumes the
        identical random stream, so all ranks select the same global indices, and this
        rank gathers and trains on rows [rank*B/world, (rank+1)*B/world) only.

        `rng="device"` (prioritized buffer): the buffer goes device-resident
        (replay_memory/device_replay.py) -- Python's `random` state is uploaded once and the
        stratified draws, tree descents and retries of sample_index_batch run in a kernel
        inside the captured graph: no host random numbers, no per-step query upload.
        `online=True` (needs rng="device"): `step(transition)` also ADDS one transition before
        drawing, the reference's online loop (reagent/gym/runners/gymrunner.py: one env step
        -> replay_buffer.add -> one update); the transition is the step's only host->device
        traffic, staged in pinned memory and copied + inserted by the same graph replay.
        `per=PrioritizedUpdate(...)` (needs rng="device", prefetch=False): prioritized
        experience replay for DQNTrainer, QRDQNTrainer and C51Trainer.  Each update weights
        its loss by the importance weights of the drawn rows and then writes their priorities
        back into the device tree, in batch order, inside the same graph; the next draw sees
        them.  The priority is computed from the TD error for DQN, and from the row's own
        distributional loss for QR-DQN (mean over the N^2 quantile pairs) and C51 (cross
        entropy).  Online, a transition staged without `priority` enters with the largest
        priority recorded so far.

        `per` with `shard` (and, for world > 1, `process_group` of that world): the tree is
        replicated, every rank draws the same global indices and computes the importance
        weights of all of them, and trains on its rows.  The priorities of all rows are then
        gathered on every rank (DeviceReplay.write_back_priorities with a PriorityShard) and
        applied in global batch order, so every rank's tree stays bit-identical;
        `self.priorities` holds the gathered global vector."""
        if isinstance(trainer, ParametricDQNTrainer):
            if per is not None:
                raise NotImplementedError("per does not cover ParametricDQNTrainer: its loss head "
                                          "has no importance weights")
            if shard is not None or process_group is not None:
                raise NotImplementedError("the ParametricDQNTrainer step is single-GPU; "
                                          "train_batch(process_group=...) runs data-parallel")
        if isinstance(trainer, DiscreteCRRTrainer):
            if per is not None:
                raise NotImplementedError("per does not cover DiscreteCRRTrainer: its critic "
                                          "head has no importance weights")
            if shard is not None or process_group is not None:
                raise NotImplementedError("the DiscreteCRRTrainer step is single-GPU; "
                                          "train_batch(process_group=...) runs data-parallel")
            if trainer.delayed_policy_update != 1:
                raise NotImplementedError(
                    "the DiscreteCRRTrainer step captures one graph, so every update trains the "
                    "actor: delayed_policy_update must be 1 (train_batch takes batch_idx)")
        # ParametricDqnInputMaker's batch (one-hot actions as features, the identity tiling of
        # the possible actions) for ParametricDQNTrainer, DiscreteDqnInputMaker's for the rest
        self._sampler = ("sample_parametric_dqn_batch" if isinstance(trainer, ParametricDQNTrainer)
                         else "sample_discrete_dqn_batch")
        if per is not None:
            if rng != "device":
                raise ValueError("per needs rng='device': the priorities live in the device tree")
            if prefetch:
                raise ValueError("per needs prefetch=False: a prefetched draw would run before "
                                 "the previous update's priority write-back")
            if type(trainer) not in self._per_trainers:
                raise NotImplementedError("per covers DQNTrainer, QRDQNTrainer and C51Trainer; "
                                          "got " + type(trainer).__name__)
        self.per = per
        if rng not in ("host", "device"):
            raise ValueError("rng must be 'host' or 'device'")
        if online and rng != "device":
            raise ValueError("online=True needs rng='device' (device-resident replay)")
        self.rng, self.online = rng, bool(online)
        self.prioritized = isinstance(replay_buffer, PrioritizedReplayBuffer)
        if rng == "device" and not self.prioritized:
            raise NotImplementedError("rng='device' covers the prioritized buffer")
        self._shard = None
        if per is not None and (shard is not None or process_group is not None):
            self._shard = _priority_shard(batch_size, shard, process_group)
        self.trainer = trainer
        self.rb = replay_buffer
        self.B_global = batch_size
        self.row0 = 0
        if shard is not None and shard[1] > 1:
            from .data_parallel import shard_rows

            self.row0, hi = shard_rows(batch_size, shard[0], shard[1])
            batch_size = hi - self.row0
        self.B = batch_size
        self.pg = process_group
        self._query_kw = _query_keyword(replay_buffer)
        self.dev = replay_buffer._dev()
        self.slots = []
        self.k = 0
        self.h2d_bytes = batch_size * 8
        self._side = torch.cuda.Stream(device=self.dev)
        self._side2 = torch.cuda.Stream(device=self.dev)
        self.d2h_bytes = 4
        self.prefetch = bool(prefetch)
        slots = 2 if self.prefetch else int(slots)  # prefetch alternates two batch sets
        replay_buffer._flush()
        self.dr = None
        if rng == "device":
            # every slot's graph adds from its own staging block
            self.dr = getattr(replay_buffer, "_device_resident", None) or DeviceReplay(
                replay_buffer, stage_rows=1, stage_slots=max(2, slots))
            if self.dr.stage_slots < slots:
                self.dr._alloc_stage(self.dr.stage_rows, slots)
            self._idx_buf = [torch.zeros(self.B_global, dtype=torch.int64, device=self.dev)
                             for _ in range(self._index_buffers)]
            self._status_host = torch.zeros(2, dtype=torch.int32).pin_memory()
            self._status_np = self._status_host.numpy()
            self.h2d_bytes = self.dr.h2d_bytes_per_add if self.online else 0
            self.d2h_bytes = 4 * self._loss_width + 8
            if per is not None:
                # the weights of all drawn rows: a shard's rows then get exactly the weights a
                # single-GPU update gives them (p_min is over the whole draw)
                self.weights = torch.empty(self.B_global, dtype=torch.float32, device=self.dev)
                self.priorities = torch.empty(self.B_global, dtype=torch.float64, device=self.dev)
        # warm-up outside capture (lazy allocations, cudaFuncSetAttribute, optimizer state)
        self._one_update(None)
        torch.cuda.synchronize()
        if self.prefetch:
            # two fixed sets of batch tensors: update k trains on set k%2 while the sampler
            # fills set (k+1)%2.  Set 0 gets the first real draw now; set 1 is only allocated
            # (given indices: no random numbers consumed).
            self._pools = [{}, {}]
            self._batches = [None, None]
            with self.rb.output_buffers(self._pools[0]):
                self._batches[0] = self._sample(None)
            with self.rb.output_buffers(self._pools[1]):
                self._batches[1] = self._sample_batch(
                    self.B, indices=self._batches[0].indices.reshape(-1))
            torch.cuda.synchronize()
        for i in range(slots):
            self.slots.append(self._capture(i))
        self._param_versions = self._versions() if hasattr(trainer, "tc_prepack") else None

    # -- parameters changed from outside (load_state_dict, manual edits) ----------------------
    def _versions(self):
        t = self.trainer
        return tuple(p._version for p in t.q_network.parameters()) + tuple(
            p._version for p in t.q_network_target.parameters())

    def invalidate_tc_images(self):
        """The captured update keeps the tensor-core weight images of K2 current by itself (the
        Adam kernel rewrites them).  If the parameters of q_network / q_network_target are
        changed OUTSIDE this object, the images must be rebuilt before the next replay: writes
        through torch (load_state_dict, `p.copy_`, ...) are detected by `step()`; call this
        after anything torch's version counters cannot see (a raw kernel writing the arena)."""
        self._param_versions = None

    def _refresh_tc_images(self):
        if not hasattr(self.trainer, "tc_prepack"):  # only DQNTrainer keeps packed images
            return
        v = self._versions()
        if v != self._param_versions:
            self.trainer._tc_images_state = None
            self.trainer.tc_prepack()  # eager, on the current stream, before the replay
            self._param_versions = v

    # -- one update on the current stream ---------------------------------------
    def _one_update(self, rnd_dev):
        # the wgmma K2 wants packed weight images: they only depend on the parameters, so they
        # are built on a side stream while the replay-sample kernel runs (fork/join is
        # captured into the graph like any other dependency)
        main = torch.cuda.current_stream()
        prepack = getattr(self.trainer, "tc_prepack", None)
        forked = False
        if prepack is not None:
            self._side.wait_stream(main)
            with torch.cuda.stream(self._side):
                forked = prepack()
        batch = self._sample(rnd_dev)
        if forked:
            main.wait_stream(self._side)
        return self._train(batch)

    def _train_batch(self, batch, **weights):
        """The trainer's update on `batch` (`importance_weights=` with per); returns the loss
        tensor a step copies to the host."""
        out = self.trainer.train_batch(batch, process_group=self.pg, **weights)
        # DiscreteCRRTrainer returns (critic losses [2], actor losses [2])
        return out[0][:1] if isinstance(self.trainer, DiscreteCRRTrainer) else out

    def _train(self, batch):
        """The update on a drawn batch; returns the loss tensor."""
        if self.per is not None:
            return self._per_train(batch)
        return self._train_batch(batch)

    def _per_train(self, batch):
        """Importance weights of the drawn rows -> weighted update -> priority write-back."""
        idx = self._idx_buf[0]
        opt = self.trainer.optimizer_of(getattr(self.trainer, self._beta_net).arena)
        opt._ensure_state()
        self.dr.importance_weights(idx, opt.step_t, self.per, self.weights)
        loss = self._train_batch(batch,
                                 importance_weights=self.weights[self.row0:self.row0 + self.B])
        write_back, inputs = _PRIORITY_SOURCES[type(self.trainer)]
        write_back(self.dr, idx, *inputs(self.trainer, self.trainer._ws), self.per,
                   self.priorities, shard=self._shard)
        return loss

    def _prefetch_update(self, i, rnd_dev, overrides=None):
        """Update on batch set i; the sampler fills set 1-i concurrently (second stream)."""
        main = torch.cuda.current_stream()
        self._side.wait_stream(main)
        self._side2.wait_stream(main)
        prepack = getattr(self.trainer, "tc_prepack", None)
        forked = False
        if prepack is not None:
            with torch.cuda.stream(self._side2):
                forked = prepack()
        with torch.cuda.stream(self._side), self.rb.output_buffers(self._pools[1 - i]):
            if self.dr is not None:
                nxt = self._device_sample(1 - i, self.online and rnd_dev is not None, stage_row=i)
            else:
                nxt = self._sample(rnd_dev, overrides)
        if forked:
            main.wait_stream(self._side2)
        loss = self._train_batch(self._batches[i])
        main.wait_stream(self._side)
        self._batches[1 - i] = nxt
        return loss

    def _host_draw(self):
        """This rank's rows of one GLOBAL host draw: (values, override positions, indices)."""
        lo, hi = self.row0, self.row0 + self.B
        if self.prioritized:
            q, pos, idxs = self.rb.host_queries(self.B_global)
            keep = [(p - lo, i) for p, i in zip(pos, idxs) if lo <= p < hi]
            return q[lo:hi], [p for p, _ in keep], [i for _, i in keep]
        n_valid = self.rb._num_valid_indices
        if n_valid == 0:
            raise RuntimeError(f"Cannot sample {self.B_global} since there are no valid indices so far.")
        return torch.randint(n_valid, (self.B_global,))[lo:hi].numpy(), [], []

    def _device_sample(self, slot: int, add: bool, stage_row: int = 0):
        """Device-resident draw: (optionally insert the staged transition,) select the global
        indices with the device MT19937 stream, gather this rank's rows."""
        if add:
            self.dr.launch_add(1, slot=stage_row, priority_from_max=self.per is not None)
        return self._gather(self.dr.draw_indices(self.B_global, out=self._idx_buf[slot]))

    def _sample_batch(self, batch_size, **kw):
        """The trainer's replay batch: sample_parametric_dqn_batch for ParametricDQNTrainer,
        sample_discrete_dqn_batch for the discrete-action trainers."""
        return getattr(self.rb, self._sampler)(batch_size, self.trainer.num_actions, **kw)

    def _gather(self, indices):
        """This rank's rows of the drawn global `indices`, as the trainer's batch."""
        return self._sample_batch(self.B, indices=indices[self.row0:self.row0 + self.B])

    def _sample(self, rnd_dev, overrides=None):
        if self.dr is not None:
            return self._device_sample(0, False)
        kw = {}
        if rnd_dev is None and self.B != self.B_global:
            q, pos, idxs = self._host_draw()
            rnd_dev = torch.from_numpy(np.ascontiguousarray(q)).to(self.dev)
            overrides = (pos, idxs) if pos else None
        if overrides is not None:
            kw["overrides"] = overrides
        if rnd_dev is not None:
            kw[self._query_kw] = rnd_dev
        return self._sample_batch(self.B, **kw)

    _loss_width = 1  # elements of the loss copied to the pinned host tensor of a step

    def _capture_device(self, i=0):
        loss_host = torch.zeros(self._loss_width, dtype=torch.float32).pin_memory()
        g = torch.cuda.CUDAGraph()
        marker = torch.zeros(1, device=self.dev)  # non-None: "inside the captured step"
        with torch.cuda.graph(g):
            if self.prefetch:
                loss = self._prefetch_update(i, marker)
            else:
                loss = self._train(self._device_sample(0, self.online, stage_row=i))
            loss_host.copy_(loss.reshape(self._loss_width), non_blocking=True)
            self._status_host.copy_(self.dr.status, non_blocking=True)
        return {"graph": g, "loss_host": loss_host, "done": torch.cuda.Event(), "used": False}

    def _capture(self, i=0):
        if self.dr is not None:
            return self._capture_device(i)
        dt = torch.float64 if self.prioritized else torch.int64
        host = torch.zeros(self.B, dtype=dt).pin_memory()
        devb = torch.zeros(self.B, dtype=dt, device=self.dev)
        loss_host = torch.zeros(1, dtype=torch.float32).pin_memory()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            devb.copy_(host, non_blocking=True)
            loss = self._prefetch_update(i, devb) if self.prefetch else self._one_update(devb)
            loss_host.copy_(loss.reshape(1), non_blocking=True)
        return {"graph": g, "host": host, "dev": devb, "loss_host": loss_host,
                "done": torch.cuda.Event(), "used": False}

    # -- public --------------------------------------------------------------------
    def step(self, transition=None) -> torch.Tensor:
        """One full update.  Returns the pinned host tensor that will hold the loss once the
        stream reaches the end of this update (call torch.cuda.current_stream().synchronize()
        or keep going: slots are recycled only after their event completed).
        `transition` (online mode): dict of the add() keyword arguments of the new transition."""
        s = self.slots[self.k % len(self.slots)]
        self.k += 1
        if s["used"]:
            s["done"].synchronize()
        self._refresh_tc_images()
        if self.dr is not None:
            return self._replay_device(s, s["graph"], s["loss_host"], transition)
        # bring device mirrors up to date OUTSIDE the captured graph (adds / set_priority)
        self.rb._flush()
        if self.prioritized:
            self.rb.sum_tree.device_heap(self.dev)
            q, pos, idxs = self._host_draw()
            if pos:  # rare retry path: resolved on the host, run this update un-captured
                qd = torch.from_numpy(q).to(self.dev)
                if self.prefetch:
                    loss = self._prefetch_update((self.k - 1) % 2, qd, overrides=(pos, idxs))
                else:
                    loss = self._train(self._sample(qd, (pos, idxs)))
                s["loss_host"].copy_(loss.reshape(1), non_blocking=True)
                s["done"].record()
                s["used"] = True
                return s["loss_host"]
            s["host"].numpy()[:] = q
        else:
            self.rb._ensure_valid_index()
            s["host"].copy_(torch.from_numpy(self._host_draw()[0]))
        s["graph"].replay()
        s["done"].record()
        s["used"] = True
        return s["loss_host"]

    def _replay_device(self, s, graph, loss_host, transition):
        """Device-resident step on slot `s` (already waited for): raise a sticky status of an
        earlier step, stage the new transition (online), replay `graph`."""
        if self._status_np[0] != 0:  # sticky device status of an earlier step
            self.dr.raise_if_failed(self._status_host)
        if self.online:
            if transition is None:
                raise ValueError(f"online {type(self).__name__}.step() needs the new transition")
            # every slot's graph copies from its own pinned staging row; the slot's previous
            # replay (and with it that H2D copy) was waited for above
            self.dr.stage(0, (self.k - 1) % len(self.slots),
                          priority_from_max=self.per is not None, **transition)
        graph.replay()
        s["done"].record()
        s["used"] = True
        return loss_host


class FusedPolicyStep(FusedDqnStep):
    """FusedDqnStep's device-resident step for the continuous-action trainers SACTrainer and
    TD3Trainer: per `step(transition)` ONE graph replay adds the transition (online), draws the
    batch with the device MT19937 stream, gathers it with `sample_policy_network_batch` (the
    actions rescaled from [action_low, action_high]) and runs the whole `train_batch`.  SAC's
    noise is drawn with torch.randn inside the graph (or comes from the trainer's `noise_hook`).

    `per=PrioritizedUpdate(...)`: the critic losses are weighted by the importance weights of
    the drawn rows (beta annealed with q1's Adam step count), and each row's priority
    (max over the critics of |q_c(s, a) - y| + eps) ** alpha is written back into the device
    tree, in batch order, inside the same graph.  The actor and alpha losses stay unweighted.

    TD3 trains its actor on every `delayed_policy_update`-th batch only, a decision taken in
    Python; one graph is captured per phase (and staging slot) and `step()` picks it from its
    own update counter.  The constructor runs one eager warm-up update, which is batch 0.
    `step()` returns the pinned host tensor that will hold [q1 loss, q2 loss] of the update.

    `shard=(rank, world)`, `process_group`: as FusedDqnStep's; each rank also draws the global
    batch's noise and uses its own rows, so that a data-parallel run equals a single-GPU run
    from the same seeds.  The losses are this rank's shard means."""

    _loss_width = 2
    _per_trainers = (SACTrainer, TD3Trainer)  # the exact types it covers, with or without per
    _index_buffers = 1
    _beta_net = "q1_network"

    def __init__(self, trainer, replay_buffer, batch_size: int, action_low, action_high,
                 online: bool = True, per: Optional[PrioritizedUpdate] = None,
                 rng: str = "device", prefetch: bool = False, slots: int = 2, shard=None,
                 process_group=None):
        if type(trainer) not in self._per_trainers:
            raise NotImplementedError("FusedPolicyStep covers SACTrainer and TD3Trainer; got "
                                      + type(trainer).__name__)
        if rng != "device":
            raise ValueError("FusedPolicyStep needs rng='device' (device-resident replay)")
        if prefetch:
            raise ValueError("FusedPolicyStep needs prefetch=False: a prefetched draw would run "
                             "before the previous update's priority write-back")
        if int(slots) < 1:
            raise ValueError("slots must be >= 1")
        if not isinstance(replay_buffer, PrioritizedReplayBuffer):
            raise NotImplementedError("FusedPolicyStep covers the prioritized buffer")
        self.action_low = np.asarray(action_low, dtype=np.float32).reshape(-1).copy()
        self.action_high = np.asarray(action_high, dtype=np.float32).reshape(-1).copy()
        # a batch_idx of each phase: TD3 with a delayed actor has two, SAC one
        self._delay = int(getattr(trainer, "delayed_policy_update", 1))
        self._phase_batch_idx = [0, 1] if (type(trainer) is TD3Trainer and self._delay != 1) else [0]
        self._updates = 0
        n0 = trainer.all_batches_processed
        # its warm-up (which also puts the action bounds on the device) is update 0
        super().__init__(trainer, replay_buffer, batch_size, slots=slots, rng="device",
                         online=online, per=per, shard=shard, process_group=process_group)
        trainer.all_batches_processed = n0 + 1  # a capture runs the Python body, not an update

    def _gather(self, indices):
        return self.rb.sample_policy_network_batch(self.B, self.action_low, self.action_high,
                                                   indices=indices[self.row0:self.row0 + self.B])

    def _one_update(self, rnd_dev):
        """One eager update (draw + train) of the next batch_idx, on the current stream: the
        constructor's warm-up, or an update run outside the captured graphs."""
        self._batch_idx = self._updates
        loss = super()._one_update(rnd_dev)
        self._updates += 1
        return loss

    def _train_batch(self, batch, **weights):
        """Returns the critic losses; importance weights weight the critics only.  A shard
        draws the global batch's noise and takes its own rows, as a single-GPU update would."""
        t = self.trainer
        t.noise_rows = (self.row0, self.B_global) if self.B != self.B_global else None
        try:
            return t.train_batch(batch, self._batch_idx, process_group=self.pg, **weights)[0]
        finally:
            t.noise_rows = None

    def _capture(self, i=0):
        graphs, hosts = [], []
        for b in self._phase_batch_idx:
            self._batch_idx = b
            c = self._capture_device(i)
            graphs.append(c["graph"])
            hosts.append(c["loss_host"])
        return {"graphs": graphs, "loss_hosts": hosts, "done": torch.cuda.Event(), "used": False}

    def step(self, transition=None) -> torch.Tensor:
        """One full update (see FusedDqnStep.step); `transition` (online mode): dict of the add()
        keyword arguments of the new transition."""
        s = self.slots[self.k % len(self.slots)]
        self.k += 1
        if s["used"]:
            s["done"].synchronize()
        phase = 0 if self._updates % self._delay == 0 else len(self._phase_batch_idx) - 1
        out = self._replay_device(s, s["graphs"][phase], s["loss_hosts"][phase], transition)
        self._updates += 1
        self.trainer.all_batches_processed += 1
        return out


assert set(FusedDqnStep._per_trainers + FusedPolicyStep._per_trainers) == set(_PRIORITY_SOURCES)


def capture_device_only(trainer, rb, batch_size, steps, queries_dev, process_group=None,
                        overlap_sampling=True):
    """`steps` consecutive updates in ONE graph with all random numbers already resident in
    HBM (queries_dev[k] is the k-th update's draw) -- the kernel-only measurement of
    bench.py.  With `overlap_sampling` the replay-sample kernel of update k+1 is captured on a
    second stream and runs concurrently with the TD / weight-gradient / Adam kernels of update
    k (the row-tile kernels leave ~20 SMs and most of HBM idle; sampling does not depend on
    the parameters, and no trainer of the path writes priorities back -- SURVEY.md fact 5)."""
    A = trainer.num_actions
    kw = _query_keyword(rb)

    def sample(k):
        return rb.sample_discrete_dqn_batch(batch_size, A, **{kw: queries_dev[k]})

    g = torch.cuda.CUDAGraph()
    keep = []  # every batch stays alive until the capture ends: no cross-stream block reuse
    side = torch.cuda.Stream()
    with torch.cuda.graph(g):
        main = torch.cuda.current_stream()
        batch = sample(0)
        keep.append(batch)
        for k in range(steps):
            nxt = None
            if overlap_sampling and k + 1 < steps:
                side.wait_stream(main)
                with torch.cuda.stream(side):
                    nxt = sample(k + 1)
                keep.append(nxt)
            loss = trainer.train_batch(batch, process_group=process_group)
            if k + 1 < steps:
                if nxt is None:
                    nxt = sample(k + 1)
                    keep.append(nxt)
                else:
                    main.wait_stream(side)
                batch = nxt
    g._rb200_keep = keep
    g._rb200_last_loss = loss  # graph-owned: the loss of the last update after every replay
    return g
