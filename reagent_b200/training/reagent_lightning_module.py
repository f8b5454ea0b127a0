"""Generator-style trainer base with the reference's protocol
(reagent/training/reagent_lightning_module.py:20-143): `train_step_gen` yields one loss per
optimizer returned by `configure_optimizers()`, `training_step(batch, batch_idx,
optimizer_idx)` advances it, the yield count is verified on the first batch.

pytorch_lightning is not a dependency here: the class is a plain nn.Module exposing the
LightningModule members the hot path touches (`log`, `logger`, `trainer.log_every_n_steps`,
`reporter`).  A Lightning-style loop is provided by reagent_b200.training.loop.
"""
import inspect
import logging

import torch

from ..optimizer import FusedAdam, SoftUpdate
from .data_parallel import dp_fused_step

logger = logging.getLogger(__name__)


class DummyExperiment:
    """pl.loggers.base.DummyExperiment stand-in: swallows every call."""

    def nop(self, *args, **kw):
        return None

    def __getattr__(self, _):
        return self.nop

    def __getitem__(self, idx):
        return self


class _TrainerStub:
    log_every_n_steps = 50


class _FusedLoss(torch.autograd.Function):
    """Gives the device-resident loss scalar a grad_fn so `loss.backward()` (what a
    Lightning-style loop calls) is legal.  The gradients were already produced by the fused
    backward kernels and sit in the network arenas; backward() is therefore a no-op."""

    @staticmethod
    def forward(ctx, loss_value, anchor):
        return loss_value.view_as(loss_value)

    @staticmethod
    def backward(ctx, grad_output):
        return None, None


class ReAgentLightningModule(torch.nn.Module):
    def __init__(self, automatic_optimization=True):
        super().__init__()
        self._automatic_optimization = automatic_optimization
        self._training_step_generator = None
        self._reporter = DummyExperiment()
        self._verified_steps = False
        self.register_buffer("_next_stopping_epoch", None)
        self.register_buffer("_cleanly_stopped", None)
        self._next_stopping_epoch = torch.tensor([-1]).int()
        self._cleanly_stopped = torch.ones(1)
        self._setup_input_type()
        self.train_batches_processed_this_epoch = 0
        self.val_batches_processed_this_epoch = 0
        self.test_batches_processed_this_epoch = 0
        self.all_batches_processed = 0
        self.logger = None
        self.trainer = _TrainerStub()
        self._logged = {}
        self._optimizers_cache = None
        # leaf that lets yielded device losses carry a grad_fn
        self._loss_anchor = torch.zeros(1, requires_grad=True)  # plain tensor: not a parameter

    # ---- reference API ------------------------------------------------------
    def _setup_input_type(self):
        self._training_batch_type = None
        sig = inspect.signature(self.train_step_gen)
        assert "training_batch" in sig.parameters
        annotation = sig.parameters["training_batch"].annotation
        if annotation == inspect.Parameter.empty:
            return
        if hasattr(annotation, "from_dict"):
            self._training_batch_type = annotation

    def set_reporter(self, reporter):
        if reporter is None:
            reporter = DummyExperiment()
        self._reporter = reporter
        return self

    @property
    def reporter(self):
        return self._reporter

    @property
    def has_real_reporter(self) -> bool:
        return not isinstance(self._reporter, DummyExperiment)

    def set_clean_stop(self, clean_stop: bool):
        self._cleanly_stopped[0] = int(clean_stop)

    def increase_next_stopping_epochs(self, num_epochs: int):
        self._next_stopping_epoch += num_epochs
        self.set_clean_stop(False)
        return self

    def log(self, name, value, **kwargs):
        self._logged[name] = value

    def train_step_gen(self, training_batch, batch_idx: int):
        raise NotImplementedError

    def soft_update_result(self) -> torch.Tensor:
        """A dummy loss to trigger soft-update (reagent_lightning_module.py:76-81)."""
        one = torch.ones(1, requires_grad=True)
        return one + one

    def fused_loss(self, loss_value: torch.Tensor) -> torch.Tensor:
        anchor = self._loss_anchor
        if anchor.device != loss_value.device:
            self._loss_anchor = torch.zeros(1, device=loss_value.device, requires_grad=True)
            anchor = self._loss_anchor
        return _FusedLoss.apply(loss_value, anchor)

    @property
    def _num_optimizing_steps(self) -> int:
        return len(self.optimizers())

    def optimizers(self, use_pl_optimizer: bool = True):
        if self._optimizers_cache is None:
            # configure_optimizers() returns {"optimizer": ...} dicts or bare optimizers
            opts = [o["optimizer"] if isinstance(o, dict) else o
                    for o in self.configure_optimizers()]
            # which optimizer trains each network arena, and which target its SoftUpdate moves
            # with it: the fast path's Adam and Polyak launches follow configure_optimizers()
            self._adam_of = {o.arena: o for o in opts if isinstance(o, FusedAdam)}
            self._polyak_of = {sa: (ta, o) for o in opts if isinstance(o, SoftUpdate)
                               for ta, sa in o._pairs}
            self._optimizers_cache = opts
        return self._optimizers_cache

    def optimizer_of(self, arena):
        """The FusedAdam / FusedAdamW of configure_optimizers() that trains `arena`."""
        self.optimizers()
        opt = self._adam_of.get(arena)
        if opt is None:
            raise KeyError(f"no optimizer of {type(self).__name__}.configure_optimizers() trains "
                           "this network (was it moved after optimizers() was first called?)")
        return opt

    def adam_step(self, arena, process_group=None, polyak: bool = True, **kw):
        """The Adam step of `arena` (data_parallel.dp_fused_step), with the Polyak update of the
        target that configure_optimizers()' SoftUpdate pairs with it folded into the same launch
        when `polyak` is set and there is one.  Returns what FusedAdam.fused_step returns."""
        opt = self.optimizer_of(arena)
        pair = self._polyak_of.get(arena) if polyak else None
        if pair is not None:
            kw.update(target=pair[0], tau=pair[1].param_groups[0]["tau"])
        return dp_fused_step(opt, process_group, **kw)

    def soft_update(self, arena):
        """The Polyak update of the target paired with `arena`, as a launch of its own (a
        batch that moves the target without an Adam step of `arena`)."""
        self.optimizers()
        target, su = self._polyak_of[arena]
        su.update(target, arena)

    def training_step(self, batch, batch_idx: int, optimizer_idx: int = 0):
        assert (optimizer_idx == 0) or (self._num_optimizing_steps > 1)
        if self._training_step_generator is None:
            if self._training_batch_type and isinstance(batch, dict):
                batch = self._training_batch_type.from_dict(batch)
            self._training_step_generator = self.train_step_gen(batch, batch_idx)
        ret = next(self._training_step_generator)
        if optimizer_idx == self._num_optimizing_steps - 1:
            if not self._verified_steps:
                try:
                    next(self._training_step_generator)
                except StopIteration:
                    self._verified_steps = True
                if not self._verified_steps:
                    raise RuntimeError(
                        "training_step_gen() yields too many times."
                        "The number of yields should match the number of optimizers,"
                        f" in this case {self._num_optimizing_steps}")
            self._training_step_generator = None
            self.all_batches_processed += 1
        return ret
