"""Batch types at the trainer boundary -- same names, fields and shapes as the reference's
`rlt` (reagent/core/types.py:48-108, :312-338, :688-816, :899-915).  Only the dense,
in-scope fields are kept; `.cuda()/.to()/.cpu()` fan out over tensor members like
TensorDataClass.__getattr__ does."""
import dataclasses
from dataclasses import dataclass, field
from typing import List, Optional

import torch


@dataclass
class TensorDataClass:
    def _map(self, fn):
        out = {}
        for f in dataclasses.fields(self):
            v = getattr(self, f.name)
            if isinstance(v, torch.Tensor):
                out[f.name] = fn(v)
            elif isinstance(v, TensorDataClass):
                out[f.name] = v._map(fn)
            else:
                out[f.name] = v
        return type(self)(**out)

    def cuda(self, *args, **kwargs):
        kwargs.setdefault("non_blocking", True)
        return self._map(lambda t: t.cuda(*args, **kwargs))

    def cpu(self):
        return self._map(lambda t: t.cpu())

    def to(self, *args, **kwargs):
        return self._map(lambda t: t.to(*args, **kwargs))

    def float(self):
        return self._map(lambda t: t.float())

    def detach(self):
        return self._map(lambda t: t.detach())

    def pin_memory(self):
        return self._map(lambda t: t.pin_memory())


@dataclass
class DocList(TensorDataClass):
    """core/types.py:250-284: the candidate documents of each row.  float_features is
    (batch_size, num_candidates, doc_dim); mask (present or not) and value (e.g. a selection
    probability) are (batch_size, num_candidates), defaulting to all present and 1."""
    float_features: torch.Tensor
    mask: torch.Tensor = None
    value: torch.Tensor = None

    def __post_init__(self):
        assert len(self.float_features.shape) == 3, f"Unexpected shape: {self.float_features.shape}"
        if self.mask is None:
            self.mask = self.float_features.new_ones(self.float_features.shape[:2], dtype=torch.bool)
        if self.value is None:
            self.value = self.float_features.new_ones(self.float_features.shape[:2])

    @torch.no_grad()
    def select_slate(self, action: torch.Tensor):
        """The documents at `action` [batch_size, slate_size] (indices into the candidates)."""
        row_idx = torch.repeat_interleave(
            torch.arange(action.shape[0], device=action.device).unsqueeze(1), action.shape[1], dim=1)
        return DocList(self.float_features[row_idx, action], self.mask[row_idx, action],
                       self.value[row_idx, action])

    def as_feature_data(self):
        _batch_size, _slate_size, feature_dim = self.float_features.shape
        return FeatureData(self.float_features.view(-1, feature_dim))


@dataclass
class FeatureData(TensorDataClass):
    # dense features, shape (batch_size, feature_dim)
    float_features: torch.Tensor
    # the candidate documents of each row (SlateQ), core/types.py:329
    candidate_docs: Optional[DocList] = None

    def __post_init__(self):
        # (batch_size, feature_dim), or (seq_len, batch_size, feature_dim) for sequences
        if self.float_features.ndim not in (2, 3):
            raise ValueError("float_features should be 2D (or 3D for a sequence); got "
                             f"{tuple(self.float_features.shape)}")


@dataclass
class ActorOutput(TensorDataClass):
    action: torch.Tensor
    log_prob: Optional[torch.Tensor] = None
    squashed_mean: Optional[torch.Tensor] = None


@dataclass
class ExtraData(TensorDataClass):
    mdp_id: Optional[torch.Tensor] = None
    sequence_number: Optional[torch.Tensor] = None
    action_probability: Optional[torch.Tensor] = None
    max_num_actions: Optional[int] = None
    metrics: Optional[torch.Tensor] = None


@dataclass
class BaseInput(TensorDataClass):
    state: FeatureData
    next_state: FeatureData
    reward: torch.Tensor
    time_diff: Optional[torch.Tensor]
    step: Optional[torch.Tensor]
    not_terminal: torch.Tensor

    def __len__(self):
        return self.state.float_features.size()[0]

    def batch_size(self):
        return len(self)


@dataclass
class DiscreteDqnInput(BaseInput):
    action: torch.Tensor = None
    next_action: torch.Tensor = None
    possible_actions_mask: torch.Tensor = None
    possible_next_actions_mask: torch.Tensor = None
    extras: Optional[ExtraData] = None

    @classmethod
    def from_dict(cls, batch):
        return cls(
            state=FeatureData(batch["state_features"]),
            next_state=FeatureData(batch["next_state_features"]),
            reward=batch["reward"],
            time_diff=batch.get("time_diff"),
            step=batch.get("step"),
            not_terminal=batch["not_terminal"],
            action=batch["action"],
            next_action=batch["next_action"],
            possible_actions_mask=batch["possible_actions_mask"],
            possible_next_actions_mask=batch["possible_next_actions_mask"],
            extras=batch.get("extras", ExtraData()),
        )


@dataclass
class PolicyNetworkInput(BaseInput):
    action: FeatureData = None
    next_action: FeatureData = None
    extras: Optional[ExtraData] = None

    @classmethod
    def from_dict(cls, batch):
        return cls(
            state=FeatureData(batch["state_features"]),
            next_state=FeatureData(batch["next_state_features"]),
            reward=batch["reward"],
            time_diff=batch.get("time_diff"),
            step=batch.get("step"),
            not_terminal=batch["not_terminal"],
            action=FeatureData(batch["action"]),
            next_action=FeatureData(batch["next_action"]),
            extras=batch.get("extras"),
        )


# ---- dense feature configuration (core/types.py:152-155, :181-215); sparse id-list features
# are out of scope of this package (SURVEY.md 8a), so the config is dense-only ----
@dataclass
class FloatFeatureInfo:
    name: str
    feature_id: int


@dataclass
class ModelFeatureConfig:
    float_feature_infos: List[FloatFeatureInfo] = field(default_factory=list)

    @property
    def only_dense(self):
        return True


@dataclass
class ParametricDqnInput(BaseInput):
    """core/types.py:867-897: actions are feature vectors; the possible (next) actions of a row
    are tiled along the batch dimension -- (batch_size * max_num_action, action_dim)."""
    action: FeatureData = None
    next_action: FeatureData = None
    possible_actions: FeatureData = None
    possible_actions_mask: torch.Tensor = None
    possible_next_actions: FeatureData = None
    possible_next_actions_mask: torch.Tensor = None
    extras: Optional[ExtraData] = None
    weight: Optional[torch.Tensor] = None

    @classmethod
    def from_dict(cls, batch):
        return cls(
            state=FeatureData(batch["state_features"]),
            action=FeatureData(batch["action"]),
            next_state=FeatureData(batch["next_state_features"]),
            next_action=FeatureData(batch["next_action"]),
            possible_actions=FeatureData(batch["possible_actions"]),
            possible_actions_mask=batch["possible_actions_mask"],
            possible_next_actions=FeatureData(batch["possible_next_actions"]),
            possible_next_actions_mask=batch["possible_next_actions_mask"],
            reward=batch["reward"],
            not_terminal=batch["not_terminal"],
            time_diff=batch.get("time_diff"),
            step=batch.get("step"),
            extras=batch.get("extras"),
            weight=batch.get("weight"),
        )


@dataclass
class SlateQInput(BaseInput):
    """core/types.py:820-863: `action` / `next_action` are (batch_size, slate_size) indices into
    the candidate docs of state / next_state; `reward` and `reward_mask` are per slate position,
    (batch_size, slate_size)."""
    action: torch.Tensor = None
    next_action: torch.Tensor = None
    reward_mask: torch.Tensor = None
    extras: Optional[ExtraData] = None

    @classmethod
    def from_dict(cls, d):
        return cls(
            state=FeatureData(
                float_features=d["state_features"],
                candidate_docs=DocList(float_features=d["candidate_features"],
                                       mask=d["item_mask"], value=d["item_probability"])),
            next_state=FeatureData(
                float_features=d["next_state_features"],
                candidate_docs=DocList(float_features=d["next_candidate_features"],
                                       mask=d["next_item_mask"], value=d["next_item_probability"])),
            action=d["action"],
            next_action=d["next_action"],
            reward=d["position_reward"],
            reward_mask=d["reward_mask"],
            time_diff=d["time_diff"],
            not_terminal=d["not_terminal"],
            step=None,
            extras=ExtraData(**{f.name: d.get(f.name) for f in dataclasses.fields(ExtraData)}),
        )


@dataclass
class BehavioralCloningModelInput(TensorDataClass):
    """core/types.py:998-1015: states, the logged action as a one-hot row per state, and the
    actions that were possible (1) or not (0)."""
    state: FeatureData
    action: torch.Tensor
    possible_actions_mask: Optional[torch.Tensor] = None

    @classmethod
    def from_dict(cls, batch):
        return cls(
            state=FeatureData(float_features=batch["state"]),
            action=batch["action"],
            possible_actions_mask=batch.get("possible_actions_mask", None),
        )

    def batch_size(self):
        assert self.state.float_features.ndim == 2
        return self.state.float_features.size()[0]


@dataclass
class PolicyGradientInput(TensorDataClass):
    """core/types.py:919-966: ONE trajectory -- its states, the logged one-hot actions [T, A],
    rewards [T] and log-probabilities [T] of the logged actions, and optionally the possible
    actions, the next states and a per-step not_terminal [T] (None: a complete episode that
    ends in a terminal state)."""
    state: FeatureData
    action: torch.Tensor
    reward: torch.Tensor
    log_prob: torch.Tensor
    possible_actions_mask: Optional[torch.Tensor] = None
    next_state: Optional[FeatureData] = None
    not_terminal: Optional[torch.Tensor] = None

    @classmethod
    def input_prototype(cls, action_dim=2, batch_size=10, state_dim=3):
        return cls(
            state=FeatureData(float_features=torch.randn(batch_size, state_dim)),
            action=torch.nn.functional.one_hot(
                torch.randint(high=action_dim, size=(batch_size,)), num_classes=action_dim),
            reward=torch.rand(batch_size),
            log_prob=torch.log(torch.rand(batch_size)),
            possible_actions_mask=torch.ones(batch_size, action_dim),
        )

    @classmethod
    def from_dict(cls, d):
        next_observation = d.get("next_observation", None)
        return cls(
            state=FeatureData(float_features=d["observation"]),
            action=d["action"],
            reward=d["reward"],
            log_prob=d["log_prob"],
            possible_actions_mask=d.get("possible_actions_mask", None),
            next_state=(FeatureData(float_features=next_observation)
                        if next_observation is not None else None),
            not_terminal=d.get("not_terminal", None),
        )

    def __len__(self):
        assert self.action.ndim == 2
        return len(self.action)

    def batch_size(self):
        return len(self)


@dataclass
class MemoryNetworkInput(BaseInput):
    """A time-major batch of sequences (reagent/core/types.py MemoryNetworkInput): state,
    next_state and action are [T, B, dim]; reward and not_terminal are [T, B]."""
    action: FeatureData = None
    valid_step: Optional[torch.Tensor] = None
    extras: ExtraData = field(default_factory=ExtraData)

    @classmethod
    def from_dict(cls, d):
        return cls(
            state=FeatureData(float_features=d["state"]),
            next_state=FeatureData(float_features=d["next_state"]),
            action=FeatureData(float_features=d["action"]),
            reward=d["reward"],
            time_diff=d["time_diff"],
            not_terminal=d["not_terminal"],
            step=d["step"],
            extras=ExtraData(**{f.name: d.get(f.name) for f in dataclasses.fields(ExtraData)}),
        )

    def __len__(self):
        if len(self.state.float_features.size()) == 2:
            return self.state.float_features.size()[0]
        elif len(self.state.float_features.size()) == 3:
            return self.state.float_features.size()[1]
        else:
            raise NotImplementedError()


@dataclass
class Seq2RewardOutput(TensorDataClass):
    acc_reward: torch.Tensor


@dataclass
class MemoryNetworkOutput(TensorDataClass):
    mus: torch.Tensor
    sigmas: torch.Tensor
    logpi: torch.Tensor
    reward: torch.Tensor
    not_terminal: torch.Tensor
    last_step_lstm_hidden: torch.Tensor
    last_step_lstm_cell: torch.Tensor
    all_steps_lstm_hidden: torch.Tensor


PADDING_SYMBOL = 0
DECODER_START_SYMBOL = 1


def _gather_rows(data: torch.Tensor, index_2d: torch.Tensor) -> torch.Tensor:
    """out[i, j] = data[i, index_2d[i, j]] (reagent/core/torch_utils.py:gather)."""
    rows = torch.arange(data.shape[0], device=data.device).unsqueeze(1)
    return data[rows, index_2d]


@dataclass
class PreprocessedRankingInput(TensorDataClass):
    """A batch of slates (reference core/types.py:453).  Every index counts the padding
    symbol 0 and the decoder start symbol 1, so candidate i is symbol i + 2."""
    state: FeatureData
    src_seq: FeatureData
    src_src_mask: Optional[torch.Tensor] = None
    tgt_in_seq: Optional[FeatureData] = None
    tgt_out_seq: Optional[FeatureData] = None
    tgt_tgt_mask: Optional[torch.Tensor] = None
    slate_reward: Optional[torch.Tensor] = None
    position_reward: Optional[torch.Tensor] = None
    src_in_idx: Optional[torch.Tensor] = None
    tgt_in_idx: Optional[torch.Tensor] = None
    tgt_out_idx: Optional[torch.Tensor] = None
    tgt_out_probs: Optional[torch.Tensor] = None
    optim_tgt_in_idx: Optional[torch.Tensor] = None
    optim_tgt_out_idx: Optional[torch.Tensor] = None
    optim_tgt_in_seq: Optional[FeatureData] = None
    optim_tgt_out_seq: Optional[FeatureData] = None
    extras: Optional[ExtraData] = field(default_factory=ExtraData)

    def batch_size(self) -> int:
        return self.state.float_features.size()[0]

    def __len__(self) -> int:
        return self.batch_size()

    @classmethod
    def from_input(cls, state: torch.Tensor, candidates: torch.Tensor, device: torch.device,
                   action: Optional[torch.Tensor] = None,
                   optimal_action: Optional[torch.Tensor] = None,
                   logged_propensities: Optional[torch.Tensor] = None,
                   slate_reward: Optional[torch.Tensor] = None,
                   position_reward: Optional[torch.Tensor] = None,
                   extras: Optional[ExtraData] = None):
        """Derive the decoder's indices and sequences from state [B, S], candidates [B, N, C]
        and the 0-based slates `action` / `optimal_action` [B, T]: tgt_out_idx = action + 2,
        tgt_in_idx = (1, tgt_out_idx[:, :-1]), and their candidate features (zeros for the start
        symbol)."""
        assert len(state.shape) == 2
        assert len(candidates.shape) == 3
        state = state.to(device)
        candidates = candidates.to(device)
        if action is not None:
            assert len(action.shape) == 2
            action = action.to(device)
        if logged_propensities is not None:
            assert len(logged_propensities.shape) == 2 and logged_propensities.shape[1] == 1
            logged_propensities = logged_propensities.to(device)
        batch_size, candidate_num, candidate_dim = candidates.shape
        if slate_reward is not None:
            assert len(slate_reward.shape) == 2 and slate_reward.shape[1] == 1
            slate_reward = slate_reward.to(device)
        if position_reward is not None:
            assert position_reward.shape == action.shape
            position_reward = position_reward.to(device)
        src_in_idx = torch.arange(candidate_num, device=device).repeat(batch_size, 1) + 2
        src_src_mask = torch.ones(batch_size, candidate_num, candidate_num,
                                  device=device).type(torch.int8)

        def process_tgt_seq(action):
            if action is None:
                return None, None, None, None, None
            output_size = action.shape[1]
            augmented = torch.cat(
                (torch.zeros(batch_size, 2, candidate_dim, device=device), candidates), dim=1)
            tgt_out_idx = action + 2
            tgt_in_idx = torch.full((batch_size, output_size), DECODER_START_SYMBOL,
                                    device=device)
            tgt_in_idx[:, 1:] = tgt_out_idx[:, :-1]
            tgt_out_seq = _gather_rows(augmented, tgt_out_idx)
            tgt_in_seq = torch.zeros(batch_size, output_size, candidate_dim, device=device)
            tgt_in_seq[:, 1:] = tgt_out_seq[:, :-1]
            tgt_tgt_mask = ~torch.triu(
                torch.ones(1, output_size, output_size, device=device, dtype=torch.bool),
                diagonal=1)
            return tgt_in_idx, tgt_out_idx, tgt_in_seq, tgt_out_seq, tgt_tgt_mask

        tgt_in_idx, tgt_out_idx, tgt_in_seq, tgt_out_seq, tgt_tgt_mask = process_tgt_seq(action)
        optim_in_idx, optim_out_idx, optim_in_seq, optim_out_seq, _ = process_tgt_seq(
            optimal_action)
        return cls.from_tensors(
            state=state, src_seq=candidates, src_src_mask=src_src_mask, tgt_in_seq=tgt_in_seq,
            tgt_out_seq=tgt_out_seq, tgt_tgt_mask=tgt_tgt_mask, slate_reward=slate_reward,
            position_reward=position_reward, src_in_idx=src_in_idx, tgt_in_idx=tgt_in_idx,
            tgt_out_idx=tgt_out_idx, tgt_out_probs=logged_propensities,
            optim_tgt_in_idx=optim_in_idx, optim_tgt_out_idx=optim_out_idx,
            optim_tgt_in_seq=optim_in_seq, optim_tgt_out_seq=optim_out_seq, extras=extras)

    @classmethod
    def from_tensors(cls, state: torch.Tensor, src_seq: torch.Tensor,
                     src_src_mask: Optional[torch.Tensor] = None,
                     tgt_in_seq: Optional[torch.Tensor] = None,
                     tgt_out_seq: Optional[torch.Tensor] = None,
                     tgt_tgt_mask: Optional[torch.Tensor] = None,
                     slate_reward: Optional[torch.Tensor] = None,
                     position_reward: Optional[torch.Tensor] = None,
                     src_in_idx: Optional[torch.Tensor] = None,
                     tgt_in_idx: Optional[torch.Tensor] = None,
                     tgt_out_idx: Optional[torch.Tensor] = None,
                     tgt_out_probs: Optional[torch.Tensor] = None,
                     optim_tgt_in_idx: Optional[torch.Tensor] = None,
                     optim_tgt_out_idx: Optional[torch.Tensor] = None,
                     optim_tgt_in_seq: Optional[torch.Tensor] = None,
                     optim_tgt_out_seq: Optional[torch.Tensor] = None,
                     extras: Optional[ExtraData] = None, **kwargs):
        """Wrap plain tensors; the sequences become FeatureData."""
        for v in (state, src_seq):
            assert isinstance(v, torch.Tensor)
        for v in (src_src_mask, tgt_in_seq, tgt_out_seq, tgt_tgt_mask, slate_reward,
                  position_reward, src_in_idx, tgt_in_idx, tgt_out_idx, tgt_out_probs,
                  optim_tgt_in_idx, optim_tgt_out_idx, optim_tgt_in_seq, optim_tgt_out_seq):
            assert v is None or isinstance(v, torch.Tensor)
        assert extras is None or isinstance(extras, ExtraData)
        fd = lambda t: None if t is None else FeatureData(float_features=t)  # noqa: E731
        return cls(
            state=FeatureData(float_features=state), src_seq=FeatureData(float_features=src_seq),
            src_src_mask=src_src_mask, tgt_in_seq=fd(tgt_in_seq), tgt_out_seq=fd(tgt_out_seq),
            tgt_tgt_mask=tgt_tgt_mask, slate_reward=slate_reward, position_reward=position_reward,
            src_in_idx=src_in_idx, tgt_in_idx=tgt_in_idx, tgt_out_idx=tgt_out_idx,
            tgt_out_probs=tgt_out_probs, optim_tgt_in_idx=optim_tgt_in_idx,
            optim_tgt_out_idx=optim_tgt_out_idx, optim_tgt_in_seq=fd(optim_tgt_in_seq),
            optim_tgt_out_seq=fd(optim_tgt_out_seq), extras=extras)


@dataclass
class RankingOutput(TensorDataClass):
    # ranked symbols (candidate i is i + 2), [B, T]
    ranked_tgt_out_idx: Optional[torch.Tensor] = None
    # the probabilities of every symbol at each decoding step, [B, T, N + 2]
    ranked_per_symbol_probs: Optional[torch.Tensor] = None
    # the probability of each ranked sequence, [B, 1]
    ranked_per_seq_probs: Optional[torch.Tensor] = None
    # [B, 1] (PER_SEQ_LOG_PROB_MODE) or [B, T, N + 2] (PER_SYMBOL_LOG_PROB_DIST_MODE)
    log_probs: Optional[torch.Tensor] = None
    encoder_scores: Optional[torch.Tensor] = None
