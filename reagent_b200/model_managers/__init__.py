"""Model managers: `build_trainer(normalization_data_map, use_gpu, reward_options=None)` with
the reference's flow (reagent/model_managers/model_manager.py:84-96 and
discrete/discrete_dqn.py:63-116, discrete/discrete_qrdqn.py:73-121,
discrete/discrete_c51dqn.py:43-88, parametric/parametric_dqn.py:45-81,
actor_critic/sac.py:80-113, actor_critic/td3.py:70-102, discrete/discrete_crr.py:104-179,
policy_gradient/reinforce.py, policy_gradient/ppo.py, model_based/world_model.py,
model_based/cross_entropy_method.py, ranking/slate_q.py): build the networks from the net
builders, copy the target, hand everything to the trainer; `create_policy` gives the online
act-time policy.  Serving modules, data modules and reporters are out of scope (SURVEY.md
section 2 rows 8, 12, 15, 16)."""
from dataclasses import dataclass, field
from typing import Union, Dict, List, Optional, Tuple

from ..core import types as rlt
from ..core.parameters import (CEMTrainerParameters, EvaluationParameters,
                               MDNRNNTrainerParameters, NormalizationData, NormalizationKey,
                               RLParameters, Seq2RewardTrainerParameters,
                               SlateQTrainerParameters)
from ..net_builder import (ActorFullyConnected, Categorical, DiscreteActorFullyConnected,
                           Dueling, DuelingQuantile, FullyConnected, GaussianFullyConnected, ParametricFullyConnected,
                           Quantile, Seq2RewardNetBuilder, ValueFullyConnected)
from ..optimizer import Optimizer__Union
from ..training import (C51Trainer, CEMTrainer, CRRWeightFn, DiscreteCRRTrainer, DQNTrainer,
                        MDNRNNTrainer, ParametricDQNTrainer, PPOTrainer, QRDQNTrainer, ReinforceTrainer,
                        SACTrainer, Seq2RewardTrainer, SlateQTrainer, TD3Trainer)


def _device(use_gpu: bool):
    if not use_gpu:
        raise RuntimeError("reagent_b200 trainers run on CUDA only; build_trainer needs use_gpu=True")
    return "cuda"


class _DiscretePolicyMixin:
    def create_policy(self, trainer_module, serving: bool = False, normalization_data_map=None):
        """Online policy (reagent/model_managers/discrete_dqn_base.py:84-103): greedy over the
        fused Q-network forward.  Serving modules are out of scope."""
        if serving:
            raise NotImplementedError("serving modules are out of scope of reagent_b200")
        from ..gym.policies import GreedyActionSampler, Policy, discrete_dqn_scorer

        return Policy(scorer=discrete_dqn_scorer(trainer_module.q_network),
                      sampler=GreedyActionSampler())


class _ActorPolicyMixin:
    def create_policy(self, trainer_module, serving: bool = False, normalization_data_map=None):
        """reagent/model_managers/actor_critic_base.py:104-118: the actor's forward is the act."""
        if serving:
            raise NotImplementedError("serving modules are out of scope of reagent_b200")
        from ..gym.policies import ActorPolicyWrapper

        return ActorPolicyWrapper(trainer_module.actor_network)


@dataclass
class DiscreteDQN(_DiscretePolicyMixin):
    actions: List[str]
    rl: RLParameters = field(default_factory=RLParameters)
    double_q_learning: bool = True
    minibatch_size: int = 1024
    optimizer: Optimizer__Union = field(default_factory=Optimizer__Union.default)
    # reagent/model_managers/discrete/discrete_dqn.py:33-36: the reference defaults to Dueling
    net_builder: Union[Dueling, FullyConnected] = field(default_factory=Dueling)
    # :37-42: the reward / CPE networks are plain FullyConnected
    cpe_net_builder: Union[Dueling, FullyConnected] = field(default_factory=FullyConnected)
    # EvaluationParameters() has calc_cpe_in_training=True, as in the reference
    # (reagent/core/parameters.py:118-120)
    eval_parameters: EvaluationParameters = field(default_factory=EvaluationParameters)
    metrics_to_score: Optional[List[str]] = None

    def build_trainer(self, normalization_data_map: Dict[str, NormalizationData], use_gpu: bool,
                      reward_options=None) -> DQNTrainer:
        """discrete_dqn.py:73-116"""
        dev = _device(use_gpu)
        s_norm = normalization_data_map[NormalizationKey.STATE]
        q_network = self.net_builder.build_q_network(None, s_norm, len(self.actions)).to(dev)
        q_network_target = q_network.get_target_network()
        reward_network = q_network_cpe = q_network_cpe_target = None
        metrics = list(self.metrics_to_score or [])
        if self.eval_parameters.calc_cpe_in_training:
            n_out = (len(metrics) + 1) * len(self.actions)  # metrics + reward
            reward_network = self.cpe_net_builder.build_q_network(None, s_norm, n_out).to(dev)
            q_network_cpe = self.cpe_net_builder.build_q_network(None, s_norm, n_out).to(dev)
            q_network_cpe_target = q_network_cpe.get_target_network()
        return DQNTrainer(
            q_network=q_network, q_network_target=q_network_target,
            reward_network=reward_network, q_network_cpe=q_network_cpe,
            q_network_cpe_target=q_network_cpe_target, metrics_to_score=metrics,
            actions=self.actions, rl=self.rl, double_q_learning=self.double_q_learning,
            minibatch_size=self.minibatch_size, optimizer=self.optimizer,
            evaluation=self.eval_parameters).to(dev)


@dataclass
class DiscreteQRDQN(_DiscretePolicyMixin):
    actions: List[str]
    rl: RLParameters = field(default_factory=RLParameters)
    double_q_learning: bool = True
    num_atoms: int = 51
    minibatch_size: int = 1024
    optimizer: Optimizer__Union = field(default_factory=Optimizer__Union.default)
    # reagent/model_managers/discrete/discrete_qrdqn.py:39-43: the reference defaults to DuelingQuantile
    net_builder: Union[DuelingQuantile, Quantile] = field(default_factory=DuelingQuantile)
    eval_parameters: EvaluationParameters = field(
        default_factory=lambda: EvaluationParameters(calc_cpe_in_training=False))

    def build_trainer(self, normalization_data_map, use_gpu: bool, reward_options=None):
        dev = _device(use_gpu)
        q_network = self.net_builder.build_q_network(
            normalization_data_map[NormalizationKey.STATE], len(self.actions),
            self.num_atoms).to(dev)
        q_network_target = q_network.get_target_network()
        return QRDQNTrainer(
            q_network=q_network, q_network_target=q_network_target, actions=self.actions,
            rl=self.rl, double_q_learning=self.double_q_learning, num_atoms=self.num_atoms,
            minibatch_size=self.minibatch_size, optimizer=self.optimizer,
            evaluation=self.eval_parameters).to(dev)


@dataclass
class DiscreteC51DQN(_DiscretePolicyMixin):
    actions: List[str]
    rl: RLParameters = field(default_factory=RLParameters)
    double_q_learning: bool = True
    num_atoms: int = 51
    qmin: float = -100
    qmax: float = 200
    minibatch_size: int = 1024
    optimizer: Optimizer__Union = field(default_factory=Optimizer__Union.default)
    net_builder: Categorical = field(default_factory=Categorical)

    def __post_init__(self):
        # discrete_c51dqn.py:43-48
        assert len(self.actions) > 1, "DiscreteC51DQN needs at least 2 actions"
        assert self.minibatch_size % 8 == 0, (
            "The minibatch size must be divisible by 8 for performance reasons.")

    def build_trainer(self, normalization_data_map, use_gpu: bool, reward_options=None):
        dev = _device(use_gpu)
        q_network = self.net_builder.build_q_network(
            normalization_data_map[NormalizationKey.STATE], len(self.actions), self.num_atoms,
            self.qmin, self.qmax).to(dev)
        q_network_target = q_network.get_target_network()
        return C51Trainer(
            q_network=q_network, q_network_target=q_network_target, actions=self.actions,
            rl=self.rl, double_q_learning=self.double_q_learning,
            minibatch_size=self.minibatch_size, num_atoms=self.num_atoms, qmin=self.qmin,
            qmax=self.qmax, optimizer=self.optimizer).to(dev)


@dataclass
class DiscreteCRR(_ActorPolicyMixin):
    """reagent/model_managers/discrete/discrete_crr.py with its `trainer_param`
    (CRRTrainerParameters) flattened into the manager.  The policy is the actor's forward
    (:181-195)."""
    actions: List[str] = field(default_factory=list)
    rl: RLParameters = field(default_factory=RLParameters)
    double_q_learning: bool = True
    q_network_optimizer: Optimizer__Union = field(default_factory=Optimizer__Union.default)
    actor_network_optimizer: Optimizer__Union = field(default_factory=Optimizer__Union.default)
    use_target_actor: bool = False
    delayed_policy_update: int = 1
    beta: float = 1.0
    entropy_coeff: float = 0.0
    clip_limit: float = 10.0
    max_weight: float = 20.0
    actor_net_builder: DiscreteActorFullyConnected = field(
        default_factory=DiscreteActorFullyConnected)
    critic_net_builder: Union[Dueling, FullyConnected] = field(default_factory=Dueling)
    cpe_net_builder: Union[Dueling, FullyConnected] = field(default_factory=FullyConnected)
    eval_parameters: EvaluationParameters = field(default_factory=EvaluationParameters)
    metrics_to_score: Optional[List[str]] = None

    def __post_init__(self):
        # :90-94
        assert len(self.actions) > 1, (
            f"DiscreteCRRModel needs at least 2 actions. Got {self.actions}.")

    @property
    def action_names(self) -> List[str]:
        return self.actions

    @property
    def rl_parameters(self) -> RLParameters:
        return self.rl

    def build_trainer(self, normalization_data_map: Dict[str, NormalizationData], use_gpu: bool,
                      reward_options=None) -> DiscreteCRRTrainer:
        """:104-179: the actor, one or two critics, the reward / CPE networks with one block of
        outputs per metric to score, every target a copy of its network."""
        dev = _device(use_gpu)
        s_norm = normalization_data_map[NormalizationKey.STATE]
        A = len(self.actions)
        actor = self.actor_net_builder.build_actor(s_norm, A).to(dev)
        q1 = self.critic_net_builder.build_q_network(None, s_norm, A).to(dev)
        q2 = q2_target = None
        if self.double_q_learning:
            q2 = self.critic_net_builder.build_q_network(None, s_norm, A).to(dev)
            q2_target = q2.get_target_network()
        metrics = list(self.metrics_to_score or [])
        reward_network = q_network_cpe = q_network_cpe_target = None
        if self.eval_parameters.calc_cpe_in_training:
            n_out = (len(metrics) + 1) * A  # metrics + reward
            reward_network = self.cpe_net_builder.build_q_network(None, s_norm, n_out).to(dev)
            q_network_cpe = self.cpe_net_builder.build_q_network(None, s_norm, n_out).to(dev)
            q_network_cpe_target = q_network_cpe.get_target_network()
        return DiscreteCRRTrainer(
            actor_network=actor, actor_network_target=actor.get_target_network(),
            q1_network=q1, q1_network_target=q1.get_target_network(),
            reward_network=reward_network, q2_network=q2, q2_network_target=q2_target,
            q_network_cpe=q_network_cpe, q_network_cpe_target=q_network_cpe_target,
            metrics_to_score=metrics, evaluation=self.eval_parameters, rl=self.rl,
            double_q_learning=self.double_q_learning,
            q_network_optimizer=self.q_network_optimizer,
            actor_network_optimizer=self.actor_network_optimizer,
            use_target_actor=self.use_target_actor, actions=self.actions,
            delayed_policy_update=self.delayed_policy_update, beta=self.beta,
            entropy_coeff=self.entropy_coeff, clip_limit=self.clip_limit,
            max_weight=self.max_weight).to(dev)


@dataclass
class ParametricDQN:
    """reagent/model_managers/parametric/parametric_dqn.py with its `trainer_param`
    (ParametricDQNTrainerParameters) flattened into the manager, as DiscreteC51DQN does."""
    rl: RLParameters = field(default_factory=RLParameters)
    double_q_learning: bool = True
    minibatches_per_step: int = 1
    optimizer: Optimizer__Union = field(default_factory=Optimizer__Union.default)
    net_builder: ParametricFullyConnected = field(default_factory=ParametricFullyConnected)
    # reagent/model_managers/parametric_dqn_base.py:55: EvaluationParameters() by default
    eval_parameters: EvaluationParameters = field(default_factory=EvaluationParameters)

    @property
    def rl_parameters(self) -> RLParameters:
        return self.rl

    def build_trainer(self, normalization_data_map, use_gpu: bool,
                      reward_options=None) -> ParametricDQNTrainer:
        """parametric_dqn.py:45-81: the q network, a reward network with one output for the
        reward and one per metric to score (get_metrics_to_score: the sorted keys of
        `reward_options.metric_reward_values`), the target as a copy of the q network."""
        dev = _device(use_gpu)
        s, a = (normalization_data_map[NormalizationKey.STATE],
                normalization_data_map[NormalizationKey.ACTION])
        q_network = self.net_builder.build_q_network(s, a).to(dev)
        metric_values = getattr(reward_options, "metric_reward_values", None)
        metrics_to_score = sorted(metric_values) if metric_values else []
        reward_network = self.net_builder.build_q_network(
            s, a, output_dim=len(metrics_to_score) + 1).to(dev)
        q_network_target = q_network.get_target_network()
        return ParametricDQNTrainer(
            q_network=q_network, q_network_target=q_network_target,
            reward_network=reward_network, rl=self.rl,
            double_q_learning=self.double_q_learning,
            minibatches_per_step=self.minibatches_per_step, optimizer=self.optimizer).to(dev)

    def create_policy(self, trainer_module, serving: bool = False, normalization_data_map=None):
        """parametric_dqn_base.py:73-103: softmax over the scores of every one-hot action at
        temperature rl.temperature.  Serving modules are out of scope."""
        if serving:
            raise NotImplementedError("serving modules are out of scope of reagent_b200")
        from ..gym.policies import Policy, SoftmaxActionSampler, parametric_dqn_scorer

        action_dim = trainer_module.q_network.action_dim
        return Policy(scorer=parametric_dqn_scorer(action_dim, trainer_module.q_network),
                      sampler=SoftmaxActionSampler(temperature=self.rl.temperature))


@dataclass
class SAC(_ActorPolicyMixin):
    """The reference manager with `trainer_param` flattened.  `value_net_builder` defaults to
    None here, so SAC() builds no state-value network; the reference's default builds one
    (value FullyConnected, [256, 128] relu).  Configurations that name a value_net_builder,
    such as the reference's Pendulum SAC and CRR configurations, get one either way."""
    rl: RLParameters = field(default_factory=RLParameters)
    actor_net_builder: GaussianFullyConnected = field(default_factory=GaussianFullyConnected)
    critic_net_builder: ParametricFullyConnected = field(default_factory=ParametricFullyConnected)
    value_net_builder: Optional[ValueFullyConnected] = None
    use_2_q_functions: bool = True
    minibatch_size: int = 1024
    entropy_temperature: float = 0.01
    logged_action_uniform_prior: bool = True
    target_entropy: float = -1.0
    q_network_optimizer: Optimizer__Union = field(default_factory=Optimizer__Union.default)
    value_network_optimizer: Optimizer__Union = field(default_factory=Optimizer__Union.default)
    actor_network_optimizer: Optimizer__Union = field(default_factory=Optimizer__Union.default)
    alpha_optimizer: Optional[Optimizer__Union] = field(default_factory=Optimizer__Union.default)
    crr_config: Optional[CRRWeightFn] = None
    backprop_through_log_prob: bool = True

    def build_trainer(self, normalization_data_map, use_gpu: bool, reward_options=None):
        dev = _device(use_gpu)
        s, a = (normalization_data_map[NormalizationKey.STATE],
                normalization_data_map[NormalizationKey.ACTION])
        actor = self.actor_net_builder.build_actor(None, s, a).to(dev)
        q1 = self.critic_net_builder.build_q_network(s, a).to(dev)
        q2 = self.critic_net_builder.build_q_network(s, a).to(dev) if self.use_2_q_functions else None
        value = (None if self.value_net_builder is None
                 else self.value_net_builder.build_value_network(s).to(dev))
        return SACTrainer(
            actor_network=actor, q1_network=q1, q2_network=q2, value_network=value, rl=self.rl,
            q_network_optimizer=self.q_network_optimizer,
            value_network_optimizer=self.value_network_optimizer,
            actor_network_optimizer=self.actor_network_optimizer,
            alpha_optimizer=self.alpha_optimizer, minibatch_size=self.minibatch_size,
            entropy_temperature=self.entropy_temperature,
            logged_action_uniform_prior=self.logged_action_uniform_prior,
            target_entropy=self.target_entropy, crr_config=self.crr_config,
            backprop_through_log_prob=self.backprop_through_log_prob).to(dev)


@dataclass
class TD3(_ActorPolicyMixin):
    rl: RLParameters = field(default_factory=RLParameters)
    actor_net_builder: ActorFullyConnected = field(default_factory=ActorFullyConnected)
    critic_net_builder: ParametricFullyConnected = field(default_factory=ParametricFullyConnected)
    use_2_q_functions: bool = True
    minibatch_size: int = 64
    noise_variance: float = 0.2
    noise_clip: float = 0.5
    delayed_policy_update: int = 2
    q_network_optimizer: Optimizer__Union = field(default_factory=Optimizer__Union.default)
    actor_network_optimizer: Optimizer__Union = field(default_factory=Optimizer__Union.default)

    def build_trainer(self, normalization_data_map, use_gpu: bool, reward_options=None):
        dev = _device(use_gpu)
        s, a = (normalization_data_map[NormalizationKey.STATE],
                normalization_data_map[NormalizationKey.ACTION])
        actor = self.actor_net_builder.build_actor(None, s, a).to(dev)
        q1 = self.critic_net_builder.build_q_network(s, a).to(dev)
        q2 = self.critic_net_builder.build_q_network(s, a).to(dev) if self.use_2_q_functions else None
        return TD3Trainer(
            actor_network=actor, q1_network=q1, q2_network=q2, rl=self.rl,
            q_network_optimizer=self.q_network_optimizer,
            actor_network_optimizer=self.actor_network_optimizer,
            minibatch_size=self.minibatch_size, noise_variance=self.noise_variance,
            noise_clip=self.noise_clip, delayed_policy_update=self.delayed_policy_update).to(dev)


class _PolicyGradientManager:
    """What Reinforce and PPO share (reagent/model_managers/policy_gradient/reinforce.py and
    ppo.py): the policy network from `policy_net_builder` (a discrete-DQN builder, because it
    takes possible_actions_mask), an optional value network, and ONE cached Policy of that
    network and a SoftmaxActionSampler, which the trainer holds and create_policy returns."""
    _name = ""
    _trainer_fields = ()

    def __post_init__(self):
        self._policy = None
        assert len(self.actions) > 1, (
            f"{self._name} needs at least 2 actions. Got {self.actions}.")

    @property
    def action_names(self) -> List[str]:
        return self.actions

    def _create_policy(self, policy_network):
        from ..gym.policies import Policy, SoftmaxActionSampler

        if self._policy is None:
            sampler = SoftmaxActionSampler(temperature=self.sampler_temperature)
            self._policy = Policy(scorer=policy_network, sampler=sampler)
        return self._policy

    def create_policy(self, trainer_module, serving: bool = False, normalization_data_map=None):
        if serving:
            raise NotImplementedError("serving modules are out of scope of reagent_b200")
        return self._create_policy(trainer_module.scorer)

    def build_trainer(self, normalization_data_map: Dict[str, NormalizationData], use_gpu: bool,
                      reward_options=None):
        dev = _device(use_gpu)
        s_norm = normalization_data_map[NormalizationKey.STATE]
        policy_network = self.policy_net_builder.build_q_network(
            None, s_norm, len(self.actions)).to(dev)
        value_net = None
        if self.value_net_builder is not None:
            value_net = self.value_net_builder.build_value_network(s_norm).to(dev)
        kw = {k: getattr(self, k) for k in self._trainer_fields}
        return self._trainer(policy=self._create_policy(policy_network), value_net=value_net,
                             actions=self.actions, **kw).to(dev)


@dataclass
class Reinforce(_PolicyGradientManager):
    """reagent/model_managers/policy_gradient/reinforce.py with its `trainer_param`
    (ReinforceTrainerParameters) flattened into the manager, as DiscreteCRR does."""
    actions: List[str] = field(default_factory=list)
    gamma: float = 0.0
    optimizer: Optimizer__Union = field(default_factory=Optimizer__Union.default)
    optimizer_value_net: Optimizer__Union = field(default_factory=Optimizer__Union.default)
    off_policy: bool = False
    reward_clip: float = 1e6
    clip_param: float = 1e6
    normalize: bool = True
    subtract_mean: bool = True
    offset_clamp_min: bool = False
    policy_net_builder: Union[Dueling, FullyConnected] = field(default_factory=Dueling)
    value_net_builder: Optional[ValueFullyConnected] = None
    sampler_temperature: float = 1.0

    _name = "REINFORCE"
    _trainer = ReinforceTrainer
    _trainer_fields = ("gamma", "optimizer", "optimizer_value_net", "off_policy", "reward_clip",
                       "clip_param", "normalize", "subtract_mean", "offset_clamp_min")


@dataclass
class PPO(_PolicyGradientManager):
    """reagent/model_managers/policy_gradient/ppo.py with its `trainer_param`
    (PPOTrainerParameters) flattened into the manager."""
    actions: List[str] = field(default_factory=list)
    gamma: float = 0.9
    optimizer: Optimizer__Union = field(default_factory=Optimizer__Union.default)
    optimizer_value_net: Optimizer__Union = field(default_factory=Optimizer__Union.default)
    reward_clip: float = 1e6
    normalize: bool = True
    subtract_mean: bool = True
    offset_clamp_min: bool = False
    update_freq: int = 1
    update_epochs: int = 1
    ppo_batch_size: int = 1
    ppo_epsilon: float = 0.2
    entropy_weight: float = 0.0
    td_error_advantage: bool = False
    policy_net_builder: Union[Dueling, FullyConnected] = field(default_factory=Dueling)
    value_net_builder: Optional[ValueFullyConnected] = None
    sampler_temperature: float = 1.0

    _name = "PPO"
    _trainer = PPOTrainer
    _trainer_fields = ("gamma", "optimizer", "optimizer_value_net", "reward_clip", "normalize",
                       "subtract_mean", "offset_clamp_min", "update_freq", "update_epochs",
                       "ppo_batch_size", "ppo_epsilon", "entropy_weight", "td_error_advantage")


@dataclass
class WorldModel:
    """reagent/model_managers/model_based/world_model.py: a MemoryNetwork trained by
    MDNRNNTrainer.  `reward_boost` is WorldModelBase's field (unused by this trainer)."""
    trainer_param: MDNRNNTrainerParameters = field(default_factory=MDNRNNTrainerParameters)
    reward_boost: Optional[Dict[str, float]] = None

    def build_trainer(self, normalization_data_map: Dict[str, NormalizationData], use_gpu: bool,
                      reward_options=None) -> MDNRNNTrainer:
        from ..models.world_model import MemoryNetwork
        from ..preprocessing.normalization import get_num_output_features

        dev = _device(use_gpu)
        p = self.trainer_param
        memory_network = MemoryNetwork(
            state_dim=get_num_output_features(
                normalization_data_map[NormalizationKey.STATE].dense_normalization_parameters),
            action_dim=p.action_dim, num_hiddens=p.hidden_size,
            num_hidden_layers=p.num_hidden_layers, num_gaussians=p.num_gaussians).to(dev)
        return MDNRNNTrainer(memory_network=memory_network, params=p)


class CEMPolicy:
    """reagent/model_managers/model_based/cross_entropy_method.py CEMPolicy: the planner's
    action, returned on the CPU as a [1, A] tensor with log_prob 0."""

    def __init__(self, cem_planner_network, discrete_action: bool):
        self.cem_planner_network = cem_planner_network
        self.discrete_action = discrete_action

    def act(self, obs: rlt.FeatureData, possible_actions_mask=None) -> rlt.ActorOutput:
        import torch

        greedy = self.cem_planner_network(obs)
        if self.discrete_action:
            _, onehot = greedy
            return rlt.ActorOutput(action=onehot.unsqueeze(0), log_prob=torch.tensor(0.0))
        return rlt.ActorOutput(action=greedy.unsqueeze(0), log_prob=torch.tensor(0.0))


@dataclass
class CrossEntropyMethod:
    """reagent/model_managers/model_based/cross_entropy_method.py: num_world_models
    MemoryNetworks, each with its MDNRNNTrainer, and the CEMPlannerNetwork over them.
    `reward_boost` is WorldModelBase's field (unused by this trainer)."""
    trainer_param: CEMTrainerParameters = field(default_factory=CEMTrainerParameters)
    reward_boost: Optional[Dict[str, float]] = None

    def create_policy(self, trainer_module, serving: bool = False, normalization_data_map=None):
        if serving:
            raise NotImplementedError("serving modules are out of scope of reagent_b200")
        assert isinstance(trainer_module, CEMTrainer)
        return CEMPolicy(trainer_module.cem_planner_network, self.discrete_action)

    def build_trainer(self, normalization_data_map: Dict[str, NormalizationData], use_gpu: bool,
                      reward_options=None) -> CEMTrainer:
        """As the reference builds it: one WorldModel trainer built and discarded (it draws its
        initial weights from torch's generator, so the models after it start from the
        reference's weights under torch.manual_seed), then num_world_models trainers, and the
        planner over their networks.  The action type and bounds come from the ACTION
        normalization: discrete unless its features are CONTINUOUS_ACTION, bounds from
        max_value / min_value."""
        import numpy as np

        from ..models.cem_planner import CEMPlannerNetwork
        from ..preprocessing.identify_types import CONTINUOUS_ACTION
        from ..preprocessing.normalization import get_num_output_features

        p = self.trainer_param
        world_model_manager = WorldModel(trainer_param=p.mdnrnn)
        world_model_manager.build_trainer(normalization_data_map, use_gpu=use_gpu,
                                          reward_options=reward_options)
        world_model_trainers = [
            world_model_manager.build_trainer(normalization_data_map, use_gpu=use_gpu,
                                              reward_options=reward_options)
            for _ in range(p.num_world_models)]
        world_model_nets = [t.memory_network for t in world_model_trainers]
        terminal_effective = p.mdnrnn.not_terminal_loss_weight > 0
        action_norm = normalization_data_map[NormalizationKey.ACTION].dense_normalization_parameters
        sorted_action_norm_vals = list(action_norm.values())
        discrete_action = sorted_action_norm_vals[0].feature_type != CONTINUOUS_ACTION
        upper = lower = None
        if not discrete_action:
            upper = np.array([v.max_value for v in sorted_action_norm_vals])
            lower = np.array([v.min_value for v in sorted_action_norm_vals])
        planner = CEMPlannerNetwork(
            mem_net_list=world_model_nets, cem_num_iterations=p.cem_num_iterations,
            cem_population_size=p.cem_population_size,
            ensemble_population_size=p.ensemble_population_size, num_elites=p.num_elites,
            plan_horizon_length=p.plan_horizon_length,
            state_dim=get_num_output_features(
                normalization_data_map[NormalizationKey.STATE].dense_normalization_parameters),
            action_dim=get_num_output_features(action_norm), discrete_action=discrete_action,
            terminal_effective=terminal_effective, gamma=p.rl.gamma, alpha=p.alpha,
            epsilon=p.epsilon, action_upper_bounds=upper, action_lower_bounds=lower)
        # kept for create_policy
        self.discrete_action = discrete_action
        return CEMTrainer(cem_planner_network=planner, world_model_trainers=world_model_trainers,
                          parameters=p)


@dataclass
class Seq2RewardModel:
    """reagent/model_managers/model_based/seq2reward_model.py: a Seq2RewardNetwork trained by
    Seq2RewardTrainer; `compress_net_builder` builds the policy network that
    CompressModelTrainer fits to its plan.  `reward_boost` is WorldModelBase's field (unused by
    this trainer)."""
    net_builder: Seq2RewardNetBuilder = field(default_factory=Seq2RewardNetBuilder)
    compress_net_builder: ValueFullyConnected = field(default_factory=ValueFullyConnected)
    trainer_param: Seq2RewardTrainerParameters = field(
        default_factory=Seq2RewardTrainerParameters)
    reward_boost: Optional[Dict[str, float]] = None

    def build_trainer(self, normalization_data_map: Dict[str, NormalizationData], use_gpu: bool,
                      reward_options=None) -> Seq2RewardTrainer:
        dev = _device(use_gpu)
        seq2reward_network = self.net_builder.build_value_network(
            normalization_data_map[NormalizationKey.STATE])
        trainer = Seq2RewardTrainer(seq2reward_network=seq2reward_network,
                                    params=self.trainer_param)
        return trainer.to(dev)


@dataclass
class SlateQ:
    """reagent/model_managers/ranking/slate_q.py and slate_q_base.py: a ParametricDQN
    FullyConnected q network over (state, item) from the STATE and ITEM normalizations, its
    target a copy, and SlateQTrainer with `trainer_param`.  slate_feature_id and slate_score_id
    are kept for the configurations that name them; the preprocessing options, the reporter and
    serving modules are out of scope."""
    slate_size: int = -1
    num_candidates: int = -1
    slate_feature_id: int = 0
    slate_score_id: Tuple[int, int] = (0, 0)
    trainer_param: SlateQTrainerParameters = field(default_factory=SlateQTrainerParameters)
    net_builder: ParametricFullyConnected = field(default_factory=ParametricFullyConnected)

    def __post_init__(self):
        assert self.slate_size > 0, f"Please set valid slate_size (currently {self.slate_size})"
        assert self.num_candidates > 0, (
            f"Please set valid num_candidates (currently {self.num_candidates})")
        self.eval_parameters = self.trainer_param.evaluation

    def build_trainer(self, normalization_data_map: Dict[str, NormalizationData], use_gpu: bool,
                      reward_options=None) -> SlateQTrainer:
        dev = _device(use_gpu)
        q_network = self.net_builder.build_q_network(
            normalization_data_map[NormalizationKey.STATE],
            normalization_data_map[NormalizationKey.ITEM]).to(dev)
        q_network_target = q_network.get_target_network()
        return SlateQTrainer(q_network=q_network, q_network_target=q_network_target,
                             slate_size=self.slate_size, **self.trainer_param.asdict()).to(dev)

    def create_policy(self, trainer_module, serving: bool = False, normalization_data_map=None):
        """slate_q_base.py:61-83: slate_q_scorer over every candidate, then the top slate_size."""
        if serving:
            raise NotImplementedError("serving modules are out of scope of reagent_b200")
        from ..gym.policies import Policy, TopKSampler, slate_q_scorer

        return Policy(scorer=slate_q_scorer(self.num_candidates, trainer_module.q_network),
                      sampler=TopKSampler(k=self.slate_size))
