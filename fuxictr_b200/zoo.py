"""Callers of the hot path: the five in-scope model forwards and one training step.

These are NOT a model-zoo rewrite.  On a machine that has the reference installed the
unmodified ``model_zoo`` classes call the patched layers (fuxictr_b200.patch.enable()).
The GPU box has no reference checkout, so parity tests and bench.py need the same
callers in-tree: each class below wires the layers exactly like the reference class of
the same name (same attribute names => same state_dict keys, same construction order =>
same RNG consumption) and nothing else.

  DeepFM   model_zoo/DeepFM/DeepFM_torch/src/DeepFM.py:41-88
  DCNv2    model_zoo/DCNv2/src/DCNv2.py:47-132
  DLRM     model_zoo/DLRM/src/DLRM.py:43-123
  DIN      model_zoo/DIN/src/DIN.py:50-149
  xDeepFM  model_zoo/xDeepFM/src/xDeepFM.py:41-97
  RankModel = the slice of BaseModel a training step touches,
             fuxictr/pytorch/models/rank_model.py:84-189, 307-323, 435-448
"""
import torch
from torch import nn

from .layers import (fused_front, FeatureEmbedding, FeatureEmbeddingDict, MLP_Block, FactorizationMachine,
                     CrossNetV2, InnerProductInteraction, DIN_Attention, Dice,
                     CompressedInteractionNet, LogisticRegression, not_in_whitelist)
from .arena import ParamArena, FusedAdam
from . import functional as F2


def _flatten(items):
    for x in items:
        if isinstance(x, (list, tuple)):
            for y in _flatten(x):
                yield y
        else:
            yield x


class RankModel(nn.Module):
    """The slice of BaseModel a training step touches: device placement, input/label extraction, loss,
    regularisation and one optimisation step (rank_model.py:84-189, 307-323)."""

    _LOSSES = ("bce", "binary_crossentropy", "binary_cross_entropy")

    def __init__(self, feature_map, model_id="RankModel", task="binary_classification", gpu=-1,
                 embedding_regularizer=None, net_regularizer=None, **kwargs):
        super(RankModel, self).__init__()
        on_gpu = gpu >= 0 and torch.cuda.is_available()
        self.device = torch.device("cuda:%d" % gpu if on_gpu else "cpu")
        self.feature_map, self.model_id = feature_map, model_id
        self._embedding_regularizer, self._net_regularizer = embedding_regularizer, net_regularizer
        self._max_gradient_norm = 10.0
        heads = {"binary_classification": nn.Sigmoid, "regression": nn.Identity}
        if task not in heads:
            raise NotImplementedError("task={} is not supported.".format(task))
        self.output_activation = heads[task]()
        self._arena = None
        self._fused_optimizer = None

    def _finish(self, kwargs, learning_rate):
        """Tail of every reference model constructor: compile (the optimizer is built over the CPU
        parameters), THEN re-initialise, THEN move — this order fixes RNG consumption and keeps the
        optimizer's Parameter objects valid (rank_model.py:92, 146-167; DeepFM.py:69-71)."""
        self.compile(kwargs.get("optimizer", "adam"), kwargs.get("loss", "binary_crossentropy"), learning_rate)
        self.reset_parameters()
        self.model_to_device()

    def compile(self, optimizer="adam", loss="binary_crossentropy", lr=1e-3):
        self._lr = lr
        self._optimizer_name = "Adam" if str(optimizer).lower() == "adam" else optimizer
        self.optimizer = getattr(torch.optim, self._optimizer_name)(self.parameters(), lr=lr)
        if loss not in self._LOSSES:
            raise NotImplementedError("loss={} is not supported on the H100 path.".format(loss))
        self.loss_fn = torch.nn.functional.binary_cross_entropy

    def reset_parameters(self):
        """Two passes in module order: xavier-normal weights / zero biases for modules that are EXACTLY
        nn.Linear or nn.Conv1d, then every module's own `init_weights` (rank_model.py:146-167)."""
        for m in self.modules():
            if type(m) in (nn.Linear, nn.Conv1d):
                nn.init.xavier_normal_(m.weight)
                if m.bias is not None:
                    m.bias.data.fill_(0)
        for m in self.modules():
            if hasattr(m, "init_weights"):
                m.init_weights()

    def model_to_device(self):
        self.to(device=self.device)

    def get_inputs(self, inputs, feature_source=None):
        """Every non-label, non-meta column the caller passed (optionally filtered by source), moved to
        the model's device (rank_model.py:169-189)."""
        specs, labels = self.feature_map.features, self.feature_map.labels
        X = dict()
        for name, column in inputs.items():
            if name in labels or specs[name]["type"] == "meta":
                continue
            if feature_source and not_in_whitelist(specs[name]["source"], feature_source):
                continue
            X[name] = column.to(self.device)
        return X

    def get_labels(self, inputs):
        y = inputs[self.feature_map.labels[0]].to(self.device)
        return y.float().view(-1, 1)

    def regularization_loss(self):
        """Sum of (lambda / p) * ||param||_p^p: embedding regulariser on the parameters of modules whose
        type is EXACTLY FeatureEmbeddingDict, net regulariser on everything else (rank_model.py:95-118)."""
        if not (self._embedding_regularizer or self._net_regularizer):
            return 0
        emb_terms = _parse_regularizer(self._embedding_regularizer)
        net_terms = _parse_regularizer(self._net_regularizer)
        total, emb_names = 0, set()
        for mod_name, module in self.named_modules():
            if type(module) != FeatureEmbeddingDict:
                continue
            for p_name, param in module.named_parameters():
                if param.requires_grad:
                    emb_names.add(mod_name + "." + p_name)
                    for p, lam in emb_terms:
                        total = total + (lam / p) * torch.norm(param, p) ** p
        for name, param in self.named_parameters():
            if param.requires_grad and name not in emb_names:
                for p, lam in net_terms:
                    total = total + (lam / p) * torch.norm(param, p) ** p
        return total

    def compute_loss(self, return_dict, y_true):
        return self.loss_fn(return_dict["y_pred"], y_true, reduction="mean") + self.regularization_loss()

    def train_step(self, batch_data):
        """rank_model.py:307-323 with torch's own optimizer (the parity path of the tests)."""
        self.optimizer.zero_grad()
        loss = self.compute_loss(self.forward(batch_data), self.get_labels(batch_data))
        loss.backward()
        nn.utils.clip_grad_norm_(self.parameters(), self._max_gradient_norm)
        self.optimizer.step()
        return loss

    # -- rank_model.py:350-398, device-resident (SURVEY.md 8f row 3) ---------------------------
    def evaluate(self, data_generator, metrics=None):
        """Same contract as BaseModel.evaluate; predictions and labels stay in HBM (no per-batch
        `.cpu().numpy()`), logloss / AUC come from csrc/metrics.cu, one small D2H at the end."""
        from .metrics import evaluate_generator
        self.materialize_tables()
        names = metrics if metrics is not None else getattr(self, "validation_metrics", ["logloss", "AUC"])
        return evaluate_generator(self, data_generator, names)

    def predict(self, data_generator):
        """BaseModel.predict: flattened float64 numpy array; one D2H for the whole generator."""
        from .metrics import predict_generator
        self.materialize_tables()
        return predict_generator(self, data_generator)

    # -- H100 extension: flat arenas + 2-kernel clip/Adam -------------------------------------
    def enable_sharding(self, group, batch_local, matrix_width, idx_dtype=torch.float64, want_fm=True):
        """Row-shard every embedding / LR table over `group` (fuxictr_b200.sharded) and route the
        sparse front through the peer-memory push/pull kernels.  Call after model_to_device() and
        before use_fused_optimizer().  Only models whose forward consumes `self._sharded_front`
        (DeepFM, DLRM) may be sharded: any other forward would keep reading the 1/world row shards
        with global ids."""
        from . import sharded as SH
        if not getattr(type(self), "_routes_sharded_front", False):
            raise NotImplementedError("%s does not route its lookups through the sharded front; row-sharding "
                                      "is implemented for DeepFM and DLRM" % type(self).__name__)
        fed = self.embedding_layer.embedding_layer
        lr_layer = self.fm.lr_layer if hasattr(self, "fm") else getattr(self, "lr_layer", None)
        names = [f for f in self.feature_map.features.keys() if f in fed.embedding_layers]
        if not all(fed._is_fusable(f) and self.feature_map.features[f]["type"] == "categorical" for f in names):
            raise NotImplementedError("sharded front needs categorical features only")
        lfed = lr_layer.embedding_layer.embedding_layer if lr_layer is not None else None
        vocabs, cols, pads, etabs, ltabs = [], [], [], [], []
        with torch.no_grad():
            for f in names:
                emb = fed.embedding_layers[f]
                vocabs.append(emb.num_embeddings)
                cols.append(self.feature_map.get_column_index(f))
                pads.append(emb.padding_idx)
                if not getattr(emb, "_b2_sharded", False):
                    emb.weight.data = SH.shard_rows(emb.weight.data, group.rank, group.world)
                    emb._b2_sharded = True
                etabs.append(emb.weight)
                if lfed is not None:
                    lemb = lfed.embedding_layers[f]
                    if not getattr(lemb, "_b2_sharded", False):
                        lemb.weight.data = SH.shard_rows(lemb.weight.data, group.rank, group.world)
                        lemb._b2_sharded = True
                    ltabs.append(lemb.weight)
        dim = fed.embedding_layers[names[0]].embedding_dim
        self._sharded_front = SH.ShardedFront(group, names, etabs, ltabs or None, vocabs, cols, pads, dim,
                                              batch_local, matrix_width, idx_dtype,
                                              bias=(lr_layer.bias if lr_layer is not None else None),
                                              want_fm=want_fm)
        self._sharded_params = etabs + ltabs
        # fused_train_step seeds backward() with 1/world, so every gradient (dense and rows) is born
        # divided by the world size: the pull and the dense all-reduce then need no scaling pass
        self._sharded_front.pull_scale = 1.0
        self._loss_grad = torch.full((), 1.0 / group.world, dtype=torch.float32, device=self.device)
        return self._sharded_front

    def _batch_matrix(self, inputs):
        """The (B, W) matrix the collator sliced `inputs` from, rebuilt from one column view's
        storage offset and row stride (the views' `_base` may be a larger tensor)."""
        name = next(iter(self.feature_map.features.keys()))
        v = inputs[name]
        col = self.feature_map.get_column_index(name)
        width = self.feature_map.input_length + len(self.feature_map.labels)
        if v.dim() != 1 or v.stride(0) < width or v.storage_offset() < col:
            raise RuntimeError("sharded front needs the batch dict to be column views of one matrix")
        mat = v.as_strided((v.shape[0], width), (v.stride(0), 1), v.storage_offset() - col)
        return mat.to(self.device)

    def _front_tables(self):
        """Embedding + LR tables read ONLY through the fused front kernels (lazy-Adam candidates)."""
        fed = self.embedding_layer.embedding_layer
        lr_layer = self.fm.lr_layer if hasattr(self, "fm") else getattr(self, "lr_layer", None)
        tabs, seen = [], set()
        for mod in ([fed] + ([lr_layer.embedding_layer.embedding_layer] if lr_layer is not None else [])):
            for f in mod._feature_map.features.keys():
                if f in mod.embedding_layers and type(mod.embedding_layers[f]) == nn.Embedding:
                    w = mod.embedding_layers[f].weight
                    if id(w) not in seen:
                        seen.add(id(w))
                        tabs.append(w)
        return tabs

    def use_fused_optimizer(self, lazy_tables=False):
        """Re-home parameters into one HBM arena and replace clip_grad_norm_ + torch Adam by
        the two-kernel FusedAdam (same arithmetic; see arena.py).  Call after model_to_device().
        lazy_tables=True (models whose tables are read only by the fused front: DeepFM, xDeepFM):
        the dense Adam semantics of the tables are evaluated row-wise and lazily — bit-identical
        results, O(batch) instead of O(vocabulary) optimizer traffic; call materialize_tables()
        before reading table weights outside the kernels (state_dict, evaluation on other paths)."""
        if self._optimizer_name != "Adam":
            raise NotImplementedError("the fused optimizer implements Adam only")
        if lazy_tables:
            if getattr(self, "_sharded_params", None):
                raise NotImplementedError("lazy tables and row-sharding are not combined yet")
            first = self._front_tables()
            self._arena = ParamArena(self, first=first)
            self._fused_optimizer = FusedAdam(self._arena, lr=self._lr, max_norm=self._max_gradient_norm)
            self._lazy = self._fused_optimizer.enable_lazy(first)
            self.optimizer = None
            return self._fused_optimizer
        # tables first (the row shards of a sharded run, else every nn.Embedding weight): the dense
        # parameters then form one contiguous tail (one all-reduce, one 3xTF32 split launch per step)
        first = getattr(self, "_sharded_params", None)
        if not first:
            first, seen = [], set()
            for m in self.modules():
                if type(m) == nn.Embedding and id(m.weight) not in seen and m.weight.requires_grad:
                    seen.add(id(m.weight))
                    first.append(m.weight)
        self._arena = ParamArena(self, first=first)
        self._fused_optimizer = FusedAdam(self._arena, lr=self._lr, max_norm=self._max_gradient_norm)
        self._fused_optimizer.sharded = bool(getattr(self, "_sharded_params", None))
        self._fused_optimizer.dense_prescaled = getattr(self, "_loss_grad", None) is not None
        front = getattr(self, "_sharded_front", None)
        if front is not None and front.group.world > 1 and hasattr(front.group, "group"):
            # real ranks (not the single-process virtual harness): overlap the dense all-reduce with the pull
            self._fused_optimizer.enable_dense_overlap()
            front.on_dense_grads_ready = self._fused_optimizer.start_dense_allreduce
        self.optimizer = None
        return self._fused_optimizer

    def materialize_tables(self):
        if getattr(self, "_lazy", None) is not None:
            self._lazy.materialize()

    def state_dict(self, *args, **kwargs):
        """Checkpoints must see up-to-date rows and moments: bring lazily evaluated tables current first."""
        self.materialize_tables()
        return super(RankModel, self).state_dict(*args, **kwargs)

    def fused_train_step(self, batch_data):
        """train_step with the arena optimizer and the fused logit+BCE kernel when the model
        exposes its pre-sigmoid logit terms (`forward_logits`)."""
        opt = self._fused_optimizer
        opt.zero_grad()
        y_true = self.get_labels(batch_data)
        if hasattr(self, "forward_logits") and not (self._embedding_regularizer or self._net_regularizer):
            loss, _ = F2.logit_bce(y_true, *self.forward_logits(batch_data))
        else:
            loss = self.compute_loss(self.forward(batch_data), y_true)
        seed = getattr(self, "_loss_grad", None)      # 1/world for row-sharded runs (see enable_sharding)
        if seed is not None:
            loss.backward(seed)
        else:
            loss.backward()
        opt.step()
        return loss


def _parse_regularizer(reg):
    """torch_utils.py:104-135: float => L2; 'l1(x)', 'l2(x)', 'l1_l2(x,y)'."""
    pairs = []
    if isinstance(reg, float):
        pairs.append((2, reg))
    elif isinstance(reg, str):
        body = reg.rstrip(")").split("(")[-1]
        if reg.startswith("l1(") or reg.startswith("l2("):
            pairs.append((int(reg[1]), float(body)))
        elif reg.startswith("l1_l2"):
            l1, l2 = body.split(",")
            pairs += [(1, float(l1)), (2, float(l2))]
        else:
            raise NotImplementedError("regularizer={} is not supported.".format(reg))
    return pairs


class DeepFM(RankModel):
    """model_zoo/DeepFM/DeepFM_torch/src/DeepFM.py:41-88: y = sigmoid(FM(X, E) + MLP(flatten(E)))."""
    _routes_sharded_front = True

    def __init__(self, feature_map, model_id="DeepFM", gpu=-1, learning_rate=1e-3, embedding_dim=10,
                 hidden_units=[64, 64, 64], hidden_activations="ReLU", net_dropout=0, batch_norm=False,
                 embedding_regularizer=None, net_regularizer=None, **kwargs):
        super(DeepFM, self).__init__(feature_map, model_id=model_id, gpu=gpu,
                                     embedding_regularizer=embedding_regularizer, net_regularizer=net_regularizer,
                                     **kwargs)
        self.embedding_layer = FeatureEmbedding(feature_map, embedding_dim)
        self.fm = FactorizationMachine(feature_map)
        self.mlp = MLP_Block(feature_map.sum_emb_out_dim(), hidden_units=hidden_units,
                             hidden_activations=hidden_activations, output_dim=1, output_activation=None,
                             dropout_rates=net_dropout, batch_norm=batch_norm)
        self._finish(kwargs, learning_rate)

    def forward_logits(self, inputs):
        if getattr(self, "_sharded_front", None) is not None:   # row-sharded tables, P2P push/pull
            from .sharded import sharded_front
            feature_emb, fm_lr = sharded_front(self._sharded_front, self._batch_matrix(inputs))
            return (fm_lr, self.mlp(feature_emb.flatten(start_dim=1)))
        X = self.get_inputs(inputs)
        fused = fused_front(self.embedding_layer, self.fm.lr_layer, X, want_fm=True)
        if fused is not None:     # gather + FM + LR in one launch
            feature_emb, fm_lr = fused
            return (fm_lr, self.mlp(feature_emb.flatten(start_dim=1)))
        if getattr(self, "_lazy", None) is not None:
            raise RuntimeError("lazy tables are only readable through the fused front (unsupported config)")
        feature_emb = self.embedding_layer(X)
        return (self.fm.fm_layer(feature_emb), self.fm.lr_layer(X),
                self.mlp(feature_emb.flatten(start_dim=1)))

    def forward(self, inputs):
        terms = self.forward_logits(inputs)
        y_pred = terms[0]
        for t in terms[1:]:
            y_pred = y_pred + t
        return {"y_pred": self.output_activation(y_pred)}


class DCNv2(RankModel):
    """model_zoo/DCNv2/src/DCNv2.py:47-132: CrossNetV2 and DNN towers combined per `model_structure`
    (crossnet_only | stacked | parallel | stacked_parallel), one Linear to the logit."""
    _STRUCTURES = ("crossnet_only", "stacked", "parallel", "stacked_parallel")

    def __init__(self, feature_map, model_id="DCNv2", gpu=-1, model_structure="parallel",
                 use_low_rank_mixture=False, low_rank=32, num_experts=4, learning_rate=1e-3,
                 embedding_dim=10, stacked_dnn_hidden_units=[], parallel_dnn_hidden_units=[],
                 dnn_activations="ReLU", num_cross_layers=3, net_dropout=0, batch_norm=False,
                 embedding_regularizer=None, net_regularizer=None, **kwargs):
        super(DCNv2, self).__init__(feature_map, model_id=model_id, gpu=gpu,
                                    embedding_regularizer=embedding_regularizer, net_regularizer=net_regularizer,
                                    **kwargs)
        if use_low_rank_mixture:
            raise NotImplementedError("CrossNetMix is outside the H100 hot path (SURVEY.md section 2 row 6)")
        if model_structure not in self._STRUCTURES:
            raise AssertionError("model_structure={} not supported!".format(model_structure))
        self.model_structure = model_structure
        has_stacked = model_structure in ("stacked", "stacked_parallel")
        has_parallel = model_structure in ("parallel", "stacked_parallel")
        self.embedding_layer = FeatureEmbedding(feature_map, embedding_dim)
        width = feature_map.sum_emb_out_dim()
        self.crossnet = CrossNetV2(width, num_cross_layers)

        def tower(units):
            return MLP_Block(width, hidden_units=units, hidden_activations=dnn_activations, output_dim=None,
                             output_activation=None, dropout_rates=net_dropout, batch_norm=batch_norm)
        left = width                                    # what the cross (or stacked) branch hands to fc
        if has_stacked:
            self.stacked_dnn = tower(stacked_dnn_hidden_units)
            left = stacked_dnn_hidden_units[-1]
        right = 0
        if has_parallel:
            self.parallel_dnn = tower(parallel_dnn_hidden_units)
            right = parallel_dnn_hidden_units[-1]
        self.fc = nn.Linear(left + right, 1)
        self._finish(kwargs, learning_rate)

    def _final_out(self, inputs):
        """DCNv2.py:108-128: what the last Linear sees for each model_structure."""
        emb = self.embedding_layer(self.get_inputs(inputs), flatten_emb=True)
        cross = self.crossnet(emb)
        left = self.stacked_dnn(cross) if hasattr(self, "stacked_dnn") else cross
        if not hasattr(self, "parallel_dnn"):
            return left
        return torch.cat([left, self.parallel_dnn(emb)], dim=-1)

    def forward_logits(self, inputs):
        final_out = self._final_out(inputs)
        return (F2.linear_act(final_out, self.fc.weight, self.fc.bias),)

    def forward(self, inputs):
        y_pred = F2.linear_act(self._final_out(inputs), self.fc.weight, self.fc.bias)
        return {"y_pred": self.output_activation(y_pred)}


class DLRM(RankModel):
    """model_zoo/DLRM/src/DLRM.py:43-123: embeddings of the non-numeric fields (+ a bottom MLP over the
    numeric ones as one more "field"), pairwise dot (or concat) interaction, top MLP with the output
    activation inside it."""
    _routes_sharded_front = True

    def __init__(self, feature_map, model_id="DLRM", gpu=-1, learning_rate=1e-3, embedding_dim=10,
                 top_mlp_units=[64, 64, 64], bottom_mlp_units=[64, 64, 64], top_mlp_activations="ReLU",
                 bottom_mlp_activations="ReLU", top_mlp_dropout=0, bottom_mlp_dropout=0,
                 interaction_op="dot", batch_norm=False, embedding_regularizer=None,
                 net_regularizer=None, **kwargs):
        super(DLRM, self).__init__(feature_map, model_id=model_id, gpu=gpu,
                                   embedding_regularizer=embedding_regularizer, net_regularizer=net_regularizer,
                                   **kwargs)
        self.dense_feats = [name for name, spec in feature_map.features.items() if spec["type"] == "numeric"]
        has_dense = len(self.dense_feats) > 0
        self.embedding_layer = FeatureEmbedding(feature_map, embedding_dim,
                                                not_required_feature_columns=self.dense_feats)
        n_fields = feature_map.num_fields - len(self.dense_feats) + int(has_dense)
        if has_dense:
            self.bottom_mlp = MLP_Block(len(self.dense_feats), hidden_units=bottom_mlp_units,
                                        hidden_activations=bottom_mlp_activations, output_dim=embedding_dim,
                                        output_activation=bottom_mlp_activations,
                                        dropout_rates=bottom_mlp_dropout, batch_norm=batch_norm)
        self.interaction_op = interaction_op
        if interaction_op == "dot":
            self.interact = InnerProductInteraction(num_fields=n_fields, output="inner_product")
            top_in = n_fields * (n_fields - 1) // 2 + (embedding_dim if has_dense else 0)
        elif interaction_op == "cat":
            self.interact = nn.Flatten(start_dim=1)
            top_in = n_fields * embedding_dim
        else:
            raise ValueError("interaction_op={} not supported.".format(interaction_op))
        self.top_mlp = MLP_Block(top_in, hidden_units=top_mlp_units, hidden_activations=top_mlp_activations,
                                 output_dim=1, output_activation=self.output_activation,
                                 dropout_rates=top_mlp_dropout, batch_norm=batch_norm)
        self._finish(kwargs, learning_rate)

    def forward(self, inputs):
        X = self.get_inputs(inputs)
        if getattr(self, "_sharded_front", None) is not None:   # row-sharded tables (SURVEY.md 8e, C5)
            from .sharded import sharded_front
            feat_emb, _ = sharded_front(self._sharded_front, self._batch_matrix(inputs))
        else:
            feat_emb = self.embedding_layer(X)
        dense_emb = None
        if self.dense_feats:        # numeric columns -> bottom MLP -> one more interaction "field" (DLRM.py:114-118)
            dense_emb = self.bottom_mlp(torch.cat([X[name] for name in self.dense_feats], dim=-1))
            feat_emb = torch.cat([feat_emb, dense_emb.unsqueeze(1)], dim=1)
        z = self.interact(feat_emb)
        if dense_emb is not None and self.interaction_op == "dot":
            z = torch.cat([z, dense_emb], dim=-1)
        return {"y_pred": self.top_mlp(z)}


class DIN(RankModel):
    """model_zoo/DIN/src/DIN.py:50-149: one DIN_Attention per (target, sequence) field pair (tuples of
    fields are concatenated), pooled sequences replace the raw ones, one DNN over all embeddings."""

    def __init__(self, feature_map, model_id="DIN", gpu=-1, dnn_hidden_units=[512, 128, 64],
                 dnn_activations="ReLU", attention_hidden_units=[64], attention_hidden_activations="Dice",
                 attention_output_activation=None, attention_dropout=0, learning_rate=1e-3,
                 embedding_dim=10, net_dropout=0, batch_norm=False,
                 din_target_field=[("item_id", "cate_id")],
                 din_sequence_field=[("click_history", "cate_history")], din_use_softmax=False,
                 embedding_regularizer=None, net_regularizer=None, **kwargs):
        super(DIN, self).__init__(feature_map, model_id=model_id, gpu=gpu,
                                  embedding_regularizer=embedding_regularizer, net_regularizer=net_regularizer,
                                  **kwargs)
        as_list = lambda v: v if isinstance(v, list) else [v]                   # noqa: E731
        self.din_target_field, self.din_sequence_field = as_list(din_target_field), as_list(din_sequence_field)
        assert len(self.din_target_field) == len(self.din_sequence_field), \
            "len(din_target_field) != len(din_sequence_field)"
        if isinstance(dnn_activations, str) and dnn_activations.lower() == "dice":
            dnn_activations = [Dice(width) for width in dnn_hidden_units]
        self.embedding_dim = embedding_dim
        self.embedding_layer = FeatureEmbeddingDict(feature_map, embedding_dim)
        heads = []
        for target in self.din_target_field:
            parts = len(target) if type(target) == tuple else 1
            heads.append(DIN_Attention(embedding_dim * parts, attention_units=attention_hidden_units,
                                       hidden_activations=attention_hidden_activations,
                                       output_activation=attention_output_activation,
                                       dropout_rate=attention_dropout, use_softmax=din_use_softmax))
        self.attention_layers = nn.ModuleList(heads)
        self.dnn = MLP_Block(feature_map.sum_emb_out_dim(), hidden_units=dnn_hidden_units,
                             hidden_activations=dnn_activations, output_dim=1,
                             output_activation=self.output_activation, dropout_rates=net_dropout,
                             batch_norm=batch_norm)
        self._finish(kwargs, learning_rate)

    def get_embedding(self, field, feature_emb_dict):
        """A tuple of fields means their embeddings side by side (DIN.py:144-149)."""
        names = field if type(field) == tuple else (field,)
        parts = [feature_emb_dict[name] for name in names]
        return parts[0] if len(parts) == 1 else torch.cat(parts, dim=-1)

    def forward(self, inputs):
        """DIN.py:109-142: attention-pool every sequence group against its target, write the pooled
        vectors back under the sequence names, then one DNN over all embeddings in FeatureMap order."""
        X = self.get_inputs(inputs)
        emb = self.embedding_layer(X)
        for head, target, sequence in zip(self.attention_layers, self.din_target_field, self.din_sequence_field):
            seq_names = list(_flatten([sequence]))
            valid = X[seq_names[0]].long() != 0            # padding id 0 marks the empty history slots
            pooled = head(self.get_embedding(target, emb), self.get_embedding(sequence, emb), valid)
            for name, piece in zip(seq_names, pooled.split(self.embedding_dim, dim=-1)):
                emb[name] = piece
        return {"y_pred": self.dnn(self.embedding_layer.dict2tensor(emb, flatten_emb=True))}


class xDeepFM(RankModel):
    """model_zoo/xDeepFM/src/xDeepFM.py:41-97: y = sigmoid(LR(X) + CIN(E) [+ DNN(flatten(E))])."""

    def __init__(self, feature_map, model_id="xDeepFM", gpu=-1, learning_rate=1e-3, embedding_dim=10,
                 dnn_hidden_units=[64, 64, 64], dnn_activations="ReLU", cin_hidden_units=[16, 16, 16],
                 net_dropout=0, batch_norm=False, embedding_regularizer=None, net_regularizer=None,
                 **kwargs):
        super(xDeepFM, self).__init__(feature_map, model_id=model_id, gpu=gpu,
                                      embedding_regularizer=embedding_regularizer, net_regularizer=net_regularizer,
                                      **kwargs)
        self.embedding_layer = FeatureEmbedding(feature_map, embedding_dim)
        self.dnn = None
        if dnn_hidden_units:
            self.dnn = MLP_Block(feature_map.sum_emb_out_dim(), hidden_units=dnn_hidden_units,
                                 hidden_activations=dnn_activations, output_dim=1, output_activation=None,
                                 dropout_rates=net_dropout, batch_norm=batch_norm)
        self.lr_layer = LogisticRegression(feature_map, use_bias=False)
        self.cin = CompressedInteractionNet(feature_map.num_fields, cin_hidden_units, output_dim=1)
        self._finish(kwargs, learning_rate)

    def forward_logits(self, inputs):
        X = self.get_inputs(inputs)
        fused = fused_front(self.embedding_layer, self.lr_layer, X, want_fm=False)
        if fused is not None:     # gather + LR in one launch
            feature_emb, lr_logit = fused
            terms = [lr_logit, self.cin(feature_emb)]
        else:
            if getattr(self, "_lazy", None) is not None:
                raise RuntimeError("lazy tables are only readable through the fused front (unsupported config)")
            feature_emb = self.embedding_layer(X)
            terms = [self.lr_layer(X), self.cin(feature_emb)]
        if self.dnn is not None:
            terms.append(self.dnn(feature_emb.flatten(start_dim=1)))
        return tuple(terms)

    def forward(self, inputs):
        terms = self.forward_logits(inputs)
        y_pred = terms[0] + terms[1]
        if len(terms) > 2:
            y_pred = y_pred + terms[2]
        return {"y_pred": self.output_activation(y_pred)}
