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
  GDCN, GDCNP  model_zoo/GDCN/src/GDCN.py
  FinalMLP     model_zoo/FinalMLP/src/FinalMLP.py
  DualMLP      model_zoo/FinalMLP/src/DualMLP.py
  MaskNet      model_zoo/MaskNet/src/MaskNet.py
  AutoInt      model_zoo/AutoInt/src/AutoInt.py
  WuKong       model_zoo/WuKong/src/WuKong.py
  FinalNet     model_zoo/FinalNet/src/FinalNet.py
  BST          model_zoo/BST/src/BST.py
  DIEN         model_zoo/DIEN/src/DIEN.py
  TransAct     model_zoo/TransAct/src/TransAct.py
  ETA, SDIM    model_zoo/LongCTR/ETA/ETA.py, model_zoo/LongCTR/SDIM/SDIM.py
  MIRRN        model_zoo/LongCTR/MIRRN/MIRRN.py
  SIM, TWIN    model_zoo/LongCTR/SIM/SIM.py, model_zoo/LongCTR/TWIN/TWIN.py
  RankModel = the slice of BaseModel a training step touches,
             fuxictr/pytorch/models/rank_model.py:84-189, 307-323, 435-448
"""
from collections import OrderedDict

import torch
from torch import nn

from .layers import (fused_front, front_plan, FeatureEmbedding, FeatureEmbeddingDict, MLP_Block, FactorizationMachine,
                     CrossNetV2, GateCorssLayer, FeatureSelection, InteractionAggregation, InnerProductInteraction,
                     SerialMaskNet, ParallelMaskNet, MultiHeadSelfAttention, WuKongLayer, wukong_stack,
                     FeatureGating, FinalBlock, BehaviorTransformer, DynamicGRU, AttentionLayer, MaskedSumPooling,
                     DIN_Attention, Dice, CompressedInteractionNet, LogisticRegression, MultiHeadTargetAttention,
                     MultiHeadTopKAttention, TransActTransformer, FilterLayer2, not_in_whitelist)
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
        `.cpu().numpy()`), logloss / AUC come from csrc/metrics.cu, one small D2H at the end.
        After enable_sharding() this is a collective call: every rank feeds its own shard of the split (generators
        of equal len(), batches of at most batch_local rows) and gets the metrics over the union of all ranks'
        rows, the same on every rank (fuxictr_b200.sharded.evaluate_sharded)."""
        from .metrics import evaluate_generator
        self.materialize_tables()
        names = metrics if metrics is not None else getattr(self, "validation_metrics", ["logloss", "AUC"])
        if getattr(self, "_sharded_front", None) is not None:
            from .sharded import evaluate_sharded
            return evaluate_sharded(self, data_generator, names)
        return evaluate_generator(self, data_generator, names)

    def predict(self, data_generator):
        """BaseModel.predict: flattened float64 numpy array; one D2H for the whole generator.  After
        enable_sharding(): a collective call that returns THIS rank's predictions, in its generator's order
        (the data-parallel meaning; fuxictr_b200.sharded.predict_sharded)."""
        from .metrics import predict_generator
        self.materialize_tables()
        if getattr(self, "_sharded_front", None) is not None:
            from .sharded import predict_sharded
            return predict_sharded(self, data_generator)
        return predict_generator(self, data_generator)

    # -- H100 extension: flat arenas + 2-kernel clip/Adam -------------------------------------
    def enable_sharding(self, group, batch_local, matrix_width, idx_dtype=torch.float64, want_fm=True):
        """Row-shard every embedding / LR table over `group` (fuxictr_b200.sharded) and route the
        sparse front through the peer-memory push/pull kernels.  Call after model_to_device() and
        before use_fused_optimizer().  Only models whose forward consumes `self._sharded_front`
        (DeepFM, DLRM, DCNv2, xDeepFM, DIN, GDCN, GDCNP, FinalMLP, DualMLP, MaskNet, AutoInt, WuKong, FinalNet, BST, DIEN)
        may be
        sharded: any
        other forward would keep reading the 1/world row shards with global ids.  Features: categorical, and unpooled sequences (DIN's histories;
        a table shared by several fields is sharded once), one common embedding dim; an LR term needs
        categorical features only.  Anything else is refused before a table is touched."""
        from . import sharded as SH
        if not getattr(type(self), "_routes_sharded_front", False):
            raise NotImplementedError("%s does not route its lookups through the sharded front; row-sharding "
                                      "is implemented for DeepFM, DLRM, DCNv2, xDeepFM, DIN, GDCN, GDCNP, FinalMLP, "
                                      "DualMLP, MaskNet, AutoInt, WuKong, FinalNet, BST and DIEN" % type(self).__name__)
        fed = self.embedding_layer
        if not isinstance(fed, FeatureEmbeddingDict):       # FeatureEmbedding wraps it; DIN holds it directly
            fed = fed.embedding_layer
        lr_layer = self.fm.lr_layer if hasattr(self, "fm") else getattr(self, "lr_layer", None)
        specs = self.feature_map.features
        names = [f for f in specs.keys() if f in fed.embedding_layers]
        for f in names:
            kind = specs[f]["type"]
            if kind not in ("categorical", "sequence") or type(fed.embedding_layers[f]) != nn.Embedding:
                raise NotImplementedError("sharded front needs categorical or sequence features (%s is %s)"
                                          % (f, kind))
            if f in fed.feature_encoders:
                raise NotImplementedError("sharded front: feature %s has an encoder (a pooled sequence's rows come "
                                          "from several owners)" % f)
        dims = set(fed.embedding_layers[f].embedding_dim for f in names)
        if len(dims) != 1:
            raise NotImplementedError("sharded front needs one common embedding dim (got %s)" % sorted(dims))
        seq_lens = [int(specs[f]["max_len"]) if specs[f]["type"] == "sequence" else 1 for f in names]
        if (lr_layer is not None or want_fm) and any(n != 1 for n in seq_lens):
            raise NotImplementedError("sharded front: an LR or FM term over sequence features is not supported")
        lfed = lr_layer.embedding_layer.embedding_layer if lr_layer is not None else None
        if lfed is not None and not all(f in lfed.embedding_layers and type(lfed.embedding_layers[f]) == nn.Embedding
                                        and f not in lfed.feature_encoders for f in names):
            raise NotImplementedError("sharded front: the LR term needs one plain table per feature")
        dim = dims.pop()
        SH.owned_capacity(group.world, batch_local, seq_lens)       # the int32 bound, before any allocation
        vocabs, cols, pads, etabs, ltabs = [], [], [], [], []
        with torch.no_grad():
            for f in names:
                emb = fed.embedding_layers[f]
                vocabs.append(emb.num_embeddings)
                col = self.feature_map.get_column_index(f)
                cols.append(col[0] if isinstance(col, list) else col)    # a sequence's columns are consecutive
                pads.append(emb.padding_idx)
                if not getattr(emb, "_b2_sharded", False):     # a shared table: sharded once, listed per field
                    emb.weight.data = SH.shard_rows(emb.weight.data, group.rank, group.world)
                    emb._b2_sharded = True
                etabs.append(emb.weight)
                if lfed is not None:
                    lemb = lfed.embedding_layers[f]
                    if not getattr(lemb, "_b2_sharded", False):
                        lemb.weight.data = SH.shard_rows(lemb.weight.data, group.rank, group.world)
                        lemb._b2_sharded = True
                    ltabs.append(lemb.weight)
        self._sharded_front = SH.ShardedFront(group, names, etabs, ltabs or None, vocabs, cols, pads, dim,
                                              batch_local, matrix_width, idx_dtype,
                                              bias=(lr_layer.bias if lr_layer is not None else None),
                                              want_fm=want_fm, seq_lens=seq_lens)
        self._sharded_params = list(self._sharded_front.distinct_tables())
        # fused_train_step seeds backward() with 1/world, so every gradient (dense and rows) is born
        # divided by the world size: the pull and the dense all-reduce then need no scaling pass
        self._sharded_front.pull_scale = 1.0
        self._loss_grad = torch.full((), 1.0 / group.world, dtype=torch.float32, device=self.device)
        return self._sharded_front

    def _batch_matrix(self, inputs):
        """The (B, W) matrix the collator sliced `inputs` from, rebuilt from one column view's
        storage offset and row stride (the views' `_base` may be a larger tensor)."""
        width = self.feature_map.input_length + len(self.feature_map.labels)
        for name in list(self.feature_map.features.keys()) + list(self.feature_map.labels):
            v = inputs.get(name)
            col = self.feature_map.get_column_index(name)
            if isinstance(col, list):   # a sequence: a column-range view (batch_views), or a copy (batch_dict)
                col = col[0]
                if v is None or v.dim() != 2 or v.stride(1) != 1:
                    continue
            elif v is None or v.dim() != 1:
                continue
            if v.stride(0) < width or v.storage_offset() < col:
                continue
            mat = v.as_strided((v.shape[0], width), (v.stride(0), 1), v.storage_offset() - col)
            return mat.to(self.device)
        raise RuntimeError("sharded front needs the batch dict to be column views of one matrix")

    def _flat_embedding(self, inputs):
        """embedding_layer(X, flatten_emb=True), or the same rows from the row-sharded front after enable_sharding()."""
        if getattr(self, "_sharded_front", None) is not None:   # row-sharded tables, P2P push/pull
            from .sharded import sharded_front
            return sharded_front(self._sharded_front, self._batch_matrix(inputs))[0].flatten(start_dim=1)
        return self.embedding_layer(self.get_inputs(inputs), flatten_emb=True)

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
        the two-kernel FusedAdam (same arithmetic; see arena.py).  Call after model_to_device()
        (and after enable_sharding() for row-sharded tables).
        lazy_tables=True (models whose every forward reads the tables through a replaying kernel:
        `_replays_lazy_tables`, i.e. DeepFM, xDeepFM, DLRM; unsharded or row-sharded): the dense Adam
        semantics of the tables are evaluated row-wise and lazily — bit-identical results, O(batch)
        instead of O(vocabulary) optimizer traffic; call materialize_tables() before reading table
        weights outside the kernels (state_dict() and evaluate() do)."""
        if self._optimizer_name != "Adam":
            raise NotImplementedError("the fused optimizer implements Adam only")
        if lazy_tables and not getattr(type(self), "_replays_lazy_tables", False):
            # any other forward reads the tables through kernels that neither replay nor enqueue: the
            # tables would silently stop training
            raise NotImplementedError("%s reads its tables through kernels without the lazy replay; lazy tables "
                                      "are implemented for DeepFM, xDeepFM and DLRM" % type(self).__name__)
        # tables first (the row shards of a sharded run, else every nn.Embedding weight): the dense
        # parameters then form one contiguous tail (one all-reduce, one 3xTF32 split launch per step)
        sharded = getattr(self, "_sharded_params", None)
        first = list(sharded) if sharded else None
        if lazy_tables and not first:
            first = self._front_tables()
        if not first:
            first, seen = [], set()
            for m in self.modules():
                if type(m) == nn.Embedding and id(m.weight) not in seen and m.weight.requires_grad:
                    seen.add(id(m.weight))
                    first.append(m.weight)
        self._arena = ParamArena(self, first=first)
        self._fused_optimizer = FusedAdam(self._arena, lr=self._lr, max_norm=self._max_gradient_norm)
        if lazy_tables:
            self._lazy = self._fused_optimizer.enable_lazy(first)
        self._fused_optimizer.sharded = bool(sharded)
        self._fused_optimizer.dense_prescaled = getattr(self, "_loss_grad", None) is not None
        front = getattr(self, "_sharded_front", None)
        if front is not None:
            self._fused_optimizer.group = front.group     # sums the norm term (and dense gradients) over the ranks
            if front.group.world > 1 and hasattr(front.group, "group"):
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

    def _table_reads(self, X):
        """(plan, lr_plan, ids, emb_tables, lr_tables) of the one fused-front launch through which this model's
        forward reads, and its backward writes, every table row of a step on inputs X; None keeps the serial
        table pass.  Only DeepFM gives one: xDeepFM and DLRM read their tables the same way, but the side pass
        made their steps slower on H100 (the CIN kernels and DLRM's 200 M-row tables need every SM; DESIGN.md 4)."""
        return None

    def fused_train_step(self, batch_data):
        """train_step with the arena optimizer and the fused logit+BCE kernel when the model
        exposes its pre-sigmoid logit terms (`forward_logits`)."""
        opt = self._fused_optimizer
        opt.zero_grad()
        regularised = bool(self._embedding_regularizer or self._net_regularizer)
        if not regularised and opt.early_tables_ok():
            # the untouched table granules get this step's update on a side stream while forward and backward run
            reads = self._table_reads(self.get_inputs(batch_data))
            if reads is not None:
                opt.start_early_tables(*reads)
        y_true = self.get_labels(batch_data)
        fused_logit = hasattr(self, "forward_logits") and not regularised
        if fused_logit:
            loss = self.fused_loss(batch_data, y_true)
        else:
            loss = self.compute_loss(self.forward(batch_data), y_true)
        seed = getattr(self, "_loss_grad", None)      # 1/world for row-sharded runs (see enable_sharding)
        # opt.step() joins the MLP's weight-gradient side stream where it first reads the dense gradients.  Only on
        # the fused-logit path, where the MLP chain is the one reader of its weights: a regulariser gives every weight
        # a second gradient, which autograd adds to the chain's on this stream, so that backward must join itself.  A
        # sharded step sums the dense gradients over the ranks from inside the backward, so it joins there too.
        opt.arena.defer_join = fused_logit and not opt.sharded
        try:
            if seed is not None:
                loss.backward(seed)
            else:
                loss.backward()
        finally:
            opt.arena.defer_join = False
        opt.step()
        return loss

    def fused_loss(self, batch_data, y_true):
        """The loss of fused_train_step's fused path: the fused logit + BCE kernel over the sum of the model's
        pre-sigmoid logit terms (`forward_logits`).  A model whose loss is not a BCE of such a sum overrides this."""
        return F2.logit_bce(y_true, *self.forward_logits(batch_data))[0]


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
    _replays_lazy_tables = True

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

    def _table_reads(self, X):
        if getattr(self, "_sharded_front", None) is not None:
            return None
        fp = front_plan(self.embedding_layer, self.fm.lr_layer, X)
        if fp is None:
            return None
        order, plan, tables, lr_plan, lr_tables = fp
        return plan, lr_plan, [X[f] for f in order], [t.weight for t in tables], [t.weight for t in lr_tables]

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
    _routes_sharded_front = True

    def __init__(self, feature_map, model_id="DCNv2", gpu=-1, model_structure="parallel",
                 use_low_rank_mixture=False, low_rank=32, num_experts=4, learning_rate=1e-3,
                 embedding_dim=10, stacked_dnn_hidden_units=[], parallel_dnn_hidden_units=[],
                 dnn_activations="ReLU", num_cross_layers=3, net_dropout=0, batch_norm=False,
                 embedding_regularizer=None, net_regularizer=None, **kwargs):
        super(DCNv2, self).__init__(feature_map, model_id=model_id, gpu=gpu,
                                    embedding_regularizer=embedding_regularizer, net_regularizer=net_regularizer,
                                    **kwargs)
        if use_low_rank_mixture:
            raise NotImplementedError(
                "zoo.DCNv2 has no low-rank mixture (arena, fused Adam, graph capture and sharding do not cover "
                "CrossNetMix); the reference DCNv2 with use_low_rank_mixture=True runs its CrossNetMix on the "
                "kernels under fuxictr_b200.patch.enable(), or build a model from layers.CrossNetMix")
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
        emb = self._flat_embedding(inputs)
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


def _gdcn_dnn_units(name, dnn_hidden_units):
    """GDCN and GDCNP need a DNN tower: the reference builds none for empty dnn_hidden_units and then fails (GDCNP
    at construction, GDCN at its first forward); refuse before anything is built."""
    if not dnn_hidden_units:
        raise ValueError("%s needs a non-empty dnn_hidden_units (its DNN tower %s)"
                         % (name, "gives the logit" if name == "GDCN" else "feeds fc"))
    return list(dnn_hidden_units)


class GDCN(RankModel):
    """model_zoo/GDCN/src/GDCN.py, GDCN: the gated cross network stacked under a DNN that ends in the logit,
    y = sigmoid(dnn(cross_net(flatten(E)))).  Unknown keyword arguments (the GDCN_test YAML's `crossing_layers`)
    are accepted and ignored, as the reference's **kwargs do."""
    _routes_sharded_front = True

    def __init__(self, feature_map, model_id="GDCN", gpu=-1, learning_rate=1e-3, embedding_dim=10,
                 dnn_hidden_units=[], dnn_activations="ReLU", num_cross_layers=3, net_dropout=0, batch_norm=False,
                 embedding_regularizer=None, net_regularizer=None, **kwargs):
        super(GDCN, self).__init__(feature_map, model_id=model_id, gpu=gpu,
                                   embedding_regularizer=embedding_regularizer, net_regularizer=net_regularizer,
                                   **kwargs)
        units = _gdcn_dnn_units("GDCN", dnn_hidden_units)
        self.embedding_layer = FeatureEmbedding(feature_map, embedding_dim)
        width = feature_map.sum_emb_out_dim()
        self.dnn = MLP_Block(width, hidden_units=units, hidden_activations=dnn_activations, output_dim=1,
                             output_activation=None, dropout_rates=net_dropout, batch_norm=batch_norm)
        self.cross_net = GateCorssLayer(width, num_cross_layers)
        self._finish(kwargs, learning_rate)

    def forward_logits(self, inputs):
        return (self.dnn(self.cross_net(self._flat_embedding(inputs))),)

    def forward(self, inputs):
        return {"y_pred": self.output_activation(self.forward_logits(inputs)[0])}


class GDCNP(RankModel):
    """model_zoo/GDCN/src/GDCN.py, GDCNP: the gated cross network beside a DNN tower, one Linear over
    [cross_net(E) | dnn(E)] to the logit.  Unknown keyword arguments are ignored as in GDCN."""
    _routes_sharded_front = True

    def __init__(self, feature_map, model_id="GDCNP", gpu=-1, learning_rate=1e-3, embedding_dim=10,
                 dnn_hidden_units=[], dnn_activations="ReLU", num_cross_layers=3, net_dropout=0, batch_norm=False,
                 embedding_regularizer=None, net_regularizer=None, **kwargs):
        super(GDCNP, self).__init__(feature_map, model_id=model_id, gpu=gpu,
                                    embedding_regularizer=embedding_regularizer, net_regularizer=net_regularizer,
                                    **kwargs)
        units = _gdcn_dnn_units("GDCNP", dnn_hidden_units)
        self.embedding_layer = FeatureEmbedding(feature_map, embedding_dim)
        width = feature_map.sum_emb_out_dim()
        self.dnn = MLP_Block(width, hidden_units=units, hidden_activations=dnn_activations, output_dim=None,
                             output_activation=None, dropout_rates=net_dropout, batch_norm=batch_norm)
        self.cross_net = GateCorssLayer(width, num_cross_layers)
        self.fc = nn.Linear(units[-1] + width, 1)
        self._finish(kwargs, learning_rate)

    def forward_logits(self, inputs):
        emb = self._flat_embedding(inputs)
        cross = self.cross_net(emb)
        return (F2.linear_act(torch.cat([cross, self.dnn(emb)], dim=1), self.fc.weight, self.fc.bias),)

    def forward(self, inputs):
        return {"y_pred": self.output_activation(self.forward_logits(inputs)[0])}


class FinalMLP(RankModel):
    """model_zoo/FinalMLP/src/FinalMLP.py, FinalMLP: two MLP towers over the flattened embedding, each fed through its
    feature-selection gate (use_fs), fused into the logit by the multi-head bilinear InteractionAggregation.  A gate
    without context features runs its MLP on one row (layers.FeatureSelection).  Unknown keyword arguments are
    accepted and ignored, as the reference's **kwargs are."""
    _routes_sharded_front = True

    def __init__(self, feature_map, model_id="FinalMLP", gpu=-1, learning_rate=1e-3, embedding_dim=10,
                 mlp1_hidden_units=[64, 64, 64], mlp1_hidden_activations="ReLU", mlp1_dropout=0, mlp1_batch_norm=False,
                 mlp2_hidden_units=[64, 64, 64], mlp2_hidden_activations="ReLU", mlp2_dropout=0, mlp2_batch_norm=False,
                 use_fs=True, fs_hidden_units=[64], fs1_context=[], fs2_context=[], num_heads=1,
                 embedding_regularizer=None, net_regularizer=None, **kwargs):
        if not mlp1_hidden_units or not mlp2_hidden_units:
            # the reference fails here too (an IndexError on mlp*_hidden_units[-1]): the fusion needs both towers
            raise ValueError("FinalMLP needs non-empty mlp1_hidden_units and mlp2_hidden_units (the towers the "
                             "fusion module combines)")
        super(FinalMLP, self).__init__(feature_map, model_id=model_id, gpu=gpu,
                                       embedding_regularizer=embedding_regularizer, net_regularizer=net_regularizer,
                                       **kwargs)
        self.embedding_layer = FeatureEmbedding(feature_map, embedding_dim)
        feature_dim = embedding_dim * feature_map.num_fields
        self.mlp1 = MLP_Block(input_dim=feature_dim, output_dim=None, hidden_units=mlp1_hidden_units,
                              hidden_activations=mlp1_hidden_activations, output_activation=None,
                              dropout_rates=mlp1_dropout, batch_norm=mlp1_batch_norm)
        self.mlp2 = MLP_Block(input_dim=feature_dim, output_dim=None, hidden_units=mlp2_hidden_units,
                              hidden_activations=mlp2_hidden_activations, output_activation=None,
                              dropout_rates=mlp2_dropout, batch_norm=mlp2_batch_norm)
        self.use_fs = use_fs
        if self.use_fs:
            self.fs_module = FeatureSelection(feature_map, feature_dim, embedding_dim, fs_hidden_units, fs1_context,
                                              fs2_context)
        self.fusion_module = InteractionAggregation(mlp1_hidden_units[-1], mlp2_hidden_units[-1], output_dim=1,
                                                    num_heads=num_heads)
        self._finish(kwargs, learning_rate)

    def enable_sharding(self, group, batch_local, matrix_width, idx_dtype=torch.float64, want_fm=True):
        """RankModel.enable_sharding for a FinalMLP whose gates have no context features: context features are
        looked up in tables of their own, which the row-sharded front does not carry."""
        if self.use_fs and (self.fs_module.fs1_context or self.fs_module.fs2_context):
            raise NotImplementedError("FinalMLP with fs1_context / fs2_context cannot be row-sharded: the gates' "
                                      "context tables are not part of the sharded front")
        return super(FinalMLP, self).enable_sharding(group, batch_local, matrix_width, idx_dtype=idx_dtype,
                                                     want_fm=want_fm)

    def forward_logits(self, inputs):
        flat_emb = self._flat_embedding(inputs)
        if self.use_fs:
            feat1, feat2 = self.fs_module(self.get_inputs(inputs), flat_emb)
        else:
            feat1, feat2 = flat_emb, flat_emb
        return (self.fusion_module(self.mlp1(feat1), self.mlp2(feat2)),)

    def forward(self, inputs):
        return {"y_pred": self.output_activation(self.forward_logits(inputs)[0])}


class DualMLP(RankModel):
    """model_zoo/FinalMLP/src/DualMLP.py, DualMLP: two MLP towers over the flattened embedding, each ending in a
    logit, summed.  Unknown keyword arguments are accepted and ignored, as the reference's **kwargs are."""
    _routes_sharded_front = True

    def __init__(self, feature_map, model_id="DualMLP", gpu=-1, learning_rate=1e-3, embedding_dim=10,
                 mlp1_hidden_units=[64, 64, 64], mlp1_hidden_activations="ReLU", mlp1_dropout=0, mlp1_batch_norm=False,
                 mlp2_hidden_units=[64, 64, 64], mlp2_hidden_activations="ReLU", mlp2_dropout=0, mlp2_batch_norm=False,
                 embedding_regularizer=None, net_regularizer=None, **kwargs):
        super(DualMLP, self).__init__(feature_map, model_id=model_id, gpu=gpu,
                                      embedding_regularizer=embedding_regularizer, net_regularizer=net_regularizer,
                                      **kwargs)
        self.embedding_layer = FeatureEmbedding(feature_map, embedding_dim)
        self.mlp1 = MLP_Block(input_dim=embedding_dim * feature_map.num_fields, output_dim=1,
                              hidden_units=mlp1_hidden_units, hidden_activations=mlp1_hidden_activations,
                              output_activation=None, dropout_rates=mlp1_dropout, batch_norm=mlp1_batch_norm)
        self.mlp2 = MLP_Block(input_dim=embedding_dim * feature_map.num_fields, output_dim=1,
                              hidden_units=mlp2_hidden_units, hidden_activations=mlp2_hidden_activations,
                              output_activation=None, dropout_rates=mlp2_dropout, batch_norm=mlp2_batch_norm)
        self._finish(kwargs, learning_rate)

    def forward_logits(self, inputs):
        flat_emb = self._flat_embedding(inputs)
        return (self.mlp1(flat_emb), self.mlp2(flat_emb))

    def forward(self, inputs):
        return {"y_pred": self.output_activation(sum(self.forward_logits(inputs)))}


class MaskNet(RankModel):
    """model_zoo/MaskNet/src/MaskNet.py, MaskNet: MaskBlocks over the flattened embedding V_emb and its per-field
    LayerNorm V_hidden (emb_layernorm), chained (SerialMaskNet, ending in fc) or side by side under an MLP
    (ParallelMaskNet).  Every block's mask MLP reads V_emb, not V_hidden, as in the reference.  V_emb's gradient is one
    buffer that every block and the embedding LayerNorm add into (functional.shared_grad).  The F embedding
    LayerNorms' weights and biases are kept in one buffer at one stride (functional.pack_field_params; the fused
    optimizer's arena keeps that layout), so their kernel reads them where they live.  Unknown keyword arguments are
    accepted and ignored, as the reference's **kwargs are."""
    _routes_sharded_front = True

    def __init__(self, feature_map, model_id="MaskNet", gpu=-1, learning_rate=1e-3, embedding_dim=10,
                 dnn_hidden_units=[64, 64, 64], dnn_hidden_activations="ReLU", model_type="SerialMaskNet",
                 parallel_num_blocks=1, parallel_block_dim=64, reduction_ratio=1, embedding_regularizer=None,
                 net_regularizer=None, net_dropout=0, emb_layernorm=True, net_layernorm=True, **kwargs):
        if model_type not in ("SerialMaskNet", "ParallelMaskNet"):
            raise ValueError("MaskNet: model_type must be 'SerialMaskNet' or 'ParallelMaskNet', got %r" % (model_type,))
        if model_type == "SerialMaskNet" and not dnn_hidden_units:
            # the reference would build no block and a bare Linear(d, 1): not a MaskNet
            raise ValueError("SerialMaskNet needs a non-empty dnn_hidden_units (its chain of mask blocks)")
        if emb_layernorm:
            bound = F2.masknet_width_bound(embedding_dim, "MaskNet embedding_dim (emb_layernorm)")
            if bound:
                raise ValueError(bound)
        super(MaskNet, self).__init__(feature_map, model_id=model_id, gpu=gpu,
                                      embedding_regularizer=embedding_regularizer, net_regularizer=net_regularizer,
                                      **kwargs)
        self.embedding_layer = FeatureEmbedding(feature_map, embedding_dim)
        if model_type == "SerialMaskNet":
            self.mask_net = SerialMaskNet(input_dim=feature_map.num_fields * embedding_dim,
                                          output_dim=1,
                                          output_activation=self.output_activation,
                                          hidden_units=dnn_hidden_units,
                                          hidden_activations=dnn_hidden_activations,
                                          reduction_ratio=reduction_ratio,
                                          dropout_rates=net_dropout,
                                          layer_norm=net_layernorm)
        else:
            self.mask_net = ParallelMaskNet(input_dim=feature_map.num_fields * embedding_dim,
                                            output_dim=1,
                                            output_activation=self.output_activation,
                                            num_blocks=parallel_num_blocks,
                                            block_dim=parallel_block_dim,
                                            hidden_units=dnn_hidden_units,
                                            hidden_activations=dnn_hidden_activations,
                                            reduction_ratio=reduction_ratio,
                                            dropout_rates=net_dropout,
                                            layer_norm=net_layernorm)
        self.num_fields = feature_map.num_fields
        if emb_layernorm:
            self.emb_norm = nn.ModuleList(nn.LayerNorm(embedding_dim) for _ in range(self.num_fields))
        else:
            self.emb_norm = None
        self._finish(kwargs, learning_rate)

    def model_to_device(self):
        super(MaskNet, self).model_to_device()
        if self.emb_norm is not None:
            F2.pack_field_params(self.emb_norm)

    def _logit_mlp(self):
        """ParallelMaskNet's MLP without its output Sigmoid (the same modules, not registered a second time)."""
        ent = self.__dict__.get("_logit_dnn")
        if ent is None:
            dnn = self.mask_net.dnn
            ent = MLP_Block.__new__(MLP_Block)
            nn.Module.__init__(ent)
            mods = list(dnn.mlp)
            ent.mlp = nn.Sequential(*(mods[:-1] if type(mods[-1]) == nn.Sigmoid else mods))
            self.__dict__["_logit_dnn"] = ent
        return ent

    def forward_logits(self, inputs):
        return (self.dense_logit(self._flat_embedding(inputs)),)

    def dense_logit(self, flat_emb):
        """The pre-sigmoid logit from the flattened embedding (B, F D): the embedding LayerNorm, the mask blocks and
        the head."""
        emb, sink = F2.shared_grad(flat_emb)
        v_hidden = emb
        if self.emb_norm is not None:
            ws, bs = [m.weight for m in self.emb_norm], [m.bias for m in self.emb_norm]
            if F2.field_param_layout(ws, bs) is None:       # moved since model_to_device (e.g. by .to())
                F2.pack_field_params(self.emb_norm)
            v_hidden = F2.field_layernorm(emb, sink, ws, bs, self.emb_norm[0].eps)
        net = self.mask_net
        if isinstance(net, SerialMaskNet):
            fc = net.fc[0]
            return F2.linear_act(net.blocks_out(emb, v_hidden, sink), fc.weight, fc.bias)
        return self._logit_mlp()(net.blocks_out(emb, v_hidden, sink))

    def forward(self, inputs):
        return {"y_pred": self.output_activation(self.forward_logits(inputs)[0])}


class AutoInt(RankModel):
    """model_zoo/AutoInt/src/AutoInt.py, AutoInt (AutoInt+ with a DNN): a stack of MultiHeadSelfAttention layers over
    the field embeddings, y = sigmoid(fc(flatten(attention(E))) [+ dnn(flatten(E))] [+ LR(X)]).  Each attention layer
    is one projection GEMM and one row kernel (layers.MultiHeadSelfAttention); in training mode with net_dropout the
    layers draw their attention-weight masks from one dropout snapshot.  An empty dnn_hidden_units builds no DNN, as
    in the reference.  Unknown keyword arguments are accepted and ignored, as the reference's **kwargs are."""
    _routes_sharded_front = True

    def __init__(self, feature_map, model_id="AutoInt", gpu=-1, learning_rate=1e-3, embedding_dim=10,
                 dnn_hidden_units=[64, 64, 64], dnn_activations="ReLU", attention_layers=2, num_heads=1,
                 attention_dim=8, net_dropout=0, batch_norm=False, layer_norm=False, use_scale=False,
                 use_wide=False, use_residual=True, embedding_regularizer=None, net_regularizer=None, **kwargs):
        assert attention_dim % num_heads == 0, \
            "attention_dim={} is not divisible by num_heads={}".format(attention_dim, num_heads)
        bound = F2.autoint_bound(feature_map.num_fields, attention_dim, num_heads)
        if bound is not None:
            raise NotImplementedError("AutoInt kernels: " + bound)
        super(AutoInt, self).__init__(feature_map, model_id=model_id, gpu=gpu,
                                      embedding_regularizer=embedding_regularizer, net_regularizer=net_regularizer,
                                      **kwargs)
        self.embedding_layer = FeatureEmbedding(feature_map, embedding_dim)
        self.lr_layer = LogisticRegression(feature_map, use_bias=False) if use_wide else None
        self.dnn = MLP_Block(input_dim=feature_map.sum_emb_out_dim(), output_dim=1, hidden_units=dnn_hidden_units,
                             hidden_activations=dnn_activations, output_activation=None, dropout_rates=net_dropout,
                             batch_norm=batch_norm) if dnn_hidden_units else None
        self.self_attention = nn.Sequential(
            *[MultiHeadSelfAttention(embedding_dim if i == 0 else attention_dim, attention_dim=attention_dim,
                                     num_heads=num_heads, dropout_rate=net_dropout, use_residual=use_residual,
                                     use_scale=use_scale, layer_norm=layer_norm)
              for i in range(attention_layers)])
        self.fc = nn.Linear(feature_map.num_fields * attention_dim, 1)
        self._finish(kwargs, learning_rate)

    def enable_sharding(self, group, batch_local, matrix_width, idx_dtype=torch.float64, want_fm=False):
        """RankModel.enable_sharding without the FM term, which AutoInt does not have: with use_wide the sharded
        front's logit is the LR term alone."""
        if want_fm:
            raise ValueError("AutoInt has no FM term: enable_sharding(..., want_fm=False)")
        return super(AutoInt, self).enable_sharding(group, batch_local, matrix_width, idx_dtype=idx_dtype,
                                                    want_fm=False)

    def _front(self, inputs):
        """(feature_emb (B, F, D), LR logit or None)."""
        if getattr(self, "_sharded_front", None) is not None:   # row-sharded tables (and LR), P2P push/pull
            from .sharded import sharded_front
            feature_emb, logit = sharded_front(self._sharded_front, self._batch_matrix(inputs))
            return feature_emb, (logit if self.lr_layer is not None else None)
        X = self.get_inputs(inputs)
        if self.lr_layer is None:
            return self.embedding_layer(X), None
        fused = fused_front(self.embedding_layer, self.lr_layer, X, want_fm=False)
        if fused is not None:     # gather + LR in one launch
            return fused
        return self.embedding_layer(X), self.lr_layer(X)

    def attention(self, feature_emb):
        """The self-attention stack on (B, F, D)."""
        mods = list(self.self_attention)
        snap = None
        if mods and self.training and mods[0].dot_attention.dropout is not None:
            snap = F2.dropout_snapshot(feature_emb.device, len(mods))
        x = feature_emb
        for i, m in enumerate(mods):
            x = m(x, snapshot=snap, layer=i, want_aux=i + 1 < len(mods))
        return x

    def forward_logits(self, inputs):
        feature_emb, lr_logit = self._front(inputs)
        attention_out = self.attention(feature_emb)
        terms = [F2.linear_act(attention_out.flatten(start_dim=1), self.fc.weight, self.fc.bias)]
        if self.dnn is not None:
            terms.append(self.dnn(feature_emb.flatten(start_dim=1)))
        if lr_logit is not None:
            terms.append(lr_logit)
        return tuple(terms)

    def forward(self, inputs):
        terms = self.forward_logits(inputs)
        y_pred = terms[0]
        for t in terms[1:]:
            y_pred = y_pred + t
        return {"y_pred": self.output_activation(y_pred)}


class WuKong(RankModel):
    """model_zoo/WuKong/src/WuKong.py, WuKong: num_wukong_layers WuKongLayers over the field embeddings, then
    y = sigmoid(fc(flatten(stack(E)))).  Each layer is the FM row kernel, the FMB's MLP, one field-axis GEMM and the
    combine row kernel (layers.WuKongLayer); the last layer writes the flatten fc reads.  fc is the reference's
    MLP_Block (with mlp_batch_norm, torch's BatchNorm1d between our Linears, as every batch_norm MLP runs).  Unknown
    keyword arguments are accepted and ignored, as the reference's **kwargs are.  Refused: fmp_rank_k=None (the
    vanilla FM), num_wukong_layers < 1 and shapes outside functional.wukong_bound."""
    _routes_sharded_front = True

    def __init__(self, feature_map, model_id="WuKong", gpu=-1, learning_rate=1e-3, embedding_dim=64,
                 num_wukong_layers=3, lcb_features=40, fmb_features=40, fmb_mlp_units=[32, 32],
                 fmb_mlp_activations="relu", fmp_rank_k=8, mlp_hidden_units=[32, 32], mlp_hidden_activations="relu",
                 mlp_batch_norm=True, layer_norm=True, net_dropout=0, embedding_regularizer=None, net_regularizer=None,
                 **kwargs):
        if num_wukong_layers < 1:
            raise NotImplementedError("WuKong needs num_wukong_layers >= 1, got %d (the reference then builds an fc "
                                      "for lcb + fmb fields over the embedding's fields)" % num_wukong_layers)
        output_features = lcb_features + fmb_features
        for fields in ((feature_map.num_fields, output_features) if num_wukong_layers > 1 or
                       feature_map.num_fields == output_features else (feature_map.num_fields,)):
            bound = F2.wukong_bound(fields, output_features, embedding_dim, fmp_rank_k)
            if bound is not None:
                raise NotImplementedError("WuKong kernels: " + bound)
        super(WuKong, self).__init__(feature_map, model_id=model_id, gpu=gpu,
                                     embedding_regularizer=embedding_regularizer, net_regularizer=net_regularizer,
                                     **kwargs)
        self.embedding_dim = embedding_dim
        self.embedding_layer = FeatureEmbedding(feature_map, embedding_dim)
        self.wukong_stack = nn.Sequential(*[
            WuKongLayer(input_features=feature_map.num_fields if i == 0 else output_features,
                        lcb_features=lcb_features, fmb_features=fmb_features, embedding_dim=embedding_dim,
                        fmp_rank_k=fmp_rank_k, fmb_mlp_units=fmb_mlp_units, fmb_mlp_activations=fmb_mlp_activations,
                        fmb_dropout=net_dropout, layer_norm=layer_norm)
            for i in range(num_wukong_layers)])
        self.fc = MLP_Block(input_dim=output_features * embedding_dim, output_dim=1, hidden_units=mlp_hidden_units,
                            hidden_activations=mlp_hidden_activations, output_activation=self.output_activation,
                            batch_norm=mlp_batch_norm)
        self._finish(kwargs, learning_rate)

    def enable_sharding(self, group, batch_local, matrix_width, idx_dtype=torch.float64, want_fm=False):
        """RankModel.enable_sharding without the FM term, which WuKong does not have."""
        if want_fm:
            raise ValueError("WuKong has no FM term: enable_sharding(..., want_fm=False)")
        return super(WuKong, self).enable_sharding(group, batch_local, matrix_width, idx_dtype=idx_dtype,
                                                   want_fm=False)

    def _logit_mlp(self):
        """fc without its output Sigmoid (the same modules, not registered a second time)."""
        ent = self.__dict__.get("_logit_fc")
        if ent is None:
            ent = MLP_Block.__new__(MLP_Block)
            nn.Module.__init__(ent)
            mods = list(self.fc.mlp)
            ent.mlp = nn.Sequential(*(mods[:-1] if type(mods[-1]) == nn.Sigmoid else mods))
            self.__dict__["_logit_fc"] = ent
        return ent

    def _feature_emb(self, inputs):
        """The field embeddings (B, F, D), from the row-sharded front after enable_sharding()."""
        if getattr(self, "_sharded_front", None) is not None:   # row-sharded tables, P2P push/pull
            from .sharded import sharded_front
            return sharded_front(self._sharded_front, self._batch_matrix(inputs))[0]
        return self.embedding_layer(self.get_inputs(inputs))

    def forward_logits(self, inputs):
        fc = self._logit_mlp()
        first = next(m for m in fc.mlp if type(m) == nn.Linear)
        flat = wukong_stack(list(self.wukong_stack), self._feature_emb(inputs),
                            want_aux=F2._tc_layer_ok(first.weight) and fc.chain_layers() is not None)
        return (fc(flat),)

    def forward(self, inputs):
        return {"y_pred": self.output_activation(self.forward_logits(inputs)[0])}


class DLRM(RankModel):
    """model_zoo/DLRM/src/DLRM.py:43-123: embeddings of the non-numeric fields (+ a bottom MLP over the
    numeric ones as one more "field"), pairwise dot (or concat) interaction, top MLP with the output
    activation inside it."""
    _routes_sharded_front = True
    _replays_lazy_tables = True

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
        elif getattr(self, "_lazy", None) is not None:     # lazy tables: read through the replaying front
            fused = fused_front(self.embedding_layer, None, X, want_fm=False)
            if fused is None:
                raise RuntimeError("lazy tables are only readable through the fused front (unsupported config)")
            feat_emb = fused[0]
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
    _routes_sharded_front = True

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
        front = getattr(self, "_sharded_front", None)
        if front is not None:       # row-sharded tables: (B, D) / (B, L, D) views of the landed rows
            from .sharded import sharded_front
            landed, _ = sharded_front(front, self._batch_matrix(inputs))
            views = front.field_views(landed)
            emb = OrderedDict((name, views[name]) for name in self.feature_map.features.keys() if name in views)
        else:
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
    _routes_sharded_front = True
    _replays_lazy_tables = True

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
        if getattr(self, "_sharded_front", None) is not None:   # row-sharded tables (and LR), P2P push/pull
            from .sharded import sharded_front
            feature_emb, lr_logit = sharded_front(self._sharded_front, self._batch_matrix(inputs))
            terms = [lr_logit, self.cin(feature_emb)]
            if self.dnn is not None:
                terms.append(self.dnn(feature_emb.flatten(start_dim=1)))
            return tuple(terms)
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


class FinalNet(RankModel):
    """model_zoo/FinalNet/src/FinalNet.py, FinalNet: block 1 (a FinalBlock over the flattened embedding, or over the
    feature gating's [e, e * gates] with use_feature_gating) and fc1; with block_type "2B" also block 2 over the plain
    flattened embedding and fc2, y_pred = sigmoid((y1 + y2) / 2) and the self-distillation loss of add_loss, which the
    fused step takes in one launch (functional.finalnet_loss).  The embedding's gradient is one shared_grad buffer that
    the gating's backward and the blocks' first dgrads add into.  Unknown keyword arguments are accepted and ignored,
    as the reference's **kwargs are.  Refused: activations other than None, ReLU and Sigmoid, shapes outside
    functional.finalnet_bound, lazy tables and enable_sharding(want_fm=True)."""
    _routes_sharded_front = True

    def __init__(self, feature_map, model_id="FinalNet", gpu=-1, learning_rate=1e-3, embedding_dim=10,
                 block_type="2B", batch_norm=True, use_feature_gating=False, block1_hidden_units=[64, 64, 64],
                 block1_hidden_activations=None, block1_dropout=0, block2_hidden_units=[64, 64, 64],
                 block2_hidden_activations=None, block2_dropout=0, residual_type="concat", embedding_regularizer=None,
                 net_regularizer=None, **kwargs):
        super(FinalNet, self).__init__(feature_map, model_id=model_id, gpu=gpu,
                                       embedding_regularizer=embedding_regularizer, net_regularizer=net_regularizer,
                                       **kwargs)
        assert block_type in ["1B", "2B"], "block_type={} not supported.".format(block_type)
        num_fields = feature_map.num_fields
        bound = F2.finalnet_bound(fields=num_fields, embedding_dim=embedding_dim) if use_feature_gating else None
        if bound is not None:
            raise NotImplementedError("FinalNet kernels: " + bound)
        self.embedding_layer = FeatureEmbedding(feature_map, embedding_dim)
        self.use_feature_gating = use_feature_gating
        if use_feature_gating:
            self.feature_gating = FeatureGating(num_fields, gate_residual="concat")
            gate_out_dim = embedding_dim * num_fields * 2
        self.block_type = block_type
        self.block1 = FinalBlock(input_dim=gate_out_dim if use_feature_gating else embedding_dim * num_fields,
                                 hidden_units=block1_hidden_units, hidden_activations=block1_hidden_activations,
                                 dropout_rates=block1_dropout, batch_norm=batch_norm, residual_type=residual_type)
        self.fc1 = nn.Linear(block1_hidden_units[-1], 1)
        if block_type == "2B":
            self.block2 = FinalBlock(input_dim=embedding_dim * num_fields, hidden_units=block2_hidden_units,
                                     hidden_activations=block2_hidden_activations, dropout_rates=block2_dropout,
                                     batch_norm=batch_norm, residual_type=residual_type)
            self.fc2 = nn.Linear(block2_hidden_units[-1], 1)
        self._finish(kwargs, learning_rate)

    def enable_sharding(self, group, batch_local, matrix_width, idx_dtype=torch.float64, want_fm=False):
        """RankModel.enable_sharding without the FM term, which FinalNet does not have."""
        if want_fm:
            raise ValueError("FinalNet has no FM term: enable_sharding(..., want_fm=False)")
        return super(FinalNet, self).enable_sharding(group, batch_local, matrix_width, idx_dtype=idx_dtype,
                                                     want_fm=False)

    def _feature_emb(self, inputs):
        """The field embeddings (B, F, D), from the row-sharded front after enable_sharding()."""
        if getattr(self, "_sharded_front", None) is not None:   # row-sharded tables, P2P push/pull
            from .sharded import sharded_front
            return sharded_front(self._sharded_front, self._batch_matrix(inputs))[0]
        return self.embedding_layer(self.get_inputs(inputs))

    def forward_logits(self, inputs):
        """(y1,) or, with 2B, (y1, y2): the blocks' pre-sigmoid logits (B, 1)."""
        feature_emb = self._feature_emb(inputs)
        flat, sink = F2.shared_grad(feature_emb.flatten(start_dim=1))
        first = F2._tc_layer_ok(self.block1.layer[0].linear.weight) if len(self.block1.layer) else False
        if self.use_feature_gating:
            x1 = self.feature_gating.run(flat, sink=sink, want_aux=first)
            out1 = self.block1.run(x1)
        else:
            out1 = self.block1.run(flat, sink=sink)
        y1 = F2.linear_act(out1, self.fc1.weight, self.fc1.bias)
        if self.block_type == "1B":
            return (y1,)
        out2 = self.block2.run(flat, sink=sink)
        return (y1, F2.linear_act(out2, self.fc2.weight, self.fc2.bias))

    def forward(self, inputs):
        logits = self.forward_logits(inputs)
        if self.block_type == "1B":
            return {"y_pred": self.output_activation(logits[0]), "y1": None, "y2": None}
        y1, y2 = logits
        return {"y_pred": self.output_activation(0.5 * (y1 + y2)), "y1": y1, "y2": y2}

    def add_loss(self, return_dict, y_true):
        """FinalNet.add_loss: BCE of y_pred, plus with 2B the two self-distillation terms against y_pred detached."""
        loss = self.loss_fn(return_dict["y_pred"], y_true, reduction="mean")
        if self.block_type == "2B":
            y1 = self.output_activation(return_dict["y1"])
            y2 = self.output_activation(return_dict["y2"])
            loss1 = self.loss_fn(y1, return_dict["y_pred"].detach(), reduction="mean")
            loss2 = self.loss_fn(y2, return_dict["y_pred"].detach(), reduction="mean")
            loss = loss + loss1 + loss2
        return loss

    def compute_loss(self, return_dict, y_true):
        return self.add_loss(return_dict, y_true) + self.regularization_loss()

    def fused_loss(self, batch_data, y_true):
        if self.block_type == "1B":
            return super(FinalNet, self).fused_loss(batch_data, y_true)
        return F2.finalnet_loss(y_true, *self.forward_logits(batch_data))[0]


class BST(RankModel):
    """model_zoo/BST/src/BST.py, BST: per (target, sequence) field pair a BehaviorTransformer over the L = max_len + 1
    tokens [history | target] (a tuple of fields: their embeddings side by side, then the position embedding), pooled
    ("mean", "sum", "target" or "concat") into a vector that replaces the sequence fields; the DNN reads the remaining
    embeddings in FeatureMap order, then the pooled vectors in pair order.  The target fields' embeddings stay in the
    DNN input too.  Each block runs on the kernels (layers.TransformerBlock); the key-padding mask comes from the
    first sequence field's ids (0 = padding).  Unknown keyword arguments are accepted and ignored, as the reference's
    **kwargs are.  Refused: model_dim % num_heads != 0 (the reference's assert), shapes outside functional.bst_bound,
    lazy tables and enable_sharding(want_fm=True)."""
    _routes_sharded_front = True

    def __init__(self, feature_map, model_id="BST", gpu=-1, dnn_hidden_units=[256, 128, 64], dnn_activations="ReLU",
                 num_heads=2, stacked_transformer_layers=1, attention_dropout=0, learning_rate=1e-3, embedding_dim=10,
                 net_dropout=0, batch_norm=False, layer_norm=True, use_residual=True,
                 bst_target_field=[("item_id", "cate_id")], bst_sequence_field=[("click_history", "cate_history")],
                 seq_pooling_type="mean", use_position_emb=True, use_causal_mask=False, embedding_regularizer=None,
                 net_regularizer=None, **kwargs):
        as_list = lambda v: v if type(v) == list else [v]                       # noqa: E731
        targets, sequences = as_list(bst_target_field), as_list(bst_sequence_field)
        assert len(targets) == len(sequences), "len(self.bst_target_field) != len(self.bst_sequence_field)"
        if seq_pooling_type not in ("mean", "sum", "target", "concat"):
            raise ValueError("seq_pooling_type={} not supported.".format(seq_pooling_type))
        dims = []
        for target, sequence in zip(targets, sequences):
            names = list(_flatten([sequence]))
            if len(list(_flatten([target]))) != len(names):
                raise ValueError("BST: target %r and sequence %r have different numbers of fields" % (target, sequence))
            model_dim = embedding_dim * (int(use_position_emb) + len(names))
            seq_len = feature_map.features[names[0]]["max_len"] + 1
            assert model_dim % num_heads == 0, "embed_dim must be divisible by num_heads"
            bound = F2.bst_bound(seq_len, model_dim, num_heads, len(names))
            if bound is not None:
                raise NotImplementedError("BST kernels: " + bound)
            dims.append((model_dim, seq_len, len(names)))
        super(BST, self).__init__(feature_map, model_id=model_id, gpu=gpu,
                                  embedding_regularizer=embedding_regularizer, net_regularizer=net_regularizer,
                                  **kwargs)
        self.bst_target_field, self.bst_sequence_field = targets, sequences
        self.use_causal_mask = use_causal_mask
        self.seq_pooling_type = seq_pooling_type
        self.embedding_dim = embedding_dim
        self.num_heads = num_heads
        self.embedding_layer = FeatureEmbeddingDict(feature_map, embedding_dim)
        self.transformer_encoders = nn.ModuleList()
        seq_out_dim = 0
        for model_dim, seq_len, parts in dims:
            width = seq_len * model_dim if seq_pooling_type == "concat" else model_dim
            seq_out_dim += width - parts * embedding_dim
            self.transformer_encoders.append(
                BehaviorTransformer(seq_len=seq_len, model_dim=model_dim, num_heads=num_heads,
                                    stacked_transformer_layers=stacked_transformer_layers,
                                    attn_dropout=attention_dropout, net_dropout=net_dropout,
                                    position_dim=embedding_dim, use_position_emb=use_position_emb,
                                    layer_norm=layer_norm, use_residual=use_residual))
        self.dnn = MLP_Block(input_dim=feature_map.sum_emb_out_dim() + seq_out_dim, output_dim=1,
                             hidden_units=dnn_hidden_units, hidden_activations=dnn_activations,
                             output_activation=self.output_activation, dropout_rates=net_dropout,
                             batch_norm=batch_norm)
        self._finish(kwargs, learning_rate)

    def enable_sharding(self, group, batch_local, matrix_width, idx_dtype=torch.float64, want_fm=False):
        """RankModel.enable_sharding without the FM term, which BST does not have."""
        if want_fm:
            raise ValueError("BST has no FM term: enable_sharding(..., want_fm=False)")
        return super(BST, self).enable_sharding(group, batch_local, matrix_width, idx_dtype=idx_dtype, want_fm=False)

    def _logit_mlp(self):
        """dnn without its output Sigmoid (the same modules, not registered a second time)."""
        ent = self.__dict__.get("_logit_dnn")
        if ent is None:
            ent = MLP_Block.__new__(MLP_Block)
            nn.Module.__init__(ent)
            mods = list(self.dnn.mlp)
            ent.mlp = nn.Sequential(*(mods[:-1] if type(mods[-1]) == nn.Sigmoid else mods))
            self.__dict__["_logit_dnn"] = ent
        return ent

    def dnn_input(self, inputs):
        """The DNN's input (B, width): the embeddings left after the sequence fields are dropped, in FeatureMap order,
        then each pair's pooled transformer output."""
        X = self.get_inputs(inputs)
        front = getattr(self, "_sharded_front", None)
        if front is not None:       # row-sharded tables: (B, D) / (B, L, D) views of the landed rows
            from .sharded import sharded_front
            landed, _ = sharded_front(front, self._batch_matrix(inputs))
            views = front.field_views(landed)
            emb = OrderedDict((name, views[name]) for name in self.feature_map.features.keys() if name in views)
        else:
            emb = self.embedding_layer(X)
        pooled = []
        for enc, target, sequence in zip(self.transformer_encoders, self.bst_target_field, self.bst_sequence_field):
            tnames, snames = list(_flatten([target])), list(_flatten([sequence]))
            valid = torch.ne(X[snames[0]], 0).to(torch.uint8)
            B, L = valid.shape[0], valid.shape[1] + 1
            out = enc.run([emb[n] for n in snames], [emb[n] for n in tnames], valid, causal=self.use_causal_mask)
            pooled.append(F2.bst_pooling(out, valid, B, L, self.seq_pooling_type))
        for sequence in self.bst_sequence_field:
            for name in _flatten([sequence]):
                emb.pop(name, None)
        return torch.cat(list(emb.values()) + pooled, dim=-1)

    def forward_logits(self, inputs):
        return (self._logit_mlp()(self.dnn_input(inputs)),)

    def forward(self, inputs):
        return {"y_pred": self.output_activation(self.forward_logits(inputs)[0])}


class DIEN(RankModel):
    """model_zoo/DIEN/src/DIEN.py, DIEN: per (target, sequence) field pair (a tuple of fields: their embeddings side by
    side) an interest extractor GRU over the history, then the interest-evolution GRU: an AUGRU or AGRU (DynamicGRU)
    driven by AttentionLayer's scores against the target, or an nn.GRU.  Its last state, then (enable_sum_pooling) the
    sequence's sum pooling and its product with the target, join the remaining 2-D embeddings in FeatureMap order
    (the neg-sequence fields left out) as the DNN's input.  A sample's length is the number of non-zero ids of its
    pair's first sequence field, and the attention mask is id > 0 position by position, as in the reference; an empty
    history gives a zero state.  The lengths are formed on the device: no row compaction, no host sync, so the step can
    be captured in a CUDA graph.  The extractor and a gru_type="GRU" evolution keep real nn.GRU children, which hold
    the weights; their forward is never called.  Unknown keyword arguments are accepted and ignored.
    Refused: gru_type="AIGRU" and aux_loss_alpha > 0 (both fail in the reference), a DNN input whose width the
    reference's formula gets wrong, din_attention with Dice, shapes outside functional.dien_bound, lazy tables and
    enable_sharding(want_fm=True)."""
    _routes_sharded_front = True

    def __init__(self, feature_map, model_id="DIEN", gpu=-1, dnn_hidden_units=[200, 80], dnn_activations="ReLU",
                 learning_rate=1e-3, embedding_dim=16, net_dropout=0, batch_norm=True,
                 dien_target_field=[("item_id", "cate_id")], dien_sequence_field=[("click_history", "cate_history")],
                 dien_neg_seq_field=[("neg_click_history", "neg_cate_history")], gru_type="AUGRU",
                 enable_sum_pooling=False, attention_dropout=0, attention_type="bilinear_attention",
                 attention_hidden_units=[80, 40], attention_activation="Dice", use_attention_softmax=True,
                 aux_hidden_units=[100, 50], aux_activation="ReLU", aux_loss_alpha=0, embedding_regularizer=None,
                 net_regularizer=None, **kwargs):
        # a tuple of fields may arrive as a list (a JSON or YAML config)
        as_list = lambda v: [tuple(f) if isinstance(f, list) else f for f in (v if isinstance(v, list) else [v])]  # noqa
        targets, sequences, negs = as_list(dien_target_field), as_list(dien_sequence_field), as_list(dien_neg_seq_field)
        assert len(targets) == len(sequences), "dien_sequence_field or dien_target_field not supported."
        if gru_type == "AIGRU":
            raise NotImplementedError("DIEN gru_type='AIGRU' is not supported: the reference fails in "
                                      "interest_emb * attn_scores, a (B, L, H) x (B, L) broadcast")
        if gru_type not in ("GRU", "AGRU", "AUGRU"):
            raise ValueError("DIEN gru_type={} is not supported.".format(gru_type))
        if aux_loss_alpha > 0:
            raise NotImplementedError("DIEN aux_loss_alpha > 0 is not supported: the reference fails in add_loss, "
                                      "where loss += alpha * aux_loss adds an (N,) vector in place into a 0-d tensor")
        if gru_type != "GRU" and attention_type == "din_attention" and \
                any(str(a).lower() == "dice" for a in as_list(attention_activation)):
            raise NotImplementedError("DIEN din_attention with Dice is not supported: the reference takes Dice's "
                                      "batch statistics over the rows of non-empty histories only")
        specs = feature_map.features
        dims = []
        for target, sequence in zip(targets, sequences):
            names = list(_flatten([sequence]))
            model_dim = embedding_dim * len(list(_flatten([target])))
            bound = F2.dien_bound(model_dim, int(specs[names[0]]["max_len"]))
            if bound is not None:
                raise NotImplementedError("DIEN kernels: " + bound)
            dims.append(model_dim)
        neg_names = list(_flatten(negs))
        ref_width = 2 * sum(dims) + feature_map.sum_emb_out_dim() - embedding_dim * len(neg_names)
        if not enable_sum_pooling:
            ref_width -= embedding_dim * len(list(_flatten(targets))) * 2
        dflt = feature_map.default_emb_dim
        width = sum(dims) * (3 if enable_sum_pooling else 1) + sum(
            spec.get("emb_output_dim", spec.get("embedding_dim", dflt)) for name, spec in specs.items()
            if spec["type"] not in ("sequence", "meta") or (spec["type"] == "sequence" and spec.get("feature_encoder")))
        if width != ref_width:
            raise NotImplementedError("DIEN: the reference sizes the DNN input as %d but feeds it %d values (neg-sequence "
                                      "fields not in the feature map, or sequence fields outside the pairs)"
                                      % (ref_width, width))
        super(DIEN, self).__init__(feature_map, model_id=model_id, gpu=gpu,
                                   embedding_regularizer=embedding_regularizer, net_regularizer=net_regularizer,
                                   **kwargs)
        self.dien_target_field, self.dien_sequence_field = targets, sequences
        self.aux_loss_alpha = aux_loss_alpha
        self.dien_neg_seq_field = negs
        self.embedding_dim = embedding_dim
        self.embedding_layer = FeatureEmbeddingDict(feature_map, embedding_dim)
        self.sum_pooling = MaskedSumPooling()
        self.gru_type = gru_type
        self.extraction_modules = nn.ModuleList()
        self.evolving_modules = nn.ModuleList()
        self.attention_modules = nn.ModuleList()
        for model_dim in dims:
            self.extraction_modules.append(nn.GRU(input_size=model_dim, hidden_size=model_dim, batch_first=True))
            if gru_type in ("AGRU", "AUGRU"):
                self.evolving_modules.append(DynamicGRU(model_dim, model_dim, gru_type=gru_type))
            else:
                self.evolving_modules.append(nn.GRU(input_size=model_dim, hidden_size=model_dim, batch_first=True))
            if gru_type in ("AGRU", "AUGRU"):
                self.attention_modules.append(
                    AttentionLayer(model_dim, attention_type=attention_type,
                                   attention_hidden_units=attention_hidden_units,
                                   attention_activation=attention_activation,
                                   use_attention_softmax=use_attention_softmax, attention_dropout=attention_dropout))
        self.enable_sum_pooling = enable_sum_pooling
        self.dnn = MLP_Block(input_dim=width, output_dim=1, hidden_units=dnn_hidden_units,
                             hidden_activations=dnn_activations, output_activation=self.output_activation,
                             dropout_rates=net_dropout, batch_norm=batch_norm)
        self._finish(kwargs, learning_rate)

    def enable_sharding(self, group, batch_local, matrix_width, idx_dtype=torch.float64, want_fm=False):
        """RankModel.enable_sharding without the FM term, which DIEN does not have."""
        if want_fm:
            raise ValueError("DIEN has no FM term: enable_sharding(..., want_fm=False)")
        return super(DIEN, self).enable_sharding(group, batch_local, matrix_width, idx_dtype=idx_dtype, want_fm=False)

    def _logit_mlp(self):
        """dnn without its output Sigmoid (the same modules, not registered a second time)."""
        ent = self.__dict__.get("_logit_dnn")
        if ent is None:
            ent = MLP_Block.__new__(MLP_Block)
            nn.Module.__init__(ent)
            mods = list(self.dnn.mlp)
            ent.mlp = nn.Sequential(*(mods[:-1] if type(mods[-1]) == nn.Sigmoid else mods))
            self.__dict__["_logit_dnn"] = ent
        return ent

    @staticmethod
    def get_embedding(field, emb):
        """A tuple of fields means their embeddings side by side (DIEN.get_embedding)."""
        parts = [emb[name] for name in (field if type(field) == tuple else (field,))]
        return parts[0] if len(parts) == 1 else torch.cat(parts, dim=-1)

    def interest(self, k, sequence_emb, target_emb, mask):
        """h_out (B, H) of pair k: the extractor GRU, the attention and the evolution GRU.  The interests' gradient is
        one buffer that the attention and the evolution GRU add into (functional.shared_grad)."""
        ext, evo = self.extraction_modules[k], self.evolving_modules[k]
        h_seq, _ = F2.gru_sequence(sequence_emb, mask, ext.weight_ih_l0, ext.bias_ih_l0, ext.weight_hh_l0,
                                   ext.bias_hh_l0)
        interest, sink = F2.shared_grad(h_seq)
        if self.gru_type == "GRU":
            return F2.gru_sequence(interest, mask, evo.weight_ih_l0, evo.bias_ih_l0, evo.weight_hh_l0,
                                   evo.bias_hh_l0, sink=sink)[1]
        scores = self.attention_modules[k].run(interest, target_emb, mask, sink=sink)
        return evo.run(interest, mask, scores, sink=sink)

    def dnn_input(self, inputs):
        X = self.get_inputs(inputs)
        front = getattr(self, "_sharded_front", None)
        if front is not None:       # row-sharded tables: (B, D) / (B, L, D) views of the landed rows
            from .sharded import sharded_front
            landed, _ = sharded_front(front, self._batch_matrix(inputs))
            views = front.field_views(landed)
            emb = OrderedDict((name, views[name]) for name in self.feature_map.features.keys() if name in views)
        else:
            emb = self.embedding_layer(X)
        parts = []
        for k, (target, sequence) in enumerate(zip(self.dien_target_field, self.dien_sequence_field)):
            target_emb = self.get_embedding(target, emb)
            sequence_emb = self.get_embedding(sequence, emb)
            mask = torch.ne(X[list(_flatten([sequence]))[0]], 0).to(torch.uint8)
            parts.append(self.interest(k, sequence_emb, target_emb, mask))
            if self.enable_sum_pooling:
                parts.append(F2.dien_sum_pool(sequence_emb, target_emb))
        negs = set(_flatten(self.dien_neg_seq_field))
        parts += [e for name, e in emb.items() if e.dim() == 2 and name not in negs]
        return torch.cat(parts, dim=-1)

    def forward_logits(self, inputs):
        return (self._logit_mlp()(self.dnn_input(inputs)),)

    def forward(self, inputs):
        return {"y_pred": self.output_activation(self.forward_logits(inputs)[0])}


class TransAct(RankModel):
    """model_zoo/TransAct/src/TransAct.py, TransAct: per (target, sequence) field pair (a tuple of fields: their
    embeddings side by side) a TransActTransformer over the L = max_len early-fusion tokens [sequence | target], whose
    output [last first_k_cols slots | out_linear(max over L)] replaces the pair's sequence fields; then DCNv2's parallel
    structure, mlp(cat([CrossNetV2(x), parallel_dnn(x)])), on x = [remaining embeddings in FeatureMap order | the
    transformer outputs in pair order].  The key-padding mask comes from the first sequence field's ids (0 = padding);
    an empty history keeps its last slot.  Unknown keyword arguments are accepted and ignored, as the reference's
    **kwargs are.  Refused: shapes outside functional.transact_bound, md % num_heads != 0 (the reference's assert),
    use_time_window_mask=True and first_k_cols outside [1, max_len] (neither trains in the reference), a DCN input
    whose width the reference's formula gets wrong, lazy tables and enable_sharding(want_fm=True)."""
    _routes_sharded_front = True

    def __init__(self, feature_map, model_id="TransAct", gpu=-1, hidden_activations="ReLU", dcn_cross_layers=3,
                 dcn_hidden_units=[256, 128, 64], mlp_hidden_units=[], num_heads=1, transformer_layers=1,
                 transformer_dropout=0, dim_feedforward=512, learning_rate=1e-3, embedding_dim=64, net_dropout=0,
                 batch_norm=False, target_item_field=[("item_id", "cate_id")],
                 sequence_item_field=[("click_history", "cate_history")], first_k_cols=1, use_time_window_mask=False,
                 time_window_ms=86400000, concat_max_pool=True, embedding_regularizer=None, net_regularizer=None,
                 **kwargs):
        # a tuple of fields may arrive as a list (a JSON or YAML config)
        as_list = lambda v: [tuple(f) if isinstance(f, list) else f for f in (v if isinstance(v, list) else [v])]  # noqa
        targets, sequences = as_list(target_item_field), as_list(sequence_item_field)
        if use_time_window_mask:
            raise NotImplementedError("TransAct use_time_window_mask=True is not supported: the reference's forward "
                                      "never passes time_interval_seq, so its mask compares None with an int")
        specs = feature_map.features
        dims, width = [], feature_map.sum_emb_out_dim()
        for sequence, target in zip(sequences, targets):
            snames, tnames = list(_flatten([sequence])), list(_flatten([target]))
            md = embedding_dim * (len(snames) + len(tnames))
            L = int(specs[snames[0]]["max_len"])
            if not 1 <= first_k_cols <= L:
                raise NotImplementedError("TransAct first_k_cols=%d is not supported: it must lie in [1, max_len = %d] "
                                          "(the reference sizes its output for first_k_cols slots but takes at most "
                                          "max_len)" % (first_k_cols, L))
            assert md % num_heads == 0, "embed_dim must be divisible by num_heads"
            bound = F2.transact_bound(L, md, num_heads, len(snames) + len(tnames))
            if bound is not None:
                raise NotImplementedError("TransAct kernels: " + bound)
            dims.append(md)
            width += (first_k_cols + int(concat_max_pool)) * md - embedding_dim * len(snames)
        names = list(_flatten(sequences))
        if len(set(names)) != len(names) or any(specs[f]["type"] != "sequence" for f in names):
            raise NotImplementedError("TransAct: every sequence field must be a sequence feature of one pair only (the "
                                      "reference sizes the DCN input for each pair's fields but pops each once)")
        super(TransAct, self).__init__(feature_map, model_id=model_id, gpu=gpu,
                                       embedding_regularizer=embedding_regularizer, net_regularizer=net_regularizer,
                                       **kwargs)
        self.target_item_field, self.sequence_item_field = targets, sequences
        self.feature_map = feature_map
        self.embedding_dim = embedding_dim
        self.embedding_layer = FeatureEmbeddingDict(feature_map, embedding_dim)
        self.transformer_encoders = nn.ModuleList()
        for md in dims:
            self.transformer_encoders.append(
                TransActTransformer(md, dim_feedforward=dim_feedforward, num_heads=num_heads,
                                    dropout=transformer_dropout, transformer_layers=transformer_layers,
                                    use_time_window_mask=use_time_window_mask, time_window_ms=time_window_ms,
                                    first_k_cols=first_k_cols, concat_max_pool=concat_max_pool))
        self.crossnet = CrossNetV2(width, dcn_cross_layers)
        self.parallel_dnn = MLP_Block(input_dim=width, output_dim=None, hidden_units=dcn_hidden_units,
                                      hidden_activations=hidden_activations, output_activation=None,
                                      dropout_rates=net_dropout, batch_norm=batch_norm)
        self.mlp = MLP_Block(input_dim=width + dcn_hidden_units[-1], output_dim=1, hidden_units=mlp_hidden_units,
                             hidden_activations=hidden_activations, output_activation=self.output_activation)
        self._finish(kwargs, learning_rate)

    def enable_sharding(self, group, batch_local, matrix_width, idx_dtype=torch.float64, want_fm=False):
        """RankModel.enable_sharding without the FM term, which TransAct does not have."""
        if want_fm:
            raise ValueError("TransAct has no FM term: enable_sharding(..., want_fm=False)")
        return super(TransAct, self).enable_sharding(group, batch_local, matrix_width, idx_dtype=idx_dtype,
                                                     want_fm=False)

    def _logit_mlp(self):
        """mlp without its output Sigmoid (the same modules, not registered a second time)."""
        ent = self.__dict__.get("_logit_head")
        if ent is None:
            ent = MLP_Block.__new__(MLP_Block)
            nn.Module.__init__(ent)
            mods = list(self.mlp.mlp)
            ent.mlp = nn.Sequential(*(mods[:-1] if type(mods[-1]) == nn.Sigmoid else mods))
            self.__dict__["_logit_head"] = ent
        return ent

    def dcn_input(self, inputs):
        """The DCN input (B, width): the embeddings left after the sequence fields are dropped, in FeatureMap order,
        then each pair's transformer output."""
        X = self.get_inputs(inputs)
        front = getattr(self, "_sharded_front", None)
        if front is not None:       # row-sharded tables: (B, D) / (B, L, D) views of the landed rows
            from .sharded import sharded_front
            landed, _ = sharded_front(front, self._batch_matrix(inputs))
            views = front.field_views(landed)
            emb = OrderedDict((name, views[name]) for name in self.feature_map.features.keys() if name in views)
        else:
            emb = self.embedding_layer(X)
        outs = []
        for enc, target, sequence in zip(self.transformer_encoders, self.target_item_field, self.sequence_item_field):
            tnames, snames = list(_flatten([target])), list(_flatten([sequence]))
            outs.append(enc.run([emb[n] for n in snames], [emb[n] for n in tnames], X[snames[0]]))
        for name in _flatten(self.sequence_item_field):
            if self.feature_map.features[name]["type"] == "sequence":
                emb.pop(name, None)
        return torch.cat(list(emb.values()) + outs, dim=-1)

    def forward_logits(self, inputs):
        x = self.dcn_input(inputs)
        return (self._logit_mlp()(torch.cat([self.crossnet(x), self.parallel_dnn(x)], dim=-1)),)

    def forward(self, inputs):
        return {"y_pred": self.output_activation(self.forward_logits(inputs)[0])}


class _LongCTRModel(RankModel):
    """What ETA and SDIM share: the LongCTR input triple (batch_dict, item_dict, mask) of the reference's
    LongCTRDataLoader, the item embeddings `embedding_layer(item_dict, flatten_emb=True)` viewed as (B, L + 1, d) with
    the target last, and a DNN over [batch embeddings, target, interests].  d = item_info_dim is the sum of the
    embedding dims of the features with source "item".  Refused: attention_dropout > 0 (the target-attention kernels
    have none), short_seq_len < 2, accumulation_steps != 1, a batch with L = 0 or L < short_seq_len (the reference's
    embedding and mask windows then differ in length), a DNN input whose width is not the reference's
    sum_emb_out_dim() + 2 item_info_dim, lazy tables and enable_sharding()."""

    def _longctr_init(self, feature_map, embedding_dim, short_seq_len, attention_dropout, accumulation_steps):
        if attention_dropout:
            raise NotImplementedError("%s: attention_dropout > 0 is not supported: the target-attention kernels have "
                                      "no dropout" % type(self).__name__)
        if short_seq_len < 2:
            raise ValueError("%s: short_seq_len must be at least 2 (the window [-short_seq_len:-1] would be empty), "
                             "got %d" % (type(self).__name__, short_seq_len))
        if accumulation_steps != 1:
            raise NotImplementedError("%s: accumulation_steps != 1 is not supported: every step updates the weights"
                                      % type(self).__name__)
        self.feature_map = feature_map
        self.embedding_dim = embedding_dim
        self.short_seq_len = short_seq_len
        self.accumulation_steps = accumulation_steps
        self.item_info_dim = 0
        for feat, spec in feature_map.features.items():
            if spec.get("source") == "item":
                self.item_info_dim += spec.get("embedding_dim", embedding_dim)

    def get_inputs(self, inputs, feature_source=None):
        """(X_dict, item_dict, mask) on the model's device (ETA.py / SDIM.py get_inputs)."""
        batch_dict, item_dict, mask = inputs
        X_dict = dict()
        for feature, value in batch_dict.items():
            if feature in self.feature_map.labels:
                continue
            feature_spec = self.feature_map.features[feature]
            if feature_spec["type"] == "meta":
                continue
            if feature_source and not_in_whitelist(feature_spec["source"], feature_source):
                continue
            X_dict[feature] = value.to(self.device)
        for item, value in item_dict.items():
            item_dict[item] = value.to(self.device)
        return X_dict, item_dict, mask.to(self.device)

    def get_labels(self, inputs):
        y = inputs[0][self.feature_map.labels[0]].to(self.device)
        return y.float().view(-1, 1)

    def get_group_id(self, inputs):
        return inputs[0][self.feature_map.group_id]

    def _logit_mlp(self, name="dnn"):
        """The MLP_Block `name` without its output Sigmoid (the same modules, not registered a second time)."""
        ent = self.__dict__.get("_logit_" + name)
        if ent is None:
            ent = MLP_Block.__new__(MLP_Block)
            nn.Module.__init__(ent)
            mods = list(getattr(self, name).mlp)
            ent.mlp = nn.Sequential(*(mods[:-1] if type(mods[-1]) == nn.Sigmoid else mods))
            self.__dict__["_logit_" + name] = ent
        return ent

    def _item_inputs(self, inputs):
        """(batch embeddings or None, item_feat_emb (B, L + 1, d), mask (B, L)); checks the DNN width."""
        batch_dict, item_dict, mask = self.get_inputs(inputs)
        emb_out = self.embedding_layer(batch_dict, flatten_emb=True) if batch_dict else None
        if mask.dim() != 2 or mask.shape[1] == 0:
            raise ValueError("%s: mask%s must be (B, L) with L >= 1" % (type(self).__name__, tuple(mask.shape)))
        B, L = mask.shape
        item_feat_emb = self.embedding_layer(item_dict, flatten_emb=True)
        if item_feat_emb.shape[-1] != self.item_info_dim or item_feat_emb.numel() != B * (L + 1) * self.item_info_dim:
            raise ValueError("%s: item_dict gives %s embeddings, expected B (L + 1) = %d rows of item_info_dim = %d"
                             % (type(self).__name__, tuple(item_feat_emb.shape), B * (L + 1), self.item_info_dim))
        width = (0 if emb_out is None else emb_out.shape[-1]) + 3 * self.item_info_dim
        ref_width = self.feature_map.sum_emb_out_dim() + 2 * self.item_info_dim
        if width != ref_width:
            raise NotImplementedError("%s: the reference sizes the DNN input as sum_emb_out_dim() + 2 item_info_dim = "
                                      "%d but this batch gives it %d values (item features in batch_dict, or a "
                                      "feature in neither dict)" % (type(self).__name__, ref_width, width))
        return emb_out, item_feat_emb.view(B, L + 1, self.item_info_dim), mask

    def forward_logits(self, inputs):
        return (self._logit_mlp()(self.dnn_input(inputs)),)

    def forward(self, inputs):
        return {"y_pred": self.output_activation(self.forward_logits(inputs)[0])}


class ETA(_LongCTRModel):
    """model_zoo/LongCTR/ETA/ETA.py, ETA: a short target attention over the last short_seq_len - 1 history items, and
    a long one over the topk history items nearest the target in SimHash Hamming distance; the DNN reads [batch
    embeddings, target, short, long].  The interest block is one autograd node on the kernels (functional.eta_interest);
    ties at equal distance go to the lower history position.  reuse_hash=False draws (B, d, hash_bits) rotations with
    torch.randn on the device every forward, as the reference does.  The frozen random_rotations stay outside the
    optimizer.  Unknown keyword arguments are accepted and ignored.  Refusals: see _LongCTRModel, and shapes outside
    functional.eta_bound."""

    def __init__(self, feature_map, model_id="ETA", gpu=-1, dnn_hidden_units=[512, 128, 64], dnn_activations="ReLU",
                 attention_dim=64, num_heads=1, use_scale=True, attention_dropout=0, reuse_hash=True, hash_bits=32,
                 topk=50, learning_rate=1e-3, embedding_dim=10, net_dropout=0, batch_norm=False, short_seq_len=50,
                 accumulation_steps=1, embedding_regularizer=None, net_regularizer=None, **kwargs):
        super(ETA, self).__init__(feature_map, model_id=model_id, gpu=gpu, embedding_regularizer=embedding_regularizer,
                                  net_regularizer=net_regularizer, **kwargs)
        self._longctr_init(feature_map, embedding_dim, short_seq_len, attention_dropout, accumulation_steps)
        bound = F2.eta_bound(self.item_info_dim, 1, topk, hash_bits)
        if bound is not None:
            raise NotImplementedError("ETA kernels: " + bound)
        self.reuse_hash = reuse_hash
        self.hash_bits = hash_bits
        self.topk = topk
        self.embedding_layer = FeatureEmbedding(feature_map, embedding_dim)
        self.short_attention = MultiHeadTargetAttention(self.item_info_dim, attention_dim, num_heads,
                                                        attention_dropout, use_scale)
        self.random_rotations = nn.Parameter(torch.randn(1, self.item_info_dim, self.hash_bits), requires_grad=False)
        self.long_attention = MultiHeadTargetAttention(self.item_info_dim, attention_dim, num_heads,
                                                       attention_dropout, use_scale)
        input_dim = feature_map.sum_emb_out_dim() + self.item_info_dim * 2
        self.dnn = MLP_Block(input_dim=input_dim, output_dim=1, hidden_units=dnn_hidden_units,
                             hidden_activations=dnn_activations, output_activation=self.output_activation,
                             dropout_rates=net_dropout, batch_norm=batch_norm)
        self._finish(kwargs, learning_rate)

    def interest(self, item_feat_emb, mask):
        """(target, short, long, positions) of functional.eta_interest."""
        if self.reuse_hash:
            rotations = self.random_rotations
        else:
            rotations = torch.randn(item_feat_emb.size(0), self.item_info_dim, self.hash_bits,
                                    device=item_feat_emb.device)
        sa, la = self.short_attention, self.long_attention
        return F2.eta_interest(item_feat_emb, mask, rotations, self.short_seq_len, self.topk, sa.num_heads,
                               sa.scale is not None, (sa.W_q.weight, sa.W_k.weight, sa.W_v.weight, sa.W_o.weight),
                               (la.W_q.weight, la.W_k.weight, la.W_v.weight, la.W_o.weight))

    def dnn_input(self, inputs):
        emb_out, item_feat_emb, mask = self._item_inputs(inputs)
        target, short, long, _ = self.interest(item_feat_emb, mask)
        return torch.cat(([emb_out] if emb_out is not None else []) + [target, short, long], dim=-1)


class SDIM(_LongCTRModel):
    """model_zoo/LongCTR/SDIM/SDIM.py, SDIM: a short target attention over the last short_seq_len - 1 history items, and
    the long interest as the mean over num_hashes SimHash hashes of the sum of the history items whose bucket matches
    the target's (each sum L2-normalised with l2_norm); the DNN reads [batch embeddings, target, long, short].  The
    interest block is one autograd node on the kernels (functional.sdim_interest), with no torch.nonzero, so the step
    never waits for the host.  reuse_hash=False draws (B, d, num_hashes, hash_bits) rotations with torch.randn on the
    device every forward.  The frozen powers_of_two and random_rotations stay outside the optimizer.  Unknown keyword
    arguments are accepted and ignored.  Refusals: see _LongCTRModel, and shapes outside functional.sdim_bound
    (hash_bits > 24 among them)."""

    def __init__(self, feature_map, model_id="SDIM", gpu=-1, dnn_hidden_units=[512, 128, 64], dnn_activations="ReLU",
                 attention_dim=64, use_qkvo=True, num_heads=1, use_scale=True, attention_dropout=0, reuse_hash=True,
                 num_hashes=1, hash_bits=4, learning_rate=1e-3, embedding_dim=10, net_dropout=0, batch_norm=False,
                 l2_norm=False, short_seq_len=50, accumulation_steps=1, embedding_regularizer=None,
                 net_regularizer=None, **kwargs):
        super(SDIM, self).__init__(feature_map, model_id=model_id, gpu=gpu, embedding_regularizer=embedding_regularizer,
                                   net_regularizer=net_regularizer, **kwargs)
        self._longctr_init(feature_map, embedding_dim, short_seq_len, attention_dropout, accumulation_steps)
        bound = F2.sdim_bound(self.item_info_dim, 1, num_hashes, hash_bits)
        if bound is not None:
            raise NotImplementedError("SDIM kernels: " + bound)
        self.reuse_hash = reuse_hash
        self.num_hashes = num_hashes
        self.hash_bits = hash_bits
        self.l2_norm = l2_norm
        self.powers_of_two = nn.Parameter(torch.tensor([2.0 ** i for i in range(hash_bits)]), requires_grad=False)
        self.embedding_layer = FeatureEmbedding(feature_map, embedding_dim)
        self.short_attention = MultiHeadTargetAttention(self.item_info_dim, attention_dim, num_heads,
                                                        attention_dropout, use_scale, use_qkvo)
        self.random_rotations = nn.Parameter(torch.randn(1, self.item_info_dim, self.num_hashes, self.hash_bits),
                                             requires_grad=False)
        input_dim = feature_map.sum_emb_out_dim() + self.item_info_dim * 2
        self.dnn = MLP_Block(input_dim=input_dim, output_dim=1, hidden_units=dnn_hidden_units,
                             hidden_activations=dnn_activations, output_activation=self.output_activation,
                             dropout_rates=net_dropout, batch_norm=batch_norm)
        self._finish(kwargs, learning_rate)

    def interest(self, item_feat_emb, mask):
        """(target, short, long) of functional.sdim_interest."""
        if self.reuse_hash:
            rotations = self.random_rotations
        else:
            rotations = torch.randn(item_feat_emb.size(0), self.item_info_dim, self.num_hashes, self.hash_bits,
                                    device=item_feat_emb.device)
        sa = self.short_attention
        weights = (sa.W_q.weight, sa.W_k.weight, sa.W_v.weight, sa.W_o.weight) if sa.use_qkvo else ()
        return F2.sdim_interest(item_feat_emb, mask, rotations, self.short_seq_len, self.l2_norm, sa.num_heads,
                                sa.scale is not None, weights)

    def dnn_input(self, inputs):
        emb_out, item_feat_emb, mask = self._item_inputs(inputs)
        target, short, long = self.interest(item_feat_emb, mask)
        return torch.cat(([emb_out] if emb_out is not None else []) + [target, long, short], dim=-1)


def _mhta_weights(att):
    return att.W_q.weight, att.W_k.weight, att.W_v.weight, att.W_o.weight


def _check_heads(name, attention_dim, num_heads):
    if num_heads < 1 or attention_dim % num_heads:
        raise ValueError("%s: attention_dim=%d is not divisible by num_heads=%d" % (name, attention_dim, num_heads))


class SIM(_LongCTRModel):
    """model_zoo/LongCTR/SIM/SIM.py, SIM: a short target attention over the last short_seq_len - 1 history items; a
    soft-search GSU that scores every history row as qk_l = (W_a t) . (W_b x_l) mask_l, pools the history with those
    scores into an auxiliary DNN over [batch embeddings, target, pooled], and keeps the topk best rows for a long target
    attention; the main DNN reads [batch embeddings, target, short, long].  forward returns {"y_pred", "y_aux"} and the
    loss is alpha BCE(y_aux) + beta BCE(y_pred).  The interest block is one autograd node on the kernels
    (functional.sim_interest).  Masked positions score 0, as in the reference, so they outrank negatively scored valid
    rows; ties go to the lower history position.  Unknown keyword arguments are accepted and ignored.  Refusals:
    gsu_type != "soft" (the reference asserts), attention_dim not divisible by num_heads, see _LongCTRModel, and shapes
    outside functional.sim_bound."""

    def __init__(self, feature_map, model_id="SIM", gpu=-1, dnn_hidden_units=[512, 128, 64], dnn_activations="ReLU",
                 attention_dropout=0, attention_dim=64, num_heads=1, gsu_type="soft", short_seq_len=50, topk=50,
                 alpha=1, beta=1, learning_rate=1e-3, embedding_dim=10, net_dropout=0, batch_norm=False,
                 accumulation_steps=1, embedding_regularizer=None, net_regularizer=None, **kwargs):
        super(SIM, self).__init__(feature_map, model_id=model_id, gpu=gpu, embedding_regularizer=embedding_regularizer,
                                  net_regularizer=net_regularizer, **kwargs)
        if gsu_type != "soft":
            raise NotImplementedError("SIM: gsu_type=%r is not supported: only the soft search exists (the reference "
                                      "asserts gsu_type == 'soft')" % (gsu_type,))
        self._longctr_init(feature_map, embedding_dim, short_seq_len, attention_dropout, accumulation_steps)
        _check_heads("SIM", attention_dim, num_heads)
        bound = F2.sim_bound(self.item_info_dim, 1, topk, num_heads)
        if bound is not None:
            raise NotImplementedError("SIM kernels: " + bound)
        self.topk = topk
        self.alpha = alpha
        self.beta = beta
        self.embedding_layer = FeatureEmbedding(feature_map, embedding_dim)
        self.W_a = nn.Linear(self.item_info_dim, attention_dim, bias=False)
        self.W_b = nn.Linear(self.item_info_dim, attention_dim, bias=False)
        self.short_attention = MultiHeadTargetAttention(self.item_info_dim, attention_dim, num_heads,
                                                        attention_dropout)
        self.long_attention = MultiHeadTargetAttention(self.item_info_dim, attention_dim, num_heads,
                                                       attention_dropout)
        input_dim = feature_map.sum_emb_out_dim() + self.item_info_dim
        self.dnn_aux = MLP_Block(input_dim=input_dim, output_dim=1, hidden_units=dnn_hidden_units,
                                 hidden_activations=dnn_activations, output_activation=self.output_activation,
                                 dropout_rates=net_dropout, batch_norm=batch_norm)
        input_dim = feature_map.sum_emb_out_dim() + self.item_info_dim * 2
        self.dnn = MLP_Block(input_dim=input_dim, output_dim=1, hidden_units=dnn_hidden_units,
                             hidden_activations=dnn_activations, output_activation=self.output_activation,
                             dropout_rates=net_dropout, batch_norm=batch_norm)
        self._finish(kwargs, learning_rate)

    def interest(self, item_feat_emb, mask):
        """(target, short, long, pooled, positions) of functional.sim_interest."""
        return F2.sim_interest(item_feat_emb, mask, self.short_seq_len, self.topk, self.short_attention.num_heads,
                               self.W_a.weight, self.W_b.weight, _mhta_weights(self.short_attention),
                               _mhta_weights(self.long_attention))

    def _logits(self, inputs):
        """(main logit, auxiliary logit), each (B, 1) before the output Sigmoid."""
        emb_out, item_feat_emb, mask = self._item_inputs(inputs)
        target, short, long, pooled, _ = self.interest(item_feat_emb, mask)
        emb = [emb_out] if emb_out is not None else []
        y = self._logit_mlp()(torch.cat(emb + [target, short, long], dim=-1))
        y_aux = self._logit_mlp("dnn_aux")(torch.cat(emb + [target, pooled], dim=-1))
        return y, y_aux

    def forward_logits(self, inputs):
        return (self._logits(inputs)[0],)

    def forward(self, inputs):
        y, y_aux = self._logits(inputs)
        return {"y_pred": self.output_activation(y), "y_aux": self.output_activation(y_aux)}

    def compute_loss(self, return_dict, y_true):
        loss_gsu = self.loss_fn(return_dict["y_aux"], y_true, reduction="mean")
        loss_esu = self.loss_fn(return_dict["y_pred"], y_true, reduction="mean")
        return self.alpha * loss_gsu + self.beta * loss_esu + self.regularization_loss()

    def fused_loss(self, batch_data, y_true):
        y, y_aux = self._logits(batch_data)
        return self.alpha * F2.logit_bce(y_true, y_aux)[0] + self.beta * F2.logit_bce(y_true, y)[0]


class TWIN(_LongCTRModel):
    """model_zoo/LongCTR/TWIN/TWIN.py, TWIN: a short target attention over the last short_seq_len - 1 history items,
    and MultiHeadTopKAttention over the whole history: per head the topk best scores, softmaxed over those k; the DNN
    reads [batch embeddings, target, short, long].  The interest block is one autograd node on the kernels
    (functional.twin_interest); ties go to the lower history position.  Unknown keyword arguments are accepted and
    ignored.  Refusals: Kc_cross_features > 0 (the reference can only broadcast its cross features at L = 1),
    attention_dim not divisible by num_heads, see _LongCTRModel, and shapes outside functional.twin_bound."""

    def __init__(self, feature_map, model_id="TWIN", gpu=-1, dnn_hidden_units=[512, 128, 64], dnn_activations="ReLU",
                 attention_dropout=0, attention_dim=64, num_heads=1, short_seq_len=50, topk=50, Kc_cross_features=0,
                 learning_rate=1e-3, embedding_dim=10, net_dropout=0, batch_norm=False, accumulation_steps=1,
                 embedding_regularizer=None, net_regularizer=None, **kwargs):
        super(TWIN, self).__init__(feature_map, model_id=model_id, gpu=gpu, embedding_regularizer=embedding_regularizer,
                                   net_regularizer=net_regularizer, **kwargs)
        if Kc_cross_features > 0:
            raise NotImplementedError("TWIN: Kc_cross_features > 0 is not supported: the reference's "
                                      "cross_feat_seq.view(B, Kc, -1) * W_c broadcasts only at L = 1")
        self._longctr_init(feature_map, embedding_dim, short_seq_len, attention_dropout, accumulation_steps)
        _check_heads("TWIN", attention_dim, num_heads)
        bound = F2.twin_bound(self.item_info_dim, 1, topk, num_heads)
        if bound is not None:
            raise NotImplementedError("TWIN kernels: " + bound)
        self.topk = topk
        self.embedding_layer = FeatureEmbedding(feature_map, embedding_dim)
        self.short_attention = MultiHeadTargetAttention(self.item_info_dim, attention_dim, num_heads,
                                                        attention_dropout)
        self.long_attention = MultiHeadTopKAttention(self.item_info_dim, Kc_cross_features, embedding_dim,
                                                     attention_dim, topk, num_heads, attention_dropout)
        input_dim = feature_map.sum_emb_out_dim() + self.item_info_dim * 2
        self.dnn = MLP_Block(input_dim=input_dim, output_dim=1, hidden_units=dnn_hidden_units,
                             hidden_activations=dnn_activations, output_activation=self.output_activation,
                             dropout_rates=net_dropout, batch_norm=batch_norm)
        self._finish(kwargs, learning_rate)

    def interest(self, item_feat_emb, mask):
        """(target, short, long, positions) of functional.twin_interest."""
        return F2.twin_interest(item_feat_emb, mask, self.short_seq_len, self.topk, self.short_attention.num_heads,
                                _mhta_weights(self.short_attention), self.long_attention.weights())

    def dnn_input(self, inputs):
        emb_out, item_feat_emb, mask = self._item_inputs(inputs)
        target, short, long, _ = self.interest(item_feat_emb, mask)
        return torch.cat(([emb_out] if emb_out is not None else []) + [target, short, long], dim=-1)


class MIRRN(_LongCTRModel):
    """model_zoo/LongCTR/MIRRN/MIRRN.py, MIRRN: a short target attention over the last short_seq_len - 1 history items;
    three SimHash retrievals of the topk history items nearest the target, the masked mean of the last 16 items and
    the masked mean of the whole history, each kept in position order, shifted by 0.02 pos[L - idx], filtered by a
    FilterLayer2 and averaged over the k slots; a long target attention over those three interests; the DNN reads
    [batch embeddings, target, short, long].  The interest block is one autograd node on the kernels
    (functional.mirrn_interest); ties at equal distance go to the lower history position.  Each FilterLayer2's
    dropout (its own out_dropout.p, 0.1 as the reference hard-codes it) runs in training mode on the Philox masks.
    reuse_hash=False draws three (d, hash_bits) rotations with torch.randn on the device every forward, in the order
    target, short, global.  The frozen random_rotations stay outside the optimizer.  Unknown keyword arguments are
    accepted and ignored.
    Refusals: see _LongCTRModel, an item width not divisible by 4 (the reference fails at its first forward), a batch
    with L > max_len, and shapes outside functional.mirrn_bound."""

    def __init__(self, feature_map, model_id="MIRRN", gpu=-1, dnn_hidden_units=[512, 128, 64],
                 dnn_activations="ReLU", attention_dim=64, num_heads=1, use_scale=True, attention_dropout=0,
                 reuse_hash=True, hash_bits=32, topk=50, max_len=1000, learning_rate=1e-3, embedding_dim=10,
                 net_dropout=0, batch_norm=False, short_seq_len=50, accumulation_steps=1, embedding_regularizer=None,
                 net_regularizer=None, **kwargs):
        super(MIRRN, self).__init__(feature_map, model_id=model_id, gpu=gpu,
                                    embedding_regularizer=embedding_regularizer, net_regularizer=net_regularizer,
                                    **kwargs)
        self._longctr_init(feature_map, embedding_dim, short_seq_len, attention_dropout, accumulation_steps)
        if self.item_info_dim % 4:
            raise ValueError("MIRRN: item_info_dim = %d (the sum of the item features' embedding dims) must be "
                             "divisible by 4, FilterLayer2's block count; the reference fails at its first forward"
                             % self.item_info_dim)
        bound = F2.mirrn_bound(self.item_info_dim, 1, topk, hash_bits)
        if bound is not None:
            raise NotImplementedError("MIRRN kernels: " + bound)
        self.reuse_hash = reuse_hash
        self.hash_bits = hash_bits
        self.topk = topk
        self.max_len = max_len
        self.embedding_layer = FeatureEmbedding(feature_map, embedding_dim)
        self.short_attention = MultiHeadTargetAttention(self.item_info_dim, attention_dim, num_heads,
                                                        attention_dropout, use_scale)
        self.pos = nn.Embedding(max_len + 1, self.item_info_dim)
        self.random_rotations = nn.Parameter(torch.randn(self.item_info_dim, self.hash_bits), requires_grad=False)
        self.MHFT_block = nn.ModuleList([FilterLayer2(topk, self.item_info_dim, F2.MIRRN_FILTER_DROPOUT, 4)
                                         for _ in range(3)])
        self.long_attention = MultiHeadTargetAttention(self.item_info_dim, attention_dim, num_heads,
                                                       attention_dropout, use_scale)
        input_dim = feature_map.sum_emb_out_dim() + self.item_info_dim * 2
        self.dnn = MLP_Block(input_dim=input_dim, output_dim=1, hidden_units=dnn_hidden_units,
                             hidden_activations=dnn_activations, output_activation=self.output_activation,
                             dropout_rates=net_dropout, batch_norm=batch_norm)
        self._finish(kwargs, learning_rate)

    def interest(self, item_feat_emb, mask):
        """(target, short, long, positions) of functional.mirrn_interest."""
        if mask.shape[1] > self.max_len:
            raise ValueError("MIRRN: the history length L = %d exceeds max_len = %d (the reference's pos embedding "
                             "has rows 0 .. max_len)" % (mask.shape[1], self.max_len))
        if self.reuse_hash:
            rotations = self.random_rotations
        else:
            rotations = torch.stack([torch.randn(self.item_info_dim, self.hash_bits, device=item_feat_emb.device)
                                     for _ in range(3)])
        blocks = self.MHFT_block
        p = [b.out_dropout.p if self.training else 0.0 for b in blocks]
        return F2.mirrn_interest(item_feat_emb, mask, rotations, self.short_seq_len, self.topk,
                                 self.short_attention.num_heads, self.short_attention.scale is not None,
                                 _mhta_weights(self.short_attention), _mhta_weights(self.long_attention),
                                 self.pos.weight, [b.complex_weight for b in blocks],
                                 [b.LayerNorm.weight for b in blocks], [b.LayerNorm.bias for b in blocks], p)

    def dnn_input(self, inputs):
        emb_out, item_feat_emb, mask = self._item_inputs(inputs)
        target, short, long, _ = self.interest(item_feat_emb, mask)
        return torch.cat(([emb_out] if emb_out is not None else []) + [target, short, long], dim=-1)
