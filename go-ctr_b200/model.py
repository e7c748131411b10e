"""Host-side mirror of the reference's plugin / operator interface for the hot path, over the C ABI.

Names, argument order and error behaviour follow the Go reference so the parity tests read like
the reference's own tests (model/model_test.go, example/movielens/dinimpl_test.go):

    recommend.SampleInfo / TrainSample           rcmd.go:56-63, 132-137
    din.NewDinNet / NewDinNetFromJson / Marshal   din.go:62-147, 171
    youtube.NewYoutubeDnn / ...FromJson / Marshal dnn.go:49-160
    model.Train / InitForwardOnlyVm / Predict     model.go:27, 215, 242
    movielens dinImpl / YoutubeDnnImpl (Fitter + PredictAbstract)   dinimpl.go:13-92, youtube.go:13-91
    mlp.SimpleMlpFitWrap / SimpleMlpPredWrap (Fitter + PredictAbstract) model/mlp/mlp.go:11-65

The gorgonia-typed half of model.Model (Fwd/Graph/Vm, model.go:16-25) has no meaning on a GPU
engine; the seam is Fitter / PredictAbstract + Train / Predict + the Marshal JSON schema
(SURVEY.md §8b).  The Go binding of the same C ABI is go/ctrb200/ctrb200.go.
"""
import json
import time
from dataclasses import dataclass, field

import numpy as np

from . import engine as _e

__all__ = ["SampleInfo", "TrainSample", "DinNet", "YoutubeDnn", "NewDinNet", "NewDinNetFromJson",
           "NewYoutubeDnn", "NewYoutubeDnnFromJson", "Train", "InitForwardOnlyVm", "Predict",
           "DinImpl", "YoutubeDnnImpl", "RocAuc32", "GroupAuc32", "ROCCurve", "PrecisionRecallCurve",
           "AveragePrecisionScore", "GroupAveragePrecision32", "AccuracyScore", "ConfusionMatrix", "PrecisionScore",
           "RecallScore", "F1Score", "FBetaScore", "PrecisionRecallFScoreSupport", "R2Score", "MeanSquaredError",
           "MeanAbsoluteError", "SimpleMlpFitWrap", "SimpleMlpPredWrap"]

mlp0_1, mlp1_2 = 200, 80          # din.go:17-18


@dataclass
class SampleInfo:                 # rcmd.go:132-137
    UserProfileRange: tuple = (0, 0)
    UserBehaviorRange: tuple = (0, 0)
    ItemFeatureRange: tuple = (0, 0)
    CtxFeatureRange: tuple = (0, 0)

    def flat(self):
        return [*self.UserProfileRange, *self.UserBehaviorRange, *self.ItemFeatureRange, *self.CtxFeatureRange]


@dataclass
class TrainSample:                # rcmd.go:56-63
    X: np.ndarray = None
    Y: np.ndarray = None
    Rows: int = 0
    XCols: int = 0
    Info: SampleInfo = field(default_factory=SampleInfo)


class _Net:
    """Common state of DinNet / YoutubeDnn: dims + weights in the Marshal layout."""
    kind = None
    d0 = d1 = 0.0

    def __init__(self, uProfileDim, uBehaviorSize, uBehaviorDim, iFeatureDim, cFeatureDim, seed=0, gemm=_e.GEMM_AUTO):
        if uBehaviorDim != iFeatureDim:           # din.go:176-178
            raise ValueError("uBehaviorDim %d != iFeatureDim %d" % (uBehaviorDim, iFeatureDim))
        self.uProfileDim, self.uBehaviorSize, self.uBehaviorDim = uProfileDim, uBehaviorSize, uBehaviorDim
        self.iFeatureDim, self.cFeatureDim = iFeatureDim, cFeatureDim
        self.seed, self.gemm = seed, gemm
        self.weights = None           # (mlp0, mlp1, mlp2, att0) host copies, set after Train / FromJson
        self.engine = None            # the "VM" (model.go:81, 237)
        self.batchSize = 0

    def _config(self, batch, pred_batch, training):
        return _e.default_config(self.kind, uP=self.uProfileDim, S=self.uBehaviorSize, D=self.uBehaviorDim,
                                 cF=self.cFeatureDim, H0=mlp0_1, H1=mlp1_2, batch=batch, pred_batch=pred_batch,
                                 dropout0=self.d0 if training else 0.0, dropout1=self.d1 if training else 0.0,
                                 seed=self.seed, gemm=self.gemm)

    def Marshal(self):
        if self.weights is None:
            if self.engine is None:
                raise RuntimeError("model has no weights yet")
            self.weights = self.engine.get_weights()
        w0, w1, w2, att = self.weights
        m = {"uProfileDim": self.uProfileDim, "uBehaviorSize": self.uBehaviorSize, "uBehaviorDim": self.uBehaviorDim,
             "iFeatureDim": self.iFeatureDim, "cFeatureDim": self.cFeatureDim,
             "mlp0": [float(v) for v in np.asarray(w0, np.float32).ravel()],
             "mlp1": [float(v) for v in np.asarray(w1, np.float32).ravel()],
             "mlp2": [float(v) for v in np.asarray(w2, np.float32).ravel()]}
        if self.kind != _e.MODEL_YOUTUBE:
            m["att0"] = [float(v) for v in np.asarray(att, np.float32).ravel()]
        return json.dumps(m).encode()

    @classmethod
    def _from_json(cls, data):
        m = json.loads(data)
        net = cls(m["uProfileDim"], m["uBehaviorSize"], m["uBehaviorDim"], m["iFeatureDim"], m["cFeatureDim"])
        net.d0 = net.d1 = 0.0     # FromJson leaves d0/d1 unset ⇒ dropout is the identity (din.go:133-145)
        inn = m["uProfileDim"] + m["uBehaviorDim"] + m["iFeatureDim"] + m["cFeatureDim"]
        att = np.asarray(m.get("att0", [1.0] * m["uBehaviorSize"]), np.float32)
        net.weights = (np.asarray(m["mlp0"], np.float32).reshape(inn, mlp0_1),
                       np.asarray(m["mlp1"], np.float32).reshape(mlp0_1, mlp1_2),
                       np.asarray(m["mlp2"], np.float32).reshape(mlp1_2, 1), att)
        return net


class DinNet(_Net):
    kind = _e.MODEL_DIN_COS
    d0 = d1 = 0.005               # din.go:204-205


class YoutubeDnn(_Net):
    kind = _e.MODEL_YOUTUBE
    d0 = d1 = 0.003               # dnn.go:136-137


def NewDinNet(uProfileDim, uBehaviorSize, uBehaviorDim, iFeatureDim, cFeatureDim, **kw):
    return DinNet(uProfileDim, uBehaviorSize, uBehaviorDim, iFeatureDim, cFeatureDim, **kw)


def NewYoutubeDnn(uProfileDim, uBehaviorSize, uBehaviorDim, iFeatureDim, cFeatureDim, **kw):
    return YoutubeDnn(uProfileDim, uBehaviorSize, uBehaviorDim, iFeatureDim, cFeatureDim, **kw)


def NewDinNetFromJson(data):
    return DinNet._from_json(data)


def NewYoutubeDnnFromJson(data):
    return YoutubeDnn._from_json(data)


def _check_dims(m, uProfileDim, uBehaviorSize, uBehaviorDim, iFeatureDim, cFeatureDim):
    if (m.uProfileDim, m.uBehaviorSize, m.uBehaviorDim, m.iFeatureDim, m.cFeatureDim) != \
            (uProfileDim, uBehaviorSize, uBehaviorDim, iFeatureDim, cFeatureDim):
        raise ValueError("model dims do not match the arguments")
    if uBehaviorDim != iFeatureDim:               # Fwd: din.go:221-223
        raise ValueError("uBehaviorDim %d != iFeatureDim %d" % (uBehaviorDim, iFeatureDim))


def Train(uProfileDim, uBehaviorSize, uBehaviorDim, iFeatureDim, cFeatureDim,
          numExamples, batchSize, epochs, earlyStop, si, inputs, targets, m):
    """model.Train (model.go:27-213).  inputs [numExamples, XCols] float32, targets [numExamples(,1)].
    Returns (epochs_run, last_cost); the Go function returns only err — errors raise here."""
    _check_dims(m, uProfileDim, uBehaviorSize, uBehaviorDim, iFeatureDim, cFeatureDim)
    inputs = np.ascontiguousarray(inputs, np.float32)
    targets = np.ascontiguousarray(targets, np.float32).reshape(-1)
    if inputs.shape[0] < numExamples or targets.size < numExamples:
        raise ValueError("numExamples exceeds the tensors")
    eng = _e.Engine(m._config(batchSize, batchSize, training=True))
    if m.weights is not None:
        eng.set_weights(*m.weights)
    else:
        eng.init_weights(m.seed)                  # G.Gaussian(0,1) / ValuesOf(1): din.go:181-191
    ep, cost = eng.train_dense(inputs[:numExamples], targets[:numExamples], si.flat(), epochs, earlyStop)
    m.weights = eng.get_weights()
    m.engine = eng
    m.batchSize = batchSize
    return ep, cost


def InitForwardOnlyVm(uProfileDim, uBehaviorSize, uBehaviorDim, iFeatureDim, cFeatureDim, batchSize, m):
    """model.InitForwardOnlyVm (model.go:215-240): builds the forward-only engine for Predict."""
    _check_dims(m, uProfileDim, uBehaviorSize, uBehaviorDim, iFeatureDim, cFeatureDim)
    if m.weights is None:
        raise RuntimeError("model has no weights")
    eng = _e.Engine(m._config(batchSize, batchSize, training=False))
    eng.set_weights(*m.weights)
    m.engine = eng
    m.batchSize = batchSize


def Predict(m, numExamples, batchSize, si, inputs):
    """model.Predict (model.go:242-353) → []float32 of length numExamples."""
    if m.engine is None:
        raise RuntimeError("InitForwardOnlyVm was not called")
    if batchSize != m.batchSize:
        raise ValueError("batchSize differs from InitForwardOnlyVm's")
    inputs = np.ascontiguousarray(inputs, np.float32)
    return m.engine.predict_dense(inputs[:numExamples], si.flat())


class _Impl:
    """example/movielens dinImpl / YoutubeDnnImpl: recommend.Fitter + recommend.PredictAbstract
    (dinimpl.go:13-92, youtube.go:13-91)."""
    _new = None
    _from_json = None

    def __init__(self, uBehaviorSize, uBehaviorDim, PredBatchSize=100, BatchSize=200, epochs=100, earlyStop=0, seed=0):
        self.uBehaviorSize, self.uBehaviorDim = uBehaviorSize, uBehaviorDim    # rcmd.UserBehaviorLen / ItemEmbDim
        self.PredBatchSize, self.BatchSize, self.epochs, self.earlyStop = PredBatchSize, BatchSize, epochs, earlyStop
        self.seed = seed
        self.learner = self.pred = self.sampleInfo = None

    def Fit(self, trainSample):
        si = trainSample.Info
        self.uProfileDim = si.UserProfileRange[1] - si.UserProfileRange[0]
        self.cFeatureDim = si.CtxFeatureRange[1] - si.CtxFeatureRange[0]
        self.iFeatureDim = self.uBehaviorDim
        self.sampleInfo = si
        if trainSample.Rows != len(trainSample.Y):       # dinimpl.go:52-56
            raise ValueError("number of examples %d and labels %d do not match" % (trainSample.Rows, len(trainSample.Y)))
        inputs = np.asarray(trainSample.X, np.float32).reshape(trainSample.Rows, trainSample.XCols)
        dims = (self.uProfileDim, self.uBehaviorSize, self.uBehaviorDim, self.iFeatureDim, self.cFeatureDim)
        self.learner = type(self)._new(*dims, seed=self.seed)
        Train(*dims, trainSample.Rows, self.BatchSize, self.epochs, self.earlyStop, si, inputs, trainSample.Y, self.learner)
        self.pred = type(self)._from_json(self.learner.Marshal())       # dinimpl.go:73-78
        InitForwardOnlyVm(*dims, self.PredBatchSize, self.pred)
        return self

    def Predict(self, X):
        X = np.asarray(X, np.float32)
        y = Predict(self.pred, X.shape[0], self.PredBatchSize, self.sampleInfo, X)
        return y.reshape(-1, 1)                                          # dinimpl.go:39


class DinImpl(_Impl):
    _new = staticmethod(NewDinNet)
    _from_json = staticmethod(NewDinNetFromJson)


class YoutubeDnnImpl(_Impl):
    _new = staticmethod(NewYoutubeDnn)
    _from_json = staticmethod(NewYoutubeDnnFromJson)


class SimpleMlpPredWrap:
    """model/mlp/mlp.go:11-39: PredictAbstract over the fitted classifier — float32 X in, float32 [n, 1] out: click
    probabilities, or the predicted labels when the classifier was fitted on labels other than 0 / 1 (pred.classes_)."""

    def __init__(self, pred, engine=None):
        self.pred = pred
        self.engine = engine          # the feature store of FitKeys: serves batch_predict_keys

    def Predict(self, X):
        X = np.asarray(X, np.float32)
        return self.pred.predict(X).reshape(-1, 1)

    def batch_predict_keys(self, user_ids, item_ids, ts):
        """Scores sample keys through the bound feature store (ctr_mlp_predict_keys), so serving.BatchPredict,
        serving.Rank and serving.Recommend serve the MLP as they serve an engine."""
        self._bound()
        return self.pred.predict_keys(self.engine, user_ids, item_ids, ts)

    def recommend(self, userId, k, now=None, exclude_history=True, exclude_seen=False):
        """The k best items of the bound feature store's whole ITEM_EMB table for one user at `now` (default: the
        current time), scored by this MLP on the device (ctr_mlp_recommend_topk).  Returns (rows [n] int32, scores [n]
        float32, logits [n] float64), best first, n <= k; serving.Recommend maps the rows to item ids.  A classifier
        with classes has no click probability to rank by: CtrError with code ESTATE.  exclude_seen drops every item the
        user's ubcache events up to `now` hold, the window's included."""
        self._bound()
        ts = int(time.time()) if now is None else int(now)
        rows, scores, logits, cnt = self.pred.recommend_topk(self.engine, [int(userId)], [ts], k, exclude_history=exclude_history,
                                                             exclude_seen=exclude_seen)
        n = int(cnt[0])
        return rows[0, :n], scores[0, :n], logits[0, :n]

    def _bound(self):
        if self.engine is None:
            raise RuntimeError("this predictor was fitted from dense X: no feature store is bound (use FitKeys)")


class SimpleMlpFitWrap:
    """model/mlp/mlp.go:41-65: Fitter over nn.MLPClassifier (main.go:42-52 builds it with NewMLPClassifier([]int{100},
    "relu", "adam", 1e-4) — pass the same through **mlp_kw).  Model is created at Fit time from the sample width.
    Labels other than 0 / 1 (ratings, say) make it a multi-class classifier whose predictor returns labels."""

    def __init__(self, **mlp_kw):
        self.mlp_kw = mlp_kw
        self.Model = None

    def Fit(self, trainSample):
        X = np.asarray(trainSample.X, np.float32).reshape(trainSample.Rows, trainSample.XCols)
        Y = np.asarray(trainSample.Y, np.float32)
        self.Model = _e.MLPClassifier(trainSample.XCols, **self.mlp_kw)
        self.Model.fit(X, Y)
        return SimpleMlpPredWrap(self.Model)

    def FitKeys(self, engine, user_ids, item_ids, ts, label):
        """rcmd.Train (rcmd.go:197-246) with this fitter, GetSample on the device: `engine` holds the id maps, the tables
        and optionally the ubcache; the sample width is its uP + S·D + D + cF.  Keys with an unknown user or item are
        dropped (Model.rows_used counts the rest).  Returns a SimpleMlpPredWrap bound to `engine`, which
        serving.BatchPredict / serving.Rank / serving.Recommend accept in place of an engine."""
        c = engine.cfg
        self.Model = _e.MLPClassifier(c.uP + c.S * c.D + c.D + c.cF, **self.mlp_kw)
        self.Model.fit_keys(engine, user_ids, item_ids, ts, label)
        return SimpleMlpPredWrap(self.Model, engine)


def RocAuc32(pred, y, engine=None):
    """utils.RocAuc32 (util.go:131-148) on the device."""
    eng = engine or _e.Engine(_e.default_config(_e.MODEL_YOUTUBE, batch=1, pred_batch=1))
    return eng.roc_auc(pred, y)


def GroupAuc32(pred, y, group, engine=None):
    """GAUC on the device (ctr_group_auc): RocAuc32 per group (normally the UserId), weighted by the groups' sample
    counts over the groups that hold both classes — the metric go-ctr's README quotes (README.md:17, 25, 33)."""
    eng = engine or _e.Engine(_e.default_config(_e.MODEL_YOUTUBE, batch=1, pred_batch=1))
    return eng.group_auc(pred, y, group)[0]


def _eval_engine(engine):
    return engine or _e.Engine(_e.default_config(_e.MODEL_YOUTUBE, batch=1, pred_batch=1))


def _column(a):
    """A vector, or a matrix of one column (the reference's *mat.Dense of one output), as a flat array."""
    a = np.asarray(a)
    if a.ndim == 2 and a.shape[1] == 1:
        return a.ravel()
    if a.ndim != 1:
        raise ValueError("expected a vector or one column, got shape %s" % (a.shape,))
    return a


def ROCCurve(Ytrue, Yscore, posLabel, engine=None):
    """metrics.ROCCurve (nn/metrics/ranking.go:71-103) on the device (ctr_roc_curve): (fpr, tpr, thresholds)."""
    return _eval_engine(engine).roc_curve(_column(Yscore), _column(Ytrue), posLabel)


def PrecisionRecallCurve(Ytrue, ProbasPred, posLabel, engine=None):
    """metrics.PrecisionRecallCurve (ranking.go:183-209) on the device (ctr_pr_curve): (precision, recall, thresholds)."""
    return _eval_engine(engine).precision_recall_curve(_column(ProbasPred), _column(Ytrue), posLabel)


def AveragePrecisionScore(Ytrue, Yscore, engine=None):
    """metrics.AveragePrecisionScore (ranking.go:212-222) of a binary target on the device (ctr_average_precision).
    Labels that are not binary raise CtrError (EINVAL) where the reference prints "unsupported" and returns 0."""
    return _eval_engine(engine).average_precision(_column(Yscore), _column(Ytrue))


def GroupAveragePrecision32(pred, y, group, engine=None):
    """Mean average precision on the device (ctr_group_average_precision): AveragePrecisionScore per group (normally
    the UserId), averaged without weights over the groups that hold a positive — MAP, next to GroupAuc32's GAUC."""
    return _eval_engine(engine).group_average_precision(pred, y, group)[0]


# ---- nn/metrics classification.go and regression.go (the averages and modes by the reference's strings) ----------
_AVERAGES = ("macro", "micro", "weighted")


def _average(average):
    if average not in _AVERAGES:
        raise ValueError("average must be one of %s, got %r" % (list(_AVERAGES), average))
    return average


def AccuracyScore(Ytrue, Ypred, normalize, sampleWeight, engine=None):
    """metrics.AccuracyScore (classification.go:12-34) on the device (ctr_accuracy_score): [n] or [n, n_out] labels,
    sampleWeight [n] (or [n, 1]) or None."""
    return _eval_engine(engine).accuracy_score(Ytrue, Ypred, normalize, sampleWeight)


def ConfusionMatrix(YTrue, YPred, sampleWeight, engine=None):
    """metrics.ConfusionMatrix (classification.go:150-153) of 1-D labels on the device (ctr_confusion_matrix): the
    [C, C] matrix over the classes of YTrue."""
    return _eval_engine(engine).confusion_matrix(_column(YTrue), _column(YPred), sampleWeight)[1]


def PrecisionRecallFScoreSupport(YTrue, YPred, beta, labels, posLabel, average, warnFor, sampleWeight, engine=None):
    """metrics.PrecisionRecallFScoreSupport (classification.go:74-148) on the device (ctr_precision_recall_fscore):
    (precision, recall, fscore, support).  "weighted" averages like "macro", as the reference does (sklearn would weight
    by support).  The reference ignores labels and warnFor; here a non-empty one raises ValueError instead of being
    dropped."""
    if labels is not None and len(labels):
        raise ValueError("labels is not used by the reference's PrecisionRecallFScoreSupport: pass None or []")
    if warnFor is not None and len(warnFor):
        raise ValueError("warnFor is not used by the reference's PrecisionRecallFScoreSupport: pass None or []")
    avg = _average(average)
    return _eval_engine(engine).precision_recall_fscore(_column(YTrue), _column(YPred), beta, avg, posLabel, sampleWeight)


def PrecisionScore(Ytrue, Ypred, average, sampleWeight, engine=None):
    """metrics.PrecisionScore (classification.go:37-42) on the device"""
    return PrecisionRecallFScoreSupport(Ytrue, Ypred, 1.0, None, -1, average, [], sampleWeight, engine)[0]


def RecallScore(Ytrue, Ypred, average, sampleWeight, engine=None):
    """metrics.RecallScore (classification.go:44-49) on the device"""
    return PrecisionRecallFScoreSupport(Ytrue, Ypred, 1.0, None, -1, average, [], sampleWeight, engine)[1]


def FBetaScore(Ytrue, Ypred, beta, average, sampleWeight, engine=None):
    """metrics.FBetaScore (classification.go:58-68) on the device"""
    return PrecisionRecallFScoreSupport(Ytrue, Ypred, beta, None, -1, average, [], sampleWeight, engine)[2]


def F1Score(Ytrue, Ypred, average, sampleWeight, engine=None):
    """metrics.F1Score (classification.go:51-56) on the device"""
    return FBetaScore(Ytrue, Ypred, 1.0, average, sampleWeight, engine)


def _multioutput(multioutput, modes):
    m = "uniform_average" if multioutput == "" else multioutput
    if m not in modes:
        raise ValueError("multioutput must be one of %s or \"\", got %r" % (list(modes), multioutput))
    return m


def R2Score(yTrue, yPred, sampleWeight, multioutput, engine=None):
    """metrics.R2Score (regression.go:83-128) on the device (ctr_r2_score): "raw_values" returns the [n_out] scores,
    "variance_weighted" and "uniform_average" (or "") one float.  A constant column is not refused."""
    m = _multioutput(multioutput, ("raw_values", "uniform_average", "variance_weighted"))
    return _eval_engine(engine).r2_score(yTrue, yPred, sampleWeight, m)


def _mean_error(kind, yTrue, yPred, sampleWeight, multioutput, engine):
    if sampleWeight is not None:
        raise ValueError("sampleWeight is not supported: the reference reads sampleWeight.At(0, j) for every sample of "
                         "column j (regression.go:163, :230), which cancels out or gives 0/0")
    m = multioutput if multioutput == "variance_weighted" else _multioutput(multioutput, ("raw_values", "uniform_average"))
    return _eval_engine(engine).mean_error(yTrue, yPred, kind, m)


def MeanSquaredError(yTrue, yPred, sampleWeight, multioutput, engine=None):
    """metrics.MeanSquaredError (regression.go:153-176) on the device (ctr_mean_error); "variance_weighted" reaches
    the C call and raises CtrError (EINVAL)."""
    return _mean_error("squared", yTrue, yPred, sampleWeight, multioutput, engine)


def MeanAbsoluteError(yTrue, yPred, sampleWeight, multioutput, engine=None):
    """metrics.MeanAbsoluteError (regression.go:220-244) on the device (ctr_mean_error)"""
    return _mean_error("absolute", yTrue, yPred, sampleWeight, multioutput, engine)
