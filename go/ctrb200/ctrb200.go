// Package ctrb200 is the cgo shim that maps go-ctr's unchanged plugin surface —
// recommend.Fitter / recommend.PredictAbstract (recommend/rcmd.go:87-97) and the
// model.Train / model.Predict call shape (model/model.go:27, 242) — onto libctr_b200.so.
//
// NOT BUILT IN THIS REPOSITORY'S CI: the build image has no Go toolchain (SURVEY.md §8b "Compile
// reality").  It is the binding a go-ctr maintainer adds; every C entry point it calls is covered
// by the Python ctypes tests in tests/, which drive the identical C ABI.
//
// Build (on a machine with Go, CUDA 12.9 and an H100):
//
//	CGO_CFLAGS="-I${CTR_B200}/include" CGO_LDFLAGS="-L${CTR_B200}/go-ctr_b200 -lctr_b200" go build ./...
package ctrb200

/*
#cgo CFLAGS:  -I${SRCDIR}/../../include
#cgo LDFLAGS: -L${SRCDIR}/../../go-ctr_b200 -lctr_b200 -Wl,-rpath,${SRCDIR}/../../go-ctr_b200
#include <stdlib.h>
#include "ctr_b200.h"
*/
import "C"

import (
	"encoding/json"
	"fmt"
	"runtime"
	"time"
	"unsafe"

	rcmd "github.com/auxten/go-ctr/recommend"
	"gorgonia.org/tensor"
)

// Kind selects the graph the engine evaluates.
type Kind int

const (
	YoutubeDnn Kind = C.CTR_MODEL_YOUTUBE // model/youtube/dnn.go
	DinCosine  Kind = C.CTR_MODEL_DIN_COS // model/din/din.go (live variant)
	DinEuclid  Kind = C.CTR_MODEL_DIN_EUC // din.go:230
)

// Engine owns one device handle (weights + HBM tables).
type Engine struct {
	h   *C.ctr_handle
	cfg C.ctr_config
}

func (e *Engine) err(rc C.int) error {
	if rc == C.CTR_OK {
		return nil
	}
	return fmt.Errorf("ctr_b200 error %d: %s", int(rc), C.GoString(C.ctr_last_error(e.h)))
}

// NewEngine mirrors din.NewDinNet / youtube.NewYoutubeDnn (din.go:171, dnn.go:119).
func NewEngine(kind Kind, uProfileDim, uBehaviorSize, uBehaviorDim, iFeatureDim, cFeatureDim, batchSize, predBatchSize int) (*Engine, error) {
	if uBehaviorDim != iFeatureDim { // din.go:176-178
		return nil, fmt.Errorf("uBehaviorDim %d != iFeatureDim %d", uBehaviorDim, iFeatureDim)
	}
	e := &Engine{}
	C.ctr_config_default(&e.cfg, C.int(kind))
	e.cfg.uP, e.cfg.S, e.cfg.D, e.cfg.cF = C.int32_t(uProfileDim), C.int32_t(uBehaviorSize), C.int32_t(uBehaviorDim), C.int32_t(cFeatureDim)
	e.cfg.batch, e.cfg.pred_batch = C.int32_t(batchSize), C.int32_t(predBatchSize)
	if rc := C.ctr_create(&e.cfg, &e.h); rc != C.CTR_OK {
		return nil, fmt.Errorf("ctr_create: %d: %s", int(rc), C.GoString(C.ctr_last_error(nil)))
	}
	runtime.SetFinalizer(e, func(e *Engine) { e.Close() })
	return e, nil
}

func (e *Engine) Close() {
	if e.h != nil {
		C.ctr_destroy(e.h)
		e.h = nil
	}
}

func f32(p []float32) *C.float { return (*C.float)(unsafe.Pointer(&p[0])) }
func i32(p []int32) *C.int32_t { return (*C.int32_t)(unsafe.Pointer(&p[0])) }

func ranges(si *rcmd.SampleInfo) [8]C.int32_t {
	return [8]C.int32_t{
		C.int32_t(si.UserProfileRange[0]), C.int32_t(si.UserProfileRange[1]),
		C.int32_t(si.UserBehaviorRange[0]), C.int32_t(si.UserBehaviorRange[1]),
		C.int32_t(si.ItemFeatureRange[0]), C.int32_t(si.ItemFeatureRange[1]),
		C.int32_t(si.CtxFeatureRange[0]), C.int32_t(si.CtxFeatureRange[1]),
	}
}

// Train has model.Train's meaning (model.go:27-213) for the engine's model.
func (e *Engine) Train(numExamples, epochs, earlyStop int, si *rcmd.SampleInfo, inputs, targets []float32, xcols int) (lastCost float32, err error) {
	r := ranges(si)
	var cost C.float
	var ran C.int32_t
	rc := C.ctr_train_dense(e.h, f32(inputs), f32(targets), C.int64_t(numExamples), C.int32_t(xcols), &r[0],
		C.int32_t(epochs), C.int32_t(earlyStop), &cost, &ran)
	return float32(cost), e.err(rc)
}

// Predict has model.Predict's meaning (model.go:242-353).
func (e *Engine) Predict(numExamples int, si *rcmd.SampleInfo, inputs []float32, xcols int) ([]float32, error) {
	r := ranges(si)
	y := make([]float32, numExamples)
	rc := C.ctr_predict_dense(e.h, f32(inputs), C.int64_t(numExamples), C.int32_t(xcols), &r[0], f32(y))
	return y, e.err(rc)
}

// UploadTable puts a feature / embedding table in HBM (replaces UserFeatureCache /
// ItemFeatureCache / itemEmbeddingMap, rcmd.go:30-36).
func (e *Engine) UploadTable(which int, rows []float32, nrows, width int) error {
	return e.err(C.ctr_table_upload(e.h, C.int(which), f32(rows), C.int64_t(nrows), C.int32_t(width)))
}

// TrainStepIdx is one inner-loop iteration of model.Train (model.go:107-196) fed by row ids.
func (e *Engine) TrainStepIdx(userRow, itemRow, histRows []int32, label []float32) (cost float32, err error) {
	var st C.ctr_step_stats
	rc := C.ctr_train_step_idx(e.h, i32(userRow), i32(itemRow), i32(histRows), f32(label), C.int32_t(len(userRow)), &st)
	return float32(st.cost), e.err(rc)
}

// PredictIdx is recommend.BatchPredict → model.Predict (rcmd.go:277-337) fed by row ids.
func (e *Engine) PredictIdx(userRow, itemRow, histRows []int32) ([]float32, error) {
	y := make([]float32, len(userRow))
	rc := C.ctr_predict_idx(e.h, i32(userRow), i32(itemRow), i32(histRows), C.int64_t(len(userRow)), f32(y))
	return y, e.err(rc)
}

// TrainIdx is one model.Train pass (one epoch) over n samples given as row ids in host memory: batches are
// copied H2D on a second stream while the previous batch computes; costs receives one BCE per batch.
func (e *Engine) TrainIdx(userRow, itemRow, histRows []int32, label []float32, costs []float32) error {
	var cp *C.float
	if len(costs) > 0 {
		cp = f32(costs)
	}
	return e.err(C.ctr_train_idx(e.h, i32(userRow), i32(itemRow), i32(histRows), f32(label), C.int64_t(len(userRow)), cp))
}

func i64(p []int64) *C.int64_t { return (*C.int64_t)(unsafe.Pointer(&p[0])) }

// LoadIDMaps replaces the strconv.Itoa-keyed caches (rcmd.go:472,483,502): userIds[r] / itemIds[r] is the
// external id of table row r.
func (e *Engine) LoadIDMaps(userIds, itemIds []int64) error {
	if err := e.err(C.ctr_idmap_build(e.h, C.CTR_IDMAP_USER, i64(userIds), C.int64_t(len(userIds)))); err != nil {
		return err
	}
	return e.err(C.ctr_idmap_build(e.h, C.CTR_IDMAP_ITEM, i64(itemIds), C.int64_t(len(itemIds))))
}

// UploadUserBehavior puts every user's (time-descending) behaviour sequence in HBM (feature/ubcache,
// prepare.go:13-38): offsets [nUsers+1], ts and itemRows [n].
func (e *Engine) UploadUserBehavior(offsets, ts []int64, itemRows []int32) error {
	return e.err(C.ctr_ubcache_upload(e.h, i64(offsets), i64(ts), i32(itemRows), C.int64_t(len(offsets)-1), C.int64_t(len(ts))))
}

// i64n / i32n are i64 / i32 for slices that may be empty (NULL then).
func i64n(p []int64) *C.int64_t {
	if len(p) == 0 {
		return nil
	}
	return i64(p)
}

func i32n(p []int32) *C.int32_t {
	if len(p) == 0 {
		return nil
	}
	return i32(p)
}

// AppendUserBehavior appends events (userRows[i] acted on itemRows[i] at ts[i]) to the device ubcache, creating it if
// none was uploaded.  Sequences stay time-descending; equal timestamps keep the most recent arrival first.
func (e *Engine) AppendUserBehavior(userRows []int32, ts []int64, itemRows []int32) error {
	if len(ts) != len(userRows) || len(itemRows) != len(userRows) {
		return fmt.Errorf("AppendUserBehavior: %d users, %d timestamps, %d items", len(userRows), len(ts), len(itemRows))
	}
	return e.err(C.ctr_ubcache_append(e.h, i32n(userRows), i64n(ts), i32n(itemRows), C.int64_t(len(userRows))))
}

// SetUserBehavior is UserBehaviorCache.BatchSet (cache.go:36-41) at row level: userRows[k]'s whole sequence becomes
// [offsets[k], offsets[k+1]) of ts / itemRows (time-descending); an empty sequence is Delete (cache.go:44-48).
func (e *Engine) SetUserBehavior(userRows []int32, offsets, ts []int64, itemRows []int32) error {
	if len(offsets) != len(userRows)+1 || len(itemRows) != len(ts) {
		return fmt.Errorf("SetUserBehavior: %d users, %d offsets, %d timestamps, %d items", len(userRows), len(offsets), len(ts), len(itemRows))
	}
	return e.err(C.ctr_ubcache_set(e.h, i32n(userRows), i64(offsets), i64n(ts), i32n(itemRows), C.int64_t(len(userRows)), C.int64_t(len(ts))))
}

// DownloadUserBehavior returns the live device ubcache as the CSR UploadUserBehavior takes.
func (e *Engine) DownloadUserBehavior() (offsets, ts []int64, itemRows []int32, err error) {
	var nu, n C.int64_t
	if err = e.err(C.ctr_ubcache_download(e.h, nil, nil, nil, 0, 0, &nu, &n)); err != nil {
		return
	}
	offsets, ts, itemRows = make([]int64, int(nu)+1), make([]int64, int(n)), make([]int32, int(n))
	err = e.err(C.ctr_ubcache_download(e.h, i64(offsets), i64n(ts), i32n(itemRows), nu, n, &nu, &n))
	return
}

// InsertIDs adds ids to a live id map (which: C.CTR_IDMAP_USER or C.CTR_IDMAP_ITEM; the map is created if none was
// loaded).  Ids the map holds keep their rows; the others get the next rows in order of first occurrence.  Returns the
// row of every id.  With world > 1 InsertIDs is collective: every rank's process calls it with its own ids (possibly
// none) and every map ends as one GPU's insert of the ranks' ids concatenated in rank order; maps that differ across
// the ranks, or an id refused on any rank, fail on every rank.
func (e *Engine) InsertIDs(which int, ids []int64) ([]int32, error) {
	if len(ids) == 0 {
		if e.cfg.world <= 1 {
			return nil, nil
		}
		return nil, e.err(C.ctr_idmap_insert(e.h, C.int(which), nil, 0, nil))
	}
	rows := make([]int32, len(ids))
	return rows, e.err(C.ctr_idmap_insert(e.h, C.int(which), i64(ids), C.int64_t(len(ids)), i32(rows)))
}

// DownloadIDs returns a map's ids in row order (ids[r] is the id of row r): with LoadIDMaps, how a map grown by
// InsertIDs is persisted and restored (checkpoints do not hold id maps).  Local: the maps of every rank are the same.
func (e *Engine) DownloadIDs(which int) ([]int64, error) {
	var n C.int64_t
	if err := e.err(C.ctr_idmap_download(e.h, C.int(which), nil, 0, &n)); err != nil {
		return nil, err
	}
	ids := make([]int64, int(n))
	return ids, e.err(C.ctr_idmap_download(e.h, C.int(which), i64n(ids), n, &n))
}

// WriteTableRows writes rows of a live table in HBM: row rows[i] becomes data[i*width : (i+1)*width].  A row past the
// end grows the table in place (the gap reads as zero); ITEM_EMB's written rows restart their row-Adam moments at zero.
// With world > 1 WriteTableRows is collective: every rank's process calls it with its own rows (possibly none) and the
// table ends as one GPU's write of the ranks' rows concatenated in rank order; a row named twice, on one rank or across
// ranks, fails on every rank.  A row-sharded table sends each row to its owner and reallocates a shard that outgrows
// its allocation at twice its rows.
func (e *Engine) WriteTableRows(which int, rows []int32, data []float32, width int) error {
	if len(rows) == 0 && e.cfg.world > 1 && len(data) == 0 {
		return e.err(C.ctr_table_write_rows(e.h, C.int(which), nil, nil, 0, C.int32_t(width)))
	}
	if len(rows) == 0 || len(data) != len(rows)*width {
		return fmt.Errorf("WriteTableRows: %d rows, %d floats, width %d", len(rows), len(data), width)
	}
	return e.err(C.ctr_table_write_rows(e.h, C.int(which), i32(rows), f32(data), C.int64_t(len(rows)), C.int32_t(width)))
}

// BatchPredict is recommend.BatchPredict (rcmd.go:277-337) over sample keys, entirely on the device.
func (e *Engine) BatchPredict(sampleKeys []rcmd.Sample) ([]float32, error) {
	n := len(sampleKeys)
	u, it, ts := make([]int64, n), make([]int64, n), make([]int64, n)
	for i, k := range sampleKeys {
		u[i], it[i], ts[i] = int64(k.UserId), int64(k.ItemId), k.Timestamp
	}
	y := make([]float32, n)
	rc := C.ctr_batch_predict_keys(e.h, i64(u), i64(it), i64(ts), C.int64_t(n), f32(y))
	return y, e.err(rc)
}

// GroupAUC is the GAUC the README quotes (README.md:17, 25, 33): utils.RocAuc32 within each group (normally the
// sample's UserId), weighted by the groups' sample counts over the groups that hold both classes; NaN when none does.
// With perGroup, groups holds the distinct ids ascending and n / pos / auc their samples, positives and AUC (NaN for a
// group with one class), so another weighting is one dot product away.
func (e *Engine) GroupAUC(pred, y []float32, group []int64, perGroup bool) (gauc float64, usedGroups int64, groups []int64, n, pos []int32, auc []float64, err error) {
	m := len(pred)
	if m == 0 || len(y) != m || len(group) != m {
		return 0, 0, nil, nil, nil, nil, fmt.Errorf("ctrb200: GroupAUC needs equally long, non-empty pred, y and group")
	}
	var g C.double
	var ng, nu C.int64_t
	var gp *C.int64_t
	var np, pp *C.int32_t
	var ap *C.double
	if perGroup {
		groups, n, pos, auc = make([]int64, m), make([]int32, m), make([]int32, m), make([]float64, m)
		gp, np, pp, ap = i64(groups), i32(n), i32(pos), (*C.double)(unsafe.Pointer(&auc[0]))
	}
	if err = e.err(C.ctr_group_auc(e.h, f32(pred), f32(y), i64(group), C.int64_t(m), &g, &ng, &nu, gp, np, pp, ap)); err != nil {
		return 0, 0, nil, nil, nil, nil, err
	}
	if perGroup {
		k := int(ng)
		groups, n, pos, auc = groups[:k], n[:k], pos[:k], auc[:k]
	}
	return float64(g), int64(nu), groups, n, pos, auc, nil
}

func f32n(p []float32) *C.float {
	if len(p) == 0 {
		return nil
	}
	return f32(p)
}

// RocAUCDist is utils.RocAuc32 over every rank's samples of a multi-GPU engine (ctr_roc_auc_dist): collective, each
// rank passing its own samples (possibly none); every rank gets the AUC of all ranks' samples concatenated in rank
// order, bit for bit what one GPU computes on them.  On a single-GPU engine it is ctr_roc_auc.
func (e *Engine) RocAUCDist(pred, y []float32) (float64, error) {
	if len(y) != len(pred) {
		return 0, fmt.Errorf("ctrb200: RocAUCDist needs equally long pred and y")
	}
	var a C.double
	err := e.err(C.ctr_roc_auc_dist(e.h, f32n(pred), f32n(y), C.int64_t(len(pred)), &a))
	return float64(a), err
}

// GroupAUCDist is GroupAUC over every rank's samples of a multi-GPU engine (ctr_group_auc_dist), with GroupAUC's
// results on every rank: those of one GPU over all ranks' samples concatenated in rank order.  Collective; a rank may
// pass no samples.  With perGroup the call runs twice, once for the group count and once for the arrays.
func (e *Engine) GroupAUCDist(pred, y []float32, group []int64, perGroup bool) (gauc float64, usedGroups int64, groups []int64, n, pos []int32, auc []float64, err error) {
	m := len(pred)
	if len(y) != m || len(group) != m {
		return 0, 0, nil, nil, nil, nil, fmt.Errorf("ctrb200: GroupAUCDist needs equally long pred, y and group")
	}
	var g C.double
	var ng, nu C.int64_t
	call := func(k int) error {
		var gp *C.int64_t
		var np, pp *C.int32_t
		var ap *C.double
		if k > 0 {
			gp, np, pp, ap = i64(groups), i32(n), i32(pos), (*C.double)(unsafe.Pointer(&auc[0]))
		}
		return e.err(C.ctr_group_auc_dist(e.h, f32n(pred), f32n(y), i64n(group), C.int64_t(m), &g, &ng, &nu, C.int64_t(k), gp, np, pp, ap))
	}
	if err = call(0); err != nil {
		return 0, 0, nil, nil, nil, nil, err
	}
	if perGroup && ng > 0 {
		k := int(ng)
		groups, n, pos, auc = make([]int64, k), make([]int32, k), make([]int32, k), make([]float64, k)
		if err = call(k); err != nil {
			return 0, 0, nil, nil, nil, nil, err
		}
	}
	return float64(g), int64(nu), groups, n, pos, auc, nil
}

func f64(p []float64) *C.double { return (*C.double)(unsafe.Pointer(&p[0])) }

// curve runs ctr_roc_curve (roc) or ctr_pr_curve with room for n + 1 points and trims the three arrays; the PR curve's
// last point has no threshold.
func (e *Engine) curve(roc bool, pred, y []float32, posLabel float64) (a, b, thresholds []float64, err error) {
	m := len(pred)
	if m == 0 || len(y) != m {
		return nil, nil, nil, fmt.Errorf("ctrb200: a curve needs equally long, non-empty pred and y")
	}
	a, b, thresholds = make([]float64, m+1), make([]float64, m+1), make([]float64, m+1)
	var k C.int64_t
	var rc C.int
	if roc {
		rc = C.ctr_roc_curve(e.h, f32(pred), f32(y), C.int64_t(m), C.double(posLabel), f64(a), f64(b), f64(thresholds), C.int64_t(m+1), &k)
	} else {
		rc = C.ctr_pr_curve(e.h, f32(pred), f32(y), C.int64_t(m), C.double(posLabel), f64(a), f64(b), f64(thresholds), C.int64_t(m+1), &k)
	}
	if err = e.err(rc); err != nil {
		return nil, nil, nil, err
	}
	nt := int(k)
	if !roc {
		nt--
	}
	return a[:k], b[:k], thresholds[:nt], nil
}

// ROCCurve is metrics.ROCCurve (nn/metrics/ranking.go:71-103) on the device: one point per distinct score from the
// highest down, (0, 0) first when the top score holds a negative; a sample is positive when y == posLabel.
func (e *Engine) ROCCurve(pred, y []float32, posLabel float64) (fpr, tpr, thresholds []float64, err error) {
	return e.curve(true, pred, y, posLabel)
}

// PrecisionRecallCurve is metrics.PrecisionRecallCurve (ranking.go:183-209) on the device: recall decreasing to the
// final (precision 1, recall 0), which has no threshold.
func (e *Engine) PrecisionRecallCurve(pred, y []float32, posLabel float64) (precision, recall, thresholds []float64, err error) {
	return e.curve(false, pred, y, posLabel)
}

// AveragePrecision is metrics.AveragePrecisionScore (ranking.go:212-222) of a binary target on the device, positives
// y == 1; NaN with no positives.  Labels that are not binary are an error where the reference returns 0.
func (e *Engine) AveragePrecision(pred, y []float32) (float64, error) {
	m := len(pred)
	if m == 0 || len(y) != m {
		return 0, fmt.Errorf("ctrb200: AveragePrecision needs equally long, non-empty pred and y")
	}
	var ap C.double
	if err := e.err(C.ctr_average_precision(e.h, f32(pred), f32(y), C.int64_t(m), &ap)); err != nil {
		return 0, err
	}
	return float64(ap), nil
}

// f64n is f64, or nil for an empty slice (the C calls' optional weights)
func f64n(p []float64) *C.double {
	if len(p) == 0 {
		return nil
	}
	return f64(p)
}

// Averages of PrecisionRecallFScore and modes of R2Score / MeanError (the reference's strings, as the C enums)
const (
	AverageMacro    = int(C.CTR_AVERAGE_MACRO)
	AverageMicro    = int(C.CTR_AVERAGE_MICRO)
	AverageWeighted = int(C.CTR_AVERAGE_WEIGHTED) // equals AverageMacro, as in the reference (classification.go:116-131)

	MultioutputRaw              = int(C.CTR_MULTIOUTPUT_RAW)
	MultioutputUniform          = int(C.CTR_MULTIOUTPUT_UNIFORM)
	MultioutputVarianceWeighted = int(C.CTR_MULTIOUTPUT_VARIANCE_WEIGHTED)

	ErrorSquared  = int(C.CTR_ERROR_SQUARED)
	ErrorAbsolute = int(C.CTR_ERROR_ABSOLUTE)
)

// AccuracyScore is metrics.AccuracyScore (classification.go:12-34) on the device: yTrue and yPred are [n, nOut]
// row-major; a row is correct when every column is equal (==).  weight is per sample (nil: all 1) and must be finite.
func (e *Engine) AccuracyScore(yTrue, yPred []float64, nOut int, weight []float64, normalize bool) (float64, error) {
	if nOut < 1 || len(yTrue) == 0 || len(yTrue)%nOut != 0 || len(yPred) != len(yTrue) || (weight != nil && len(weight) != len(yTrue)/nOut) {
		return 0, fmt.Errorf("ctrb200: AccuracyScore needs [n, nOut] yTrue and yPred and nil or n weights")
	}
	norm := 0
	if normalize {
		norm = 1
	}
	var r C.double
	if err := e.err(C.ctr_accuracy_score(e.h, f64(yTrue), f64(yPred), C.int64_t(len(yTrue)/nOut), C.int32_t(nOut), f64n(weight), C.int32_t(norm), &r)); err != nil {
		return 0, err
	}
	return float64(r), nil
}

// ConfusionMatrix is metrics.ConfusionMatrix (classification.go:150-178) of 1-D labels on the device: the classes of
// yTrue ascending and the [C, C] matrix, row-major.  A prediction between two classes counts as the higher one; one
// above the largest class, or a NaN, is an error.
func (e *Engine) ConfusionMatrix(yTrue, yPred, weight []float64) (classes, cm []float64, err error) {
	m := len(yTrue)
	if m == 0 || len(yPred) != m || (weight != nil && len(weight) != m) {
		return nil, nil, fmt.Errorf("ctrb200: ConfusionMatrix needs equally long, non-empty yTrue, yPred (and weight)")
	}
	var nc C.int32_t
	classes = make([]float64, m)
	if err = e.err(C.ctr_confusion_matrix(e.h, f64(yTrue), f64(yPred), C.int64_t(m), f64n(weight), f64(classes), nil,
		C.int64_t(int64(m)*int64(m)), &nc)); err != nil {
		return nil, nil, err
	}
	cm = make([]float64, int(nc)*int(nc))
	if err = e.err(C.ctr_confusion_matrix(e.h, f64(yTrue), f64(yPred), C.int64_t(m), f64n(weight), nil, f64(cm),
		C.int64_t(len(cm)), &nc)); err != nil {
		return nil, nil, err
	}
	return classes[:nc], cm, nil
}

// PrecisionRecallFScore is metrics.PrecisionRecallFScoreSupport (classification.go:74-148) on the device: the class
// posLabel's precision, recall, F-beta and support, or with posLabel < 0 the average (AverageMacro, AverageMicro or
// AverageWeighted; support 0).  PrecisionScore, RecallScore and F1Score are beta = 1, FBetaScore the beta given.
// perClass holds [C, 4] rows (p, r, f, support).
func (e *Engine) PrecisionRecallFScore(yTrue, yPred, weight []float64, beta float64, average, posLabel int) (p, r, f, support float64, perClass []float64, err error) {
	m := len(yTrue)
	if m == 0 || len(yPred) != m || (weight != nil && len(weight) != m) {
		return 0, 0, 0, 0, nil, fmt.Errorf("ctrb200: PrecisionRecallFScore needs equally long, non-empty yTrue, yPred (and weight)")
	}
	var cp, cr, cf, cs C.double
	var nc C.int32_t
	perClass = make([]float64, 4*m)
	if err = e.err(C.ctr_precision_recall_fscore(e.h, f64(yTrue), f64(yPred), C.int64_t(m), f64n(weight), C.double(beta),
		C.int32_t(average), C.int32_t(posLabel), &cp, &cr, &cf, &cs, f64(perClass), C.int64_t(m), &nc)); err != nil {
		return 0, 0, 0, 0, nil, err
	}
	return float64(cp), float64(cr), float64(cf), float64(cs), perClass[:4*int(nc)], nil
}

// R2Score is metrics.R2Score (regression.go:83-128) on the device over [n, nOut] row-major targets: nOut scores for
// MultioutputRaw, else one.  weight is per sample (nil: all 1).  A constant column is not an error.
func (e *Engine) R2Score(yTrue, yPred []float64, nOut int, weight []float64, multioutput int) ([]float64, error) {
	if nOut < 1 || len(yTrue) == 0 || len(yTrue)%nOut != 0 || len(yPred) != len(yTrue) || (weight != nil && len(weight) != len(yTrue)/nOut) {
		return nil, fmt.Errorf("ctrb200: R2Score needs [n, nOut] yTrue and yPred and nil or n weights")
	}
	out := make([]float64, nOut)
	if err := e.err(C.ctr_r2_score(e.h, f64(yTrue), f64(yPred), C.int64_t(len(yTrue)/nOut), C.int32_t(nOut), f64n(weight), C.int32_t(multioutput), f64(out))); err != nil {
		return nil, err
	}
	if multioutput != MultioutputRaw {
		out = out[:1]
	}
	return out, nil
}

// MeanError is metrics.MeanSquaredError (kind ErrorSquared) or MeanAbsoluteError (ErrorAbsolute) (regression.go:153-244)
// on the device, without sample weights: nOut column means for MultioutputRaw, their mean for MultioutputUniform.
func (e *Engine) MeanError(yTrue, yPred []float64, nOut, kind, multioutput int) ([]float64, error) {
	if nOut < 1 || len(yTrue) == 0 || len(yTrue)%nOut != 0 || len(yPred) != len(yTrue) {
		return nil, fmt.Errorf("ctrb200: MeanError needs [n, nOut] yTrue and yPred")
	}
	out := make([]float64, nOut)
	if err := e.err(C.ctr_mean_error(e.h, f64(yTrue), f64(yPred), C.int64_t(len(yTrue)/nOut), C.int32_t(nOut), C.int32_t(kind), C.int32_t(multioutput), f64(out))); err != nil {
		return nil, err
	}
	if multioutput != MultioutputRaw {
		out = out[:1]
	}
	return out, nil
}

// GroupAveragePrecision is the mean average precision (MAP) over groups (normally the sample's UserId): AveragePrecision
// within each group, averaged without weights over the groups that hold a positive; NaN when none does.  With
// perGroup, groups holds the distinct ids ascending and n / pos / ap their samples, positives and AP (NaN without a
// positive), so another weighting is one dot product away.
func (e *Engine) GroupAveragePrecision(pred, y []float32, group []int64, perGroup bool) (mapScore float64, usedGroups int64, groups []int64, n, pos []int32, ap []float64, err error) {
	m := len(pred)
	if m == 0 || len(y) != m || len(group) != m {
		return 0, 0, nil, nil, nil, nil, fmt.Errorf("ctrb200: GroupAveragePrecision needs equally long, non-empty pred, y and group")
	}
	var r C.double
	var ng, nu C.int64_t
	var gp *C.int64_t
	var np, pp *C.int32_t
	var app *C.double
	if perGroup {
		groups, n, pos, ap = make([]int64, m), make([]int32, m), make([]int32, m), make([]float64, m)
		gp, np, pp, app = i64(groups), i32(n), i32(pos), f64(ap)
	}
	if err = e.err(C.ctr_group_average_precision(e.h, f32(pred), f32(y), i64(group), C.int64_t(m), &r, &ng, &nu, gp, np, pp, app)); err != nil {
		return 0, 0, nil, nil, nil, nil, err
	}
	if perGroup {
		k := int(ng)
		groups, n, pos, ap = groups[:k], n[:k], pos[:k], ap[:k]
	}
	return float64(r), int64(nu), groups, n, pos, ap, nil
}

// Search is search.Searcher (feature/embedding/search/search.go:66-134) over the ITEM_EMB table on the device: the k
// rows most cosine-similar to each query. queries holds nq float64 vectors of the table's width (SearchVector; rows,
// if not nil, names a row to exclude per query, -1 for none), or is nil and rows holds the query rows (SearchInternal,
// with the word→row map on the Go side). outRows / sims are [nq*k] in rank order; counts[i] is the true number of
// results of query i, the positions past it hold row -1 and similarity 0.
// With a row-sharded ITEM_EMB (world > 1, large table) Search is collective: every rank's process calls it with the
// same arguments and each receives the same complete result, bit-identical to one GPU holding the whole table;
// arguments that differ between the ranks fail on every rank. No Sync is needed after training.
func (e *Engine) Search(queries []float64, rows []int32, k int) (outRows []int32, sims []float64, counts []int32, err error) {
	nq := len(rows)
	var qp *C.double
	var rp *C.int32_t
	if len(queries) > 0 {
		nq = len(queries) / int(e.cfg.D)
		if rows != nil && len(rows) != nq {
			return nil, nil, nil, fmt.Errorf("ctrb200: len(rows) must equal the number of queries")
		}
		qp = (*C.double)(unsafe.Pointer(&queries[0]))
	}
	if len(rows) > 0 {
		rp = i32(rows)
	}
	if nq == 0 || k < 1 {
		return nil, nil, nil, fmt.Errorf("ctrb200: Search needs at least one query and k >= 1")
	}
	outRows = make([]int32, nq*k)
	sims = make([]float64, nq*k)
	counts = make([]int32, nq)
	rc := C.ctr_knn_search(e.h, qp, rp, C.int64_t(nq), C.int32_t(k), i32(outRows), (*C.double)(unsafe.Pointer(&sims[0])), i32(counts))
	if err = e.err(rc); err != nil {
		return nil, nil, nil, err
	}
	return outRows, sims, counts, nil
}

// Recommend is the default recall recommend/api.go:115-118 leaves as a todo: for each user row, every ITEM_EMB row is
// scored with the trained model as the sample (userRows[j], item, histRows[j*S:(j+1)*S]) and the k best are returned,
// logit descending then row ascending. excludeHistory drops the items of the user's valid history rows. outRows /
// scores / logits are [nu*k]; counts[j] is the true number of results of user j, the positions past it hold row -1,
// score 0 and logit 0.
// With a row-sharded ITEM_EMB (world > 1, large table) Recommend is collective, under the same rule as Search.
func (e *Engine) Recommend(userRows, histRows []int32, k int, excludeHistory bool) (outRows []int32, scores, logits []float32, counts []int32, err error) {
	return e.recommend(userRows, histRows, nil, k, windowMode(excludeHistory))
}

// RecommendSeen is Recommend that never lists an item the user has already seen: besides the valid history rows, the
// item of every event of the user's device behaviour cache with timestamp <= maxTs[j] (0: every event) is excluded.
// maxTs has one cut per user. With a row-sharded ITEM_EMB RecommendSeen is collective like Recommend, and every rank
// must pass the same maxTs. The rank that owns a row decides whether it is seen: row g is excluded when it is a valid
// history row, or when the behaviour cache of rank g % world holds such an event for item g. Apply every cache upload,
// append and set on every rank; then the result equals one GPU holding the whole table and that cache.
func (e *Engine) RecommendSeen(userRows, histRows []int32, maxTs []int64, k int) (outRows []int32, scores, logits []float32, counts []int32, err error) {
	if len(maxTs) != len(userRows) {
		return nil, nil, nil, nil, fmt.Errorf("ctrb200: RecommendSeen needs one maxTs per user")
	}
	return e.recommend(userRows, histRows, maxTs, k, C.CTR_EXCLUDE_SEEN)
}

// windowMode is the exclusion mode of an excludeHistory flag
func windowMode(excludeHistory bool) C.int32_t {
	if excludeHistory {
		return C.CTR_EXCLUDE_WINDOW
	}
	return C.CTR_EXCLUDE_NONE
}

func (e *Engine) recommend(userRows, histRows []int32, maxTs []int64, k int, mode C.int32_t) (outRows []int32, scores, logits []float32, counts []int32, err error) {
	nu := len(userRows)
	if nu == 0 || k < 1 || len(histRows) != nu*int(e.cfg.S) {
		return nil, nil, nil, nil, fmt.Errorf("ctrb200: Recommend needs at least one user, k >= 1 and S history rows per user")
	}
	outRows = make([]int32, nu*k)
	scores = make([]float32, nu*k)
	logits = make([]float32, nu*k)
	counts = make([]int32, nu)
	rc := C.ctr_recommend_topk_ex(e.h, i32(userRows), i32(histRows), i64n(maxTs), C.int64_t(nu), C.int32_t(k), mode, i32(outRows), f32(scores),
		f32(logits), i32(counts))
	if err = e.err(rc); err != nil {
		return nil, nil, nil, nil, err
	}
	return outRows, scores, logits, counts, nil
}

// RankItems is the full-catalogue rank of held-out items: for key i, every ITEM_EMB row is scored as Recommend scores it
// for (userRows[i], histRows[i*S:(i+1)*S]) and ranks[i] is the place itemRows[i] would take in that list (1 = first),
// or -1 when it can never be listed (outside the table, in an excluded history, or a NaN logit). For every k up to
// 1024, Recommend(k) lists the item exactly when 0 < rank <= k, at position rank-1, with logits[i] as its logit.
// With a row-sharded ITEM_EMB (world > 1, large table) RankItems is collective, under the same rule as Search.
func (e *Engine) RankItems(userRows, histRows, itemRows []int32, excludeHistory bool) (ranks []int64, logits []float32, err error) {
	return e.rankItems(userRows, histRows, nil, itemRows, windowMode(excludeHistory))
}

// RankItemsSeen ranks as RecommendSeen lists: key i's seen set (its history rows and the items of the user's cached
// events with timestamp <= maxTs[i]) is removed from the catalogue, and a target in it ranks -1. This is the filtered
// full-ranking protocol; with maxTs[i] the held-out event's time, no later event is excluded. With a row-sharded
// ITEM_EMB it is collective, under RecommendSeen's owner rule: a target's verdict comes from the rank that owns it.
func (e *Engine) RankItemsSeen(userRows, histRows []int32, maxTs []int64, itemRows []int32) (ranks []int64, logits []float32, err error) {
	if len(maxTs) != len(userRows) {
		return nil, nil, fmt.Errorf("ctrb200: RankItemsSeen needs one maxTs per key")
	}
	return e.rankItems(userRows, histRows, maxTs, itemRows, C.CTR_EXCLUDE_SEEN)
}

func (e *Engine) rankItems(userRows, histRows []int32, maxTs []int64, itemRows []int32, mode C.int32_t) (ranks []int64, logits []float32, err error) {
	n := len(userRows)
	if n == 0 || len(itemRows) != n || len(histRows) != n*int(e.cfg.S) {
		return nil, nil, fmt.Errorf("ctrb200: RankItems needs at least one key, one item and S history rows per key")
	}
	ranks = make([]int64, n)
	logits = make([]float32, n)
	if err = e.err(C.ctr_rank_items_ex(e.h, i32(userRows), i32(histRows), i64n(maxTs), i32(itemRows), C.int64_t(n), mode, i64(ranks), f32(logits))); err != nil {
		return nil, nil, err
	}
	return ranks, logits, nil
}

// RankMetrics turns ranks from RankItems into HR@k, Recall@k and NDCG@k for every k in ks, and MRR; groups[i] names key
// i's group (normally its user). A rank of -1 is a miss. Host only: no engine is needed.
func RankMetrics(ranks, groups []int64, ks []int32) (hit, recall, ndcg []float64, mrr float64, err error) {
	n := len(ranks)
	if n == 0 || len(groups) != n || len(ks) == 0 {
		return nil, nil, nil, 0, fmt.Errorf("ctrb200: RankMetrics needs equally long, non-empty ranks and groups and at least one k")
	}
	hit, recall, ndcg = make([]float64, len(ks)), make([]float64, len(ks)), make([]float64, len(ks))
	var m C.double
	rc := C.ctr_rank_metrics(i64(ranks), i64(groups), C.int64_t(n), i32(ks), C.int32_t(len(ks)), (*C.double)(unsafe.Pointer(&hit[0])),
		(*C.double)(unsafe.Pointer(&recall[0])), (*C.double)(unsafe.Pointer(&ndcg[0])), &m)
	if rc != C.CTR_OK {
		return nil, nil, nil, 0, fmt.Errorf("ctr_rank_metrics: %d: %s", int(rc), C.GoString(C.ctr_last_error(nil)))
	}
	return hit, recall, ndcg, float64(m), nil
}

// SaveCheckpoint / LoadCheckpoint: binary snapshot of weights, Adam moments, step counter and tables.
func (e *Engine) SaveCheckpoint(path string) error {
	cs := C.CString(path)
	defer C.free(unsafe.Pointer(cs))
	return e.err(C.ctr_checkpoint_save(e.h, cs))
}
func (e *Engine) LoadCheckpoint(path string) error {
	cs := C.CString(path)
	defer C.free(unsafe.Pointer(cs))
	return e.err(C.ctr_checkpoint_load(e.h, cs))
}

// dinModel is the reference's JSON schema (din.go:41-52; dnn.go:38-47 without att0).
type dinModel struct {
	UProfileDim   int       `json:"uProfileDim"`
	UBehaviorSize int       `json:"uBehaviorSize"`
	UBehaviorDim  int       `json:"uBehaviorDim"`
	IFeatureDim   int       `json:"iFeatureDim"`
	CFeatureDim   int       `json:"cFeatureDim"`
	Mlp0          []float32 `json:"mlp0"`
	Mlp1          []float32 `json:"mlp1"`
	Mlp2          []float32 `json:"mlp2"`
	Att0          []float32 `json:"att0,omitempty"`
}

// Marshal emits exactly what DinNet.Marshal / YoutubeDnn.Marshal emit (din.go:62, dnn.go:49), so
// din.NewDinNetFromJson can load an engine-trained model and vice versa.
func (e *Engine) Marshal() ([]byte, error) {
	in := int(e.cfg.uP + 2*e.cfg.D + e.cfg.cF)
	m := dinModel{UProfileDim: int(e.cfg.uP), UBehaviorSize: int(e.cfg.S), UBehaviorDim: int(e.cfg.D),
		IFeatureDim: int(e.cfg.D), CFeatureDim: int(e.cfg.cF),
		Mlp0: make([]float32, in*int(e.cfg.H0)), Mlp1: make([]float32, int(e.cfg.H0*e.cfg.H1)),
		Mlp2: make([]float32, int(e.cfg.H1)), Att0: make([]float32, int(e.cfg.S))}
	if err := e.err(C.ctr_get_weights(e.h, f32(m.Mlp0), f32(m.Mlp1), f32(m.Mlp2), f32(m.Att0))); err != nil {
		return nil, err
	}
	if Kind(e.cfg.model) == YoutubeDnn {
		m.Att0 = nil
	}
	return json.Marshal(m)
}

// LoadJSON is NewDinNetFromJson / NewYoutubeDnnFromJson for the engine (din.go:82, dnn.go:63).
func (e *Engine) LoadJSON(data []byte) error {
	var m dinModel
	if err := json.Unmarshal(data, &m); err != nil {
		return err
	}
	var att *C.float
	if len(m.Att0) > 0 {
		att = f32(m.Att0)
	}
	return e.err(C.ctr_set_weights(e.h, f32(m.Mlp0), f32(m.Mlp1), f32(m.Mlp2), att))
}

// Impl is the drop-in for example/movielens dinImpl / YoutubeDnnImpl (dinimpl.go:13-92,
// youtube.go:13-91): it satisfies recommend.Fitter and recommend.PredictAbstract, so
// recommend.Train(ctx, recSys, &ctrb200.Impl{...}) (rcmd.go:196,229) works unchanged.
type Impl struct {
	Kind                               Kind
	PredBatchSize, BatchSize, Epochs   int
	EarlyStop                          int
	UBehaviorSize, UBehaviorDim        int // rcmd.UserBehaviorLen, rcmd.ItemEmbDim
	sampleInfo                         *rcmd.SampleInfo
	xcols                              int
	pred                               *Engine
}

// Fit implements recommend.Fitter (rcmd.go:95-97); body follows dinImpl.Fit (dinimpl.go:44-92).
func (d *Impl) Fit(trainSample *rcmd.TrainSample) (rcmd.PredictAbstract, error) {
	uP := trainSample.Info.UserProfileRange[1] - trainSample.Info.UserProfileRange[0]
	cF := trainSample.Info.CtxFeatureRange[1] - trainSample.Info.CtxFeatureRange[0]
	d.sampleInfo, d.xcols = &trainSample.Info, trainSample.XCols
	if trainSample.Rows != len(trainSample.Y) {
		return nil, fmt.Errorf("number of examples %d and labels %d do not match", trainSample.Rows, len(trainSample.Y))
	}
	learner, err := NewEngine(d.Kind, uP, d.UBehaviorSize, d.UBehaviorDim, d.UBehaviorDim, cF, d.BatchSize, d.BatchSize)
	if err != nil {
		return nil, err
	}
	defer learner.Close()
	if _, err = learner.Train(trainSample.Rows, d.Epochs, d.EarlyStop, d.sampleInfo, trainSample.X, trainSample.Y, trainSample.XCols); err != nil {
		return nil, err
	}
	js, err := learner.Marshal() // learner → JSON → predictor, dinimpl.go:73-89
	if err != nil {
		return nil, err
	}
	pred, err := NewEngine(d.Kind, uP, d.UBehaviorSize, d.UBehaviorDim, d.UBehaviorDim, cF, d.PredBatchSize, d.PredBatchSize)
	if err != nil {
		return nil, err
	}
	if err = pred.LoadJSON(js); err != nil {
		return nil, err
	}
	d.pred = pred
	return d, nil
}

// Predict implements recommend.PredictAbstract (rcmd.go:87-89); body follows dinImpl.Predict
// (dinimpl.go:32-42), including returning nil on failure.
func (d *Impl) Predict(X tensor.Tensor) tensor.Tensor {
	numPred := X.Shape()[0]
	y, err := d.pred.Predict(numPred, d.sampleInfo, X.Data().([]float32), d.xcols)
	if err != nil {
		return nil
	}
	return tensor.NewDense(tensor.Float32, tensor.Shape{numPred, 1}, tensor.WithBacking(y))
}

// TrainKeys is recommend.Train's sample path (rcmd.go:197-246) on the device: the samples go down as keys (28 bytes
// each), GetSample's assembly (id maps, drop-unknown, history window at the sample's timestamp; rcmd.go:339-460) and
// model.Train's epoch loop run in HBM.  Needs LoadIDMaps (and UploadUserBehavior for DIN's history).
func (e *Engine) TrainKeys(samples []rcmd.Sample, epochs, earlyStop int) (lastCost float32, rowsUsed int64, err error) {
	n := len(samples)
	u, it, ts, y := make([]int64, n), make([]int64, n), make([]int64, n), make([]float32, n)
	for i, s := range samples {
		u[i], it[i], ts[i], y[i] = int64(s.UserId), int64(s.ItemId), s.Timestamp, s.Label
	}
	var cost C.float
	var ran C.int32_t
	var used C.int64_t
	rc := C.ctr_train_keys(e.h, i64(u), i64(it), i64(ts), f32(y), C.int64_t(n), C.int32_t(epochs), C.int32_t(earlyStop), &cost, &ran, &used)
	return float32(cost), int64(used), e.err(rc)
}

// TrainItemEmbedding is recommend.Train's embedding stage (GetItemEmbeddingModelFromUb + GenEmbeddingMap32 and the
// itemEmbeddingMap lookups, rcmd.go:207-213, 502, 519, 538-545) on the device: itemIds is what ItemSeqGenerator yields,
// as int64, in corpus order.  Words are numbered by first appearance, embedding.TrainEmbedding(itemSeq, window, D, iter)
// runs on them, and ITEM_EMB row r becomes the vector of the item LoadIDMaps put at row r (zeros when the item never
// occurs).  No table crosses PCIe.  Returns the item id of every word in word-id order (SaveVectors, Searcher).  With
// world > 1 TrainItemEmbedding is collective: every rank's process calls it with its own shard of the stream (possibly
// empty), words are numbered by first appearance in the ranks' shards concatenated in rank order (the same ids on every
// rank), each rank trains its shard with the replicas averaged, and each rank writes the ITEM_EMB rows it holds; item
// maps or arguments that differ across the ranks, or a stream empty on every rank, fail on every rank.  The returned
// vocabulary is whole and the same on every rank.
func (e *Engine) TrainItemEmbedding(itemIds []int64, window, iter int) ([]int64, error) {
	if len(itemIds) == 0 && e.cfg.world <= 1 {
		return nil, fmt.Errorf("TrainItemEmbedding: empty item stream")
	}
	var cfg C.ctr_i2v_config
	C.ctr_i2v_config_default(&cfg)
	cfg.dim, cfg.window, cfg.iter = e.cfg.D, C.int32_t(window), C.int32_t(iter)
	capacity := len(itemIds)
	if e.cfg.world > 1 { // room for every item-map row as well; only other ranks' unmapped ids can exceed it
		var rows C.int64_t
		if err := e.err(C.ctr_idmap_download(e.h, C.CTR_IDMAP_ITEM, nil, 0, &rows)); err == nil {
			capacity += int(rows)
		}
	}
	vocab := make([]int64, capacity+1)
	var v C.int32_t
	rc := C.ctr_item_emb_train(e.h, &cfg, i64n(itemIds), C.int64_t(len(itemIds)), i64(vocab), C.int64_t(len(vocab)), &v, nil)
	if err := e.err(rc); err != nil {
		return nil, err
	}
	if int(v) > len(vocab) { // other ranks' unmapped ids: the handle kept the whole vocabulary
		vocab = make([]int64, int(v))
		if err := e.err(C.ctr_item_emb_vocab(e.h, i64(vocab), C.int64_t(len(vocab)), &v)); err != nil {
			return nil, err
		}
	}
	return vocab[:int(v)], nil
}

// SetTableOptimizer selects how embedding rows learn (engine extension; the reference keeps them frozen,
// din.go:161-169): C.CTR_TABLE_FROZEN | SGD | SGD_DETERMINISTIC | ADAM.  Call before NewEngine's ctr_create in a
// custom constructor, or use NewEngineWith.
func NewEngineWith(kind Kind, uP, S, D, cF, batchSize, predBatchSize, tableOpt int, tableLr float32) (*Engine, error) {
	e := &Engine{}
	C.ctr_config_default(&e.cfg, C.int(kind))
	e.cfg.uP, e.cfg.S, e.cfg.D, e.cfg.cF = C.int32_t(uP), C.int32_t(S), C.int32_t(D), C.int32_t(cF)
	e.cfg.batch, e.cfg.pred_batch = C.int32_t(batchSize), C.int32_t(predBatchSize)
	e.cfg.table_opt, e.cfg.table_lr = C.int32_t(tableOpt), C.float(tableLr)
	if rc := C.ctr_create(&e.cfg, &e.h); rc != C.CTR_OK {
		return nil, fmt.Errorf("ctr_create: %d: %s", int(rc), C.GoString(C.ctr_last_error(nil)))
	}
	runtime.SetFinalizer(e, func(e *Engine) { e.Close() })
	return e, nil
}

// ---- model/mlp: drop-in for mlp.SimpleMlpFitWrap / SimpleMlpPredWrap (model/mlp/mlp.go:11-65) -----------------

// MlpFitWrap satisfies recommend.Fitter like mlp.SimpleMlpFitWrap{Model: nn.NewMLPClassifier([]int{100}, "relu",
// "adam", 1e-4)} (main.go:42-52): float32 TrainSample in, float64 training on the device.  The fields after Seed
// carry the names of BaseMultilayerPerceptron64's (basemlp64.go:25-50); a zero value means the reference default,
// and pointer fields exist where zero is itself a meaningful setting.  Fit returns an error for what the engine
// does not build (solver "lbfgs", EarlyStopping, BatchNormalize) instead of training something else.
// Labels: when every Y is 0 or 1 the classifier has one logistic output and predicts click probabilities.  Any other
// labels (ratings, say) are classes, as the reference's LabelBinarizer64 makes them: one softmax output per distinct
// value (one logistic output for a single value), and the predictor returns the predicted label of each row.  A NaN
// label or more than 1024 distinct labels is an error.
type MlpFitWrap struct {
	Hidden      []int   // HiddenLayerSizes, default {100}
	Activation  int     // C.CTR_MLP_RELU (default) | CTR_MLP_LOGISTIC | CTR_MLP_IDENTITY | CTR_MLP_TANH
	Alpha       float64 // 1e-4
	MaxIter     int     // 200
	Adaptive    bool    // LearningRate == "adaptive"
	Seed        uint32

	Solver            string   // "adam" (default) | "sgd"
	LearningRate      string   // "constant" (default, or "adaptive" when Adaptive) | "invscaling" | "adaptive"
	LearningRateInit  float64  // 1e-3
	PowerT            float64  // .5 (invscaling)
	Momentum          *float64 // .9 (sgd), in [0, 1]
	NesterovsMomentum *bool    // true (sgd)
	WeightDecay       float64  // 0, in [0, 1)
	BatchSize         int      // 200; clipped to the sample count
	Tol               float64  // 1e-4
	NIterNoChange     int      // 10
	Shuffle           *bool    // true
	EarlyStopping     bool     // not built: an error
	BatchNormalize    bool     // not built: an error
}

// MlpPredWrap satisfies recommend.PredictAbstract like mlp.SimpleMlpPredWrap.
type MlpPredWrap struct {
	m     *C.ctr_mlp
	xcols int
}

// create maps the options onto a classifier (or a one-target regressor) of xcols inputs, or refuses what the engine
// does not build.
func (f *MlpFitWrap) create(xcols int, regressor bool) (*C.ctr_mlp, error) {
	var cfg C.ctr_mlp_config
	C.ctr_mlp_config_default(&cfg, C.int32_t(xcols))
	if len(f.Hidden) > 0 {
		cfg.n_layers = C.int32_t(len(f.Hidden) + 2)
		for i, u := range f.Hidden {
			cfg.units[i+1] = C.int32_t(u)
		}
		cfg.units[len(f.Hidden)+1] = 1
	}
	cfg.hidden_act = C.int32_t(f.Activation)
	if f.Alpha != 0 {
		cfg.alpha = C.double(f.Alpha)
	}
	if f.MaxIter != 0 {
		cfg.max_iter = C.int32_t(f.MaxIter)
	}
	if f.Adaptive {
		cfg.adaptive = 1
	}
	cfg.seed = C.uint32_t(f.Seed)
	if f.LearningRateInit != 0 {
		cfg.lr_init = C.double(f.LearningRateInit)
	}
	if f.BatchSize != 0 {
		cfg.batch = C.int32_t(f.BatchSize)
	}
	if f.Tol != 0 {
		cfg.tol = C.double(f.Tol)
	}
	if f.NIterNoChange != 0 {
		cfg.n_iter_no_change = C.int32_t(f.NIterNoChange)
	}
	if f.Shuffle != nil && !*f.Shuffle {
		cfg.shuffle = 0
	}
	var opts C.ctr_mlp_options
	C.ctr_mlp_options_default(&opts)
	switch f.Solver {
	case "", "adam":
	case "sgd":
		opts.solver = C.CTR_MLP_SOLVER_SGD
	case "lbfgs":
		return nil, fmt.Errorf("MlpFitWrap: solver lbfgs is not built: the reference runs gonum's optimize.Minimize (basemlp64.go:675-727), which cannot be restated here")
	default:
		return nil, fmt.Errorf("MlpFitWrap: solver %q is not one of adam, sgd", f.Solver)
	}
	switch f.LearningRate {
	case "":
		if f.Adaptive {
			opts.lr_schedule = C.CTR_MLP_LR_ADAPTIVE
		}
	case "constant":
		opts.lr_schedule = C.CTR_MLP_LR_CONSTANT
	case "invscaling":
		opts.lr_schedule = C.CTR_MLP_LR_INVSCALING
	case "adaptive":
		opts.lr_schedule = C.CTR_MLP_LR_ADAPTIVE
		cfg.adaptive = 1
	default:
		return nil, fmt.Errorf("MlpFitWrap: learning rate %q is not one of constant, invscaling, adaptive", f.LearningRate)
	}
	if f.EarlyStopping {
		return nil, fmt.Errorf("MlpFitWrap: EarlyStopping is not built: the reference scores raw probabilities by exact-equality accuracy (basemlp64.go:933-938) and restores a best-parameter copy it never wrote (:850-853)")
	}
	if f.BatchNormalize {
		return nil, fmt.Errorf("MlpFitWrap: BatchNormalize is not built: the reference normalises in training only, never in predict (:347-351, :897-915)")
	}
	if f.PowerT != 0 {
		opts.power_t = C.double(f.PowerT)
	}
	if f.Momentum != nil {
		opts.momentum = C.double(*f.Momentum)
	}
	if f.NesterovsMomentum != nil && !*f.NesterovsMomentum {
		opts.nesterov = 0
	}
	opts.weight_decay = C.double(f.WeightDecay)
	var m *C.ctr_mlp
	if regressor {
		if rc := C.ctr_mlp_regressor_create(&cfg, &opts, &m); rc != C.CTR_OK {
			return nil, fmt.Errorf("ctr_mlp_regressor_create: %d: %s", int(rc), C.GoString(C.ctr_mlp_last_error(nil)))
		}
	} else if rc := C.ctr_mlp_create_ex(&cfg, &opts, &m); rc != C.CTR_OK {
		return nil, fmt.Errorf("ctr_mlp_create_ex: %d: %s", int(rc), C.GoString(C.ctr_mlp_last_error(nil)))
	}
	return m, nil
}

func (f *MlpFitWrap) Fit(trainSample *rcmd.TrainSample) (rcmd.PredictAbstract, error) {
	return f.fit(trainSample, false)
}

func (f *MlpFitWrap) fit(trainSample *rcmd.TrainSample, regressor bool) (rcmd.PredictAbstract, error) {
	m, err := f.create(trainSample.XCols, regressor)
	if err != nil {
		return nil, err
	}
	var iters C.int32_t
	if rc := C.ctr_mlp_fit(m, f32(trainSample.X), f32(trainSample.Y), C.int64_t(trainSample.Rows), C.int32_t(trainSample.XCols), &iters, nil); rc != C.CTR_OK {
		err := fmt.Errorf("ctr_mlp_fit: %d: %s", int(rc), C.GoString(C.ctr_mlp_last_error(m)))
		C.ctr_mlp_destroy(m)
		return nil, err
	}
	p := &MlpPredWrap{m: m, xcols: trainSample.XCols}
	runtime.SetFinalizer(p, func(p *MlpPredWrap) { C.ctr_mlp_destroy(p.m) })
	return p, nil
}

// Predict follows SimpleMlpPredWrap.Predict (mlp.go:15-39), including nil on failure: probabilities, or the predicted
// labels of a classifier fitted on labels other than 0 / 1.
func (p *MlpPredWrap) Predict(X tensor.Tensor) tensor.Tensor {
	n := X.Shape()[0]
	y := make([]float32, n)
	if rc := C.ctr_mlp_predict(p.m, f32(X.Data().([]float32)), C.int64_t(n), C.int32_t(p.xcols), f32(y)); rc != C.CTR_OK {
		return nil
	}
	return tensor.NewDense(tensor.Float32, tensor.Shape{n, 1}, tensor.WithBacking(y))
}

// Score is MLPRegressor.Score (multilayer_perceptron.go:64-70) of a predictor MlpRegressorFitWrap made: R² of its
// predictions on X against Y, one target per row.  A constant Y, or a classifier's predictor, is an error.
func (p *MlpPredWrap) Score(X tensor.Tensor, Y []float32) (float64, error) {
	n := X.Shape()[0]
	if len(Y) != n {
		return 0, fmt.Errorf("MlpPredWrap.Score: %d targets for %d rows", len(Y), n)
	}
	var r2 C.double
	if rc := C.ctr_mlp_score(p.m, f32(X.Data().([]float32)), f32(Y), C.int64_t(n), C.int32_t(p.xcols), &r2); rc != C.CTR_OK {
		return 0, fmt.Errorf("ctr_mlp_score: %d: %s", int(rc), C.GoString(C.ctr_mlp_last_error(p.m)))
	}
	return float64(r2), nil
}

// Accuracy is MLPClassifier.Score (multilayer_perceptron.go:127-133) of a classifier's predictor: the share of rows
// whose prediction equals Y.  With classes the prediction is the class label; a binary model compares its float64
// probability itself, as the reference does, so only probabilities of exactly 0 or 1 count.  A regressor's predictor
// is an error (its score is Score).
func (p *MlpPredWrap) Accuracy(X tensor.Tensor, Y []float32) (float64, error) {
	n := X.Shape()[0]
	if len(Y) != n {
		return 0, fmt.Errorf("MlpPredWrap.Accuracy: %d labels for %d rows", len(Y), n)
	}
	var acc C.double
	if rc := C.ctr_mlp_accuracy(p.m, f32(X.Data().([]float32)), f32(Y), C.int64_t(n), C.int32_t(p.xcols), &acc); rc != C.CTR_OK {
		return 0, fmt.Errorf("ctr_mlp_accuracy: %d: %s", int(rc), C.GoString(C.ctr_mlp_last_error(p.m)))
	}
	return float64(acc), nil
}

// MlpRegressorFitWrap satisfies recommend.Fitter with nn.NewMLPRegressor (multilayer_perceptron.go:19-28) in place of
// the classifier, with MlpFitWrap's options and refusals.  Each TrainSample.Y is the target: a rating, say.  Some
// target not 0 or 1 gives an identity output trained on square_loss, and the predictor returns predicted values, which
// Recommend then ranks; targets all 0 or 1 give the binary classifier exactly.  A NaN or infinite target is an error.
type MlpRegressorFitWrap struct{ MlpFitWrap }

func (f *MlpRegressorFitWrap) Fit(trainSample *rcmd.TrainSample) (rcmd.PredictAbstract, error) {
	return f.fit(trainSample, true)
}

// FitKeys is rcmd.Train (rcmd.go:197-246) with this fitter, with GetSample (rcmd.go:339-460) on the device: e is the
// feature store (id maps, tables, optional ubcache), samples are its keys.  Samples whose user or item is unknown are
// dropped; rowsUsed counts the rest.  The classifier has e's uP + S·D + D + cF inputs and trains bit for bit as Fit
// would on the rows GetSample builds.  The options and refusals are Fit's.  The predictor serves keys through e.
// FitKeys needs a single-GPU feature store: on a multi-GPU one use FitKeysDist.
func (f *MlpFitWrap) FitKeys(e *Engine, samples []rcmd.Sample) (*MlpPredWrap, int64, error) {
	return f.fitKeys(e, samples, false, false)
}

// FitKeys is MlpFitWrap.FitKeys with the regressor: each sample's Label is its target.
func (f *MlpRegressorFitWrap) FitKeys(e *Engine, samples []rcmd.Sample) (*MlpPredWrap, int64, error) {
	return f.fitKeys(e, samples, true, false)
}

// FitKeysDist is FitKeys on a multi-GPU feature store, a row-sharded ITEM_EMB included (ctr_mlp_fit_keys_dist).  With
// world > 1 it is collective: every rank calls it with its own samples (possibly none) and the same fitter options, and
// every rank's predictor ends as FitKeys on one GPU over all ranks' samples concatenated in rank order, bit for bit;
// rowsUsed counts the survivors of all ranks.  Each sample is windowed by the ubcache of the rank that passed it.  Options
// that differ across ranks are CTR_EINVAL everywhere; any other refusal is the lowest failing rank's on every rank.  On a
// single-GPU store it is FitKeys.
func (f *MlpFitWrap) FitKeysDist(e *Engine, samples []rcmd.Sample) (*MlpPredWrap, int64, error) {
	return f.fitKeys(e, samples, false, true)
}

// FitKeysDist is MlpFitWrap.FitKeysDist with the regressor: each sample's Label is its target.
func (f *MlpRegressorFitWrap) FitKeysDist(e *Engine, samples []rcmd.Sample) (*MlpPredWrap, int64, error) {
	return f.fitKeys(e, samples, true, true)
}

func (f *MlpFitWrap) fitKeys(e *Engine, samples []rcmd.Sample, regressor, dist bool) (*MlpPredWrap, int64, error) {
	n := len(samples)
	if n == 0 && !(dist && e.cfg.world > 1) {
		return nil, 0, fmt.Errorf("MlpFitWrap.FitKeys: no samples")
	}
	xcols := int(e.cfg.uP + e.cfg.S*e.cfg.D + e.cfg.D + e.cfg.cF)
	m, err := f.create(xcols, regressor)
	if err != nil {
		return nil, 0, err
	}
	u, it, ts, y := make([]int64, n), make([]int64, n), make([]int64, n), make([]float32, n)
	for i, s := range samples {
		u[i], it[i], ts[i], y[i] = int64(s.UserId), int64(s.ItemId), s.Timestamp, s.Label
	}
	var iters C.int32_t
	var used C.int64_t
	var rc C.int
	name := "ctr_mlp_fit_keys"
	if dist {
		name = "ctr_mlp_fit_keys_dist"
		var yp *C.float // a rank without samples passes null arrays
		if n > 0 {
			yp = f32(y)
		}
		rc = C.ctr_mlp_fit_keys_dist(m, e.h, i64n(u), i64n(it), i64n(ts), yp, C.int64_t(n), &iters, nil, &used)
	} else {
		rc = C.ctr_mlp_fit_keys(m, e.h, i64(u), i64(it), i64(ts), f32(y), C.int64_t(n), &iters, nil, &used)
	}
	if rc != C.CTR_OK {
		err := fmt.Errorf("%s: %d: %s", name, int(rc), C.GoString(C.ctr_mlp_last_error(m)))
		C.ctr_mlp_destroy(m)
		return nil, int64(used), err
	}
	p := &MlpPredWrap{m: m, xcols: xcols}
	runtime.SetFinalizer(p, func(p *MlpPredWrap) { C.ctr_mlp_destroy(p.m) })
	return p, int64(used), nil
}

// BatchPredict is recommend.BatchPredict (rcmd.go:277-337) for the MLP over the feature store e: an unknown key scores
// as an all-zero row, except key 0, which is an error.  On a row-sharded ITEM_EMB (world > 1) each rank scores its own
// keys under (*Engine).BatchPredict's rule: Sync on every rank and a barrier between training and prediction.
func (p *MlpPredWrap) BatchPredict(e *Engine, sampleKeys []rcmd.Sample) ([]float32, error) {
	n := len(sampleKeys)
	if n == 0 {
		return nil, fmt.Errorf("MlpPredWrap.BatchPredict: no sample keys")
	}
	u, it, ts := make([]int64, n), make([]int64, n), make([]int64, n)
	for i, k := range sampleKeys {
		u[i], it[i], ts[i] = int64(k.UserId), int64(k.ItemId), k.Timestamp
	}
	y := make([]float32, n)
	if rc := C.ctr_mlp_predict_keys(p.m, e.h, i64(u), i64(it), i64(ts), C.int64_t(n), f32(y)); rc != C.CTR_OK {
		return nil, fmt.Errorf("ctr_mlp_predict_keys: %d: %s", int(rc), C.GoString(C.ctr_mlp_last_error(p.m)))
	}
	return y, nil
}

// Rank is recommend.Rank (rcmd.go:248-275) for the MLP: itemIds scored for one user at the current time, in the
// caller's order.
func (p *MlpPredWrap) Rank(e *Engine, userId int, itemIds []int) ([]rcmd.ItemScore, error) {
	now := time.Now().Unix()
	keys := make([]rcmd.Sample, len(itemIds))
	for i, id := range itemIds {
		keys[i] = rcmd.Sample{UserId: userId, ItemId: id, Timestamp: now}
	}
	y, err := p.BatchPredict(e, keys)
	if err != nil {
		return nil, err
	}
	out := make([]rcmd.ItemScore, len(itemIds))
	for i, id := range itemIds {
		out[i] = rcmd.ItemScore{ItemId: id, Score: y[i]}
	}
	return out, nil
}

// Recommend is the default recall of recommend/api.go's empty itemIdList (api.go:115-118) for the MLP: every ITEM_EMB
// row of the feature store e scored for each user, windowed at ts[j], and the best k kept on the device (logit
// descending, then row ascending).  outRows, scores and logits are [len(userIds)·k]; counts[j] results of user j are
// valid.  Each score is what BatchPredict returns for (user, the row's item id, ts[j]).  An unknown user is an error,
// and so is a classifier fitted on labels other than 0 / 1: it predicts labels, so it has no click probability to
// rank items by (CTR_ESTATE, with nothing written).
// With a row-sharded ITEM_EMB (world > 1) Recommend is collective, under the same rule as (*Engine).Recommend: every
// rank calls it with the same users, ts and k and gets the same result; the users' windows are rank 0's.
func (p *MlpPredWrap) Recommend(e *Engine, userIds []int, ts []int64, k int, excludeHistory bool) (outRows []int32, scores []float32, logits []float64, counts []int32, err error) {
	return p.recommend(e, userIds, ts, k, windowMode(excludeHistory))
}

// RecommendSeen is Recommend that never lists an item the user has already seen: every item of the user's cached events
// with timestamp <= ts[j] (0: every event), the window's included.
func (p *MlpPredWrap) RecommendSeen(e *Engine, userIds []int, ts []int64, k int) (outRows []int32, scores []float32, logits []float64, counts []int32, err error) {
	return p.recommend(e, userIds, ts, k, C.CTR_EXCLUDE_SEEN)
}

func (p *MlpPredWrap) recommend(e *Engine, userIds []int, ts []int64, k int, mode C.int32_t) (outRows []int32, scores []float32, logits []float64, counts []int32, err error) {
	nu := len(userIds)
	if nu == 0 || k < 1 || len(ts) != nu {
		return nil, nil, nil, nil, fmt.Errorf("MlpPredWrap.Recommend needs at least one user, one ts per user and k >= 1")
	}
	u := make([]int64, nu)
	for i, id := range userIds {
		u[i] = int64(id)
	}
	outRows = make([]int32, nu*k)
	scores = make([]float32, nu*k)
	logits = make([]float64, nu*k)
	counts = make([]int32, nu)
	if rc := C.ctr_mlp_recommend_topk_ex(p.m, e.h, i64(u), i64(ts), C.int64_t(nu), C.int32_t(k), mode, i32(outRows), f32(scores),
		(*C.double)(unsafe.Pointer(&logits[0])), i32(counts)); rc != C.CTR_OK {
		return nil, nil, nil, nil, fmt.Errorf("ctr_mlp_recommend_topk_ex: %d: %s", int(rc), C.GoString(C.ctr_mlp_last_error(p.m)))
	}
	return outRows, scores, logits, counts, nil
}

// RankItems is the full-catalogue rank of held-out items for the MLP: key i is (userIds[i], itemIds[i], ts[i]), the
// user's window cut at ts[i] as Recommend cuts it, and ranks[i] the place the item would take in Recommend's list for
// (userIds[i], ts[i]), or -1 when it can never be listed (an unknown item id, an excluded window row, a NaN logit).
// logits[i] is the list's float64 logit for the item. An unknown user is an error.  With a row-sharded ITEM_EMB it is
// collective, as Recommend.
func (p *MlpPredWrap) RankItems(e *Engine, userIds, itemIds []int, ts []int64, excludeHistory bool) (ranks []int64, logits []float64, err error) {
	return p.rankItems(e, userIds, itemIds, ts, windowMode(excludeHistory))
}

// RankItemsSeen ranks as RecommendSeen lists: every item of the user's cached events with timestamp <= ts[i] is removed
// from the catalogue, and a target among them ranks -1.
func (p *MlpPredWrap) RankItemsSeen(e *Engine, userIds, itemIds []int, ts []int64) (ranks []int64, logits []float64, err error) {
	return p.rankItems(e, userIds, itemIds, ts, C.CTR_EXCLUDE_SEEN)
}

func (p *MlpPredWrap) rankItems(e *Engine, userIds, itemIds []int, ts []int64, mode C.int32_t) (ranks []int64, logits []float64, err error) {
	n := len(userIds)
	if n == 0 || len(itemIds) != n || len(ts) != n {
		return nil, nil, fmt.Errorf("MlpPredWrap.RankItems needs at least one key and one item and ts per key")
	}
	u, it := make([]int64, n), make([]int64, n)
	for i := range userIds {
		u[i], it[i] = int64(userIds[i]), int64(itemIds[i])
	}
	ranks = make([]int64, n)
	logits = make([]float64, n)
	if rc := C.ctr_mlp_rank_items_ex(p.m, e.h, i64(u), i64(it), i64(ts), C.int64_t(n), mode, i64(ranks),
		(*C.double)(unsafe.Pointer(&logits[0]))); rc != C.CTR_OK {
		return nil, nil, fmt.Errorf("ctr_mlp_rank_items_ex: %d: %s", int(rc), C.GoString(C.ctr_mlp_last_error(p.m)))
	}
	return ranks, logits, nil
}
