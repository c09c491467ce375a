"""Host driver pieces of `deepconsensus run` that touch the model (mirror of the hot-path part of
`deepconsensus/inference/quick_inference.py`).

  InferenceOptions        quick_inference.py:238-275 (same field names)
  batch_examples          quick_inference.py:304-338
  run_model_on_examples   quick_inference.py:341-415   <- the drop-in: same signature, same return
  initialize_model        quick_inference.py:485-532   (weights come from an .npz / dict instead of a
                                                         TF checkpoint; see INTEGRATION.md)

`run_model_on_examples` hands the stacked rows to the CUDA engine, which returns the per-position
base and quality characters directly (the device epilogue does argmax / Phred / calibration /
clip / round, quick_inference.py:377-389); the host only slices bytes into `DCModelOutput`s.
"""
from __future__ import annotations

import dataclasses
from typing import Any, Dict, Iterable, Iterator, List, Optional, Tuple, Union

import numpy as np

from deepconsensus_b200 import calibration as calibration_lib
from deepconsensus_b200 import constants
from deepconsensus_b200 import engine as engine_lib
from deepconsensus_b200 import params as params_lib
from deepconsensus_b200 import stitch_utils
from deepconsensus_b200 import utils
from deepconsensus_b200 import weights as weights_lib


@dataclasses.dataclass
class InferenceOptions:
  """Options used across the inference stages (quick_inference.py:238-275)."""
  max_length: int
  example_height: int
  max_passes: int
  min_quality: int
  min_length: int
  batch_size: int
  use_ccs_bq: bool
  cpus: int
  skip_windows_above: int
  use_saved_model: bool
  max_base_quality: int
  dc_calibration_values: calibration_lib.QualityCalibrationValues
  ccs_calibration_values: calibration_lib.QualityCalibrationValues


def format_rows(subreads: np.ndarray, params: params_lib.Params) -> np.ndarray:
  """Shape check only: the PW/IP/SN clipping of data_providers.format_rows (:128-184) runs on the
  device inside the embedding kernel, so rows are passed through unmodified."""
  rows = np.asarray(subreads, dtype=constants.NP_DATA_TYPE)
  if rows.ndim == 2:
    rows = rows[..., None]
  if rows.shape != (params.total_rows, params.max_length, 1):
    raise ValueError("expected subreads of shape %s, got %s" %
                     ((params.total_rows, params.max_length, 1), rows.shape))
  return rows


def process_feature_dict(features: Dict[str, Any], params: params_lib.Params) -> Dict[str, Any]:
  """data_providers.process_feature_dict (:187-223) without TensorFlow."""
  return {
      "rows": format_rows(features["subreads"], params),
      "label": np.array([]),
      "num_passes": features["subreads/num_passes"],
      "window_pos": features["window_pos"],
      "name": features["name"],
      "ccs_base_quality_scores": features["ccs_base_quality_scores"],
      "ec": features["ec"],
      "np_num_passes": features["np_num_passes"],
      "rq": features["rq"],
      "rg": features["rg"],
  }


def batch_examples(feature_dicts: List[Dict[str, Any]], model_params: params_lib.Params,
                   options: InferenceOptions) -> Iterator[Dict[str, Any]]:
  """Stack values for each feature, `options.batch_size` windows at a time (quick_inference.py:304-338)."""
  processed = [process_feature_dict(fd, model_params) for fd in feature_dicts]
  for i in range(0, len(processed), options.batch_size):
    one_batch = processed[i:i + options.batch_size]
    yield {key: np.stack([x[key] for x in one_batch]) for key in constants.DC_FEATURES}


def run_model_on_examples(feature_dicts: List[Dict[str, Any]], model: engine_lib.B200Model,
                          model_params: params_lib.Params,
                          options: InferenceOptions) -> List[stitch_utils.DCModelOutput]:
  """Runs the model over windows and returns one DCModelOutput per window (quick_inference.py:341-415)."""
  predictions: List[stitch_utils.DCModelOutput] = []
  batches = batch_examples(feature_dicts, model_params, options)
  for data, out in engine_lib.pipelined(batches, lambda d: model.submit(d["rows"]), model.wait, model.drain):
    bases, quals = out["bases"], out["quals"]
    for i in range(bases.shape[0]):
      predictions.append(stitch_utils.DCModelOutput(
          window_pos=data["window_pos"][i], molecule_name=data["name"][i], ec=data["ec"][i],
          np_num_passes=data["np_num_passes"][i], rq=data["rq"][i], rg=data["rg"][i],
          sequence=bases[i].tobytes().decode("ascii"),
          quality_string=quals[i].tobytes().decode("ascii")))
  return predictions


def process_skipped_window(feature_dict: Dict[str, Any], options: InferenceOptions) -> stitch_utils.DCModelOutput:
  """A window that is not sent to the model adopts the CCS bases and (calibrated, capped) CCS base qualities
  (quick_inference.py:567-594)."""
  rows = feature_dict["subreads"]
  ccs_index = params_lib.get_indices(options.max_passes, options.use_ccs_bq)[4]
  ccs = rows[ccs_index[0], :, 0]
  ccs_seq = utils.encoded_sequence_to_string(ccs)
  ccs_quality_scores = feature_dict["ccs_base_quality_scores"]
  if options.ccs_calibration_values.enabled:
    ccs_quality_scores = calibration_lib.calibrate_quality_scores(ccs_quality_scores, options.ccs_calibration_values)
  ccs_quality_scores = np.minimum(ccs_quality_scores, options.max_base_quality)
  ccs_quality_scores = ccs_quality_scores.astype(dtype=np.int32)
  return stitch_utils.DCModelOutput(
      window_pos=feature_dict["window_pos"], molecule_name=feature_dict["name"], sequence=ccs_seq,
      quality_string=utils.quality_scores_to_string(ccs_quality_scores), ec=feature_dict["ec"],
      np_num_passes=feature_dict["np_num_passes"], rq=feature_dict["rq"], rg=feature_dict["rg"])


def split_skipped_windows(feature_dicts_for_zmws: Iterable[Iterable[Dict[str, Any]]], options: InferenceOptions
                          ) -> Tuple[List[Dict[str, Any]], List[stitch_utils.DCModelOutput]]:
  """The skip decision of `inference_on_n_zmws` (quick_inference.py:657-676): overflowing windows, and windows whose
  CCS already averages above `skip_windows_above`, bypass the model and adopt the CCS call."""
  for_model, skipped = [], []
  for one_zmw in feature_dicts_for_zmws:
    for window in one_zmw:
      skip_example = False
      if window["overflow"]:
        skipped.append(process_skipped_window(window, options))
        skip_example = True
      if options.skip_windows_above and not skip_example:
        if utils.avg_phred(window["ccs_base_quality_scores"]) > options.skip_windows_above:
          skipped.append(process_skipped_window(window, options))
          skip_example = True
      if not skip_example:
        for_model.append(window)
  return for_model, skipped


def run_model_and_stitch(feature_dicts: List[Dict[str, Any]], model: engine_lib.B200Model,
                         model_params: params_lib.Params, options: InferenceOptions,
                         outcome_counter: stitch_utils.OutcomeCounter,
                         skipped_outputs: Optional[List[stitch_utils.DCModelOutput]] = None
                         ) -> List[Optional[str]]:
  """Windows -> FASTQ records without per-window Python objects: `run_model_on_examples`, the merge with the windows
  that bypassed the model, the sort, and per read `stitch_utils.stitch_to_fastq` (quick_inference.py:341-415, :686 and
  :721-760), with the byte work on the device.

  `feature_dicts`: the windows to score (the `for_model` list of `split_skipped_windows`).  `skipped_outputs`: the
  DCModelOutputs `split_skipped_windows` produced for overflow / high-quality windows (`process_skipped_window`); they
  are interleaved with the model's outputs exactly as the reference does -- concatenate, sort by (molecule_name,
  window_pos), group by name (quick_inference.py:686,721-736).  Returns one FASTQ record (or None when a filter drops
  the read) per read, in sorted-name order; `outcome_counter` is updated like the reference's.
  """
  from deepconsensus_b200 import stitch_gpu
  L = int(model_params.max_length)
  names, positions, bases, quals = [], [], [], []
  batches = batch_examples(feature_dicts, model_params, options)
  for data, out in engine_lib.pipelined(batches, lambda d: model.submit(d["rows"]), model.wait, model.drain):
    bases.append(out["bases"])
    quals.append(out["quals"])
    names.extend(_as_str(x) for x in data["name"])
    positions.extend(int(x) for x in data["window_pos"])
  # skipped windows: L characters, or any width for an overflow window (CCS smart windows keep it whole)
  skipped = [(np.frombuffer(o.sequence.encode("latin-1"), np.uint8), np.frombuffer(o.quality_string.encode("latin-1"), np.uint8))
             for o in (skipped_outputs or [])]
  for o, (sb, sq) in zip(skipped_outputs or [], skipped):
    if len(sb) != len(sq):
      raise ValueError("skipped window %s@%s: sequence and quality string differ in length" % (o.molecule_name, o.window_pos))
    names.append(_as_str(o.molecule_name))
    positions.append(int(o.window_pos))
  if not names:
    return []
  order = sorted(range(len(names)), key=lambda i: (names[i], positions[i]))     # quick_inference.py:721-728
  names = [names[i] for i in order]
  positions = [positions[i] for i in order]
  if all(len(sb) == L for sb, _ in skipped):
    all_b = np.concatenate(bases + [np.stack([sb for sb, _ in skipped])] if skipped else bases)
    all_q = np.concatenate(quals + [np.stack([sq for _, sq in skipped])] if skipped else quals)
    return stitch_gpu.stitch_batch_to_fastq(model, all_b[order], all_q[order], names, positions, L, options.min_quality,
                                            options.min_length, outcome_counter)
  rows_b = [r for b in bases for r in b] + [sb for sb, _ in skipped]
  rows_q = [r for q in quals for r in q] + [sq for _, sq in skipped]
  win_off = np.zeros(len(order) + 1, np.int64)
  np.cumsum([len(rows_b[i]) for i in order], out=win_off[1:])
  return stitch_gpu.stitch_batch_to_fastq(model, np.concatenate([rows_b[i] for i in order]),
                                          np.concatenate([rows_q[i] for i in order]), names, positions, L,
                                          options.min_quality, options.min_length, outcome_counter, win_off=win_off)


def skip_decisions(model: engine_lib.B200Model, ccs_bq: np.ndarray, skip_windows_above: float) -> np.ndarray:
  """avg_phred(ccs_base_quality_scores) > skip_windows_above for every window of int16 [n, L] (quick_inference.py:
  663-672), decided by dcb_skip_mask; windows within 1e-7 of the threshold are re-decided with the reference's NumPy
  expression.  Returns bool [n]."""
  mask, _ = model.skip_mask(ccs_bq, skip_windows_above)
  for i in np.nonzero(mask == 2)[0]:
    mask[i] = utils.avg_phred(ccs_bq[i].astype(np.int64)) > skip_windows_above
  return mask.astype(bool)


def inference_on_zmw_windows(feature_dicts_for_zmws: Iterable[Iterable[Dict[str, Any]]], model: engine_lib.B200Model,
                             model_params: params_lib.Params, options: InferenceOptions,
                             outcome_counter: stitch_utils.OutcomeCounter) -> List[Optional[str]]:
  """The model-facing part of `inference_on_n_zmws` + the stitching of `run()` for a batch of ZMWs
  (quick_inference.py:657-686,721-760) with every per-window / per-read byte and arithmetic step on the device:

    skip decision   avg_phred(ccs_base_quality_scores) > skip_windows_above     dcb_skip_mask
    model           run_model_on_examples on the windows that are not skipped    dcb_submit / dcb_wait
    skipped windows process_skipped_window: adopt CCS bases / calibrated quals    dcb_fill_skipped
    stitch          sort by (name, window_pos), stitch_to_fastq per read          dcb_stitch_fastq

  Returns one FASTQ record (or None) per read in sorted-name order -- identical to the reference flow built from
  `split_skipped_windows`, `run_model_on_examples`, `sorted(...)` and `stitch_utils.stitch_to_fastq`.  Overflow windows
  may have any width, as `to_features_dict` makes them with CCS smart windows (pre_lib.py:683-697): they adopt their
  CCS at full width.
  """
  L = int(model_params.max_length)
  windows = [w for one_zmw in feature_dicts_for_zmws for w in one_zmw]
  if not windows:
    return []
  # windows grouped by read name, in order of appearance: the stable sort by (name, window_pos) of
  # quick_inference.py:721-728 is then the sort by name of the reads and by position inside each
  by_name: Dict[str, List[int]] = {}
  for i, w in enumerate(windows):
    by_name.setdefault(_as_str(w["name"]), []).append(i)
  windows = [windows[i] for ids in by_name.values() for i in ids]
  rows_of = lambda i: np.asarray(windows[i]["subreads"])
  ccs_row = params_lib.get_indices(options.max_passes, options.use_ccs_bq)[4][0]
  bq_full = [np.asarray(w["ccs_base_quality_scores"]) for w in windows]
  bq = np.stack([q[:L] for q in bq_full]).astype(np.int16)
  skip = np.array([bool(w.get("overflow", False)) for w in windows])
  wide = {i: (rows_of(i)[ccs_row, :, 0].astype(np.uint8), bq_full[i].astype(np.int16))
          for i in range(len(windows)) if rows_of(i).shape[1] != L}
  for i in wide:
    if not skip[i]:
      raise ValueError("window %s@%s is %d columns wide but not an overflow window" %
                       (_as_str(windows[i]["name"]), windows[i]["window_pos"], rows_of(i).shape[1]))

  def score(scored):       # run_model_on_examples' batches, two submissions in flight
    cursor = 0
    batches = batch_examples([windows[i] for i in scored], model_params, options)
    for _, out in engine_lib.pipelined(batches, lambda d: model.submit(d["rows"]), model.wait, model.drain):
      k = out["bases"].shape[0]
      yield scored[cursor:cursor + k], out["bases"], out["quals"]
      cursor += k
  score.batches = True

  fastq, rec_off, passed, _ = _skip_score_stitch(
      model, model_params, options, outcome_counter, list(by_name), np.array([len(v) for v in by_name.values()]),
      np.array([int(w["window_pos"]) for w in windows], np.int64), bq, skip, score,
      lambda skipped: np.stack([rows_of(i)[ccs_row, :L, 0] for i in skipped]).astype(np.uint8), wide=wide or None)
  return [fastq[int(rec_off[z]):int(rec_off[z + 1])].decode("latin-1") if passed[z] else None for z in range(len(passed))]


def inference_on_packed_zmws(zmws: List[Dict[str, Any]], model: engine_lib.B200Model, model_params: params_lib.Params,
                             options: InferenceOptions, outcome_counter: stitch_utils.OutcomeCounter
                             ) -> Tuple[bytes, np.ndarray, np.ndarray, List[str]]:
  """`inference_on_zmw_windows` without any per-window Python object: `zmws` are the per-ZMW array bundles of
  `preprocess.BamFeatureStream.next_zmw(want_rows=False, want_packed=True)` (packed rows, window_pos, ccs_bq, overflow,
  name).  Skip decision, model (dcb_forward_packed), skipped-window fill, sort and stitch as there.

  Returns (fastq bytes, rec_off, passed, names): read z (sorted-name order) has the record
  fastq[rec_off[z]:rec_off[z + 1]] when passed[z].
  """
  L, P = int(model_params.max_length), int(model_params.max_passes)
  zmws = [z for z in zmws if len(z["window_pos"])]
  if not zmws:
    return b"", np.zeros(1, np.int64), np.zeros(0, bool), []
  packed = np.concatenate([z["packed"] for z in zmws])

  def score(idx):
    out = model.forward_packed(packed[idx])
    return out["bases"], out["quals"]

  wide = None
  if "overflow_ccs_ids" in zmws[0]:                    # BamFeatureStream(use_ccs_smart_windows=True)
    wide, base = {}, 0
    for z in zmws:
      o = 0
      for i in np.nonzero(z["overflow"])[0]:
        w = int(z["window_width"][i])
        wide[base + int(i)] = (z["overflow_ccs_ids"][o:o + w], z["overflow_ccs_bq"][o:o + w])
        o += w
      base += len(z["window_pos"])
  return _skip_score_stitch(
      model, model_params, options, outcome_counter, [z["name"] for z in zmws], np.array([len(z["window_pos"]) for z in zmws]),
      np.concatenate([z["window_pos"] for z in zmws]).astype(np.int64), np.concatenate([z["ccs_bq"] for z in zmws]),
      np.concatenate([z["overflow"] for z in zmws]).astype(bool), score,
      lambda skipped: packed[skipped][:, 3 * P * L:3 * P * L + L], wide=wide)    # the CCS plane of the packed rows


def inference_on_record_zmws(zmws: List[Dict[str, Any]], model: engine_lib.B200Model, model_params: params_lib.Params,
                             options: InferenceOptions, outcome_counter: stitch_utils.OutcomeCounter, ins_trim: int = 5,
                             stats: Optional[Dict[str, Any]] = None) -> Tuple[bytes, np.ndarray, np.ndarray, List[str]]:
  """`inference_on_packed_zmws` with the feature construction on the device: `zmws` are the raw-record bundles of
  `preprocess.BamFeatureStream.next_zmw_records()`.  dcb_features_layout spaces the reads and returns what the skip
  decision needs; rows are laid out (dcb_features_pack) only for the windows the model scores, in device memory that
  dcb_forward_packed reads in place; skipped windows take their CCS ids and qualities from the layout.  Same return
  value, and the same bytes, as `inference_on_packed_zmws` on the host-built windows of the same ZMWs.  `stats`, when
  given, accumulates "windows" and "windows_skipped"."""
  if not zmws:
    return b"", np.zeros(1, np.int64), np.zeros(0, bool), []
  lay = model.features_layout(engine_lib.concat_records(zmws), ins_trim)
  counts = lay["zmw_windows"]
  if stats is not None:
    stats["windows"] = stats.get("windows", 0) + int(counts.sum())
  has = np.nonzero(counts)[0]
  if not len(has):
    return b"", np.zeros(1, np.int64), np.zeros(0, bool), []
  rows_dev = model.alloc_device(options.batch_size * model.packed_window_bytes)

  def score(idx):
    bases, quals = np.empty((len(idx), model.max_length), np.uint8), np.empty((len(idx), model.max_length), np.uint8)
    model.features_pack(idx, out=rows_dev)
    model.forward_packed_raw(rows_dev, len(idx), engine_lib.DCB_ROWS_ON_DEVICE, bases.ctypes.data, quals.ctypes.data)
    return bases, quals

  wide = None
  if "window_width" in lay:                            # CCS smart windows: overflow windows adopt their full-width CCS
    over = np.nonzero(lay["overflow"])[0]
    full = model.features_ccs(over, lay["window_width"][over])
    wide = {int(i): (full["ccs_ids"][full["off"][j]:full["off"][j + 1]], full["ccs_bq"][full["off"][j]:full["off"][j + 1]])
            for j, i in enumerate(over)}
  try:
    return _skip_score_stitch(model, model_params, options, outcome_counter, [zmws[k]["name"] for k in has], counts[has],
                              lay["window_pos"].astype(np.int64), lay["ccs_bq"], lay["overflow"].astype(bool), score,
                              lambda skipped: lay["ccs_ids"][skipped], stats, wide=wide)
  finally:
    model.free_device(rows_dev)


def _skip_score_stitch(model, model_params, options, outcome_counter, names_z, counts, pos, bq, skip, score, ccs_ids_of,
                       stats=None, wide=None):
  """The part of `inference_on_n_zmws` behind the features, for windows given as arrays (ZMW k owns counts[k]
  consecutive windows): skip decision, `score(window indices) -> (bases, quals)` for the rest in batches of
  options.batch_size, skipped-window fill from `ccs_ids_of(window indices)`, sort and stitch.  `score` may instead be
  a generator function `score(all scored indices)` yielding (indices, bases, quals) batch by batch (marked by the
  attribute `batches`), so that the caller keeps its own submission pipeline.

  wide: CCS smart windows -- {window index: (ccs ids, ccs base qualities)} at full width for every overflow window.
  Those windows are always skipped and keep their width through the fill and the stitch; every other window is L
  wide (quick_inference.py:661-664, process_skipped_window)."""
  from deepconsensus_b200 import stitch_gpu
  L = int(model_params.max_length)
  n = len(pos)
  if options.skip_windows_above:
    skip = skip | skip_decisions(model, bq, options.skip_windows_above)
  if stats is not None:
    stats["windows_skipped"] = stats.get("windows_skipped", 0) + int(skip.sum())
  # sort by (name, window_pos): ZMW order by name, windows inside a ZMW by position (quick_inference.py:721-728)
  zorder = sorted(range(len(names_z)), key=lambda k: names_z[k])
  starts = np.concatenate([[0], np.cumsum(counts)])
  order = np.concatenate([starts[k] + np.argsort(pos[starts[k]:starts[k + 1]], kind="stable") for k in zorder])
  dest = np.empty(n, np.int64)
  dest[order] = np.arange(n)
  scored, skipped = np.nonzero(~skip)[0], np.nonzero(skip)[0]
  names_sorted = [names_z[k] for k in zorder for _ in range(counts[k])]

  def scored_batches():
    if getattr(score, "batches", False):
      yield from score(scored)
      return
    for b0 in range(0, len(scored), options.batch_size):        # batch_examples (quick_inference.py:304-338)
      idx = scored[b0:b0 + options.batch_size]
      yield (idx,) + tuple(score(idx))

  if wide is None:
    all_b, all_q = np.empty((n, L), np.uint8), np.empty((n, L), np.uint8)
    for idx, b, q in scored_batches():
      all_b[dest[idx]], all_q[dest[idx]] = b, q
    if len(skipped):
      model.fill_skipped(ccs_ids_of(skipped), bq[skipped], dest[skipped].astype(np.int32), all_b, all_q,
                         calibration=options.ccs_calibration_values)
    win_off = None
  else:
    width = np.full(n, L, np.int64)
    for i, (ids, _) in wide.items():
      width[i] = len(ids)
    win_off = np.zeros(n + 1, np.int64)
    np.cumsum(width[order], out=win_off[1:])
    all_b, all_q = np.empty(int(win_off[-1]), np.uint8), np.empty(int(win_off[-1]), np.uint8)
    cols = np.arange(L)
    for idx, b, q in scored_batches():
      at = win_off[dest[idx]][:, None] + cols
      all_b[at], all_q[at] = b, q
    if len(skipped):
      narrow = ccs_ids_of(skipped)
      parts = [wide[i] if i in wide else (narrow[j], bq[i]) for j, i in enumerate(skipped)]
      src_off = np.zeros(len(skipped) + 1, np.int64)
      np.cumsum([len(p[0]) for p in parts], out=src_off[1:])
      model.fill_skipped_ragged(np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]), src_off,
                                dest[skipped], win_off, all_b, all_q, calibration=options.ccs_calibration_values)
  fastq, rec_off, passed = stitch_gpu.stitch_batch_to_fastq_bytes(model, all_b, all_q, names_sorted, pos[order].tolist(), L,
                                                                  options.min_quality, options.min_length, outcome_counter,
                                                                  win_off=win_off)
  return fastq, rec_off, passed, [names_z[k] for k in zorder]


def _as_str(x) -> str:
  return x.decode() if isinstance(x, (bytes, np.bytes_)) else str(x)


def load_weights_npz(path: str) -> weights_lib.Weights:
  """Variables exported as an .npz keyed by the checkpoint variable names."""
  with np.load(path) as z:
    return {k: z[k] for k in z.files}


def load_weights(checkpoint_path: str) -> weights_lib.Weights:
  """What `--checkpoint` may point at (quick_inference.py:515-529): a TF2 checkpoint prefix (".../checkpoint-50"), its
  `.index` file, a directory holding a `checkpoint` state file -- read without TensorFlow by `tf_checkpoint` -- or an
  .npz export of the same variables."""
  if checkpoint_path.endswith(".npz"):
    return load_weights_npz(checkpoint_path)
  from deepconsensus_b200 import tf_checkpoint
  return tf_checkpoint.load_variables(tf_checkpoint.resolve_prefix(checkpoint_path))


def read_params_from_json(checkpoint_path: str) -> params_lib.Params:
  """params.json next to the checkpoint (model_utils.read_params_from_json, model_utils.py:434-465)."""
  return params_lib.read_params_from_json(checkpoint_path)


def initialize_model(checkpoint_path: str, params: params_lib.Params, options: InferenceOptions,
                     weights: Optional[weights_lib.Weights] = None, device: int = 0, precision: str = "bf16"
                     ) -> Tuple[engine_lib.B200Model, params_lib.Params]:
  """Builds the engine for `params` and loads variables (quick_inference.py:485-532).

  `checkpoint_path`: a TF2 checkpoint (prefix / directory / .index) or an .npz export; `weights` overrides it.
  Like the reference's `assert_existing_objects_matched()`, a variable the model needs but the checkpoint lacks (or
  holds with another shape) raises; extra keys (optimizer slots) are ignored as with `expect_partial()`.
  """
  params_lib.modify_params(params, max_length=options.max_length, is_training=False)
  if weights is None:
    weights = load_weights(checkpoint_path)
  model = engine_lib.B200Model(params, weights, max_batch=options.batch_size, device=device,
                               max_base_quality=options.max_base_quality,
                               calibration=options.dc_calibration_values, precision=precision)
  return model, params
