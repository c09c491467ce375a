"""Reader of the reference's labelled tf.Examples (`*.tfrecord.gz` written by preprocess in training mode), without
TensorFlow.

  * framing: GZIP'd TFRecord -- u64 length, masked crc32c of the length, payload, masked crc32c of the payload.  A CRC
    mismatch or a truncated record raises `TFRecordError`; nothing is skipped.
  * payload: a tf.Example; the fields `data_providers.parse_example` reads in non-inference mode
    (models/data_providers.py:41-58,226-297): name, window_pos, subreads/encoded (raw float32) + subreads/shape,
    subreads/num_passes, ccs_base_quality_scores, label/encoded (raw float32) + label/shape.
  * file arguments: a glob or a list of globs, expanded as `data_providers.create_glob_list` does
    (data_providers.py:367-374: each pattern in turn, files in the order the glob returns them).

`read_examples` returns rows float32 [N, R, L] exactly as stored (NOT clipped: `format_rows`' clipping happens in the
engine's embedding kernel), labels as u8 ids [N, L] over ' ATCG', and the per-window metadata.
"""
from __future__ import annotations

import glob as glob_lib
import gzip
import struct
from typing import Dict, Iterator, List, Sequence, Union

import numpy as np

from deepconsensus_b200 import tf_checkpoint


class TFRecordError(ValueError):
  pass


def create_glob_list(paths: Union[str, Sequence[str]]) -> List[str]:
  """data_providers.create_glob_list: every pattern expanded in turn (sorted, as tf.io.gfile.glob returns)."""
  if isinstance(paths, str):
    paths = [paths]
  out: List[str] = []
  for p in paths:
    out.extend(sorted(glob_lib.glob(p)))
  return out


def iter_records(path: str) -> Iterator[bytes]:
  """Payloads of one GZIP'd TFRecord file, in order, with both CRCs checked."""
  with gzip.open(path, "rb") as f:
    data = f.read()
  pos, n = 0, len(data)
  while pos < n:
    if pos + 12 > n:
      raise TFRecordError("%s: truncated record header at byte %d" % (path, pos))
    length, len_crc = struct.unpack_from("<QI", data, pos)
    if tf_checkpoint.mask_crc(tf_checkpoint.crc32c(data[pos:pos + 8])) != len_crc:
      raise TFRecordError("%s: length CRC mismatch at byte %d" % (path, pos))
    start = pos + 12
    if start + length + 4 > n:
      raise TFRecordError("%s: truncated record at byte %d" % (path, pos))
    payload = data[start:start + length]
    (data_crc,) = struct.unpack_from("<I", data, start + length)
    if tf_checkpoint.mask_crc(tf_checkpoint.crc32c(payload)) != data_crc:
      raise TFRecordError("%s: data CRC mismatch in the record at byte %d" % (path, pos))
    yield payload
    pos = start + length + 4


def _packed_varints(buf: bytes) -> List[int]:
  out, pos = [], 0
  while pos < len(buf):
    v, pos = tf_checkpoint._varint(buf, pos)
    out.append(tf_checkpoint._signed64(v))
  return out


def parse_example(payload: bytes) -> Dict[str, Union[List[bytes], List[float], List[int]]]:
  """tf.Example -> {feature name: list of values} (bytes_list / float_list / int64_list)."""
  feats: Dict[str, Union[List[bytes], List[float], List[int]]] = {}
  for f1, _, features in tf_checkpoint._proto_fields(payload):            # Example.features = 1
    if f1 != 1:
      continue
    for f2, _, entry in tf_checkpoint._proto_fields(features):            # Features.feature = 1 (map entry)
      if f2 != 1:
        continue
      key, value = None, b""
      for f3, _, v in tf_checkpoint._proto_fields(entry):
        if f3 == 1:
          key = v.decode()
        elif f3 == 2:
          value = v
      vals: list = []
      for kind, _, lst in tf_checkpoint._proto_fields(value):             # Feature: 1 bytes, 2 float, 3 int64
        for f4, wt, v in tf_checkpoint._proto_fields(lst):
          if f4 != 1:
            continue
          if kind == 1:
            vals.append(v)
          elif kind == 2:
            vals.extend(np.frombuffer(v, "<f4").tolist() if wt == 2 else [struct.unpack("<f", struct.pack("<I", v))[0]])
          elif kind == 3:
            vals.extend(_packed_varints(v) if wt == 2 else [tf_checkpoint._signed64(v)])
      if key is not None:
        feats[key] = vals
  return feats


_REQUIRED = ("name", "window_pos", "subreads/encoded", "subreads/shape", "subreads/num_passes", "ccs_base_quality_scores",
             "label/encoded", "label/shape")


def read_examples(paths: Union[str, Sequence[str]], limit: int = -1) -> Dict[str, np.ndarray]:
  """Labelled windows of every file matching `paths` (in create_glob_list order), at most `limit` (-1: all).

  Returns rows float32 [N, R, L], labels uint8 [N, L] (0..4 = ' ATCG'), names (object [N]), window_pos int32 [N],
  num_passes int32 [N], ccs_base_quality_scores int16 [N, L]."""
  files = create_glob_list(paths)
  if not files:
    raise FileNotFoundError("no files match %s" % (paths,))
  rows, labels, names, pos, npass, bq = [], [], [], [], [], []
  for path in files:
    for payload in iter_records(path):
      if 0 <= limit <= len(rows):
        break
      f = parse_example(payload)
      missing = [k for k in _REQUIRED if k not in f]
      if missing:
        raise TFRecordError("%s: example without %s (not a training-mode example?)" % (path, missing))
      shape = [int(s) for s in f["subreads/shape"]]
      r = np.frombuffer(f["subreads/encoded"][0], "<f4")
      if r.size != int(np.prod(shape)):
        raise TFRecordError("%s: subreads/encoded has %d values for shape %s" % (path, r.size, shape))
      r = r.reshape(shape[0], shape[1])
      lab = np.frombuffer(f["label/encoded"][0], "<f4")
      if lab.size != int(np.prod([int(s) for s in f["label/shape"]])) or lab.size != shape[1]:
        raise TFRecordError("%s: label of %d values for windows of length %d" % (path, lab.size, shape[1]))
      if lab.min() < 0 or lab.max() > 4:
        raise TFRecordError("%s: label id outside 0..4" % path)
      rows.append(r)
      labels.append(lab.astype(np.uint8))            # tf.cast(float -> int32) truncates; the ids are integers
      names.append(f["name"][0].decode())
      pos.append(int(f["window_pos"][0]))
      npass.append(int(f["subreads/num_passes"][0]))
      bq.append(np.asarray(f["ccs_base_quality_scores"], np.int16))
    if 0 <= limit <= len(rows):
      break
  shapes = {r.shape for r in rows}
  if len(shapes) > 1:
    raise TFRecordError("windows of different shapes: %s" % sorted(shapes))
  L = rows[0].shape[1] if rows else 0
  return dict(rows=np.stack(rows) if rows else np.zeros((0, 0, 0), np.float32),
              labels=np.stack(labels) if labels else np.zeros((0, L), np.uint8),
              names=np.array(names, dtype=object), window_pos=np.array(pos, np.int32),
              num_passes=np.array(npass, np.int32),
              ccs_base_quality_scores=np.stack(bq) if bq else np.zeros((0, L), np.int16))


# ----------------------------------------------------------------------------------------------- writer
def _varint(v: int) -> bytes:
  v &= (1 << 64) - 1
  out = bytearray()
  while True:
    b = v & 0x7F
    v >>= 7
    if v:
      out.append(b | 0x80)
    else:
      out.append(b)
      return bytes(out)


def _field(num: int, payload: bytes) -> bytes:
  return _varint(num << 3 | 2) + _varint(len(payload)) + payload


def serialize_example(features: Dict[str, Union[List[bytes], List[int]]]) -> bytes:
  """tf.Example with bytes_list (values of type bytes) and int64_list (ints) features, keys in the dict's order."""
  entries = b""
  for key, vals in features.items():
    if vals and isinstance(vals[0], (bytes, bytearray)):
      lst = _field(1, b"".join(_field(1, bytes(v)) for v in vals))                 # Feature.bytes_list = 1
    else:
      lst = _field(3, _field(1, b"".join(_varint(int(v)) for v in vals)))          # Feature.int64_list = 3, packed
    entries += _field(1, _field(1, key.encode()) + _field(2, lst))                # Features.feature map entry
  return _field(1, entries)                                                        # Example.features = 1


def frame_record(payload: bytes) -> bytes:
  """TFRecord framing: u64 length, masked crc32c of it, payload, masked crc32c of the payload."""
  length = struct.pack("<Q", len(payload))
  return (length + struct.pack("<I", tf_checkpoint.mask_crc(tf_checkpoint.crc32c(length))) + payload +
          struct.pack("<I", tf_checkpoint.mask_crc(tf_checkpoint.crc32c(payload))))


def dc_example(rows: np.ndarray, num_passes: int, name: str, window_pos: int, ccs_bq: np.ndarray,
               label: "np.ndarray | None" = None) -> bytes:
  """DcExample.tf_example (pre_lib.py:764-787) serialised: rows float32 [R, L] stored as [R, L, 1], the CCS base
  qualities, and with a label (ids over ' ATCG', [L]) label/encoded float32 and label/shape."""
  rows = np.ascontiguousarray(rows, "<f4")
  f: Dict[str, Union[List[bytes], List[int]]] = {
      "subreads/encoded": [rows.tobytes()], "subreads/shape": [rows.shape[0], rows.shape[1], 1],
      "subreads/num_passes": [int(num_passes)], "name": [name.encode()], "window_pos": [int(window_pos)],
      "ccs_base_quality_scores": [int(v) for v in np.asarray(ccs_bq).reshape(-1)]}
  if label is not None:
    lab = np.ascontiguousarray(label, "<f4")
    f["label/encoded"] = [lab.tobytes()]
    f["label/shape"] = [lab.shape[0]]
  return serialize_example(f)


class TFRecordWriter:
  """GZIP'd TFRecord file (what tf.io.TFRecordWriter with compression_type='GZIP' writes; the compressed stream need not
  be byte-identical)."""

  def __init__(self, path: str):
    self._f = gzip.open(path, "wb")

  def write(self, payload: bytes) -> None:
    self._f.write(frame_record(payload))

  def close(self) -> None:
    self._f.close()
