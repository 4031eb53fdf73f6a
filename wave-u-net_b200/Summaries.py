"""TensorBoard event files - the scalar summaries of the reference's tf.summary.FileWriter (Training.py:80-81,88,106
`sep_loss`; Test.py:41,81-82 `test_loss`), written without TensorFlow.

    with Summaries.EventFileWriter(os.path.join(model_config["log_dir"], str(experiment_id))) as w:
        w.add_scalar("sep_loss", loss, step, wall_time)
    Summaries.read_scalars(path)          # [(wall_time, step, tag, value)], both CRCs of every record checked

Format (restated from the published TensorFlow sources, tensorflow/core/util/event.proto, core/framework/summary.proto and
core/lib/io/record_writer.cc; tests/test_summaries.py pins it byte for byte against TensorBoard's own EventFileWriter):

  file   events.out.tfevents.<%010d unix seconds>.<hostname>.<pid>.<n>, n counting the writers of this process, so that two
         writers opened in the same second and directory write two files (TensorBoard reads any name containing "tfevents")
  record uint64 length (little-endian) | uint32 masked CRC-32C of those 8 bytes | payload | uint32 masked CRC-32C of payload
  Event  1: wall_time (double)  2: step (int64)  3: file_version (string)  5: summary (Summary); the first record of a file is
         Event{wall_time, file_version: "brain.Event:2"}
  Summary 1: value (repeated Summary.Value);  Summary.Value  1: tag (string)  2: simple_value (float)

The messages are proto3: wall_time, step and tag are written only when they are not zero / empty; file_version, summary and
simple_value sit in oneofs and are always written.  The FileWriter's graph_def and meta_graph_def events are not written:
there is no TensorFlow graph here to describe.
"""
import itertools
import os
import socket
import struct
import time

import numpy as np

import wun
from TFCheckpoint import CheckpointError, _fields, mask_crc, put_varint, unmask_crc

FILE_VERSION = "brain.Event:2"
_writer_ids = itertools.count()


class EventFileError(ValueError):
    pass


def _bytes_field(out, field, payload):
    out.append(field << 3 | 2)
    put_varint(out, len(payload))
    out += payload


def encode_event(wall_time, step=0, file_version=None, tag=None, value=None):
    """Serialised Event: the file_version record (file_version given) or one scalar summary (tag, value)."""
    out = bytearray()
    wt = struct.pack("<d", float(wall_time))
    if wt != bytes(8):
        out += b"\x09" + wt                                                   # 1: wall_time
    if step:
        out.append(0x10); put_varint(out, int(step))                          # 2: step
    if file_version is not None:
        _bytes_field(out, 3, file_version.encode("utf-8"))                    # 3: file_version
    else:
        val = bytearray()
        if tag:
            _bytes_field(val, 1, tag.encode("utf-8"))                         # Summary.Value 1: tag
        val += b"\x15" + np.float32(value).tobytes()                          # Summary.Value 2: simple_value (little-endian)
        summary = bytearray()
        _bytes_field(summary, 1, val)                                         # Summary 1: value
        _bytes_field(out, 5, summary)                                         # 5: summary
    return bytes(out)


def decode_event(payload):
    """Serialised Event -> {"wall_time", "step", "file_version" (or None), "values": [(tag, simple_value)]}."""
    e = {"wall_time": 0.0, "step": 0, "file_version": None, "values": []}
    try:
        for fn, wt, v in _fields(payload):
            if fn == 1 and wt == 1:
                e["wall_time"] = struct.unpack("<d", struct.pack("<Q", v))[0]
            elif fn == 2 and wt == 0:
                e["step"] = v - (1 << 64) if v >= 1 << 63 else v
            elif fn == 3 and wt == 2:
                e["file_version"] = v.decode("utf-8")
            elif fn == 5 and wt == 2:
                for f2, w2, val in _fields(v):
                    if f2 != 1 or w2 != 2:
                        continue
                    tag, simple = "", None
                    for f3, w3, x in _fields(val):
                        if f3 == 1 and w3 == 2:
                            tag = x.decode("utf-8")
                        elif f3 == 2 and w3 == 5:
                            simple = struct.unpack("<f", struct.pack("<I", x))[0]
                    if simple is not None:
                        e["values"].append((tag, simple))
    except (CheckpointError, struct.error, UnicodeDecodeError) as ex:
        raise EventFileError("malformed Event record: %s" % ex)
    return e


def frame_record(payload):
    """TFRecord framing of one payload."""
    header = struct.pack("<Q", len(payload))
    return (header + struct.pack("<I", mask_crc(wun.crc32c(header))) + payload +
            struct.pack("<I", mask_crc(wun.crc32c(payload))))


def read_records(path):
    """The payloads of a TFRecord file, each record's length and payload CRCs checked."""
    with open(path, "rb") as f:
        data = f.read()
    out, pos = [], 0
    while pos < len(data):
        if pos + 12 > len(data):
            raise EventFileError("%s: truncated record header at offset %d" % (path, pos))
        header = data[pos:pos + 8]
        n = struct.unpack("<Q", header)[0]
        if unmask_crc(struct.unpack_from("<I", data, pos + 8)[0]) != wun.crc32c(header):
            raise EventFileError("%s: record length checksum mismatch at offset %d" % (path, pos))
        if pos + 12 + n + 4 > len(data):
            raise EventFileError("%s: truncated record at offset %d" % (path, pos))
        payload = data[pos + 12:pos + 12 + n]
        if unmask_crc(struct.unpack_from("<I", data, pos + 12 + n)[0]) != wun.crc32c(payload):
            raise EventFileError("%s: record payload checksum mismatch at offset %d" % (path, pos))
        out.append(payload)
        pos += 12 + n + 4
    return out


def read_scalars(path):
    """[(wall_time, step, tag, value)] of the scalar summaries of an events file, in file order."""
    out = []
    for payload in read_records(path):
        e = decode_event(payload)
        out.extend((e["wall_time"], e["step"], tag, value) for tag, value in e["values"])
    return out


class EventFileWriter(object):
    """A new events file in `logdir` (created if missing), opened with its file_version record, as tf.summary.FileWriter
    opens one.  add_scalar(tag, value, step, wall_time=None) appends a scalar summary (value rounded to float32; wall_time
    defaults to now); flush() pushes what was written to the file; close() flushes and closes it."""

    def __init__(self, logdir):
        os.makedirs(logdir, exist_ok=True)
        now = time.time()
        name = "events.out.tfevents.%010d.%s.%d.%d" % (now, socket.gethostname(), os.getpid(), next(_writer_ids))
        self.path = os.path.join(logdir, name)
        self._f = open(self.path, "xb")
        self._f.write(frame_record(encode_event(now, file_version=FILE_VERSION)))

    def add_scalar(self, tag, value, step, wall_time=None):
        self._f.write(frame_record(encode_event(time.time() if wall_time is None else wall_time, step, tag=tag, value=value)))

    def flush(self):
        self._f.flush()

    def close(self):
        if not self._f.closed:
            self._f.flush()
            self._f.close()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def write_scalar(logdir, tag, value, step):
    """One scalar summary in a new events file of `logdir` (what Test.test's FileWriter writes); returns the file's path."""
    with EventFileWriter(logdir) as w:
        w.add_scalar(tag, value, step)
    return w.path
