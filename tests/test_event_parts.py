"""The part files of a `pio export` directory (events.export_parts and friends), which the streamed device read and the host
mirror both take: name order, what is skipped, part boundaries and the mapping of global lines back to parts."""
import json

from universal_recommender_b200 import events as E


def line(k: int, name: str = "buy") -> bytes:
    return json.dumps({"event": name, "entityType": "user", "entityId": f"u{k}", "targetEntityType": "item",
                       "targetEntityId": f"i{k % 7}", "eventTime": "2020-01-01T00:00:00.%03dZ" % (k % 1000)}).encode()


def write_export(d, parts: dict):
    d.mkdir(exist_ok=True)
    for name, data in parts.items():
        (d / name).write_bytes(data)
    return d


def test_parts_in_name_order_without_markers_checksums_hidden_or_empty_files(tmp_path):
    d = write_export(tmp_path / "export", {
        "part-00010": line(10) + b"\n", "part-00002": line(2) + b"\n", "part-00000": b"", "_SUCCESS": b"",
        ".part-00002.crc": b"x", "part-00002.crc": b"x", ".hidden": b"x", "_temporary": b"x"})
    (d / "part-00003").mkdir()   # not a file
    assert [p.rsplit("/", 1)[1] for p in E.export_parts(d)] == ["part-00002", "part-00010"]


def test_a_part_without_a_final_newline_does_not_join_the_next_part(tmp_path):
    d = write_export(tmp_path / "export", {"part-00000": line(0) + b"\n" + line(1), "part-00001": line(2) + b"\r\n" + line(3)})
    joined = E.join_parts(E.export_parts(d))
    assert joined == line(0) + b"\n" + line(1) + b"\n" + line(2) + b"\r\n" + line(3) + b"\n"
    assert [e[0] for e in E.read_export(str(d)).events] == ["u0", "u1", "u2", "u3"]


def test_global_lines_map_to_part_and_line(tmp_path):
    d = write_export(tmp_path / "export", {"part-00000": line(0) + b"\n" + line(1), "part-00001": b"\n".join(line(k) for k in range(3)) + b"\n",
                                           "part-00002": line(9)})
    counts = [E.part_lines(p) for p in E.export_parts(d)]
    assert counts == [2, 3, 1]
    want = [(0, 0), (0, 1), (1, 0), (1, 1), (1, 2), (2, 0)]
    assert [E.locate_line(counts, g) for g in range(6)] == want


def test_read_export_of_a_directory_equals_read_export_of_the_joined_bytes(tmp_path):
    rows = [line(k, ["buy", "view"][k % 2]) for k in range(40)]
    rows += [b'{"event":"$set","entityType":"item","entityId":"i1","properties":{"a":1},"eventTime":"2020-01-01T00:00:00Z"}']
    d = write_export(tmp_path / "export", {"part-%05d" % k: b"\n".join(rows[k * 10:(k + 1) * 10]) for k in range(5)})
    want = E.read_export(b"\n".join(rows))
    got = E.read_export(str(d))
    assert (got.names, got.events, got.ranking_events, got.set_events) == (want.names, want.events, want.ranking_events, want.set_events)
