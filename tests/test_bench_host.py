"""CPU: host-side logic of bench.py that does not need a GPU -- the watchdog / time-budget wrapper around the secondary blocks
of the bench line, and the parser that takes roofline.traffic from an ncu summary."""
import io
import json
import time

import bench


def test_secondary_blocks_return_values_errors_and_skips():
    line = {"metric": "m"}
    sb = bench.SecondaryBlocks(0, line, budget_s=30.0, exit_fn=lambda code: None, out=io.StringIO())
    assert sb.run("ok", 5, lambda: {"value": 1}) == {"value": 1}
    err = sb.run("boom", 5, lambda: 1 / 0)
    assert "ZeroDivisionError" in err["error"]
    assert "incomplete" not in line
    spent = bench.SecondaryBlocks(0, line, budget_s=0.0, exit_fn=lambda code: None, out=io.StringIO())
    called = []
    assert spent.run("late", 5, lambda: called.append(1)) == {"skipped": "secondary time budget spent"}
    assert not called and line["incomplete"] == ["late: skipped, secondary time budget spent"]


def test_secondary_block_watchdog_prints_the_line_and_exits():
    line = {"metric": "m", "value": 1.0}
    out, exits = io.StringIO(), []
    sb = bench.SecondaryBlocks(0, line, budget_s=0.3 + 3.0, exit_fn=exits.append, out=out)   # limit = min(block limit, budget left)
    t0 = time.monotonic()
    sb.run("hangs", 0.3, lambda: time.sleep(1.2))            # the real exit_fn is os._exit: here the block simply outlives its limit
    assert exits == [0] and time.monotonic() - t0 >= 1.0
    printed = json.loads(out.getvalue().strip())
    assert printed["value"] == 1.0 and printed["incomplete"] == ["hangs: watchdog timeout"]
    # the other ranks print nothing and exit too
    out2, exits2 = io.StringIO(), []
    bench.SecondaryBlocks(1, None, budget_s=10.0, exit_fn=exits2.append, out=out2).run("hangs", 0.2, lambda: time.sleep(0.6))
    assert exits2 == [0] and out2.getvalue() == ""


def test_roofline_traffic_is_parsed_from_the_newest_ncu_summary(tmp_path):
    assert bench.conv_traffic_from_profile(str(tmp_path)) == (None, None)   # no capture: no traffic figure
    prof = tmp_path / "profiles"
    prof.mkdir()
    rows = [["Section Name", "Metric Name", "Metric Unit", "Metric Value"],
            ["Memory", "dram__bytes_read.sum", "Mbyte", "51.04"], ["Memory", "dram__bytes_write.sum", "Kbyte", "3,300"]]
    (prof / "r01_prof_conv_a_summary.csv").write_text("Memory,dram__bytes_read.sum,byte,1\nMemory,dram__bytes_write.sum,byte,2\n")
    (prof / "r02_prof_conv_b_summary.csv").write_text("\n".join(",".join(f'"{c}"' if "," in c else c for c in r) for r in rows) + "\n")
    traffic, src = bench.conv_traffic_from_profile(str(tmp_path))
    assert src == "profiles/r02_prof_conv_b_summary.csv"
    assert traffic == 51.04e6 + 3.3e6
