"""The captioner's weight-only int8 mode on the host: the int8 header against its bindings and the library's exports,
the `--llava_int8` flag, the agent's `weights=` check, and the quantization rule on hand-made rows.  Nothing here
launches a kernel."""
import os
import re

import pytest

from llava_int8_cases import hand_rows, quantize_rows_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declarations(header: str) -> dict:
    src = re.sub(r"/\*.*?\*/", " ", open(os.path.join(ROOT, "include", header)).read(), flags=re.S)
    return dict(re.findall(r"\b(uav_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", src))


def test_int8_header_matches_bindings_and_exports(uav_lib):
    import ctypes as C
    from upscale_a_video_b200 import _lib
    decls = _declarations("uav_b200_int8.h")
    assert set(decls) == set(_lib.declared_int8_symbols()) == {"uav_quantize_rows_int8", "uav_dequantize_rows_int8",
                                                                "uav_gemv_rows_int8"}
    kinds = {"int": C.c_int, "int64_t": C.c_int64}
    for name, params in decls.items():
        assert hasattr(uav_lib, name), f"{name} declared in include/uav_b200_int8.h but not exported"
        want = [C.c_void_p if "*" in p or p.strip().startswith("uav_stream_t") else kinds[p.strip().rsplit(" ", 1)[0]]
                for p in params.split(",")]
        assert _lib._INT8_PROTOS[name] == want, name
    # the main header and its binding table are unchanged
    main = _declarations("uav_b200.h")
    assert len(main) == 64 and not set(main) & set(decls)
    assert set(main) == set(_lib.declared_symbols())
    assert uav_lib.uav_launch_count() == 0


def test_cli_llava_int8_flag(capsys):
    from upscale_a_video_b200 import cli
    a = cli.parse_args(["--llava_path", "L", "--llava_int8"])
    assert a.llava_int8 and cli.use_llava(a)
    assert not cli.parse_args(["--llava_path", "L"]).llava_int8
    for argv in (["--llava_int8"], ["--llava_path", "L", "--no_llava", "--llava_int8"]):
        capsys.readouterr()
        with pytest.raises(SystemExit):
            cli.parse_args(argv)
        assert "--llava_int8 needs the captioner" in capsys.readouterr().err
    with pytest.raises(SystemExit):
        cli.parse_args(["--llava_path", "L", "--load_8bit_llava", "--llava_int8"])
    err = capsys.readouterr().err
    assert "no LLaVA captioner" in err and "--llava_int8" in err


def test_agent_weights_checked_before_loading(tmp_path):
    from upscale_a_video_b200 import LLavaAgent
    from upscale_a_video_b200.llava import load_decoder
    missing = str(tmp_path / "no-such-model")
    for bad in ("int4", "fp32", None):
        with pytest.raises(ValueError, match="weights="):
            LLavaAgent(missing, weights=bad)
    with pytest.raises(ValueError, match="weights="):
        load_decoder(missing, None, "cpu", weights="int4")
    with pytest.raises(NotImplementedError, match="weights='int8'"):
        LLavaAgent(missing, load_8bit=True)


def test_quantization_rule_on_hand_made_rows():
    w, expect = hand_rows()
    q, s = quantize_rows_ref(w)
    assert q.dtype == expect.dtype and q.tolist() == expect.tolist()
    assert s.tolist() == w.float().abs().amax(1).tolist()
    # spot checks of the rows' intent: ties to even, zero row, negative absmax, the fp16 extremes, subnormals
    assert q[0, :10].tolist() == [127, 0, 2, 2, 0, -2, -2, 126, 4, -126]
    assert not q[1].any() and s[1] == 0
    assert q[3, :4].tolist() == [-127, 42, 85, -64]
    assert q[4, :5].tolist() == [127, -127, 64, 0, -32]
    assert q[5, 6] == 127 and s[5] == 1023 * 2.0 ** -24
