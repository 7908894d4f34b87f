"""Construction of `protobuf_to_arrow` / `arrow_to_protobuf` (processor/protobuf.rs:71-95, 197-232 and
component/protobuf.rs:41-113): configuration shape, `.proto` discovery, parsing, type resolution and message lookup all
happen on the host, so every error is checked here without a GPU."""
import pytest

from arkflow_b200.processor import (ArkError, ArrowToProtobufProcessor, ProtobufToArrowProcessor, build_processor, init)

BOTH = (ProtobufToArrowProcessor, ArrowToProtobufProcessor)


def write(d, name, text):
    d.mkdir(parents=True, exist_ok=True)
    (d / name).write_text(text)
    return d


def cfg(d, message="pkg.M", **kw):
    return {"proto_inputs": [str(d)], "message_type": message, **kw}


def expect(cls, config, kind, prefix):
    with pytest.raises(ArkError) as e:
        cls(config)
    assert e.value.kind == kind, e.value.message
    assert e.value.message.startswith(prefix), e.value.message
    return e.value.message


SIMPLE = 'syntax = "proto3";\npackage pkg;\nmessage M { int64 timestamp = 1; double value = 2; string sensor = 3; }\n'


def test_missing_configuration(lib):
    expect(ProtobufToArrowProcessor, None, "Config", "ProtobufToArrow processor configuration is missing")
    expect(ArrowToProtobufProcessor, None, "Config", "ArrowToProtobuf processor configuration is missing")


@pytest.mark.parametrize("cls", BOTH)
def test_shape_errors_are_serialization(lib, tmp_path, cls):
    d = write(tmp_path / "p", "m.proto", SIMPLE)
    for bad in ({"proto_inputs": [str(d)]}, {"message_type": "pkg.M"}, {"proto_inputs": str(d), "message_type": "pkg.M"},
                {"proto_inputs": [str(d)], "message_type": 3}, {"proto_inputs": [1], "message_type": "pkg.M"},
                {"proto_inputs": [str(d)], "message_type": "pkg.M", "proto_includes": "x"}, []):
        expect(cls, bad, "Serialization", "")
    expect(ProtobufToArrowProcessor, cfg(d, value_field=5), "Serialization", "")
    expect(ArrowToProtobufProcessor, cfg(d, fields_to_include="sensor"), "Serialization", "")


@pytest.mark.parametrize("cls", BOTH)
def test_no_proto_files(lib, tmp_path, cls):
    write(tmp_path / "empty", "notes.txt", "message M {}")
    write(tmp_path / "empty" / "sub", "deeper.proto", SIMPLE)  # subdirectories are not searched
    for dirs in ([str(tmp_path / "empty")], [str(tmp_path / "does_not_exist")], []):
        expect(cls, {"proto_inputs": dirs, "message_type": "pkg.M"}, "Config", "No proto files found in the specified paths")


@pytest.mark.parametrize("text", [
    "syntax = \"proto3\";\npackage pkg;\nmessage M { int64 x = 1 }\n",                       # missing ';'
    "syntax = \"proto3\";\npackage pkg;\nmessage M { Missing x = 1; }\n",                    # unresolvable type
    "syntax = \"proto3\";\npackage pkg;\nmessage M { int32 x = 1; int32 y = 1; }\n",         # duplicate number
    "syntax = \"proto3\";\npackage pkg;\nmessage M { int32 x = 1 [default = 3]; }\n",        # defaults are proto2 only
    "syntax = \"proto2\";\npackage pkg;\nmessage M { int32 x = 1; }\n",                      # proto2 needs a label
    "syntax = \"proto4\";\nmessage M {}\n",
    "syntax = \"proto3\";\npackage pkg;\nmessage M { int32 x = 0; }\n",
    "syntax = \"proto3\";\npackage pkg;\n/* unterminated comment\nmessage M {}\n",
    "syntax = \"proto3\";\npackage pkg;\nimport \"google/protobuf/timestamp.proto\";\nmessage M { google.protobuf.Timestamp t = 1; }\n",
    "syntax = \"proto2\";\npackage pkg;\nenum E { A = 1; }\nmessage M { optional E e = 1 [default = B]; }\n",
    "syntax = \"proto3\";\npackage pkg;\nmessage A { message B {} }\nmessage M { B b = 1; }\n",  # B is only visible inside A
])
def test_parse_and_resolution_failures(lib, tmp_path, text):
    d = write(tmp_path / "p", "m.proto", text)
    for cls in BOTH:
        expect(cls, cfg(d), "Config", "Failed to parse the proto file: ")


def test_unknown_message(lib, tmp_path):
    d = write(tmp_path / "p", "m.proto", SIMPLE)
    for cls in BOTH:
        msg = expect(cls, cfg(d, "pkg.Nope"), "Config", "The message type could not be found: pkg.Nope")
        assert msg == "The message type could not be found: pkg.Nope"
        expect(cls, cfg(d, "M"), "Config", "The message type could not be found: M")  # names are fully qualified


def test_parser_accepts_the_language(lib, tmp_path):
    inc = tmp_path / "inc"
    write(inc / "dep", "shared.proto", 'syntax = "proto3";\npackage dep.v1;\nmessage Shared { sint32 v = 1; }\nenum Level { LOW = 0; HIGH = 1; }\n')
    write(inc / "dep", "weak.proto", 'syntax = "proto2";\npackage dep.v1;\nmessage Weak { optional int32 w = 1; }\n')
    d = write(tmp_path / "p", "main.proto", r'''
// line comment
syntax = "proto2";   /* block
comment */
package pkg.sub;
import public "dep/shared.proto";
import weak "dep/weak.proto";
option java_package = "com.example";
option (my.custom) = { a: 1 b: "x" };

message Outer {
  option deprecated = true;
  optional int32 a = 1 [default = -0x10, deprecated = true];
  required string s = 2 [default = "t\x41b\101é" " more"];
  optional Color c = 3 [default = BLUE];
  enum Color { option allow_alias = true; RED = 1; BLUE = 2; AZURE = 2; }
  message Inner {
    optional double d = 1 [default = -inf];
    optional Color c = 2;                  // Outer.Color, found from the enclosing scope
    optional .pkg.sub.Outer.Inner self = 3;
  }
  optional Inner inner = 4;
  oneof choice { int64 x = 5; string y = 6; }
  map<string, dep.v1.Shared> m = 7;
  repeated int32 r = 8 [packed = true];
  reserved 10 to 12, 15;
  reserved "old";
  extensions 100 to 199;
  optional group G = 9 { optional int32 q = 1; }
  optional dep.v1.Shared sh = 13;
  optional dep.v1.Level lv = 14 [default = HIGH];
  optional float f = 16 [default = nan];
  optional bool b = 17 [default = true];
  optional bytes z = 18 [default = "\000\377"];
  optional uint64 u = 19 [default = 18446744073709551615];
}
extend Outer { optional int32 ext = 100; }
service Svc { rpc Do(Outer) returns (Outer) { option deprecated = true; } }
message Other { optional Outer.Inner i = 1; optional sub.Outer o = 2; }
''')
    c = {"proto_inputs": [str(d)], "proto_includes": [str(d), str(inc)]}
    for cls in BOTH:
        for m in ("pkg.sub.Outer", "pkg.sub.Outer.Inner", "pkg.sub.Other", "pkg.sub.Outer.G", "dep.v1.Shared"):
            cls(dict(c, message_type=m))
    # without proto_includes the import is looked up under proto_inputs only
    expect(ProtobufToArrowProcessor, {"proto_inputs": [str(d)], "message_type": "pkg.sub.Outer"}, "Config",
           "Failed to parse the proto file: ")
    # proto3 features: optional, no labels
    d3 = write(tmp_path / "p3", "m.proto", 'syntax = "proto3";\npackage a.b;\nmessage M { optional int32 x = 1; int32 y = 2; }\n')
    ProtobufToArrowProcessor(cfg(d3, "a.b.M"))


def test_registry_builds_both(lib, tmp_path):
    d = write(tmp_path / "p", "m.proto", SIMPLE)
    init()
    assert isinstance(build_processor({"type": "protobuf_to_arrow", **cfg(d)}), ProtobufToArrowProcessor)
    assert isinstance(build_processor({"type": "arrow_to_protobuf", **cfg(d), "fields_to_include": ["sensor"]}), ArrowToProtobufProcessor)
    with pytest.raises(ArkError) as e:
        build_processor({"type": "protobuf_to_arrow"})
    assert e.value.kind == "Config"
