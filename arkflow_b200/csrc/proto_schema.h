// proto_schema.h — message descriptors read from `.proto` files, for the protobuf_to_arrow / arrow_to_protobuf
// processors (csrc/protobuf.cu).  Stands in for component::protobuf::parse_proto_file
// (crates/arkflow-plugin/src/component/protobuf.rs:41-113: protobuf-parse's pure parser + typecheck) and
// prost-reflect's DescriptorPool::get_message_by_name (processor/protobuf.rs:73-95).  Host code only: building a
// descriptor needs no CUDA device.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

namespace ark {

// FieldDescriptorProto.Type numbering
enum class PbKind : uint8_t {
  Double = 1, Float = 2, Int64 = 3, UInt64 = 4, Int32 = 5, Fixed64 = 6, Fixed32 = 7, Bool = 8, String = 9,
  Group = 10, Message = 11, Bytes = 12, UInt32 = 13, Enum = 14, SFixed32 = 15, SFixed64 = 16, SInt32 = 17, SInt64 = 18
};

struct PbField {
  std::string name;
  int32_t number = 0;
  PbKind kind = PbKind::Int32;
  bool repeated = false;     // `repeated` and map fields
  bool is_map = false;
  bool presence = false;     // explicit presence: proto2 optional / required, proto3 `optional`, oneof members
  int oneof = -1;            // index of the declared oneof that holds the field, else -1
  std::string type_name;     // message / group / enum: the fully qualified name
  // the value of an absent field: proto2's [default = …], else zero / false / "" / the enum's first value
  uint64_t default_bits = 0; // integers and bool as their two's-complement value; float / double as IEEE bits
  std::string default_bytes; // string / bytes
};

struct PbMessage {
  std::string full_name;
  std::vector<PbField> fields;  // in declaration order
};

// Reads every `*.proto` file directly inside each directory of `inputs` (imports resolved against `includes`) and
// returns the message named `message_type` (fully qualified, e.g. "pkg.Outer.Inner").  Raises ArkError Config with the
// reference's messages: "No proto files found in the specified paths…", "Failed to parse the proto file: …",
// "The message type could not be found: …".
PbMessage load_proto_message(const std::vector<std::string>& inputs, const std::vector<std::string>& includes,
                             const std::string& message_type);

// prost-reflect's Kind name of a field, e.g. "Int32", "Message(pkg.M)"
std::string pb_kind_debug(const PbField& f);

}  // namespace ark
