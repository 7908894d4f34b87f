// abi.h — the contract every extern "C" entry point of include/arkflow_b200.h keeps:
//  * no exception leaves it: guarded() turns one into an ark_status and the thread-local message of ark_last_error;
//  * a moved-in ArrowArray / ArrowDeviceArray is adopted (adopt_array) BEFORE the guard, so it is released on every path,
//    and a released one is rejected by adopted() / device_view();
//  * a processor handle of the wrong type is rejected by proc_of();
//  * `out` / `out_schema` are zeroed on entry (zero_out), so an early return is ProcessResult::None.
#pragma once
#include <cstring>
#include <memory>
#include <new>
#include <string>

#include "engine.h"

struct ark_proc {
  std::unique_ptr<ark::Processor> impl;
};

namespace ark {

template <typename F>
int guarded(F&& f) {
  try {
    f();
    return ARK_OK;
  } catch (const ArkError& e) {
    set_last_error(e.what());
    return e.code;
  } catch (const std::bad_alloc&) {
    set_last_error("out of host memory");
    return ARK_ERR_PROCESS;
  } catch (const std::exception& e) {
    set_last_error(e.what());
    return ARK_ERR_PROCESS;
  }
}

// The array an entry point adopted from its caller.
inline const ArrowArray* adopted(const BufferPtr& owner) {
  if (!owner) fail(ARK_ERR_PROCESS, "input array already released");
  return (const ArrowArray*)owner.get();
}

// `in` with its array replaced by the adopted one (adopt_array left `in->array` released).
inline ArrowDeviceArray device_view(const ArrowDeviceArray& in, const BufferPtr& owner) {
  ArrowDeviceArray view = in;
  view.array = *adopted(owner);
  return view;
}

inline Processor* proc_of(ark_proc_t* p, const char* type) {
  if (!p || !p->impl || strcmp(p->impl->type(), type) != 0)
    fail(ARK_ERR_PROCESS, std::string(strchr("aeiou", type[0]) ? "handle is not an " : "handle is not a ") + type + " processor");
  return p->impl.get();
}

inline SqlProcessor* as_sql(ark_proc_t* p) { return static_cast<SqlProcessor*>(proc_of(p, "sql")); }

template <typename Out>  // ArrowArray or ArrowDeviceArray
void zero_out(Out* out, ArrowSchema* out_schema) {
  if (out) memset(out, 0, sizeof(*out));
  if (out_schema) memset(out_schema, 0, sizeof(*out_schema));
}

}  // namespace ark
