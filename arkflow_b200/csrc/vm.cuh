// vm.cuh — device-side interpreter for VmProgram (see vm.h for the semantics being restated).
#pragma once
#include "bitmap.cuh"
#include "vm.h"

namespace ark {

struct VmVal {
  uint64_t bits;
  bool valid;
};

// IEEE-754 totalOrder key: monotone map from f64 bits to int64 (arrow-rs f64::total_cmp).
__device__ __forceinline__ int64_t f64_total_key(uint64_t bits) {
  int64_t s = (int64_t)bits;
  return s ^ (int64_t)(((uint64_t)(s >> 63)) >> 1);
}

__device__ __forceinline__ bool cmp_apply(int32_t cmp, int c /* -1,0,1 */) {
  switch (cmp) {
    case CMP_EQ: return c == 0;
    case CMP_NE: return c != 0;
    case CMP_LT: return c < 0;
    case CMP_LE: return c <= 0;
    case CMP_GT: return c > 0;
    default: return c >= 0;
  }
}

__device__ __forceinline__ bool cmp_i64(int32_t cmp, int64_t a, int64_t b) {
  switch (cmp) {
    case CMP_EQ: return a == b;
    case CMP_NE: return a != b;
    case CMP_LT: return a < b;
    case CMP_LE: return a <= b;
    case CMP_GT: return a > b;
    default: return a >= b;
  }
}

// lexicographic byte comparison, shorter-is-smaller on a common prefix (arrow-ord on &[u8])
__device__ inline int bytes_cmp(const uint8_t* a, int32_t la, const uint8_t* b, int32_t lb) {
  int32_t n = la < lb ? la : lb;
  for (int32_t i = 0; i < n; ++i) {
    int d = (int)a[i] - (int)b[i];
    if (d != 0) return d < 0 ? -1 : 1;
  }
  return la < lb ? -1 : (la > lb ? 1 : 0);
}

static __device__ __noinline__ VmVal vm_eval(const VmProgram& prog, const ColView* cols, int64_t row, int32_t* err) {
  VmVal r[VM_MAX_REGS];
#pragma unroll 1
  for (int pc = 0; pc < prog.n_instr; ++pc) {
    const VmInstr in = prog.instr[pc];
    VmVal out;
    out.bits = 0;
    out.valid = true;
    switch (in.op) {
      case VM_LOAD_I64:
      case VM_LOAD_F64: {
        const ColView& c = cols[in.a];
        out.valid = col_valid(c, row);
        out.bits = out.valid ? ((const uint64_t*)c.data)[row] : 0;
        break;
      }
      case VM_LOAD_BOOL: {
        const ColView& c = cols[in.a];
        out.valid = col_valid(c, row);
        out.bits = out.valid ? (uint64_t)bit_get((const uint8_t*)c.data, row + c.data_bit0) : 0;
        break;
      }
      case VM_CONST: out.bits = prog.consts[in.aux]; break;
      case VM_NULL: out.valid = false; break;
      case VM_ADD_I64: out.valid = r[in.a].valid && r[in.b].valid; out.bits = r[in.a].bits + r[in.b].bits; break;
      case VM_SUB_I64: out.valid = r[in.a].valid && r[in.b].valid; out.bits = r[in.a].bits - r[in.b].bits; break;
      case VM_MUL_I64: out.valid = r[in.a].valid && r[in.b].valid; out.bits = r[in.a].bits * r[in.b].bits; break;
      case VM_DIV_I64:
      case VM_MOD_I64: {
        out.valid = r[in.a].valid && r[in.b].valid;
        if (out.valid) {
          int64_t x = (int64_t)r[in.a].bits, y = (int64_t)r[in.b].bits;
          if (y == 0) { *err = VMERR_DIV_ZERO; out.valid = false; }
          else if (x == INT64_MIN && y == -1) {
            *err = in.op == VM_DIV_I64 ? VMERR_OVERFLOW : VMERR_OVERFLOW_MOD;
            out.valid = false;
          } else out.bits = (uint64_t)(in.op == VM_DIV_I64 ? x / y : x % y);
        }
        break;
      }
      case VM_NEG_I64: out.valid = r[in.a].valid; out.bits = 0 - r[in.a].bits; break;
      case VM_ADD_F64: case VM_SUB_F64: case VM_MUL_F64: case VM_DIV_F64: case VM_MOD_F64: {
        out.valid = r[in.a].valid && r[in.b].valid;
        double x = __longlong_as_double((long long)r[in.a].bits), y = __longlong_as_double((long long)r[in.b].bits), z;
        if (in.op == VM_ADD_F64) z = x + y;
        else if (in.op == VM_SUB_F64) z = x - y;
        else if (in.op == VM_MUL_F64) z = x * y;
        else if (in.op == VM_DIV_F64) z = x / y;
        else z = fmod(x, y);
        out.bits = (uint64_t)__double_as_longlong(z);
        break;
      }
      case VM_NEG_F64: out.valid = r[in.a].valid; out.bits = r[in.a].bits ^ 0x8000000000000000ull; break;
      case VM_I64_TO_F64:
        out.valid = r[in.a].valid;
        out.bits = (uint64_t)__double_as_longlong((double)(int64_t)r[in.a].bits);
        break;
      case VM_F64_TO_I64: {
        out.valid = r[in.a].valid;
        if (out.valid) {
          double x = __longlong_as_double((long long)r[in.a].bits);
          // arrow-cast (safe=false): NaN / out-of-range is an error; in-range truncates toward zero
          if (!(x > -9223372036854777856.0 && x < 9223372036854775808.0)) { *err = VMERR_CAST; out.valid = false; }
          else out.bits = (uint64_t)(int64_t)x;
        }
        break;
      }
      case VM_BOOL_TO_I64: out.valid = r[in.a].valid; out.bits = r[in.a].bits & 1; break;
      case VM_I64_TO_BOOL: out.valid = r[in.a].valid; out.bits = r[in.a].bits != 0; break;
      case VM_F64_TO_BOOL:
        out.valid = r[in.a].valid;
        out.bits = __longlong_as_double((long long)r[in.a].bits) != 0.0;
        break;
      case VM_CMP_I64:
        out.valid = r[in.a].valid && r[in.b].valid;
        out.bits = cmp_i64(in.aux, (int64_t)r[in.a].bits, (int64_t)r[in.b].bits);
        break;
      case VM_CMP_F64:
        out.valid = r[in.a].valid && r[in.b].valid;
        out.bits = cmp_i64(in.aux, f64_total_key(r[in.a].bits), f64_total_key(r[in.b].bits));
        break;
      case VM_CMP_BOOL:
        out.valid = r[in.a].valid && r[in.b].valid;
        out.bits = cmp_i64(in.aux, (int64_t)(r[in.a].bits & 1), (int64_t)(r[in.b].bits & 1));
        break;
      case VM_CMP_STR_CONST: {
        const ColView& c = cols[in.a];
        out.valid = col_valid(c, row);
        if (out.valid) {
          int32_t o0 = c.offsets[row], o1 = c.offsets[row + 1];
          int cc = bytes_cmp((const uint8_t*)c.data + o0, o1 - o0, prog.str_bytes[in.b], prog.str_len[in.b]);
          out.bits = cmp_apply(in.aux, cc);
        }
        break;
      }
      case VM_CMP_STR_COL: {
        const ColView& ca = cols[in.a];
        const ColView& cb = cols[in.b];
        out.valid = col_valid(ca, row) && col_valid(cb, row);
        if (out.valid) {
          int32_t a0 = ca.offsets[row], a1 = ca.offsets[row + 1];
          int32_t b0 = cb.offsets[row], b1 = cb.offsets[row + 1];
          int cc = bytes_cmp((const uint8_t*)ca.data + a0, a1 - a0, (const uint8_t*)cb.data + b0, b1 - b0);
          out.bits = cmp_apply(in.aux, cc);
        }
        break;
      }
      case VM_AND: {  // Kleene
        bool av = r[in.a].valid, bv = r[in.b].valid;
        bool at = r[in.a].bits & 1, bt = r[in.b].bits & 1;
        if ((av && !at) || (bv && !bt)) { out.valid = true; out.bits = 0; }
        else if (av && bv) { out.valid = true; out.bits = 1; }
        else out.valid = false;
        break;
      }
      case VM_OR: {
        bool av = r[in.a].valid, bv = r[in.b].valid;
        bool at = r[in.a].bits & 1, bt = r[in.b].bits & 1;
        if ((av && at) || (bv && bt)) { out.valid = true; out.bits = 1; }
        else if (av && bv) { out.valid = true; out.bits = 0; }
        else out.valid = false;
        break;
      }
      case VM_NOT: out.valid = r[in.a].valid; out.bits = (r[in.a].bits & 1) ^ 1; break;
      case VM_IS_NULL: out.bits = !r[in.a].valid; break;
      case VM_IS_NOT_NULL: out.bits = r[in.a].valid; break;
      case VM_IS_NULL_COL: out.bits = !col_valid(cols[in.a], row); break;
      case VM_IS_NOT_NULL_COL: out.bits = col_valid(cols[in.a], row); break;
      default: break;
    }
    r[in.dst] = out;
  }
  return r[prog.result_reg];
}

}  // namespace ark
