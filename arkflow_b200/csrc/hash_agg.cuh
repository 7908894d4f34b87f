// hash_agg.cuh — parameter blocks of the GROUP BY hash-aggregate kernels.
#pragma once
#include "vm.h"

namespace ark {

// 16-byte group key word stored in the table.  Utf8/Binary keys up to 12 bytes live inline
// ("German string": 12 bytes + u32 length); longer keys store a 4-byte prefix + the row index of
// the first row that inserted them (their bytes are compared against that row of the input).
struct __align__(16) Key16 {
  unsigned long long lo, hi;
};

constexpr unsigned long long KEY_EMPTY = 0xFFFFFFFFFFFFFFFFull;  // lo == hi == KEY_EMPTY ⇒ empty slot
constexpr unsigned KEYTAG_NULL = 0xFFFFFFFEu;                    // tag (top 32 bits of hi) of the NULL key
constexpr unsigned KEYTAG_LONG = 0x80000000u;                    // | length for keys longer than 12 bytes
constexpr unsigned KEYTAG_INT = 0x40000000u;                     // Int64 / Bool key: lo = value
constexpr unsigned KEYTAG_PAIR = 0x20000000u;                    // two GROUP BY keys: lo = row that first held the pair, low 32 bits of hi = top
                                                                 // 32 bits of the pair's hash (compared first; also decides the owner rank)

// Table layout.  Slot s lives in bucket s / 4, lane s % 4.  A bucket is
//   [Key16 key[4]]  (64 bytes = two 32-byte sectors)  followed by  [u64 acc_a[4]] (one sector) per accumulator a,
// i.e. 128 bytes — one cache line — for the usual two accumulators.  A probe reads the four keys of a bucket at once
// (two 128-bit requests, one per sector) instead of walking 32-byte slots one L2 round trip at a time: at load 0.48 the longest
// chain among the 32 lanes of a warp drops from 6.3 slot probes to 1.9 bucket probes (simulated, 10^6 keys in 2^21
// slots), and that longest chain is what a warp waits for.
constexpr int TBL_B = 4;
__host__ __device__ inline int table_bucket_stride(int n_acc) { return 64 + 32 * n_acc; }
__host__ __device__ inline unsigned long long table_bytes(unsigned long long capacity, int n_acc) {
  return (capacity / TBL_B) * (unsigned long long)table_bucket_stride(n_acc);
}
#ifdef __CUDACC__
static __device__ __forceinline__ Key16* tbl_key(uint8_t* t, unsigned long long s, int bstride) {
  return reinterpret_cast<Key16*>(t + (s >> 2) * (unsigned long long)bstride + (s & 3) * 16);
}
static __device__ __forceinline__ const Key16* tbl_key(const uint8_t* t, unsigned long long s, int bstride) {
  return reinterpret_cast<const Key16*>(t + (s >> 2) * (unsigned long long)bstride + (s & 3) * 16);
}
static __device__ __forceinline__ unsigned long long* tbl_acc(uint8_t* t, unsigned long long s, int a, int bstride) {
  return reinterpret_cast<unsigned long long*>(t + (s >> 2) * (unsigned long long)bstride + 64 + a * 32 + (s & 3) * 8);
}
static __device__ __forceinline__ const unsigned long long* tbl_acc(const uint8_t* t, unsigned long long s, int a, int bstride) {
  return reinterpret_cast<const unsigned long long*>(t + (s >> 2) * (unsigned long long)bstride + 64 + a * 32 + (s & 3) * 8);
}
#endif

enum AccKind : int32_t {
  ACC_COUNT_STAR = 0,
  ACC_COUNT,     // non-null values of arg
  ACC_SUM_I64,   // wrapping
  ACC_SUM_F64,   // arg converted to f64 when arg_is_f64 == 0 (AVG over Int64)
  ACC_MIN_I64, ACC_MAX_I64,
  ACC_MIN_F64, ACC_MAX_F64,  // on the totalOrder key
};

// COUNT(*) has no argument and COUNT(x) needs only x's validity; every other accumulator reads x's 8-byte values
__host__ __device__ inline bool acc_reads_values(int kind) { return kind != ACC_COUNT_STAR && kind != ACC_COUNT; }

enum KeyKind : int32_t { KEY_NONE = 0, KEY_INT64 = 1, KEY_BYTES = 2, KEY_BOOL = 3, KEY_PAIR = 4 /* two key columns */ };

constexpr int AGG_MAX_ACC = 8;
constexpr int AGG_MAX_PROGS = 2;

struct AccParam {
  int32_t kind;
  int32_t arg_slot;    // column slot, or -1
  int32_t arg_prog;    // program index, or -1
  int32_t arg_is_f64;  // type of the argument value
  int32_t acc_index;   // which accumulator lane of the table bucket (see "table layout" above)
  int32_t pad;
};

struct AggParams {
  int64_t n_rows;
  int32_t pred_kind;   // 0 none, 1 simple, 2 VM
  int32_t sp_slot, sp_cmp, sp_is_f64;
  uint64_t sp_const;
  int32_t key_kind;
  int32_t key_slot;
  int32_t n_acc;
  int32_t key_slot2;   // KEY_PAIR: the second key column; key_kind1 / key_kind2 = the kinds of the two columns
  int32_t key_kind1, key_kind2;
  ColView cols[MAX_COLS];
  AccParam accs[AGG_MAX_ACC];
  VmProgram pred;
  VmProgram progs[AGG_MAX_PROGS];
  uint8_t* table;            // capacity / 4 buckets of bucket_stride bytes (table layout above)
  unsigned long long mask;   // capacity - 1 (slots); bucket mask = mask >> 2
  int32_t bucket_stride;     // table_bucket_stride(n_acc)
  int32_t pad2;
  unsigned int* group_count; // number of occupied slots
  unsigned int max_groups;   // load-factor limit; beyond it the kernel raises `overflow`
  int32_t* overflow;
  int32_t* error;
  int32_t* long_seen;        // set when a key longer than 12 bytes (stored by row reference) was met: the table cannot outlive the batch
};

}  // namespace ark
