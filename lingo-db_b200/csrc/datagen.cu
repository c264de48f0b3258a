// datagen.cu — device twin of the deterministic TPC-H-shaped generator (tpch_gen.h): fills Arrow
// physical column buffers directly in HBM so SF100 tables never cross PCIe.  Bit-identical to
// datagen_host.cpp (tests/test_gpu_datagen.py).  Not on the query hot path.
#include "context.h"
#include "tpch_gen.h"
#include "dbgen_gen.h"
#include "../../include/ldb_datagen.h"

using namespace ldbgen;

namespace {
Scale toScale(const LdbGenScale* g) {
   Scale s;
   s.seed = g->seed;
   s.nOrders = g->n_orders;
   s.nCustomer = g->n_customer;
   s.nSupplier = g->n_supplier;
   s.nPart = g->n_part;
   return s;
}
__device__ __forceinline__ void storeDec(uint8_t* col, int64_t i, int64_t v) {
   longlong2 x;
   x.x = v;
   x.y = v >> 63;
   reinterpret_cast<longlong2*>(col)[i] = x;
}
__global__ void lineitemKernel(Scale s, int64_t rowBegin, int64_t n, LdbGenLineitemCols c) {
   for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) {
      LineItem l = lineItem(s, rowBegin + i);
      if (c.l_orderkey) c.l_orderkey[i] = l.orderkey;
      if (c.l_partkey) c.l_partkey[i] = l.partkey;
      if (c.l_suppkey) c.l_suppkey[i] = l.suppkey;
      if (c.l_quantity) storeDec(c.l_quantity, i, l.quantity);
      if (c.l_extendedprice) storeDec(c.l_extendedprice, i, l.extendedprice);
      if (c.l_discount) storeDec(c.l_discount, i, l.discount);
      if (c.l_tax) storeDec(c.l_tax, i, l.tax);
      if (c.l_returnflag) c.l_returnflag[i] = l.returnflag;
      if (c.l_linestatus) c.l_linestatus[i] = l.linestatus;
      if (c.l_shipdate) c.l_shipdate[i] = l.shipdate;
      if (c.l_commitdate) c.l_commitdate[i] = l.commitdate;
      if (c.l_receiptdate) c.l_receiptdate[i] = l.receiptdate;
   }
}
__global__ void ordersKernel(Scale s, int64_t rowBegin, int64_t n, LdbGenOrdersCols c) {
   for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) {
      int64_t o = rowBegin + i;
      if (c.o_orderkey) c.o_orderkey[i] = orderKey(o);
      if (c.o_custkey) c.o_custkey[i] = orderCustKey(s, o);
      if (c.o_orderdate) c.o_orderdate[i] = orderDate(s, o);
      if (c.o_shippriority) c.o_shippriority[i] = orderShipPriority(s, o);
   }
}
__global__ void customerFixedKernel(Scale s, int64_t rowBegin, int64_t n, LdbGenCustomerCols c, int32_t* segLengths) {
   for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) {
      int64_t r = rowBegin + i;
      if (c.c_custkey) c.c_custkey[i] = (int32_t) (r + 1);
      if (c.c_nationkey) c.c_nationkey[i] = customerNationKey(s, r);
      if (segLengths) segLengths[i] = segmentLen(customerSegment(s, r));
   }
}
__global__ void customerBytesKernel(Scale s, int64_t rowBegin, int64_t n, const int32_t* offsets, uint8_t* data) {
   for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) {
      int32_t seg = customerSegment(s, rowBegin + i);
      int32_t len = segmentLen(seg), off = offsets[i];
      for (int32_t k = 0; k < len; k++) data[off + k] = (uint8_t) segmentChar(seg, k);
   }
}
__global__ void supplierKernel(Scale s, int64_t rowBegin, int64_t n, LdbGenSupplierCols c) {
   for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) {
      int64_t r = rowBegin + i;
      if (c.s_suppkey) c.s_suppkey[i] = (int32_t) (r + 1);
      if (c.s_nationkey) c.s_nationkey[i] = supplierNationKey(s, r);
   }
}
__global__ void partFixedKernel(Scale s, int64_t rowBegin, int64_t n, LdbGenPartCols c, int32_t* nameLengths) {
   for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) {
      int64_t r = rowBegin + i;
      if (c.p_partkey) c.p_partkey[i] = (int32_t) (r + 1);
      if (nameLengths) nameLengths[i] = partNameLen(s, r);
   }
}
__global__ void partBytesKernel(Scale s, int64_t rowBegin, int64_t n, const int32_t* offsets, uint8_t* data) {
   for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) partNameWrite(s, rowBegin + i, data + offsets[i]);
}
__global__ void partsuppKernel(Scale s, int64_t rowBegin, int64_t n, LdbGenPartsuppCols c) {
   for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) {
      int64_t r = rowBegin + i;
      if (c.ps_partkey) c.ps_partkey[i] = partSuppPartKey(r);
      if (c.ps_suppkey) c.ps_suppkey[i] = partSuppSuppKey(s, r);
      if (c.ps_supplycost) storeDec(c.ps_supplycost, i, partSuppSupplyCost(s, r));
   }
}
// ---- dbgen-faithful variant (dbgen_gen.h): one thread per ORDER for lineitem (1..7 lines at the order's first row)
__global__ void dbgenLineCountsKernel(int64_t orderBegin, int64_t n, int32_t* counts) {
   for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) counts[i] = ldbdbgen::orderLineCount(orderBegin + i);
}
__global__ void dbgenLineitemKernel(ldbdbgen::Scale s, int64_t orderBegin, int64_t n, const int64_t* firstRow, LdbGenLineitemCols c) {
   for (int64_t o = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; o < n; o += (int64_t) gridDim.x * blockDim.x) {
      ldbdbgen::Line lines[7];
      const int32_t cnt = ldbdbgen::orderLines(s, orderBegin + o, lines);
      const int32_t key = ldbdbgen::orderKey(orderBegin + o);
      for (int32_t k = 0; k < cnt; k++) {
         const int64_t i = firstRow[o] + k;
         const ldbdbgen::Line& l = lines[k];
         if (c.l_orderkey) c.l_orderkey[i] = key;
         if (c.l_partkey) c.l_partkey[i] = l.partkey;
         if (c.l_suppkey) c.l_suppkey[i] = l.suppkey;
         if (c.l_quantity) storeDec(c.l_quantity, i, l.quantity);
         if (c.l_extendedprice) storeDec(c.l_extendedprice, i, l.extendedprice);
         if (c.l_discount) storeDec(c.l_discount, i, l.discount);
         if (c.l_tax) storeDec(c.l_tax, i, l.tax);
         if (c.l_returnflag) c.l_returnflag[i] = l.returnflag;
         if (c.l_linestatus) c.l_linestatus[i] = l.linestatus;
         if (c.l_shipdate) c.l_shipdate[i] = l.shipdate;
         if (c.l_commitdate) c.l_commitdate[i] = l.commitdate;
         if (c.l_receiptdate) c.l_receiptdate[i] = l.receiptdate;
      }
   }
}
__global__ void dbgenOrdersKernel(ldbdbgen::Scale s, int64_t rowBegin, int64_t n, LdbGenOrdersCols c) {
   for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) {
      const int64_t o = rowBegin + i;
      if (c.o_orderkey) c.o_orderkey[i] = ldbdbgen::orderKey(o);
      if (c.o_custkey) c.o_custkey[i] = ldbdbgen::orderCustKey(s, o);
      if (c.o_orderdate) c.o_orderdate[i] = ldbdbgen::orderDateRaw(o) - ldbdbgen::kEpochOffset;
      if (c.o_shippriority) c.o_shippriority[i] = 0;
   }
}
// table: 0 customer (fixed columns + segment lengths), 1 supplier, 2 part (key + name lengths), 3 partsupp
__global__ void dbgenSmallFixedKernel(ldbdbgen::Scale s, int table, int64_t rowBegin, int64_t n, int32_t* key, int32_t* second, uint8_t* dec, int32_t* lengths) {
   for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) {
      const int64_t r = rowBegin + i;
      if (table == 0) {
         if (key) key[i] = (int32_t) (r + 1);
         if (second) second[i] = ldbdbgen::customerNationKey(r);
         if (lengths) lengths[i] = ldbdbgen::segmentLen(ldbdbgen::customerSegment(r));
      } else if (table == 1) {
         if (key) key[i] = (int32_t) (r + 1);
         if (second) second[i] = ldbdbgen::supplierNationKey(r);
      } else if (table == 2) {
         if (key) key[i] = (int32_t) (r + 1);
         if (lengths) lengths[i] = ldbdbgen::partNameLen(r);
      } else {
         if (key) key[i] = (int32_t) (r / 4 + 1);
         if (second) second[i] = ldbdbgen::partSuppSuppKey(s, r);
         if (dec) storeDec(dec, i, ldbdbgen::partSuppSupplyCost(r));
      }
   }
}
// table: 0 customer c_mktsegment bytes, 2 part p_name bytes
__global__ void dbgenBytesKernel(int table, int64_t rowBegin, int64_t n, const int32_t* offsets, uint8_t* data) {
   for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) {
      if (table == 0) {
         const int32_t seg = ldbdbgen::customerSegment(rowBegin + i), len = ldbdbgen::segmentLen(seg), off = offsets[i];
         for (int32_t k = 0; k < len; k++) data[off + k] = (uint8_t) ldbdbgen::segmentChar(seg, k);
      } else {
         ldbdbgen::partNameWrite(rowBegin + i, data + offsets[i]);
      }
   }
}
int gridFor(LdbContext* ctx, int64_t n) { return (int) std::min<int64_t>(std::max<int64_t>((n + 255) / 256, 1), (int64_t) ctx->smCount * 16); }
} // namespace
using ldb::guarded;

extern "C" {
int ldb_gpu_datagen_lineitem(LdbContext* ctx, const LdbGenScale* g, int64_t row_begin, int64_t n_rows, const LdbGenLineitemCols* c, LdbError* err) {
   return guarded(err, [&] {
      LDB_CUDA(cudaSetDevice(ctx->device));
      lineitemKernel<<<gridFor(ctx, n_rows), 256, 0, ctx->compute>>>(toScale(g), row_begin, n_rows, *c);
      LDB_CUDA(cudaGetLastError());
   });
}
int ldb_gpu_datagen_orders(LdbContext* ctx, const LdbGenScale* g, int64_t row_begin, int64_t n_rows, const LdbGenOrdersCols* c, LdbError* err) {
   return guarded(err, [&] {
      LDB_CUDA(cudaSetDevice(ctx->device));
      ordersKernel<<<gridFor(ctx, n_rows), 256, 0, ctx->compute>>>(toScale(g), row_begin, n_rows, *c);
      LDB_CUDA(cudaGetLastError());
   });
}
int ldb_gpu_datagen_customer_fixed(LdbContext* ctx, const LdbGenScale* g, int64_t row_begin, int64_t n_rows, const LdbGenCustomerCols* c, int32_t* dev_seg_lengths, LdbError* err) {
   return guarded(err, [&] {
      LDB_CUDA(cudaSetDevice(ctx->device));
      customerFixedKernel<<<gridFor(ctx, n_rows), 256, 0, ctx->compute>>>(toScale(g), row_begin, n_rows, *c, dev_seg_lengths);
      LDB_CUDA(cudaGetLastError());
   });
}
int ldb_gpu_datagen_customer_bytes(LdbContext* ctx, const LdbGenScale* g, int64_t row_begin, int64_t n_rows, const int32_t* dev_offsets, uint8_t* dev_data, LdbError* err) {
   return guarded(err, [&] {
      LDB_CUDA(cudaSetDevice(ctx->device));
      customerBytesKernel<<<gridFor(ctx, n_rows), 256, 0, ctx->compute>>>(toScale(g), row_begin, n_rows, dev_offsets, dev_data);
      LDB_CUDA(cudaGetLastError());
   });
}
int ldb_gpu_datagen_supplier(LdbContext* ctx, const LdbGenScale* g, int64_t row_begin, int64_t n_rows, const LdbGenSupplierCols* c, LdbError* err) {
   return guarded(err, [&] {
      LDB_CUDA(cudaSetDevice(ctx->device));
      supplierKernel<<<gridFor(ctx, n_rows), 256, 0, ctx->compute>>>(toScale(g), row_begin, n_rows, *c);
      LDB_CUDA(cudaGetLastError());
   });
}
int ldb_gpu_datagen_part_fixed(LdbContext* ctx, const LdbGenScale* g, int64_t row_begin, int64_t n_rows, const LdbGenPartCols* c, int32_t* dev_name_lengths, LdbError* err) {
   return guarded(err, [&] {
      LDB_CUDA(cudaSetDevice(ctx->device));
      partFixedKernel<<<gridFor(ctx, n_rows), 256, 0, ctx->compute>>>(toScale(g), row_begin, n_rows, *c, dev_name_lengths);
      LDB_CUDA(cudaGetLastError());
   });
}
int ldb_gpu_datagen_part_bytes(LdbContext* ctx, const LdbGenScale* g, int64_t row_begin, int64_t n_rows, const int32_t* dev_offsets, uint8_t* dev_data, LdbError* err) {
   return guarded(err, [&] {
      LDB_CUDA(cudaSetDevice(ctx->device));
      partBytesKernel<<<gridFor(ctx, n_rows), 256, 0, ctx->compute>>>(toScale(g), row_begin, n_rows, dev_offsets, dev_data);
      LDB_CUDA(cudaGetLastError());
   });
}
int ldb_gpu_datagen_partsupp(LdbContext* ctx, const LdbGenScale* g, int64_t row_begin, int64_t n_rows, const LdbGenPartsuppCols* c, LdbError* err) {
   return guarded(err, [&] {
      LDB_CUDA(cudaSetDevice(ctx->device));
      partsuppKernel<<<gridFor(ctx, n_rows), 256, 0, ctx->compute>>>(toScale(g), row_begin, n_rows, *c);
      LDB_CUDA(cudaGetLastError());
   });
}
// ---- dbgen-faithful variant
static ldbdbgen::Scale toDbgenScale(const LdbGenScale* g) { return ldbdbgen::Scale{g->n_orders, g->n_customer, g->n_supplier, g->n_part}; }
int ldb_gpu_dbgen_line_counts(LdbContext* ctx, const LdbGenScale*, int64_t order_begin, int64_t n_orders, int32_t* dev_counts, LdbError* err) {
   return guarded(err, [&] {
      LDB_CUDA(cudaSetDevice(ctx->device));
      dbgenLineCountsKernel<<<gridFor(ctx, n_orders), 256, 0, ctx->compute>>>(order_begin, n_orders, dev_counts);
      LDB_CUDA(cudaGetLastError());
   });
}
int ldb_gpu_dbgen_lineitem(LdbContext* ctx, const LdbGenScale* g, int64_t order_begin, int64_t n_orders, const int64_t* dev_first_row, const LdbGenLineitemCols* c, LdbError* err) {
   return guarded(err, [&] {
      LDB_CUDA(cudaSetDevice(ctx->device));
      dbgenLineitemKernel<<<gridFor(ctx, n_orders), 256, 0, ctx->compute>>>(toDbgenScale(g), order_begin, n_orders, dev_first_row, *c);
      LDB_CUDA(cudaGetLastError());
   });
}
int ldb_gpu_dbgen_orders(LdbContext* ctx, const LdbGenScale* g, int64_t row_begin, int64_t n_rows, const LdbGenOrdersCols* c, LdbError* err) {
   return guarded(err, [&] {
      LDB_CUDA(cudaSetDevice(ctx->device));
      dbgenOrdersKernel<<<gridFor(ctx, n_rows), 256, 0, ctx->compute>>>(toDbgenScale(g), row_begin, n_rows, *c);
      LDB_CUDA(cudaGetLastError());
   });
}
int ldb_gpu_dbgen_small_fixed(LdbContext* ctx, const LdbGenScale* g, int32_t table, int64_t row_begin, int64_t n_rows, int32_t* dev_key, int32_t* dev_second, uint8_t* dev_decimal, int32_t* dev_lengths, LdbError* err) {
   return guarded(err, [&] {
      LDB_CUDA(cudaSetDevice(ctx->device));
      dbgenSmallFixedKernel<<<gridFor(ctx, n_rows), 256, 0, ctx->compute>>>(toDbgenScale(g), table, row_begin, n_rows, dev_key, dev_second, dev_decimal, dev_lengths);
      LDB_CUDA(cudaGetLastError());
   });
}
int ldb_gpu_dbgen_bytes(LdbContext* ctx, const LdbGenScale*, int32_t table, int64_t row_begin, int64_t n_rows, const int32_t* dev_offsets, uint8_t* dev_data, LdbError* err) {
   return guarded(err, [&] {
      LDB_CUDA(cudaSetDevice(ctx->device));
      dbgenBytesKernel<<<gridFor(ctx, n_rows), 256, 0, ctx->compute>>>(table, row_begin, n_rows, dev_offsets, dev_data);
      LDB_CUDA(cudaGetLastError());
   });
}
}
