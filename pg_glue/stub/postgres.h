/*
 * pg_glue/stub/postgres.h -- a TYPE-CHECKING SHIM, not PostgreSQL.
 *
 * This image has no PostgreSQL headers (and no network), so the glue in pg_glue/ cannot be built against the
 * real server here.  To keep it honest C rather than prose, it is compiled with
 *     gcc -fsyntax-only -Wall -Werror -I pg_glue/stub -I include pg_glue/<file>.c     (tests/test_pg_glue.py)
 * against this one header, which declares -- with PostgreSQL 16-18's names, argument orders and field names --
 * exactly the server and Citus interfaces the glue touches.  Every other header under stub/ includes this one.
 * Declarations only; nothing here is copied code.  Where a Citus type is mirrored, the reference file:line is
 * given so that a maintainer can check the field lists when building against the real headers
 * (make -C pg_glue PG_CONFIG=... uses those and never sees this directory).
 */
#ifndef PG_GLUE_STUB_POSTGRES_H
#define PG_GLUE_STUB_POSTGRES_H

#include <stdbool.h>
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

/* ---- c.h ---- */
typedef uintptr_t Datum;
typedef unsigned int Oid;
typedef int16_t int16;
typedef int32_t int32;
typedef int64_t int64;
typedef uint8_t uint8;
typedef uint16_t uint16;
typedef uint32_t uint32;
typedef uint64_t uint64;
typedef size_t Size;
typedef int16 AttrNumber;
typedef uint32 BlockNumber;
typedef int Buffer;
typedef char *Pointer;
typedef struct varlena { char vl_len_[4]; char vl_dat[]; } varlena;
typedef varlena bytea;
typedef varlena text;
#define InvalidOid ((Oid) 0)
#define PGDLLEXPORT
#define pg_attribute_noreturn() __attribute__((noreturn))
#define PG_MODULE_MAGIC extern int pg_glue_module_magic
#define BLCKSZ 8192
#define Assert(x) ((void) 0)
#define Min(a, b) ((a) < (b) ? (a) : (b))
#define Max(a, b) ((a) > (b) ? (a) : (b))
#define lengthof(a) (sizeof(a) / sizeof((a)[0]))

/* ---- elog.h ---- */
#define ERROR 21
#define WARNING 19
#define NOTICE 18
#define DEBUG1 14
#define ERRCODE_FEATURE_NOT_SUPPORTED 1
#define ERRCODE_INTERNAL_ERROR 2
#define ERRCODE_DATA_CORRUPTED 3
#define ERRCODE_OUT_OF_MEMORY 4
#define ERRCODE_INVALID_PARAMETER_VALUE 5
int errcode(int sqlerrcode);
int errmsg(const char *fmt, ...) __attribute__((format(printf, 1, 2)));
int errdetail(const char *fmt, ...) __attribute__((format(printf, 1, 2)));
int errhint(const char *fmt, ...) __attribute__((format(printf, 1, 2)));
void pg_glue_ereport(int elevel, ...);
#define ereport(elevel, ...) pg_glue_ereport(elevel, __VA_ARGS__)
void elog(int elevel, const char *fmt, ...) __attribute__((format(printf, 2, 3)));

/* ---- palloc.h / memutils.h ---- */
typedef struct MemoryContextData *MemoryContext;
extern MemoryContext CurrentMemoryContext;
void *palloc(Size size);
void *palloc0(Size size);
void *repalloc(void *pointer, Size size);
void pfree(void *pointer);
char *pstrdup(const char *in);
MemoryContext MemoryContextSwitchTo(MemoryContext context);
MemoryContext AllocSetContextCreateInternal(MemoryContext parent, const char *name, Size minContextSize, Size initBlockSize, Size maxBlockSize);
#define ALLOCSET_DEFAULT_SIZES 0, 8 * 1024, 8 * 1024 * 1024
#define AllocSetContextCreate AllocSetContextCreateInternal
void MemoryContextDelete(MemoryContext context);
typedef void (*MemoryContextCallbackFunction)(void *arg);
typedef struct MemoryContextCallback { MemoryContextCallbackFunction func; void *arg; struct MemoryContextCallback *next; } MemoryContextCallback;
void MemoryContextRegisterResetCallback(MemoryContext context, MemoryContextCallback *cb);

/* ---- postgres.h Datum conversions ---- */
#define DatumGetInt64(X) ((int64) (X))
#define Int64GetDatum(X) ((Datum) (X))
#define DatumGetInt32(X) ((int32) (X))
#define Int32GetDatum(X) ((Datum) (X))
#define DatumGetInt16(X) ((int16) (X))
#define Int16GetDatum(X) ((Datum) (X))
#define DatumGetBool(X) ((bool) ((X) != 0))
#define BoolGetDatum(X) ((Datum) ((X) ? 1 : 0))
#define DatumGetObjectId(X) ((Oid) (X))
#define ObjectIdGetDatum(X) ((Datum) (X))
#define DatumGetPointer(X) ((Pointer) (X))
#define PointerGetDatum(X) ((Datum) (X))
#define DatumGetCString(X) ((char *) DatumGetPointer(X))
#define CStringGetDatum(X) PointerGetDatum(X)
double DatumGetFloat8(Datum X);
Datum Float8GetDatum(double X);
float DatumGetFloat4(Datum X);
#define VARHDRSZ 4
#define VARDATA(PTR) (((varlena *) (PTR))->vl_dat)
#define VARSIZE(PTR) (*(uint32 *) (PTR) >> 2)
#define SET_VARSIZE(PTR, len) (*(uint32 *) (PTR) = ((uint32) (len)) << 2)
#define VARDATA_ANY(PTR) VARDATA(PTR)
#define VARSIZE_ANY_EXHDR(PTR) (VARSIZE(PTR) - VARHDRSZ)

/* ---- pg_list.h ---- */
typedef struct List { int length; void **elements; } List;
typedef struct ListCell { void *ptr_value; } ListCell;
#define NIL ((List *) NULL)
int list_length(const List *l);
List *lappend(List *list, void *datum);
List *lappend_int(List *list, int datum);
List *list_make1_impl(void *datum);
#define list_make1(x) list_make1_impl(x)
#define list_make2(a, b) lappend(list_make1_impl(a), b)
void *list_nth(const List *list, int n);
List *list_delete_ptr(List *list, void *datum);
#define linitial(l) list_nth(l, 0)
#define lsecond(l) list_nth(l, 1)
#define foreach(cell, lst) for (int cell##__i = 0; (cell) = NULL, cell##__i < list_length(lst) && ((cell) = (ListCell *) &(lst)->elements[cell##__i], true); cell##__i++)
#define lfirst(lc) ((lc)->ptr_value)
#define lfirst_node(type, lc) ((type *) lfirst(lc))

/* ---- nodes ---- */
typedef enum NodeTag { T_Invalid = 0, T_Var, T_Const, T_OpExpr, T_BoolExpr, T_Aggref, T_TargetEntry, T_RelabelType, T_CustomScan, T_CustomScanState,
					   T_CustomPath, T_Query, T_NullTest, T_FuncExpr, T_ScalarArrayOpExpr, T_CaseExpr, T_CaseWhen, T_CaseTestExpr,
					   T_CoalesceExpr, T_NullIfExpr } NodeTag;
typedef struct Node { NodeTag type; } Node;
#define nodeTag(nodeptr) (((const Node *) (nodeptr))->type)
#define IsA(nodeptr, _type_) (nodeTag(nodeptr) == T_##_type_)
#define castNode(_type_, nodeptr) ((_type_ *) (nodeptr))
void *newNodeImpl(Size size, NodeTag tag);
#define makeNode(_type_) ((_type_ *) newNodeImpl(sizeof(_type_), T_##_type_))
typedef struct Bitmapset Bitmapset;
typedef struct Expr { NodeTag type; } Expr;
typedef struct Var { Expr xpr; int varno; AttrNumber varattno; Oid vartype; int32 vartypmod; Oid varcollid; unsigned varlevelsup; } Var;
typedef struct Const { Expr xpr; Oid consttype; int32 consttypmod; Oid constcollid; int constlen; Datum constvalue; bool constisnull; bool constbyval; } Const;
typedef struct OpExpr { Expr xpr; Oid opno; Oid opfuncid; Oid opresulttype; bool opretset; Oid opcollid; Oid inputcollid; List *args; } OpExpr;
typedef enum BoolExprType { AND_EXPR, OR_EXPR, NOT_EXPR } BoolExprType;
typedef struct BoolExpr { Expr xpr; BoolExprType boolop; List *args; } BoolExpr;
typedef struct RelabelType { Expr xpr; Expr *arg; Oid resulttype; } RelabelType;
typedef struct ScalarArrayOpExpr { Expr xpr; Oid opno; Oid opfuncid; Oid hashfuncid; Oid negfuncid; bool useOr; Oid inputcollid; List *args; int location; } ScalarArrayOpExpr;
typedef enum NullTestType { IS_NULL, IS_NOT_NULL } NullTestType;
typedef struct NullTest { Expr xpr; Expr *arg; NullTestType nulltesttype; bool argisrow; int location; } NullTest;
typedef struct CaseExpr { Expr xpr; Oid casetype; Oid casecollid; Expr *arg; List *args; Expr *defresult; int location; } CaseExpr;
typedef struct CaseWhen { Expr xpr; Expr *expr; Expr *result; int location; } CaseWhen;
typedef struct CaseTestExpr { Expr xpr; Oid typeId; int32 typeMod; Oid collation; } CaseTestExpr;
typedef struct CoalesceExpr { Expr xpr; Oid coalescetype; Oid coalescecollid; List *args; int location; } CoalesceExpr;
typedef OpExpr NullIfExpr;                      /* [PG] an OpExpr of the "=" operator, tagged T_NullIfExpr */
typedef struct Aggref { Expr xpr; Oid aggfnoid; Oid aggtype; List *args; List *aggorder; List *aggdistinct; Expr *aggfilter; bool aggstar; char aggkind; } Aggref;
typedef struct TargetEntry { Expr xpr; Expr *expr; AttrNumber resno; char *resname; unsigned ressortgroupref; bool resjunk; } TargetEntry;
typedef struct SortGroupClause { NodeTag type; unsigned tleSortGroupRef; Oid eqop; } SortGroupClause;
Const *makeConst(Oid consttype, int32 consttypmod, Oid constcollid, int constlen, Datum constvalue, bool constisnull, bool constbyval);
TargetEntry *get_sortgroupref_tle(unsigned sortref, List *targetList);

/* ---- catalog/pg_type.h, pg_operator.h: the few OIDs the glue names (stable built-in OIDs) ---- */
#define BOOLOID 16
#define BYTEAOID 17
#define INT8OID 20
#define INT2OID 21
#define INT4OID 23
#define TEXTOID 25
#define OIDOID 26
#define FLOAT4OID 700
#define FLOAT8OID 701
#define DATEOID 1082
#define TIMESTAMPOID 1114
#define TIMESTAMPTZOID 1184
#define NUMERICOID 1700
#define CSTRINGOID 2275
#define INTERNALOID 2281
#define BTLessStrategyNumber 1
#define BTLessEqualStrategyNumber 2
#define BTEqualStrategyNumber 3
#define BTGreaterEqualStrategyNumber 4
#define BTGreaterStrategyNumber 5
#define BTREE_AM_OID 403
char *get_func_name(Oid funcid);
Oid get_opcode(Oid opno);
char *get_opname(Oid opno);
int get_op_opfamily_strategy(Oid opno, Oid opfamily);
Oid get_opfamily_member(Oid opfamily, Oid lefttype, Oid righttype, int16 strategy);
Oid GetDefaultOpClass(Oid type_id, Oid am_id);
Oid get_opclass_family(Oid opclass);
void get_typlenbyvalalign(Oid typid, int16 *typlen, bool *typbyval, char *typalign);
Oid get_commutator(Oid opno);
Oid get_negator(Oid opno);
Oid get_element_type(Oid typid);

/* ---- fmgr.h ---- */
typedef struct FmgrInfo { void *fn_addr; Oid fn_oid; short fn_nargs; bool fn_strict; void *fn_extra; MemoryContext fn_mcxt; Node *fn_expr; } FmgrInfo;
typedef struct NullableDatum { Datum value; bool isnull; } NullableDatum;
typedef struct FunctionCallInfoBaseData { FmgrInfo *flinfo; Node *context; Node *resultinfo; Oid fncollation; bool isnull; short nargs; NullableDatum args[8]; } FunctionCallInfoBaseData;
typedef FunctionCallInfoBaseData *FunctionCallInfo;
typedef Datum (*PGFunction)(FunctionCallInfo fcinfo);
#define PG_FUNCTION_ARGS FunctionCallInfo fcinfo
#define PG_FUNCTION_INFO_V1(funcname) extern PGDLLEXPORT Datum funcname(PG_FUNCTION_ARGS)
#define PG_NARGS() (fcinfo->nargs)
#define PG_ARGISNULL(n) (fcinfo->args[n].isnull)
#define PG_GETARG_DATUM(n) (fcinfo->args[n].value)
#define PG_GETARG_POINTER(n) DatumGetPointer(PG_GETARG_DATUM(n))
#define PG_GETARG_OID(n) DatumGetObjectId(PG_GETARG_DATUM(n))
#define PG_GETARG_INT32(n) DatumGetInt32(PG_GETARG_DATUM(n))
#define PG_GETARG_INT64(n) DatumGetInt64(PG_GETARG_DATUM(n))
#define PG_GETARG_BOOL(n) DatumGetBool(PG_GETARG_DATUM(n))
#define PG_GETARG_TEXT_PP(n) ((text *) PG_GETARG_POINTER(n))
#define PG_GETARG_CSTRING(n) DatumGetCString(PG_GETARG_DATUM(n))
#define PG_GETARG_ARRAYTYPE_P(n) ((ArrayType *) PG_GETARG_POINTER(n))
#define PG_RETURN_DATUM(x) return (x)
#define PG_RETURN_POINTER(x) return PointerGetDatum(x)
#define PG_RETURN_CSTRING(x) return CStringGetDatum(x)
#define PG_RETURN_NULL() do { fcinfo->isnull = true; return (Datum) 0; } while (0)
#define PG_RETURN_VOID() return (Datum) 0
Datum DirectFunctionCall1Coll(PGFunction func, Oid collation, Datum arg1);
Datum DirectFunctionCall3Coll(PGFunction func, Oid collation, Datum arg1, Datum arg2, Datum arg3);
#define DirectFunctionCall1(func, arg1) DirectFunctionCall1Coll(func, InvalidOid, arg1)
#define DirectFunctionCall3(func, a, b, c) DirectFunctionCall3Coll(func, InvalidOid, a, b, c)
Oid get_fn_expr_argtype(FmgrInfo *flinfo, int argnum);
int AggCheckCallContext(FunctionCallInfo fcinfo, MemoryContext *aggcontext);
Datum numeric_in(PG_FUNCTION_ARGS);
Datum numeric_out(PG_FUNCTION_ARGS);
Datum int8out(PG_FUNCTION_ARGS);
char *text_to_cstring(const text *t);
text *cstring_to_text(const char *s);
typedef struct ArrayType ArrayType;
ArrayType *DatumGetArrayTypeP(Datum d);
void deconstruct_array(ArrayType *array, Oid elmtype, int elmlen, bool elmbyval, char elmalign, Datum **elemsp, bool **nullsp, int *nelemsp);
void getTypeOutputInfo(Oid type, Oid *typOutput, bool *typIsVarlena);
char *OidOutputFunctionCall(Oid functionId, Datum val);
Datum OidInputFunctionCall(Oid functionId, char *str, Oid typioparam, int32 typmod);
void getTypeInputInfo(Oid type, Oid *typInput, Oid *typIOParam);

/* ---- syscache: pg_aggregate / pg_proc rows the aggregate shim looks at ---- */
typedef struct HeapTupleData *HeapTuple;
typedef struct FormData_pg_aggregate { Oid aggfnoid; char aggkind; int16 aggnumdirectargs; Oid aggtransfn; Oid aggfinalfn; Oid aggcombinefn; Oid aggserialfn;
									   Oid aggdeserialfn; Oid aggtranstype; } FormData_pg_aggregate;
typedef FormData_pg_aggregate *Form_pg_aggregate;
typedef struct NameData { char data[64]; } NameData;
#define NameStr(name) ((name).data)
typedef struct FormData_pg_proc { Oid oid; NameData proname; Oid pronamespace; int16 pronargs; Oid prorettype; } FormData_pg_proc;
typedef FormData_pg_proc *Form_pg_proc;
enum SysCacheIdentifier { AGGFNOID, PROCOID };
HeapTuple SearchSysCache1(int cacheId, Datum key1);
void ReleaseSysCache(HeapTuple tuple);
#define HeapTupleIsValid(tuple) ((tuple) != NULL)
void *GETSTRUCT(HeapTuple tuple);
#define PG_CATALOG_NAMESPACE 11

/* ---- tupdesc / tuptable / heap tuples ---- */
typedef struct FormData_pg_attribute { Oid atttypid; int16 attlen; AttrNumber attnum; bool attbyval; char attalign; bool attisdropped; bool attnotnull; int32 atttypmod; } FormData_pg_attribute;
typedef FormData_pg_attribute *Form_pg_attribute;
typedef struct TupleDescData { int natts; FormData_pg_attribute attrs[1]; } TupleDescData;
typedef TupleDescData *TupleDesc;
#define TupleDescAttr(tupdesc, i) (&(tupdesc)->attrs[(i)])
TupleDesc CreateTemplateTupleDesc(int natts);
void TupleDescInitEntry(TupleDesc desc, AttrNumber attributeNumber, const char *attributeName, Oid oidtypeid, int32 typmod, int attdim);
TupleDesc BlessTupleDesc(TupleDesc tupdesc);
typedef struct TupleTableSlot { NodeTag type; uint16 tts_flags; AttrNumber tts_nvalid; TupleDesc tts_tupleDescriptor; Datum *tts_values; bool *tts_isnull; } TupleTableSlot;
TupleTableSlot *ExecClearTuple(TupleTableSlot *slot);
TupleTableSlot *ExecStoreVirtualTuple(TupleTableSlot *slot);
void heap_deform_tuple(HeapTuple tuple, TupleDesc tupleDesc, Datum *values, bool *isnull);
HeapTuple heap_form_tuple(TupleDesc tupleDescriptor, const Datum *values, const bool *isnull);
typedef struct Tuplestorestate Tuplestorestate;
void tuplestore_putvalues(Tuplestorestate *state, TupleDesc tdesc, const Datum *values, const bool *isnull);
void tuplestore_puttuple(Tuplestorestate *state, HeapTuple tuple);

/* ---- relations, buffers, snapshots ---- */
typedef struct RelFileLocator { Oid spcOid; Oid dbOid; Oid relNumber; } RelFileLocator;
typedef struct RelationData { RelFileLocator rd_locator; TupleDesc rd_att; Oid rd_id; } RelationData;
typedef RelationData *Relation;
#define RelationGetDescr(relation) ((relation)->rd_att)
#define RelationGetRelid(relation) ((relation)->rd_id)
typedef int LOCKMODE;
#define AccessShareLock 1
#define NoLock 0
Relation table_open(Oid relationId, LOCKMODE lockmode);
void table_close(Relation relation, LOCKMODE lockmode);
typedef enum ForkNumber { MAIN_FORKNUM = 0 } ForkNumber;
typedef enum ReadBufferMode { RBM_NORMAL } ReadBufferMode;
BlockNumber RelationGetNumberOfBlocksInFork(Relation relation, ForkNumber forkNum);
#define RelationGetNumberOfBlocks(reln) RelationGetNumberOfBlocksInFork(reln, MAIN_FORKNUM)
Buffer ReadBufferExtended(Relation reln, ForkNumber forkNum, BlockNumber blockNum, ReadBufferMode mode, void *strategy);
void LockBuffer(Buffer buffer, int mode);
#define BUFFER_LOCK_SHARE 1
#define BUFFER_LOCK_UNLOCK 0
void ReleaseBuffer(Buffer buffer);
void UnlockReleaseBuffer(Buffer buffer);
typedef char *Page;
Page BufferGetPage(Buffer buffer);
typedef struct SnapshotData *Snapshot;
Snapshot GetActiveSnapshot(void);
Snapshot GetTransactionSnapshot(void);

/* ---- planner ---- */
typedef struct Query { NodeTag type; List *targetList; List *groupClause; Node *havingQual; List *sortClause; bool hasAggs; bool hasWindowFuncs; bool hasDistinctOn;
					   List *distinctClause; List *groupingSets; List *rtable; } Query;
typedef struct PlannerInfo { NodeTag type; Query *parse; List *processed_tlist; } PlannerInfo;
typedef double Cost;
typedef struct PathTarget { NodeTag type; List *exprs; } PathTarget;
typedef enum RelOptKind { RELOPT_BASEREL, RELOPT_JOINREL, RELOPT_UPPER_REL } RelOptKind;
typedef struct RestrictInfo { NodeTag type; Expr *clause; } RestrictInfo;
typedef struct RelOptInfo { NodeTag type; RelOptKind reloptkind; Bitmapset *relids; double rows; PathTarget *reltarget; List *pathlist; unsigned relid; List *baserestrictinfo; } RelOptInfo;
typedef struct RangeTblEntry { NodeTag type; int rtekind; Oid relid; char relkind; } RangeTblEntry;
#define RTE_RELATION 0
RangeTblEntry *planner_rt_fetch_impl(unsigned rti, PlannerInfo *root);
#define planner_rt_fetch(rti, root) planner_rt_fetch_impl(rti, root)
typedef struct Path { NodeTag type; NodeTag pathtype; RelOptInfo *parent; PathTarget *pathtarget; double rows; Cost startup_cost; Cost total_cost; List *pathkeys; } Path;
struct CustomPathMethods;
typedef struct CustomPath { Path path; uint32 flags; List *custom_paths; List *custom_private; const struct CustomPathMethods *methods; } CustomPath;
typedef struct Plan { NodeTag type; List *targetlist; List *qual; struct Plan *lefttree; } Plan;
typedef struct Scan { Plan plan; unsigned scanrelid; } Scan;
struct CustomScanMethods;
typedef struct CustomScan { Scan scan; uint32 flags; List *custom_plans; List *custom_exprs; List *custom_private; List *custom_scan_tlist; Bitmapset *custom_relids;
							const struct CustomScanMethods *methods; } CustomScan;
typedef struct CustomPathMethods
{
	const char *CustomName;
	struct Plan *(*PlanCustomPath)(PlannerInfo *root, RelOptInfo *rel, struct CustomPath *best_path, List *tlist, List *clauses, List *custom_plans);
} CustomPathMethods;
typedef struct CustomScanMethods { const char *CustomName; Node *(*CreateCustomScanState)(CustomScan *cscan); } CustomScanMethods;
void RegisterCustomScanMethods(const CustomScanMethods *methods);
typedef enum UpperRelationKind { UPPERREL_SETOP, UPPERREL_PARTIAL_GROUP_AGG, UPPERREL_GROUP_AGG, UPPERREL_WINDOW, UPPERREL_DISTINCT, UPPERREL_ORDERED,
								 UPPERREL_FINAL } UpperRelationKind;
typedef void (*create_upper_paths_hook_type)(PlannerInfo *root, UpperRelationKind stage, RelOptInfo *input_rel, RelOptInfo *output_rel, void *extra);
extern PGDLLEXPORT create_upper_paths_hook_type create_upper_paths_hook;
void add_path(RelOptInfo *parent_rel, Path *new_path);

/* ---- executor ---- */
typedef struct EState { NodeTag type; Snapshot es_snapshot; MemoryContext es_query_cxt; } EState;
typedef struct ExprContext ExprContext;
typedef struct PlanState { NodeTag type; Plan *plan; EState *state; TupleTableSlot *ps_ResultTupleSlot; ExprContext *ps_ExprContext; } PlanState;
/* executor/executor.h (ExecProcNode is a static inline there: the same call) */
PlanState *ExecInitNode(Plan *node, EState *estate, int eflags);
TupleTableSlot *ExecProcNode(PlanState *node);
void ExecEndNode(PlanState *node);
void ExecReScan(PlanState *node);
typedef struct ScanState { PlanState ps; Relation ss_currentRelation; TupleTableSlot *ss_ScanTupleSlot; } ScanState;
struct CustomExecMethods;
typedef struct CustomScanState { ScanState ss; uint32 flags; List *custom_ps; Size pscan_len; const struct CustomExecMethods *methods; } CustomScanState;
typedef struct ExplainState ExplainState;
typedef struct CustomExecMethods
{
	const char *CustomName;
	void (*BeginCustomScan)(CustomScanState *node, EState *estate, int eflags);
	TupleTableSlot *(*ExecCustomScan)(CustomScanState *node);
	void (*EndCustomScan)(CustomScanState *node);
	void (*ReScanCustomScan)(CustomScanState *node);
	void (*MarkPosCustomScan)(CustomScanState *node);
	void (*RestrPosCustomScan)(CustomScanState *node);
	Size (*EstimateDSMCustomScan)(CustomScanState *node, void *pcxt);
	void (*InitializeDSMCustomScan)(CustomScanState *node, void *pcxt, void *coordinate);
	void (*ReInitializeDSMCustomScan)(CustomScanState *node, void *pcxt, void *coordinate);
	void (*InitializeWorkerCustomScan)(CustomScanState *node, void *toc, void *coordinate);
	void (*ShutdownCustomScan)(CustomScanState *node);
	void (*ExplainCustomScan)(CustomScanState *node, List *ancestors, ExplainState *es);
} CustomExecMethods;
void ExplainPropertyInteger(const char *qlabel, const char *unit, int64 value, ExplainState *es);
void ExplainPropertyText(const char *qlabel, const char *value, ExplainState *es);
void ExplainPropertyFloat(const char *qlabel, const char *unit, double value, int ndigits, ExplainState *es);

/* ---- funcapi.h (set-returning function in materialize mode) ---- */
typedef struct ReturnSetInfo { NodeTag type; ExprContext *econtext; TupleDesc expectedDesc; int allowedModes; int returnMode; Tuplestorestate *setResult; TupleDesc setDesc; } ReturnSetInfo;
void InitMaterializedSRF(FunctionCallInfo fcinfo, uint32 flags);

/* ===================================================================================== *
 *  Citus interfaces the glue plugs into (mirrors; the real build includes the reference's headers).
 * ===================================================================================== */
/* include/columnar/columnar_compression.h:17-27 */
typedef enum CompressionType { COMPRESSION_TYPE_INVALID = -1, COMPRESSION_NONE = 0, COMPRESSION_PG_LZ = 1, COMPRESSION_LZ4 = 2, COMPRESSION_ZSTD = 3,
							   COMPRESSION_COUNT } CompressionType;
/* include/columnar/columnar.h:85-111 */
typedef struct ColumnChunkSkipNode
{
	bool hasMinMax;
	Datum minimumValue;
	Datum maximumValue;
	uint64 rowCount;
	uint64 valueChunkOffset;
	uint64 valueLength;
	uint64 existsChunkOffset;
	uint64 existsLength;
	uint64 decompressedValueSize;
	CompressionType valueCompressionType;
	int valueCompressionLevel;
} ColumnChunkSkipNode;
/* include/columnar/columnar.h:119-125 */
typedef struct StripeSkipList { ColumnChunkSkipNode **chunkSkipNodeArray; uint32 *chunkGroupRowCounts; uint32 columnCount; uint32 chunkCount; } StripeSkipList;
/* include/columnar/columnar_metadata.h:21-42 */
typedef struct StripeMetadata
{
	uint64 fileOffset;
	uint64 dataLength;
	uint32 columnCount;
	uint32 chunkCount;
	uint32 chunkGroupRowCount;
	uint64 rowCount;
	uint64 id;
	uint64 firstRowNumber;
	bool aborted;
	bool insertedByCurrentXact;
} StripeMetadata;
typedef enum StripeWriteStateEnum { STRIPE_WRITE_FLUSHED, STRIPE_WRITE_ABORTED, STRIPE_WRITE_IN_PROGRESS } StripeWriteStateEnum;
List *StripesForRelfilelocator(Relation rel);                                                     /* columnar_metadata.h:60 */
StripeWriteStateEnum StripeWriteState(StripeMetadata *stripeMetadata);                            /* columnar_metadata.c:897 */
StripeSkipList *ReadStripeSkipList(Relation rel, uint64 stripe, TupleDesc tupleDescriptor, uint32 chunkCount, Snapshot snapshot);   /* columnar.h:307 */
bool IsColumnarTableAmTable(Oid relationId);                                                     /* columnar_tableam.h */
extern bool EnableColumnarQualPushdown;                                                           /* columnar_customscan.c:225-236 GUC */
/* include/distributed/tuple_destination.h:45-62 */
typedef struct Task Task;
typedef struct TupleDestinationStats { uint64 totalIntermediateResultSize; } TupleDestinationStats;
typedef struct TupleDestination TupleDestination;
struct TupleDestination
{
	void (*putTuple)(TupleDestination *self, Task *task, int placementIndex, int queryNumber, HeapTuple tuple, uint64 tupleLibpqSize);
	TupleDesc (*tupleDescForQuery)(TupleDestination *self, int queryNumber);
	TupleDestinationStats *tupleDestinationStats;
};
/* executor/intermediate_results.c: per-transaction result directory and file names of a partitioned result */
char *QueryResultFileName(const char *resultId);
void CreateIntermediateResultsDirectory(void);
int pg_glue_open_result_file(const char *path);
void pg_glue_write_result_file(int fd, const void *data, size_t len);
void pg_glue_close_result_file(int fd);

#endif
