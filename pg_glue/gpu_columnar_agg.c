/*
 * gpu_columnar_agg.c -- PostgreSQL-side glue: a "GpuColumnarAgg" CustomScan that replaces the worker task's
 *     Agg <- Custom Scan (ColumnarScan)
 * subtree with one call into libcitus_gpu.so (include/citus_gpu.h).
 *
 * What it mirrors in the reference (file:line under the Citus sources' src/):
 *   registration     backend/columnar/columnar_customscan.c:155-175 (CustomScanMethods / CustomExecMethods),
 *                    :199-200, :265 (hook chaining, RegisterCustomScanMethods)
 *   path injection   the reference injects at set_rel_pathlist_hook (:269-351) because it replaces a SCAN; an
 *                    aggregate replacement has to be offered one level up: create_upper_paths_hook, UPPERREL_GROUP_AGG
 *   stripe listing   backend/columnar/columnar_reader.c:687-734 AdvanceStripeRead: stripes visible to the snapshot,
 *                    unflushed ones skipped (StripeWriteState), skip lists by ReadStripeSkipList
 *                    (backend/columnar/columnar_metadata.c:717-832)
 *   page access      backend/columnar/columnar_storage.c:463-492 ColumnarStorageRead / :669-689 ReadFromBlock: here the
 *                    8 KB pages are copied out of shared_buffers once per scan into one image the library DMAs from
 *   execution        ColumnarScan_ExecCustomScan :1907-1913 returns one slot per call; so does this node: the first call
 *                    runs the fused kernel, later calls stream the partial-aggregate rows
 *   errors           the library returns codes, never longjmps; every non-zero code becomes ereport(ERROR) here
 *
 * A query shape the library does not cover (CG_EUNSUPPORTED at plan time) simply gets no GpuColumnarAgg path: the
 * reference's own Agg <- ColumnarScan plan runs.  A composite GROUP BY key (three or four columns, a column wider than 4
 * bytes, or a nullable column in a two-column key) can also be refused at execution time, because its code domain
 * depends on the data: such a node keeps the reference plan as its child and runs it instead, before any scan.  Built against the real headers with `make -C pg_glue`; type-checked in
 * this repository against pg_glue/stub/ (tests/test_pg_glue.py).
 */
#include "postgres.h"

#include "access/table.h"
#include "catalog/pg_type.h"
#include "commands/explain.h"
#include "executor/executor.h"
#include "executor/tuptable.h"
#include "fmgr.h"
#include "nodes/extensible.h"
#include "nodes/makefuncs.h"
#include "optimizer/pathnode.h"
#include "optimizer/planner.h"
#include "storage/bufmgr.h"
#include "utils/array.h"
#include "utils/builtins.h"
#include "utils/lsyscache.h"
#include "utils/memutils.h"
#include "utils/numeric.h"
#include "utils/rel.h"
#include "utils/snapmgr.h"

#include "columnar/columnar.h"
#include "columnar/columnar_metadata.h"

#include "citus_gpu.h"

PG_MODULE_MAGIC;

void _PG_init(void);

/* what one output column of the node is made of */
typedef enum GpuOutKind { GPU_OUT_KEY, GPU_OUT_COUNT, GPU_OUT_SUM_NUMERIC, GPU_OUT_SUM_INT8, GPU_OUT_SUM_FLOAT8, GPU_OUT_MINMAX,
						  GPU_OUT_VARIANCE } GpuOutKind;

typedef struct GpuOutColumn
{
	int32 kind;          /* GpuOutKind */
	int32 index;         /* group column number / aggregate number in the CgScanDesc */
	Oid type;            /* result type */
	int32 scale;         /* numeric display scale of a sum over scaled integers (0 for plain int8) */
	int32 final;         /* GPU_OUT_VARIANCE: CG_VAR_POP / CG_VAR_SAMP / CG_STDDEV_POP / CG_STDDEV_SAMP */
} GpuOutColumn;

/* the plan-time product: travels in CustomScan.custom_private as one bytea Const (so that copyObject works) */
typedef struct GpuAggPlan
{
	Oid relid;
	CgScanDesc desc;
	int32 nout;
	GpuOutColumn out[CG_MAX_AGGS + CG_MAX_GROUP_COLS];
} GpuAggPlan;

typedef struct GpuColumnarAggState
{
	CustomScanState css;         /* must be first (columnar_customscan.c:65-71 does the same) */
	GpuAggPlan plan;
	CgPartial *partial;
	CgScanStats stats;
	/* result rows fetched from the device */
	int64 ngroups, next;
	int64 *keys;
	uint8 *key_nulls;
	int64 *sum_hi;
	uint64 *sum_lo;
	int64 *count;
	int64 *minmax;
	double *fsum;
	uint64 *sumsq;       /* [cells * 3]: sum(x^2) of the variance aggregates */
	/* composite key: the decoded key columns of every group, [group][column] */
	int64 *key_values;
	uint8 *key_value_nulls;
	bool done_scan;
	/* composite key: the reference Agg <- ColumnarScan plan, run when the library refuses the key domain */
	PlanState *child;
	bool use_child;
} GpuColumnarAggState;

static create_upper_paths_hook_type prev_create_upper_paths_hook = NULL;
static bool gpu_device_ready = false;

/* ------------------------------------------------------------------------------------ *
 *  library errors -> ereport
 * ------------------------------------------------------------------------------------ */
static void
gpu_check(int rc)
{
	if (rc == CG_OK)
		return;
	int sqlstate = rc == CG_EUNSUPPORTED ? ERRCODE_FEATURE_NOT_SUPPORTED :
				   rc == CG_ECORRUPT ? ERRCODE_DATA_CORRUPTED :
				   rc == CG_ENOMEM ? ERRCODE_OUT_OF_MEMORY : ERRCODE_INTERNAL_ERROR;
	ereport(ERROR, (errcode(sqlstate), errmsg("citus_gpu: %s", cg_last_error())));
}

/* CUDA is initialised lazily in the backend that needs it, never in the postmaster (a forked CUDA context is unusable) */
static void
gpu_ensure_device(void)
{
	if (gpu_device_ready)
		return;
	gpu_check(cg_init(0));
	gpu_device_ready = true;
}

/* ------------------------------------------------------------------------------------ *
 *  plan time: does the worker query fit the library's plan language?
 * ------------------------------------------------------------------------------------ */
static bool
type_is_supported(Oid type, int *attlen, int *type_class)
{
	switch (type)
	{
		case INT8OID: case TIMESTAMPOID: case TIMESTAMPTZOID: *attlen = 8; *type_class = CG_TYPE_INT; return true;
		case INT4OID: case DATEOID: *attlen = 4; *type_class = CG_TYPE_INT; return true;
		case INT2OID: *attlen = 2; *type_class = CG_TYPE_INT; return true;
		case BOOLOID: *attlen = 1; *type_class = CG_TYPE_INT; return true;        /* one byte, 0 / 1 */
		case FLOAT8OID: *attlen = 8; *type_class = CG_TYPE_FLOAT; return true;
		case FLOAT4OID: *attlen = 4; *type_class = CG_TYPE_FLOAT; return true;
		default: return false;
	}
}

static Var *
strip_to_var(Node *node)
{
	while (node && IsA(node, RelabelType))
		node = (Node *) ((RelabelType *) node)->arg;
	return (node && IsA(node, Var)) ? (Var *) node : NULL;
}

/* btree strategy of an operator on the column's default operator class, 0 if it has none ("<>" is its negator) */
static int
btree_strategy(Oid opno, Oid type)
{
	Oid opclass = GetDefaultOpClass(type, BTREE_AM_OID);
	if (opclass == InvalidOid)
		return 0;
	return get_op_opfamily_strategy(opno, get_opclass_family(opclass));
}

/* the pairs of column types a column atom compares: integers of any width, floats of any width, and bool, date, timestamp,
 * timestamptz each with itself.  date / timestamp / timestamptz against one another are refused: their comparison converts
 * units (and, for timestamptz, uses the session time zone), so it is not a comparison of the decoded integers */
static bool
column_pair_supported(Oid a, Oid b)
{
	const bool ia = a == INT2OID || a == INT4OID || a == INT8OID, ib = b == INT2OID || b == INT4OID || b == INT8OID;
	const bool fa = a == FLOAT4OID || a == FLOAT8OID, fb = b == FLOAT4OID || b == FLOAT8OID;
	if (ia || ib)
		return ia && ib;
	if (fa || fb)
		return fa && fb;
	return a == b && (a == BOOLOID || a == DATEOID || a == TIMESTAMPOID || a == TIMESTAMPTZOID);
}

/* btree strategy -> the atom's operator ("<>", the negator of "=", has no strategy); -1 for anything else */
static int
strategy_op(int strategy, Oid opno)
{
	switch (strategy)
	{
		case BTLessStrategyNumber: return CG_OP_LT;
		case BTLessEqualStrategyNumber: return CG_OP_LE;
		case BTEqualStrategyNumber: return CG_OP_EQ;
		case BTGreaterEqualStrategyNumber: return CG_OP_GE;
		case BTGreaterStrategyNumber: return CG_OP_GT;
		default: return strcmp(get_opname(opno), "<>") == 0 ? CG_OP_NE : -1;
	}
}

/* "Var op Var" over two columns of the scanned relation -> a CG_OP_COL_* atom; false for any other pair of types */
static bool
translate_column_atom(Var *x, Var *y, Oid opno, TupleDesc tupdesc, CgQual *qual)
{
	int attlen, type_class;
	if (x->varno != y->varno || x->varlevelsup != 0 || y->varlevelsup != 0 || x->varattno <= 0 || x->varattno > tupdesc->natts ||
		y->varattno <= 0 || y->varattno > tupdesc->natts || !type_is_supported(x->vartype, &attlen, &type_class) ||
		!type_is_supported(y->vartype, &attlen, &type_class) || !column_pair_supported(x->vartype, y->vartype))
		return false;
	/* the strategy in the left type's default operator family, which holds the cross-type operators of its family */
	const int cgop = strategy_op(btree_strategy(opno, x->vartype), opno);
	if (cgop < 0)
		return false;
	qual->column = x->varattno - 1;
	qual->op = CG_OP_COL_LT + (cgop - CG_OP_LT);
	qual->konst = y->varattno - 1;
	return true;
}

/* one WHERE atom "Var op Const" (or commuted) or "Var op Var" -> CgQual; false when it is anything else */
static bool
translate_atom(OpExpr *op, TupleDesc tupdesc, CgQual *qual)
{
	if (list_length(op->args) != 2)
		return false;
	Node *l = (Node *) linitial(op->args), *r = (Node *) lsecond(op->args);
	if (strip_to_var(l) && strip_to_var(r))
		return translate_column_atom(strip_to_var(l), strip_to_var(r), op->opno, tupdesc, qual);
	Var *var = strip_to_var(l);
	Const *konst = (r && IsA(r, Const)) ? (Const *) r : NULL;
	Oid opno = op->opno;
	if (var == NULL || konst == NULL)
	{
		var = strip_to_var(r);
		konst = (l && IsA(l, Const)) ? (Const *) l : NULL;
		opno = get_commutator(op->opno);
		if (var == NULL || konst == NULL || opno == InvalidOid)
			return false;
	}
	if (konst->constisnull || var->varattno <= 0 || var->varattno > tupdesc->natts)
		return false;
	int attlen, type_class;
	if (!type_is_supported(var->vartype, &attlen, &type_class) || konst->consttype != var->vartype)
		return false;
	int cgop = strategy_op(btree_strategy(opno, var->vartype), opno);
	if (cgop < 0)
		return false;
	qual->column = var->varattno - 1;
	qual->op = cgop;
	if (type_class == CG_TYPE_FLOAT)
	{
		double d = var->vartype == FLOAT4OID ? (double) DatumGetFloat4(konst->constvalue) : DatumGetFloat8(konst->constvalue);
		memcpy(&qual->konst, &d, sizeof d);
	}
	else
		qual->konst = attlen == 8 ? DatumGetInt64(konst->constvalue) :
					  attlen == 4 ? (int64) DatumGetInt32(konst->constvalue) :
					  attlen == 2 ? (int64) DatumGetInt16(konst->constvalue) : (int64) DatumGetBool(konst->constvalue);
	return true;
}

static int64 datum_to_i64(Datum d, Oid type);

/* "x = ANY(array)" / "x <> ALL(array)" -- how PostgreSQL plans IN and NOT IN lists -- over a non-NULL constant array of the
 * column's own type, with the type's btree equality (or its negator) -> a CG_OP_IN / CG_OP_NOT_IN atom whose list is appended
 * to desc's list table: the elements as written, NULLs counted.  false for anything else, an empty array, or a full table */
static bool
translate_saop(ScalarArrayOpExpr *saop, TupleDesc tupdesc, CgScanDesc *desc, CgQual *qual)
{
	if (list_length(saop->args) != 2)
		return false;
	Var *var = strip_to_var((Node *) linitial(saop->args));
	Node *r = (Node *) lsecond(saop->args);
	Const *arr = (r && IsA(r, Const)) ? (Const *) r : NULL;
	if (var == NULL || arr == NULL || arr->constisnull || var->varattno <= 0 || var->varattno > tupdesc->natts)
		return false;
	int attlen, type_class;
	if (!type_is_supported(var->vartype, &attlen, &type_class) || get_element_type(arr->consttype) != var->vartype)
		return false;
	if (saop->useOr ? btree_strategy(saop->opno, var->vartype) != BTEqualStrategyNumber
					: (get_negator(saop->opno) == InvalidOid || btree_strategy(get_negator(saop->opno), var->vartype) != BTEqualStrategyNumber))
		return false;
	int16 typlen;
	bool typbyval;
	char typalign;
	get_typlenbyvalalign(var->vartype, &typlen, &typbyval, &typalign);
	Datum *elems;
	bool *nulls;
	int n;
	deconstruct_array(DatumGetArrayTypeP(arr->constvalue), var->vartype, typlen, typbyval, typalign, &elems, &nulls, &n);
	int nvalues = 0;
	for (int i = 0; i < n; i++)
		nvalues += !nulls[i];
	if (n == 0 || desc->nin_lists >= CG_MAX_IN_LISTS || desc->nin_values + nvalues > CG_MAX_IN_VALUES)
		return false;
	CgInList *list = &desc->in_lists[desc->nin_lists];
	list->first = desc->nin_values;
	list->nvalues = nvalues;
	list->nnulls = n - nvalues;
	list->reserved = 0;
	for (int i = 0; i < n; i++)
		if (!nulls[i])
			desc->in_values[desc->nin_values++] = datum_to_i64(elems[i], var->vartype);     /* konst's convention */
	qual->column = var->varattno - 1;
	qual->op = saop->useOr ? CG_OP_IN : CG_OP_NOT_IN;
	qual->konst = desc->nin_lists++;
	return true;
}

/* "x IS [NOT] NULL" over a column of a supported type -> CG_OP_IS_NULL / CG_OP_IS_NOT_NULL */
static bool
translate_nulltest(NullTest *nt, TupleDesc tupdesc, CgQual *qual)
{
	Var *var = strip_to_var((Node *) nt->arg);
	int attlen, type_class;
	if (nt->argisrow || var == NULL || var->varattno <= 0 || var->varattno > tupdesc->natts ||
		!type_is_supported(var->vartype, &attlen, &type_class))
		return false;
	qual->column = var->varattno - 1;
	qual->op = nt->nulltesttype == IS_NULL ? CG_OP_IS_NULL : CG_OP_IS_NOT_NULL;
	qual->konst = 0;
	return true;
}

/* a bare bool column `flag` as the atom "flag = 1", and NOT flag as "flag = 0" (a NULL flag stays UNKNOWN either way) */
static bool
translate_bool_var(Node *node, bool negated, TupleDesc tupdesc, CgQual *qual)
{
	Var *var = strip_to_var(node);
	if (var == NULL || var->vartype != BOOLOID || var->varattno <= 0 || var->varattno > tupdesc->natts)
		return false;
	qual->column = var->varattno - 1;
	qual->op = CG_OP_EQ;
	qual->konst = negated ? 0 : 1;
	return true;
}

/* boolean tree -> atoms appended to atoms[0 .. *natoms) (at most max_atoms) + postfix tokens appended to tokens[0 .. *ntokens)
 * (at most CG_MAX_QEXPR): the WHERE list (quals / qual_expr), aggregate FILTERs (filter_quals / filter_expr[a]) and the
 * predicate arguments of bool_and / bool_or / every (filter_quals / arg_expr[a]).  An atom is "Var op Const", "Var op Var"
 * (column_pair_supported), a bare bool Var, NOT over a bare bool Var, an IN / NOT IN list over a Var (its list goes to
 * desc's list table) or "Var IS [NOT] NULL".
 * false when a node is anything else or the tree is too big */
static bool
translate_where(Node *node, TupleDesc tupdesc, CgScanDesc *desc, CgQual *atoms, int32_t *natoms, int max_atoms, int8_t *tokens,
				int32_t *ntokens)
{
	if (IsA(node, BoolExpr))
	{
		BoolExpr *b = (BoolExpr *) node;
		if (b->boolop == NOT_EXPR)
		{
			/* only NOT over a bare bool column: its negation is the atom "flag = 0" */
			if (list_length(b->args) != 1 || *natoms >= max_atoms || *ntokens >= CG_MAX_QEXPR ||
				!translate_bool_var((Node *) linitial(b->args), true, tupdesc, &atoms[*natoms]))
				return false;
			tokens[(*ntokens)++] = (int8_t) (*natoms)++;
			return true;
		}
		ListCell *lc;
		int n = 0;
		foreach(lc, b->args)
		{
			if (!translate_where((Node *) lfirst(lc), tupdesc, desc, atoms, natoms, max_atoms, tokens, ntokens))
				return false;
			if (n++ > 0)
			{
				if (*ntokens >= CG_MAX_QEXPR)
					return false;
				tokens[(*ntokens)++] = b->boolop == AND_EXPR ? CG_QX_AND : CG_QX_OR;
			}
		}
		return n > 0;
	}
	if (*natoms >= max_atoms || *ntokens >= CG_MAX_QEXPR)
		return false;
	bool ok;
	if (IsA(node, OpExpr))
		ok = translate_atom((OpExpr *) node, tupdesc, &atoms[*natoms]);
	else if (IsA(node, ScalarArrayOpExpr))
		ok = translate_saop((ScalarArrayOpExpr *) node, tupdesc, desc, &atoms[*natoms]);
	else if (IsA(node, NullTest))
		ok = translate_nulltest((NullTest *) node, tupdesc, &atoms[*natoms]);
	else
		ok = translate_bool_var(node, false, tupdesc, &atoms[*natoms]);
	if (!ok)
		return false;
	tokens[(*ntokens)++] = (int8_t) (*natoms)++;
	return true;
}

/* the argument forms a CASE arm reads (include/citus_gpu.h, CgCaseArm): int2 / int4 / int8, or float8 for a float CASE */
static bool
case_type_supported(Oid type)
{
	return type == INT2OID || type == INT4OID || type == INT8OID || type == FLOAT8OID;
}

/* a CASE result: a Var of the CASE's own type (through strip_to_var) -> a bare-column product, a Const of that type -> a
 * constant, a NULL Const -> the NULL result; false for anything else (casts, arithmetic) */
static bool
translate_case_result(Node *node, Oid type, TupleDesc tupdesc, CgCaseArm *arm)
{
	Var *var = strip_to_var(node);
	if (var != NULL)
	{
		if (var->varattno <= 0 || var->varattno > tupdesc->natts || var->vartype != type)
			return false;
		arm->form = CG_CASE_PRODUCT;
		arm->nfactors = 1;
		arm->column[0] = var->varattno - 1;
		arm->a[0] = 0;
		if (type == FLOAT8OID) { double one = 1.0; memcpy(&arm->b[0], &one, sizeof one); }
		else arm->b[0] = 1;
		return true;
	}
	if (node == NULL || !IsA(node, Const) || ((Const *) node)->consttype != type)
		return false;
	const Const *k = (const Const *) node;
	arm->form = k->constisnull ? CG_CASE_NULL : CG_CASE_CONST;
	arm->a[0] = k->constisnull ? 0 : datum_to_i64(k->constvalue, type);      /* float8 bits for a float CASE */
	return true;
}

/* "x = k" over a column and a non-NULL constant of its type with the type's btree equality -> one atom of the pool, appended
 * to the arm's WHEN tree (the simple CASE's "CASE x WHEN k" and NULLIF's test) */
static bool
case_equality_atom(Var *var, Const *k, Oid opno, TupleDesc tupdesc, CgScanDesc *desc, CgCaseArm *arm)
{
	int attlen, type_class;
	if (var == NULL || k == NULL || k->constisnull || var->varattno <= 0 || var->varattno > tupdesc->natts ||
		!type_is_supported(var->vartype, &attlen, &type_class) || k->consttype != var->vartype ||
		btree_strategy(opno, var->vartype) != BTEqualStrategyNumber || desc->nfilter_quals >= CG_MAX_FILTER_QUALS || arm->nwhen >= CG_MAX_QEXPR)
		return false;
	CgQual *q = &desc->filter_quals[desc->nfilter_quals];
	q->column = var->varattno - 1;
	q->op = CG_OP_EQ;
	q->konst = datum_to_i64(k->constvalue, var->vartype);
	arm->when[arm->nwhen++] = (int8_t) desc->nfilter_quals++;
	return true;
}

/* the next free arm of the descriptor (zeroed), NULL when CG_MAX_CASE_ARMS are taken */
static CgCaseArm *
next_arm(CgScanDesc *desc)
{
	if (desc->ncase_arms >= CG_MAX_CASE_ARMS)
		return NULL;
	CgCaseArm *arm = &desc->case_arms[desc->ncase_arms++];
	memset(arm, 0, sizeof *arm);
	return arm;
}

/*
 * A conditional aggregate argument -> the arms of aggregate desc->naggs (include/citus_gpu.h, CgScanDesc.case_arms):
 *   CASE WHEN c THEN r ... [ELSE r] END     each WHEN through translate_where into the filter atom pool
 *   CASE x WHEN k THEN r ... END            each WHEN a CaseTestExpr = Const, as the atom "x = k"
 *   COALESCE(x, k)                          WHEN x IS NOT NULL THEN x ELSE k
 *   NULLIF(x, k)                            WHEN x = k THEN NULL ELSE x
 * with results as translate_case_result takes them, of int2 / int4 / int8 or float8.  *type = the argument's type.  false
 * (the reference's executor runs the query) for any other form, or when the pool or the arm table is full.
 */
static bool
translate_case_arg(Node *arg, TupleDesc tupdesc, CgScanDesc *desc, Oid *type)
{
	const int a = desc->naggs, first = desc->ncase_arms;
	CgCaseArm *arm;
	if (IsA(arg, CaseExpr))
	{
		CaseExpr *ce = (CaseExpr *) arg;
		*type = ce->casetype;
		Var *subject = ce->arg != NULL ? strip_to_var((Node *) ce->arg) : NULL;
		if (!case_type_supported(*type) || (ce->arg != NULL && subject == NULL))
			return false;
		ListCell *lc;
		foreach(lc, ce->args)
		{
			CaseWhen *w = (CaseWhen *) lfirst(lc);
			if ((arm = next_arm(desc)) == NULL)
				return false;
			if (ce->arg != NULL)
			{
				/* the simple form: the planner wrote each WHEN as "CaseTestExpr = Const" */
				OpExpr *op = IsA(w->expr, OpExpr) ? (OpExpr *) w->expr : NULL;
				if (op == NULL || list_length(op->args) != 2 || !IsA((Node *) linitial(op->args), CaseTestExpr) ||
					!IsA((Node *) lsecond(op->args), Const) ||
					!case_equality_atom(subject, (Const *) lsecond(op->args), op->opno, tupdesc, desc, arm))
					return false;
			}
			else if (!translate_where((Node *) w->expr, tupdesc, desc, desc->filter_quals, &desc->nfilter_quals, CG_MAX_FILTER_QUALS, arm->when,
									  &arm->nwhen))
				return false;
			if (!translate_case_result((Node *) w->result, *type, tupdesc, arm))
				return false;
		}
		/* [PG] a CASE without ELSE has a NULL Const as its defresult */
		if (ce->defresult != NULL && ((arm = next_arm(desc)) == NULL || !translate_case_result((Node *) ce->defresult, *type, tupdesc, arm)))
			return false;
	}
	else if (IsA(arg, CoalesceExpr))
	{
		CoalesceExpr *co = (CoalesceExpr *) arg;
		*type = co->coalescetype;
		Var *x = list_length(co->args) == 2 ? strip_to_var((Node *) linitial(co->args)) : NULL;
		if (!case_type_supported(*type) || x == NULL || x->varattno <= 0 || x->varattno > tupdesc->natts || desc->nfilter_quals >= CG_MAX_FILTER_QUALS ||
			(arm = next_arm(desc)) == NULL)
			return false;
		CgQual *q = &desc->filter_quals[desc->nfilter_quals];
		q->column = x->varattno - 1;
		q->op = CG_OP_IS_NOT_NULL;
		q->konst = 0;
		arm->when[arm->nwhen++] = (int8_t) desc->nfilter_quals++;
		if (!translate_case_result((Node *) linitial(co->args), *type, tupdesc, arm) || (arm = next_arm(desc)) == NULL ||
			!translate_case_result((Node *) lsecond(co->args), *type, tupdesc, arm) || arm->form != CG_CASE_CONST)
			return false;
	}
	else if (IsA(arg, NullIfExpr))
	{
		NullIfExpr *ni = (NullIfExpr *) arg;
		*type = ni->opresulttype;
		Var *x = list_length(ni->args) == 2 ? strip_to_var((Node *) linitial(ni->args)) : NULL;
		Node *k = list_length(ni->args) == 2 ? (Node *) lsecond(ni->args) : NULL;
		if (!case_type_supported(*type) || k == NULL || !IsA(k, Const) || (arm = next_arm(desc)) == NULL ||
			!case_equality_atom(x, (Const *) k, ni->opno, tupdesc, desc, arm))
			return false;
		arm->form = CG_CASE_NULL;
		if ((arm = next_arm(desc)) == NULL || !translate_case_result((Node *) x, *type, tupdesc, arm))
			return false;
	}
	else
		return false;
	desc->case_first[a] = first;
	desc->case_narms[a] = desc->ncase_arms - first;
	return desc->case_narms[a] > 0;
}

/* the most accumulator words the library can lay out for the aggregate list (include/citus_gpu.h, CG_MAX_WORDS): word 0
 * plus per aggregate its widest form, whatever the term bounds turn out to be */
static int
worst_case_words(const CgScanDesc *desc)
{
	int words = 1;
	for (int a = 0; a < desc->naggs; a++)
		switch (desc->aggs[a].kind)
		{
			case CG_AGG_COUNT_STAR: case CG_AGG_COUNT: words += 1; break;
			case CG_AGG_SUM: words += 3; break;
			case CG_AGG_VARIANCE: words += 7; break;
			default: words += 2; break;
		}
	return words;
}

/* the worker half of the aggregate split names plain built-ins (planner/multi_logical_optimizer.c:3160-3484) */
static bool
translate_aggref(Aggref *agg, TupleDesc tupdesc, CgScanDesc *desc, GpuOutColumn *out)
{
	if (agg->aggdistinct != NIL || agg->aggorder != NIL || agg->aggkind != 'n' || desc->naggs >= CG_MAX_AGGS)
		return false;
	const char *name = get_func_name(agg->aggfnoid);
	CgAggSpec *spec = &desc->aggs[desc->naggs];
	memset(spec, 0, sizeof *spec);
	/* FILTER (WHERE ...): the worker aggregate keeps it (multi_logical_optimizer.c:3279-3280, 3479), so it is evaluated
	 * here, into the filter atom pool; a filter the atom language cannot express keeps the reference's executor.  (avg's
	 * sum and count parts are one aggregate here: its non-NULL count rides along with the sum, under the same filter.) */
	desc->nfilter_expr[desc->naggs] = 0;
	if (agg->aggfilter != NULL &&
		!translate_where((Node *) agg->aggfilter, tupdesc, desc, desc->filter_quals, &desc->nfilter_quals, CG_MAX_FILTER_QUALS,
						 desc->filter_expr[desc->naggs], &desc->nfilter_expr[desc->naggs]))
		return false;
	out->index = desc->naggs;
	out->scale = 0;
	if (agg->aggstar && strcmp(name, "count") == 0)
	{
		spec->kind = CG_AGG_COUNT_STAR;
		out->kind = GPU_OUT_COUNT; out->type = INT8OID;
		desc->naggs++;
		return true;
	}
	if (list_length(agg->args) != 1)
		return false;
	Node *arg = (Node *) ((TargetEntry *) linitial(agg->args))->expr;
	if (strcmp(name, "bool_and") == 0 || strcmp(name, "bool_or") == 0 || strcmp(name, "every") == 0)
	{
		/* the argument is a predicate (a bool column or any tree translate_where accepts), written into the atom pool it
		 * shares with the FILTERs; three-valued: an UNKNOWN row is no input, no input at all is NULL (count 0) */
		spec->kind = strcmp(name, "bool_or") == 0 ? CG_AGG_BOOL_OR : CG_AGG_BOOL_AND;
		desc->narg_expr[desc->naggs] = 0;
		if (!translate_where(arg, tupdesc, desc, desc->filter_quals, &desc->nfilter_quals, CG_MAX_FILTER_QUALS, desc->arg_expr[desc->naggs],
							 &desc->narg_expr[desc->naggs]))
			return false;
		out->kind = GPU_OUT_MINMAX; out->type = BOOLOID;
		desc->naggs++;
		return true;
	}
	/* the argument: a bare column, or a conditional expression whose arms read columns and constants (translate_case_arg);
	 * vtype = its type either way */
	Var *var = strip_to_var(arg);
	const bool is_case = var == NULL;
	Oid vtype;
	desc->case_narms[desc->naggs] = 0;
	if (is_case)
	{
		if (!translate_case_arg(arg, tupdesc, desc, &vtype))
			return false;
		spec->nfactors = 0;
		spec->is_float = vtype == FLOAT8OID;
	}
	else
	{
		int attlen, type_class;
		if (var->varattno <= 0 || var->varattno > tupdesc->natts || !type_is_supported(var->vartype, &attlen, &type_class))
			return false;
		vtype = var->vartype;
		spec->nfactors = 1;
		spec->column[0] = var->varattno - 1;
		spec->is_float = type_class == CG_TYPE_FLOAT;
		spec->a[0] = 0;
		if (spec->is_float) { double one = 1.0; memcpy(&spec->b[0], &one, sizeof one); }
		else spec->b[0] = 1;
	}
	if (strcmp(name, "count") == 0)
	{
		spec->kind = CG_AGG_COUNT;
		if (!is_case) { spec->is_float = 0; spec->b[0] = 1; }
		out->kind = GPU_OUT_COUNT; out->type = INT8OID;
	}
	else if (strcmp(name, "sum") == 0)
	{
		spec->kind = CG_AGG_SUM;
		if (spec->is_float) { out->kind = GPU_OUT_SUM_FLOAT8; out->type = vtype == FLOAT4OID ? FLOAT4OID : FLOAT8OID; }
		else if (vtype == INT8OID) { out->kind = GPU_OUT_SUM_NUMERIC; out->type = NUMERICOID; }   /* [PG] sum(int8) is numeric */
		else if (vtype == INT4OID || vtype == INT2OID) { out->kind = GPU_OUT_SUM_INT8; out->type = INT8OID; }
		else return false;
		if (vtype == FLOAT4OID) return false;          /* [PG] sum(float4) accumulates in float4: not what the kernels do */
	}
	else if (strcmp(name, "min") == 0 || strcmp(name, "max") == 0 || strcmp(name, "any_value") == 0)
	{
		/* any_value(x): any non-NULL input -- the minimum is one */
		spec->kind = name[1] == 'a' ? CG_AGG_MAX : CG_AGG_MIN;
		out->kind = GPU_OUT_MINMAX; out->type = vtype;
	}
	else if (strcmp(name, "var_pop") == 0 || strcmp(name, "var_samp") == 0 || strcmp(name, "variance") == 0 ||
			 strcmp(name, "stddev_pop") == 0 || strcmp(name, "stddev_samp") == 0 || strcmp(name, "stddev") == 0)
	{
		/* over int2 / int4 / int8 PostgreSQL keeps N, sum(x) and sum(x^2) as exact integers and the result is numeric: one
		 * state for all six names, the name picks the final function (cg_numeric_var_out).  A float argument keeps the
		 * reference's executor (float8_accum cannot be matched bit for bit) */
		if (vtype != INT2OID && vtype != INT4OID && vtype != INT8OID)
			return false;
		const bool pop = strcmp(name, "var_pop") == 0 || strcmp(name, "stddev_pop") == 0;
		spec->kind = CG_AGG_VARIANCE;
		out->kind = GPU_OUT_VARIANCE; out->type = NUMERICOID;
		out->final = strncmp(name, "var", 3) == 0 ? (pop ? CG_VAR_POP : CG_VAR_SAMP) : (pop ? CG_STDDEV_POP : CG_STDDEV_SAMP);
	}
	else if (strcmp(name, "bit_and") == 0 || strcmp(name, "bit_or") == 0)
	{
		/* bare int2 / int4 / int8 column; the result has the argument's type (words hold it sign-extended) */
		if (is_case || (vtype != INT2OID && vtype != INT4OID && vtype != INT8OID))
			return false;
		spec->kind = name[4] == 'a' ? CG_AGG_BIT_AND : CG_AGG_BIT_OR;
		out->kind = GPU_OUT_MINMAX; out->type = var->vartype;
	}
	else
		return false;                                           /* anything else keeps the reference's executor */
	desc->naggs++;
	return true;
}

static bool
translate_query(PlannerInfo *root, RelOptInfo *input_rel, GpuAggPlan *plan)
{
	Query *q = root->parse;
	if (!q->hasAggs || q->hasWindowFuncs || q->hasDistinctOn || q->distinctClause != NIL || q->groupingSets != NIL || q->havingQual != NULL)
		return false;
	if (input_rel->reloptkind != RELOPT_BASEREL)
		return false;
	RangeTblEntry *rte = planner_rt_fetch(input_rel->relid, root);
	if (rte->rtekind != RTE_RELATION || !IsColumnarTableAmTable(rte->relid))
		return false;
	memset(plan, 0, sizeof *plan);
	plan->relid = rte->relid;
	plan->desc.enable_qual_pushdown = EnableColumnarQualPushdown ? 1 : 0;
	Relation rel = table_open(rte->relid, AccessShareLock);
	TupleDesc tupdesc = RelationGetDescr(rel);
	bool ok = true;
	ListCell *lc;
	/* WHERE: the implicit AND-list of restriction clauses */
	int nclauses = 0;
	foreach(lc, input_rel->baserestrictinfo)
	{
		RestrictInfo *ri = (RestrictInfo *) lfirst(lc);
		if (!(ok = translate_where((Node *) ri->clause, tupdesc, &plan->desc, plan->desc.quals, &plan->desc.nquals, CG_MAX_QUALS, plan->desc.qual_expr,
								   &plan->desc.nqual_expr)))
			break;
		if (nclauses++ > 0)
		{
			if (plan->desc.nqual_expr >= CG_MAX_QEXPR) { ok = false; break; }
			plan->desc.qual_expr[plan->desc.nqual_expr++] = CG_QX_AND;
		}
	}
	/* GROUP BY plain integer columns.  One column, and two NOT NULL columns of at most 4 bytes, keep the one-column and
	 * packed two-column key forms; anything wider, or a two-column key with a nullable column (whose NULL the packed form
	 * refuses at run time), takes the composite key, whose bounds run_scan reads from the skip lists */
	bool composite = false;
	foreach(lc, q->groupClause)
	{
		if (!ok) break;
		SortGroupClause *sgc = (SortGroupClause *) lfirst(lc);
		TargetEntry *tle = get_sortgroupref_tle(sgc->tleSortGroupRef, q->targetList);
		Var *var = strip_to_var((Node *) tle->expr);
		int attlen, type_class;
		if (var == NULL || var->varattno <= 0 || var->varattno > tupdesc->natts || plan->desc.ngroup_cols >= CG_MAX_GROUP_COLS ||
			!type_is_supported(var->vartype, &attlen, &type_class) || type_class != CG_TYPE_INT)
			ok = false;
		else
		{
			composite |= attlen > 4 || !TupleDescAttr(tupdesc, var->varattno - 1)->attnotnull;
			plan->desc.group_cols[plan->desc.ngroup_cols++] = var->varattno - 1;
		}
	}
	plan->desc.composite_key = plan->desc.ngroup_cols > 2 || (plan->desc.ngroup_cols == 2 && composite);
	/* target list: group columns and aggregates, in output order */
	foreach(lc, q->targetList)
	{
		if (!ok) break;
		TargetEntry *tle = (TargetEntry *) lfirst(lc);
		if (tle->resjunk || plan->nout >= (int) lengthof(plan->out)) { ok = false; break; }
		GpuOutColumn *out = &plan->out[plan->nout];
		if (IsA(tle->expr, Aggref))
			ok = translate_aggref((Aggref *) tle->expr, tupdesc, &plan->desc, out);
		else
		{
			Var *var = strip_to_var((Node *) tle->expr);
			ok = false;
			for (int g = 0; var != NULL && g < plan->desc.ngroup_cols; g++)
				if (plan->desc.group_cols[g] == var->varattno - 1)
				{
					out->kind = GPU_OUT_KEY; out->index = g; out->type = var->vartype; ok = true;
				}
		}
		plan->nout++;
	}
	table_close(rel, AccessShareLock);
	/* the library refuses an aggregate list whose words pass CG_MAX_WORDS, and only at run time, when the bounds are known:
	 * a list that could pass it keeps the reference executor */
	return ok && plan->desc.naggs > 0 && worst_case_words(&plan->desc) <= CG_MAX_WORDS;
}

/* ------------------------------------------------------------------------------------ *
 *  path / plan / state creation
 * ------------------------------------------------------------------------------------ */
static Plan *GpuColumnarAgg_PlanCustomPath(PlannerInfo *root, RelOptInfo *rel, CustomPath *best_path, List *tlist, List *clauses, List *custom_plans);
static Node *GpuColumnarAgg_CreateCustomScanState(CustomScan *cscan);
static void GpuColumnarAgg_Begin(CustomScanState *node, EState *estate, int eflags);
static TupleTableSlot *GpuColumnarAgg_Exec(CustomScanState *node);
static void GpuColumnarAgg_End(CustomScanState *node);
static void GpuColumnarAgg_ReScan(CustomScanState *node);
static void GpuColumnarAgg_Explain(CustomScanState *node, List *ancestors, ExplainState *es);

static const CustomPathMethods GpuColumnarAggPathMethods = {
	.CustomName = "GpuColumnarAgg",
	.PlanCustomPath = GpuColumnarAgg_PlanCustomPath,
};

static const CustomScanMethods GpuColumnarAggScanMethods = {
	.CustomName = "GpuColumnarAgg",
	.CreateCustomScanState = GpuColumnarAgg_CreateCustomScanState,
};

static const CustomExecMethods GpuColumnarAggExecMethods = {
	.CustomName = "GpuColumnarAgg",
	.BeginCustomScan = GpuColumnarAgg_Begin,
	.ExecCustomScan = GpuColumnarAgg_Exec,
	.EndCustomScan = GpuColumnarAgg_End,
	.ReScanCustomScan = GpuColumnarAgg_ReScan,
	.ExplainCustomScan = GpuColumnarAgg_Explain,
};

static void
GpuColumnarAggUpperPaths(PlannerInfo *root, UpperRelationKind stage, RelOptInfo *input_rel, RelOptInfo *output_rel, void *extra)
{
	if (prev_create_upper_paths_hook)
		prev_create_upper_paths_hook(root, stage, input_rel, output_rel, extra);
	if (stage != UPPERREL_GROUP_AGG)
		return;
	GpuAggPlan *plan = palloc0(sizeof(GpuAggPlan));
	if (!translate_query(root, input_rel, plan))
		return;
	CustomPath *cpath = makeNode(CustomPath);
	cpath->path.pathtype = T_CustomScan;
	cpath->path.parent = output_rel;
	cpath->path.pathtarget = output_rel->reltarget;
	cpath->path.rows = output_rel->rows;
	/* one kernel pass at HBM speed: cheaper than any row-at-a-time plan over the same relation */
	cpath->path.startup_cost = 0;
	cpath->path.total_cost = input_rel->rows * 1e-6;
	cpath->methods = &GpuColumnarAggPathMethods;
	if (plan->desc.composite_key)
	{
		/* the composite key's domain is known only at execution time, where cg_partial_create may refuse it: the cheapest
		 * reference path becomes the node's child.  It is taken out of the pathlist because add_path frees the paths the
		 * GPU path displaces. */
		Path *ref = NULL;
		ListCell *lc;
		foreach(lc, output_rel->pathlist)
		{
			Path *p = (Path *) lfirst(lc);
			if (ref == NULL || p->total_cost < ref->total_cost)
				ref = p;
		}
		if (ref == NULL)
			return;
		output_rel->pathlist = list_delete_ptr(output_rel->pathlist, ref);
		cpath->custom_paths = list_make1(ref);
	}
	bytea *blob = palloc(VARHDRSZ + sizeof(GpuAggPlan));
	SET_VARSIZE(blob, VARHDRSZ + sizeof(GpuAggPlan));
	memcpy(VARDATA(blob), plan, sizeof(GpuAggPlan));
	cpath->custom_private = list_make1(makeConst(BYTEAOID, -1, InvalidOid, -1, PointerGetDatum(blob), false, false));
	add_path(output_rel, (Path *) cpath);
}

static Plan *
GpuColumnarAgg_PlanCustomPath(PlannerInfo *root, RelOptInfo *rel, CustomPath *best_path, List *tlist, List *clauses, List *custom_plans)
{
	CustomScan *cscan = makeNode(CustomScan);
	cscan->scan.plan.targetlist = tlist;
	cscan->scan.scanrelid = 0;                       /* not a scan of one base relation's tuples: it emits aggregate rows */
	cscan->custom_scan_tlist = tlist;
	cscan->custom_private = best_path->custom_private;
	cscan->custom_plans = custom_plans;                /* composite key: the reference plan (GpuColumnarAggUpperPaths) */
	cscan->methods = &GpuColumnarAggScanMethods;
	(void) root; (void) rel; (void) clauses;
	return (Plan *) cscan;
}

static Node *
GpuColumnarAgg_CreateCustomScanState(CustomScan *cscan)
{
	GpuColumnarAggState *state = (GpuColumnarAggState *) newNodeImpl(sizeof(GpuColumnarAggState), T_CustomScanState);
	state->css.methods = &GpuColumnarAggExecMethods;
	Const *blob = (Const *) linitial(cscan->custom_private);
	memcpy(&state->plan, VARDATA(DatumGetPointer(blob->constvalue)), sizeof(GpuAggPlan));
	return (Node *) state;
}

/* ------------------------------------------------------------------------------------ *
 *  execution
 * ------------------------------------------------------------------------------------ */
static int64
datum_to_i64(Datum d, Oid type)
{
	switch (type)
	{
		case INT8OID: case TIMESTAMPOID: case TIMESTAMPTZOID: return DatumGetInt64(d);
		case INT4OID: case DATEOID: return (int64) DatumGetInt32(d);
		case INT2OID: return (int64) DatumGetInt16(d);
		case BOOLOID: return (int64) DatumGetBool(d);
		case FLOAT8OID: { double x = DatumGetFloat8(d); int64 v; memcpy(&v, &x, sizeof v); return v; }
		case FLOAT4OID: { double x = (double) DatumGetFloat4(d); int64 v; memcpy(&v, &x, sizeof v); return v; }
		default: return 0;
	}
}

/*
 * The relation as the library wants it (CgRelation): the main fork's pages as one image + the stripes visible to the
 * snapshot + their skip lists.  CgSkipNode / CgStripe are field-for-field conversions of ColumnChunkSkipNode /
 * StripeMetadata (different order and widths: this function IS the mapping).
 */
static void
build_relation_image(Relation rel, Snapshot snapshot, CgRelation *out)
{
	TupleDesc tupdesc = RelationGetDescr(rel);
	int natts = tupdesc->natts;
	CgColumnDesc *cols = palloc0(sizeof(CgColumnDesc) * natts);
	for (int c = 0; c < natts; c++)
	{
		int attlen = 8, type_class = CG_TYPE_INT;
		Form_pg_attribute att = TupleDescAttr(tupdesc, c);
		if (att->attisdropped || !type_is_supported(att->atttypid, &attlen, &type_class))
			attlen = att->attlen > 0 && att->attlen <= 8 && att->attbyval ? att->attlen : 8;   /* never read: only planned columns are staged */
		cols[c].attlen = attlen;
		cols[c].type_class = type_class;
	}
	List *stripes = StripesForRelfilelocator(rel);           /* snapshot-aware catalog scan of columnar.stripe */
	int nstripes = 0, nnodes = 0;
	ListCell *lc;
	foreach(lc, stripes)
	{
		StripeMetadata *s = (StripeMetadata *) lfirst(lc);
		if (StripeWriteState(s) != STRIPE_WRITE_FLUSHED)     /* columnar_reader.c:721-728 */
			continue;
		nstripes++;
		nnodes += (int) (s->columnCount * s->chunkCount);
	}
	CgStripe *cs = palloc0(sizeof(CgStripe) * Max(nstripes, 1));
	CgSkipNode *cn = palloc0(sizeof(CgSkipNode) * Max(nnodes, 1));
	int si = 0, base = 0;
	foreach(lc, stripes)
	{
		StripeMetadata *s = (StripeMetadata *) lfirst(lc);
		if (StripeWriteState(s) != STRIPE_WRITE_FLUSHED)
			continue;
		StripeSkipList *skip = ReadStripeSkipList(rel, s->id, tupdesc, s->chunkCount, snapshot);
		CgStripe *d = &cs[si++];
		d->id = s->id; d->file_offset = s->fileOffset; d->data_length = s->dataLength; d->row_count = s->rowCount;
		d->first_row_number = s->firstRowNumber; d->column_count = s->columnCount; d->chunk_row_count = s->chunkGroupRowCount;
		d->chunk_count = s->chunkCount; d->skipnode_base = (uint32) base;
		for (uint32 c = 0; c < s->columnCount; c++)
			for (uint32 k = 0; k < s->chunkCount; k++)
			{
				const ColumnChunkSkipNode *n = &skip->chunkSkipNodeArray[c][k];
				CgSkipNode *o = &cn[base + c * s->chunkCount + k];
				Oid type = TupleDescAttr(tupdesc, c)->atttypid;
				int attlen, type_class;
				o->has_minmax = n->hasMinMax && type_is_supported(type, &attlen, &type_class);
				o->min_value = o->has_minmax ? datum_to_i64(n->minimumValue, type) : 0;
				o->max_value = o->has_minmax ? datum_to_i64(n->maximumValue, type) : 0;
				o->row_count = n->rowCount;
				o->value_offset = n->valueChunkOffset; o->value_length = n->valueLength;
				o->exists_offset = n->existsChunkOffset; o->exists_length = n->existsLength;
				o->decompressed_size = n->decompressedValueSize;
				o->compression_type = (int32) n->valueCompressionType;
				o->compression_level = n->valueCompressionLevel;
			}
		base += (int) (s->columnCount * s->chunkCount);
	}
	/* the pages, as they sit in shared_buffers: one share-locked copy per block */
	BlockNumber nblocks = RelationGetNumberOfBlocks(rel);
	uint8 *pages = palloc((Size) Max(nblocks, 1) * BLCKSZ);
	for (BlockNumber b = 0; b < nblocks; b++)
	{
		Buffer buf = ReadBufferExtended(rel, MAIN_FORKNUM, b, RBM_NORMAL, NULL);
		LockBuffer(buf, BUFFER_LOCK_SHARE);
		memcpy(pages + (Size) b * BLCKSZ, BufferGetPage(buf), BLCKSZ);
		UnlockReleaseBuffer(buf);
	}
	out->pages = pages; out->nblocks = nblocks;
	out->stripes = cs; out->nstripes = nstripes;
	out->nodes = cn; out->nnodes = nnodes;
	out->columns = cols; out->natts = natts;
}

static void
GpuColumnarAgg_Begin(CustomScanState *node, EState *estate, int eflags)
{
	/* everything on the GPU happens at the first Exec call: EXPLAIN without ANALYZE must not touch it.  The reference
	 * child of a composite-key node is initialised here like any subplan (EXPLAIN shows it under the node). */
	GpuColumnarAggState *state = (GpuColumnarAggState *) node;
	CustomScan *cscan = (CustomScan *) node->ss.ps.plan;
	if (cscan->custom_plans != NIL)
	{
		state->child = ExecInitNode((Plan *) linitial(cscan->custom_plans), estate, eflags);
		node->custom_ps = list_make1(state->child);
	}
}

static void
run_scan(GpuColumnarAggState *state)
{
	EState *estate = state->css.ss.ps.state;
	MemoryContext old = MemoryContextSwitchTo(estate->es_query_cxt);
	gpu_ensure_device();
	Relation rel = table_open(state->plan.relid, AccessShareLock);
	CgRelation image;
	build_relation_image(rel, estate->es_snapshot ? estate->es_snapshot : GetActiveSnapshot(), &image);
	CgScanDesc *desc = &state->plan.desc;
	int64 key_min = 0, key_max = -1, rows = 0;
	int64 bounds[CG_MAX_AGGS];
	gpu_check(cg_relation_bounds(&image, desc, &key_min, &key_max, bounds, &rows));
	for (int a = 0; a < desc->naggs; a++)
		desc->aggs[a].term_abs_bound = bounds[a];
	int rc = CG_OK;
	if (desc->composite_key)
	{
		/* per-column bounds over the chunk groups the scan keeps; a domain the library refuses (D > 2^63, or a column
		 * without min / max) runs the reference child instead, before anything is scanned */
		int64 lo[CG_MAX_GROUP_COLS], hi[CG_MAX_GROUP_COLS];
		rc = cg_relation_key_bounds(&image, desc, lo, hi);
		for (int g = 0; rc == CG_OK && g < desc->ngroup_cols; g++)
		{
			desc->key_col_min[g] = lo[g];
			desc->key_col_max[g] = hi[g];
		}
	}
	if (rc == CG_OK)
		rc = cg_partial_create(desc, image.columns, image.natts, key_min, key_max, Max(rows, 1), &state->partial);
	if (rc == CG_EUNSUPPORTED && state->child != NULL)
	{
		table_close(rel, AccessShareLock);
		state->use_child = true;
		state->done_scan = true;
		MemoryContextSwitchTo(old);
		return;
	}
	gpu_check(rc);
	rc = cg_scan_relation(&image, desc, state->partial, &state->stats);
	if (rc == CG_ERETRY_UNPACKED)
	{
		/* an optimistic packed accumulator overflowed: nothing wrong was produced; rescan with wide accumulators */
		gpu_check(cg_partial_set_packing(state->partial, 0));
		gpu_check(cg_partial_reset(state->partial));
		rc = cg_scan_relation(&image, desc, state->partial, &state->stats);
	}
	gpu_check(rc);
	int64 n = 0;
	gpu_check(cg_partial_ngroups(state->partial, &n));
	Size cells = (Size) Max(n, 1) * Max(desc->naggs, 1);
	state->keys = palloc(sizeof(int64) * Max(n, 1)); state->key_nulls = palloc(Max(n, 1));
	state->sum_hi = palloc(sizeof(int64) * cells); state->sum_lo = palloc(sizeof(uint64) * cells);
	state->count = palloc(sizeof(int64) * cells); state->minmax = palloc(sizeof(int64) * cells);
	state->fsum = palloc(sizeof(double) * cells);
	state->sumsq = palloc(sizeof(uint64) * 3 * cells);
	gpu_check(cg_partial_fetch_ex(state->partial, Max(n, 1), state->keys, state->key_nulls, state->sum_hi, state->sum_lo, state->count,
								  state->minmax, state->fsum, state->sumsq, &state->ngroups));
	if (desc->composite_key)
	{
		/* the key arrays hold composite codes: the key columns come from the library's decoder */
		Size kcells = (Size) Max(state->ngroups, 1) * desc->ngroup_cols;
		state->key_values = palloc(sizeof(int64) * kcells);
		state->key_value_nulls = palloc(kcells);
		gpu_check(cg_group_key_decode(desc, state->ngroups, state->keys, state->key_values, state->key_value_nulls));
	}
	table_close(rel, AccessShareLock);
	state->next = 0;
	state->done_scan = true;
	MemoryContextSwitchTo(old);
}

static Datum
i64_to_datum(int64 v, Oid type)
{
	switch (type)
	{
		case INT4OID: case DATEOID: return Int32GetDatum((int32) v);
		case INT2OID: return Int16GetDatum((int16) v);
		case BOOLOID: return BoolGetDatum(v != 0);
		case FLOAT8OID: { double x; memcpy(&x, &v, sizeof x); return Float8GetDatum(x); }
		default: return Int64GetDatum(v);
	}
}

static TupleTableSlot *
GpuColumnarAgg_Exec(CustomScanState *node)
{
	GpuColumnarAggState *state = (GpuColumnarAggState *) node;
	if (!state->done_scan)
		run_scan(state);
	if (state->use_child)
		return ExecProcNode(state->child);             /* the reference plan's rows have the node's target list */
	TupleTableSlot *slot = node->ss.ps.ps_ResultTupleSlot;
	ExecClearTuple(slot);
	if (state->next >= state->ngroups)
		return slot;                                   /* empty slot = end of scan */
	const int64 g = state->next++;
	const int na = state->plan.desc.naggs;
	for (int i = 0; i < state->plan.nout; i++)
	{
		const GpuOutColumn *out = &state->plan.out[i];
		const int64 cell = g * na + out->index;
		slot->tts_isnull[i] = false;
		switch ((GpuOutKind) out->kind)
		{
			case GPU_OUT_KEY:
			{
				if (state->plan.desc.composite_key)
				{
					const Size kc = (Size) g * state->plan.desc.ngroup_cols + out->index;
					slot->tts_isnull[i] = state->key_value_nulls[kc] != 0;
					slot->tts_values[i] = i64_to_datum(state->key_values[kc], out->type);
					break;
				}
				/* two group columns travel packed: low 32 bits the first, high 32 bits the second */
				int64 k = state->keys[g];
				if (state->plan.desc.ngroup_cols == 2)
					k = out->index == 0 ? (int64) (int32) (uint32) k : (int64) (int32) ((uint64) k >> 32);
				slot->tts_isnull[i] = state->key_nulls[g] != 0;
				slot->tts_values[i] = i64_to_datum(k, out->type);
				break;
			}
			case GPU_OUT_COUNT:
				slot->tts_values[i] = Int64GetDatum(state->count[cell]);
				break;
			case GPU_OUT_SUM_NUMERIC:
			{
				char buf[64];
				if (state->count[cell] == 0) { slot->tts_isnull[i] = true; break; }      /* sum over no non-NULL input is NULL */
				gpu_check(cg_numeric_out(state->sum_hi[cell], state->sum_lo[cell], out->scale, buf, sizeof buf));
				slot->tts_values[i] = DirectFunctionCall3(numeric_in, CStringGetDatum(buf), ObjectIdGetDatum(InvalidOid), Int32GetDatum(-1));
				break;
			}
			case GPU_OUT_SUM_INT8:
				if (state->count[cell] == 0) { slot->tts_isnull[i] = true; break; }
				slot->tts_values[i] = Int64GetDatum((int64) state->sum_lo[cell]);
				break;
			case GPU_OUT_SUM_FLOAT8:
				if (state->count[cell] == 0) { slot->tts_isnull[i] = true; break; }
				slot->tts_values[i] = Float8GetDatum(state->fsum[cell]);
				break;
			case GPU_OUT_MINMAX:
				if (state->count[cell] == 0) { slot->tts_isnull[i] = true; break; }
				slot->tts_values[i] = i64_to_datum(state->minmax[cell], out->type);
				break;
			case GPU_OUT_VARIANCE:
			{
				/* numeric_stddev_internal's text: up to 1000 fraction digits */
				char buf[1200];
				int32 isnull = 0;
				gpu_check(cg_numeric_var_out(out->final, state->count[cell], state->sum_hi[cell], state->sum_lo[cell], &state->sumsq[cell * 3],
											 out->scale, buf, sizeof buf, &isnull));
				if (isnull) { slot->tts_isnull[i] = true; break; }
				slot->tts_values[i] = DirectFunctionCall3(numeric_in, CStringGetDatum(buf), ObjectIdGetDatum(InvalidOid), Int32GetDatum(-1));
				break;
			}
		}
	}
	return ExecStoreVirtualTuple(slot);
}

static void
GpuColumnarAgg_End(CustomScanState *node)
{
	GpuColumnarAggState *state = (GpuColumnarAggState *) node;
	if (state->partial)
		cg_partial_free(state->partial);
	state->partial = NULL;
	if (state->child)
		ExecEndNode(state->child);
	state->child = NULL;
}

static void
GpuColumnarAgg_ReScan(CustomScanState *node)
{
	GpuColumnarAggState *state = (GpuColumnarAggState *) node;
	if (state->use_child)
		ExecReScan(state->child);
	state->next = 0;                                   /* the aggregate rows are still there */
}

/* the counters ColumnarScan's EXPLAIN ANALYZE prints (columnar_customscan.c:1966-1999), plus the device's */
static void
GpuColumnarAgg_Explain(CustomScanState *node, List *ancestors, ExplainState *es)
{
	GpuColumnarAggState *state = (GpuColumnarAggState *) node;
	(void) ancestors;
	if (!state->done_scan)
		return;
	if (state->use_child)
	{
		ExplainPropertyText("GPU Path", "refused the composite key domain: the reference plan ran", es);
		return;
	}
	ExplainPropertyInteger("Rows Removed by Filter", NULL, state->stats.rows_removed_by_filter, es);
	ExplainPropertyInteger("Columnar Chunk Groups Removed by Filter", NULL, state->stats.chunk_groups_filtered, es);
	ExplainPropertyInteger("GPU Bytes Scanned", "B", state->stats.bytes_scanned, es);
	ExplainPropertyFloat("GPU Kernel Time", "ms", state->stats.kernel_ms, 3, es);
}

void
_PG_init(void)
{
	RegisterCustomScanMethods(&GpuColumnarAggScanMethods);
	prev_create_upper_paths_hook = create_upper_paths_hook;
	create_upper_paths_hook = GpuColumnarAggUpperPaths;
}
