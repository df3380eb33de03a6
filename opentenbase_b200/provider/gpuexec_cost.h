/*
 * gpuexec_cost.h — what the GPU path costs, in the planner's own units.
 *
 * Pure C without backend headers: gpuexec_provider.c includes it, tests/test_provider_cost_cpu.py compiles it alone.
 *
 * The reference prices a sequential scan as  seq_page_cost * pages + (cpu_tuple_cost + qual cost) * tuples
 * (cost_seqscan, src/backend/optimizer/path/costsize.c:327-394, all quantities per datanode through PAGES_PER_DN /
 * TUPLES_PER_DN, optimizer/paths.h:62-67), a hash join as the sum of its inputs plus hashing and matching per tuple
 * (final_cost_hashjoin, :3788) and a hashed aggregate as its input plus cpu_operator_cost per aggregate and grouping
 * column per tuple plus cpu_tuple_cost per group (cost_agg, :2451).  The unit is "one sequential page fetch".
 *
 * The GPU path reads the same pages through shared_buffers — the disk term is the reference's, unchanged — but pays
 * per PAGE, not per tuple, on the host (heapgetpage()'s visibility pass and one memcpy into the pinned ring), moves the
 * pages over PCIe while the host prepares the next batch (the slower of the two counts), runs a few passes over the
 * staged columns at HBM speed, and has a fixed price before the first row (context, plan compile, kernel launches,
 * result fetch) that keeps small queries on the CPU.  It is a blocking node: everything but the output rows is
 * start-up cost, as in cost_agg's AGG_HASHED case.
 *
 * Rates are GUCs of the provider (gpuexec.cost_unit_us, gpuexec.host_page_us, gpuexec.pcie_gb_s, gpuexec.hbm_gb_s,
 * gpuexec.startup_us) with defaults taken from bench.py on an H100 host.
 */
#ifndef GPUEXEC_COST_H
#define GPUEXEC_COST_H

typedef struct gpuexec_cost_params
{
	double		seq_page_cost;		/* the planner's GUCs (optimizer/cost.h:62-66); defaults 1.0 / 0.01 */
	double		cpu_tuple_cost;
	double		cost_unit_us;		/* microseconds one unit of cost stands for */
	double		host_page_us;		/* heapgetpage() + memcpy of one 8 KB page into the staging ring */
	double		pcie_gb_s;			/* host -> device copy rate of pinned memory */
	double		hbm_gb_s;			/* what the kernels sustain over the staged columns */
	double		startup_us;			/* fixed price of one GPU sub-plan */
} gpuexec_cost_params;

#define GPUEXEC_PAGE_BYTES		8192.0
#define GPUEXEC_DEVICE_PASSES	3.0		/* loader (deform), build / probe, aggregate: each touches the staged bytes about once */

static inline void
gpuexec_default_cost_params(gpuexec_cost_params *p)
{
	p->seq_page_cost = 1.0;
	p->cpu_tuple_cost = 0.01;
	p->cost_unit_us = 10.0;			/* 8 KB at ~0.8 GB/s: a sequential read that is not entirely cached */
	p->host_page_us = 1.5;			/* bench.py e2e_pages on two H100 hosts: one host thread feeds the ring at 5.6-6.9 GB/s */
	p->pcie_gb_s = 50.0;			/* bench.py e2e on two H100 hosts: 48.9-54.0 GB/s, same-run copy ceiling 50.5-55.3 GB/s */
	p->hbm_gb_s = 3000.0;			/* what the fused kernels sustain over the staged columns (H100: 3.35 TB/s HBM3) */
	p->startup_us = 1500.0;			/* context already created; plan compile + ~20 launches + result fetch */
}

/*
 * pages          heap pages the sub-plan reads on this datanode (all its base relations)
 * staged_bytes   bytes of the referenced columns once deformed, plus the join table
 * groups         rows the node returns
 */
static inline void
gpuexec_path_cost(const gpuexec_cost_params *p, double pages, double staged_bytes, double groups,
				  double *startup_cost, double *total_cost)
{
	double		unit = p->cost_unit_us > 0 ? p->cost_unit_us : 1.0;
	double		disk = p->seq_page_cost * pages;
	double		host_us = p->host_page_us * pages;
	double		pcie_us = pages * GPUEXEC_PAGE_BYTES / (p->pcie_gb_s * 1e3);	/* GB/s = 1e3 bytes per microsecond */
	double		device_us = GPUEXEC_DEVICE_PASSES * staged_bytes / (p->hbm_gb_s * 1e3);
	double		feed_us = host_us > pcie_us ? host_us : pcie_us;				/* the ring overlaps the two */
	double		run = disk + (feed_us + device_us + p->startup_us) / unit;

	if (groups < 1)
		groups = 1;
	*startup_cost = run;
	*total_cost = run + p->cpu_tuple_cost * groups;
}

/*
 * staged_bytes of a right semi / right anti join (gx_hash_agg_right): the hashed relation's referenced columns, read by
 * the build, by the compaction of the consumed rows and by the aggregate over them (three passes); its join table
 * (16-byte slots at load factor <= 2/3: 32 B per row) and match bitmap; and the probe side's key and qual columns once.
 */
static inline double
gpuexec_right_join_bytes(double build_rows, double build_row_bytes, double probe_rows, double probe_row_bytes)
{
	return build_rows * (3.0 * build_row_bytes + 32.0 + 0.125) + probe_rows * probe_row_bytes;
}

#endif							/* GPUEXEC_COST_H */
