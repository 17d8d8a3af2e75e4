/* The CPU stand-in engine (mock_engine.c) with snapshot-chain calls, TEST INFRASTRUCTURE ONLY
 * (tests/test_chain_policy_logic.py).  Every snapshot call is logged in order ("save_set", "load_set",
 * "load_chain", "base", "d<k>", "refused" for a delta the engines hold no chain state for), and writes
 * a file of MOCK_BASE_BYTES (a base; the chain id in its first 8 bytes, 0 for cmb200_save_set) or
 * MOCK_DELTA_BYTES (a delta) through <path>.tmp and a rename, so that a driver can see which file each
 * tick of the drop-in's CMB200_CHECKPOINT_DELTAS policy writes and which files the directory keeps.
 * cmb200_load_chain counts the deltas .d1, .d2, ... that exist and leaves chain state when
 * MOCK_LOAD_WHOLE=1.  Nothing of the product links against this file. */
#include "mock_engine.c"

#include <stdio.h>

struct cmb200_snapshot { char path[2300], tmp[2310]; uint64_t id; int k; };

static pthread_mutex_t chain_mu = PTHREAD_MUTEX_INITIALIZER;
static char call_log[16384];
static uint64_t chain_id, next_id = 1;          /* the engines' chain state: 0 = none */
static int chain_k;

static void log_call(const char *what) {
	pthread_mutex_lock(&chain_mu);
	if (strlen(call_log) + strlen(what) + 2 < sizeof(call_log)) {
		strcat(call_log, what);
		strcat(call_log, " ");
	}
	pthread_mutex_unlock(&chain_mu);
}

static long env_num(const char *name, long dflt) {
	const char *v = getenv(name);
	return v && *v ? strtol(v, NULL, 0) : dflt;
}

static int write_file(const char *path, long bytes, uint64_t id) {
	FILE *f = fopen(path, "wb");
	if (!f) return -1;
	int ok = fwrite(&id, 8, 1, f) == 1;
	for (long i = 8; ok && i < bytes; i++) ok = fputc(0, f) != EOF;
	return fclose(f) == 0 && ok ? 0 : -1;
}

static uint64_t base_id(const char *path) {
	uint64_t id = 0;
	FILE *f = fopen(path, "rb");
	if (f) {
		if (fread(&id, 8, 1, f) != 1) id = 0;
		fclose(f);
	}
	return id;
}

int cmb200_save_set(cmb200_engine *const *engines, int g, const char *path, uint64_t *records_out) {
	(void)engines; (void)g;
	log_call("save_set");
	if (records_out) *records_out = 0;
	return write_file(path, env_num("MOCK_BASE_BYTES", 4096), 0);
}

int cmb200_load_set(cmb200_engine *const *engines, int g, const char *path, uint64_t *records_out) {
	(void)engines; (void)g; (void)path;
	log_call("load_set");
	if (records_out) *records_out = 0;
	return 0;
}

cmb200_snapshot *cmb200_chain_begin(cmb200_engine *const *engines, int g, const char *base_path, int delta) {
	(void)engines; (void)g;
	cmb200_snapshot *s = calloc(1, sizeof(*s));
	char what[32];
	pthread_mutex_lock(&chain_mu);
	const uint64_t have = chain_id;
	const int k = chain_k + 1;
	if (!delta) s->id = next_id++;
	pthread_mutex_unlock(&chain_mu);
	if (delta) {
		if (!have || base_id(base_path) != have) {
			log_call("refused");
			snprintf(err_buf, sizeof(err_buf), "mock: no chain state for this base");
			free(s);
			return NULL;
		}
		s->id = have; s->k = k;
		snprintf(s->path, sizeof(s->path), "%s.d%d", base_path, k);
		snprintf(what, sizeof(what), "d%d", k);
	} else {
		snprintf(s->path, sizeof(s->path), "%s", base_path);
		snprintf(what, sizeof(what), "base");
	}
	log_call(what);
	snprintf(s->tmp, sizeof(s->tmp), "%s.tmp", s->path);
	if (write_file(s->tmp, delta ? env_num("MOCK_DELTA_BYTES", 512) : env_num("MOCK_BASE_BYTES", 4096), delta ? 0 : s->id)) {
		free(s);
		return NULL;
	}
	return s;
}

int cmb200_snapshot_finish(cmb200_snapshot *s, uint64_t *records_out) {
	if (records_out) *records_out = 0;
	const int rc = rename(s->tmp, s->path) == 0 ? 0 : -1;
	if (rc == 0) {
		pthread_mutex_lock(&chain_mu);
		chain_id = s->id; chain_k = s->k;
		pthread_mutex_unlock(&chain_mu);
	}
	free(s);
	return rc;
}

int cmb200_load_chain(cmb200_engine *const *engines, int g, const char *base_path, uint64_t *records_out,
    uint32_t *deltas_out) {
	(void)engines; (void)g;
	log_call("load_chain");
	char p[2300];
	uint32_t k = 0;
	for (;; k++) {
		snprintf(p, sizeof(p), "%s.d%u", base_path, k + 1);
		if (access(p, R_OK) != 0) break;
	}
	pthread_mutex_lock(&chain_mu);
	chain_id = env_num("MOCK_LOAD_WHOLE", 0) ? base_id(base_path) : 0;
	chain_k = (int)k;
	pthread_mutex_unlock(&chain_mu);
	if (records_out) *records_out = 0;
	if (deltas_out) *deltas_out = k;
	return 0;
}

/* the calls logged so far, space-separated */
void mock_chain_log(char *out, size_t cap) {
	pthread_mutex_lock(&chain_mu);
	snprintf(out, cap, "%s", call_log);
	pthread_mutex_unlock(&chain_mu);
}
