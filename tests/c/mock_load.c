/* The CPU stand-in engine of mock_chain.c with the background-load calls, TEST INFRASTRUCTURE ONLY
 * (tests/test_load_background_logic.py).  cmb200_load_open, each cmb200_load_step and cmb200_load_close
 * are logged ("load_open", "load_step", "load_close") in the call log of mock_chain.c.  A step blocks
 * until the driver calls mock_load_release(); then the load ends at the next step.  MOCK_LOAD_OPEN_FAIL=1
 * makes cmb200_load_open fail, so that the drop-in falls back to the blocking load.  Nothing of the
 * product links against this file. */
#include "mock_chain.c"

struct cmb200_loader { int steps; };

static pthread_mutex_t load_mu = PTHREAD_MUTEX_INITIALIZER;
static pthread_cond_t load_cv = PTHREAD_COND_INITIALIZER;
static int load_released;

void mock_load_release(void) {
	pthread_mutex_lock(&load_mu);
	load_released = 1;
	pthread_cond_broadcast(&load_cv);
	pthread_mutex_unlock(&load_mu);
}

/* a mark of the driver's in the call log */
void mock_log_mark(const char *what) { log_call(what); }

cmb200_loader *cmb200_load_open(cmb200_engine *const *engines, int g, const char *base_path) {
	(void)engines; (void)g; (void)base_path;
	if (env_num("MOCK_LOAD_OPEN_FAIL", 0)) {
		snprintf(err_buf, sizeof(err_buf), "mock: no background load");
		return NULL;
	}
	log_call("load_open");
	return calloc(1, sizeof(struct cmb200_loader));
}

uint64_t cmb200_load_total(const cmb200_loader *l) { (void)l; return 100; }

int cmb200_load_step(cmb200_loader *l, size_t max_records, uint64_t *loaded_out) {
	(void)max_records;
	if (l->steps++ == 0) log_call("load_step");
	pthread_mutex_lock(&load_mu);
	while (!load_released)
		pthread_cond_wait(&load_cv, &load_mu);
	pthread_mutex_unlock(&load_mu);
	if (loaded_out) *loaded_out = 100;
	return 0;
}

int cmb200_load_close(cmb200_loader *l, uint64_t *records_out, uint32_t *deltas_out) {
	log_call("load_close");
	free(l);
	if (records_out) *records_out = 100;
	if (deltas_out) *deltas_out = 0;
	return 0;
}
