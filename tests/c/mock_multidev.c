/* The CPU stand-in engine (mock_engine.c) as the engines of a sharded map (CMB200_DEVICES), TEST
 * INFRASTRUCTURE ONLY (tests/test_multidevice_logic.py).  It compiles mock_engine.c into this file with
 * engine creation and destruction renamed and wraps them: every engine remembers the device and the
 * capacity it was created with (mock_engine_config), a "machine" of MOCK_DEVICES devices refuses any
 * other ordinal, and the engines alive are counted (mock_engines_alive), so that a map that cannot
 * start all of its engines can be seen to keep none.  The snapshot set calls and the page moves of the
 * _dev calls fail as the stand-in's cmb200_save / cmb200_load and device-memory calls do: the stand-in
 * has neither files nor device memory.  Nothing of the product links against this file. */
#define cmb200_engine_create mock_base_engine_create
#define cmb200_engine_destroy mock_base_engine_destroy
#include "mock_engine.c"
#undef cmb200_engine_create
#undef cmb200_engine_destroy

#define MOCK_DEVICES 8
#define MOCK_ENGINES 256

static struct {
	pthread_mutex_t mu;
	cmb200_engine *eng[MOCK_ENGINES];
	int device[MOCK_ENGINES];
	uint64_t capacity[MOCK_ENGINES];
	int alive;
} md = { PTHREAD_MUTEX_INITIALIZER, { 0 }, { 0 }, { 0 }, 0 };

cmb200_engine *cmb200_engine_create(const cmb200_config *cfg) {
	if (cfg->device >= MOCK_DEVICES) {
		snprintf(err_buf, sizeof(err_buf), "mock: no device %d", cfg->device);
		return NULL;
	}
	cmb200_engine *e = mock_base_engine_create(cfg);
	pthread_mutex_lock(&md.mu);
	for (int i = 0; i < MOCK_ENGINES; i++)
		if (!md.eng[i]) { md.eng[i] = e; md.device[i] = cfg->device; md.capacity[i] = cfg->capacity; break; }
	md.alive++;
	pthread_mutex_unlock(&md.mu);
	return e;
}

void cmb200_engine_destroy(cmb200_engine *e) {
	if (!e) return;
	pthread_mutex_lock(&md.mu);
	for (int i = 0; i < MOCK_ENGINES; i++)
		if (md.eng[i] == e) md.eng[i] = NULL;
	md.alive--;
	pthread_mutex_unlock(&md.mu);
	mock_base_engine_destroy(e);
}

/* device and capacity engine e was created with; -1 if it is not alive */
int mock_engine_config(cmb200_engine *e, int *device, uint64_t *capacity) {
	int rc = -1;
	pthread_mutex_lock(&md.mu);
	for (int i = 0; i < MOCK_ENGINES; i++)
		if (md.eng[i] == e) { *device = md.device[i]; *capacity = md.capacity[i]; rc = 0; }
	pthread_mutex_unlock(&md.mu);
	return rc;
}

int mock_engines_alive(void) {
	pthread_mutex_lock(&md.mu);
	const int n = md.alive;
	pthread_mutex_unlock(&md.mu);
	return n;
}

int cmb200_save_set(cmb200_engine *const *engines, int g, const char *path, uint64_t *records_out) {
	(void)engines; (void)g; (void)path; if (records_out) *records_out = 0; return -1;
}
int cmb200_load_set(cmb200_engine *const *engines, int g, const char *path, uint64_t *records_out) {
	(void)engines; (void)g; (void)path; if (records_out) *records_out = 0; return -1;
}
int cmb200_move_pages(cmb200_engine *e, size_t n, void *dst, const uint32_t *dst_idx, const void *src, const uint32_t *src_idx) {
	(void)e; (void)n; (void)dst; (void)dst_idx; (void)src; (void)src_idx;
	snprintf(err_buf, sizeof(err_buf), "mock: no device memory"); return -1;
}
int cmb200_copy_peer(cmb200_engine *dst_e, void *dst, cmb200_engine *src_e, const void *src, size_t bytes) {
	(void)dst_e; (void)dst; (void)src_e; (void)src; (void)bytes;
	snprintf(err_buf, sizeof(err_buf), "mock: no device memory"); return -1;
}
