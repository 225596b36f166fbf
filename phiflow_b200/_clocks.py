"""nvidia-smi clock / throttle sampling during timed regions."""
import subprocess
import threading
import time


class ClockSampler(threading.Thread):
    """Samples nvidia-smi clocks / throttle reasons during the timed region, with the card's name and power limit."""
    QUERY = 'clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,' \
            'clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap,power.limit,name'

    def __init__(self, index=0):
        super().__init__(daemon=True)
        self.index, self.samples, self.stop_flag = index, [], False

    def run(self):
        while not self.stop_flag:
            try:
                out = subprocess.check_output(['nvidia-smi', f'--query-gpu={self.QUERY}', '--format=csv,noheader,nounits',
                                               '-i', str(self.index)], timeout=5).decode().strip()
                self.samples.append([v.strip() for v in out.split(',')])
            except Exception:
                pass
            time.sleep(0.2)

    def summary(self):
        self.stop_flag = True
        if not self.samples:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"], "gpu": None, "power_limit_w": None}
        sm = sorted(float(s[0]) for s in self.samples)
        names = ['hw_slowdown', 'hw_thermal_slowdown', 'sw_thermal_slowdown', 'sw_power_cap']
        reasons = [n for i, n in enumerate(names) if any(s[2 + i] == 'Active' for s in self.samples)]
        return {"sm_mhz": sm[len(sm) // 2], "sm_max_mhz": float(self.samples[0][1]), "reasons": reasons, "samples": len(sm),
                "gpu": self.samples[0][7], "power_limit_w": self.samples[0][6]}
